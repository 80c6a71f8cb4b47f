"""Launch-by-launch replay of flow propagation on the H100: every fgt_prop_step, fgt_prop_gather and fgt_prop_fuse launch
of real `get_flowNN_gradient` calls runs on the GPU and then, on CPU copies of the buffers it referenced as they were
before the launch, through the interpreter of tests/prop_emulator.py (the Replayer of tests/test_kernel_replay_gpu.py
with that interpreter). Both slots' state buffers start as 0xA5 bytes (have 0xA5 and nn_t negative both mean "no
neighbour"), so a store the interpreter does not make cannot hide behind a zero.

Bars, per launch (every byte the interpreter does not write must be unchanged, for all three):
- fgt_prop_step: nn_y, nn_x, nn_t, have and cuv bit-identical. Every operation is correctly rounded on both sides
  (the kernel's _rn intrinsics and IEEE double sqrt; numpy's fp32 / fp64 arithmetic), so there is nothing to allow.
- fgt_prop_gather: bit-identical (fp32 remap, the same operations in the same order).
- fgt_prop_fuse: tofill exact. Where the weights are exact (one candidate, or den == 0 and equal weights) the output is
  bit-identical. Elsewhere it must be fp32(v), v the interpreter's float64 value, except where fp32(v - e m) and
  fp32(v + e m) differ, e = 8 * 2^-53 and m = |g_b w0| + |g_f w1| (|v| without cancellation), where either neighbour
  is accepted: device double `exp` and numpy's may differ by an ulp, which is the only legitimate difference. With a
  subnormal confidence c that ulp is 2^-1074 absolute, so e grows by 2^-1072 / c there (tests/prop_emulator.fuse_ulps).

Cases: the three edge clips of tests/test_prop_kernels.py, the three golden clips, synth.prop_inputs(seed=7) at
240 x 432 with N = 10, and 720 x 1280 with N = 3, where the step launch's pixels outnumber its capped grid
(num_sms * 16 blocks of 256) and the grid-stride loop runs.

Observed on an H100 80GB HBM3 (700 W power limit), largest error in units of the bar over all launches: step 0 and
gather 0 (bit-identical everywhere); fuse 0: every fused value is fp32(v), also at the 32 elements inside the exemption (equal-weight
means that land exactly on an fp32 tie, and pairs of subnormal confidences). The file's 8 tests take 36 s.

Each of these changes to prop.cu fails a test here: np.round's half-to-even replaced by truncation (`(int)ny`), and
remap's 1/32-quantised fraction replaced by x - floor(x), and the case-2 fmax by fmin (the decisions clip and every
clip from the goldens up); `diff <= thres` (only the decisions clip: its 3-4-5 round trip); `iy < H` for the direct
neighbour (the decisions clip, prop_small, prop_mid, 240 x 432 and 720 x 1280); the fusion's den == 0 branch removed
(only the fusion clip at alpha 1e-3).
"""
import argparse
import collections
import time

import numpy as np
import pytest
import torch

from fgt_b200 import lib, propagation, synth
from tests.prop_emulator import PROP_ENTRIES, PropEmulator, fuse_ulps
from tests.test_kernel_replay_gpu import Replayer
from tests.test_prop_kernels import GOLDEN_CLIPS, edge_clips, golden_inputs

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


class PropReplayer(Replayer):
    """`exempt` counts the fused elements inside the exp exemption, and those of them that are not fp32(v)."""

    emulator = PropEmulator

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.exempt = collections.Counter()

    def _compare(self, name, cargs, emu, before, after, work):
        self._check_untouched(name, emu, before, after, work)
        key = {w.untyped_storage().data_ptr(): b for b, w in work.items()}
        for i, (kind, fl, idx, _, _) in enumerate(emu.records):
            b = key[fl.untyped_storage().data_ptr()]
            g = torch.empty(0, dtype=fl.dtype).set_(after[b].untyped_storage(), fl.storage_offset(), fl.shape, (1,))
            got, want = g[idx], fl[idx]
            if name == "fgt_prop_fuse" and kind == "f32":   # records: tofill, gx, gy
                f, k = emu.fuse, ("gx", "gy")[i - 1]
                ulps, exempt = fuse_ulps(got.numpy(), f["v"][k], f["mag"][k], f["exact"], f["cmin"])
                err = float(ulps.max()) if ulps.size else 0.0
                self.exempt["elements"] += int(exempt.sum())
                self.exempt["off fp32(v)"] += int((exempt & (ulps > 0)).sum())
                self.maxima[(name, kind)] = max(self.maxima[(name, kind)], err)
                assert err <= 1.0, f"{name}: {int(np.isinf(ulps).sum())} values outside the bar, max {err} ulp"
                continue
            same = (got.view(torch.uint8).view(-1, got.element_size()) ==
                    want.view(torch.uint8).view(-1, want.element_size())).all(1)
            bad = int((~same).sum())
            self.maxima[(name, kind)] = max(self.maxima[(name, kind)], float(bad))
            assert bad == 0, f"{name} ({kind}): {bad} of {len(idx)} stored values differ from the interpreter"


def _sentinel_state(N, H, W, dev):
    s = _plain_state(N, H, W, dev)
    for v in s.values():
        v.view(torch.uint8).fill_(0xA5)
    return s


_plain_state = propagation.slot_state


def _replay(inputs, thres, alpha, what, monkeypatch):
    gx, gy, mask, ff, fb = inputs
    N = mask.shape[2]
    monkeypatch.setattr(propagation, "slot_state", _sentinel_state)
    args = argparse.Namespace(Nonlocal=False, consistencyThres=thres, alpha=alpha)
    saved = lib.load()
    rep = PropReplayer(saved, PROP_ENTRIES, device_type=DEV.type)
    lib._lib = rep
    try:
        with np.errstate(invalid="ignore", over="ignore"):
            propagation.get_flowNN_gradient(args, gx.copy(), gy.copy(), mask, mask, ff, fb, None, None)
    finally:
        lib._lib = saved
        rep._st.clear()
    rep.report(what)
    print(f"[{what}] fuse: exempt elements {dict(rep.exempt)}")
    assert rep.launches == {"fgt_prop_step": 2 * (N - 1), "fgt_prop_gather": 2 * N, "fgt_prop_fuse": 1}
    return rep


@pytest.mark.parametrize("case", range(3))
def test_replay_edge_clips(case, monkeypatch):
    name, inputs, thres, alpha = edge_clips()[case]
    _replay(inputs, thres, alpha, name, monkeypatch)


@pytest.mark.parametrize("name", GOLDEN_CLIPS)
def test_replay_golden_clips(name, monkeypatch):
    inputs, thres, alpha = golden_inputs(name)
    _replay(inputs, thres, alpha, name, monkeypatch)


def test_replay_240x432_n10(monkeypatch):
    _replay(synth.prop_inputs(seed=7, H=240, W=432, N=10), 5.0, 0.1, "240x432 N=10", monkeypatch)


def test_replay_720x1280_grid_stride(monkeypatch):
    H, W = 720, 1280
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    assert H * W > sms * 16 * 256, "the step grid covers every pixel in one stride"
    t0 = time.time()
    _replay(synth.prop_inputs(seed=8, H=H, W=W, N=3), 5.0, 0.1, "720x1280 N=3", monkeypatch)
    print(f"[720x1280 N=3] replay {time.time() - t0:.1f} s")
