"""The small RAFT model (the reference's --small) on the CPU: the oracle against goldens of the unmodified reference
(tests/golden/raft_s_*.npz), the module's state-dict contract and refusals, the constructor's choice of model, the whole
native forward through the float64 interpreters of its launches, and the --small switch of both command lines."""
import argparse

import pytest
import torch
import torch.nn.functional as F

from fgt_b200 import lib, synth
from oracle import raft_small_oracle as RSO
from tests.kernel_emulator import KernelEmulator, _KernelEntry, _raw
from tests.test_launch_trace import recording
from tests.util import assert_close, load_golden


def _args(**kw):
    return argparse.Namespace(**{**dict(small=True, mixed_precision=False, alternate_corr=False), **kw})


class _Stop(Exception):
    pass


@pytest.mark.parametrize("name", ["raft_s_i6", "raft_s_i20"])
def test_oracle_matches_reference_golden(name):
    g = load_golden(name)
    m = g["meta"]
    sd = synth.raft_small_state_dict(seed=m["seed"])
    im1, im2 = synth.raft_inputs(seed=m["seed"] + 1, H=m["H"], W=m["W"])
    with torch.no_grad():
        lo, up = RSO.raft_small_forward(sd, im1, im2, iters=m["iters"])
    assert_close(lo, g["lo"], 2e-5, name + " low-res flow")
    assert_close(up, g["up"], 2e-5, name + " upsampled flow")


def test_state_dict_contract_and_dataparallel_roundtrip():
    from fgt_b200.raft_small import SmallRAFT
    sd = synth.raft_small_state_dict(seed=3)
    dp = torch.nn.DataParallel(SmallRAFT(_args()))
    dp.load_state_dict({"module." + k: v for k, v in sd.items()})
    model = dp.module
    got = model.state_dict()
    assert set(got.keys()) == set(sd.keys()) and len(got) == 106
    for k, v in sd.items():
        assert torch.equal(got[k].cpu(), v), k
    assert (model.args.corr_levels, model.args.corr_radius) == (4, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        model(*synth.raft_inputs(seed=0, H=64, W=64), iters=1, test_mode=True)  # CPU tensors: no fallback


def test_constructor_chooses_the_model_and_refusals():
    from fgt_b200 import raft_model
    from fgt_b200.raft_small import SmallRAFT, make_raft
    assert type(make_raft(_args(small=False))) is raft_model.RAFT
    assert type(make_raft(_args())) is SmallRAFT
    with pytest.raises(ValueError, match="small"):
        raft_model.RAFT(_args())
    for build in (SmallRAFT, make_raft):
        with pytest.raises(ValueError, match="mixed_precision is not implemented for the small model"):
            build(_args(mixed_precision=True))
    m = SmallRAFT(_args())
    m.args.mixed_precision = True   # read on every forward, like the reference
    with pytest.raises(ValueError, match="not implemented"):
        m(*synth.raft_inputs(seed=0, H=64, W=64), iters=1, test_mode=True)


class _Upflow8Entry(_KernelEntry):
    def __call__(self, *args):
        a = {k: _raw(v, t) for k, v, t in zip(lib.PROTOS[self.name].names, args, self.argtypes)}
        self.emu.forms.add((self.name, ()))
        self.emu._upflow8(a)
        return 0


class SmallRaftEmulator(KernelEmulator):
    """The float64 interpreters of tests/kernel_emulator.py plus fgt_upflow8: 8 * bilinear x8 with align_corners=True,
    source index scale * dst with scale = (in - 1) / (out - 1) (0 for a 1-pixel side), as ATen's upsample_bilinear2d."""

    def __getattr__(self, name):
        if name == "fgt_upflow8":
            e = _Upflow8Entry(self, name)
            setattr(self, name, e)
            return e
        return super().__getattr__(name)

    def _upflow8(self, a):
        n, h, w = a["n"], a["h"], a["w"]
        f = self.f32(a["flow_nchw"], n * 2 * h * w).view(n, 2, h, w)

        def axis(size):
            dst = torch.arange(8 * size, dtype=torch.float64)
            src = dst * ((size - 1) / (8 * size - 1))
            i0 = src.long()
            return i0, (i0 + 1).clamp(max=size - 1), src - i0

        y0, y1, ly = axis(h)
        x0, x1, lx = axis(w)
        ly, lx = ly[:, None], lx[None, :]
        top = (1 - lx) * f[:, :, y0][:, :, :, x0] + lx * f[:, :, y0][:, :, :, x1]
        bot = (1 - lx) * f[:, :, y1][:, :, :, x0] + lx * f[:, :, y1][:, :, :, x1]
        up = 8.0 * ((1 - ly) * top + ly * bot)
        self.st32(a["out"], torch.arange(up.numel()), up)


def _emulated(fn):
    with torch.no_grad(), recording(SmallRaftEmulator()) as emu:
        out = fn()
    return out, emu


def test_upflow8_interpreter_matches_interpolate():
    for h, w in ((3, 5), (1, 4), (4, 1), (1, 1)):
        flow = torch.randn(2, 2, h, w, generator=torch.Generator().manual_seed(h * 10 + w))
        out = torch.full((2, 2, 8 * h, 8 * w), -1234.5)
        _emulated(lambda: lib.upflow8(flow, h, w, out, n=2))
        ref = 8 * F.interpolate(flow.double(), size=(8 * h, 8 * w), mode="bilinear", align_corners=True)
        assert (out.double() - ref).abs().max() <= 1e-6 * (1 + ref.abs().max()), (h, w)


def test_small_forward_in_float64():
    """The whole native forward (every GEMM, lookup, norm and upflow8 launch) interpreted in float64, against the
    reference's golden and the oracle."""
    from fgt_b200.raft_small import SmallRAFT
    g = load_golden("raft_s_i6")
    meta = g["meta"]
    sd = synth.raft_small_state_dict(seed=meta["seed"])
    m = SmallRAFT(_args())
    m.load_state_dict(sd)
    im1, im2 = synth.raft_inputs(seed=meta["seed"] + 1, H=meta["H"], W=meta["W"])
    (lo, up), emu = _emulated(lambda: m._forward_impl(im1, im2, meta["iters"], None, True))
    assert ("fgt_upflow8", ()) in emu.forms and ("fgt_corr_lookup", ("split", 4, 3)) in emu.forms
    assert_close(lo, g["lo"], 1e-4, "small RAFT low vs reference golden")
    assert_close(up, g["up"], 1e-4, "small RAFT up vs reference golden")
    with torch.no_grad():
        olo, oup = RSO.raft_small_forward(sd, im1, im2, iters=meta["iters"])
    assert_close(up, oup, 1e-4, "small RAFT up vs oracle")


# ------------------------------------------------------------------------------------------------ command lines
def test_pipeline_command_line_small(monkeypatch):
    from fgt_b200 import pipeline
    base = ["--path", "frames", "--path_mask", "masks", "--outroot", "out"]
    assert pipeline.arg_parser().parse_args(base).small is False
    seen = {}

    def fake_load(raft_model, lafc_ckpts, fgt_ckpts, device, mixed_precision=False, small=False):
        seen["small"] = small
        raise _Stop

    monkeypatch.setattr(pipeline, "load_models", fake_load)
    for argv, want in (([], False), (["--small"], True)):
        with pytest.raises(_Stop):
            pipeline.main(base + argv)
        assert seen.pop("small") is want


def _capture_constructor(monkeypatch):
    from fgt_b200 import raft_small
    seen = {}

    def fake(args):
        seen["args"] = args
        raise _Stop

    monkeypatch.setattr(raft_small, "make_raft", fake)
    return seen


def test_load_models_builds_the_small_model(monkeypatch):
    from fgt_b200 import pipeline
    seen = _capture_constructor(monkeypatch)
    for flag in (False, True):
        with pytest.raises(_Stop):
            pipeline.load_models("raft.pth", "lafc", "fgt", torch.device("cpu"), small=flag)
        assert seen.pop("args").small is flag
    with pytest.raises(_Stop):
        pipeline.load_models("raft.pth", "lafc", "fgt", torch.device("cpu"))
    assert seen.pop("args").small is False


def test_flow_extract_command_line_small(monkeypatch):
    from fgt_b200 import flow_extract
    seen = _capture_constructor(monkeypatch)
    for argv, want in (([], False), (["--small"], True)):
        with pytest.raises(_Stop):
            flow_extract.main(["--path", "videos", "--outroot", "flows"] + argv)
        assert seen.pop("args").small is want


def test_dropin_exports_the_constructor():
    import importlib
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "dropin"))
    try:
        sys.modules.pop("RAFT", None)
        R = importlib.import_module("RAFT")
        from fgt_b200.raft_small import make_raft
        assert R.RAFT is make_raft
    finally:
        sys.path.remove(os.path.join(root, "dropin"))
        sys.modules.pop("RAFT", None)
