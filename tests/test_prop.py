"""Flow-guided gradient propagation (SURVEY §8 row a9): numpy oracle vs reference goldens and vs
cv2.remap (CPU); CUDA path vs oracle + goldens (GPU). Bars against the goldens: mask_tofill identical,
gradients within 1e-5 absolute (SURVEY §8d). Against the oracle, through the interpreter of
tests/prop_emulator.py (bit-identical to the oracle, tests/test_prop_kernels.py): mask_tofill identical,
every gradient the fusion does not write bit-identical, the fused ones fp32 of the float64 fusion except
within an ulp where device and numpy `exp` may round apart (tests/prop_emulator.fuse_ulps)."""
import argparse

import numpy as np
import pytest

from fgt_b200 import synth
from oracle import prop_oracle as PO
from tests.prop_emulator import emulate, fuse_ulps
from tests.util import load_golden

CASES = ["prop_small", "prop_thres1", "prop_mid"]


def _inputs(meta):
    return synth.prop_inputs(seed=meta["seed"], H=meta["H"], W=meta["W"], N=meta["N"])


def _check(meta, g, mask, ox, oy, om, tol):
    hole = np.repeat(mask[:, :, None, :], 3, axis=2)
    tofill = np.unpackbits(g["tofill"])[: mask.size].reshape(mask.shape).astype(bool)
    assert np.array_equal(om, tofill), "mask_tofill differs from the reference"
    assert np.abs(ox[hole] - g["gx_hole"]).max() <= tol
    assert np.abs(oy[hole] - g["gy_hole"]).max() <= tol


def _vs_oracle(inputs, thres, alpha, rx, ry, rm):
    """The whole-run bars against the oracle (see the module docstring)."""
    gx, gy, mask, ff, fb = inputs
    ex, ey, em, emu = emulate(gx, gy, mask, ff, fb, thres, alpha)
    ox, oy, om = PO.get_flownn_gradient(gx, gy, mask, ff, fb, thres, alpha)
    assert np.array_equal(em, om) and np.array_equal(ex, ox) and np.array_equal(ey, oy)
    assert np.array_equal(rm, om), "mask_tofill differs from the oracle"
    f = emu.fuse
    for k, got, want in (("gx", rx, ox), ("gy", ry, oy)):
        got = np.ascontiguousarray(got.transpose(3, 0, 1, 2)).reshape(-1)
        want = np.ascontiguousarray(want.transpose(3, 0, 1, 2)).reshape(-1)
        rest = np.ones(got.size, dtype=bool)
        rest[f["idx"]] = False
        assert np.array_equal(got[rest].view(np.uint32), want[rest].view(np.uint32)), "unfused gradients changed"
        ulps, _ = fuse_ulps(got[f["idx"]], f["v"][k], f["mag"][k], f["exact"], f["cmin"])
        assert ulps.size == 0 or ulps.max() <= 1.0, f"{k}: fused gradients outside the bar"


def test_remap_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    img = rng.standard_normal((40, 50, 3)).astype(np.float32)
    x = (rng.random((1, 4000)) * 60 - 5).astype(np.float32)
    y = (rng.random((1, 4000)) * 50 - 5).astype(np.float32)
    ref = cv2.remap(img, x, y, cv2.INTER_LINEAR)
    assert np.abs(ref[0] - PO.remap_q32(img, x[0], y[0])).max() <= 1e-6
    exact = PO.remap_q32(img, np.array([3.0, 7.5], np.float32), np.array([2.0, 4.25], np.float32))
    assert np.allclose(exact[0], img[2, 3]) and np.allclose(exact[1], 0.75 * 0.5 * (img[4, 7] + img[4, 8]) +
                                                            0.25 * 0.5 * (img[5, 7] + img[5, 8]), atol=1e-6)


@pytest.mark.parametrize("name", CASES)
def test_prop_oracle_vs_golden(name):
    g = load_golden(name)
    gx, gy, mask, ff, fb = _inputs(g["meta"])
    ox, oy, om = PO.get_flownn_gradient(gx, gy, mask, ff, fb, g["meta"]["thres"], 0.1)
    _check(g["meta"], g, mask, ox, oy, om, 1e-6)
    keep = ~np.repeat(mask[:, :, None, :], 3, axis=2)
    assert np.array_equal(ox[keep], gx[keep])  # pixels outside the holes are untouched


def test_prop_no_cpu_fallback_and_nonlocal_rejected():
    import torch
    from fgt_b200.propagation import get_flowNN_gradient
    gx, gy, mask, ff, fb = synth.prop_inputs(seed=0, H=32, W=32, N=3)
    with pytest.raises(ValueError):
        get_flowNN_gradient(argparse.Namespace(Nonlocal=True, consistencyThres=5, alpha=0.1), gx, gy, mask, mask, ff, fb)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):
            get_flowNN_gradient(argparse.Namespace(Nonlocal=False, consistencyThres=5, alpha=0.1), gx, gy, mask, mask,
                                ff, fb)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_prop_gpu(name):
    from fgt_b200.propagation import get_flowNN_gradient
    g = load_golden(name)
    gx, gy, mask, ff, fb = _inputs(g["meta"])
    args = argparse.Namespace(Nonlocal=False, consistencyThres=g["meta"]["thres"], alpha=0.1)
    gx_in, gy_in = gx.copy(), gy.copy()
    rx, ry, rm = get_flowNN_gradient(args, gx_in, gy_in, mask.copy(), mask.copy(), ff, fb, None, None)
    assert rx is gx_in and ry is gy_in  # fused in place like the reference
    assert rx.shape == gx.shape and rm.shape == mask.shape and rm.dtype == bool
    _check(g["meta"], g, mask, rx, ry, rm, 1e-5)
    _vs_oracle((gx, gy, mask, ff, fb), g["meta"]["thres"], 0.1, rx, ry, rm)


@pytest.mark.gpu
def test_prop_gpu_432x240_properties():
    """BASELINE-size clip: untouched outside holes, filled + tofill partition the hole set, idempotent."""
    from fgt_b200.propagation import get_flowNN_gradient
    gx, gy, mask, ff, fb = synth.prop_inputs(seed=7, H=240, W=432, N=10)
    args = argparse.Namespace(Nonlocal=False, consistencyThres=5.0, alpha=0.1)
    rx, ry, rm = get_flowNN_gradient(args, gx.copy(), gy.copy(), mask, mask, ff, fb)
    keep = ~np.repeat(mask[:, :, None, :], 3, axis=2)
    assert np.array_equal(rx[keep], gx[keep]) and np.array_equal(ry[keep], gy[keep])
    assert not (rm & ~mask).any()
    rx2, ry2, rm2 = get_flowNN_gradient(args, gx.copy(), gy.copy(), mask, mask, ff, fb)
    assert np.array_equal(rx, rx2) and np.array_equal(rm, rm2)
    _vs_oracle((gx, gy, mask, ff, fb), 5.0, 0.1, rx, ry, rm)
