"""Flow warping error (fgt_b200/warp_error.py, oracle/warp_error_oracle.py) on the CPU: the oracle's warp and occlusion
test against the unmodified reference functions (tests/golden/warp_error.npz), the float64 composition against numpy,
the InputPadder pads, the host API's refusals and the C ABI declaration."""
import os

import numpy as np
import pytest
import torch

from fgt_b200 import lib
from fgt_b200 import warp_error as WE
from oracle import warp_error_oracle as WO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "warp_error.npz")
# Frame sizes whose InputPadder pads the golden records.
PAD_SIZES = [(8, 8), (7, 9), (37, 53), (240, 432), (256, 432), (480, 854), (1080, 1920), (2, 2), (63, 17)]
# Cases stored whole (inputs and outputs); LARGE stores outputs at SAMPLES seeded positions and regenerates its inputs.
LARGE = {"driver_240x430": (19, 2, 3, 240, 430)}
SAMPLES = 4096


def _image(rng, b, c, h, w):
    return (rng.integers(0, 256, (b, c, h, w)).astype(np.float32) / np.float32(255)).astype(np.float32)


def _smooth_flow(rng, b, h, w, scale):
    """Smooth random flows: coarse noise upsampled, as real flows vary slowly."""
    coarse = rng.standard_normal((b, 2, h // 16 + 2, w // 16 + 2)) * scale
    ys = np.linspace(0, coarse.shape[2] - 1.001, h)
    xs = np.linspace(0, coarse.shape[3] - 1.001, w)
    y0, x0 = ys.astype(int), xs.astype(int)
    fy, fx = (ys - y0)[:, None], (xs - x0)[None, :]
    c = coarse
    out = (c[:, :, y0][:, :, :, x0] * (1 - fy) * (1 - fx) + c[:, :, y0 + 1][:, :, :, x0] * fy * (1 - fx)
           + c[:, :, y0][:, :, :, x0 + 1] * (1 - fy) * fx + c[:, :, y0 + 1][:, :, :, x0 + 1] * fy * fx)
    return out.astype(np.float32)


def _random_case(seed, b, c, h, w, scale=3.0):
    rng = np.random.default_rng(seed)
    img = _image(rng, b, c, h, w)
    f = _smooth_flow(rng, b, h, w, scale) + (rng.standard_normal((b, 2, h, w)) * 0.05).astype(np.float32)
    bw = -f + (rng.standard_normal((b, 2, h, w)) * 0.35).astype(np.float32)
    return img, f.astype(np.float32), bw.astype(np.float32)


def _integer_case(seed, b, c, h, w):
    rng = np.random.default_rng(seed)
    img = _image(rng, b, c, h, w)
    f = rng.integers(-4, 5, (b, 2, h, w)).astype(np.float32)
    bw = rng.integers(-4, 5, (b, 2, h, w)).astype(np.float32)
    return img, f, bw


def _leaving_case(seed, b, c, h, w):
    rng = np.random.default_rng(seed)
    img = _image(rng, b, c, h, w)
    f = (rng.standard_normal((b, 2, h, w)) * np.array([w, h], np.float32).reshape(1, 2, 1, 1)).astype(np.float32)
    bw = -f + rng.standard_normal((b, 2, h, w)).astype(np.float32)
    return img, f, bw


def _threshold_case(seed, b, c, h, w):
    """Integer forward flow (a, 0) per row and B = (-a + d, 0): the sample lands on a pixel centre, so the test reads
    d^2 > 0.01 (a^2 + (d - a)^2) + 0.5. d is that equation's root moved by -8..8 float32 ulps."""
    rng = np.random.default_rng(seed)
    img = _image(rng, b, c, h, w)
    a = rng.integers(-3, 4, (b, h, 1)).astype(np.float64) * np.ones((1, 1, w))
    root = (-0.02 * a + np.sqrt((0.02 * a) ** 2 + 4 * 0.99 * (0.02 * a * a + 0.5))) / (2 * 0.99)
    d = root.astype(np.float32)
    for _ in range(8):
        step = rng.integers(-1, 2, d.shape)
        d = np.where(step > 0, np.nextafter(d, np.float32(np.inf)), np.where(step < 0, np.nextafter(d, np.float32(-np.inf)), d))
    f = np.stack([a, np.zeros_like(a)], 1).astype(np.float32)
    bw = np.stack([(-a + d).astype(np.float32), np.zeros_like(d)], 1).astype(np.float32)
    return img, f, bw


def _zero_case(seed, b, c, h, w):
    rng = np.random.default_rng(seed)
    img = np.repeat(_image(rng, 1, c, h, w), b, axis=0)
    z = np.zeros((b, 2, h, w), np.float32)
    return img, z, z.copy()


# name: (generator, seed, b, c, h, w); the generator returns (image [b,c,h,w] on 0..1, F [b,2,h,w], B [b,2,h,w]).
CASES = {
    "odd_7x9": (_random_case, 1, 2, 3, 7, 9),
    "odd_37x53": (_random_case, 2, 2, 1, 37, 53),
    "not8_30x46": (_random_case, 3, 1, 3, 30, 46),
    "tiny_2x2": (_random_case, 4, 2, 3, 2, 2),
    "integer_24x40": (_integer_case, 5, 2, 3, 24, 40),
    "leaving_20x31": (_leaving_case, 6, 2, 3, 20, 31),
    "threshold_33x47": (_threshold_case, 7, 2, 1, 33, 47),
    "zero_16x23": (_zero_case, 8, 2, 3, 16, 23),
}


def case_inputs(name):
    if name in LARGE:
        seed, b, c, h, w = LARGE[name]
        return _random_case(seed, b, c, h, w)
    gen, *args = CASES[name]
    return gen(*args)


def sample_positions(name, shape):
    """The seeded flat positions of a LARGE case's sampled outputs."""
    return np.random.default_rng(LARGE[name][0] + 1000).choice(int(np.prod(shape)), SAMPLES, replace=False)


def _golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_golden(name):
    g = _golden()
    img, f, b = (torch.from_numpy(g[f"{name}/{k}"]) for k in ("image", "flow_fw", "flow_bw"))
    assert np.array_equal(WO.image_warp(img, f).numpy(), g[f"{name}/warped"])
    assert np.array_equal(WO.fb_occlusion(f, b).numpy().astype(np.uint8), g[f"{name}/occ"])


def test_oracle_matches_reference_golden_sampled():
    g = _golden()
    for name in LARGE:
        img, f, b = (torch.from_numpy(x) for x in case_inputs(name))
        warped, occ = WO.image_warp(img, f).numpy(), WO.fb_occlusion(f, b).numpy().astype(np.uint8)
        assert np.array_equal(warped.reshape(-1)[sample_positions(name, warped.shape)], g[f"{name}/warped"])
        assert np.array_equal(occ.reshape(-1)[sample_positions(name, occ.shape)], g[f"{name}/occ"])


def test_golden_covers_the_threshold_and_the_frame_border():
    g = _golden()
    assert 0.2 < g["threshold_33x47/occ"].mean() < 0.8         # both sides of the threshold
    lf = g["leaving_20x31/flow_fw"]
    x = np.arange(31)[None, None, :] + lf[:, 0]
    assert ((x < 0) | (x > 30)).mean() > 0.3                     # many samples leave the frame
    assert np.array_equal(g["integer_24x40/flow_fw"], np.round(g["integer_24x40/flow_fw"]))


def test_linspace_matches_numpy():
    for n in (2, 3, 7, 9, 17, 53, 240, 432, 480, 854, 1080, 1920, 4096):
        assert np.array_equal(WO.linspace32(n), np.linspace(-1, 1, n).astype(np.float32)), n


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(0)
    a, b, c = (torch.from_numpy(rng.standard_normal(20000).astype(np.float32)) for _ in range(3))
    got = WO.fma32(a, b, c).numpy()
    from fractions import Fraction
    for i in range(0, 20000, 97):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        cands = [lo, np.nextafter(lo, np.float32(-np.inf)), np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.float32(v).view(np.int32)) & 1))
        assert got[i] == best, i


def test_input_pads_match_reference_padder():
    g = _golden()
    for (h, w), pads in zip(PAD_SIZES, g["pads"]):
        assert WE.input_pads(h, w) == pads.tolist(), (h, w)


def _numpy_sums(frames, warped, valid, masks):
    """The float64 composition, pixel loop by numpy rows: (sum M*err, sum M, sum M*hole*err, sum M*hole)."""
    it = frames.astype(np.float32) / np.float32(255)
    out = []
    for t in range(warped.shape[0]):
        err = ((it[t].astype(np.float64) - warped[t].transpose(1, 2, 0).astype(np.float64)) ** 2).sum(-1)
        mt = valid[t].astype(np.float64)
        hole = (masks[t] != 0) if masks is not None else np.zeros_like(mt, bool)
        out.append([(mt * err).sum(), mt.sum(), (mt * err)[hole].sum(), mt[hole].sum()])
    return np.array(out)


def test_composition_matches_numpy():
    rng = np.random.default_rng(3)
    N, H, W, C = 4, 19, 27, 3
    frames = rng.integers(0, 256, (N, H, W, C)).astype(np.uint8)
    f = (rng.standard_normal((N - 1, 2, H, W)) * 2).astype(np.float32)
    b = -f + (rng.standard_normal((N - 1, 2, H, W)) * 0.6).astype(np.float32)
    masks = (rng.random((N, H, W)) < 0.3).astype(np.uint8)
    warped, valid = WO.pair_maps(frames, f, b)
    assert 0 < valid.mean() < 1
    sums = WO.pair_sums(frames, warped, valid, masks)
    ref = _numpy_sums(frames, warped.numpy(), valid.numpy(), masks)
    np.testing.assert_allclose(sums, ref, rtol=1e-13, atol=0)
    r = WO.report(sums)
    np.testing.assert_allclose(r["per_pair_ewarp"], ref[:, 0] / ref[:, 1], rtol=1e-15)
    assert r["ewarp_pairs"] == N - 1 and r["ewarp_hole_pairs"] == N - 1


def test_empty_mask_is_nan_and_left_out_of_the_mean():
    sums = np.array([[2.0, 4.0, 1.0, 2.0], [5.0, 0.0, 0.0, 0.0], [3.0, 3.0, 0.0, 0.0]])
    for r in (WO.report(sums), WE.report(sums, True)):
        assert np.array_equal(r["per_pair_ewarp"][[0, 2]], [0.5, 1.0]) and np.isnan(r["per_pair_ewarp"][1])
        assert r["ewarp"] == 0.75 and r["ewarp_pairs"] == 2
        assert r["per_pair_ewarp_hole"][0] == 0.5 and np.isnan(r["per_pair_ewarp_hole"][1:]).all()
        assert r["ewarp_hole"] == 0.5 and r["ewarp_hole_pairs"] == 1
    r = WE.report(np.zeros((2, 4)), False)
    assert np.isnan(r["ewarp"]) and r["ewarp_pairs"] == 0 and "ewarp_hole" not in r


@pytest.mark.parametrize("C", [1, 3])
def test_static_clip_with_zero_flows_scores_zero(C):
    rng = np.random.default_rng(5)
    frames = np.repeat(rng.integers(0, 256, (1, 31, 45, C)).astype(np.uint8), 3, axis=0)
    z = np.zeros((2, 2, 31, 45), np.float32)
    r = WO.warp_error(frames, z, z)
    assert r["ewarp_pairs"] == 2 and 0 <= r["ewarp"] < 1e-10
    # the reference's own align_corners=False sample half-blends the border with zeros: far from 0
    img = torch.from_numpy(frames[1:].astype(np.float32) / np.float32(255)).permute(0, 3, 1, 2)
    off = torch.nn.functional.grid_sample(img, torch.from_numpy(np.stack(np.meshgrid(
        WO.linspace32(45), WO.linspace32(31)), -1)[None].repeat(2, 0)), align_corners=False)
    assert ((off - img) ** 2).sum(1).mean() > 1e-3


def test_host_api_refuses_bad_arguments():
    u8 = lambda *s: np.zeros(s, np.uint8)
    fl = lambda n, h, w: (np.zeros((n, 2, h, w), np.float32),) * 2
    with pytest.raises(ValueError, match="N >= 2"):
        WE.warp_error(u8(1, 8, 8, 3), flows=fl(0, 8, 8))
    with pytest.raises(ValueError, match="H >= 2"):
        WE.warp_error(u8(3, 1, 8, 3), flows=fl(2, 1, 8))
    with pytest.raises(ValueError, match="W >= 2"):
        WE.warp_error(u8(3, 8, 1, 3), flows=fl(2, 8, 1))
    with pytest.raises(ValueError, match="C = 1 or 3"):
        WE.warp_error(u8(3, 8, 8, 2), flows=fl(2, 8, 8))
    with pytest.raises(ValueError, match="C = 1 or 3"):
        WE.warp_error(u8(3, 8, 8, 4), flows=fl(2, 8, 8))
    with pytest.raises(ValueError, match=r"\[N,H,W,C\]"):
        WE.warp_error(u8(3, 8, 8), flows=fl(2, 8, 8))
    with pytest.raises(ValueError, match="masks"):
        WE.warp_error(u8(3, 8, 8, 3), masks=u8(3, 8, 9), flows=fl(2, 8, 8))
    with pytest.raises(ValueError, match="forward flows"):
        WE.warp_error(u8(3, 8, 8, 3), flows=(np.zeros((3, 2, 8, 8), np.float32), fl(2, 8, 8)[1]))
    with pytest.raises(ValueError, match="backward flows"):
        WE.warp_error(u8(3, 8, 8, 3), flows=(fl(2, 8, 8)[0], np.zeros((2, 2, 8, 7), np.float32)))
    with pytest.raises(ValueError, match="pair"):
        WE.warp_error(u8(3, 8, 8, 3), flows=fl(2, 8, 8)[:1])
    with pytest.raises(ValueError, match="RAFT"):
        WE.warp_error(u8(3, 8, 8, 3))
    with pytest.raises(TypeError, match="uint8 or float32"):
        WE.warp_error(np.zeros((3, 8, 8, 3), np.float64), flows=fl(2, 8, 8))


def test_cpu_device_is_refused_without_fallback():
    z = np.zeros((2, 2, 8, 8), np.float32)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        WE.warp_error(np.zeros((3, 8, 8, 3), np.uint8), flows=(z, z), device="cpu")


def test_header_declares_the_entries():
    p = lib.PROTOS["fgt_warp_error"]
    assert p.names == ["frames", "frame_dtype", "masks", "flow_f", "flow_b", "N", "H", "W", "C", "workspace",
                       "workspace_bytes", "out", "warped", "valid", "stream"]
    assert p.stream and p.restype is __import__("ctypes").c_int
    ws = lib.PROTOS["fgt_warp_error_workspace"]
    assert ws.names == ["N", "H", "W", "C"] and not ws.stream


def test_command_line_requires_result_and_model():
    with pytest.raises(SystemExit):
        WE._parser().parse_args(["--result", "x"])
    a = WE._parser().parse_args(["--result", "x", "--raft_model", "m.pth", "--small", "--mixed_precision", "--gpu", "1"])
    assert a.small and a.mixed_precision and a.gpu == 1 and a.mask is None
