"""Flow warping error on the device (fgt_b200/warp_error.py, csrc/warp_error.cu) against the unmodified reference's
outputs (tests/golden/warp_error.npz) and the oracle (oracle/warp_error_oracle.py) run on the CPU."""
import argparse

import numpy as np
import pytest
import torch

from fgt_b200 import lib, synth
from fgt_b200 import warp_error as WE
from oracle import warp_error_oracle as WO
from tests.test_warp_error import CASES, GOLDEN

pytestmark = pytest.mark.gpu

# The kernel repeats the oracle's float32 operations one for one (the three fused multiply-adds of the bilinear sum
# included), so warped values and occlusion decisions are expected to be identical. An occlusion decision may differ
# only where the oracle's |F + B(x+F)|^2 lies within THRESH_ULPS float32 ulps of its threshold, and on at most
# MAX_NEAR_FLIPS of those pixels per call.
THRESH_ULPS = 4
MAX_NEAR_FLIPS = 0
# Per-pair float64 sums: the kernel's tile order against numpy's pairwise sums of the same terms.
SUM_RTOL = 1e-12
WARPED_SENTINEL = -12345.0
VALID_SENTINEL = 0xA5


def _clip(seed, N, H, W, C, dtype, masks=True, scale=3.0):
    """A seeded clip [N,H,W,C] with smooth, mostly consistent flows (F, B) [N-1,2,H,W] and masks [N,H,W]."""
    rng = np.random.default_rng(seed)
    base = rng.random((N, H, W, C)) * 255
    frames = base.astype(np.float32) if dtype == "f32" else np.floor(base).astype(np.uint8)
    coarse = rng.standard_normal((N - 1, 2, H // 16 + 2, W // 16 + 2)) * scale
    f = torch.nn.functional.interpolate(torch.from_numpy(coarse), size=(H, W), mode="bilinear",
                                        align_corners=True).numpy().astype(np.float32)
    b = (-f + rng.standard_normal(f.shape) * 0.35).astype(np.float32)
    m = (rng.random((N, H, W)) < 0.3).astype(np.uint8) * rng.integers(1, 256, (N, H, W)).astype(np.uint8) if masks else None
    return frames, m, f, b


def _near_threshold(f, b):
    """Pixels whose occlusion test lies within THRESH_ULPS ulps of its threshold (the oracle's float32 values)."""
    f, b = torch.as_tensor(f), torch.as_tensor(b)
    bw = WO.image_warp(b, f)
    lhs = WO.length_sq(f + bw)[:, 0].numpy()
    thr = (WO.ALPHA1 * (WO.length_sq(f) + WO.length_sq(bw)) + WO.ALPHA2)[:, 0].numpy()
    return np.abs(lhs - thr) <= THRESH_ULPS * np.spacing(thr)


def _check_maps(res, frames, f, b, masks):
    warped, valid = WO.pair_maps(frames, f, b)
    ref_w = warped.permute(0, 2, 3, 1).numpy()
    assert np.array_equal(res["warped"], ref_w), f"{np.count_nonzero(res['warped'] != ref_w)} warped values differ"
    flips = res["valid"] != valid.numpy().astype(np.uint8)
    assert not np.any(flips & ~_near_threshold(f, b))
    assert np.count_nonzero(flips) <= MAX_NEAR_FLIPS
    # the sums on the kernel's own maps
    own = WO.pair_sums(frames, torch.from_numpy(res["warped"]).permute(0, 3, 1, 2), torch.from_numpy(res["valid"]),
                       masks)
    np.testing.assert_allclose(res["sums"], own, rtol=SUM_RTOL, atol=0)
    return own


@pytest.mark.parametrize("name", sorted(CASES))
def test_kernel_matches_reference_golden(name):
    g = np.load(GOLDEN)
    img, f, b = g[f"{name}/image"], g[f"{name}/flow_fw"], g[f"{name}/flow_bw"]
    # frame t+1 of the clip is the golden's image t; the images are k / 255, so the uint8 clip reproduces them
    u8 = np.rint(img.transpose(0, 2, 3, 1) * 255).astype(np.uint8)
    frames = np.concatenate([u8[:1], u8])
    res = WE.warp_error(frames, flows=(f, b), return_maps=True)
    assert np.array_equal(res["warped"], g[f"{name}/warped"].transpose(0, 2, 3, 1))
    assert np.array_equal(res["valid"], 1 - g[f"{name}/occ"][:, 0])


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("dtype", ["u8", "f32"])
@pytest.mark.parametrize("with_masks", [False, True])
@pytest.mark.parametrize("shape", [(2, 37, 53), (5, 97, 131), (3, 240, 432)])
def test_kernel_matches_oracle(shape, dtype, C, with_masks):
    N, H, W = shape
    frames, masks, f, b = _clip(N * 1000 + H + C, N, H, W, C, dtype, with_masks)
    res = WE.warp_error(torch.from_numpy(frames).cuda(), masks, flows=(torch.from_numpy(f).cuda(), b),
                        return_maps=True)
    own = _check_maps(res, frames, f, b, masks)
    r = WO.report(own, masks is not None)
    np.testing.assert_allclose(res["per_pair_ewarp"], r["per_pair_ewarp"], rtol=SUM_RTOL)
    assert res["ewarp"] == pytest.approx(r["ewarp"], rel=SUM_RTOL)
    assert ("ewarp_hole" in res) == with_masks


def test_chunked_long_clip_is_bit_identical_to_one_call(monkeypatch):
    N, H, W, C = 23, 64, 90, 3
    frames, masks, f, b = _clip(77, N, H, W, C, "u8")
    whole = WE.warp_error(frames, masks, flows=(f, b), return_maps=True)
    per_ws = lib.call("fgt_warp_error_workspace", 2, H, W, C)
    monkeypatch.setattr(WE, "WORKSPACE_BUDGET", 5 * (H * W * (C + 1 + 16 + 4 * C + 1) + per_ws))   # chunks of 5 pairs
    before = lib.COUNTERS["launches"]
    chunked = WE.warp_error(frames, masks, flows=(f, b), return_maps=True)
    assert lib.COUNTERS["launches"] - before == 2 * 5                                        # 22 pairs: 5 chunks
    for k in ("sums", "warped", "valid"):
        assert np.array_equal(whole[k], chunked[k]), k
    _check_maps(chunked, frames, f, b, masks)


def test_two_runs_are_bit_identical():
    frames, masks, f, b = _clip(5, 6, 480, 854, 3, "u8")
    dev = torch.device("cuda:0")
    args = (torch.from_numpy(frames).to(dev), torch.from_numpy(masks).to(dev))
    fl = (torch.from_numpy(f).to(dev), torch.from_numpy(b).to(dev))
    r1, r2 = WE.warp_error(*args, flows=fl), WE.warp_error(*args, flows=fl)
    assert np.array_equal(r1["sums"], r2["sums"])
    assert r1["ewarp_pairs"] == 5 and 0 < r1["ewarp"] < 1


@pytest.mark.parametrize("dtype", ["u8", "f32"])
def test_static_clip_with_zero_flows_scores_zero(dtype):
    frames, _, _, _ = _clip(9, 1, 121, 203, 3, dtype, masks=False)
    frames = np.repeat(frames, 4, axis=0)
    z = np.zeros((3, 2, 121, 203), np.float32)
    res = WE.warp_error(frames, np.ones((4, 121, 203), np.uint8), flows=(z, z))
    assert res["ewarp_pairs"] == 3 and res["ewarp_hole_pairs"] == 3
    assert 0 <= res["ewarp"] < 1e-10 and 0 <= res["ewarp_hole"] < 1e-10
    assert np.array_equal(res["sums"][:, 1], np.full(3, 121.0 * 203))


def test_outputs_are_fully_written_and_nothing_else():
    N, H, W, C = 4, 45, 70, 3
    frames, masks, f, b = _clip(13, N, H, W, C, "f32")
    dev = torch.device("cuda:0")
    v, m, ff, fb = (torch.from_numpy(x).to(dev) for x in (frames, masks, f, b))
    need = lib.call("fgt_warp_error_workspace", N, H, W, C)
    pad = 1024
    ws = torch.full((need + 2 * pad,), 0x5A, dtype=torch.uint8, device=dev)
    out = torch.full((N - 1, 4), float("nan"), dtype=torch.float64, device=dev)
    warped = torch.full(((N - 1) * H * W * C + 2 * pad,), WARPED_SENTINEL, dtype=torch.float32, device=dev)
    valid = torch.full(((N - 1) * H * W + 2 * pad,), VALID_SENTINEL, dtype=torch.uint8, device=dev)
    ws0, w0, v0 = ws.clone(), warped.clone(), valid.clone()
    p = lambda t: t.data_ptr() + pad * t.element_size()
    lib.call("fgt_warp_error", v, lib.METRIC_F32, m, ff, fb, N, H, W, C, p(ws), need, out, p(warped), p(valid),
             kernels=2)
    torch.cuda.synchronize()
    for t, t0, n in ((ws, ws0, need), (warped, w0, (N - 1) * H * W * C), (valid, v0, (N - 1) * H * W)):
        assert torch.equal(t[:pad], t0[:pad]) and torch.equal(t[pad + n:], t0[pad + n:])
    wv, vv = warped[pad:pad + (N - 1) * H * W * C], valid[pad:pad + (N - 1) * H * W]
    assert not torch.any(wv == WARPED_SENTINEL) and torch.all(vv <= 1)
    res = {"warped": wv.view(N - 1, H, W, C).cpu().numpy(), "valid": vv.view(N - 1, H, W).cpu().numpy(),
           "sums": out.cpu().numpy()}
    _check_maps(res, frames, f, b, masks)
    # without maps the sums are the same, bit for bit
    out2 = torch.zeros_like(out)
    lib.call("fgt_warp_error", v, lib.METRIC_F32, m, ff, fb, N, H, W, C, p(ws), need, out2, None, None, kernels=2)
    assert torch.equal(out, out2)


def test_c_abi_refuses_bad_arguments():
    dev = torch.device("cuda:0")
    v = torch.zeros(3, 20, 20, 3, dtype=torch.uint8, device=dev)
    fl = torch.zeros(2, 2, 20, 20, dtype=torch.float32, device=dev)
    need = lib.call("fgt_warp_error_workspace", 3, 20, 20, 3)
    ws = torch.zeros(need, dtype=torch.uint8, device=dev)
    out = torch.zeros(2, 4, dtype=torch.float64, device=dev)
    U8 = lib.METRIC_U8
    with pytest.raises(RuntimeError, match="workspace of"):
        lib.call("fgt_warp_error", v, U8, None, fl, fl, 3, 20, 20, 3, ws, need - 1, out, None, None)
    with pytest.raises(RuntimeError, match="dtype"):
        lib.call("fgt_warp_error", v, 7, None, fl, fl, 3, 20, 20, 3, ws, need, out, None, None)
    with pytest.raises(RuntimeError, match="at least 2"):
        lib.call("fgt_warp_error", v, U8, None, fl, fl, 1, 20, 20, 3, ws, need, out, None, None)
    with pytest.raises(RuntimeError, match="2x2"):
        lib.call("fgt_warp_error", v, U8, None, fl, fl, 3, 1, 20, 3, ws, need, out, None, None)
    with pytest.raises(RuntimeError, match="channels"):
        lib.call("fgt_warp_error", v, U8, None, fl, fl, 3, 20, 20, 2, ws, need, out, None, None)
    with pytest.raises(RuntimeError, match="null"):
        lib.call("fgt_warp_error", v, U8, None, fl, None, 3, 20, 20, 3, ws, need, out, None, None)


@pytest.mark.parametrize("small", [False, True])
def test_raft_flows_end_to_end_match_the_oracle(small):
    from fgt_b200 import raft_small
    from fgt_b200.raft_model import RAFT
    dev = torch.device("cuda:0")
    if small:
        raft = raft_small.SmallRAFT(argparse.Namespace(small=True, mixed_precision=False, alternate_corr=False))
        raft.load_state_dict(synth.raft_small_state_dict(seed=34))
    else:
        raft = RAFT(argparse.Namespace(small=False, mixed_precision=False, alternate_corr=False))
        raft.load_state_dict(synth.raft_state_dict(seed=33))
    raft = raft.to(dev).eval()
    N, H, W = 6, 60, 90                                       # padded to 64 x 96 for RAFT
    rng = np.random.default_rng(21)
    scene = np.floor(rng.random((H + 16, W + 16, 3)) * 255).astype(np.uint8)
    frames = np.stack([scene[k:k + H, 2 * k:2 * k + W] for k in range(N)])
    masks = np.zeros((N, H, W), np.uint8)
    masks[:, 20:40, 30:60] = 255
    res = WE.warp_error(frames, masks, raft=raft, iters=4, return_maps=True)
    ff, fb = WE.raft_flows(torch.from_numpy(frames).to(dev), raft, iters=4)
    assert tuple(ff.shape) == (N - 1, 2, H, W) and tuple(fb.shape) == (N - 1, 2, H, W)
    f, b = ff.cpu().numpy(), fb.cpu().numpy()
    own = _check_maps(res, frames, f, b, masks)
    ref = WO.warp_error(frames, f, b, masks)
    for k in ("per_pair_ewarp", "per_pair_ewarp_hole"):
        np.testing.assert_allclose(res[k], ref[k], rtol=SUM_RTOL)
    assert res["ewarp_pairs"] == WO.report(own)["ewarp_pairs"]
