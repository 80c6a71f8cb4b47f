"""Flow colour coding on the GPU (csrc/flowviz.cu through fgt_b200/flowviz.py) against the numpy oracle, and the
pipeline's visualisation switches end to end on GpuBackend.

Bars (tests/test_flowviz.py check_images): within one level everywhere, identical on at least 99.99 % of the values,
identical on the cases whose angles are exact. The device's atan2f and the host's float32 arctan2 may differ by an ulp;
everything else is rounded as numpy rounds it."""
import os

import numpy as np
import pytest
import torch

from fgt_b200 import flowviz, lib, synth
from oracle import flowviz_oracle as FO
from tests.test_flowviz import CASES, check_images, golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F32 = np.float32


@pytest.mark.parametrize("name", list(CASES))
def test_golden_cases_against_oracle_and_reference(name):
    flows, rgb, bgr = golden()[name]
    exact = CASES[name][1]
    got = flowviz.flow_to_image(flows, device=DEV)
    check_images(got, FO.flow_images(flows), exact, f"{name} vs oracle")
    check_images(got, rgb, exact, f"{name} vs reference")
    got_bgr = flowviz.flow_to_image(torch.from_numpy(flows).to(DEV), convert_to_bgr=True)
    assert got_bgr.is_cuda and got_bgr.dtype == torch.uint8
    assert np.array_equal(got_bgr.cpu().numpy(), got[..., ::-1])
    check_images(got_bgr.cpu().numpy(), bgr, exact, f"{name} bgr vs reference")


def test_single_image_and_signed_zero_selects_wheel_ends():
    f = CASES["signed_zeros"][0]()[0]
    got = flowviz.flow_to_image(f, device=DEV)
    assert got.shape == (4, 4, 3) and np.array_equal(got, FO.flow_to_image(f))
    assert not np.array_equal(got[0, 1], got[0, 2])           # (1, +0) and (1, -0): entries 0 and 54


def test_1080p_batch():
    flows = synth.vis_flows(41, 3, 1080, 1920)
    check_images(flowviz.flow_to_image(flows, device=DEV), FO.flow_images(flows), False, "1080p")


def test_batched_equals_per_image_calls():
    flows = np.concatenate([synth.vis_flows(51, 5, 37, 53) * s for s in (F32(0.1), F32(40.0))], 0)
    flows[3] = 0.0
    batched = flowviz.flow_to_image(flows, device=DEV)
    single = np.stack([flowviz.flow_to_image(f, device=DEV) for f in flows])
    assert np.array_equal(batched, single)
    per = 8 * 37 * 53
    import fgt_b200.flowviz as FV
    old = FV.HOST_BUDGET
    try:
        FV.HOST_BUDGET = 3 * per                                 # host input in chunks of 3, 3, 3, 1
        assert np.array_equal(flowviz.flow_to_image(flows, device=DEV), batched)
    finally:
        FV.HOST_BUDGET = old


def test_sentinels_around_output_and_workspace_stay_untouched():
    B, H, W = 3, 45, 77                                          # H*W odd: no image starts on a 4-pixel boundary
    flows = torch.from_numpy(synth.vis_flows(61, B, H, W)).to(DEV)
    pad = 4096
    out = torch.full((pad + B * H * W * 3 + pad,), 0xA5, dtype=torch.uint8, device=DEV)
    ws_bytes = lib.call("fgt_flow_to_image_workspace", B, H, W)
    ws = torch.full((pad + ws_bytes + pad,), 0x5A, dtype=torch.uint8, device=DEV)
    mx = torch.full((B + 2,), -7.0, dtype=torch.float32, device=DEV)
    lib.call("fgt_flow_to_image", flows, B, H, W, 0, ws[pad:], ws_bytes, out[pad:], mx[1:], kernels=2)
    torch.cuda.synchronize()
    o, w, m = out.cpu().numpy(), ws.cpu().numpy(), mx.cpu().numpy()
    assert (o[:pad] == 0xA5).all() and (o[pad + B * H * W * 3:] == 0xA5).all()
    assert (w[:pad] == 0x5A).all() and (w[pad + ws_bytes:] == 0x5A).all()
    assert m[0] == -7.0 and m[-1] == -7.0
    f = flows.cpu().numpy()
    assert np.array_equal(m[1:-1], [np.sqrt(np.square(x[..., 0]) + np.square(x[..., 1])).max() for x in f])
    check_images(o[pad:pad + B * H * W * 3].reshape(B, H, W, 3), FO.flow_images(f), False, "sentinels")


def test_non_finite_raises_and_bad_arguments_are_refused():
    flows = synth.vis_flows(71, 4, 16, 24)
    for bad in (np.nan, np.inf, -np.inf):
        f = flows.copy()
        f[2, 5, 7, 1] = bad
        with pytest.raises(ValueError, match=r"\[2\].*NaN or Inf"):
            flowviz.flow_to_image(f, device=DEV)
    t = torch.zeros(1, 4, 4, 2, device=DEV)
    with pytest.raises(RuntimeError, match="workspace"):
        lib.call("fgt_flow_to_image", t, 1, 4, 4, 0, t, 0, t, None)
    with pytest.raises(RuntimeError, match="empty"):
        lib.call("fgt_flow_to_image_workspace", 0, 4, 4)
    with pytest.raises(RuntimeError, match="aligned"):
        ws = torch.empty(64, dtype=torch.uint8, device=DEV)
        lib.call("fgt_flow_to_image", t.data_ptr() + 4, 1, 1, 1, 0, ws, 64, ws, None)


def test_two_launches_per_call():
    flows = torch.from_numpy(synth.vis_flows(81, 6, 64, 96)).to(DEV)
    n0 = lib.COUNTERS["launches"]
    flowviz.flow_to_image(flows)
    assert lib.COUNTERS["launches"] - n0 == 2


def test_command_line_end_to_end_on_gpu_backend(tmp_path, monkeypatch):
    """All four switches on GpuBackend with synthetic weights: the driver's file tree, flow PNGs in the oracle's colours
    of the written .flo files, and frames/ and result.mp4 byte-identical to a run without the switches.
    The pipeline itself runs once and its result is replayed for the second command line: two runs of it on the GPU
    are not bit-identical (the fp64 reductions of the flow diffusion, the Poisson blend and RAFT's instance norm
    accumulate with atomics), and what is checked here is that the switches change nothing the writers produce. That
    the result does not depend on vis_out is checked on the deterministic CPU backend (tests/test_flowviz.py)."""
    from fgt_b200 import io as IO
    from fgt_b200 import pipeline as PL
    from tests.test_pipeline import _setup, _write_ckpts
    _, _, frames, masks, args, cfg, sds = _setup()
    tmp = str(tmp_path)
    _write_ckpts(tmp, cfg, sds)
    IO.write_frames(os.path.join(tmp, "in"), frames, mp4=False)
    IO.write_frames(os.path.join(tmp, "msk"), [np.repeat(m[..., None], 3, -1) for m in masks], mp4=False)
    real, seen = PL.video_inpainting, {}

    def once(*a, vis_out=None, **k):
        if not seen:
            seen["vis"] = {}
            seen["comp"] = real(*a, vis_out=seen["vis"], **k)
            seen["backend"] = a[2]
        if vis_out is not None:
            vis_out.update(seen["vis"])
        return seen["comp"]

    monkeypatch.setattr(PL, "video_inpainting", once)
    base = ["--path", os.path.join(tmp, "in", "frames"), "--path_mask", os.path.join(tmp, "msk", "frames"),
            "--raft_model", os.path.join(tmp, "raft.pth"), "--lafc_ckpts", os.path.join(tmp, "lafc"),
            "--fgt_ckpts", os.path.join(tmp, "fgt"), "--imgH", str(args.imgH), "--imgW", str(args.imgW),
            "--flow_mask_dilates", str(args.flow_mask_dilates), "--frame_dilates", str(args.frame_dilates)]
    PL.main(base + ["--outroot", os.path.join(tmp, "vis"), "--vis_flows", "--vis_completed_flows", "--vis_prop",
                    "--vis_frame"])
    PL.main(base + ["--outroot", os.path.join(tmp, "plain")])
    assert isinstance(seen["backend"], PL.GpuBackend)
    tree = lambda r: sorted(os.path.relpath(os.path.join(d, f), r) for d, _, fs in os.walk(r) for f in fs)
    plain, vis = os.path.join(tmp, "plain"), os.path.join(tmp, "vis")
    N = len(frames)
    extra = sorted(set(tree(vis)) - set(tree(plain)))
    want = []
    for sub in ("flow", "completed_flow"):
        for mode in ("forward", "backward"):
            want += [f"{sub}/{mode}_flo/{i:05d}.flo" for i in range(N - 1)]
            want += [f"{sub}/{mode}_png/{i:05d}.png" for i in range(N - 1)]
    for d, ext in (("prop_frames", "png"), ("masks_left", "png"), ("prop_frames_npy", "npy"), ("masks_left_npy", "npy")):
        want += [f"{d}/{i:05d}.{ext}" for i in range(N)]
    assert extra == sorted(want) and set(tree(plain)) <= set(tree(vis))
    for p in tree(plain):                                      # frames/*.png and result.mp4
        with open(os.path.join(plain, p), "rb") as a, open(os.path.join(vis, p), "rb") as b:
            assert a.read() == b.read(), p
    from PIL import Image
    for sub in ("flow", "completed_flow"):
        for mode in ("forward", "backward"):
            fl = np.stack([IO.read_flo(os.path.join(vis, sub, f"{mode}_flo", f"{i:05d}.flo")) for i in range(N - 1)])
            png = np.stack([np.array(Image.open(os.path.join(vis, sub, f"{mode}_png", f"{i:05d}.png")))
                            for i in range(N - 1)])
            check_images(png, FO.flow_images(fl), False, f"{sub}/{mode}")
