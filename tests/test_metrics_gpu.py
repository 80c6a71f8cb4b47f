"""Quality metrics on the device (fgt_b200/metrics.py, csrc/metrics.cu) against the reference's outputs
(tests/golden/metrics.npz) and the float64 oracle (oracle/metrics_oracle.py)."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

from fgt_b200 import lib
from fgt_b200 import metrics as M
from fgt_b200 import pipeline as PL
from fgt_b200 import synth
from oracle import metrics_oracle as MO
from tests.test_metrics import CASES, GOLDEN, KEYS, ORACLE_GOLDEN_GAP, case_inputs, rel_err

pytestmark = pytest.mark.gpu

# The kernels filter separably and sum in another order than the oracle's direct 11x11 sum and numpy's pairwise means,
# so they differ from the oracle as the oracle differs from cv2: GPU_TOL is 100 times the measured CPU bound.
GPU_TOL = 100 * ORACLE_GOLDEN_GAP


def _oracle(res, gts):
    with ThreadPoolExecutor(max_workers=PL.HOST_THREADS) as pool:
        return MO.clip_metrics(res, gts, map_fn=pool.map)


def _check(got, ref, tol=GPU_TOL):
    for k in KEYS:
        assert rel_err(got["per_frame"][k], ref["per_frame"][k]) <= tol, k
    for k in KEYS[:4]:
        assert got[k] == pytest.approx(ref[k], rel=tol), k


@pytest.mark.parametrize("name", sorted(CASES))
def test_matches_reference_golden_and_oracle(name):
    res, gts = case_inputs(name)
    got = M.frame_metrics(res, gts)
    gd = np.load(GOLDEN)
    for k in KEYS:
        assert rel_err(got["per_frame"][k], gd[f"{name}/{k}"]) <= GPU_TOL, k
    _check(got, _oracle(res, gts))


@pytest.mark.parametrize("shape", [(80, 256, 432, 3), (3, 720, 1280, 3), (5, 11, 11, 3), (4, 33, 65, 1),
                                   (3, 77, 43, 3)])
@pytest.mark.parametrize("dtype", ["u8", "f32"])
def test_matches_oracle(shape, dtype):
    N, H, W, C = shape
    res, gts = synth.metric_pair(11 + H, N, H, W, C, "noise" if H % 2 == 0 else "blur", dtype)
    got = M.frame_metrics(torch.from_numpy(res).cuda(), torch.from_numpy(gts).cuda())
    _check(got, _oracle(res, gts))


def test_mixed_dtypes_match_oracle():
    res, gts = synth.metric_pair(21, 4, 64, 96, 3, "noise", "f32")
    res8 = np.floor(res + 0.5).astype(np.uint8)
    _check(M.frame_metrics(res8, gts), _oracle(res8, gts))
    _check(M.frame_metrics(gts, res8), _oracle(gts, res8))


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("dtype", ["u8", "f32"])
def test_identical_frames_are_exactly_100_and_1(C, dtype):
    _, gts = synth.metric_pair(31, 6, 70, 90, C, "same", dtype)
    got = M.frame_metrics(gts, gts.copy())
    assert np.all(got["per_frame"]["psnr"] == 100.0) and np.all(got["per_frame"]["ssim"] == 1.0)
    assert np.all(got["per_frame"]["ssim_channels"] == 1.0)
    assert np.all(got["per_frame"]["l1"] == 0.0) and np.all(got["per_frame"]["l2"] == 0.0)
    assert got["psnr"] == 100.0 and got["ssim"] == 1.0


def test_bit_identical_across_batch_sizes_and_chunkings(monkeypatch):
    res, gts = synth.metric_pair(41, 24, 96, 160, 3, "noise", "u8")
    whole = M.frame_metrics(res, gts)
    singles = [M.frame_metrics(res[i:i + 1], gts[i:i + 1]) for i in range(0, 24, 5)]
    for j, i in enumerate(range(0, 24, 5)):
        for k in KEYS:
            assert np.array_equal(whole["per_frame"][k][i], singles[j]["per_frame"][k][0]), k
    per = 96 * 160 * 3 * 2 + lib.call("fgt_metrics_workspace", 1, 96, 160, 3)
    monkeypatch.setattr(M, "WORKSPACE_BUDGET", 7 * per)                      # chunks of 7, 7, 7, 3 frames
    chunked = M.frame_metrics(res, gts)
    for k in KEYS:
        assert np.array_equal(whole["per_frame"][k], chunked["per_frame"][k]), k


def _kernel_nodes(fn):
    """Kernel nodes of the CUDA graph captured from fn(): what fn enqueues, read from the driver rather than from a
    profiler's activity records."""
    import ctypes
    cu = ctypes.CDLL("libcuda.so.1")
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        fn()
    graph = ctypes.c_void_p(g.raw_cuda_graph())
    n = ctypes.c_size_t(0)
    assert cu.cuGraphGetNodes(graph, None, ctypes.byref(n)) == 0
    nodes = (ctypes.c_void_p * n.value)()
    assert cu.cuGraphGetNodes(graph, nodes, ctypes.byref(n)) == 0
    kinds = []
    for node in nodes:
        t = ctypes.c_int(-1)
        assert cu.cuGraphNodeGetType(ctypes.c_void_p(node), ctypes.byref(t)) == 0
        kinds.append(t.value)
    del g
    return sum(1 for t in kinds if t == 0)                                   # CU_GRAPH_NODE_TYPE_KERNEL


@pytest.mark.parametrize("N", [1, 40])
def test_launch_count_does_not_depend_on_n(N):
    a, b = (torch.from_numpy(x).cuda() for x in synth.metric_pair(51, N, 128, 200, 3, "noise", "u8"))
    M.frame_metrics(a, b)                                                   # warm-up
    before = lib.COUNTERS["launches"]
    M.frame_metrics(a, b)
    assert lib.COUNTERS["launches"] - before == 2
    need = lib.call("fgt_metrics_workspace", N, 128, 200, 3)
    ws = torch.empty(need, dtype=torch.uint8, device=a.device)
    out = torch.empty(N, 4, dtype=torch.float64, device=a.device)
    sc = torch.empty(N, 3, dtype=torch.float64, device=a.device)
    U8 = lib.METRIC_U8
    assert _kernel_nodes(lambda: lib.call("fgt_metrics", a, U8, b, U8, N, 128, 200, 3, ws, need, out, sc, kernels=2)) == 2


@pytest.mark.parametrize("dtype", ["u8", "f32"])
def test_writes_nothing_outside_outputs_and_workspace(dtype):
    N, H, W, C = 5, 50, 70, 3
    res, gts = synth.metric_pair(61, N, H, W, C, "noise", dtype)
    dev = torch.device("cuda:0")
    pad = 4096
    code = lib.METRIC_U8 if dtype == "u8" else lib.METRIC_F32

    def guarded(x):
        t = torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1)).to(dev)
        buf = torch.full((t.numel() + 2 * pad,), 0xA5, dtype=torch.uint8, device=dev)
        buf[pad:pad + t.numel()] = t
        return buf

    need = lib.call("fgt_metrics_workspace", N, H, W, C)
    a, b = guarded(res), guarded(gts)
    ws = torch.full((need + 2 * pad,), 0x5A, dtype=torch.uint8, device=dev)
    out = torch.full((N * 4 * 8 + 2 * pad,), 0x3C, dtype=torch.uint8, device=dev)
    sc = torch.full((N * C * 8 + 2 * pad,), 0xC3, dtype=torch.uint8, device=dev)
    a0, b0, ws0, out0, sc0 = (t.clone() for t in (a, b, ws, out, sc))
    p = lambda t: t.data_ptr() + pad
    lib.call("fgt_metrics", p(a), code, p(b), code, N, H, W, C, p(ws), need, p(out), p(sc), kernels=2)
    torch.cuda.synchronize()
    assert torch.equal(a, a0) and torch.equal(b, b0)
    for t, t0, n in ((ws, ws0, need), (out, out0, N * 4 * 8), (sc, sc0, N * C * 8)):
        assert torch.equal(t[:pad], t0[:pad]) and torch.equal(t[pad + n:], t0[pad + n:])
    vals = out[pad:pad + N * 32].view(torch.float64).view(N, 4).cpu().numpy()
    ref = _oracle(res, gts)
    for j, k in enumerate(KEYS[:4]):
        assert rel_err(vals[:, j], ref["per_frame"][k]) <= GPU_TOL, k
    # without the per-channel output the frame values are the same, bit for bit
    out2 = torch.zeros(N, 4, dtype=torch.float64, device=dev)
    lib.call("fgt_metrics", p(a), code, p(b), code, N, H, W, C, p(ws), need, out2, None, kernels=2)
    assert np.array_equal(out2.cpu().numpy(), vals)


def test_c_abi_refuses_bad_arguments():
    dev = torch.device("cuda:0")
    a = torch.zeros(2, 20, 20, 3, dtype=torch.uint8, device=dev)
    need = lib.call("fgt_metrics_workspace", 2, 20, 20, 3)
    ws = torch.zeros(need, dtype=torch.uint8, device=dev)
    out = torch.zeros(2, 4, dtype=torch.float64, device=dev)
    U8 = lib.METRIC_U8
    with pytest.raises(RuntimeError, match="workspace of"):
        lib.call("fgt_metrics", a, U8, a, U8, 2, 20, 20, 3, ws, need - 1, out, None)
    with pytest.raises(RuntimeError, match="dtype"):
        lib.call("fgt_metrics", a, U8, a, 7, 2, 20, 20, 3, ws, need, out, None)
    with pytest.raises(RuntimeError, match="11x11"):
        lib.call("fgt_metrics", a, U8, a, U8, 2, 10, 20, 3, ws, need, out, None)
    with pytest.raises(RuntimeError, match="channels"):
        lib.call("fgt_metrics", a, U8, a, U8, 2, 20, 20, 2, ws, need, out, None)
    with pytest.raises(RuntimeError, match="null"):
        lib.call("fgt_metrics", a, U8, a, U8, 2, 20, 20, 3, ws, need, None, None)


def test_scores_a_pipeline_result_against_its_unmasked_frames():
    from tests.test_native_gpu import _backend
    frames, masks = synth.pipeline_clip(seed=5, N=7, H=64, W=96)
    args = PL.make_args(imgH=64, imgW=96, flow_mask_dilates=3, frame_dilates=1)
    out = np.stack(PL.video_inpainting(frames, masks, _backend(64, 96), args))
    gts = np.stack(frames)
    assert out.shape == gts.shape and out.dtype == np.uint8
    got = M.frame_metrics(out, gts)
    _check(got, _oracle(out, gts))
    assert np.all(got["per_frame"]["psnr"] < 100) and np.all(got["per_frame"]["ssim"] < 1)
