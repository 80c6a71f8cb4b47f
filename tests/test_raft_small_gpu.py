"""The small RAFT model (the reference's --small) on sm_90a: the native forward against the goldens of the unmodified
reference (tests/golden/raft_s_*.npz) and the CPU oracle at all four geometries, batching, warm start, non-test mode,
CUDA-graph replay, fgt_upflow8 against F.interpolate in float64, and a short pipeline run with load_models(small=True)."""
import argparse
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fgt_b200 import lib, synth
from oracle import raft_small_oracle as RSO
from tests.util import REL_TOL, assert_close, load_golden

pytestmark = pytest.mark.gpu


def _model(seed):
    from fgt_b200.raft_small import make_raft
    sd = synth.raft_small_state_dict(seed=seed)
    m = make_raft(argparse.Namespace(small=True, mixed_precision=False, alternate_corr=False))
    m.load_state_dict(sd)
    return m.cuda().eval(), sd


@pytest.mark.parametrize("name", ["raft_s_i6", "raft_s_i20", "raft_s_full_i20", "raft_s_720p_i20"])
def test_small_forward_vs_golden_and_oracle(name):
    g = load_golden(name)
    m = g["meta"]
    model, sd = _model(m["seed"])
    im1, im2 = synth.raft_inputs(seed=m["seed"] + 1, H=m["H"], W=m["W"])
    with torch.no_grad():
        lo, up = model(im1.cuda(), im2.cuda(), iters=m["iters"], test_mode=True)
    assert tuple(lo.shape) == (1, 2, m["H"] // 8, m["W"] // 8) and tuple(up.shape) == (1, 2, m["H"], m["W"])
    assert_close(lo, g["lo"], REL_TOL, name + " low vs reference golden")
    if "up" in g:
        assert_close(up, g["up"], REL_TOL, name + " up vs reference golden")
    else:
        assert_close(up.reshape(-1).cpu()[torch.from_numpy(g["up_idx"])], g["up_val"], REL_TOL, name + " up samples")
    with torch.no_grad():
        olo, oup = RSO.raft_small_forward(sd, im1, im2, iters=m["iters"])
    assert_close(lo, olo, REL_TOL, name + " low vs oracle")
    assert_close(up, oup, REL_TOL, name + " up vs oracle")


def test_batch3_flow_init_and_non_test_mode():
    """n=3 pairs in one call against the oracle and three single calls (instance-norm partial sums split differently:
    1e-4, not bit equality); a zero flow_init equals none; non-test mode returns one flow per iteration, the last
    equal to test mode's."""
    model, sd = _model(3)
    im1, im2 = synth.raft_inputs(seed=13, H=128, W=160, n=3)
    with torch.no_grad():
        lo, up = model(im1.cuda(), im2.cuda(), iters=5, test_mode=True)
        olo, oup = RSO.raft_small_forward(sd, im1, im2, iters=5)
    assert tuple(lo.shape) == (3, 2, 16, 20) and tuple(up.shape) == (3, 2, 128, 160)
    assert_close(lo, olo, REL_TOL, "batch low vs oracle")
    assert_close(up, oup, REL_TOL, "batch up vs oracle")
    with torch.no_grad():
        for i in range(3):
            lo1, up1 = model(im1[i:i + 1].cuda(), im2[i:i + 1].cuda(), iters=5, test_mode=True)
            assert_close(lo[i:i + 1], lo1, 1e-4, f"batch vs single pair {i}")
            assert_close(up[i:i + 1], up1, 1e-4, f"batch vs single pair {i} (up)")
        init = torch.randn(3, 2, 16, 20, generator=torch.Generator().manual_seed(2))
        wlo, wup = model(im1.cuda(), im2.cuda(), iters=3, flow_init=init.cuda(), test_mode=True)
        z0, zu = model(im1.cuda(), im2.cuda(), iters=3, flow_init=torch.zeros(3, 2, 16, 20).cuda(), test_mode=True)
        n0, nu = model(im1.cuda(), im2.cuda(), iters=3, test_mode=True)
        seq = model(im1.cuda(), im2.cuda(), iters=3, test_mode=False)
        olo_w, oup_w = RSO.raft_small_forward(sd, im1, im2, iters=3, flow_init=init)
    assert torch.equal(zu, nu) and torch.equal(z0, n0)
    assert_close(wup, oup_w, REL_TOL, "flow_init vs oracle")
    assert isinstance(seq, list) and len(seq) == 3 and torch.equal(seq[-1], nu)


def test_graph_replay_equals_eager():
    model, _ = _model(5)
    im1, im2 = synth.raft_inputs(seed=6, H=128, W=192, n=2)
    a, b = im1.cuda(), im2.cuda()
    with torch.no_grad():
        lo_e, up_e = model(a, b, iters=4, test_mode=True)
        seq_e = model(a, b, iters=2, test_mode=False)
        model.enable_cuda_graph(True)
        for _ in range(3):   # eager first call, capture, replay
            lo_g, up_g = model(a, b, iters=4, test_mode=True)
            seq_g = model(a, b, iters=2, test_mode=False)
        model.enable_cuda_graph(False)
    assert torch.equal(lo_g, lo_e) and torch.equal(up_g, up_e)
    assert len(seq_g) == 2 and all(torch.equal(x, y) for x, y in zip(seq_g, seq_e))


@pytest.mark.parametrize("n,h,w", [(2, 17, 23), (1, 60, 108), (3, 1, 9), (1, 6, 1), (2, 1, 1)])
def test_upflow8_vs_interpolate(n, h, w):
    flow = torch.randn(n, 2, h, w, generator=torch.Generator().manual_seed(h * 100 + w)) * 5
    out = torch.full((n, 2, 8 * h, 8 * w), float("nan"), device="cuda")
    lib.upflow8(flow.cuda(), h, w, out, n=n)
    torch.cuda.synchronize()
    ref = 8 * F.interpolate(flow.double(), size=(8 * h, 8 * w), mode="bilinear", align_corners=True)
    err = (out.cpu().double() - ref).abs().max().item()
    assert err <= 1e-5 * (1 + ref.abs().max().item()), err


def test_pipeline_with_small_model_matches_oracle_raft(tmp_path):
    """load_models(small=True) from checkpoints in the driver's layout; the flows of a short object-removal run match a
    run whose backend computes the flows with the oracle's small RAFT (every later stage on the GPU in both)."""
    from fgt_b200 import pipeline as PL
    from tests.test_pipeline import _setup, _write_ckpts
    g, st, frames, masks, args, cfg, sds = _setup()
    sds = dict(sds, raft=synth.raft_small_state_dict(seed=9))
    _write_ckpts(str(tmp_path), cfg, sds)
    dev = torch.device("cuda:0")
    backend, lafc_cfg = PL.load_models(os.path.join(str(tmp_path), "raft.pth"), os.path.join(str(tmp_path), "lafc"),
                                       os.path.join(str(tmp_path), "fgt"), dev, small=True)
    from fgt_b200.raft_small import SmallRAFT
    assert type(backend.raft) is SmallRAFT
    comp, stages = PL.video_inpainting(frames, masks, backend, args, lafc_cfg["num_flows"], lafc_cfg["flow_interval"],
                                       return_stages=True)
    assert len(comp) == len(frames) and comp[0].shape == frames[0].shape and comp[0].dtype == np.uint8

    def oracle_pairs(img1, img2, iters):
        with torch.no_grad():
            return torch.cat([RSO.raft_small_forward(sds["raft"], img1[i:i + 1], img2[i:i + 1], iters=iters)[1]
                              for i in range(img1.shape[0])], 0).numpy()

    backend.raft_pairs = oracle_pairs
    _, ostages = PL.video_inpainting(frames, masks, backend, args, lafc_cfg["num_flows"], lafc_cfg["flow_interval"],
                                     return_stages=True)
    for k in ("flow_f", "flow_b"):
        assert_close(stages[k], ostages[k], REL_TOL, k + " of the small model vs the oracle")
