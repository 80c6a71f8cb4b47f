"""GPU parity of the full FGT forward (fgt_b200.fgt_model.Model, every op an sm_90a kernel behind
the C-ABI) against (a) the CPU oracle on the same seeded inputs and (b) the committed golden
outputs of the unmodified reference. Tolerance: north_star's 1e-3 relative (rel-L2 and max/max)."""
import pytest
import torch

from fgt_b200 import synth
from tests.util import REL_TOL, assert_close, load_golden

pytestmark = pytest.mark.gpu


def _run(meta, capture=False):
    from fgt_b200.fgt_model import Model
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = tuple(meta["res"])
    sd = synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=meta["seed"], regime=meta["regime"])
    model = Model(cfg)
    model.load_state_dict(sd)
    model = model.cuda()
    fr, fl, mk = synth.fgt_inputs(seed=meta["seed"] + 2, t=meta["t"], H=meta["H"], W=meta["W"])
    cap = {} if capture else None
    model.net.capture = cap
    with torch.no_grad():
        out = model(fr.cuda(), fl.cuda(), mk.cuda())
    torch.cuda.synchronize()
    return out, cap, sd, (fr, fl, mk)


@pytest.mark.parametrize("name", ["fgt_small_scaled", "fgt_small_default", "fgt_runtime_geo"])
def test_fgt_small_vs_golden_and_oracle(name):
    from oracle import fgt_oracle as O
    g = load_golden(name)
    out, cap, sd, (fr, fl, mk) = _run(g["meta"], capture=True)
    assert tuple(out.shape) == tuple(g["out"].shape)
    assert_close(out, g["out"], REL_TOL, name + " vs reference golden")
    with torch.no_grad():
        ref, inter = O.fgt_forward(O.strip_net(sd), fr, fl, mk, return_intermediates=True)
    assert_close(out, ref, REL_TOL, name + " vs oracle")
    bt = g["meta"]["t"]
    for key in ("tok0", "ftok", "t0", "s0", "tok_final"):
        assert_close(cap[key].reshape(bt, -1, cap[key].shape[-1]), inter[key], REL_TOL, f"{name}:{key}")
    assert_close(cap["enc"].permute(0, 3, 1, 2), inter["enc"], REL_TOL, f"{name}:enc")


def test_fgt_full_t10_vs_golden():
    """BASELINE config 2: 432x240, T=10, against the sampled reference output."""
    g = load_golden("fgt_full_t10")
    out, _, _, _ = _run(g["meta"])
    assert tuple(out.shape) == (10, 3, 240, 432)
    assert torch.isfinite(out).all()
    assert_close(out.reshape(-1).cpu()[torch.from_numpy(g["idx"])], g["val"], REL_TOL, "fgt_full_t10 samples")
    assert abs(out.double().norm().item() - float(g["l2"])) / float(g["l2"]) < REL_TOL


def test_fgt_batch2_and_odd_t():
    """b=2 and odd t exercise the zone bookkeeping (b*4 zones, Lz not a multiple of 8)."""
    from oracle import fgt_oracle as O
    from fgt_b200.fgt_model import Model
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    sd = synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=5)
    model = Model(cfg)
    model.load_state_dict(sd)
    model = model.cuda()
    fr, fl, mk = synth.fgt_inputs(seed=9, t=3, H=64, W=96, b=2)
    with torch.no_grad():
        out = model(fr.cuda(), fl.cuda(), mk.cuda())
        ref = O.fgt_forward(O.strip_net(sd), fr, fl, mk)
    assert_close(out, ref, REL_TOL, "b=2,t=3")
    # determinism / idempotence: a second call on the same buffers gives the same bits
    with torch.no_grad():
        out2 = model(fr.cuda(), fl.cuda(), mk.cuda())
    assert torch.equal(out, out2)


def test_fgt_720p_padded_geometry():
    """BASELINE config 5 geometry (720x1280): tokens 60x107 -> temporal zones padded by one column,
    spatial grid padded to 64x112 (112 windows, 448 pooled tokens = 7 global key tiles). T=2 keeps the
    CPU oracle to a few seconds."""
    from oracle import fgt_oracle as O
    from fgt_b200.fgt_model import Model
    cfg = dict(synth.CFG_A)
    sd = synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=6)
    model = Model(cfg)
    model.load_state_dict(sd)
    model = model.cuda()
    fr, fl, mk = synth.fgt_inputs(seed=11, t=2, H=720, W=1280)
    with torch.no_grad():
        out = model(fr.cuda(), fl.cuda(), mk.cuda())
        ref = O.fgt_forward(O.strip_net(sd), fr, fl, mk)
    assert tuple(out.shape) == (2, 3, 720, 1280)
    assert_close(out, ref, REL_TOL, "720p T=2")


def test_clip_streamer_matches_direct_calls():
    """fgt_b200.streaming.ClipStreamer (H2D / forward / D2H on three streams, two slots) returns, in order,
    exactly what direct Model.forward calls return — with and without CUDA-graph replay."""
    from fgt_b200.fgt_model import Model
    from fgt_b200.streaming import ClipStreamer
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    sd = synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=8)
    model = Model(cfg)
    model.load_state_dict(sd)
    model = model.cuda()
    clips = [[t.contiguous().pin_memory() for t in synth.fgt_inputs(seed=20 + i, t=3, H=64, W=96)] for i in range(5)]
    with torch.no_grad():
        direct = [model(*[t.cuda() for t in c]).cpu() for c in clips]
    for graph in (False, True):
        model.net.enable_cuda_graph(graph)
        st = ClipStreamer(model, clips[0])
        got = [o.clone() for o in st.run(clips)]
        assert len(got) == 5
        for i, (a, b) in enumerate(zip(got, direct)):
            assert torch.equal(a, b), f"clip {i} (graph={graph})"
    model.net.enable_cuda_graph(False)


def test_fgt_driver_default_size_256x432():
    """The driver's default working size (--imgH 256 --imgW 432, tool/video_inpainting.py:829-830) on a checkpoint
    configured for 240x432: runtime geometry 22x36 tokens (temporal zones 11x18, spatial grid padded to 24x40), first
    window of a 10-frame clip (t=6). Sampled reference output + norm."""
    g = load_golden("fgt_driver_256x432_t6")
    out, _, _, _ = _run(g["meta"])
    assert tuple(out.shape) == (6, 3, 256, 432)
    assert torch.isfinite(out).all()
    assert_close(out.reshape(-1).cpu()[torch.from_numpy(g["idx"])], g["val"], REL_TOL, "fgt_driver_256x432 samples")
    assert abs(out.double().norm().item() - float(g["l2"])) / float(g["l2"]) < REL_TOL
