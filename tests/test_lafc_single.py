"""The single-frame ("2D") LAFC of FGT's validation on the CPU: the oracle against goldens of the unmodified reference
(tests/golden/lafc_single_*.npz), the module's state-dict contract and refusals, the C-ABI call sequence of one forward
against its case of the launch-trace golden, and the whole native forward through the float64 interpreters of its
launches."""
import json

import pytest
import torch

from fgt_b200 import synth
from oracle import lafc_single_oracle as LSO
from tests.kernel_emulator import emulating_all
from tests.test_launch_trace import load_golden as load_trace_golden
from tests.test_launch_trace import recording
from tests.util import assert_close, load_golden

FULL = ["lafc_single_scaled", "lafc_single_kaiming", "lafc_single_odd"]
SAMPLED = ["lafc_single_full_scaled", "lafc_single_full_kaiming"]


def setup(meta):
    """(state dict, flows, masks) of a golden's meta."""
    sd = synth.lafc_single_state_dict(seed=meta["seed"], regime=meta["regime"])
    fl, mk = synth.lafc_single_inputs(seed=meta["seed"] + 1, n=meta["n"], H=meta["H"], W=meta["W"])
    return sd, fl, mk


def strip(sd):
    return {k[4:]: v for k, v in sd.items()}


def model(sd=None):
    from fgt_b200.lafc_single import Model
    m = Model(synth.CFG_LAFC_SINGLE)
    if sd is not None:
        m.load_state_dict(sd)
    return m


@pytest.mark.parametrize("name", FULL + SAMPLED)
def test_oracle_matches_reference_golden(name):
    g = load_golden(name)
    sd, fl, mk = setup(g["meta"])
    with torch.no_grad():
        flow, edge = LSO.lafc_single_forward(strip(sd), fl, mk)
    if "flow" in g:
        assert_close(flow, g["flow"], 1e-6, name + " flow")
        assert_close(edge, g["edge"], 1e-6, name + " edge")
    else:
        assert_close(flow.reshape(-1)[torch.from_numpy(g["flow_idx"])], g["flow_val"], 1e-6, name + " flow")
        assert_close(edge.reshape(-1)[torch.from_numpy(g["edge_idx"])], g["edge_val"], 1e-6, name + " edge")
        assert abs(flow.double().norm().item() - float(g["flow_l2"])) <= 1e-6 * float(g["flow_l2"])


def test_state_dict_matches_the_reference_keys_and_shapes():
    g = load_golden("lafc_single_scaled")
    got = model().state_dict()
    assert list(got) == [str(k) for k in g["keys"]]
    assert [repr(tuple(v.shape)) for v in got.values()] == [str(s) for s in g["shapes"]]
    m = model(synth.lafc_single_state_dict(seed=1))
    with pytest.raises(RuntimeError, match="CUDA"):
        m(*synth.lafc_single_inputs(seed=0, n=1, H=32, W=32))   # CPU tensors: no fallback


@pytest.mark.parametrize("key,value", [("conv_type", "gated"), ("conv_type", "partial"), ("PASSMASK", 0),
                                       ("use_bias", 0), ("in_channel", 4)])
def test_refuses_what_it_does_not_implement(key, value):
    from fgt_b200.lafc_single import Model
    with pytest.raises(ValueError, match="2D LAFC"):
        Model({**synth.CFG_LAFC_SINGLE, key: value})


def test_refuses_edges_and_bad_geometry():
    m = model(synth.lafc_single_state_dict(seed=1))
    fl, mk = synth.lafc_single_inputs(seed=0, n=1, H=32, W=32)
    with pytest.raises(ValueError, match="edges"):
        m(fl, mk, torch.zeros(1, 1, 32, 32))
    with recording(), pytest.raises(ValueError, match="divisible by 4"):
        m.net._forward_impl(fl[:, :, :30], mk[:, :, :30])
    with recording(), pytest.raises(ValueError, match=r"masks \[n,1,H,W\]"):
        m.net._forward_impl(fl, mk[:, :, :16])


def test_res_blocks_are_separate_blocks():
    """make_layer builds resBlocks independent blocks (unlike the P3D LAFC's one shared block)."""
    cfg = {**synth.CFG_LAFC_SINGLE, "resBlocks": 2}
    from fgt_b200.lafc_single import Model
    keys = set(Model(cfg).state_dict())
    assert keys == set(synth.lafc_single_param_shapes(cfg))
    assert "net.res_blocks.1.conv2.weight" in keys


def trace():
    """The recorded C-ABI calls of one forward: 64 x 96, n = 2."""
    m = model(synth.lafc_single_state_dict(seed=5))
    fl, mk = synth.lafc_single_inputs(seed=6, n=2, H=64, W=96)
    with torch.no_grad(), recording() as rec:
        m.net._forward_impl(fl, mk)
    return json.loads(json.dumps(rec.calls))


def test_launch_trace_matches_golden():
    want = load_trace_golden()["lafc_single"]
    got = trace()
    assert [c[0] for c in got] == [c[0] for c in want], "entry sequence differs"
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"call {i} ({g[0]}) differs"


def test_forward_in_float64():
    """Every launch of one forward (im2col, GEMMs, upsampling) interpreted in float64, against the reference's golden
    and the oracle, at the bar the other networks' float64 forwards meet."""
    g = load_golden("lafc_single_scaled")
    sd, fl, mk = setup(g["meta"])
    m = model(sd)
    with torch.no_grad(), emulating_all():
        flow, edge = m.net._forward_impl(fl, mk)
    assert_close(flow, g["flow"], 2.2e-5, "2D LAFC flow vs reference golden")
    assert_close(edge, g["edge"], 2.2e-5, "2D LAFC edge vs reference golden")
    with torch.no_grad():
        rf, re_ = LSO.lafc_single_forward(strip(sd), fl, mk)
    assert_close(flow, rf, 2.2e-5, "2D LAFC flow vs oracle")
    assert_close(edge, re_, 2.2e-5, "2D LAFC edge vs oracle")
