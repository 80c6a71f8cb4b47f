"""LAFC flow completion (SURVEY §8 row a8): oracle vs reference goldens (CPU) and the sm_90a path
vs oracle + goldens (GPU)."""
import pytest
import torch

from fgt_b200 import synth
from oracle import lafc_oracle as LO
from tests.util import REL_TOL, assert_close, load_golden


def _setup(meta):
    sd = synth.make_state_dict(synth.lafc_param_shapes(), seed=meta["seed"], regime=meta["regime"])
    fl, mk = synth.lafc_inputs(seed=meta["seed"] + 1, H=meta["H"], W=meta["W"])
    return sd, fl, mk


def _strip(sd):
    return {k[4:]: v for k, v in sd.items()}


@pytest.mark.parametrize("name", ["lafc_small_scaled", "lafc_small_kaiming"])
def test_lafc_oracle_small(name):
    g = load_golden(name)
    sd, fl, mk = _setup(g["meta"])
    with torch.no_grad():
        flow, edge = LO.lafc_forward(_strip(sd), fl, mk)
    assert_close(flow, g["flow"], 2e-5, name + " flow")
    assert_close(edge, g["edge"], 2e-5, name + " edge")


def test_lafc_oracle_full_sampled():
    g = load_golden("lafc_full")
    sd, fl, mk = _setup(g["meta"])
    with torch.no_grad():
        flow, edge = LO.lafc_forward(_strip(sd), fl, mk)
    assert_close(flow.reshape(-1)[torch.from_numpy(g["flow_idx"])], g["flow_val"], 2e-5, "lafc_full flow")
    assert_close(edge.reshape(-1)[torch.from_numpy(g["edge_idx"])], g["edge_val"], 2e-5, "lafc_full edge")


def test_lafc_state_dict_contract():
    from fgt_b200.lafc_model import Model
    m = Model(synth.CFG_LAFC)
    shapes = synth.lafc_param_shapes()
    sd = m.state_dict()
    assert set(sd.keys()) == set(shapes.keys())
    for k, s in shapes.items():
        assert tuple(sd[k].shape) == tuple(s), k
    with pytest.raises(RuntimeError):
        m(*synth.lafc_inputs(seed=0, H=32, W=32))  # CPU tensors: no fallback


def _run_gpu(meta):
    from fgt_b200.lafc_model import Model
    sd, fl, mk = _setup(meta)
    m = Model(synth.CFG_LAFC)
    m.load_state_dict(sd)
    m = m.cuda()
    with torch.no_grad():
        flow, edge = m(fl.cuda(), mk.cuda())
    torch.cuda.synchronize()
    return flow, edge, sd, fl, mk


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["lafc_small_scaled", "lafc_small_kaiming"])
def test_lafc_gpu_small(name):
    g = load_golden(name)
    flow, edge, sd, fl, mk = _run_gpu(g["meta"])
    assert tuple(flow.shape) == (1, 2, 64, 96) and tuple(edge.shape) == (1, 1, 64, 96)
    assert_close(flow, g["flow"], REL_TOL, name + " flow vs reference golden")
    assert_close(edge, g["edge"], REL_TOL, name + " edge vs reference golden")
    with torch.no_grad():
        rf, re_ = LO.lafc_forward(_strip(sd), fl, mk)
    assert_close(flow, rf, REL_TOL, name + " flow vs oracle")
    assert_close(edge, re_, REL_TOL, name + " edge vs oracle")


@pytest.mark.gpu
def test_lafc_gpu_full_sampled():
    g = load_golden("lafc_full")
    flow, edge, _, _, _ = _run_gpu(g["meta"])
    assert_close(flow.reshape(-1).cpu()[torch.from_numpy(g["flow_idx"])], g["flow_val"], REL_TOL, "lafc_full flow")
    assert_close(edge.reshape(-1).cpu()[torch.from_numpy(g["edge_idx"])], g["edge_val"], REL_TOL, "lafc_full edge")
    assert abs(flow.double().norm().item() - float(g["flow_l2"])) / float(g["flow_l2"]) < REL_TOL
