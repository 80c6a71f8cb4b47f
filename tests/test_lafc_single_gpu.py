"""The 2D LAFC on the H100: against the reference goldens and the oracle in both weight regimes, at t = 1, 3 and 13
(240 x 432, sampled) and an odd size; CUDA-graph replay against eager; and a launch-by-launch replay of a 240 x 432
forward (every launch, the GEMMs included) against the float64 interpreters, as tests/test_kernel_replay_gpu.py does
for the other networks."""
import pytest
import torch

from fgt_b200 import synth
from oracle import lafc_single_oracle as LSO
from tests.test_lafc_single import FULL, SAMPLED, model, setup, strip
from tests.util import REL_TOL, assert_close, load_golden

pytestmark = pytest.mark.gpu


def _run(m, fl, mk):
    with torch.no_grad():
        flow, edge = m(fl.cuda(), mk.cuda())
    torch.cuda.synchronize()
    return flow.cpu(), edge.cpu()


@pytest.mark.parametrize("name", FULL)
def test_against_golden_and_oracle(name):
    g = load_golden(name)
    sd, fl, mk = setup(g["meta"])
    m = model(sd).cuda()
    flow, edge = _run(m, fl, mk)
    assert flow.shape == fl.shape and edge.shape == mk.shape
    assert_close(flow, g["flow"], REL_TOL, name + " flow vs reference golden")
    assert_close(edge, g["edge"], REL_TOL, name + " edge vs reference golden")
    with torch.no_grad():
        rf, re_ = LSO.lafc_single_forward(strip(sd), fl, mk)
    assert_close(flow, rf, REL_TOL, name + " flow vs oracle")
    assert_close(edge, re_, REL_TOL, name + " edge vs oracle")
    # t = 1: the first frame alone gives the golden's first frame
    f1, e1 = _run(m, fl[:1], mk[:1])
    assert_close(f1, g["flow"][:1], REL_TOL, name + " t=1 flow")
    assert_close(e1, g["edge"][:1], REL_TOL, name + " t=1 edge")


@pytest.mark.parametrize("name", SAMPLED)
def test_240x432_t13_sampled(name):
    g = load_golden(name)
    sd, fl, mk = setup(g["meta"])
    flow, edge = _run(model(sd).cuda(), fl, mk)
    assert_close(flow.reshape(-1)[torch.from_numpy(g["flow_idx"])], g["flow_val"], REL_TOL, name + " flow")
    assert_close(edge.reshape(-1)[torch.from_numpy(g["edge_idx"])], g["edge_val"], REL_TOL, name + " edge")
    assert abs(flow.double().norm().item() - float(g["flow_l2"])) <= REL_TOL * float(g["flow_l2"])
    assert abs(edge.double().norm().item() - float(g["edge_l2"])) <= REL_TOL * float(g["edge_l2"])


def test_graph_replay_equals_eager():
    g = load_golden("lafc_single_odd")
    sd, fl, mk = setup(g["meta"])
    m = model(sd).cuda()
    eager = _run(m, fl, mk)
    m.net.enable_cuda_graph()
    for seed in (0, 1):   # first call eager, then captured, then replayed with other inputs
        _run(m, *synth.lafc_single_inputs(seed=seed, n=fl.shape[0], H=fl.shape[2], W=fl.shape[3]))
    for a, b in zip(_run(m, fl, mk), eager):
        assert torch.equal(a, b)


def test_replay_240x432_every_launch():
    from tests.test_kernel_replay_gpu import replaying
    sd = synth.lafc_single_state_dict(seed=5)
    m = model(sd).cuda()
    fl, mk = (x.cuda() for x in synth.lafc_single_inputs(seed=6, n=1, H=240, W=432))
    with torch.no_grad():
        m.net._forward_impl(fl, mk)
        with replaying() as r:
            m.net._forward_impl(fl, mk)
    r.report("lafc_single_240x432")
    assert sum(r.launches.values()) == 26
