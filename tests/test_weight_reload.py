"""Loading weights drops every cache derived from the old ones, whichever module the load is called on.

`nn.Module.load_state_dict` reaches submodules through `_load_from_state_dict`, not through their own
`load_state_dict`, so a load through the reference-compatible wrapper (`fgt_model.Model`, `lafc_model.Model`,
`nn.DataParallel(RAFT)`) must still invalidate the network's packed weights and captured CUDA graphs: otherwise the next
forward runs the old weights, and a graph replay reads the old packed weights' addresses."""
import argparse

import torch

from fgt_b200 import synth

CPU = torch.device("cpu")


def _fgt(seed):
    from fgt_b200.fgt_model import Model
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    return Model(cfg), synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=seed)


def _lafc(seed):
    from fgt_b200.lafc_model import Model
    return Model(synth.CFG_LAFC), synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=seed)


def _raft(seed):
    from fgt_b200.raft_model import RAFT
    dp = torch.nn.DataParallel(RAFT(argparse.Namespace(small=False, mixed_precision=False, alternate_corr=False)))
    return dp, {"module." + k: v for k, v in synth.raft_state_dict(seed=seed).items()}


def _net(wrapper):
    return wrapper.module if isinstance(wrapper, torch.nn.DataParallel) else wrapper.net


def _equal(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_equal(a[k], b[k]) for k in a)
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b)
    return a == b


def test_load_through_the_wrapper_drops_packed_weights_and_graphs():
    for make in (_fgt, _lafc, _raft):
        wrapper, sd_old = make(1)
        wrapper.load_state_dict(sd_old)
        net = _net(wrapper)
        net._pack(CPU)
        net.enable_cuda_graph(True)
        net._graphed(("key",), lambda x: x, torch.zeros(1))   # first call of a key runs eagerly and records it
        assert net._packed and net._graphs

        _, sd_new = make(2)
        wrapper.load_state_dict(sd_new)
        assert not net._packed and not net._graphs, make.__name__

        fresh, _ = make(2)
        fresh.load_state_dict(sd_new)
        assert _equal(net._pack(CPU), _net(fresh)._pack(CPU)), make.__name__
