"""Forward flow splatting (SURVEY §8 row a10: LAFC/models/utils/flow_warp.py — never called by the reference, but
named by the north star). Oracle vs the reference golden on the CPU; CUDA kernel vs oracle and golden on the GPU
(float atomics: summation order differs from the reference's sequential put_, tolerance 1e-5 of the value range)."""
import numpy as np
import pytest
import torch

from fgt_b200 import synth
from oracle import flow_warp_oracle as FO
from tests.util import load_golden


@pytest.mark.parametrize("mode", ["forward", "backward"])
def test_oracle_matches_reference_golden(mode):
    g = load_golden("flow_warp")
    feat, flow = synth.flow_warp_inputs(seed=g["meta"]["seed"])
    out = FO.flow_prop(feat, flow, mode)
    assert np.abs(out.numpy() - g[mode]).max() < 1e-5
    # identity flow: a pixel receives its own value with weight 1 plus neighbours' contributions; zero flow everywhere
    # gives back the input (weights e^0 on itself, e^-1, e^-1, e^-2 pushed to the right/down neighbours)
    z = FO.flow_prop(feat, torch.zeros_like(flow), mode)
    assert torch.isfinite(z).all() and z.shape == feat.shape


def test_oracle_partition_of_unity_for_constant_features():
    feat = torch.ones(1, 3, 12, 16)
    _, flow = synth.flow_warp_inputs(seed=3, b=1, c=3, h=12, w=16)
    out = FO.flow_prop(feat, flow)
    assert ((out - 1).abs() < 1e-5)[out != 0].all() and ((out == 0) | ((out - 1).abs() < 1e-5)).all()


@pytest.mark.parametrize("mode", ["forward", "backward"])
def test_kernel_target_logic_on_host_matches_oracle(mode):
    """The kernel's per-pixel function (splat_targets, __host__ __device__) run on the host for every source pixel;
    the scatter assembled in numpy equals the oracle."""
    import ctypes
    from fgt_b200 import lib
    L = lib.load()
    feat, flow = synth.flow_warp_inputs(seed=4, b=1, c=2, h=9, w=11)
    f, fl = feat.numpy(), flow.numpy()
    acc = np.zeros_like(f, dtype=np.float64)
    osum = np.zeros(f.shape[2:], dtype=np.float64)
    ti, tj, ok = (np.zeros(4, np.int32) for _ in range(3))
    wt = np.zeros(4, np.float32)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    for i in range(f.shape[2]):
        for j in range(f.shape[3]):
            assert L.fgt_flow_splat_targets_host(float(fl[0, 1, i, j]), float(fl[0, 0, i, j]), i, j, f.shape[2], f.shape[3],
                                                 int(mode == "backward"), P(ti), P(tj), P(wt), P(ok)) == 0
            for q in range(4):
                if ok[q]:
                    acc[0, :, ti[q], tj[q]] += f[0, :, i, j].astype(np.float64) * wt[q]
                    osum[ti[q], tj[q]] += wt[q]
    out = np.where(osum > 0, acc / np.where(osum > 0, osum, 1), acc)
    assert np.abs(out - FO.flow_prop(feat, flow, mode).numpy()).max() < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["forward", "backward"])
def test_gpu_flow_warp_vs_golden_and_oracle(mode):
    from fgt_b200 import flow_warp as FW
    g = load_golden("flow_warp")
    feat, flow = synth.flow_warp_inputs(seed=g["meta"]["seed"])
    out = FW.flow_prop(feat.cuda(), flow.cuda(), mode).cpu()
    scale = float(np.abs(g[mode]).max())
    assert np.abs(out.numpy() - g[mode]).max() < 1e-5 * max(scale, 1.0)
    assert (out - FO.flow_prop(feat, flow, mode)).abs().max().item() < 1e-5 * max(scale, 1.0)
    with pytest.raises(RuntimeError):
        FW.flow_prop(feat, flow, mode)
