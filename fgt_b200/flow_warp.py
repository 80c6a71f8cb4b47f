"""Drop-in for LAFC/models/utils/flow_warp.py (`flow_prop`, `warp`): forward splatting of features along a flow
with Gaussian weights (SURVEY §8 row a10 — dead code in the reference, named by the north star). csrc/splat.cu;
no CPU fallback. Flow channel 0 shifts columns, channel 1 rows, exactly as the reference's (confusingly named)
code does (flow_warp.py:24-25,60-77)."""
import torch

from . import lib


def warp(feat, flow, mode):
    if mode not in ("forward", "backward"):
        raise AssertionError("Invalid mode: {}".format(mode))
    if not feat.is_cuda:
        raise RuntimeError("fgt_b200.flow_warp runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    b, c, h, w = feat.shape
    if tuple(flow.shape) != (b, 2, h, w):
        raise ValueError(f"flow_warp: flow {tuple(flow.shape)} does not match features {tuple(feat.shape)}")
    feat = feat.float().contiguous()
    flow = flow.to(feat.device).float().contiguous()
    out = torch.empty_like(feat)
    wsum = torch.empty(b, h, w, dtype=torch.float32, device=feat.device)
    lib.call("fgt_flow_splat", feat, flow, b, c, h, w, int(mode == "backward"), out, wsum, kernels=2)
    return out


def flow_prop(feat, flow, mode="forward"):
    """flow_warp.py:4-18."""
    return warp(feat, flow, mode)
