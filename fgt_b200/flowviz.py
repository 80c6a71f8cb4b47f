"""Flow colour coding on the GPU: RAFT/utils/flow_viz.py `flow_to_image` (the Middlebury colour wheel, each flow
normalised by its own maximum radius), for a whole batch of flows in one launch pair (csrc/flowviz.cu; definition:
oracle/flowviz_oracle.py). The driver colours every flow it writes with `--vis_flows` this way (tool/video_inpainting.py
:274-282); `python -m fgt_b200.pipeline --vis_flows / --vis_completed_flows` does it here.

Rounding follows numpy's on the float32 flows, operation by operation, except the angle: the device's atan2f and the
host's float32 arctan2 may differ by an ulp, which moves a few values in a million by one level. A NaN or Inf in a
flow raises ValueError (the reference raises IndexError). There is no CPU fallback.
"""
import numpy as np
import torch

from . import lib

HOST_BUDGET = 1 << 30     # bytes of flows copied to the device per launch pair when the input is a host array


def _device(flows, device):
    if device is not None:
        dev = torch.device(device)
    elif torch.is_tensor(flows) and flows.is_cuda:
        dev = flows.device
    elif torch.cuda.is_available():
        dev = torch.device("cuda", torch.cuda.current_device())
    else:
        dev = None
    if dev is None or dev.type != "cuda":
        raise RuntimeError("fgt_b200.flowviz runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    return dev


def _colour(x, bgr, out, first=0):
    """x: contiguous float32 [B,H,W,2] on the device -> out uint8 [B,H,W,3]; raises ValueError on NaN / Inf (naming
    the flows by their index in the caller's batch, x[0] being flow `first`)."""
    B, H, W, _ = x.shape
    ws = torch.empty(lib.call("fgt_flow_to_image_workspace", B, H, W), dtype=torch.uint8, device=x.device)
    maxima = torch.empty(B, dtype=torch.float32, device=x.device)
    lib.call("fgt_flow_to_image", x, B, H, W, 1 if bgr else 0, ws, ws.numel(), out, maxima, kernels=2)
    bad = (first + np.flatnonzero(np.isnan(maxima.cpu().numpy()))).tolist()
    if bad:
        raise ValueError(f"flow_to_image: flow{'s' if len(bad) > 1 else ''} {bad[:8]} of the batch hold NaN or Inf")


def flow_to_image(flows, convert_to_bgr=False, device=None):
    """flows: float32 [H,W,2] or [B,H,W,2] (u, v), a numpy array or a tensor -> uint8 [H,W,3] / [B,H,W,3] colour
    images (RGB, or BGR with convert_to_bgr), each flow divided by its own maximum radius + 1e-5 as flow_to_image
    does. A numpy input gives a numpy output (long batches are copied to the device in chunks); a tensor gives a
    tensor on `device` (default: the input's CUDA device, else the current one)."""
    is_np = not torch.is_tensor(flows)
    t = torch.from_numpy(np.asarray(flows)) if is_np else flows
    if t.dtype != torch.float32:
        raise TypeError(f"flow_to_image: flows must be float32, got {t.dtype}")
    if t.dim() not in (3, 4) or t.shape[-1] != 2:
        raise ValueError(f"flow_to_image: flows {tuple(t.shape)} must be [H,W,2] or [B,H,W,2]")
    single = t.dim() == 3
    if single:
        t = t.unsqueeze(0)
    B, H, W, _ = t.shape
    if B == 0 or H == 0 or W == 0:
        raise ValueError(f"flow_to_image: flows {tuple(t.shape)} are empty")
    dev = _device(flows, device)
    # device-resident flows go in one launch pair (up to 65535 images); host flows in chunks of HOST_BUDGET bytes
    chunk = max(1, min(B, 65535, B if t.device == dev else HOST_BUDGET // (8 * H * W)))
    with torch.cuda.device(dev):
        out = torch.empty(B, H, W, 3, dtype=torch.uint8, device=dev)
        for s in range(0, B, chunk):
            e = min(B, s + chunk)
            _colour(t[s:e].to(dev).contiguous(), convert_to_bgr, out[s:e], s)
        if is_np:
            out = out.cpu().numpy()
    return out[0] if single else out
