"""H100-native flow-guided gradient propagation behind the reference's function signature.

Drop-in for /root/reference/tool/get_flowNN_gradient.py: `get_flowNN_gradient(args, gradient_x,
gradient_y, mask_RGB, mask, videoFlowF, videoFlowB, None, None) -> (gradient_x, gradient_y,
mask_tofill)` with numpy arrays in the reference's layouts (call site tool/video_inpainting.py:623).
The sequential frame loop stays on the host (2(N-1) step launches, 2N gather launches, one fusion);
all per-pixel work runs in prop.cu. PyTorch only moves the arrays to the device and back.
"""
import numpy as np
import torch

from . import lib


def get_flowNN_gradient(args, gradient_x, gradient_y, mask_RGB, mask, videoFlowF, videoFlowB,
                        videoNonLocalFlowF=None, videoNonLocalFlowB=None, device="cuda:0"):
    if getattr(args, "Nonlocal", False):
        raise ValueError("fgt_b200 implements Nonlocal=False (the driver's setting, video_inpainting.py:796)")
    if not torch.cuda.is_available():
        raise RuntimeError("fgt_b200 get_flowNN_gradient needs a CUDA (sm_90a) device; there is no CPU fallback")
    dev = torch.device(device)
    thres, alpha = float(args.consistencyThres), float(args.alpha)
    m = torch.from_numpy(np.ascontiguousarray(mask.astype(np.uint8).transpose(2, 0, 1))).to(dev)  # [N,H,W]
    ff = torch.from_numpy(np.ascontiguousarray(videoFlowF.astype(np.float32).transpose(3, 0, 1, 2))).to(dev)
    fb = torch.from_numpy(np.ascontiguousarray(videoFlowB.astype(np.float32).transpose(3, 0, 1, 2))).to(dev)
    gx0 = torch.from_numpy(np.ascontiguousarray(gradient_x.astype(np.float32).transpose(3, 0, 1, 2))).to(dev)
    gy0 = torch.from_numpy(np.ascontiguousarray(gradient_y.astype(np.float32).transpose(3, 0, 1, 2))).to(dev)
    tofill = propagate(m, ff, fb, gx0, gy0, thres, alpha)
    out_x = gx0.permute(1, 2, 3, 0).cpu().numpy()
    out_y = gy0.permute(1, 2, 3, 0).cpu().numpy()
    # the reference fuses into its inputs in place and returns them (get_flowNN_gradient.py:517-534)
    if isinstance(gradient_x, np.ndarray) and gradient_x.dtype == np.float32 and gradient_x.flags.writeable:
        np.copyto(gradient_x, out_x)
        np.copyto(gradient_y, out_y)
        out_x, out_y = gradient_x, gradient_y
    return out_x, out_y, tofill.permute(1, 2, 0).cpu().numpy().astype(bool)


def slot_state(N, H, W, dev):
    """One NN slot's dense state (include/fgt_b200.h), with no neighbour anywhere."""
    return dict(ny=torch.zeros(N, H, W, dtype=torch.float64, device=dev),
                nx=torch.zeros(N, H, W, dtype=torch.float64, device=dev),
                nt=torch.full((N, H, W), -1, dtype=torch.int32, device=dev),
                have=torch.zeros(N, H, W, dtype=torch.uint8, device=dev),
                cuv=torch.zeros(N, H, W, 2, dtype=torch.float64, device=dev))


def propagate(m, ff, fb, gx0, gy0, thres, alpha):
    """The launch sequence on tensors in the kernels' layouts: mask m uint8 [N,H,W], flows [N-1,H,W,2], gradients
    [N,H,W,3] (fused in place). Returns mask_tofill, uint8 [N,H,W]."""
    N, H, W = m.shape
    dev = m.device
    state = [slot_state(N, H, W, dev) for _ in (0, 1)]
    # pass 1: backward-flow neighbours, frames 1..N-1; pass 2: forward-flow neighbours, frames N-2..0
    for t in range(1, N):
        s0 = state[0]
        lib.call("fgt_prop_step", m, fb[t - 1], ff[t - 1], H, W, t, t - 1, thres, s0["ny"], s0["nx"], s0["nt"], s0["have"],
                 s0["cuv"])
    for t in range(N - 2, -1, -1):
        s1 = state[1]
        lib.call("fgt_prop_step", m, ff[t], fb[t], H, W, t, t + 1, thres, s1["ny"], s1["nx"], s1["nt"], s1["have"],
                 s1["cuv"])
    cand = []
    for slot, order in ((0, range(N)), (1, range(N - 1, -1, -1))):
        gx, gy = gx0.clone(), gy0.clone()
        s_ = state[slot]
        for s in order:
            lib.call("fgt_prop_gather", m, s_["ny"], s_["nx"], s_["nt"], N, H, W, s, gx, gy)
        cand.append((gx, gy))
    tofill = torch.empty(N, H, W, dtype=torch.uint8, device=dev)
    lib.call("fgt_prop_fuse", m, state[0]["have"], state[1]["have"], state[0]["cuv"], state[1]["cuv"], N, H, W, alpha,
             cand[0][0], cand[0][1], cand[1][0], cand[1][1], gx0, gy0, tofill)
    return tofill
