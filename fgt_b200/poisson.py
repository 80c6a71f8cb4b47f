"""Drop-in for tool/utils/Poisson_blend_img.py (`Poisson_blend_img`, `getUnfilledMask`), batched on the GPU:
all frames x colour channels of a clip are solved together by matrix-free LSQR in fp64 (csrc/poisson.cu) with
scipy's recurrences and stopping tests, instead of one sparse assembly + three `scipy.sparse.linalg.lsqr`
calls + two O(hole pixels) Python loops per frame (Poisson_blend_img.py:35-38,139-170). The reference's answer
is the LSQR iterate at which the default stopping rule (atol = btol = 1e-6) fires, so that rule is reproduced
rather than replaced by a tighter solve; results agree with the reference to ~1e-6 on [0,1] images (the
reference's own bidiagonalisation runs in float32). There is no CPU fallback.
"""
import ctypes

import numpy as np
import torch

from . import lib

CHUNK = 48            # iterations per graph replay = between convergence checks (one host sync each)
MAX_ITERS = None      # None: scipy's own limit iter_lim = 2*H*W (then istop = 7 and the iterate is returned as is)


def _dev(device):
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("fgt_b200 Poisson blending runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    return dev


def _mask(m, dev, shape, name):
    if m is None:
        return None
    t = (torch.as_tensor(np.asarray(m) if not torch.is_tensor(m) else m).to(dev) != 0).to(torch.uint8).contiguous()
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"poisson: {name} {tuple(t.shape)} must be {tuple(shape)}")
    return t


def poisson_blend_batch(trg, gx, gy, hole, gmask=None, edge=None, device=None, return_info=False,
                        atol=1e-6, btol=1e-6, conlim=1e8, max_iters=MAX_ITERS, use_graph=True):
    """trg [F,H,W,3], gx [F,H,W-1,3], gy [F,H-1,W,3] (forward differences of the source), hole [F,H,W],
    optional gmask / edge [F,H,W] -> (blend float64 [F,H,W,3], UnfilledMask bool [F,H,W]) on the device
    (+ per-system (istop, itn) int tensors [F,3] with return_info). max_iters is scipy's iter_lim (default 2*H*W): a
    system still running at iteration max_iters stops there with istop 7 and returns its iterate. use_graph: replay
    each chunk of iterations as one CUDA graph (default) or launch its kernels one by one."""
    dev = _dev(device)
    # host arrays cross the bus in their own dtype (float32 in the driver) and are widened on the device (exact)
    t64 = lambda a: torch.as_tensor(np.ascontiguousarray(a) if not torch.is_tensor(a) else a).to(dev).to(torch.float64).contiguous()
    trg, gx, gy = t64(trg), t64(gx), t64(gy)
    if trg.dim() != 4 or trg.shape[3] != 3:
        raise ValueError(f"poisson: target {tuple(trg.shape)} must be [F,H,W,3]")
    F, H, W, C = trg.shape
    if H < 2 or W < 2:
        raise ValueError("poisson: images must be at least 2x2")
    if tuple(gx.shape) != (F, H, W - 1, C) or tuple(gy.shape) != (F, H - 1, W, C):
        raise ValueError(f"poisson: gradients {tuple(gx.shape)} / {tuple(gy.shape)} must be "
                         f"{(F, H, W - 1, C)} / {(F, H - 1, W, C)}")
    hole = _mask(hole, dev, (F, H, W), "holeMask")
    gmask = _mask(gmask, dev, (F, H, W), "gradientMask")
    edge = _mask(edge, dev, (F, H, W), "edge")
    S = F * C
    z64 = lambda *s: torch.zeros(*s, dtype=torch.float64, device=dev)
    code = torch.zeros(F, H, W, dtype=torch.uint8, device=dev)
    u = z64(F, 4, H * W, C)
    v, w, x = z64(F, H * W, C), z64(F, H * W, C), z64(F, H * W, C)
    iter_lim = 2 * H * W                               # scipy.sparse.linalg.lsqr's default for an [m, H*W] system
    if max_iters is not None:
        if max_iters < 1:
            raise ValueError(f"poisson: max_iters {max_iters} must be at least 1")
        iter_lim = min(max_iters, iter_lim)            # the device-side test k >= iter_lim stops every system there
    slots = iter_lim + CHUNK + 2                       # a replay may run past the last stop by < CHUNK (frozen) iterations
    bb, aa, ww = z64(slots * S), z64(slots * S), z64(slots * S)
    state = z64(2, S, 16)
    plist = torch.zeros(F, H * W, dtype=torch.int32, device=dev)    # uint32 entries: pixel | code << 24, 0 = none
    cnt = torch.zeros(F, dtype=torch.int32, device=dev)
    kctr = torch.zeros(2, dtype=torch.int32, device=dev)             # device-side iteration index (csrc/poisson.cu)
    lib.call("fgt_poisson_setup", trg, gx, gy, hole, gmask, edge, F, H, W, code, u, bb, plist, cnt)
    clr = torch.empty(2, F, H, W, dtype=torch.uint8, device=dev)
    lib.call("fgt_poisson_unfilled", hole, gmask, F, H, W, clr)
    max_cnt = int(cnt.max())                           # pixels owning equations, largest frame (one host sync)
    iter_args = (plist, max_cnt, F, H, W, u, v, w, x, bb, aa, ww, state, kctr, CHUNK, atol, btol, conlim, iter_lim)
    exec_ = ctypes.c_void_p()
    if use_graph:
        lib.call("fgt_poisson_graph_create", *iter_args, ctypes.byref(exec_))
    k = 0
    try:
        while True:
            if k > iter_lim + CHUNK:                   # cannot happen: every system stops by iteration iter_lim (istop 7)
                raise RuntimeError(f"poisson: LSQR did not stop within {iter_lim} iterations")
            if use_graph:
                lib.call("fgt_poisson_graph_launch", exec_, kernels=2 * CHUNK)
            else:
                lib.call("fgt_poisson_iters", *iter_args, kernels=2 * CHUNK)
            k += CHUNK
            last = state[(k - 1) & 1]                     # written by iteration k-1
            if bool((last[:, 12] != 0).all()):             # one host sync per CHUNK iterations
                break
    finally:
        if exec_:
            lib.call("fgt_poisson_graph_destroy", exec_)
    out = torch.empty_like(trg)
    unf = torch.empty(F, H, W, dtype=torch.uint8, device=dev)
    lib.call("fgt_poisson_finish", trg, hole, x, F, H, W, out, clr, unf)
    unf = unf.bool()
    if return_info:
        return out, unf, last[:, 13].to(torch.int64).view(F, C), last[:, 14].to(torch.int64).view(F, C)
    return out, unf


def Poisson_blend_img(imgTrg, imgSrc_gx, imgSrc_gy, holeMask, gradientMask=None, edge=None):
    """tool/utils/Poisson_blend_img.py:19-44 for one frame: numpy in, (imgBlend float64 [H,W,3], UnfilledMask bool)
    numpy out. Non-ndarray gradientMask / edge mean "none", as in the reference (:23-27)."""
    gm = gradientMask[None] if isinstance(gradientMask, np.ndarray) else None
    ed = edge[None] if isinstance(edge, np.ndarray) else None
    out, unf = poisson_blend_batch(np.asarray(imgTrg)[None], np.asarray(imgSrc_gx)[None], np.asarray(imgSrc_gy)[None],
                                   np.asarray(holeMask)[None], gm, ed)
    return out[0].cpu().numpy(), unf[0].cpu().numpy()


def poisson_blend_clip(video, gradient_x, gradient_y, mask, mask_gradient):
    """The driver's per-frame loop (tool/video_inpainting.py:643-656) as ONE batch, in the driver's array layout:
    video [H,W,3,N], gradient_x / gradient_y [H,W,3,N], mask / mask_gradient [H,W,N] -> (blend [N,H,W,3] float64,
    UnfilledMask [N,H,W] bool) numpy. Frames whose mask is empty are returned unchanged with an empty mask, as
    the driver skips them (:647)."""
    H, W = mask.shape[:2]
    mv = lambda a: np.ascontiguousarray(np.moveaxis(a, -1, 0))
    out, unf = poisson_blend_batch(mv(video), mv(gradient_x[:, :W - 1]), mv(gradient_y[:H - 1]), mv(mask), mv(mask_gradient))
    return out.cpu().numpy(), unf.cpu().numpy()


def getUnfilledMask(holeMask, gradientMask):
    """tool/utils/Poisson_blend_img.py:270-309: numpy [H,W] in, bool [H,W] out."""
    dev = _dev(None)
    hole = _mask(np.asarray(holeMask)[None], dev, (1,) + tuple(np.asarray(holeMask).shape), "holeMask")
    gm = _mask(np.asarray(gradientMask)[None], dev, tuple(hole.shape), "gradientMask")
    _, H, W = hole.shape
    clr = torch.empty(2, 1, H, W, dtype=torch.uint8, device=dev)
    lib.call("fgt_poisson_unfilled", hole, gm, 1, H, W, clr)
    return ((hole != 0) & (clr[0] == 0) & (clr[1] == 0))[0].cpu().numpy()
