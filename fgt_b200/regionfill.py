"""Drop-in for tool/utils/region_fill.py (`regionfill`) and the driver's `diffusion()`
(tool/video_inpainting.py:44-52), batched on the GPU: all images of a call are solved together by
matrix-free conjugate gradients in fp64 (csrc/laplace.cu) instead of one sparse direct solve per image
and channel. Results agree with the reference's spsolve to the CG tolerance (default: relative residual
1e-12, i.e. ~1e-9 px on flows); there is no CPU fallback.
"""
import numpy as np
import torch

from . import lib

CHUNK = 64           # iterations between convergence checks (one host sync each)
MAX_ITERS = None     # None: max(10000, 50 * (H + W)) — CG on a hole of diameter d needs ~25 d iterations at tol 1e-12


def _dev(device):
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("fgt_b200 regionfill runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    return dev


def regionfill_batch(images, masks, tol=1e-12, device=None, return_iters=False, max_iters=MAX_ITERS):
    """images [B,H,W] float (numpy or tensor), masks [B,H,W] bool/uint8 -> float64 tensor [B,H,W] on the device:
    harmonic fill inside each mask, the image unchanged outside."""
    dev = _dev(device)
    img = torch.as_tensor(images).to(dev, torch.float64).contiguous()
    msk = (torch.as_tensor(masks).to(dev) != 0).to(torch.uint8).contiguous()
    if img.dim() != 3 or img.shape != msk.shape:
        raise ValueError(f"regionfill: images {tuple(img.shape)} and masks {tuple(msk.shape)} must both be [B,H,W]")
    B, H, W = img.shape
    if max_iters is None:
        max_iters = max(10000, 50 * (H + W))
    full = msk.flatten(1).all(dim=1)
    if bool(full.any()):
        raise ValueError("regionfill: a mask covers its whole image (singular system; the reference fails too)")
    x, r, p0, p1, ap = (torch.empty_like(img) for _ in range(5))
    # per-iteration scalars <r,r> and <p,Ap> of every image: one slot per iteration, never reset (csrc/laplace.cu)
    rr = torch.zeros((max_iters + 1) * B, dtype=torch.float64, device=dev)
    pap = torch.zeros(max_iters * B, dtype=torch.float64, device=dev)
    lib.call("fgt_regionfill_init", img, msk, B, H, W, x, r, p0, rr)
    rr0 = rr[:B].clone()
    k = 0
    while k < max_iters:
        n = min(CHUNK, max_iters - k)
        lib.call("fgt_regionfill_iters", msk, B, H, W, x, r, p0, p1, ap, rr, pap, k, n, kernels=2 * n)
        k += n
        if bool((rr[k * B:(k + 1) * B] <= (tol * tol) * rr0).all()):   # one host sync per CHUNK iterations
            break
    else:
        raise RuntimeError(f"regionfill: CG did not reach relative residual {tol:g} in {max_iters} iterations")
    out = torch.empty_like(img)
    lib.call("fgt_regionfill_finish", img, msk, img.numel(), x, out)
    return (out, k) if return_iters else out


def regionfill(I, mask, factor=1.0):
    """tool/utils/region_fill.py:7-17 for one image: numpy in, float64 numpy out."""
    if factor != 1.0:
        raise ValueError("fgt_b200 regionfill implements factor=1.0 (the driver's call, video_inpainting.py:49-50)")
    mask = np.asarray(mask)
    if np.count_nonzero(mask) == 0:
        return np.asarray(I).copy()
    return regionfill_batch(np.asarray(I)[None], mask[None])[0].cpu().numpy()


def diffusion(flows, masks):
    """tool/video_inpainting.py:44-52: flows [N,H,W,2], masks [N,H,W,1] -> list of N float64 arrays [H,W,2];
    the 2N solves run as one batch."""
    flows, masks = np.asarray(flows), np.asarray(masks)
    N = flows.shape[0]
    imgs = np.concatenate([flows[..., 0], flows[..., 1]], 0)
    m = np.concatenate([masks[..., 0], masks[..., 0]], 0)
    out = regionfill_batch(imgs, m).cpu().numpy()
    return [np.stack([out[i], out[N + i]], -1) for i in range(N)]
