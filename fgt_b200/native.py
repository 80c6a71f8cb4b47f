"""Native-resolution output of the pipeline on the device: the working-resolution result upscaled to the input frames'
size and pasted into the original frames inside a feathered band around the mask, so that only the neighbourhood of the
hole is resampled (csrc/native.cu; the definition is written out in oracle/native_oracle.py, which the kernels equal
bit for bit). No CPU fallback.
"""
import math

import numpy as np
import torch

from . import lib, morph


def _dev(device):
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("fgt_b200.native runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    return dev


def _u8(x, dev, what):
    t = torch.as_tensor(np.ascontiguousarray(x) if not torch.is_tensor(x) else x)
    if t.dtype != torch.uint8:
        raise TypeError(f"composite_native: {what} must be uint8, got {t.dtype}")
    return t.to(dev).contiguous()


def native_window(h, w, imgH, imgW, frame_dilates):
    """(k, r): the blend window's half-width k = ceil(s) and the L1 radius r = ceil(s * (frame_dilates + 2)) + 2 around
    the hole that is pure upscaled result, s = max(h / imgH, w / imgW)."""
    s = max(h / imgH, w / imgW)
    return int(math.ceil(s)), int(math.ceil(s * (frame_dilates + 2))) + 2


def composite_native(comp, frames, masks, frame_dilates, device=None):
    """comp uint8 [N,imgH,imgW,3] (the pipeline's output), frames uint8 [N,h,w,3] (the original frames), masks
    [N,h,w] / [N,h,w,C] per frame or one [h,w] / [h,w,C] for every frame (counted once); a pixel is in the hole when any
    channel is non-zero. numpy arrays or tensors. Returns a uint8 tensor [N,h,w,3] on the device."""
    dev = _dev(device)
    cp, fr = _u8(comp, dev, "comp"), _u8(frames, dev, "frames")
    if fr.dim() != 4 or cp.dim() != 4 or cp.shape[0] != fr.shape[0] or cp.shape[3] != fr.shape[3]:
        raise ValueError(f"composite_native: comp {tuple(cp.shape)} and frames {tuple(fr.shape)} must be [N,imgH,imgW,C] "
                         "and [N,h,w,C]")
    N, h, w, C = fr.shape
    imgH, imgW = cp.shape[1:3]
    m = torch.as_tensor(np.ascontiguousarray(masks) if not torch.is_tensor(masks) else masks).to(dev)
    given = tuple(m.shape)
    if m.dim() == 2 or (m.dim() == 3 and tuple(m.shape) != (N, h, w)):     # one mask for every frame
        m = m[None]
    hole = (m != 0).any(-1) if m.dim() == 4 else m != 0
    if hole.dim() != 3 or tuple(hole.shape[1:]) != (h, w) or hole.shape[0] not in (1, N):
        raise ValueError(f"composite_native: masks {given} do not match frames {tuple(fr.shape)}")
    M = hole.shape[0]
    shared = int(M == 1)
    k, r = native_window(h, w, imgH, imgW, frame_dilates)
    nbytes = lib.call("fgt_native_workspace", M, h, w, k)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    D = morph.binary_dilation(hole, r + 2 * k, device=dev)              # bool storage: one byte, 0 / 1
    lib.call("fgt_native_count", D, M, h, w, k, ws, nbytes, kernels=2)
    out = torch.empty_like(fr)
    lib.call("fgt_native_composite", cp, N, imgH, imgW, fr, h, w, C, shared, k, ws, nbytes, out)
    return out
