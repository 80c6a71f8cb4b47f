"""Device-side mask / resize glue of the driver (SURVEY 8f rank 3): the calls tool/video_inpainting.py makes to
scipy.ndimage (binary_dilation :551-556, binary_fill_holes :637) and cv2.resize (:268 flows, :546 masks) — and the
F.interpolate of the input frames (:478-483) — as batched kernels on tensors that stay on the GPU. Mask results are
bit-identical to the libraries'; the bilinear resize agrees to float32 rounding. No CPU fallback.
"""
import numpy as np
import torch

from . import lib


def _dev(device):
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("fgt_b200.morph runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    return dev


def _mask_u8(m, dev):
    t = torch.as_tensor(np.ascontiguousarray(m) if not torch.is_tensor(m) else m).to(dev)
    if t.dim() == 2:
        t = t[None]
    if t.dim() != 3:
        raise ValueError(f"mask batch {tuple(t.shape)} must be [B,H,W] (or [H,W])")
    return (t != 0).to(torch.uint8).contiguous()


def binary_dilation(masks, iterations=1, device=None):
    """scipy.ndimage.binary_dilation(m, iterations=n) for every image of [B,H,W] -> bool tensor [B,H,W] on the device."""
    dev = _dev(device)
    m = _mask_u8(masks, dev)
    if iterations < 1:
        raise ValueError("binary_dilation: iterations must be >= 1 (scipy's 'repeat until stable' mode is not used by the driver)")
    B, H, W = m.shape
    tmp, out = torch.empty_like(m), torch.empty_like(m)
    lib.call("fgt_binary_dilate", m, B, H, W, iterations, tmp, out, kernels=iterations)
    return out.bool()


def binary_fill_holes(masks, device=None, passes_per_check=3):
    """scipy.ndimage.binary_fill_holes(m) for every image of [B,H,W] -> bool tensor [B,H,W] on the device."""
    dev = _dev(device)
    m = _mask_u8(masks, dev)
    B, H, W = m.shape
    reach = torch.empty_like(m)
    changed = torch.zeros(1, dtype=torch.int32, device=dev)
    lib.call("fgt_fill_holes_init", m, B, H, W, reach, kernels=0)   # a memset
    for _ in range(H * W):                      # terminates: every pass but the last adds at least one pixel
        lib.call("fgt_fill_holes_pass", m, B, H, W, reach, changed, passes_per_check, kernels=2 * passes_per_check)
        if int(changed.item()) == 0:            # one host sync per group of passes
            break
    out = torch.empty_like(m)
    lib.call("fgt_fill_holes_finish", reach, B, H, W, out)
    return out.bool()


def resize_nearest(masks, size, device=None):
    """cv2.resize(m, dsize=(W', H'), interpolation=cv2.INTER_NEAREST) for uint8 [B,H,W] or [B,H,W,C]; size = (H', W')."""
    dev = _dev(device)
    t = torch.as_tensor(np.ascontiguousarray(masks) if not torch.is_tensor(masks) else masks).to(dev, torch.uint8).contiguous()
    squeeze = t.dim() == 3
    if squeeze:
        t = t[..., None]
    B, H, W, C = t.shape
    out = torch.empty(B, size[0], size[1], C, dtype=torch.uint8, device=dev)
    lib.call("fgt_resize_nearest_u8", t, B, H, W, C, size[0], size[1], out)
    return out[..., 0] if squeeze else out


def resize_bilinear(x, size, layout="nhwc", channel_scale=None, device=None):
    """Bilinear resize of float32 images to size = (H', W'): layout "nhwc" [B,H,W,C] follows cv2.resize(INTER_LINEAR)
    (the driver's flow resize; channel_scale = (sx, sy) multiplies channels 0 / 1 of the result like :266-267),
    layout "nchw" [B,C,H,W] follows F.interpolate(mode="bilinear", align_corners=False) (the frame resize, :478-483)."""
    dev = _dev(device)
    t = torch.as_tensor(np.ascontiguousarray(x) if not torch.is_tensor(x) else x).to(dev, torch.float32).contiguous()
    if t.dim() != 4:
        raise ValueError(f"resize_bilinear: {tuple(t.shape)} must be 4-D")
    nchw = layout == "nchw"
    B, H, W, C = (t.shape[0], t.shape[2], t.shape[3], t.shape[1]) if nchw else tuple(t.shape)
    out = torch.empty((B, C, size[0], size[1]) if nchw else (B, size[0], size[1], C), dtype=torch.float32, device=dev)
    s0, s1 = channel_scale if channel_scale is not None else (1.0, 1.0)
    lib.call("fgt_resize_bilinear_f32", t, B, H, W, C, size[0], size[1], 1 if nchw else 0, float(s0), float(s1), out)
    return out
