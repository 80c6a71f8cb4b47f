"""cv2.inpaint(..., cv2.INPAINT_TELEA) on the device, byte-identical to OpenCV, and the driver's gradient preparation
around it (tool/video_inpainting.py:583-614) as device kernels. TELEA is a sequential fast-marching method, but its
fill order, distances and weights depend on the mask alone: the kernels plan every distinct mask once (serially, one
CTA per mask) and then fill every image level by level in parallel (csrc/inpaint.cu). No CPU fallback.
"""
import numpy as np
import torch

from . import lib

WORKSPACE_BUDGET = 1 << 30     # bytes of plan workspace per launch; larger batches of distinct masks run in chunks


def _dev(device):
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("fgt_b200.inpaint runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    return dev


def _u8(x, dev):
    t = torch.as_tensor(np.ascontiguousarray(x) if not torch.is_tensor(x) else x)
    if t.dtype != torch.uint8 and t.dtype != torch.bool:
        raise TypeError(f"inpaint_telea: uint8 images / masks expected, got {t.dtype}")
    return t.to(dev, torch.uint8).contiguous()


def inpaint_telea(images, masks, radius=3, device=None, timing=None):
    """cv2.inpaint(img, mask, radius, cv2.INPAINT_TELEA) for a batch [B,H,W,C] or one image [H,W,C] / [H,W] of uint8
    (C = 1 or 3). masks: uint8 or bool [B,H,W], or one [H,W] mask for every image (planned once); non-zero = hole.
    The radius must round to 3, the driver's and the only radius verified byte-identical (others raise).
    Returns a uint8 tensor of the images' shape on the device. `timing`: a dict that receives the plan and fill times
    in ms from CUDA events (synchronises)."""
    dev = _dev(device)
    img = _u8(images, dev)
    single = img.dim() < 4
    if img.dim() == 2:
        img = img[None, :, :, None]
    elif img.dim() == 3:
        img = img[None]
    if img.dim() != 4:
        raise ValueError(f"inpaint_telea: images {tuple(img.shape)} must be [B,H,W,C], [H,W,C] or [H,W]")
    B, H, W, C = img.shape
    m = _u8(masks, dev)
    if m.dim() == 3 and m.shape[0] == 1:
        m = m[0]
    if m.dim() == 2:
        if tuple(m.shape) != (H, W):
            raise ValueError(f"inpaint_telea: mask {tuple(m.shape)} does not match images {tuple(img.shape)}")
        stride = 0
    elif m.dim() == 3 and tuple(m.shape) == (B, H, W):
        stride = H * W
    else:
        raise ValueError(f"inpaint_telea: masks {tuple(m.shape)} must be [H,W] or [B,H,W] for images {tuple(img.shape)}")
    per_mask = lib.call("fgt_inpaint_telea_workspace", 1, H, W)
    out = torch.empty_like(img)
    chunk = B if stride == 0 else max(1, min(B, WORKSPACE_BUDGET // per_mask))
    ws = torch.empty(per_mask * (1 if stride == 0 else chunk), dtype=torch.uint8, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)] if timing is not None else None
    plan_ms = fill_ms = 0.0
    for s in range(0, B, chunk):
        e = min(B, s + chunk)
        if ev:
            ev[0].record()
        lib.call("fgt_inpaint_telea_plan", m.data_ptr() + s * stride, 1 if stride == 0 else e - s, H, W, float(radius),
                 ws, ws.numel(), kernels=2)                # marches + levels
        if ev:
            ev[1].record()
        lib.call("fgt_inpaint_telea_fill", img[s], e - s, H, W, C, 1 if stride == 0 else 0, float(radius), ws, ws.numel(),
                 out[s])
        if ev:
            ev[2].record()
            ev[2].synchronize()
            plan_ms += ev[0].elapsed_time(ev[1])
            fill_ms += ev[1].elapsed_time(ev[2])
    if timing is not None:
        timing["plan_ms"] = timing.get("plan_ms", 0.0) + plan_ms
        timing["fill_ms"] = timing.get("fill_ms", 0.0) + fill_ms
    if single:
        out = out[0] if images.ndim == 3 else out[0, :, :, 0]
    return out


def inpaint_telea_host(image, mask, radius=3):
    """The same algorithm (radius 3 only) for one uint8 image [H,W] / [H,W,C] on the CPU (fgt_inpaint_telea_host) — a
    verification tool for machines without a GPU, not a fallback: nothing on the product path calls it."""
    img = np.ascontiguousarray(image, dtype=np.uint8)
    m = np.ascontiguousarray(np.asarray(mask) != 0, dtype=np.uint8)
    if img.ndim not in (2, 3) or m.shape != img.shape[:2]:
        raise ValueError(f"inpaint_telea_host: image {img.shape} / mask {m.shape} must be [H,W(,C)] / [H,W]")
    out = np.empty_like(img)
    C = 1 if img.ndim == 2 else img.shape[2]
    lib.call("fgt_inpaint_telea_host", img.ctypes.data, m.ctypes.data, img.shape[0], img.shape[1], C, float(radius),
             out.ctypes.data)
    return out


def prepare_gradients(video, mask, mask_dilated, device=None):
    """The device form of pipeline.prepare_gradients: video [H,W,3,N] float32 (BGR, 0..1), mask / mask_dilated [H,W,N]
    bool -> (gx, gy) [H,W,3,N] float32, stored frame-major. Zeroes the hole of `video` in place like the driver.
    Bit-identical to the host stage (float32 *255 -> uint8, TELEA radius 3, /255, forward differences)."""
    dev = _dev(device)
    video = np.asarray(video)
    if video.dtype != np.float32 or video.ndim != 4 or video.shape[2] != 3:
        raise ValueError(f"prepare_gradients: video {video.shape} {video.dtype} must be float32 [H,W,3,N]")
    H, W, _, N = video.shape
    frames = np.moveaxis(video, -1, 0)                                   # [N,H,W,3] (a view)
    hole = np.ascontiguousarray(np.moveaxis(np.asarray(mask), -1, 0)).astype(bool)
    v = torch.from_numpy(np.ascontiguousarray(frames)).to(dev)
    m = torch.from_numpy(hole).to(dev).to(torch.uint8)
    md = torch.from_numpy(np.ascontiguousarray(np.moveaxis(np.asarray(mask_dilated), -1, 0)).astype(np.uint8)).to(dev)
    u8 = torch.empty((N, H, W, 3), dtype=torch.uint8, device=dev)
    lib.call("fgt_grad_prep_pre", v, m, N, H, W, u8)
    filled = inpaint_telea(u8, m, 3, device=dev)
    gx = torch.empty((N, H, W, 3), dtype=torch.float32, device=dev)
    gy = torch.empty_like(gx)
    lib.call("fgt_grad_prep_post", filled, md, N, H, W, gx, gy)
    frames[hole] = 0                                                     # :592, in place
    return np.moveaxis(gx.cpu().numpy(), 0, -1), np.moveaxis(gy.cpu().numpy(), 0, -1)
