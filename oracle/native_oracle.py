"""Native-resolution output of the pipeline (TEST INFRASTRUCTURE — the definition the device stage
fgt_b200/native.py / csrc/native.cu must equal byte for byte).

The network runs at the working size imgH x imgW; the user's frames are h x w. The stage upscales the pipeline's
working-resolution result `comp` to h x w and pastes it into the original frames inside a feathered band around the
mask, so that pixels far from the hole keep their original values:

    s = max(h / imgH, w / imgW),  k = ceil(s),  r = ceil(s * (frame_dilates + 2)) + 2
    D = scipy.ndimage.binary_dilation(hole, iterations = r + 2k)        (default cross, like the driver's dilations)
    c(y, x) = number of D pixels in the (2k+1) x (2k+1) window centred on (y, x);  A = (2k+1)^2
              (a window position outside the image counts as the nearest image pixel)
    up = bilinear resampling of comp to h x w in cv2's fixed-point INTER_LINEAR arithmetic (upscale below)
    out = (c * up + (A - c) * frame + A // 2) // A                          per channel, in integers

The L-infinity window of half-width k fits inside the L1 (cross) dilation of 2k, so c = A and out = up on every pixel
within L1 distance r of the hole; r bounds the native footprint of the working-resolution hole (the cv2-nearest resize
of the mask, dilated frame_dilates times: at most s * (frame_dilates + 2) native pixels from the hole, plus 2 for the
roundings of the two nearest-neighbour maps). Beyond L1 distance r + 4k, c = 0 and out is the original pixel. Both
hold at the image border too because the window replicates the edge: clamping a window position into the image moves
it towards the centre pixel. (Counting outside positions as 0 instead would blend the original frame, object included,
into hole pixels within k of the border.)
Everything is integer, so the device stage and this restatement agree bit for bit.
"""
import math

import numpy as np
import scipy.ndimage

COEF_BITS = 11                       # cv2's INTER_RESIZE_COEF_BITS: 8U weights are 11-bit fixed point


def native_window(h, w, imgH, imgW, frame_dilates):
    """(k, r) of the definition above for native size h x w and working size imgH x imgW."""
    s = max(h / imgH, w / imgW)
    return int(math.ceil(s)), int(math.ceil(s * (frame_dilates + 2))) + 2


def axis_coords(src, dst):
    """cv2 INTER_LINEAR's source index and 11-bit weights along one axis: x = float32((d + 0.5) * scale - 0.5) with the
    scale in double as cv2 computes it (1 / (dst / src)), i = floor(x), f = x - i; i < 0 -> (0, f = 0),
    i >= src - 1 -> (src - 1, f = 0). Returns (i0, i1, w0, w1), int64 arrays of length dst; w = round-half-even of
    2048 * (1 - f) and 2048 * f in float32."""
    scale = 1.0 / (dst / src)
    x = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    i = np.floor(x).astype(np.int64)
    f = (x - i.astype(np.float32)).astype(np.float32)
    low, high = i < 0, i >= src - 1
    i[low], f[low] = 0, 0
    i[high], f[high] = src - 1, 0
    one = np.float32(1 << COEF_BITS)
    w0 = np.rint(one * (np.float32(1) - f)).astype(np.int64)
    w1 = np.rint(one * f).astype(np.int64)
    return i, np.minimum(i + 1, src - 1), w0, w1


def upscale(comp, h, w):
    """comp uint8 [..., H, W, C] -> uint8 [..., h, w, C]: the horizontal pass exact in integers, the vertical pass
    rounded as cv2's vectorised 8U code does, (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2.
    Within 1 level of cv2.resize(comp, (w, h), interpolation=cv2.INTER_LINEAR)."""
    c = np.asarray(comp).astype(np.int64)
    H, W = c.shape[-3], c.shape[-2]
    x0, x1, a0, a1 = axis_coords(W, w)
    y0, y1, b0, b1 = axis_coords(H, h)
    rows = c[..., x0, :] * a0[:, None] + c[..., x1, :] * a1[:, None]           # [..., H, w, C]
    s0, s1 = rows[..., y0, :, :], rows[..., y1, :, :]                           # [..., h, w, C]
    v = (((b0[:, None, None] * (s0 >> 4)) >> 16) + ((b1[:, None, None] * (s1 >> 4)) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def window_count(D, k):
    """c: the number of set pixels of D [..., h, w] in the (2k+1) x (2k+1) window around every pixel, a window position
    outside the image counting as the nearest image pixel (edge replication)."""
    d = np.asarray(D).astype(np.int64)
    pad = [(0, 0)] * (d.ndim - 2) + [(k, k), (k, k)]
    cs = np.pad(np.pad(d, pad, mode="edge"), [(0, 0)] * (d.ndim - 2) + [(1, 0), (1, 0)]).cumsum(-1).cumsum(-2)
    n = 2 * k + 1
    return cs[..., n:, n:] - cs[..., :-n, n:] - cs[..., n:, :-n] + cs[..., :-n, :-n]


def counts(hole, h, w, imgH, imgW, frame_dilates):
    """(c, A) for bool holes [M, h, w]."""
    k, r = native_window(h, w, imgH, imgW, frame_dilates)
    D = np.stack([scipy.ndimage.binary_dilation(x, iterations=r + 2 * k) for x in hole])
    return window_count(D, k), (2 * k + 1) ** 2


def composite_native(comp, frames, masks, frame_dilates):
    """comp uint8 [N, imgH, imgW, 3], frames uint8 [N, h, w, 3], masks [N, h, w] / [N, h, w, C] per frame or one
    [h, w] / [h, w, C] for every frame (non-zero in any channel = hole) -> uint8 [N, h, w, 3]."""
    comp, frames = np.asarray(comp), np.asarray(frames)
    N, h, w, _ = frames.shape
    imgH, imgW = comp.shape[1:3]
    m = np.asarray(masks)
    if m.ndim == 3 and m.shape != (N, h, w):             # one colour mask
        m = m[None]
    elif m.ndim == 2:
        m = m[None]
    hole = (m != 0).any(-1) if m.ndim == 4 else m != 0
    c, A = counts(hole, h, w, imgH, imgW, frame_dilates)
    c = np.broadcast_to(c, (N, h, w))[..., None]
    up = upscale(comp, h, w).astype(np.int64)
    out = (c * up + (A - c) * frames.astype(np.int64) + A // 2) // A
    return out.astype(np.uint8)
