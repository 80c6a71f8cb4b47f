"""Oracle of the flow warping error (TEST INFRASTRUCTURE — see oracle/fgt_oracle.py; kernel: csrc/warp_error.cu).

Restates the reference's `image_warp` and `fbConsistencyCheck` (FGT/models/utils/fbConsistencyCheck.py:8-48; the copy
under LAFC/ is identical) as explicit float32 operations, with the one documented departure: the bilinear sample is
grid_sample's align_corners=True form, the convention the reference's linspace grid is built for. Step by step:
  - grid: np.linspace(-1, 1, n), i.e. i * (2 / (n - 1)) - 1 in float64 with the last point set to 1, cast to float32;
  - the flow divided by s = (n - 1) / 2 (a float32 division), added to the grid;
  - unnormalised as ATen's align-corners grid sampler does, (g + 1) * s, then floor, the distances w = x - floor(x),
    e = 1 - w (likewise n, s along y) and the weights nw = s*e, ne = s*w, sw = n*e, se = n*w;
  - the sum as ATen's vectorised CPU sampler computes it: nw_v*nw rounded, then three fused multiply-adds with
    ne_v*ne, sw_v*sw and se_v*se, with zero for corners outside the image (its AVX2 / AVX-512 code is compiled with FMA
    contraction, and the golden pins that order);
  - length_sq and the occlusion test |F + B(x+F)|^2 > 0.01 * (|F|^2 + |B(x+F)|^2) + 0.5, each operation in float32.
Every other operation is a single rounded float32 operation, on the CPU or on a CUDA device, and fma32 is exact on
both, so the results are the same on both. Pinned by tests/golden/warp_error.npz (outputs of the unmodified reference
functions on the CPU).

The score composes these in float64: per pair t, e_t = sum_x M(x) sum_c (I_t - W_t)^2 / sum_x M(x), and e_hole_t the
same restricted to M * hole_t; an empty mask gives NaN, which is left out of the clip's mean."""
import numpy as np
import torch

ALPHA1, ALPHA2 = 0.01, 0.5


def linspace32(n):
    """np.linspace(-1, 1, n).astype(float32), restated: float64 i * step - 1, the last point exactly 1."""
    y = np.arange(n, dtype=np.float64) * (2.0 / (n - 1)) + -1.0
    y[-1] = 1.0
    return y.astype(np.float32)


def _f32(v, like):
    """A float32 0-dim tensor on like's device: dividing by it is a true division on CUDA too (not x * (1 / v))."""
    return torch.tensor(v, dtype=torch.float32, device=like.device)


def fma32(a, b, c):
    """Correctly rounded float32 a * b + c: the float64 product is exact, the float64 sum is rounded to odd (exact when
    its error is zero, else the neighbour with an odd last bit), and a round-to-odd float64 rounds to float32 as the
    exact value would."""
    p = a.double() * b.double()
    c = c.double()
    s = p + c
    bb = s - p
    t = (p - (s - bb)) + (c - bb)                          # s + t == p + c exactly (TwoSum)
    even = (s.view(torch.int64) & 1) == 0
    s = torch.where((t != 0) & even, torch.nextafter(s, torch.where(t > 0, s + 1, s - 1)), s)
    return s.float()


def image_warp(image, flow):
    """image [b,c,h,w], flow [b,2,h,w] float32 (pixels, x first) -> [b,c,h,w] float32: image sampled at x + flow."""
    b, c, h, w = image.shape
    dev = image.device
    sx, sy = _f32((w - 1.0) / 2.0, flow), _f32((h - 1.0) / 2.0, flow)
    gx = torch.from_numpy(linspace32(w)).to(dev).view(1, 1, w)
    gy = torch.from_numpy(linspace32(h)).to(dev).view(1, h, 1)
    x = (gx + flow[:, 0] / sx + 1.0) * sx
    y = (gy + flow[:, 1] / sy + 1.0) * sy
    x0, y0 = torch.floor(x), torch.floor(y)
    wd = x - x0
    ed = 1.0 - wd
    nd = y - y0
    sd = 1.0 - nd
    flat = image.reshape(b, c, h * w)
    out = None
    for wgt, xs, ys in ((sd * ed, x0, y0), (sd * wd, x0 + 1, y0), (nd * ed, x0, y0 + 1), (nd * wd, x0 + 1, y0 + 1)):
        ok = (xs >= 0) & (xs < w) & (ys >= 0) & (ys < h)
        idx = torch.where(ok, ys * w + xs, torch.zeros_like(xs)).long().reshape(b, 1, h * w).expand(b, c, h * w)
        v = torch.where(ok.view(b, 1, h, w), torch.gather(flat, 2, idx).view(b, c, h, w), torch.zeros((), device=dev))
        wgt = wgt.view(b, 1, h, w).expand(b, c, h, w)
        out = v * wgt if out is None else fma32(v, wgt, out)
    return out


def length_sq(x):
    return x[:, 0:1] * x[:, 0:1] + x[:, 1:2] * x[:, 1:2]


def fb_occlusion(flow_fw, flow_bw, alpha1=ALPHA1, alpha2=ALPHA2):
    """fbConsistencyCheck's first output: [b,1,h,w] float32, 1 where the forward flow fails the check."""
    bw_warped = image_warp(flow_bw, flow_fw)
    diff = flow_fw + bw_warped
    thresh = alpha1 * (length_sq(flow_fw) + length_sq(bw_warped)) + alpha2
    return (length_sq(diff) > thresh).float()


def normalise(frames):
    """float32 [N,H,W,C] frames (uint8 or float32 on 0..255) -> float32 [N,C,H,W] I = V / 255."""
    v = torch.as_tensor(np.asarray(frames)).float()
    return (v / _f32(255.0, v)).permute(0, 3, 1, 2)


def pair_maps(frames, flows_f, flows_b):
    """(warped [P,C,H,W] float32 = frame t+1 brought to frame t, valid [P,H,W] float32 = 1 - occlusion) of every pair,
    on the device of flows_f."""
    f = torch.as_tensor(flows_f)
    img = normalise(frames).to(f.device)
    warped = image_warp(img[1:], f)
    valid = 1.0 - fb_occlusion(f, torch.as_tensor(flows_b).to(f.device))[:, 0]
    return warped, valid


def pair_sums(frames, warped, valid, masks=None):
    """float64 [P,4]: (sum M*err, sum M, sum M*hole*err, sum M*hole) per pair, err = sum_c (I_t - W_t)^2 with each
    float32 value cast to float64 first; the hole columns are 0 without masks. warped [P,C,H,W], valid [P,H,W]."""
    it = normalise(frames)[:-1].double().cpu().numpy()
    err = ((it - torch.as_tensor(warped).double().cpu().numpy()) ** 2).sum(axis=1)
    m = torch.as_tensor(valid).double().cpu().numpy()
    out = np.zeros((m.shape[0], 4))
    out[:, 0] = (m * err).sum(axis=(1, 2))
    out[:, 1] = m.sum(axis=(1, 2))
    if masks is not None:
        hole = (np.asarray(masks)[:-1] != 0).astype(np.float64)
        out[:, 2] = (m * hole * err).sum(axis=(1, 2))
        out[:, 3] = (m * hole).sum(axis=(1, 2))
    return out


def report(sums, masks=True):
    """The report of per-pair sums [P,4]: per-pair errors (NaN for an empty mask), their means over the pairs that
    have one, and those pairs' counts."""
    sums = np.asarray(sums, np.float64)
    res = {}
    for key, col in (("ewarp", 0), ("ewarp_hole", 2)):
        if key == "ewarp_hole" and not masks:
            continue
        with np.errstate(invalid="ignore", divide="ignore"):
            per = np.where(sums[:, col + 1] > 0, sums[:, col] / sums[:, col + 1], np.nan)
        ok = ~np.isnan(per)
        res[key] = float(np.mean(per[ok])) if ok.any() else float("nan")
        res[f"{key}_pairs"] = int(ok.sum())
        res[f"per_pair_{key}"] = per
    return res


def warp_error(frames, flows_f, flows_b, masks=None):
    """The whole score on the oracle's own maps (see report)."""
    warped, valid = pair_maps(frames, flows_f, flows_b)
    return report(pair_sums(frames, warped, valid, masks), masks is not None)
