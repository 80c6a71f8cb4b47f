"""Quality metrics of inpainted frames against ground truth (TEST INFRASTRUCTURE — the definition that
fgt_b200/metrics.py / csrc/metrics.cu are checked against; nothing under fgt_b200/ imports it).

Restates, in float64 numpy, the reference's FGT/metrics:
    psnr.py:5-10      mse = mean((a - b)^2); 100 if mse == 0 else 20 log10(255 / sqrt(mse))
    ssim.py:5-25      calculate_ssim: w = g g^T with g = cv2.getGaussianKernel(11, 1.5) (:11-12); mu = w * x at the
                      valid positions [5:-5, 5:-5] (:14-15); sigma1^2 = w * a^2 - mu1^2, sigma2^2 = w * b^2 - mu2^2,
                      sigma12 = w * ab - mu1 mu2 (:16-21); the map ((2 mu1 mu2 + C1)(2 sigma12 + C2)) /
                      ((mu1^2 + mu2^2 + C1)(sigma1^2 + sigma2^2 + C2)) with C1 = (0.01*255)^2, C2 = (0.03*255)^2
                      (:6-7, :23-24), averaged (:25)
    ssim.py:28-46     ssim: one plane for [H,W] or [H,W,1], the mean of the three planes' SSIM for [H,W,3]
    __init__.py:9-31  calculate_metrics: L1 = mean|a - b|, L2 = sqrt(sum (a - b)^2) / (H*W*C) per frame (:17-19),
                      and the means over the frames under the keys l1, l2, psnr, ssim (:26-31)
The 11x11 correlation is a direct float64 sum (scipy.ndimage.correlate; the border mode never reaches the valid
positions) where ssim.py calls cv2.filter2D; the two agree to about 1e-13 on the 0..255 scale.

Two deliberate differences: inputs are converted to float64 before any arithmetic (psnr.py and calculate_metrics
subtract uint8 arrays with wrap-around when handed uint8), and frames smaller than the 11x11 window raise ValueError
(the reference averages an empty map and returns NaN).
"""
import math

import cv2
import numpy as np
import scipy.ndimage

KEYS = ("l1", "l2", "psnr", "ssim")
RADIUS = 5
C1 = (0.01 * 255) ** 2
C2 = (0.03 * 255) ** 2


_WINDOW = np.outer(cv2.getGaussianKernel(11, 1.5), cv2.getGaussianKernel(11, 1.5).T)      # ssim.py:11-12


def _valid(x):
    return scipy.ndimage.correlate(x, _WINDOW, mode="constant")[RADIUS:-RADIUS, RADIUS:-RADIUS]


def ssim_plane(a, b):
    """calculate_ssim for one [H,W] plane pair (any real dtype; converted to float64)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    mu1, mu2 = _valid(a), _valid(b)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 ** 2, mu2 ** 2, mu1 * mu2
    sigma1_sq = _valid(a ** 2) - mu1_sq
    sigma2_sq = _valid(b ** 2) - mu2_sq
    sigma12 = _valid(a * b) - mu1_mu2
    ssim_map = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))
    return ssim_map.mean()


def check_pair(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        raise ValueError(f"metrics: result {a.shape} and ground truth {b.shape} differ in shape")
    if a.ndim != 3 or a.shape[2] not in (1, 3):
        raise ValueError(f"metrics: frames {a.shape} must be [H,W,C] with C = 1 or 3")
    if a.shape[0] < 11 or a.shape[1] < 11:
        raise ValueError(f"metrics: frames of {a.shape[0]}x{a.shape[1]} are smaller than the 11x11 SSIM window")
    return a.astype(np.float64), b.astype(np.float64)


def frame_metrics(a, b):
    """(l1, l2, psnr, ssim, per-channel ssim) of one [H,W,C] frame pair."""
    a, b = check_pair(a, b)
    H, W, C = a.shape
    d = a - b
    mse = np.mean(d ** 2)
    psnr = 100.0 if mse == 0 else 20 * math.log10(255.0 / math.sqrt(mse))
    per = np.array([ssim_plane(a[:, :, c], b[:, :, c]) for c in range(C)])
    return np.mean(np.abs(d)), np.sum(d ** 2) ** 0.5 / (H * W * C), float(psnr), float(per.mean() if C == 3 else per[0]), per


def clip_metrics(results, gts, map_fn=map):
    """calculate_metrics over [N,H,W,C] clips, in the layout of fgt_b200.metrics.frame_metrics: the clip means under
    'l1', 'l2', 'psnr', 'ssim', and under 'per_frame' the float64 arrays [N] of each metric plus 'ssim_channels' [N,C].
    `map_fn` maps the per-frame function over the frame indices (a thread pool's map spreads them over host threads)."""
    results, gts = np.asarray(results), np.asarray(gts)
    if results.shape != gts.shape or results.ndim != 4:
        raise ValueError(f"metrics: clips {results.shape} / {gts.shape} must both be [N,H,W,C]")
    rows = list(map_fn(lambda i: frame_metrics(results[i], gts[i]), range(len(results))))
    per = {k: np.array([r[j] for r in rows], dtype=np.float64) for j, k in enumerate(KEYS)}
    per["ssim_channels"] = np.stack([r[4] for r in rows])
    return {**{k: float(np.mean(per[k])) for k in KEYS}, "per_frame": per}
