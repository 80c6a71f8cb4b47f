"""Quality metrics of inpainted clips against ground truth on the GPU: the reference's PSNR (FGT/metrics/psnr.py), its
MATLAB-style Gaussian SSIM (FGT/metrics/ssim.py) and the L1 / L2 errors of FGT/metrics/__init__.py calculate_metrics,
for every frame of a clip in one batched launch pair (csrc/metrics.cu; definition: oracle/metrics_oracle.py).

Inputs are uint8 or float32 on the 0..255 scale and are converted to float64 before any arithmetic. Unlike psnr.py and
calculate_metrics handed uint8 arrays, a difference therefore never wraps around modulo 256. Frames smaller than the
11x11 SSIM window raise ValueError (the reference returns NaN). There is no CPU fallback.

    python -m fgt_b200.metrics --result out/frames --gt gt_frames [--gpu N]     # one JSON object on stdout
"""
import argparse
import json
import sys

import numpy as np
import torch

from . import lib

KEYS = ("l1", "l2", "psnr", "ssim")       # calculate_metrics' keys, in the order of the kernel's output columns
WORKSPACE_BUDGET = 1 << 30                # bytes of device copies and workspace per launch; longer clips run in chunks
_DTYPES = {torch.uint8: lib.METRIC_U8, torch.float32: lib.METRIC_F32}


def _clip(x, what):
    t = x if torch.is_tensor(x) else torch.as_tensor(np.ascontiguousarray(x))
    if t.dtype not in _DTYPES:
        raise TypeError(f"frame_metrics: {what} must be uint8 or float32, got {t.dtype}")
    return t


def frame_metrics(results, gts, device=None):
    """results, gts: [N,H,W,C] clips (numpy arrays or tensors, uint8 or float32, C = 1 or 3, H and W >= 11) on the
    0..255 scale. Returns calculate_metrics' dict: the clip means under 'l1', 'l2', 'psnr', 'ssim' (floats), and under
    'per_frame' the float64 arrays [N] of each metric plus 'ssim_channels' [N,C], the SSIM of each channel.
    Runs on `device` (default: the inputs' CUDA device, else the current one)."""
    a, b = _clip(results, "results"), _clip(gts, "gts")
    if a.dim() != 4 or tuple(a.shape) != tuple(b.shape):
        raise ValueError(f"frame_metrics: results {tuple(a.shape)} and gts {tuple(b.shape)} must be [N,H,W,C] of one shape")
    N, H, W, C = a.shape
    if N == 0 or C not in (1, 3):
        raise ValueError(f"frame_metrics: clips {tuple(a.shape)} need N >= 1 and C = 1 or 3")
    if H < 11 or W < 11:
        raise ValueError(f"frame_metrics: frames of {H}x{W} are smaller than the 11x11 SSIM window")
    if device is None:
        dev = a.device if a.is_cuda else b.device if b.is_cuda else None
    else:
        dev = torch.device(device)
    if dev is None:
        if not torch.cuda.is_available():
            raise RuntimeError("fgt_b200.metrics runs on a CUDA (sm_90a) device only; there is no CPU fallback")
        dev = torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("fgt_b200.metrics runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    per_ws = lib.call("fgt_metrics_workspace", 1, H, W, C)
    per_frame = H * W * C * (a.element_size() + b.element_size()) + per_ws
    chunk = max(1, min(N, 65535 // C, WORKSPACE_BUDGET // per_frame))
    with torch.cuda.device(dev):
        out = torch.empty(N, 4, dtype=torch.float64, device=dev)
        per_c = torch.empty(N, C, dtype=torch.float64, device=dev)
        ws = torch.empty(chunk * per_ws, dtype=torch.uint8, device=dev)
        for s in range(0, N, chunk):
            e = min(N, s + chunk)
            ca, cb = a[s:e].to(dev).contiguous(), b[s:e].to(dev).contiguous()
            lib.call("fgt_metrics", ca, _DTYPES[a.dtype], cb, _DTYPES[b.dtype], e - s, H, W, C, ws, ws.numel(), out[s:e],
                     per_c[s:e], kernels=2)
        vals, chans = out.cpu().numpy(), per_c.cpu().numpy()
    res = {k: float(np.mean(vals[:, j])) for j, k in enumerate(KEYS)}
    res["per_frame"] = {k: vals[:, j].copy() for j, k in enumerate(KEYS)}
    res["per_frame"]["ssim_channels"] = chans
    return res


def _parser():
    p = argparse.ArgumentParser(prog="python -m fgt_b200.metrics",
                                description="PSNR, SSIM, L1 and L2 of result frames against ground-truth frames, as "
                                            "FGT/metrics defines them, computed on the GPU; prints one JSON object")
    p.add_argument("--result", required=True, help="directory of result frames (*.png / *.jpg), e.g. the pipeline's "
                                                   "OUTROOT/frames")
    p.add_argument("--gt", required=True, help="directory of ground-truth frames, in the same order")
    p.add_argument("--gpu", type=int, default=0, help="CUDA device index")
    return p


def main(argv=None):
    """The command line: returns the dict it prints (per-frame values as lists)."""
    from . import io
    p = _parser()
    args = p.parse_args(argv)
    res, gt = io.read_frames(args.result), io.read_frames(args.gt)
    if len(res) != len(gt):
        p.error(f"{args.result} holds {len(res)} frames and {args.gt} holds {len(gt)}")
    for i, (r, g) in enumerate(zip(res, gt)):
        if r.shape != g.shape:
            p.error(f"frame {i}: result {r.shape} and ground truth {g.shape} differ in size")
    if len({r.shape for r in res}) != 1:
        p.error(f"{args.result}: frames of different sizes")
    m = frame_metrics(np.stack(res), np.stack(gt), device=f"cuda:{args.gpu}")
    out = {"frames": len(res), **{k: m[k] for k in KEYS},
           "per_frame": {k: v.tolist() for k, v in m["per_frame"].items()}}
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main(sys.argv[1:])
