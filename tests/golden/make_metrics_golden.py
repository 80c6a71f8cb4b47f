"""Writes metrics.npz: the reference's own quality metrics of seeded frame pairs (tests/test_metrics.py CASES).

    python tests/golden/make_metrics_golden.py

Runs the UNMODIFIED FGT/metrics/psnr.py and ssim.py of a reference checkout (REF, as in make_golden.py), each loaded
on its own by file path: the package's __init__.py imports skimage, which these two do not need. L1 and L2 are
calculate_metrics' expressions (FGT/metrics/__init__.py:17-19). Every input is converted to float64 before it reaches
the reference, which is the project's definition (psnr.py would otherwise subtract uint8 arrays with wrap-around).
Only the outputs are stored; the inputs are regenerated from their seeds.
"""
import importlib.util
import os
import sys

import numpy as np

REF = "/root/reference/FGT/metrics"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.test_metrics import CASES, GOLDEN, case_inputs  # noqa: E402


def _load(name):
    spec = importlib.util.spec_from_file_location(f"ref_metrics_{name}", os.path.join(REF, f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference(results, gts):
    psnr, ssim = _load("psnr").psnr, _load("ssim")
    out = {k: [] for k in ("l1", "l2", "psnr", "ssim", "ssim_channels")}
    for r, g in zip(results.astype(np.float64), gts.astype(np.float64)):
        H, W, C = r.shape
        residual = r - g
        out["l1"].append(np.mean(np.abs(residual)))
        out["l2"].append(np.sum(residual ** 2) ** 0.5 / (H * W * C))
        out["psnr"].append(psnr(r, g))
        out["ssim"].append(ssim.ssim(r, g))
        out["ssim_channels"].append([ssim.calculate_ssim(r[:, :, c], g[:, :, c]) for c in range(C)])
    return {k: np.array(v, dtype=np.float64) for k, v in out.items()}


if __name__ == "__main__":
    arrs = {}
    for name in CASES:
        for k, v in reference(*case_inputs(name)).items():
            arrs[f"{name}/{k}"] = v
        print(name, {k: arrs[f"{name}/{k}"][:2].tolist() for k in ("psnr", "ssim")})
    np.savez_compressed(GOLDEN, **arrs)
