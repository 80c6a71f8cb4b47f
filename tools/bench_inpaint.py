"""TELEA timing: cv2.inpaint on the pipeline's host pool (HOST_THREADS) against the device kernels (fgt_b200/inpaint.py)
at the driver's three call sites, N = 80 frames: prepare_gradients and blend_frames at 256x432 with per-frame object
masks, extrapolate with the shared border mask of the 2x canvas (the clip at 256x432 in 512x864), and object masks at
1280x720. Rounds alternate host and device; every round's time is reported, with the spread. Device: plan and fill
times from CUDA events on device-resident inputs, the split of the plan into its two serial kernels (fast marches,
levels) from torch.profiler in a separate run, and the whole call (uint8 in and out of host memory) from a synchronised
host clock.
Outputs are checked byte for byte against cv2. Prints one JSON line."""
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import inpaint, pipeline as PL  # noqa: E402

N = 80


def object_masks(g, N, H, W):
    m = np.zeros((N, H, W), np.uint8)
    for b in range(N):
        cx, cy = int(W * (0.3 + 0.4 * b / N)), int(H * 0.5)
        cv2.ellipse(m[b], (cx, cy), (int(W * 0.1), int(H * 0.15)), 15.0, 0, 360, 1, -1)
        m[b] = cv2.dilate(m[b], np.ones((9, 9), np.uint8))
    return m


def cases(g):
    fr = g.integers(0, 256, (N, 256, 432, 3), dtype=np.uint8)
    fr = np.stack([cv2.GaussianBlur(f, (0, 0), 2) for f in fr])
    yield "object_256x432", fr, object_masks(g, N, 256, 432)
    ring = np.ones((512, 864), np.uint8)
    ring[128:384, 216:648] = 0
    big = np.zeros((N, 512, 864, 3), np.uint8)
    big[:, 128:384, 216:648] = fr
    yield "extrapolation_512x864", big, ring
    hd = np.stack([cv2.GaussianBlur(g.integers(0, 256, (720, 1280, 3), dtype=np.uint8), (0, 0), 2) for _ in range(N)])
    yield "object_1280x720", hd, object_masks(g, N, 720, 1280)


def host_pool(fr, mk):
    out = [None] * len(fr)

    def one(i):
        out[i] = cv2.inpaint(fr[i], mk[i] if mk.ndim == 3 else mk, 3, cv2.INPAINT_TELEA)
    t0 = time.perf_counter()
    PL._per_frame(one, len(fr))
    return time.perf_counter() - t0, np.stack(out)


def device(fr, mk):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = inpaint.inpaint_telea(fr, mk).cpu().numpy()
    return time.perf_counter() - t0, out


def kernel_times(fr, mk, rounds):
    x, m = torch.from_numpy(fr).cuda(), torch.from_numpy(np.ascontiguousarray(mk)).cuda()
    inpaint.inpaint_telea(x, m)
    plan, fill = [], []
    for _ in range(rounds):                                             # CUDA events around the plan and the fill
        t = {}
        inpaint.inpaint_telea(x, m, timing=t)
        plan.append(round(t["plan_ms"], 2))
        fill.append(round(t["fill_ms"], 2))
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        inpaint.inpaint_telea(x, m)
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        for k in ("march_kernel", "levels_kernel"):
            if k in ev.key:
                split[k] = round(ev.device_time_total / 1e3 / max(ev.count, 1), 2)
    return dict(plan_ms_events=plan, fill_ms_events=fill, plan_split_ms_profiler=split)


def main():
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 3
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip(), host_threads=PL.HOST_THREADS, cpu_count=os.cpu_count(), frames=N)
    g = np.random.default_rng(0)
    for name, fr, mk in cases(g):
        device(fr[:2], mk if mk.ndim == 2 else mk[:2])                     # warm-up
        hs, ds, same = [], [], True
        for _ in range(rounds):
            th, ref = host_pool(fr, mk)
            td, got = device(fr, mk)
            hs.append(round(th * 1e3, 2))
            ds.append(round(td * 1e3, 2))
            same = same and np.array_equal(ref, got)
        hole = int((mk != 0).sum()) if mk.ndim == 3 else int((mk != 0).sum()) * N
        res[name] = dict(hole_px_total=hole, host_pool_ms=hs, device_call_ms=ds,
                         host_spread_ms=round(max(hs) - min(hs), 2), device_spread_ms=round(max(ds) - min(ds), 2),
                         device=kernel_times(fr, mk, rounds), h2d_bytes=int(fr.nbytes + mk.nbytes),
                         d2h_bytes=int(fr.nbytes), bytes_identical_to_cv2=bool(same))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
