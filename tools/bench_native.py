"""Timing of the native-resolution output stage (fgt_b200/native.py): 80 frames of 1080x1920 from a 256x432 working size,
and 80 frames of 720x1280 at a working size of 720x1280 (s = 1), object masks from synth.pipeline_clip's generator
scaled up with cv2's nearest-neighbour resize, frame_dilates 0.

Device: the whole stage (hole, dilation r + 2k passes, counts, composite) between CUDA events on device-resident inputs
after warm-up, every round reported; the split between its kernels from torch.profiler in a separate run. Bytes are the
algorithmic bytes of each kernel computed from the shapes (uint8 masks, uint16 counts, 3-byte pixels), over the time,
against the H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth. Host: the same stage with cv2.resize, scipy's
binary_dilation, numpy box sums and blend on the pipeline's host pool (HOST_THREADS). The device output of the first
and last frame is checked against oracle/native_oracle.py. Prints a table and one JSON line."""
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np
import scipy.ndimage
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import native, pipeline as PL, synth  # noqa: E402
from oracle import native_oracle as NO  # noqa: E402

N = 80
HBM_BPS = 3.35e12
CASES = [("1080x1920_from_256x432", 1080, 1920, 256, 432), ("720x1280_at_720x1280", 720, 1280, 720, 1280)]


def inputs(h, w, imgH, imgW):
    # pipeline_clip's texture allows 25 frames of motion: four 20-frame clips
    parts = [synth.pipeline_clip(seed=7 + s, N=N // 4, H=imgH, W=imgW) for s in range(4)]
    comp = np.stack([f for fr, _ in parts for f in fr])
    masks = [m for _, ms in parts for m in ms]
    frames = np.stack([cv2.resize(c, (w, h), interpolation=cv2.INTER_LINEAR) for c in comp])
    masks = np.stack([cv2.resize(m, (w, h), interpolation=cv2.INTER_NEAREST) for m in masks])
    return comp, frames, masks


def stage_bytes(h, w, imgH, imgW, k, r):
    px = N * h * w
    return dict(hole=2 * px, dilate=(r + 2 * k) * 2 * px, count=5 * px,
                composite=px * (3 + 3 + 2) + N * imgH * imgW * 3)


def host_stage(comp, frames, masks, k, r):
    A = (2 * k + 1) ** 2
    out = np.empty_like(frames)
    h, w = frames.shape[1:3]

    def one(i):
        up = cv2.resize(comp[i], (w, h), interpolation=cv2.INTER_LINEAR).astype(np.int32)
        D = scipy.ndimage.binary_dilation(masks[i] != 0, iterations=r + 2 * k)
        c = NO.window_count(D, k).astype(np.int32)[..., None]
        out[i] = (c * up + (A - c) * frames[i] + A // 2) // A
    t0 = time.perf_counter()
    PL._per_frame(one, N)
    return time.perf_counter() - t0


def device_ms(comp, frames, masks, rounds):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    native.composite_native(comp, frames, masks, 0)                        # warm-up
    ms = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        ev[0].record()
        native.composite_native(comp, frames, masks, 0)
        ev[1].record()
        ev[1].synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
    return ms


def kernel_split(comp, frames, masks):
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        native.composite_native(comp, frames, masks, 0)
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        for key, name in (("dilate_cross_kernel", "dilate"), ("count_rows_kernel", "count"), ("count_cols_kernel", "count"),
                          ("composite_kernel", "composite")):
            if key in ev.key:
                split[name] = split.get(name, 0.0) + ev.device_time_total / 1e3
    other = sum(ev.device_time_total for ev in prof.key_averages()) / 1e3 - sum(split.values())
    split["hole"] = max(other, 0.0)                                         # the mask -> hole conversion (torch)
    return split


def main():
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 5
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip(), host_threads=PL.HOST_THREADS, cpu_count=os.cpu_count(), frames=N)
    print(f"{res['gpu']}; host pool {PL.HOST_THREADS} threads of {os.cpu_count()} CPUs; {N} frames")
    print(f"{'case':26s} {'device ms':>18s} {'GB':>6s} {'% HBM':>6s} {'composite ms':>13s} {'% HBM':>6s} {'host ms':>18s}")
    for name, h, w, imgH, imgW in CASES:
        comp, frames, masks = inputs(h, w, imgH, imgW)
        k, r = native.native_window(h, w, imgH, imgW, 0)
        dev = [torch.from_numpy(a).cuda() for a in (comp, frames, masks)]
        got = native.composite_native(*dev, 0).cpu().numpy()
        exact = all(np.array_equal(got[i], NO.composite_native(comp[i:i + 1], frames[i:i + 1], masks[i], 0)[0])
                    for i in (0, N - 1))
        ms = device_ms(*dev, rounds)
        split = kernel_split(*dev)
        host = [round(host_stage(comp, frames, masks, k, r) * 1e3, 1) for _ in range(max(2, rounds // 2))]
        nb = stage_bytes(h, w, imgH, imgW, k, r)
        best = min(ms)
        res[name] = dict(k=k, r=r, dilate_passes=r + 2 * k, device_stage_ms=[round(x, 3) for x in ms],
                         kernel_ms_profiler={a: round(b, 3) for a, b in split.items()}, bytes=nb,
                         stage_hbm_share=round(sum(nb.values()) / (best * 1e-3) / HBM_BPS, 3),
                         composite_hbm_share=round(nb["composite"] / (split["composite"] * 1e-3) / HBM_BPS, 3),
                         host_pool_ms=host, device_equals_oracle=bool(exact))
        e = res[name]
        print(f"{name:26s} {min(ms):8.2f}-{max(ms):8.2f} {sum(nb.values()) / 1e9:6.2f} {100 * e['stage_hbm_share']:5.1f}% "
              f"{split['composite']:13.3f} {100 * e['composite_hbm_share']:5.1f}% {min(host):8.1f}-{max(host):8.1f}")
        del dev
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
