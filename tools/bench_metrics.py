"""Timing of clip scoring (fgt_b200/metrics.py: PSNR, SSIM, L1, L2 of every frame) on the GPU against the float64
oracle (oracle/metrics_oracle.py, numpy + scipy) on the pipeline's host pool (HOST_THREADS), for 80 uint8 RGB frames
at the driver's 256x432 and at 720x1280.

Device: frame_metrics between CUDA events, once from host numpy arrays (the host-to-device copies included, which is
what a caller holding frames on the host pays) and once from device-resident tensors; host: the oracle under a
wall clock. After a warm-up of both, the paths alternate for --rounds rounds and every round is reported. The split
between the two kernels comes from one torch.profiler session after the timed rounds. FLOPs and bytes are the
algorithm's, computed from the shapes (ALG_FLOPS per valid position and channel, RESID_FLOPS per pixel and channel;
each input byte read once), over the time of one fgt_metrics call (both kernels, CUDA events over 20 calls), against
the H100 SXM data sheet (34 TFLOP/s FP64 without tensor cores, 3.35 TB/s HBM3). The card's name and power limit are read in the same run. Prints a table and one JSON line."""
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import lib, metrics as M, pipeline as PL, synth  # noqa: E402
from oracle import metrics_oracle as MO  # noqa: E402

N = 80
FP64_FLOPS = 34e12
HBM_BPS = 3.35e12
# per valid SSIM position and channel: 5 x 11 FMAs along rows and along columns (2 FLOPs each), the products a^2, b^2,
# ab, and 18 operations of the map and its sum. Per pixel and channel: difference, square-accumulate, |d| accumulate.
ALG_FLOPS = 2 * 2 * 5 * 11 + 3 + 18
RESID_FLOPS = 4
CASES = [("256x432", 256, 432), ("720x1280", 720, 1280)]


def work(H, W, C=3, elem=1):
    flops = N * C * (ALG_FLOPS * (H - 10) * (W - 10) + RESID_FLOPS * H * W)
    return flops, 2 * N * H * W * C * elem


def gpu_ms(a, b):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    r = M.frame_metrics(a, b)                     # ends with the device-to-host copy of the results
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]), r


def host_ms(a, b, pool):
    t0 = time.perf_counter()
    r = MO.clip_metrics(a, b, map_fn=pool.map)
    return (time.perf_counter() - t0) * 1e3, r


def kernel_ms(a, b, reps=20):
    """Mean time of one fgt_metrics call (both kernels) on device-resident inputs, between CUDA events."""
    N_, H, W, C = a.shape
    need = lib.call("fgt_metrics_workspace", N_, H, W, C)
    ws = torch.empty(need, dtype=torch.uint8, device=a.device)
    out = torch.empty(N_, 4, dtype=torch.float64, device=a.device)
    args = (a, lib.METRIC_U8, b, lib.METRIC_U8, N_, H, W, C, ws, need, out, None)
    lib.call("fgt_metrics", *args, kernels=2)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        lib.call("fgt_metrics", *args, kernels=2)
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def kernel_split(pairs):
    """{case: {tile, reduce} ms} from one torch.profiler session that scores each case once, in order."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for a, b in pairs.values():
            M.frame_metrics(a, b)
        torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if "metrics_" in e.name and e.device_type == torch.autograd.DeviceType.CUDA),
                  key=lambda e: e.time_range.start)
    tiles = [e for e in kern if "metrics_tile_kernel" in e.name]
    reds = [e for e in kern if "metrics_reduce_kernel" in e.name]
    if not len(tiles) == len(reds) == len(pairs):                        # one chunk, so one kernel pair, per case
        return {name: dict(tile=float("nan"), reduce=float("nan")) for name in pairs}
    return {name: dict(tile=t.time_range.elapsed_us() / 1e3, reduce=r.time_range.elapsed_us() / 1e3)
            for name, t, r in zip(pairs, tiles, reds)}


def main():
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 3
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip().splitlines()[0] if q.stdout.strip() else torch.cuda.get_device_name(0),
               host_threads=PL.HOST_THREADS, cpu_count=os.cpu_count(), frames=N, rounds=rounds)
    print(f"{res['gpu']}; host pool {PL.HOST_THREADS} threads of {os.cpu_count()} CPUs; {N} uint8 RGB frames")
    pairs = {}
    with ThreadPoolExecutor(max_workers=PL.HOST_THREADS) as pool:
        for name, H, W in CASES:
            a, b = synth.metric_pair(100 + H, N, H, W, 3, "noise", "u8")
            da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
            pairs[name] = (da, db)
            gpu_ms(a, b), gpu_ms(da, db), host_ms(a[:8], b[:8], pool)              # warm-up
            t_host_in, t_dev, t_pool = [], [], []
            for _ in range(rounds):
                t_host_in.append(gpu_ms(a, b)[0])
                ms, got = gpu_ms(da, db)
                t_dev.append(ms)
                ms, ref = host_ms(a, b, pool)
                t_pool.append(ms)
            err = max(float(np.max(np.abs(got["per_frame"][k] - ref["per_frame"][k]) / np.abs(ref["per_frame"][k])))
                      for k in ("l1", "l2", "psnr", "ssim"))
            kms = kernel_ms(da, db)
            flops, nbytes = work(H, W)
            res[name] = dict(gpu_from_host_ms=[round(x, 3) for x in t_host_in], gpu_on_device_ms=[round(x, 3) for x in t_dev],
                             kernels_ms_events=round(kms, 4), alg_flops=flops, alg_bytes=nbytes,
                             fp64_share=round(flops / (kms * 1e-3) / FP64_FLOPS, 4),
                             hbm_share=round(nbytes / (kms * 1e-3) / HBM_BPS, 4),
                             host_pool_ms=[round(x, 1) for x in t_pool], max_rel_vs_oracle=err)
    for name, split in kernel_split(pairs).items():
        res[name]["kernel_ms_profiler"] = {k: round(v, 4) for k, v in split.items()}
    print(f"{'case':10s} {'gpu from host ms':>18s} {'gpu on device ms':>18s} {'kernels ms':>10s} {'tile / reduce ms':>17s} "
          f"{'FP64':>6s} {'HBM':>6s} {'host pool ms':>18s} {'max rel vs oracle':>18s}")
    for name, _, _ in CASES:
        e = res[name]
        h, d, p, sp = e["gpu_from_host_ms"], e["gpu_on_device_ms"], e["host_pool_ms"], e["kernel_ms_profiler"]
        print(f"{name:10s} {min(h):8.2f}-{max(h):8.2f} {min(d):8.3f}-{max(d):8.3f} {e['kernels_ms_events']:10.3f} "
              f"{sp['tile']:8.3f} / {sp['reduce']:6.3f} {100 * e['fp64_share']:5.1f}% {100 * e['hbm_share']:5.1f}% "
              f"{min(p):8.0f}-{max(p):8.0f} {e['max_rel_vs_oracle']:18.2e}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
