"""Timing of the flow colour coding (fgt_b200/flowviz.py, csrc/flowviz.cu) and of the pipeline's visualisation
switches, alternated in one run:

* device: flow_to_image of 158 flows of 256x432 (an 80-frame clip's raw and completed flows, both directions) and of 80
  flows of 1080x1920, from device-resident tensors. Per call between CUDA events (both kernels plus the 4*B-byte
  readback of the per-image maxima that the NaN / Inf check needs); one fgt_flow_to_image call (both kernels) between
  CUDA events over 20 calls; the split between the kernels from one torch.profiler session. The HBM share is the
  kernels' algorithmic traffic, BYTES_PER_PIXEL = 8 (max pass reads u, v) + 8 + 3 (colour
  pass reads u, v and writes RGB), over the time of one fgt_flow_to_image call, against the H100 SXM data sheet's 3.35 TB/s.
* host: the numpy definition (oracle/flowviz_oracle.py, which equals RAFT/utils/flow_viz.py flow_to_image) of the
  same flows on the pipeline's host pool (HOST_THREADS), under a wall clock.
* command line: `python -m fgt_b200.pipeline` (main()) on a synthetic clip of --frames frames of 256x432 with synthetic
  weights, without switches and with --vis_flows --vis_completed_flows --vis_prop, after one warm-up run. The models are
  built once, outside the timed calls.

The card's name and power limit are read in the same run. Prints a table and one JSON line."""
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import flowviz, io as IO, lib, pipeline as PL, synth  # noqa: E402
from oracle import flowviz_oracle as FO  # noqa: E402
from tools.bench_pipeline import models  # noqa: E402

HBM_BPS = 3.35e12
BYTES_PER_PIXEL = 8 + 8 + 3
CASES = [("158 x 256x432", 158, 256, 432), ("80 x 1080x1920", 80, 1080, 1920)]


def device_ms(x, reps=10):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(reps):
        out = flowviz.flow_to_image(x)
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]) / reps, out


def kernel_ms(x, reps=20):
    """Mean time of one fgt_flow_to_image call (both kernels, no readback) on device-resident flows, between CUDA
    events."""
    B, H, W, _ = x.shape
    ws = torch.empty(lib.call("fgt_flow_to_image_workspace", B, H, W), dtype=torch.uint8, device=x.device)
    out = torch.empty(B, H, W, 3, dtype=torch.uint8, device=x.device)
    args = (x, B, H, W, 0, ws, ws.numel(), out, None)
    lib.call("fgt_flow_to_image", *args, kernels=2)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        lib.call("fgt_flow_to_image", *args, kernels=2)
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def kernel_split(xs, reps=5):
    """{case: (max pass, colour pass) ms per call} from one torch.profiler session that colours each case `reps`
    times, in order (NaN when the profiler saw no kernels)."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for x in xs.values():
            for _ in range(reps):
                flowviz.flow_to_image(x)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                 and "flowviz" in e.name), key=lambda e: e.time_range.start)
    mx = [e.time_range.elapsed_us() / 1e3 for e in ev if "flow_max_kernel" in e.name]
    col = [e.time_range.elapsed_us() / 1e3 for e in ev if "flow_colour_kernel" in e.name]
    if not len(mx) == len(col) == reps * len(xs):
        return {name: (float("nan"), float("nan")) for name in xs}
    return {name: (float(np.mean(mx[i * reps:(i + 1) * reps])), float(np.mean(col[i * reps:(i + 1) * reps])))
            for i, name in enumerate(xs)}


def host_ms(flows, pool):
    t0 = time.perf_counter()
    out = list(pool.map(FO.flow_to_image, flows))
    return (time.perf_counter() - t0) * 1e3, out


def cli_runs(n_frames, rounds):
    H, W = 256, 432
    frames, masks = synth.pipeline_clip(seed=5, N=n_frames, H=H, W=W)
    be, _ = models(H, W)
    PL.load_models = lambda *a, **k: (be, dict(synth.CFG_LAFC))
    res = {"plain": [], "vis": []}
    with tempfile.TemporaryDirectory() as tmp:
        IO.write_frames(os.path.join(tmp, "in"), frames, mp4=False)
        IO.write_frames(os.path.join(tmp, "msk"), [np.repeat(m[..., None], 3, -1) for m in masks], mp4=False)
        base = ["--path", os.path.join(tmp, "in", "frames"), "--path_mask", os.path.join(tmp, "msk", "frames"),
                "--imgH", str(H), "--imgW", str(W)]
        sw = ["--vis_flows", "--vis_completed_flows", "--vis_prop"]
        PL.main(base + ["--outroot", os.path.join(tmp, "warm")] + sw)
        for r in range(rounds):
            for key, extra in (("plain", []), ("vis", sw)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                PL.main(base + ["--outroot", os.path.join(tmp, f"{key}{r}")] + extra)
                res[key].append(round(time.perf_counter() - t0, 3))
        # two pipeline runs are not bit-identical (fp64 atomics in diffusion, Poisson and RAFT's instance norm), so
        # this reports how far apart the frames of the runs with and without the switches are, not an identity
        rd = lambda key, r: np.stack(IO.read_frames(os.path.join(tmp, f"{key}{r}", "frames"))).astype(np.int16)
        res["frames_max_level_diff"] = max(int(np.abs(rd("plain", r) - rd("vis", r)).max()) for r in range(rounds))
    return res


def main():
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 3
    n_frames = int(sys.argv[sys.argv.index("--frames") + 1]) if "--frames" in sys.argv else 20
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip().splitlines()[0] if q.stdout.strip() else torch.cuda.get_device_name(0),
               host_threads=PL.HOST_THREADS, cpu_count=os.cpu_count(), rounds=rounds)
    print(f"{res['gpu']}; host pool {PL.HOST_THREADS} threads of {os.cpu_count()} CPUs")
    xs = {}
    with ThreadPoolExecutor(max_workers=PL.HOST_THREADS) as pool:
        for name, B, H, W in CASES:
            flows = synth.vis_flows(90 + B, B, H, W)
            x = xs[name] = torch.from_numpy(flows).cuda()
            device_ms(x, 2), host_ms(flows[:8], pool)                                    # warm-up
            t_dev, t_host = [], []
            for _ in range(rounds):
                ms, got = device_ms(x)
                t_dev.append(ms)
                ms, ref = host_ms(flows, pool)
                t_host.append(ms)
            d = np.abs(got.cpu().numpy().astype(np.int16) - np.stack(ref).astype(np.int16))
            kms = kernel_ms(x)
            nbytes = BYTES_PER_PIXEL * B * H * W
            res[name] = dict(device_call_ms=[round(v, 3) for v in t_dev], kernels_ms_events=round(kms, 4),
                             alg_bytes=nbytes, hbm_share=round(nbytes / (kms * 1e-3) / HBM_BPS, 4),
                             host_pool_ms=[round(v, 1) for v in t_host], max_level_diff=int(d.max()),
                             values_differing=int((d != 0).sum()), values=int(d.size))
    for name, (k_max, k_col) in kernel_split(xs).items():
        res[name]["kernel_ms_profiler"] = dict(max=round(k_max, 4), colour=round(k_col, 4))
    res["cli_s"] = cli_runs(n_frames, max(2, rounds - 1))
    res["cli_frames"] = n_frames
    print(f"{'case':16s} {'device call ms':>18s} {'kernels ms':>10s} {'max / colour ms':>17s} {'HBM':>6s} "
          f"{'host pool ms':>20s} {'diff vs numpy':>16s}")
    for name, *_ in CASES:
        e = res[name]
        dv, hp, sp = e["device_call_ms"], e["host_pool_ms"], e["kernel_ms_profiler"]
        print(f"{name:16s} {min(dv):8.3f}-{max(dv):8.3f} {e['kernels_ms_events']:10.3f} {sp['max']:7.3f} / "
              f"{sp['colour']:7.3f} {100 * e['hbm_share']:5.1f}% {min(hp):9.1f}-{max(hp):9.1f} "
              f"{e['values_differing']:>6d} of {e['values']:.1e}")
    print(f"command line, {n_frames} frames of 256x432: without switches {res['cli_s']['plain']} s, with "
          f"--vis_flows --vis_completed_flows --vis_prop {res['cli_s']['vis']} s, frames of the two at most "
          f"{res['cli_s']['frames_max_level_diff']} levels apart")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
