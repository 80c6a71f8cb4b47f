"""LAFC flow completion: fp32 path vs mixed-precision path (P3DNet.enable_mixed_precision) on the same model and inputs.

For each workload (256x432 and 480x864, T=3, one triplet per forward as `lafc_complete` calls it; synthetic weights of
the shipped configuration), after warm-up of both paths (CUDA-graph replay, as a clip's triplets run), the two paths
alternate round by round; each round times --steps forwards with CUDA events. Reported: min-max per path, the speed-up
of the medians and the gap of the medians over the larger spread. Then a per-kernel split of one eager forward of each
path (CUDA events around each launch). Last, one pipeline run of an --frames-frame 256x432 clip per LAFC precision
(RAFT and FGT in fp32), timed stage by stage with a device synchronise after every backend call, which gives LAFC's
share of the run. The card's name and power limit are read in the same call.

    python tools/bench_lafc_precision.py [--rounds 8] [--steps 20] [--frames 80] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fgt_b200 import lib, synth  # noqa: E402
from fgt_b200.lafc_model import Model  # noqa: E402

WORKLOADS = [("256x432_t3", 256, 432), ("480x864_t3", 480, 864)]


def _gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unavailable ({e})"


def _time(model, inp, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        model(*inp)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def run(name, H, W, rounds, steps):
    dev = torch.device("cuda:0")
    model = Model(dict(synth.CFG_LAFC))
    model.load_state_dict(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=5))
    model = model.to(dev).eval()
    net = model.net
    inp = tuple(z.to(dev) for z in synth.lafc_inputs(seed=6, H=H, W=W))
    res = dict(workload=name)
    with torch.no_grad():
        out = {}
        for m in (False, True):
            net.enable_mixed_precision(m)
            out[m] = model(*inp)
        res["mixed_vs_fp32_flow_max_px"] = (out[True][0] - out[False][0]).abs().max().item()
        res["mixed_vs_fp32_flow_rel_l2"] = ((out[True][0] - out[False][0]).norm() / out[False][0].norm()).item()
        # per-kernel split (eager, profiler on)
        split = {}
        for m in (False, True):
            net.enable_mixed_precision(m)
            model(*inp)
            torch.cuda.synchronize()
            lib.profile_start()
            model(*inp)
            recs = lib.profile_stop()
            agg = defaultdict(float)
            for kern, _tag, _fl, _by, ms, _sc in recs:
                agg[kern] += ms
            split["mixed" if m else "fp32"] = {k: round(v, 4) for k, v in sorted(agg.items(), key=lambda kv: -kv[1])}
        res["kernel_ms"] = split
        # timing: CUDA graphs, warm-up of both paths, then alternating rounds
        net.enable_cuda_graph(True)
        for m in (False, True):
            net.enable_mixed_precision(m)
            for _ in range(3):
                model(*inp)
        torch.cuda.synchronize()
        times = {False: [], True: []}
        for r in range(rounds):
            for m in ((False, True) if r % 2 == 0 else (True, False)):
                net.enable_mixed_precision(m)
                times[m].append(_time(model, inp, steps))
        net.enable_cuda_graph(False)
        net.enable_mixed_precision(False)
    f, x = np.array(times[False]), np.array(times[True])
    res.update(rounds_ms=dict(fp32=[round(v, 4) for v in f], mixed=[round(v, 4) for v in x]),
               fp32_ms_min_max=[float(f.min()), float(f.max())], mixed_ms_min_max=[float(x.min()), float(x.max())],
               fp32_ms_median=float(np.median(f)), mixed_ms_median=float(np.median(x)),
               speedup=float(np.median(f) / np.median(x)),
               gap_over_spread=float((np.median(f) - np.median(x)) / max(np.ptp(f), np.ptp(x), 1e-9)))
    del model
    torch.cuda.empty_cache()
    return res


def pipeline_share(N, H=256, W=432):
    """One pipeline run of an N-frame clip per LAFC precision, stage by stage (Timed from tools/bench_pipeline.py);
    a 10-frame run of the same size first warms up each backend (module load, workspaces, graphs)."""
    from fgt_b200 import pipeline as PL
    from tools.bench_pipeline import Timed, models
    frames, masks = synth.pipeline_clip(seed=5, N=N, H=H, W=W)
    args = PL.make_args(imgH=H, imgW=W, flow_mask_dilates=3, frame_dilates=1)
    out = {}
    for mixed in (False, True):
        be, _ = models(H, W)
        be.lafc.net.enable_mixed_precision(mixed)
        PL.video_inpainting(frames[:10], masks[:10], be, args)
        tb = Timed(be, True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        PL.video_inpainting(frames, masks, tb, args)
        torch.cuda.synchronize()
        tot = time.perf_counter() - t0
        stages = {k: round(v, 4) for k, v in sorted(tb.t.items(), key=lambda kv: -kv[1])}
        out["lafc_mixed" if mixed else "lafc_fp32"] = dict(
            seconds=round(tot, 4), stage_seconds=stages, lafc_seconds=stages.get("lafc_complete", 0.0),
            lafc_share=round(stages.get("lafc_complete", 0.0) / tot, 4), lafc_forwards=2 * (N - 1))
        del be
        torch.cuda.empty_cache()
    return dict(clip=f"{N}x{H}x{W}", **out)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--frames", type=int, default=80, help="frames of the pipeline clip (0: skip the pipeline run)")
    ap.add_argument("--only", default=None, help="run one workload by name")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lafc_precision needs a CUDA device")
    out = dict(gpu=_gpu_info(), results=[])
    print("gpu:", out["gpu"], flush=True)
    for name, H, W in WORKLOADS:
        if a.only and name != a.only:
            continue
        r = run(name, H, W, a.rounds, a.steps)
        out["results"].append(r)
        print(json.dumps(r), flush=True)
    if a.frames:
        out["pipeline"] = pipeline_share(a.frames)
        print(json.dumps(out["pipeline"]), flush=True)
    out["gpu_after"] = _gpu_info()
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
