"""RAFT's basic model against its small model (the reference's --small), both fp32.

(1) One forward of 20 iterations in test_mode at 480x864 with batch 1 and 4 (the pipeline's raft_batch) and at
720x1280, synthetic weights (synth.raft_state_dict / synth.raft_small_state_dict) and seeded inputs. Timing: CUDA
events around one forward, after warm-up of both models, the two alternated round by round in one call; every round is
reported; eagerly (one ctypes launch per kernel) and as CUDA-graph replay (enable_cuda_graph), the two timed in
separate alternations. Profile: a separate torch.profiler run per model and geometry, CUDA time split by kernel name.
(2) The RAFT stage's share of a whole pipeline run (fgt_b200.pipeline.video_inpainting on synth.pipeline_clip, 256x432,
so RAFT runs at 512x864) with the small model off and on, a device synchronise after every stage call, after a 10-frame
warm-up run of each; the two alternated.

The card's name, power limit and max SM clock are printed with the numbers. Prints a table and one JSON line (also
written to --json PATH when given).

    python tools/bench_raft_small.py [--rounds 8] [--frames 80] [--pipeline-rounds 2] [--no-profile] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import pipeline as PL, synth  # noqa: E402
from fgt_b200.raft_small import make_raft  # noqa: E402
from tools.bench_pipeline import Timed, models  # noqa: E402
from tools.bench_raft_precision import kernel_split  # noqa: E402

CASES = [("480x864_b1", 1, 480, 864), ("480x864_b4", 4, 480, 864), ("720x1280_b1", 1, 720, 1280)]
ITERS = 20


def raft(small, seed=7):
    m = make_raft(argparse.Namespace(small=small, mixed_precision=False, alternate_corr=False))
    m.load_state_dict((synth.raft_small_state_dict if small else synth.raft_state_dict)(seed=seed))
    return m.cuda().eval()


def forward_ms(model, a, b):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    model(a, b, iters=ITERS, test_mode=True)
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1])


def forwards(ns, nets, res, graph):
    mode = "CUDA-graph replay" if graph else "eager"
    print(f"RAFT forward, {ITERS} iterations, test_mode, fp32, {mode}, {ns.rounds} alternated rounds")
    print(f"{'case':13s} {'basic ms (min-max)':>20s} {'small ms (min-max)':>20s} {'speed-up':>8s} {'gap/spread':>10s}")
    for m in nets.values():
        m.enable_cuda_graph(graph)
    for name, n, H, W in CASES:
        im1, im2 = synth.raft_inputs(seed=8, H=H, W=W, n=n)
        a, b = im1.cuda(), im2.cuda()
        times = {False: [], True: []}
        with torch.no_grad():
            for sm in (False, True):   # warm-up: packing, workspaces, module load (and graph capture)
                nets[sm](a, b, iters=ITERS, test_mode=True)
                forward_ms(nets[sm], a, b)
                forward_ms(nets[sm], a, b)
            for r in range(ns.rounds):
                for sm in ((False, True) if r % 2 == 0 else (True, False)):
                    times[sm].append(forward_ms(nets[sm], a, b))
            split = {} if ns.no_profile or graph else {("small" if sm else "basic"): kernel_split(nets[sm], a, b)
                                              for sm in (False, True)}
        tb, ts = times[False], times[True]
        spread = max(max(tb) - min(tb), max(ts) - min(ts))
        gap = statistics.median(tb) - statistics.median(ts)
        res[("graph_" if graph else "") + name] = dict(batch=n, H=H, W=W, basic_ms=[round(x, 3) for x in tb], small_ms=[round(x, 3) for x in ts],
                         speedup_median=round(statistics.median(tb) / statistics.median(ts), 3),
                         gap_over_spread=round(gap / spread, 2) if spread > 0 else None, profile=split)
        r = res[("graph_" if graph else "") + name]
        print(f"{name:13s} {min(tb):9.2f}-{max(tb):9.2f} {min(ts):9.2f}-{max(ts):9.2f} {r['speedup_median']:7.2f}x "
              f"{r['gap_over_spread'] if r['gap_over_spread'] is not None else float('nan'):10.1f}")
        for tag, sp in split.items():
            print(f"  {tag} profile, {sp['total_ms']:.2f} ms of kernels:")
            for k, ms, cnt in sp["kernels"]:
                print(f"    {ms:9.3f} ms {cnt:5d}x  {k}")
        del a, b
        torch.cuda.empty_cache()
    for m in nets.values():
        m.enable_cuda_graph(False)


def pipeline_share(ns, nets, res):
    H, W = 256, 432
    be, _ = models(H, W)
    args = PL.make_args(imgH=H, imgW=W, flow_mask_dilates=3, frame_dilates=1)
    clip = synth.pipeline_clip(seed=5, N=ns.frames, H=H, W=W)
    warm = synth.pipeline_clip(seed=5, N=10, H=H, W=W)
    runs = {False: [], True: []}
    for sm in (False, True):
        be.raft = nets[sm]
        PL.video_inpainting(*warm, be, args)
    for r in range(ns.pipeline_rounds):
        for sm in ((False, True) if r % 2 == 0 else (True, False)):
            be.raft = nets[sm]
            tb = Timed(be, True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            PL.video_inpainting(*clip, tb, args)
            torch.cuda.synchronize()
            tot = time.perf_counter() - t0
            runs[sm].append(dict(seconds=round(tot, 3), raft_seconds=round(tb.t["raft_pairs"], 3),
                                 raft_share=round(tb.t["raft_pairs"] / tot, 4)))
    res[f"pipeline_{ns.frames}x{H}x{W}"] = {("small" if sm else "basic"): v for sm, v in runs.items()}
    print(f"pipeline, {ns.frames} frames of {H}x{W} (RAFT at {2 * H}x{2 * W}), {ns.pipeline_rounds} alternated rounds")
    for sm in (False, True):
        for v in runs[sm]:
            print(f"  {'small' if sm else 'basic'}: {v['seconds']:.3f} s, RAFT {v['raft_seconds']:.3f} s "
                  f"({100 * v['raft_share']:.1f} %)")


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--frames", type=int, default=80)
    ap.add_argument("--pipeline-rounds", type=int, default=2)
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--json", default=None, help="also write the JSON result line to this file")
    ns = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_raft_small needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip() or torch.cuda.get_device_name(0), iters=ITERS, rounds=ns.rounds)
    print(res["gpu"])
    nets = {sm: raft(sm) for sm in (False, True)}
    forwards(ns, nets, res, graph=False)
    forwards(ns, nets, res, graph=True)
    if ns.frames > 0:
        pipeline_share(ns, nets, res)
    line = json.dumps(res)
    print(line)
    if ns.json:
        with open(ns.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
