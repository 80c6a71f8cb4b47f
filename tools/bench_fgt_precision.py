"""FGT generator: fp32 path vs mixed-precision path (FGT.enable_mixed_precision) on the same model and inputs.

For each workload (432x240 T=10 and 1280x720 T=10, synthetic weights of the shipped configuration), after warm-up of
both paths (CUDA-graph replay, as a long clip runs), the two paths alternate round by round; each round times
--steps forwards with CUDA events. Every round is reported. Then, in separate runs: a per-kernel split of one eager
forward of each path (CUDA events around each launch), and the accuracy figures: E_ref = rel-L2 of the reference
under CUDA autocast against the fp32 reference, the mixed path against autocast (and the ratio to E_ref), and the
uint8-level histogram of the mixed path against the fp32 path.

    python tools/bench_fgt_precision.py [--rounds 8] [--steps 5] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fgt_b200 import lib, synth  # noqa: E402
from fgt_b200.fgt_model import Model  # noqa: E402

WORKLOADS = [("432x240_t10", 240, 432, 10), ("1280x720_t10", 720, 1280, 10)]


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def _u8(x):
    return ((x.float().clamp(-1, 1) + 1) / 2 * 255).round().to(torch.int16)


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


def run(name, H, W, T, rounds, steps):
    from oracle import fgt_oracle as O
    dev = torch.device("cuda:0")
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (H, W)
    sd = synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=1)
    model = Model(cfg)
    model.load_state_dict(sd)
    model = model.to(dev)
    net = model.net
    inp = tuple(z.to(dev) for z in synth.fgt_inputs(seed=3, t=T, H=H, W=W))
    res = dict(workload=name)
    with torch.no_grad():
        # accuracy (eager)
        out = {}
        for m in (False, True):
            net.enable_mixed_precision(m)
            out[m] = model(*inp).float()
        sdc = {k: v.to(dev) for k, v in O.strip_net(sd).items()}
        ref32 = O.fgt_forward(sdc, *inp).float()
        with torch.autocast("cuda", dtype=torch.float16):
            refac = O.fgt_forward(sdc, *inp).float()
        del sdc
        e_ref, e_mix = _rel(refac, ref32), _rel(out[True], refac)
        lv = (_u8(out[True]) - _u8(out[False])).abs().cpu().numpy()
        res.update(E_ref=e_ref, mixed_vs_autocast=e_mix, ratio_to_E_ref=e_mix / e_ref,
                   fp32_vs_fp32_oracle=_rel(out[False], ref32), mixed_vs_fp32=_rel(out[True], out[False]),
                   uint8_hist_vs_fp32={int(v): int(c) for v, c in zip(*np.unique(lv, return_counts=True))})
        del ref32, refac, out
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
            split["mixed" if m else "fp32"] = {k: round(v, 3) for k, v in sorted(agg.items(), key=lambda kv: -kv[1])}
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
    res.update(rounds_ms=dict(fp32=[round(v, 3) for v in f], mixed=[round(v, 3) for v in x]),
               fp32_ms_median=float(np.median(f)), mixed_ms_median=float(np.median(x)),
               speedup=float(np.median(f) / np.median(x)),
               gap_over_spread=float((np.median(f) - np.median(x)) / max(np.ptp(f), np.ptp(x), 1e-9)))
    del model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--only", default=None, help="run one workload by name")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fgt_precision needs a CUDA device")
    out = dict(gpu=_gpu_info(), results=[])
    print("gpu:", out["gpu"], flush=True)
    for name, H, W, T in WORKLOADS:
        if a.only and name != a.only:
            continue
        r = run(name, H, W, T, a.rounds, a.steps)
        out["results"].append(r)
        print(json.dumps(r), flush=True)
    out["gpu_after"] = _gpu_info()
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
