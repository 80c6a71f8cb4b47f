"""RAFT fp32 against mixed precision (`args.mixed_precision`, the reference's --mixed_precision): one forward of 20
iterations in test_mode at 480x864 with batch 1 and 4 (the pipeline's raft_batch) and at 720x1280, synthetic weights
(synth.raft_state_dict) and seeded inputs.

Timing: CUDA events around one forward, after warm-up of both paths, the two paths alternated round by round in one
call; every round is reported. Profile: a separate torch.profiler run per path and geometry, CUDA time split by kernel
name. Accuracy: mean end-point error of the mixed path against the fp32 path at 1/8 resolution, and E_ref, the same
statistic of the oracle under CUDA autocast against the fp32 oracle (the reference's own mixed-precision error;
skipped at 720x1280, where the fp32 oracle's correlation volume alone is 0.8 GB per copy). Prints a table and one JSON
line (also written to --json PATH when given).

    python tools/bench_raft_precision.py [--rounds 8] [--no-profile] [--no-oracle] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import synth  # noqa: E402
from fgt_b200.raft_model import RAFT  # noqa: E402
from oracle import raft_mixed_oracle as RO  # noqa: E402

CASES = [("480x864_b1", 1, 480, 864), ("480x864_b4", 4, 480, 864), ("720x1280_b1", 1, 720, 1280)]
ITERS = 20


def forward_ms(model, a, b):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    model(a, b, iters=ITERS, test_mode=True)
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1])


def kernel_split(model, a, b, top=12):
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        model(a, b, iters=ITERS, test_mode=True)
        torch.cuda.synchronize()
    rows = sorted(((ev.key, ev.device_time_total / 1e3, ev.count) for ev in prof.key_averages() if ev.device_time_total > 0),
                  key=lambda r: -r[1])
    total = sum(r[1] for r in rows)
    return dict(total_ms=round(total, 3), kernels=[(k[:90], round(ms, 3), n) for k, ms, n in rows[:top]])


def epe(x, y):
    return (x.float() - y.float()).norm(dim=1).mean().item()


def oracle_epe(sd, im1, im2):
    sdc = {k: v.cuda() for k, v in sd.items()}
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            lo16, _ = RO.raft_forward(sdc, im1, im2, iters=ITERS, mixed_precision=True)
            lo32, _ = RO.raft_forward(sdc, im1, im2, iters=ITERS)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    return lo16, lo32


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--json", default=None, help="also write the JSON result line to this file")
    ns = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_raft_precision needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip() or torch.cuda.get_device_name(0), iters=ITERS, rounds=ns.rounds)
    print(f"{res['gpu']}; RAFT forward, {ITERS} iterations, test_mode, {ns.rounds} alternated rounds")
    print(f"{'case':13s} {'fp32 ms (min-max)':>20s} {'mixed ms (min-max)':>20s} {'speed-up':>8s} {'gap/spread':>10s} "
          f"{'EPE mix-fp32':>12s} {'E_ref':>10s}")
    sd = synth.raft_state_dict(seed=7)
    models = {}
    for mixed in (False, True):
        m = RAFT(argparse.Namespace(small=False, mixed_precision=mixed, alternate_corr=False))
        m.load_state_dict(sd)
        models[mixed] = m.cuda().eval()
    for name, n, H, W in CASES:
        im1, im2 = synth.raft_inputs(seed=8, H=H, W=W, n=n)
        a, b = im1.cuda(), im2.cuda()
        times = {False: [], True: []}
        with torch.no_grad():
            lo = {mx: models[mx](a, b, iters=ITERS, test_mode=True)[0] for mx in (False, True)}  # warm-up + outputs
            for mx in (False, True):
                forward_ms(models[mx], a, b)
            for r in range(ns.rounds):
                for mx in ((False, True) if r % 2 == 0 else (True, False)):
                    times[mx].append(forward_ms(models[mx], a, b))
            e = dict(epe_mixed_vs_fp32=epe(lo[True], lo[False]), flow_mag=lo[False].float().norm(dim=1).mean().item())
            if not ns.no_oracle and H * W <= 480 * 864:
                o16, o32 = oracle_epe(sd, a, b)
                e.update(E_ref=epe(o16, o32), epe_mixed_vs_autocast=epe(lo[True], o16))
                del o16, o32
            split = {}
            if not ns.no_profile:
                split = {("mixed" if mx else "fp32"): kernel_split(models[mx], a, b) for mx in (False, True)}
        t32, t16 = times[False], times[True]
        spread = max(max(t32) - min(t32), max(t16) - min(t16))
        gap = statistics.median(t32) - statistics.median(t16)
        res[name] = dict(batch=n, H=H, W=W, fp32_ms=[round(x, 3) for x in t32], mixed_ms=[round(x, 3) for x in t16],
                         speedup_median=round(statistics.median(t32) / statistics.median(t16), 3),
                         gap_over_spread=round(gap / spread, 2) if spread > 0 else None,
                         **{k: round(v, 6) for k, v in e.items()}, profile=split)
        r = res[name]
        print(f"{name:13s} {min(t32):9.2f}-{max(t32):9.2f} {min(t16):9.2f}-{max(t16):9.2f} {r['speedup_median']:7.2f}x "
              f"{r['gap_over_spread'] if r['gap_over_spread'] is not None else float('nan'):10.1f} "
              f"{e['epe_mixed_vs_fp32']:12.3e} {e.get('E_ref', float('nan')):10.3e}")
        for tag, sp in split.items():
            print(f"  {tag} profile, {sp['total_ms']:.2f} ms of kernels:")
            for k, ms, cnt in sp["kernels"]:
                print(f"    {ms:9.3f} ms {cnt:5d}x  {k}")
        del a, b, lo
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if ns.json:
        with open(ns.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
