"""Per-launch timing (CUDA events) of one FGT forward at 432x240 T=10 under the previous GEMM tile schedule
(fgt_debug_gemm_serial_epilogue(1)) and the current one, side by side: every launch with its tag, both times and their
ratio, then the gemm_tc and all-launch sums. Needs a GPU."""
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import lib, synth  # noqa: E402
from bench import build_model, T, H, W  # noqa: E402
from tools.gemm_epilogue_probe import card  # noqa: E402


def per_launch(model, clip, reps=5):
    with torch.no_grad():
        for _ in range(3):
            model(*clip)
        lib.profile_start()
        for _ in range(reps):
            model(*clip)
        recs = lib.profile_stop()
    n = len(recs) // reps
    return [(recs[i][0], recs[i][1], sum(recs[i + r * n][4] for r in range(reps)) / reps) for i in range(n)]


def main():
    dev = torch.device("cuda:0")
    print(f"card: {card()}")
    L = lib.load()
    L.fgt_debug_gemm_serial_epilogue.argtypes = [ctypes.c_int]
    model, _ = build_model(dev)
    clip = [t.to(dev) for t in synth.fgt_inputs(seed=3, t=T, H=H, W=W)]
    runs = {}
    for sched in ("serial", "overlap", "serial2", "overlap2"):  # alternated twice: the second pair shows the noise
        L.fgt_debug_gemm_serial_epilogue(1 if sched.startswith("serial") else 0)
        try:
            runs[sched] = per_launch(model, clip)
        finally:
            L.fgt_debug_gemm_serial_epilogue(0)
    old, new = runs["serial"], runs["overlap"]
    assert [r[:2] for r in old] == [r[:2] for r in new], "the two schedules ran different launch sequences"
    print(f"{'kernel':14s} {'tag':14s} {'serial ms':>10s} {'overlap ms':>11s} {'new/old':>8s}")
    for (k, tag, t0), (_, _, t1) in zip(old, new):
        print(f"{k:14s} {tag:14s} {t0:10.4f} {t1:11.4f} {t1 / t0:8.3f}")
    for sched in ("serial", "overlap", "serial2", "overlap2"):
        g = sum(t for k, _, t in runs[sched] if k == "gemm_tc")
        a = sum(t for _, _, t in runs[sched])
        print(f"{sched:9s} gemm_tc sum {g:8.3f} ms   all launches {a:8.3f} ms")


if __name__ == "__main__":
    main()
