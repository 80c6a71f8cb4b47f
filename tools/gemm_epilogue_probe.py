"""How much of a GEMM tile's time no MMA hides: times fgt_gemm_tc at M=7200 (the transformer's token count) for
N in {512, 1536} and K in {64, 256, 512, 1024, 2048} with two epilogues, under the previous tile schedule
(fgt_debug_gemm_serial_epilogue(1)) and the current one, fits time = a + b * K per epilogue and prints the intercept a
(per-launch cost that does not scale with K: epilogues, pipeline fill / drain, wave tail) next to the K=512 time.
Needs a GPU."""
import ctypes
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import lib, packing  # noqa: E402

M, NS, KS, BN, REPS = 7200, (512, 1536), (64, 256, 512, 1024, 2048), 128, 200


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def time_ms(fn):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / REPS


def main():
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    print(f"card: {card()}")
    L = lib.load()
    L.fgt_debug_gemm_serial_epilogue.argtypes = [ctypes.c_int]
    for N in NS:
        x = torch.randn(M, N, device=dev)
        xs = lib.empty_split((M, N), dev)
        b = torch.randn(N, device=dev)
        res = {}
        for K in KS:
            a = lib.to_split(torch.randn(M, K, device=dev))
            w = packing.pack_weight(torch.randn(N, K, device=dev) / K ** 0.5).to(dev)
            seg = [lib.ASeg(a, K, M)]
            for sched in ("serial", "overlap"):
                L.fgt_debug_gemm_serial_epilogue(1 if sched == "serial" else 0)
                try:
                    # out-projection / ffn2 epilogue: x += A W^T + b (fp32 read + fp32 write) and the split copy of x
                    res[("residual", sched, K)] = time_ms(
                        lambda: lib.gemm_tc(seg, w, N, out_w=M, bn=BN, bias=b, aux=x, aux_mode=lib.AUX_ADD, out_f32=x,
                                            out_split=xs))
                    res[("split", sched, K)] = time_ms(lambda: lib.gemm_tc(seg, w, N, out_w=M, bn=BN, bias=b,
                                                                           out_split=xs))
                finally:
                    L.fgt_debug_gemm_serial_epilogue(0)
        print(f"\nM={M} N={N} bn={BN}, {REPS} back-to-back launches per point (CUDA events)")
        print(f"{'epilogue':10s} {'schedule':9s} " + " ".join(f"{'K=' + str(k):>9s}" for k in KS) +
              f" {'intercept':>10s} {'us/K64':>8s} {'icpt/K512':>10s}")
        for epi in ("residual", "split"):
            for sched in ("serial", "overlap"):
                ys = [res[(epi, sched, k)] * 1e3 for k in KS]
                n = len(KS)
                mx, my = sum(KS) / n, sum(ys) / n
                slope = sum((k - mx) * (y - my) for k, y in zip(KS, ys)) / sum((k - mx) ** 2 for k in KS)
                icpt = my - slope * mx
                print(f"{epi:10s} {sched:9s} " + " ".join(f"{y:8.1f}u" for y in ys) +
                      f" {icpt:9.1f}u {slope * 64:7.2f}u {icpt / ys[KS.index(512)]:10.1%}")


if __name__ == "__main__":
    main()
