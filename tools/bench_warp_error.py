"""Timing of the flow warping error (fgt_b200/warp_error.py, csrc/warp_error.cu) on the GPU, for uint8 RGB clips with
hole masks at 480x854 (N = 80) and 1080x1920 (N = 30), and of a whole `python -m fgt_b200.warp_error` run.

Kernels: one fgt_warp_error call (tile + reduce kernel, no maps) on device-resident inputs, CUDA events around REPS
calls. Eager: the same work as the reference's functions would do it with torch on the same GPU (image_warp's linspace
grid and F.grid_sample with align_corners=True for B and for frame t+1, the forward occlusion test of
fbConsistencyCheck, the float64 masked sums). After a warm-up of both, the two alternate for --rounds rounds; min-max
over rounds is reported. Bytes are the algorithm's per pixel and pair (F_t and the 2-channel B_t sample, 8 + 8; frames
t and t+1, 2 C; the hole, 1) over the kernel time, against the H100 SXM data sheet's 3.35 TB/s HBM3.
Command line: main() of fgt_b200.warp_error on N_CLI PNG frames at 480x854 with synthetic RAFT weights (the speed of
RAFT does not depend on the weights' values), split by timing raft_flows and the scoring of the same clip on its own.
The card's name and power limit are read in the same run. Prints a table and one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import lib, synth  # noqa: E402
from fgt_b200 import warp_error as WE  # noqa: E402

HBM_BPS = 3.35e12
CASES = [("480x854", 480, 854, 80), ("1080x1920", 1080, 1920, 30)]
N_CLI = 20
REPS = 10


def clip(seed, N, H, W, dev):
    """A smooth texture translating by (1, 2) px per frame, a moving box hole, and smooth flows near (2, 1)."""
    g = torch.Generator().manual_seed(seed)
    big = torch.nn.functional.interpolate(torch.rand(1, 3, (H + 2 * N) // 8 + 2, (W + 2 * N) // 8 + 2, generator=g),
                                          size=(H + 2 * N, W + 2 * N), mode="bilinear", align_corners=False)[0]
    frames = torch.stack([big[:, i:i + H, 2 * i:2 * i + W] for i in range(N)]).permute(0, 2, 3, 1)
    frames = (frames * 255).to(torch.uint8).contiguous().to(dev)
    masks = torch.zeros(N, H, W, dtype=torch.uint8, device=dev)
    masks[:, H // 3:H // 2, W // 3:W // 2] = 1
    f = torch.tensor([2.0, 1.0]).view(1, 2, 1, 1) + 0.3 * torch.randn(N - 1, 2, H, W, generator=g)
    return frames, masks, f.float().to(dev).contiguous(), (-f).float().to(dev).contiguous()


def alg_bytes(N, H, W, C=3):
    return (N - 1) * H * W * (8 + 8 + 2 * C + 1)


def kernel_call(frames, masks, f, b):
    N, H, W, C = frames.shape
    need = lib.call("fgt_warp_error_workspace", N, H, W, C)
    ws = torch.empty(need, dtype=torch.uint8, device=frames.device)
    out = torch.empty(N - 1, 4, dtype=torch.float64, device=frames.device)
    return lambda: lib.call("fgt_warp_error", frames, lib.METRIC_U8, masks, f, b, N, H, W, C, ws, need, out, None, None,
                            kernels=2)


def eager_call(frames, masks, f, b):
    """The reference's operations, eagerly by torch: image_warp twice, the forward test, the float64 sums."""
    N, H, W, C = frames.shape
    x = torch.from_numpy(np.linspace(-1, 1, W).astype(np.float32)).to(frames.device)
    y = torch.from_numpy(np.linspace(-1, 1, H).astype(np.float32)).to(frames.device)
    grid = torch.stack(torch.meshgrid(x, y, indexing="xy"), -1)[None]

    def image_warp(img, flow):
        fl = torch.cat([flow[:, 0:1] / ((W - 1.0) / 2.0), flow[:, 1:2] / ((H - 1.0) / 2.0)], 1).permute(0, 2, 3, 1)
        return F.grid_sample(img, grid + fl, mode="bilinear", padding_mode="zeros", align_corners=True)

    def length_sq(v):
        return torch.sum(torch.square(v), dim=1, keepdim=True)

    def run():
        img = frames.permute(0, 3, 1, 2).float() / 255
        bw = image_warp(b, f)
        occ = (length_sq(f + bw) > 0.01 * (length_sq(f) + length_sq(bw)) + 0.5).float()
        m = (1 - occ)[:, 0].double()
        err = ((img[:-1].double() - image_warp(img[1:], f).double()) ** 2).sum(1)
        hole = (masks[:-1] != 0).double()
        return torch.stack([(m * err).sum((1, 2)), m.sum((1, 2)), (m * hole * err).sum((1, 2)), (m * hole).sum((1, 2))], 1)
    return run


def timed_ms(fn, reps=REPS):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def wall_s(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def command_line(dev, tmp):
    """(total, raft, scoring) seconds of one command-line run and of its two parts on the same clip."""
    from PIL import Image
    frames, masks, _, _ = clip(7, N_CLI, 480, 854, dev)
    fdir, mdir = os.path.join(tmp, "frames"), os.path.join(tmp, "masks")
    os.makedirs(fdir), os.makedirs(mdir)
    for i, (fr, mk) in enumerate(zip(frames.cpu().numpy(), masks.cpu().numpy())):
        Image.fromarray(fr).save(os.path.join(fdir, "%05d.png" % i))
        Image.fromarray(mk * 255).save(os.path.join(mdir, "%05d.png" % i))
    ckpt = os.path.join(tmp, "raft-synth.pth")
    torch.save({"module." + k: v for k, v in synth.raft_state_dict(seed=3).items()}, ckpt)
    argv = ["--result", fdir, "--mask", mdir, "--raft_model", ckpt, "--gpu", str(dev.index or 0)]
    WE.main(argv)                                                                # warm-up: weights, graphs
    total, _ = wall_s(lambda: WE.main(argv))
    raft = WE.load_raft(ckpt, device=dev)
    WE.raft_flows(frames[:2], raft)
    t_raft, (ff, fb) = wall_s(lambda: WE.raft_flows(frames, raft))
    t_score, _ = wall_s(lambda: WE.warp_error(frames.cpu().numpy(), masks.cpu().numpy(), flows=(ff, fb)))
    return total, t_raft, t_score


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_warp_error needs a CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip().splitlines()[0] if q.stdout.strip() else torch.cuda.get_device_name(0),
               rounds=args.rounds, reps=REPS)
    print(res["gpu"])
    for name, H, W, N in CASES:
        data = clip(11 + H, N, H, W, dev)
        kern, eager = kernel_call(*data), eager_call(*data)
        kern(), eager()                                                          # warm-up
        ref = eager()
        t_k, t_e = [], []
        for _ in range(args.rounds):
            t_k.append(timed_ms(kern))
            t_e.append(timed_ms(eager))
        r = WE.warp_error(*data[:2], flows=data[2:])
        got = r["sums"]
        e_ref = (ref[:, 0] / ref[:, 1]).cpu().numpy()
        nbytes = alg_bytes(N, H, W)
        res[name] = dict(frames=N, kernels_ms=[round(x, 4) for x in t_k], eager_ms=[round(x, 3) for x in t_e],
                         alg_bytes=nbytes, hbm_share_best=round(nbytes / (min(t_k) * 1e-3) / HBM_BPS, 4),
                         ewarp=r["ewarp"],
                         max_rel_ewarp_vs_eager=float(np.max(np.abs(r["per_pair_ewarp"] - e_ref) / np.abs(e_ref))),
                         valid_pixels_kernel=float(got[:, 1].sum()), valid_pixels_eager=float(ref[:, 1].sum()))
        del data, kern, eager
        torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as tmp:
        total, t_raft, t_score = command_line(dev, tmp)
    res["command_line_480x854"] = dict(frames=N_CLI, total_s=round(total, 3), raft_s=round(t_raft, 3),
                                       scoring_s=round(t_score, 3))
    print(f"{'case':10s} {'kernels ms':>18s} {'eager ms':>18s} {'HBM (best)':>10s}")
    for name, _, _, _ in CASES:
        e = res[name]
        k, g = e["kernels_ms"], e["eager_ms"]
        print(f"{name:10s} {min(k):8.3f}-{max(k):8.3f} {min(g):8.2f}-{max(g):8.2f} {100 * e['hbm_share_best']:9.1f}%")
    c = res["command_line_480x854"]
    print(f"command line, {N_CLI} frames 480x854: {c['total_s']:.2f} s total; RAFT {c['raft_s']:.2f} s, scoring "
          f"{c['scoring_s']:.3f} s")
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
