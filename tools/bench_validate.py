"""Times FGT's validation (fgt_b200.validate) on a seeded DAVIS-like set: 10 videos of 60-90 frames at 854 x 480
(JPEG frames, rectangular masks, 854 x 480 .flo files), evaluated at 240 x 432 with the 2D LAFC and the FGT generator
on seeded synthetic weights.

Reports, per video and summed: the wall time of each stage (decode / resize, flow preparation, diffusion, 2D LAFC,
FGT, scoring), each followed by a device synchronise; the 2D LAFC forward alone at t = 8 (the validation's frame
count) with CUDA events, eager and replayed as a CUDA graph; and the CPU oracle (oracle/validate_oracle.py) timed on one
video. The card's name and power limit are read with nvidia-smi in the same run. Prints a table and one JSON line.

    python tools/bench_validate.py [--videos 10] [--rounds 20] [--no-oracle] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fgt_b200 import synth  # noqa: E402
from fgt_b200 import validate as V  # noqa: E402

H, W = 240, 432


def _events(fn, rounds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return dict(median_ms=ts[len(ts) // 2], min_ms=ts[0], max_ms=ts[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--json", default=None)
    ns = ap.parse_args()
    from fgt_b200.fgt_model import Model as FGTModel
    from fgt_b200.lafc_single import Model as LAFCSingle
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip() or torch.cuda.get_device_name(0), size=f"{W}x{H}")
    fgt_cfg = dict(synth.CFG_A, input_resolution=(H, W))
    fgt_sd = synth.make_state_dict(synth.fgt_param_shapes(fgt_cfg), seed=1)
    lafc_sd = synth.lafc_single_state_dict(seed=2)
    fgt, lafc = FGTModel(fgt_cfg), LAFCSingle(synth.CFG_LAFC_SINGLE)
    fgt.load_state_dict(fgt_sd)
    lafc.load_state_dict(lafc_sd)
    fgt, lafc = fgt.cuda().eval(), lafc.cuda().eval()
    g = torch.Generator().manual_seed(0)
    videos = tuple((f"video_{i:02d}", int(torch.randint(60, 91, (1,), generator=g))) for i in range(ns.videos))
    with tempfile.TemporaryDirectory() as root:
        t0 = time.perf_counter()
        # only the .flo files the frame set reads (about 8 of each video's 60-90): 3.3 MB each at 854 x 480
        need = lambda n: [int(os.path.basename(p)[:5]) for p in V.flow_files("", V.frame_ids(n), n)]  # noqa: E731
        roots = synth.validation_set(root, seed=7, videos=videos, H=480, W=854, flow_hw=(480, 854), flow_ids=need)
        res["dataset_write_s"] = round(time.perf_counter() - t0, 2)
        V.validate(lafc, fgt, *roots, limit=1)                       # warm-up: packing, workspaces, kernel attributes
        times = {}
        t0 = time.perf_counter()
        out = V.validate(lafc, fgt, *roots, times=times)
        torch.cuda.synchronize()
        res["validate_wall_s"] = round(time.perf_counter() - t0, 3)
        res["videos"] = len(out["videos"])
        res["stage_s"] = {k: round(times[k], 4) for k in V.STAGES}
        res["per_video_ms"] = {k: round(1e3 * times[k] / len(out["videos"]), 2) for k in V.STAGES}
        res["mean_psnr"] = out["mean"]["psnr"]
        if not ns.no_oracle:
            from oracle import validate_oracle as VO
            from oracle.fgt_oracle import strip_net
            name = videos[0][0]
            t0 = time.perf_counter()
            VO.validate_video(strip_net(lafc_sd), strip_net(fgt_sd), *[os.path.join(r, name) for r in roots], W, H)
            res["oracle_one_video_s"] = round(time.perf_counter() - t0, 2)
            res["oracle_threads"] = torch.get_num_threads()
    fl, mk = (x.cuda() for x in synth.lafc_single_inputs(seed=3, n=8, H=H, W=W))
    with torch.no_grad():
        res["lafc_t8_eager"] = _events(lambda: lafc(fl, mk), ns.rounds)
        lafc.net.enable_cuda_graph()
        res["lafc_t8_graph"] = _events(lambda: lafc(fl, mk), ns.rounds)
    for k, v in res.items():
        print(f"{k:22s} {v}")
    line = json.dumps(res)
    print(line)
    if ns.json:
        with open(ns.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
