"""Whole-pipeline timing (RAFT -> diffusion + LAFC -> propagation -> Poisson -> FGT stage; fgt_b200.pipeline) on
synthetic clips: (a) the parity clip of tests/golden (7 frames of 64x96, RAFT at 128x192) with the CPU oracle
backend timed next to it, (b) BASELINE config 2's shape (10 frames of 240x432, RAFT at 480x864). Per-stage wall
times with a device synchronise after every backend call. Prints one JSON object. Run under gpurun."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import pipeline as PL, synth  # noqa: E402
from fgt_b200.fgt_model import Model as FGTModel  # noqa: E402
from fgt_b200.lafc_model import Model as LAFCModel  # noqa: E402
from fgt_b200.raft_model import RAFT  # noqa: E402

dev = torch.device("cuda:0")


class Timed:
    """Wraps a backend: accumulates wall time per stage method (synchronising the device after each call)."""

    def __init__(self, inner, sync):
        self.inner, self.sync, self.t = inner, sync, {}

    def __getattr__(self, name):
        fn = getattr(self.inner, name)

        def call(*a, **kw):
            t0 = time.perf_counter()
            out = fn(*a, **kw)
            if self.sync:
                torch.cuda.synchronize()
            self.t[name] = self.t.get(name, 0.0) + time.perf_counter() - t0
            return out
        return call


def models(H, W, seeds=(31, 32, 33), dev=dev):
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (H, W)
    sds = dict(fgt=synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=seeds[0]),
               lafc=synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=seeds[1]),
               raft=synth.raft_state_dict(seed=seeds[2]))
    fgt = FGTModel(cfg); fgt.load_state_dict(sds["fgt"]); fgt = fgt.to(dev)
    lafc = LAFCModel(dict(synth.CFG_LAFC)); lafc.load_state_dict(sds["lafc"]); lafc = lafc.to(dev)
    raft = RAFT(argparse.Namespace(small=False, mixed_precision=False, alternate_corr=False))
    raft.load_state_dict(sds["raft"]); raft = raft.to(dev).eval()
    # --device-inpaint: the opt-in device TELEA and gradient preparation instead of cv2 on the host pool (A/B runs)
    return PL.GpuBackend(raft, lafc, fgt, device=dev, host_inpaint="--device-inpaint" not in sys.argv), sds


def run(N, H, W, reps):
    frames, masks = synth.pipeline_clip(seed=5, N=N, H=H, W=W)
    args = PL.make_args(imgH=H, imgW=W, flow_mask_dilates=3, frame_dilates=1)
    be, sds = models(H, W)
    PL.video_inpainting(frames, masks, be, args)                       # warm-up (workspaces, module load)
    best = None
    for _ in range(reps):
        tb = Timed(be, True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = PL.video_inpainting(frames, masks, tb, args)
        torch.cuda.synchronize()
        tot = time.perf_counter() - t0
        if best is None or tot < best["seconds"]:
            best = dict(seconds=tot, frames_per_s=N / tot, gpu_stage_seconds={k: round(v, 4) for k, v in tb.t.items()},
                        host_glue_seconds=round(tot - sum(tb.t.values()), 4))
    return best, frames, masks, args, sds, out


def main():
    res = {}
    best, frames, masks, args, sds, out = run(7, 64, 96, 3)
    res["clip_7x64x96"] = best
    if "--no-cpu" not in sys.argv:
        from oracle import fgt_oracle as O
        from oracle.pipeline_oracle import OracleBackend
        ob = Timed(OracleBackend(sds["raft"], O.strip_net(sds["lafc"]), O.strip_net(sds["fgt"])), False)
        t0 = time.perf_counter()
        ref = PL.video_inpainting(frames, masks, ob, args)
        tot = time.perf_counter() - t0
        d = np.abs(np.stack(out).astype(np.int16) - np.stack(ref).astype(np.int16))
        res["clip_7x64x96"]["cpu_oracle"] = dict(seconds=tot, frames_per_s=7 / tot, stage_seconds={k: round(v, 3) for k, v in ob.t.items()},
                                                 threads=torch.get_num_threads(), mean_abs_diff_levels=float(d.mean()),
                                                 frac_over_2_levels=float((d > 2).mean()))
    res["clip_10x240x432"] = run(10, 240, 432, 2)[0]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
