"""Dataset pre-processing of the reference's tool/flow_extract.py: forward and backward RAFT flows of every video in
a directory, written as Middlebury `.flo` files (<outroot>/<video>/forward_flo/%05d.flo, backward_flo/%05d.flo;
flow_extract.py:64-105). The frames are resized with `cv2.resize` like the reference (:142-145), all pairs of a video run
through the batched RAFT of the GPU backend (or any callable with its signature), and the files are written with
fgt_b200.io.write_flo (byte-identical to the reference's writer).

    python -m fgt_b200.flow_extract --path videos/ --outroot flows/ --model raft-things.pth [--width 432 --height 256]
                                    [--mixed_precision] [--small]
"""
import argparse
import os

import cv2
import numpy as np
import torch

from . import io as IO


def extract_video(frames_u8, raft_pairs, outdir, width=432, height=256, iters=20):
    """frames_u8: list of RGB uint8 [h,w,3]; raft_pairs(img1 [n,3,H,W], img2, iters) -> [n,2,H,W] flows (numpy).
    Writes forward_flo / backward_flo under outdir and returns (forward, backward) as [N-1,H,W,2] float32."""
    video = []
    for img in frames_u8:
        img = np.asarray(img)
        if width != 0 and height != 0:
            img = cv2.resize(img, (width, height), cv2.INTER_LINEAR)        # same positional call as the reference
        video.append(torch.from_numpy(img.astype(np.uint8)).permute(2, 0, 1).float())
    video = torch.stack(video, dim=0)
    if video.shape[2] % 8 or video.shape[3] % 8:
        raise ValueError(f"flow_extract: frame size {tuple(video.shape[2:])} must be divisible by 8 for RAFT")
    out = []
    for mode, (a, b) in (("forward", (video[:-1], video[1:])), ("backward", (video[1:], video[:-1]))):
        flows = np.ascontiguousarray(np.asarray(raft_pairs(a, b, iters)).transpose(0, 2, 3, 1)).astype(np.float32)
        d = os.path.join(outdir, mode + "_flo")
        os.makedirs(d, exist_ok=True)
        for i in range(flows.shape[0]):
            IO.write_flo(os.path.join(d, "%05d.flo" % i), flows[i])
        out.append(flows)
    return tuple(out)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--path", required=True, help="directory with one sub-directory of frames per video")
    ap.add_argument("--expdir", default=None, help="videos listed in this directory are skipped")
    ap.add_argument("--outroot", required=True)
    ap.add_argument("--width", type=int, default=432)
    ap.add_argument("--height", type=int, default=256)
    ap.add_argument("--model", default="../weight/raft-things.pth", help="RAFT checkpoint ('module.'-prefixed keys)")
    ap.add_argument("--gpu", type=int, default=0)
    ap.add_argument("--mixed_precision", action="store_true",
                    help="run RAFT with fp16 tensor-core operands, as the reference's autocast mode")
    ap.add_argument("--small", action="store_true",
                    help="run RAFT's small model (RAFT-S; --model must then be a small-model checkpoint such as "
                         "raft-small.pth)")
    ns = ap.parse_args(argv)
    from . import raft_small
    from .pipeline import GpuBackend
    dev = torch.device("cuda", ns.gpu)
    raft = torch.nn.DataParallel(raft_small.make_raft(argparse.Namespace(small=ns.small, mixed_precision=ns.mixed_precision,
                                                                         alternate_corr=False)))
    raft.load_state_dict(torch.load(ns.model, map_location="cpu"))
    backend = GpuBackend(raft.module.to(dev).eval(), None, None, device=dev)
    skip = set(os.listdir(ns.expdir)) if ns.expdir and os.path.isdir(ns.expdir) else set()
    videos = sorted(os.listdir(ns.path))
    for k, vid in enumerate(videos, 1):
        if vid in skip:
            print(f"[{k}]/[{len(videos)}] Video {vid} skipped")
            continue
        frames = IO.read_frames(os.path.join(ns.path, vid))
        extract_video(frames, backend.raft_pairs, os.path.join(ns.outroot, vid), ns.width, ns.height)
        print(f"[{k}]/[{len(videos)}] Video {vid}: {2 * (len(frames) - 1)} flows written")


if __name__ == "__main__":
    main()
