"""Temporal consistency of an inpainted clip on the GPU: the flow warping error (E_warp), which needs no ground truth
(csrc/warp_error.cu; definition: oracle/warp_error_oracle.py).

Definition. A clip V of N >= 2 frames [N,H,W,C] (uint8 or float32 on the 0..255 scale, C = 1 or 3, H and W >= 2),
optional hole masks [N,H,W] (non-zero = hole), forward flows F_t (t -> t+1) and backward flows B_t (t+1 -> t), each
[N-1,2,H,W] float32 in pixels, x first. For each pair t = 0..N-2, with I = float32(V) / 255:
  W_t = image_warp(I_{t+1}, F_t)                   frame t+1 brought to frame t
  M_t = 1 - fbConsistencyCheck(F_t, B_t)[0]        1 where |F + B(x+F)|^2 <= 0.01 (|F|^2 + |B(x+F)|^2) + 0.5
  e_t = sum_x M_t(x) sum_c (I_t(x,c) - W_t(x,c))^2 / sum_x M_t(x)
each float32 value cast to float64 before the subtraction, the sums in float64. With masks, e_hole_t is the same sum
restricted to M_t * hole_t (the hole of frame t). A pair whose mask is empty gives NaN and is left out of the mean.
image_warp and fbConsistencyCheck are the reference's (FGT/models/utils/fbConsistencyCheck.py), float32 operation for
operation, with one deliberate departure: the bilinear sample uses grid_sample's align_corners=True convention, the one
the reference's np.linspace(-1, 1, n) grid is built for (it puts -1 and 1 on the centres of the border pixels). Under
the default align_corners=False that the reference runs, a zero flow is not the identity: it samples pixel j at
j W / (W - 1) - 1/2, half-blending the border rows and columns with the zero padding, so a static clip would score a
non-zero error.

Flows. By default they come from RAFT (`raft`, e.g. fgt_b200.raft_model.RAFT or raft_small.SmallRAFT) on the scored
clip itself: iters=20, test_mode=True, on the 0..255 frames (a one-channel clip is repeated to three channels), F from
(t, t+1) and B from (t+1, t), in batches of RAFT_BATCH pairs. Frames whose H or W is not a multiple of 8 are padded as
the reference's InputPadder does (RAFT/utils/utils.py, 'sintel' mode, replicate) and the flows unpadded. Callers may
pass their own flows=(F, B) instead, e.g. the flows of the original video. Flows are never resized. There is no CPU
fallback.

    python -m fgt_b200.warp_error --result out/frames [--mask masks] --raft_model raft-things.pth [--small]
                                  [--mixed_precision] [--gpu N]       # one JSON object on stdout
"""
import argparse
import json
import sys

import numpy as np
import torch
import torch.nn.functional as F

from . import lib

WORKSPACE_BUDGET = 1 << 30                # bytes of device inputs, flows, workspace and maps per launch
RAFT_BATCH = 4                            # pairs per RAFT forward, as GpuBackend.raft_pairs
_DTYPES = {torch.uint8: lib.METRIC_U8, torch.float32: lib.METRIC_F32}


def input_pads(H, W):
    """InputPadder(dims).pad's F.pad amounts in 'sintel' mode: [left, right, top, bottom] up to multiples of 8."""
    pad_ht = (((H // 8) + 1) * 8 - H) % 8
    pad_wd = (((W // 8) + 1) * 8 - W) % 8
    return [pad_wd // 2, pad_wd - pad_wd // 2, pad_ht // 2, pad_ht - pad_ht // 2]


def _tensor(x):
    return x if torch.is_tensor(x) else torch.as_tensor(np.ascontiguousarray(x))


def _device(device, *ts):
    if device is not None:
        dev = torch.device(device)
    else:
        dev = next((t.device for t in ts if t is not None and t.is_cuda), None)
        if dev is None and torch.cuda.is_available():
            dev = torch.device("cuda", torch.cuda.current_device())
    if dev is None or dev.type != "cuda":
        raise RuntimeError("fgt_b200.warp_error runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    return dev


def raft_flows(frames, raft, iters=20):
    """RAFT flows of consecutive frames: frames [n,H,W,C] (tensor on the RAFT's device, 0..255) -> (F, B), float32
    [n-1,2,H,W] on that device, F_t from (t, t+1) and B_t from (t+1, t)."""
    n, H, W, C = frames.shape
    img = frames.permute(0, 3, 1, 2).float()
    if C == 1:
        img = img.expand(n, 3, H, W)
    pads = input_pads(H, W)
    if any(pads):
        img = F.pad(img, pads, mode="replicate")
    img = img.contiguous()
    Hp, Wp = img.shape[2], img.shape[3]
    fw, bw = [], []
    with torch.no_grad():
        for s in range(0, n - 1, RAFT_BATCH):
            e = min(n - 1, s + RAFT_BATCH)
            a, b = img[s:e], img[s + 1:e + 1]
            for out, (i1, i2) in ((fw, (a, b)), (bw, (b, a))):
                _, up = raft(i1, i2, iters=iters, test_mode=True)
                out.append(up.float()[:, :, pads[2]:Hp - pads[3], pads[0]:Wp - pads[1]])
    return torch.cat(fw).contiguous(), torch.cat(bw).contiguous()


def report(sums, with_holes):
    """The score from the per-pair sums [P,4] (sum M*err, sum M, sum M*hole*err, sum M*hole)."""
    sums = np.asarray(sums, np.float64)
    res = {"pairs": int(sums.shape[0])}
    for key, col in (("ewarp", 0), ("ewarp_hole", 2))[:2 if with_holes else 1]:
        with np.errstate(invalid="ignore", divide="ignore"):
            per = np.where(sums[:, col + 1] > 0, sums[:, col] / sums[:, col + 1], np.nan)
        ok = ~np.isnan(per)
        res[key] = float(np.mean(per[ok])) if ok.any() else float("nan")
        res[f"{key}_pairs"] = int(ok.sum())
        res[f"per_pair_{key}"] = per
    return res


def warp_error(frames, masks=None, flows=None, raft=None, iters=20, device=None, return_maps=False):
    """E_warp of a clip (see the module docstring). frames [N,H,W,C] uint8 or float32 (numpy or tensor); masks [N,H,W]
    (non-zero = hole) or None; flows = (F, B), each [N-1,2,H,W] in pixels, or None to run `raft` on the clip.
    Returns {'pairs', 'ewarp', 'ewarp_pairs', 'per_pair_ewarp' (float64 [N-1], NaN for an empty mask), 'sums' (float64
    [N-1,4]: sum M*err, sum M, sum M*hole*err, sum M*hole)}, with masks also 'ewarp_hole', 'ewarp_hole_pairs' and
    'per_pair_ewarp_hole'; with return_maps also 'warped' (float32 [N-1,H,W,C], frame t+1 warped to frame t on the
    0..1 scale) and 'valid' (uint8 [N-1,H,W], M_t). Runs on `device` (default: the inputs' CUDA device, else the
    current one)."""
    v = _tensor(frames)
    if v.dtype not in _DTYPES:
        raise TypeError(f"warp_error: frames must be uint8 or float32, got {v.dtype}")
    if v.dim() != 4:
        raise ValueError(f"warp_error: frames {tuple(v.shape)} must be [N,H,W,C]")
    N, H, W, C = v.shape
    if N < 2 or H < 2 or W < 2 or C not in (1, 3):
        raise ValueError(f"warp_error: frames {tuple(v.shape)} need N >= 2, H >= 2, W >= 2 and C = 1 or 3")
    m = None
    if masks is not None:
        m = _tensor(masks)
        if tuple(m.shape) != (N, H, W):
            raise ValueError(f"warp_error: masks {tuple(m.shape)} must be [N,H,W] = {(N, H, W)}")
    fl = None
    if flows is not None:
        if len(flows) != 2:
            raise ValueError("warp_error: flows must be a pair (forward, backward)")
        fl = [_tensor(f) for f in flows]
        for name, f in zip(("forward", "backward"), fl):
            if tuple(f.shape) != (N - 1, 2, H, W):
                raise ValueError(f"warp_error: {name} flows {tuple(f.shape)} must be [N-1,2,H,W] = {(N - 1, 2, H, W)}")
            if not f.is_floating_point():
                raise TypeError(f"warp_error: {name} flows must be floating point, got {f.dtype}")
    elif raft is None:
        raise ValueError("warp_error: pass flows=(forward, backward) or a RAFT model to compute them")
    if iters < 1:
        raise ValueError(f"warp_error: iters = {iters} must be at least 1")
    dev = _device(device, v, m, *(fl or ()))

    P = N - 1
    per_ws = lib.call("fgt_warp_error_workspace", 2, H, W, C)
    per_pair = H * W * (C * v.element_size() + 1 + 16) + per_ws + (H * W * (4 * C + 1) if return_maps else 0)
    chunk = max(1, min(P, 65535, WORKSPACE_BUDGET // per_pair))
    sums = np.empty((P, 4))
    warped = np.empty((P, H, W, C), np.float32) if return_maps else None
    valid = np.empty((P, H, W), np.uint8) if return_maps else None
    with torch.cuda.device(dev):
        out = torch.empty(P, 4, dtype=torch.float64, device=dev)
        ws = torch.empty(chunk * per_ws, dtype=torch.uint8, device=dev)
        wmap = torch.empty(chunk, H, W, C, dtype=torch.float32, device=dev) if return_maps else None
        vmap = torch.empty(chunk, H, W, dtype=torch.uint8, device=dev) if return_maps else None
        for s in range(0, P, chunk):
            e = min(P, s + chunk)
            cv = v[s:e + 1].to(dev).contiguous()
            cm = (m[s:e + 1].to(dev) != 0).to(torch.uint8).contiguous() if m is not None else None
            if fl is not None:
                ff, fb = (f[s:e].to(dev, torch.float32).contiguous() for f in fl)
            else:
                ff, fb = raft_flows(cv, raft, iters)
            lib.call("fgt_warp_error", cv, _DTYPES[v.dtype], cm, ff, fb, e - s + 1, H, W, C, ws, ws.numel(), out[s:e],
                     wmap, vmap, kernels=2)
            if return_maps:
                warped[s:e] = wmap[:e - s].cpu().numpy()
                valid[s:e] = vmap[:e - s].cpu().numpy()
        sums[:] = out.cpu().numpy()
    res = report(sums, m is not None)
    res["sums"] = sums
    if return_maps:
        res["warped"], res["valid"] = warped, valid
    return res


def load_raft(path, small=False, mixed_precision=False, device="cuda"):
    """A RAFT checkpoint ('module.'-prefixed keys) as fgt_b200.flow_extract loads it, on `device`, in eval mode."""
    from . import raft_small
    raft = torch.nn.DataParallel(raft_small.make_raft(argparse.Namespace(small=small, mixed_precision=mixed_precision,
                                                                         alternate_corr=False)))
    raft.load_state_dict(torch.load(path, map_location="cpu"))
    return raft.module.to(device).eval()


def _parser():
    p = argparse.ArgumentParser(prog="python -m fgt_b200.warp_error",
                                description="Flow warping error (temporal consistency, no ground truth needed) of a "
                                            "clip, computed on the GPU with RAFT flows of the clip itself; prints one "
                                            "JSON object")
    p.add_argument("--result", required=True, help="directory of frames (*.png / *.jpg), e.g. the pipeline's "
                                                   "OUTROOT/frames")
    p.add_argument("--mask", default=None, help="directory of hole masks in the same order and size (non-zero = "
                                                "hole); adds the error inside the holes")
    p.add_argument("--raft_model", required=True, help="RAFT checkpoint ('module.'-prefixed keys)")
    p.add_argument("--small", action="store_true", help="the checkpoint is RAFT's small model (RAFT-S)")
    p.add_argument("--mixed_precision", action="store_true",
                   help="run RAFT with fp16 tensor-core operands, as the reference's autocast mode")
    p.add_argument("--gpu", type=int, default=0, help="CUDA device index")
    return p


def main(argv=None):
    """The command line: returns the dict it prints (per-pair values as lists, NaN as null)."""
    from . import io
    p = _parser()
    args = p.parse_args(argv)
    frames = io.read_frames(args.result)
    if len({f.shape for f in frames}) != 1:
        p.error(f"{args.result}: frames of different sizes")
    if len(frames) < 2:
        p.error(f"{args.result}: {len(frames)} frame(s); at least 2 are needed")
    masks = None
    if args.mask is not None:
        masks = io.read_masks(args.mask)
        if len(masks) != len(frames):
            p.error(f"{args.result} holds {len(frames)} frames and {args.mask} holds {len(masks)} masks")
        if any(mk.shape != frames[0].shape[:2] for mk in masks):
            p.error(f"{args.mask}: masks must be {frames[0].shape[0]}x{frames[0].shape[1]}, the frames' size")
        masks = np.stack(masks)
    dev = torch.device("cuda", args.gpu)
    raft = load_raft(args.raft_model, args.small, args.mixed_precision, dev)
    r = warp_error(np.stack(frames), masks, raft=raft, device=dev)
    nan = lambda x: None if np.isnan(x) else float(x)
    out = {"frames": len(frames), "pairs": r["pairs"]}
    for key in ("ewarp", "ewarp_hole"):
        if key in r:
            out[key], out[f"{key}_pairs"] = nan(r[key]), r[f"{key}_pairs"]
            out[f"per_pair_{key}"] = [nan(x) for x in r[f"per_pair_{key}"]]
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main(sys.argv[1:])
