"""FGT's own validation (FGT/networks/network.py:258-352, Network._validate) per video: the frame set around a pivot,
frames, masks and pre-extracted flows resized to the working size, the flows diffused into the hole, completed by
the single-frame LAFC (fgt_b200.lafc_single) and normalised, the FGT generator run on the masked frames, and the
composite scored against the frames with PSNR, SSIM, L1 and L2.

    python -m fgt_b200.validate --frame_root JPEGImages/480p --mask_root rectMask_96 --flow_root flows \\
        --flow_ckpt LAFC_single_ckpt/ --fgt_ckpts FGT_ckpt/ [--limit 10] [--vis_dir DIR] [--gpu N]

prints one JSON object: each video's l1, l2, psnr, ssim and frame count, their means, and the skipped videos with the
reason. The data layout is the reference's valid_config.yaml: <frame_root>/<video>/%05d.jpg,
<mask_root>/<video>/*.png and <flow_root>/<video>/{forward,backward}_flo/%05d.flo (fgt_b200.flow_extract writes it).

What runs where: JPEG decoding and the frame and mask resizes stay on the host with Pillow and cv2, as in the
reference (cv2 hands 3-channel and float64 resizes to IPP; DESIGN.md section 1). The flow resize (the bit-exact
cv2-compatible kernel), the flow scaling, the diffusion (batched regionfill), both networks, the normalisation, the
composite and the uint8 quantisation run on the GPU (csrc/validate.cu); there is no CPU fallback.

The reference's behaviour is kept, quirks included:
- Frame set (:276-279, get_ref_index :356-361): the video length is the number of mask PNGs; the neighbours are
  range(max(0, pivot - n // 2), min(L, pivot + n // 2)) (n // 2 on both sides: 4 frames for n = 5); the references
  are every ref_length-th frame that is not a neighbour; the order is references first, then neighbours.
- Frames (read_frames :363-373): a video with 30 or fewer *.jpg is skipped; frames are read by name (%05d.jpg),
  decoded to RGB by Pillow (what imageio.imread does) and resized by cv2.resize(frame, (w, h), cv2.INTER_LINEAR),
  whose third positional argument is `dst`: the default bilinear interpolation.
- Masks (read_masks :457-468): a video with fewer than 30 PNGs is skipped; masks are taken by position in the sorted
  file list, not by name; cv2.resize(mask / 255., (w, h), cv2.INTER_NEAREST) is again bilinear (the flag lands in
  `dst`), and every value above 0 becomes 1: the hole comes out about one pixel wider than a nearest resize makes it.
- Flows (read_flows :412-435): 'for' reads forward_flo/ with no shift, 'back' backward_flo/ with shift -1, 'bi' raises
  NotImplementedError; the index is clamped to [0, L - 2]; each flow is resized bilinearly and scaled as
  u / pre_w * w and v / pre_h * h in float32, in that order.
- Diffusion (diffusion_flow :383-388): regionfill(flow_c * (1 - mask), mask) per channel in float64; the values inside
  the hole do not enter the fill, so the flows go to the batched solver as they are.
- norm_flows (:80-84) divides each frame's channel by its maximum, not its absolute maximum.
- FGT: frames / 127.5 - 1, masked = frames * (1 - masks), one forward over all t frames (b = 1), and
  comp = out * m + frames * (1 - m).
- Scoring (metrics_calc :354-365): clip((x + 1) / 2 * 255, 0, 255).astype(uint8) of the composite and of the frames.

Where the numbers depart from _validate's own: calculate_metrics (FGT/metrics/__init__.py) scores the uint8 arrays with
skimage's PSNR and SSIM and subtracts them as uint8, so its L1 / L2 residuals wrap around modulo 256. This command
scores with fgt_b200.metrics.frame_metrics: the reference's own psnr.py and MATLAB-style Gaussian SSIM (ssim.py) and the
L1 / L2 of calculate_metrics on float64 differences that never wrap. Also departing from the reference: the videos are
taken in sorted order (os.listdir's order is arbitrary), and a video is skipped before its flows are read (the
reference reads them first, and fails on a short video whose flows are missing).
"""
import argparse
import glob
import json
import os
import sys
import time

import cv2
import numpy as np
import torch
from PIL import Image

from . import io as IO
from . import lib, metrics, morph
from .regionfill import regionfill_batch

DIRECTIONS = {"for": ("forward_flo", 0), "back": ("backward_flo", -1)}
STAGES = ("decode_resize", "flow_prep", "diffusion", "lafc", "fgt", "scoring")


class SkipVideo(Exception):
    """A video _validate leaves out (it prints "doesn't have enough frames")."""


def frame_ids(video_len, pivot=20, num_frames=5, ref_length=10):
    """The frame set of one video (network.py:276-279, 356-361): references first, then neighbours."""
    neighbours = list(range(max(0, pivot - num_frames // 2), min(video_len, pivot + num_frames // 2)))
    refs = [i for i in range(0, video_len, ref_length) if i not in neighbours]
    return refs + neighbours


def flow_files(flow_dir, ids, video_len, direction="for"):
    """The .flo path read for each frame id (read_flows :412-430): shifted, then clamped to [0, video_len - 2]."""
    if direction == "bi":
        raise NotImplementedError("Bidirectional flows processing are not implemented")
    if direction not in DIRECTIONS:
        raise ValueError(f"Unknown flow direction: {direction}")
    sub, shift = DIRECTIONS[direction]
    top = video_len - 1
    out = []
    for i in ids:
        i += shift
        if i >= top:
            i = top - 1
        if i < 0:
            i = 0
        out.append(os.path.join(flow_dir, sub, f"{i:05d}.flo"))
    return out


def read_frames(frame_dir, width, height, ids):
    """uint8 [t,h,w,3] RGB frames (read_frames :363-373); SkipVideo when the video has 30 or fewer *.jpg."""
    n = len(glob.glob(os.path.join(frame_dir, "*.jpg")))
    if n <= 30:
        raise SkipVideo(f"{n} *.jpg frames; more than 30 are needed")
    out = []
    for i in ids:
        path = os.path.join(frame_dir, f"{i:05d}.jpg")
        with Image.open(path) as im:
            if im.mode != "RGB":
                raise ValueError(f"{path}: a {im.mode} image; the validation takes RGB frames")
            frame = np.asarray(im)
        out.append(cv2.resize(frame, (width, height), cv2.INTER_LINEAR))
    return np.stack(out, 0)


def read_masks(mask_dir, width, height, ids):
    """uint8 [t,h,w] 0 / 1 masks (read_masks :457-468); SkipVideo when the video has fewer than 30 PNGs."""
    paths = sorted(glob.glob(os.path.join(mask_dir, "*.png")))
    if len(paths) < 30:
        raise SkipVideo(f"{len(paths)} *.png masks; at least 30 are needed")
    out = []
    for i in ids:
        m = cv2.imread(paths[i], 0)
        if m is None:
            raise ValueError(f"{paths[i]}: not a readable image")
        m = cv2.resize(m / 255., (width, height), cv2.INTER_NEAREST)   # bilinear: the flag is the `dst` argument
        out.append((m > 0).astype(np.uint8))
    return np.stack(out, 0)


def read_flows(paths, width, height, device):
    """float32 [t,h,w,2] on the device: each .flo resized bilinearly as cv2.resize does and scaled by (w / pre_w,
    h / pre_h) as u / pre_w * w (read_flows :428-433). Flows of one size are resized in one launch."""
    raw = [IO.read_flo(p) for p in paths]
    out = torch.empty(len(raw), height, width, 2, dtype=torch.float32, device=device)
    for shape in dict.fromkeys(f.shape for f in raw):
        idx = [i for i, f in enumerate(raw) if f.shape == shape]
        r = morph.resize_bilinear(np.stack([raw[i] for i in idx], 0), (height, width), device=device)
        lib.call("fgt_valid_flow_scale", r, r.numel() // 2, float(shape[1]), float(width), float(shape[0]),
                 float(height))
        out[idx] = r
    return out


class _Clock:
    """Per-stage wall time, with a device synchronise before each reading (off when `times` is None)."""

    def __init__(self, times, device):
        self.times, self.device = times, device
        self.t = time.perf_counter() if times is not None else None

    def __call__(self, stage):
        if self.times is None:
            return
        torch.cuda.synchronize(self.device)
        now = time.perf_counter()
        self.times[stage] = self.times.get(stage, 0.0) + now - self.t
        self.t = now


def validate_video(lafc, fgt, frame_dir, mask_dir, flow_dir, width=432, height=240, num_frames=5, ref_length=10,
                   pivot=20, flow_direction="for", device=None, vis_dir=None, stages=None, times=None):
    """One video of Network._validate. lafc: fgt_b200.lafc_single.Model, fgt: fgt_b200.fgt_model.Model, both on
    `device`. Returns {'l1', 'l2', 'psnr', 'ssim', 'frames'}; raises SkipVideo for a video _validate skips.
    stages: a dict that receives the intermediate device tensors; times: a dict that accumulates the wall seconds of
    each of STAGES (synchronising after each)."""
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("fgt_b200.validate runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    clock = _Clock(times, dev)
    video_len = len(glob.glob(os.path.join(mask_dir, "*.png")))
    ids = frame_ids(video_len, pivot, num_frames, ref_length)
    frames = read_frames(frame_dir, width, height, ids)
    masks = read_masks(mask_dir, width, height, ids)
    t, H, W = len(ids), height, width
    frames_d = torch.from_numpy(frames).to(dev)
    masks_d = torch.from_numpy(masks).to(dev)
    clock("decode_resize")
    flows = read_flows(flow_files(flow_dir, ids, video_len, flow_direction), W, H, dev)
    clock("flow_prep")
    filled = regionfill_batch(flows.permute(3, 0, 1, 2).reshape(2 * t, H, W), torch.cat([masks_d, masks_d]), device=dev)
    diffused = filled.view(2, t, H, W).permute(1, 0, 2, 3).float().contiguous()
    clock("diffusion")
    frames_n = torch.empty(t, 3, H, W, dtype=torch.float32, device=dev)
    masked = torch.empty_like(frames_n)
    masks_f = torch.empty(t, 1, H, W, dtype=torch.float32, device=dev)
    lib.call("fgt_valid_inputs", frames_d, masks_d, t, H, W, frames_n, masked, masks_f)
    with torch.no_grad():
        completed = lafc(diffused, masks_f)[0]
    fmax = torch.empty(t * 2, dtype=torch.float32, device=dev)
    lib.call("fgt_plane_max", completed, t * 2, H * W, fmax)
    normed = torch.empty_like(completed)
    lib.call("fgt_valid_norm_flows", completed, fmax, t * 2, H * W, normed)
    clock("lafc")
    with torch.no_grad():
        out = fgt(masked.view(1, t, 3, H, W), normed.view(1, t, 2, H, W), masks_f.view(1, t, 1, H, W))
    out = out.float().contiguous()
    clock("fgt")
    comp_u8 = torch.empty(t, H, W, 3, dtype=torch.uint8, device=dev)
    frames_u8 = torch.empty_like(comp_u8)
    lib.call("fgt_valid_score", out, frames_n, masks_f, t, H, W, comp_u8, frames_u8)
    m = metrics.frame_metrics(comp_u8, frames_u8, device=dev)
    clock("scoring")
    if stages is not None:
        stages.update(ids=ids, frames=frames, masks=masks, flows=flows, diffused=diffused, completed=completed,
                      normed=normed, masked=masked, out=out, comp_u8=comp_u8, frames_u8=frames_u8)
    if vis_dir is not None:
        write_vis(vis_dir, out, masks_f, frames_n, masked)
    return dict(l1=m["l1"], l2=m["l2"], psnr=m["psnr"], ssim=m["ssim"], frames=t)


def _as_png_u8(canvas):
    """imageio's conversion of a float image it is asked to write as 8-bit (image_as_uint): [0, 1] data is scaled by
    255, anything else stretched from its own min..max to 0..255; both then rounded by + 0.499999999 and truncation."""
    mi, ma = float(np.nanmin(canvas)), float(np.nanmax(canvas))
    if mi >= 0 and ma <= 1:
        v = canvas.astype(np.float64) * 255.0 + 0.499999999
    elif ma == mi:
        return canvas.astype(np.uint8)
    else:
        v = (canvas.astype(np.float64) - mi) / (ma - mi) * 255.0 + 0.499999999
    return v.astype(np.uint8)


def write_vis(out_dir, out, masks_f, frames_n, masked):
    """vis_frames (network.py:470-489): result_compare_%05d.png canvases of (result | frame | masked frame) with 20
    black columns between them, result = out * m + frames * (1 - m), all as clip((x + 1) / 2 * 255, 0, 255)."""
    os.makedirs(out_dir, exist_ok=True)
    m = masks_f.cpu().numpy()
    res = out.cpu().numpy() * m + frames_n.cpu().numpy() * (1 - m)
    imgs = [np.clip(((x.transpose(0, 2, 3, 1) + 1) / 2) * 255, 0, 255) for x in (res, frames_n.cpu().numpy(),
                                                                              masked.cpu().numpy())]
    t, h, w, _ = imgs[0].shape
    gap = 20
    for i in range(t):
        canvas = np.zeros((h, w * 3 + gap * 2, 3))
        canvas[:, 0:w] = imgs[0][i]
        canvas[:, w + gap:2 * w + gap] = imgs[1][i]
        canvas[:, 2 * (w + gap):] = imgs[2][i]
        Image.fromarray(_as_png_u8(canvas)).save(os.path.join(out_dir, f"result_compare_{i:05d}.png"))


def validate(lafc, fgt, frame_root, mask_root, flow_root, limit=None, vis_dir=None, times=None, **kw):
    """Network._validate over the videos of flow_root (sorted; the first `limit`). Returns {'videos': {name: scores},
    'mean': {metric: mean over the scored videos}, 'skipped': {name: reason}}."""
    names = sorted(os.listdir(flow_root))
    if limit is not None:
        names = names[:limit]
    videos, skipped = {}, {}
    for name in names:
        try:
            videos[name] = validate_video(lafc, fgt, os.path.join(frame_root, name), os.path.join(mask_root, name),
                                          os.path.join(flow_root, name),
                                          vis_dir=None if vis_dir is None else os.path.join(vis_dir, name),
                                          times=times, **kw)
        except SkipVideo as e:
            skipped[name] = str(e)
    mean = {k: float(np.mean([v[k] for v in videos.values()])) for k in metrics.KEYS} if videos else {}
    return dict(videos=videos, mean=mean, skipped=skipped)


def load_models(flow_ckpt, fgt_ckpts, device):
    """init_flow_model (network.py:42-48) and the generator, each from a reference checkpoint directory (one *.tar
    with `model_state_dict`, one *.yaml config; FGT/train.py:45-50)."""
    from .fgt_model import Model as FGTModel
    from .lafc_single import Model as LAFCSingle
    from .pipeline import load_ckpt_dir
    sd, cfg = load_ckpt_dir(flow_ckpt)
    lafc = LAFCSingle(cfg)
    lafc.load_state_dict(sd)
    sd, cfg = load_ckpt_dir(fgt_ckpts)
    fgt = FGTModel(cfg)
    fgt.load_state_dict(sd)
    return lafc.to(device).eval(), fgt.to(device).eval()


def arg_parser():
    p = argparse.ArgumentParser(prog="python -m fgt_b200.validate", description=__doc__.split("\n\n")[0],
                                formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--frame_root", required=True, help="<frame_root>/<video>/%%05d.jpg")
    p.add_argument("--mask_root", required=True, help="<mask_root>/<video>/*.png")
    p.add_argument("--flow_root", required=True, help="<flow_root>/<video>/{forward,backward}_flo/%%05d.flo; its "
                   "subdirectories are the videos")
    p.add_argument("--flow_ckpt", required=True, help="directory of the 2D LAFC checkpoint (*.tar) and config (*.yaml)")
    p.add_argument("--fgt_ckpts", required=True, help="directory of the FGT checkpoint (*.tar) and config (*.yaml)")
    p.add_argument("--width", type=int, default=432)
    p.add_argument("--height", type=int, default=240)
    p.add_argument("--num_frames", type=int, default=5, help="neighbour span around the pivot")
    p.add_argument("--ref_length", type=int, default=10, help="stride of the reference frames")
    p.add_argument("--pivot", type=int, default=20)
    p.add_argument("--flow_direction", default="for", choices=["for", "back", "bi"],
                   help="'bi' is not implemented (as in the reference)")
    p.add_argument("--limit", type=int, default=None,
                   help="validate the first N videos in sorted order; the reference takes the first 10 of "
                        "os.listdir(flow_root), so --limit 10 reproduces its cap")
    p.add_argument("--vis_dir", default=None, help="write <vis_dir>/<video>/result_compare_%%05d.png")
    p.add_argument("--gpu", type=int, default=0)
    return p


def main(argv=None):
    ns = arg_parser().parse_args(argv)
    if ns.flow_direction == "bi":
        raise NotImplementedError("Bidirectional flows processing are not implemented")
    dev = torch.device("cuda", ns.gpu)
    lafc, fgt = load_models(ns.flow_ckpt, ns.fgt_ckpts, dev)
    res = validate(lafc, fgt, ns.frame_root, ns.mask_root, ns.flow_root, limit=ns.limit, vis_dir=ns.vis_dir,
                   width=ns.width, height=ns.height, num_frames=ns.num_frames, ref_length=ns.ref_length,
                   pivot=ns.pivot, flow_direction=ns.flow_direction, device=dev)
    json.dump(res, sys.stdout)
    sys.stdout.write("\n")
    return res


if __name__ == "__main__":
    main()
