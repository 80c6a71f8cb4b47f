"""CPU oracle for one video of FGT's validation (TEST INFRASTRUCTURE — see oracle/fgt_oracle.py header).

Restates /root/reference/FGT/networks/network.py:258-352 (Network._validate) for one video with the other oracles:
get_ref_index :356-361, read_frames :363-373 and read_masks :457-468 (Pillow + cv2 on the host, as the reference),
read_flows :412-435 (cv2.resize + the float32 vector scaling), diffusion_flow :383-388 (regionfill_oracle),
the 2D LAFC (lafc_single_oracle), norm_flows :80-84, FGT (fgt_oracle), the composite :310 and metrics_calc :354-365
with metrics_oracle in place of calculate_metrics (the project's metric definitions; see fgt_b200/validate.py).
The data-loading steps are pinned bit for bit by tests/golden/validate_*.npz (the unmodified network.py methods).
"""
import glob
import os

import cv2
import numpy as np
import torch
from PIL import Image

from oracle import fgt_oracle, lafc_single_oracle, metrics_oracle, regionfill_oracle


def ref_ids(video_len, pivot=20, num_frames=5, ref_length=10):
    neighbours = [i for i in range(max(0, pivot - num_frames // 2), min(video_len, pivot + num_frames // 2))]
    return [i for i in range(0, video_len, ref_length) if i not in neighbours] + neighbours


def read_frames(frame_dir, width, height, ids):
    if len(glob.glob(os.path.join(frame_dir, "*.jpg"))) <= 30:
        return []
    return [cv2.resize(np.asarray(Image.open(os.path.join(frame_dir, f"{i:05d}.jpg"))), (width, height))
            for i in ids]


def read_masks(mask_dir, width, height, ids):
    paths = sorted(glob.glob(os.path.join(mask_dir, "*.png")))
    if len(paths) < 30:
        return []
    out = []
    for i in ids:
        m = cv2.resize(cv2.imread(paths[i], 0) / 255., (width, height))
        m[m > 0] = 1
        out.append(m[:, :, None])
    return out


def _read_flo(path):
    with open(path, "rb") as f:
        assert np.fromfile(f, np.float32, 1)[0] == 202021.25
        w, h = np.fromfile(f, np.int32, 2)
        return np.fromfile(f, np.float32, 2 * w * h).reshape(h, w, 2)


def read_flows(flow_dir, width, height, ids, frame_max, direction="for"):
    sub, shift = {"for": ("forward_flo", 0), "back": ("backward_flo", -1)}[direction]
    out = []
    for i in ids:
        i = min(i + shift, frame_max - 1)
        i = max(i, 0)
        flow = _read_flo(os.path.join(flow_dir, sub, f"{i:05d}.flo"))
        ph, pw = flow.shape[:2]
        flow = cv2.resize(flow, (width, height))
        flow[:, :, 0] = flow[:, :, 0] / pw * width
        flow[:, :, 1] = flow[:, :, 1] / ph * height
        out.append(flow)
    return out


def validate_video(lafc_sd, fgt_sd, frame_dir, mask_dir, flow_dir, width, height, num_frames=5, ref_length=10,
                   pivot=20, direction="for", num_blocks=8):
    """lafc_sd / fgt_sd: state dicts with 'net.' stripped. Returns (metrics dict, stages dict), or None for a video
    _validate skips."""
    video_len = len(glob.glob(os.path.join(mask_dir, "*.png")))
    ids = ref_ids(video_len, pivot, num_frames, ref_length)
    frames = read_frames(frame_dir, width, height, ids)
    masks = read_masks(mask_dir, width, height, ids)
    if frames == [] or masks == []:
        return None
    flows = read_flows(flow_dir, width, height, ids, video_len - 1, direction)
    diffused = []
    for f, m in zip(flows, masks):
        d = np.zeros(f.shape)
        for c in range(2):
            d[:, :, c] = regionfill_oracle.regionfill(f[:, :, c] * (1 - m[:, :, 0]), m[:, :, 0])
        diffused.append(d)
    fr = torch.from_numpy(np.transpose(np.stack(frames), (0, 3, 1, 2))).unsqueeze(0).float() / 127.5 - 1
    mk = torch.from_numpy(np.transpose(np.stack(masks), (0, 3, 1, 2))).unsqueeze(0).float()
    fl = torch.from_numpy(np.transpose(np.stack(diffused), (0, 3, 1, 2))).float()
    t = len(ids)
    with torch.no_grad():
        completed = lafc_single_oracle.lafc_single_forward(lafc_sd, fl, mk[0])[0]
        mx = completed.reshape(1, t, 2, -1).max(-1, keepdim=True)[0]
        normed = completed.reshape(1, t, 2, height, width) / mx.unsqueeze(-1)
        masked = fr * (1 - mk)
        out = fgt_oracle.fgt_forward(fgt_sd, masked, normed, mk, num_blocks=num_blocks)
    f = fr[0]
    m = mk[0]
    comp = out * m + f * (1 - m)
    q = lambda x: np.clip((x.permute(0, 2, 3, 1).numpy() + 1) / 2 * 255, 0, 255).astype(np.uint8)  # noqa: E731
    comp_u8, frames_u8 = q(comp), q(f)
    res = metrics_oracle.clip_metrics(comp_u8, frames_u8)
    stages = dict(ids=ids, frames=np.stack(frames), masks=np.stack(masks)[..., 0], flows=np.stack(flows),
                  diffused=np.stack(diffused), completed=completed, normed=normed[0], out=out, comp_u8=comp_u8,
                  frames_u8=frames_u8)
    return dict(l1=res["l1"], l2=res["l2"], psnr=res["psnr"], ssim=res["ssim"], frames=t), stages
