"""The FGT stage of the driver — the window loop around `Model.forward` and the compositing of its output
(tool/video_inpainting.py:686-745) — device-resident: the clip is uploaded once, every window's inputs are
gathered by one kernel, the model output is composed into the clip by one kernel, and one uint8 clip comes
back, instead of a `.cpu()` round trip per window plus one per frame (:726-733). csrc/clip.cu performs the
reference's float32 / uint8 arithmetic operation for operation, so with the same model output the composite is
bit-identical. There is no CPU fallback.
"""
import numpy as np
import torch

from . import lib
from .parallel import window_schedule


def _i32(ids, dev):
    return torch.tensor(list(ids), dtype=torch.int32, device=dev)


def prepare_clip(frame_blends, mask, video_flow_f, device):
    """The driver's tensor preparation (:686-707) up to the device: frameBlends (list of [H,W,3] BGR arrays in
    [0,1], or an [N,H,W,3] array) -> frames [N,3,H,W] float32 RGB; mask [H,W,N] bool -> [N,H,W] uint8; completed
    forward flows [H,W,2,N-1] -> [N,2,H,W] float32 with the last flow repeated (:702-704)."""
    fb = np.stack(frame_blends, 0) if isinstance(frame_blends, (list, tuple)) else np.asarray(frame_blends)
    fb = fb[..., ::-1]                                                         # BGR -> RGB (:688-689)
    frames = torch.from_numpy(np.ascontiguousarray(np.transpose(fb, (0, 3, 1, 2)))).float().to(device)
    masks = torch.from_numpy(np.ascontiguousarray(np.moveaxis(np.asarray(mask), -1, 0)).astype(np.uint8)).to(device)
    fl = np.moveaxis(np.asarray(video_flow_f), -1, 0)                          # [N-1,H,W,2]
    fl = np.concatenate([fl, fl[-1:]], 0)
    flows = torch.from_numpy(np.ascontiguousarray(np.transpose(fl, (0, 3, 1, 2)))).float().to(device)
    return frames.contiguous(), masks.contiguous(), flows.contiguous()


def inpaint_clip_device(model, frames, masks, flows, step=10, num_ref=-1, neighbor_stride=5):
    """frames [N,3,H,W] float32 in [0,1], masks [N,H,W] uint8, flows [N,2,H,W] float32, all on one CUDA device ->
    composed clip uint8 [N,H,W,3] on the device. `model(masked_frames[1,t,3,H,W], flows[1,t,2,H,W],
    masks[1,t,1,H,W]) -> [t,3,H,W]` is the drop-in FGT model (or anything with that signature)."""
    if not frames.is_cuda:
        raise RuntimeError("fgt_b200.clip runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    dev = frames.device
    N, _, H, W = frames.shape
    if tuple(masks.shape) != (N, H, W) or tuple(flows.shape) != (N, 2, H, W):
        raise ValueError(f"clip: masks {tuple(masks.shape)} / flows {tuple(flows.shape)} do not match frames {tuple(frames.shape)}")
    frames, flows = frames.float().contiguous(), flows.float().contiguous()
    masks = (masks != 0).to(torch.uint8).contiguous()
    fmax = torch.empty(N, 2, dtype=torch.float32, device=dev)
    lib.call("fgt_plane_max", flows, N * 2, H * W, fmax)
    comp = torch.empty(N, H, W, 3, dtype=torch.float32, device=dev)
    seen = [False] * N
    for f, neighbor_ids, ref_ids in window_schedule(N, neighbor_stride, step, num_ref):
        ids = neighbor_ids + ref_ids
        t, k = len(ids), len(neighbor_ids)
        d_ids = _i32(ids, dev)
        w_frames = torch.empty(1, t, 3, H, W, dtype=torch.float32, device=dev)
        w_flows = torch.empty(1, t, 2, H, W, dtype=torch.float32, device=dev)
        w_masks = torch.empty(1, t, 1, H, W, dtype=torch.float32, device=dev)
        lib.call("fgt_window_gather", frames, masks, flows, fmax, d_ids, t, H, W, w_frames, w_flows, w_masks)
        with torch.no_grad():
            filled = model(w_frames, w_flows, w_masks)
        filled = filled.float().contiguous()
        if tuple(filled.shape) != (t, 3, H, W):
            raise ValueError(f"clip: model returned {tuple(filled.shape)}, expected {(t, 3, H, W)}")
        first = torch.tensor([0 if seen[i] else 1 for i in neighbor_ids], dtype=torch.uint8, device=dev)
        lib.call("fgt_window_compose", filled, frames, masks, d_ids, first, k, H, W, comp)
        for i in neighbor_ids:
            seen[i] = True
    assert all(seen)
    out = torch.empty(N, H, W, 3, dtype=torch.uint8, device=dev)
    lib.call("fgt_comp_to_u8", comp, comp.numel(), out)
    return out


def inpaint_clip(model, frame_blends, mask, video_flow_f, step=10, num_ref=-1, neighbor_stride=5, device=None):
    """Driver-layout front end (numpy in, list of N uint8 [H,W,3] RGB frames out — `comp_frames` at :745)."""
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("fgt_b200.clip runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    frames, masks, flows = prepare_clip(frame_blends, mask, video_flow_f, dev)
    out = inpaint_clip_device(model, frames, masks, flows, step, num_ref, neighbor_stride).cpu().numpy()
    return [out[i] for i in range(out.shape[0])]
