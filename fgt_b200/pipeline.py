"""The driver's object-removal pipeline (tool/video_inpainting.py:418-745, `video_inpainting(args)`) on arrays
instead of directories, with every heavy stage on the GPU:

    frames, masks ──► RAFT flows (batched pairs) ──► flow diffusion (batched CG) + LAFC completion
                 ──► gradient propagation ──► Poisson blending (batched LSQR) ──► FGT windows + compositing

The calls the reference makes to third-party image code run as device kernels when the backend provides them
(`GpuBackend` does): `cv2.resize` of flows and masks (:264-267,:544-546), `scipy.ndimage.binary_dilation /
binary_fill_holes` (:549-561,:637-640), and — with `GpuBackend(..., host_inpaint=False)` — `cv2.inpaint` (TELEA,
:316-320,:591-599,:663-671, byte-identical, fgt_b200/inpaint.py) with the gradient preparation around it. By default
TELEA stays on the host pool, where it is faster; the `F.interpolate` of the input frames (:478-483) is host-side
too. The stage implementations come from a backend object; `GpuBackend`
(default) binds the fgt_b200 modules, and the parity tests plug the CPU oracle into the same glue, so the glue
itself is verified against a full run of the unmodified reference driver (tests/golden/pipeline_*.npz).
There is no CPU fallback in this module: GpuBackend raises without a CUDA device.
With `native=True` the result is returned at the input frames' size instead of the working size (fgt_b200/native.py).
"""
import argparse
import os
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np
import scipy.ndimage
import torch
import torch.nn.functional as F

HOST_THREADS = max(1, min(8, os.cpu_count() or 1))   # per-frame host work (TELEA, differences) runs on a small pool
# GpuBackend keeps cv2.inpaint on the host pool unless built with host_inpaint=False: the device TELEA is byte-identical
# but its serial planning made it slower than 8 cv2 threads at the driver's sizes on an H100 (DESIGN §8)
HOST_INPAINT_DEFAULT = True


def _frame_major(n, h, w, c=None, dtype=np.float32):
    """Zero array indexed [H,W,(C,)N] like the driver's clips but stored frame-major, so that a frame `a[..., i]` is
    contiguous (the driver's own layout makes every per-frame operation a stride-N gather)."""
    base = np.zeros((n, h, w) + (() if c is None else (c,)), dtype=dtype)
    return np.moveaxis(base, 0, -1)


def _per_frame(fn, n):
    if HOST_THREADS == 1 or n == 1:
        return [fn(i) for i in range(n)]
    with ThreadPoolExecutor(max_workers=min(HOST_THREADS, n)) as pool:
        return list(pool.map(fn, range(n)))


DEFAULTS = dict(mode="object_removal", imgH=256, imgW=432, flow_mask_dilates=8, frame_dilates=0, consistencyThres=5.0,
                alpha=0.1, Nonlocal=False, step=10, num_ref=-1, neighbor_stride=5, raft_iters=20, H_scale=2.0, W_scale=2.0)
MODES = ("object_removal", "watermark_removal", "video_extrapolation")


def make_args(**kw):
    """Namespace with the driver's argparse defaults (:764-855) overridden by keyword."""
    unknown = set(kw) - set(DEFAULTS)
    if unknown:
        raise TypeError(f"unknown pipeline options: {sorted(unknown)}")
    return argparse.Namespace(**{**DEFAULTS, **kw})


def indices_gen(pivot, interval, frames, t):
    """indicesGen (:90-100): `frames` indices centred on pivot, reflected at both ends of [0, t-1]."""
    out = []
    for i in range(-(frames // 2), frames // 2 + 1):
        idx = abs(pivot + interval * i)
        out.append(2 * (t - 1) - idx if idx > t - 1 else idx)
    return out


def gradient_mask(mask):
    """gradient_mask (:74-87): the mask OR-ed with itself shifted up and left (pixels whose forward difference
    touches the hole)."""
    m = np.asarray(mask).astype(bool)
    up = np.zeros_like(m); up[:-1] = m[1:]
    left = np.zeros_like(m); left[:, :-1] = m[:, 1:]
    return m | up | left


# ------------------------------------------------------------------------------------------------ stages
def load_clip(frames_u8, args, masks_u8=None):
    """:452-497 — uint8 RGB frames [N,h,w,3] -> (video [N,3,imgH,imgW], video_flow [N,3,flowH,flowW]) float32 0..255.
    RAFT sees frames at twice the working resolution when imgH < 350 (:440-443). In watermark_removal mode the frames
    are multiplied by (1 - mask) at their native size before any resizing (:454-473; masks [N,h,w] or [N,h,w,3],
    non-zero = watermark)."""
    flow_hw = (args.imgH * 2, args.imgW * 2) if args.imgH < 350 else (args.imgH, args.imgW)
    video, video_flow = [], []
    for k, fr in enumerate(frames_u8):
        t = torch.from_numpy(np.ascontiguousarray(fr).astype(np.uint8)).permute(2, 0, 1).float().unsqueeze(0)
        if masks_u8 is not None:
            m = np.asarray(masks_u8[k]).astype(np.uint8)
            m = torch.from_numpy(np.ascontiguousarray(m if m.ndim == 3 else m[..., None])).permute(2, 0, 1).float().unsqueeze(0)
            m[m > 0] = 1
            t = t * (1 - m)
        t = F.interpolate(t, size=(args.imgH, args.imgW), mode="bilinear", align_corners=False)
        video.append(t)
        video_flow.append(F.interpolate(t, size=flow_hw, mode="bilinear", align_corners=False))
    return torch.cat(video, 0), torch.cat(video_flow, 0)


def extrapolate(video, flow_f, flow_b, h_scale, w_scale, backend=None):
    """extrapolation (:286-335): a canvas H_scale x W_scale as large (rounded down to multiples of 4) with the clip in
    the middle; the border is the hole. The frames are TELEA-inpainted into the border right away (all frames in one
    device batch with one shared mask when the backend has `inpaint_telea`), the flows are zero there.
    Returns (video, flow_f, flow_b, flow_mask [H',W'] bool, mask_dilated [H',W'] bool)."""
    H, W, _, N = video.shape
    He, We = int(h_scale * H), int(w_scale * W)
    He, We = He - He % 4, We - We % 4
    y0, x0 = int((He - H) / 2), int((We - W) / 2)
    flow_mask = np.ones((He, We), dtype=bool)
    flow_mask[y0:y0 + H, x0:x0 + W] = False
    big = _frame_major(N, He, We, 3)
    big[y0:y0 + H, x0:x0 + W] = video

    def fill(i):
        big[:, :, :, i] = cv2.inpaint((big[:, :, :, i] * 255).astype(np.uint8), flow_mask.astype(np.uint8), 3,
                                      cv2.INPAINT_TELEA).astype(np.float32) / 255.0

    if backend is not None and hasattr(backend, "inpaint_telea"):
        frames = np.moveaxis(big, -1, 0)                                  # [N,He,We,3] view
        done = backend.inpaint_telea((frames * 255).astype(np.uint8), flow_mask.astype(np.uint8))
        frames[...] = done.astype(np.float32) / 255.0
    else:
        _per_frame(fill, N)
    ff = np.zeros((He, We, 2, N - 1), dtype=np.float32)
    fb = np.zeros((He, We, 2, N - 1), dtype=np.float32)
    ff[y0:y0 + H, x0:x0 + W] = flow_f
    fb[y0:y0 + H, x0:x0 + W] = flow_b
    return big, ff, fb, flow_mask, gradient_mask(flow_mask)


def compute_flows(backend, video_flow, args, mode):
    """calculate_flow (:232-283): RAFT on consecutive frames (forward i -> i+1, backward i+1 -> i), resized to the
    working resolution with the flow vectors rescaled. Returns [imgH,imgW,2,N-1] float32."""
    a, b = (video_flow[:-1], video_flow[1:]) if mode == "forward" else (video_flow[1:], video_flow[:-1])
    flows = backend.raft_pairs(a, b, args.raft_iters)                   # [N-1,2,h,w]
    out = np.empty((args.imgH, args.imgW, 2, flows.shape[0]), dtype=np.float32)   # (the driver grows it by concatenation)
    if hasattr(backend, "resize_flows") and flows.shape[0] and tuple(flows.shape[2:]) != (args.imgH, args.imgW):
        # device kernel for cv2.resize(INTER_LINEAR) + the rescaling of the flow vectors, all pairs in one batch
        out[...] = np.moveaxis(backend.resize_flows(flows, args.imgH, args.imgW), 0, -1)
        return out
    for i in range(flows.shape[0]):
        flow = np.ascontiguousarray(flows[i].transpose(1, 2, 0))
        h, w = flow.shape[:2]
        if h != args.imgH or w != args.imgW:
            flow = cv2.resize(flow, (args.imgW, args.imgH), cv2.INTER_LINEAR)   # same positional call as the driver
            flow[:, :, 0] *= float(args.imgW) / float(w)
            flow[:, :, 1] *= float(args.imgH) / float(h)
        out[..., i] = flow
    return out


def prepare_masks(masks_u8, args, backend=None):
    """:539-567 — per-frame uint8 masks [N,h,w] (non-zero = hole) -> (mask, mask_dilated, flow_mask) bool [H,W,N].
    A backend with `dilate_masks` (the GPU backend) runs the resize + both dilations of all frames as batched device
    kernels (bit-identical to cv2.resize INTER_NEAREST / scipy.ndimage.binary_dilation)."""
    if backend is not None and hasattr(backend, "dilate_masks") and len(masks_u8) and \
            all(np.asarray(m).ndim == 2 and np.asarray(m).shape == np.asarray(masks_u8[0]).shape for m in masks_u8):
        m0 = backend.resize_masks(np.stack([np.asarray(m).astype(np.uint8) for m in masks_u8], 0), args.imgH, args.imgW)
        fm = backend.dilate_masks(m0, args.flow_mask_dilates) if args.flow_mask_dilates > 0 else m0
        mk = backend.dilate_masks(m0, args.frame_dilates) if args.frame_dilates > 0 else m0
        st = lambda a: np.moveaxis(np.ascontiguousarray(a).astype(bool), 0, -1)
        # (without dilation the driver keeps the resized uint8 values; every consumer only tests them for non-zero)
        return st(mk), st(np.stack([gradient_mask(x) for x in mk.astype(bool)], 0)), st(fm)
    mask, dilated, flow_mask = [], [], []
    for m in masks_u8:
        m = np.asarray(m)
        if m.ndim == 3:                                   # a colour mask file: the driver reads it with .convert("L") (:543)
            from PIL import Image
            m = np.array(Image.fromarray(m.astype(np.uint8)).convert("L"))
        m = cv2.resize(np.ascontiguousarray(m).astype(np.uint8), dsize=(args.imgW, args.imgH), interpolation=cv2.INTER_NEAREST)
        flow_mask.append(scipy.ndimage.binary_dilation(m, iterations=args.flow_mask_dilates) if args.flow_mask_dilates > 0 else m)
        if args.frame_dilates > 0:
            m = scipy.ndimage.binary_dilation(m, iterations=args.frame_dilates)
        mask.append(m)
        dilated.append(gradient_mask(m))
    st = lambda xs: np.moveaxis(np.stack(xs, 0).astype(bool), 0, -1)        # [H,W,N] view, frame-major storage
    return st(mask), st(dilated), st(flow_mask)


def complete_flows(backend, flows, flow_mask, mode, num_flows, flow_interval):
    """complete_flow (:338-385): diffuse the holes of every flow, run LAFC on (pivot ± interval) triplets, keep the
    network output inside the hole and the measured flow outside. flows [H,W,2,N-1] -> [H,W,2,N-1] float32."""
    masks = np.moveaxis(flow_mask, -1, 0)[..., None]                     # [N,H,W,1]
    masks = masks[:-1] if mode == "forward" else masks[1:]
    fl = np.moveaxis(flows, -1, 0)                                       # [N-1,H,W,2]
    diffused = backend.diffusion(fl, masks)                              # list of [H,W,2] float64
    to_cthw = lambda a: np.ascontiguousarray(np.transpose(np.stack(a, 0) if isinstance(a, list) else a, (3, 0, 1, 2))).astype(np.float32)
    fl_t, mk_t, df_t = to_cthw(fl), to_cthw(masks), to_cthw(diffused)    # [c,t,H,W]
    t = df_t.shape[1]
    triplets = [indices_gen(i, flow_interval, num_flows, t) for i in range(t)]
    out = backend.lafc_complete(fl_t, mk_t, df_t, triplets, num_flows // 2)   # [t,2,H,W]
    return np.ascontiguousarray(np.transpose(out, (2, 3, 1, 0)))


def prepare_gradients(video, mask, mask_dilated, backend=None):
    """:583-614 — zero the hole (in place, like the driver), TELEA-inpaint it for a plausible initialisation, take
    forward differences and zero them wherever they touch the hole. video [H,W,3,N] float32 (BGR, 0..1). A backend
    with `prepare_gradients` runs the whole stage on the device (bit-identical)."""
    if backend is not None and hasattr(backend, "prepare_gradients"):
        return backend.prepare_gradients(video, mask, mask_dilated)
    H, W, _, N = video.shape
    gx = _frame_major(N, H, W, 3)                      # last column / row stay zero (:601-606)
    gy = _frame_major(N, H, W, 3)

    def one(i):
        img = video[:, :, :, i]
        img[mask[:, :, i], :] = 0
        img = cv2.inpaint((img * 255).astype(np.uint8), mask[:, :, i].astype(np.uint8), 3, cv2.INPAINT_TELEA).astype(np.float32) / 255.0
        gx[:, :W - 1, :, i] = np.diff(img, axis=1)
        gy[:H - 1, :, :, i] = np.diff(img, axis=0)
        gx[mask_dilated[:, :, i], :, i] = 0
        gy[mask_dilated[:, :, i], :, i] = 0

    _per_frame(one, N)                                  # frames are independent; each task writes its own frame
    return gx, gy


def blend_frames(backend, video, gx, gy, mask, mask_gradient):
    """:636-681 — fill the holes of the propagated-gradient mask, Poisson-blend every frame that still has a hole
    (all of them in one batch), TELEA-inpaint what the blend could not reach, mark it green in the frames handed to
    the transformer. Updates `video` and `mask` in place like the driver; returns the list of frames."""
    H, W, _, N = video.shape

    def fill(i):
        mask_gradient[:, :, i] = scipy.ndimage.binary_fill_holes(mask_gradient[:, :, i]).astype(bool)

    if hasattr(backend, "fill_holes"):                   # batched device kernel, bit-identical to scipy's
        mask_gradient[...] = np.moveaxis(backend.fill_holes(np.moveaxis(mask_gradient, -1, 0)), 0, -1)
    else:
        _per_frame(fill, N)
    todo = [i for i in range(N) if mask[:, :, i].sum() > 0]

    def solve(ids):
        return backend.poisson_frames([video[:, :, :, i] for i in ids], [gx[:, 0:W - 1, :, i] for i in ids],
                                      [gy[0:H - 1, :, :, i] for i in ids], [mask[:, :, i] for i in ids],
                                      [mask_gradient[:, :, i] for i in ids])

    # The driver wraps each frame's blend in try/except and falls back to (video_comp[..., i], mask[..., i]) (:648-660).
    # The batched solve is retried frame by frame when it fails, so one bad frame cannot take the clip down.
    blends = []
    if todo:
        try:
            blends = solve(todo)
        except Exception:  # noqa: BLE001 - mirrors the driver's bare except
            for i in todo:
                try:
                    blends.append(solve([i])[0])
                except Exception:  # noqa: BLE001
                    blends.append((video[:, :, :, i].astype(np.float64), mask[:, :, i].copy()))
    slot = {i: k for k, i in enumerate(todo)}
    filled = None
    if todo and hasattr(backend, "inpaint_telea"):       # every frame's leftover TELEA in one device batch
        filled = backend.inpaint_telea(np.stack([(np.clip(b, 0, 1.0) * 255).astype(np.uint8) for b, _ in blends], 0),
                                       np.stack([u.astype(np.uint8) for _, u in blends], 0))

    def finish(i):
        if i not in slot:
            return video[:, :, :, i]
        blend, unfilled = blends[slot[i]]
        blend = np.clip(blend, 0, 1.0)
        u8 = filled[slot[i]] if filled is not None else \
            cv2.inpaint((blend * 255).astype(np.uint8), unfilled.astype(np.uint8), 3, cv2.INPAINT_TELEA)
        tmp = u8.astype(np.float32) / 255.0
        blend[unfilled, :] = tmp[unfilled, :]
        video[:, :, :, i] = blend
        mask[:, :, i] = unfilled
        shown = blend.copy()
        shown[unfilled, :] = [0, 1.0, 0]          # green = not filled by propagation (:678-679); masked out for the model
        return shown

    return _per_frame(finish, N)


# ------------------------------------------------------------------------------------------------ backend
class GpuBackend:
    """Stage implementations on the fgt_b200 kernels. raft / lafc / fgt are the drop-in modules (already on the
    device, weights loaded); lafc_config provides num_flows / flow_interval like the driver's LAFC yaml."""

    def __init__(self, raft, lafc, fgt, device=None, raft_batch=4, host_inpaint=HOST_INPAINT_DEFAULT):
        if not torch.cuda.is_available():
            raise RuntimeError("fgt_b200.pipeline.GpuBackend needs a CUDA (sm_90a) device; there is no CPU fallback")
        self.dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.raft, self.lafc, self.fgt = raft, lafc, fgt
        self.fgt_model = fgt          # the callable the FGT stage evaluates per window (ShardedBackend swaps it)
        self.raft_batch = raft_batch
        if not host_inpaint:          # opt-in: TELEA and the gradient preparation on the device (byte-identical)
            self.inpaint_telea, self.prepare_gradients = self._inpaint_telea, self._prepare_gradients

    def raft_pairs(self, img1, img2, iters):
        outs = []
        with torch.no_grad():
            for s in range(0, img1.shape[0], self.raft_batch):
                a, b = img1[s:s + self.raft_batch].to(self.dev), img2[s:s + self.raft_batch].to(self.dev)
                _, up = self.raft(a, b, iters=iters, test_mode=True)
                outs.append(up.float().cpu())
        return torch.cat(outs, 0).numpy()

    def diffusion(self, flows, masks):
        from .regionfill import diffusion
        return diffusion(flows, masks)

    # ---- the driver's mask / resize glue as device kernels (fgt_b200/morph.py): numpy in, numpy out
    def resize_masks(self, masks, H, W):
        from . import morph
        return masks if tuple(masks.shape[1:]) == (H, W) else morph.resize_nearest(masks, (H, W), device=self.dev).cpu().numpy()

    def dilate_masks(self, masks, iterations):
        from . import morph
        return morph.binary_dilation(masks, iterations, device=self.dev).cpu().numpy()

    def fill_holes(self, masks):
        from . import morph
        return morph.binary_fill_holes(masks, device=self.dev).cpu().numpy()

    def resize_flows(self, flows, H, W):
        """[n,2,h,w] RAFT flows -> [n,H,W,2] at the working resolution, vectors rescaled (:264-268)."""
        from . import morph
        n, _, h, w = flows.shape
        x = torch.as_tensor(flows).to(self.dev).permute(0, 2, 3, 1).contiguous()
        return morph.resize_bilinear(x, (H, W), channel_scale=(float(W) / float(w), float(H) / float(h)),
                                     device=self.dev).cpu().numpy()

    def flow_images(self, flows, convert_to_bgr=False):
        """flow_viz.flow_to_image of every flow in [n,H,W,2] float32 in one batched device call -> numpy uint8
        [n,H,W,3] (fgt_b200/flowviz.py)."""
        from . import flowviz
        return flowviz.flow_to_image(np.ascontiguousarray(flows, dtype=np.float32), convert_to_bgr, device=self.dev)

    def _inpaint_telea(self, images, masks):
        """cv2.inpaint(..., 3, INPAINT_TELEA) of uint8 [B,H,W,3] with masks [B,H,W] or one [H,W] -> numpy uint8."""
        from . import inpaint
        return inpaint.inpaint_telea(images, masks, 3, device=self.dev).cpu().numpy()

    def _prepare_gradients(self, video, mask, mask_dilated):
        from . import inpaint
        return inpaint.prepare_gradients(video, mask, mask_dilated, device=self.dev)

    def composite_native(self, comp, frames, masks, frame_dilates):
        """The working-resolution result pasted into the input frames at their size (fgt_b200/native.py) -> numpy
        uint8 [N,h,w,3]."""
        from . import native
        return native.composite_native(comp, frames, masks, frame_dilates, device=self.dev).cpu().numpy()

    def lafc_complete(self, flows, masks, diffused, triplets, pivot):
        fl, mk, df = (torch.from_numpy(a).to(self.dev).unsqueeze(0) for a in (flows, masks, diffused))   # [1,c,t,H,W]
        out = []
        with torch.no_grad():
            for idx in triplets:
                cand_masks = mk[:, :, idx]
                res = self.lafc(df[:, :, idx], cand_masks, None)
                res = res[0] if isinstance(res, (tuple, list)) else res
                pm = cand_masks[:, :, pivot]
                out.append(res * pm + fl[:, :, idx][:, :, pivot] * (1 - pm))
        return torch.cat(out, 0).float().cpu().numpy()

    def propagate(self, args, gx, gy, mask, mask_gradient, flow_f, flow_b):
        from .propagation import get_flowNN_gradient
        return get_flowNN_gradient(args, gx, gy, mask, mask_gradient, flow_f, flow_b, None, None, device=str(self.dev))

    POISSON_BYTES_PER_PIXEL = 364   # fp64 solver state (u, v, w, x, target, result) + the 2*H*W per-iteration scalar slots
    POISSON_BUDGET_BYTES = 8 << 30  # frames per batch are bounded by this much device memory (results are per-frame independent)

    def poisson_frames(self, trg, gx, gy, hole, gmask):
        from .poisson import poisson_blend_batch
        st = lambda xs: np.ascontiguousarray(np.stack(xs, 0))
        n = len(trg)
        if n == 0:
            return []
        H, W = trg[0].shape[:2]
        per = max(1, int(self.POISSON_BUDGET_BYTES // (self.POISSON_BYTES_PER_PIXEL * H * W)))
        res = []
        for s in range(0, n, per):
            e = min(n, s + per)
            t = st(trg[s:e])
            out, unf = poisson_blend_batch(t, st(gx[s:e]), st(gy[s:e]), st(hole[s:e]), st(gmask[s:e]), device=self.dev)
            if t.dtype == np.float32:    # every value of the blend is then a float32 (float64(float32(x)) in the hole, the
                out = out.float()        # float32 target outside): half the bytes back over the bus, widened exactly on the host
            out, unf = out.cpu().numpy().astype(np.float64), unf.cpu().numpy()
            res += [(out[i], unf[i]) for i in range(out.shape[0])]
        return res

    def fgt_stage(self, frame_blends, mask, flow_f, step, num_ref, neighbor_stride):
        from .clip import inpaint_clip
        return inpaint_clip(self.fgt_model, frame_blends, mask, flow_f, step, num_ref, neighbor_stride, device=self.dev)


class ShardedBackend:
    """Multi-GPU execution of the pipeline (SURVEY §8e): wraps any backend and shards the independent work items
    of every stage over the ranks of a torch.distributed group — RAFT pairs, diffusion solves, LAFC triplets, Poisson
    frames, FGT windows (balanced by frames per window) — with one all-gather per stage, so that every rank holds the
    complete stage output (131 MB of flows at N=80, 240x432) before the next stage starts. The propagation is
    sequential over frames and runs replicated. One process per GPU (torchrun); NCCL moves device tensors over
    NVLink, gloo (CPU tests) host tensors. Results are bit-identical to the unsharded backend: every item is
    computed by exactly the same call, only by a different rank."""

    def __init__(self, inner, group=None):
        import torch.distributed as dist
        if not dist.is_initialized():
            raise RuntimeError("ShardedBackend needs an initialised torch.distributed process group")
        self.inner, self.group, self.dist = inner, group, dist
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        nccl = dist.get_backend(group) == "nccl"
        self.comm_dev = torch.device("cuda", torch.cuda.current_device()) if nccl else torch.device("cpu")

    def __getattr__(self, name):
        # the mask / resize glue kernels are cheap and run replicated on every rank: delegate when the inner backend has them
        if name in ("resize_masks", "dilate_masks", "fill_holes", "resize_flows", "inpaint_telea", "prepare_gradients",
                    "composite_native") and hasattr(self.inner, name):
            return getattr(self.inner, name)
        raise AttributeError(name)

    def _mine(self, n, costs=None):
        from .parallel import shard_items
        return shard_items(n, self.rank, self.world, costs)

    def _gather(self, local, n, costs=None):
        """local: array [k, ...] of this rank's items (k may be 0 -> pass the trailing shape via a [0, ...] array);
        returns [n, ...] in item order on every rank."""
        from .parallel import shard_items
        owners = [shard_items(n, r, self.world, costs) for r in range(self.world)]
        kmax = max(len(o) for o in owners)
        local = np.ascontiguousarray(local)
        if n == 0 or kmax == 0:                          # nothing to exchange (e.g. a one-frame clip has no RAFT pairs)
            return np.zeros((0,) + local.shape[1:], dtype=local.dtype)
        pad = np.zeros((kmax,) + local.shape[1:], dtype=local.dtype)
        pad[:local.shape[0]] = local
        t = torch.from_numpy(pad.view(np.uint8).reshape(kmax, -1)).to(self.comm_dev)
        parts = [torch.empty_like(t) for _ in range(self.world)]
        self.dist.all_gather(parts, t.contiguous(), group=self.group)           # raw bytes: exact on every backend
        out = np.zeros((n,) + local.shape[1:], dtype=local.dtype)
        for r, ids in enumerate(owners):
            if ids:
                rows = parts[r].cpu().numpy().view(local.dtype).reshape((kmax,) + local.shape[1:])
                out[ids] = rows[:len(ids)]
        return out

    def raft_pairs(self, img1, img2, iters):
        n = img1.shape[0]
        mine = self._mine(n)
        h, w = img1.shape[2], img1.shape[3]
        local = self.inner.raft_pairs(img1[mine], img2[mine], iters) if mine else np.zeros((0, 2, h, w), np.float32)
        return self._gather(np.asarray(local, dtype=np.float32), n)

    def diffusion(self, flows, masks):
        n = flows.shape[0]
        mine = self._mine(n)
        local = np.stack(self.inner.diffusion(flows[mine], masks[mine]), 0) if mine else np.zeros((0,) + flows.shape[1:], np.float64)
        out = self._gather(np.asarray(local, dtype=np.float64), n)
        return [out[i] for i in range(n)]

    def lafc_complete(self, flows, masks, diffused, triplets, pivot):
        n = len(triplets)
        mine = self._mine(n)
        H, W = flows.shape[2], flows.shape[3]
        local = self.inner.lafc_complete(flows, masks, diffused, [triplets[i] for i in mine], pivot) if mine else np.zeros((0, 2, H, W), np.float32)
        return self._gather(np.asarray(local, dtype=np.float32), n)

    def propagate(self, *a):
        return self.inner.propagate(*a)                       # sequential over frames: replicas only

    def poisson_frames(self, trg, gx, gy, hole, gmask):
        n = len(trg)
        if n == 0:
            return []
        mine = self._mine(n)
        pick = lambda xs: [xs[i] for i in mine]
        res = self.inner.poisson_frames(pick(trg), pick(gx), pick(gy), pick(hole), pick(gmask)) if mine else []
        shp = tuple(np.asarray(trg[0]).shape)
        blend = np.stack([r[0] for r in res], 0) if res else np.zeros((0,) + shp, np.float64)
        unf = np.stack([r[1] for r in res], 0).astype(np.uint8) if res else np.zeros((0,) + shp[:2], np.uint8)
        blend, unf = self._gather(np.asarray(blend, dtype=np.float64), n), self._gather(unf, n)
        return [(blend[i], unf[i].astype(bool)) for i in range(n)]

    def fgt_stage(self, frame_blends, mask, flow_f, step, num_ref, neighbor_stride):
        """Windows shard over the ranks (cost = frames per window). Pass 1: the stage runs with a model proxy that
        evaluates only this rank's windows (the others return zeros; the composite of this pass is discarded) and
        keeps their outputs; all-gather; pass 2: the stage runs again with a proxy that replays every window's output,
        so the compositing — including the order-dependent 0.5/0.5 averaging — is exactly the unsharded one."""
        from .parallel import window_schedule
        sched = window_schedule(len(frame_blends), neighbor_stride, step, num_ref)
        costs = [len(nb) + len(ref) for _, nb, ref in sched]
        mine = set(self._mine(len(sched), costs))
        real, kept, calls = self.inner.fgt_model, {}, [0]

        def first_pass(frames, flows, masks):
            wi = calls[0]
            calls[0] += 1
            if wi in mine:
                kept[wi] = real(frames, flows, masks)
                return kept[wi]
            return torch.zeros(frames.shape[1], 3, frames.shape[3], frames.shape[4], dtype=torch.float32, device=frames.device)

        try:
            self.inner.fgt_model = first_pass
            self.inner.fgt_stage(frame_blends, mask, flow_f, step, num_ref, neighbor_stride)
            tmax = max(costs)
            some = next(iter(kept.values())) if kept else None
            H, W = np.asarray(frame_blends[0]).shape[:2]
            local = np.zeros((len(kept), tmax, 3, H, W), np.float32)
            for j, wi in enumerate(sorted(kept)):
                local[j, :costs[wi]] = kept[wi].detach().float().cpu().numpy()
            allw = self._gather(local, len(sched), costs)
            dev = some.device if some is not None else None
            calls[0] = 0

            def second_pass(frames, flows, masks):
                wi = calls[0]
                calls[0] += 1
                return torch.from_numpy(allw[wi, :costs[wi]]).to(frames.device if dev is None else dev)

            self.inner.fgt_model = second_pass
            return self.inner.fgt_stage(frame_blends, mask, flow_f, step, num_ref, neighbor_stride)
        finally:
            self.inner.fgt_model = real


# ------------------------------------------------------------------------------------------------ driver
def _check_native(frames_u8, masks_u8, backend, args):
    if args.mode == "video_extrapolation":
        raise ValueError("native=True: video_extrapolation has no original frame to paste the result into")
    if not hasattr(backend, "composite_native"):
        raise TypeError(f"native=True needs a backend with composite_native ({type(backend).__name__} has none)")
    sizes = {np.asarray(f).shape[:2] for f in frames_u8}
    if len(sizes) != 1:
        raise ValueError(f"native=True needs frames of one size (got {sorted(sizes)})")
    (hw,) = sizes
    bad = [np.asarray(m).shape for m in masks_u8 if np.asarray(m).shape[:2] != hw]
    if bad or len(masks_u8) != len(frames_u8):
        raise ValueError(f"native=True: {len(masks_u8)} masks for {len(frames_u8)} frames of {hw}"
                         + (f"; mask sizes {bad[:3]}" if bad else ""))


def composite_native(backend, comp, frames_u8, masks_u8, args):
    """The working-resolution frames `comp` upscaled to the input size and pasted into the input frames as given (with
    the watermark in watermark_removal) inside a feathered band around the mask (fgt_b200/native.py). Returns a list of
    N uint8 RGB frames [h,w,3]."""
    out = backend.composite_native(np.stack(comp), np.stack([np.asarray(f) for f in frames_u8]),
                                   np.stack([np.asarray(m) for m in masks_u8]), args.frame_dilates)
    return list(np.asarray(out))


def video_inpainting(frames_u8, masks_u8, backend, args=None, num_flows=3, flow_interval=3, return_stages=False,
                     native=False, vis_out=None):
    """The driver on arrays: frames_u8 [N,h,w,3] RGB uint8 (the PNGs the driver reads), masks_u8 [N,h,w] (non-zero =
    remove; ignored by video_extrapolation) -> list of N uint8 RGB frames (what the driver writes to result.mp4).
    `args`: make_args(...), `args.mode` one of object_removal (default), watermark_removal (frames are masked before
    resizing, :454-473), video_extrapolation (the clip is placed in a larger canvas whose border is inpainted,
    :516-537); num_flows / flow_interval are the LAFC config entries the driver reads (:352).
    native=True returns the frames at the input size h x w instead of imgH x imgW: the result is upscaled and pasted
    into the input frames around the mask by `backend.composite_native` (object and watermark removal; every frame and
    mask of one size). With return_stages the working-resolution frames are then in stages["comp"].
    vis_out: a dict that receives what the driver's visualisation switches write (write_visualisations): "flow_f" /
    "flow_b", the RAFT flows at imgH x imgW before video_extrapolation places them on its canvas (--vis_flows);
    "done_f" / "done_b", the completed flows (--vis_completed_flows); "prop_frames", the list of BGR frames after
    propagation, each with its own dtype (float64 where the Poisson blend ran, float32 elsewhere), and "masks_left",
    the [H,W,N] mask of what propagation could not fill (--vis_prop)."""
    args = args or make_args()
    if args.mode not in MODES:
        raise ValueError(f"Accepted modes: {MODES}, but input is {args.mode}")
    if native:
        _check_native(frames_u8, masks_u8, backend, args)
    video, video_flow = load_clip(frames_u8, args, masks_u8 if args.mode == "watermark_removal" else None)
    flow_f = compute_flows(backend, video_flow, args, "forward")
    flow_b = compute_flows(backend, video_flow, args, "backward")
    if vis_out is not None:
        vis_out.update(flow_f=flow_f, flow_b=flow_b)
    # [H,W,3(BGR),N] in 0..1 (:499-501), stored frame-major so that every per-frame view is contiguous
    video = np.moveaxis(np.ascontiguousarray(video.permute(0, 2, 3, 1).numpy()[..., ::-1]) / 255.0, 0, -1)
    assert video.dtype == np.float32
    if args.mode == "video_extrapolation":
        N = video.shape[3]
        video, flow_f, flow_b, fm2, md2 = extrapolate(video, flow_f, flow_b, args.H_scale, args.W_scale, backend)
        tile = lambda m: np.moveaxis(np.repeat(m[None], N, 0), 0, -1)           # the same mask for every frame (:531-535)
        mask, mask_dilated, flow_mask = tile(fm2), tile(md2), tile(fm2)
    else:
        mask, mask_dilated, flow_mask = prepare_masks(masks_u8, args, backend)
    done_f = complete_flows(backend, flow_f, flow_mask, "forward", num_flows, flow_interval)
    done_b = complete_flows(backend, flow_b, flow_mask, "backward", num_flows, flow_interval)
    gx, gy = prepare_gradients(video, mask, mask_dilated, backend)
    gx, gy, mask_gradient = backend.propagate(args, gx, gy, mask, mask_dilated, done_f, done_b)
    frame_blends = blend_frames(backend, video, gx, gy, mask, np.array(mask_gradient, dtype=bool))
    if vis_out is not None:
        vis_out.update(done_f=done_f, done_b=done_b, prop_frames=list(frame_blends), masks_left=mask.copy())
    comp = backend.fgt_stage(frame_blends, mask, done_f, args.step, args.num_ref, args.neighbor_stride)
    out = composite_native(backend, comp, frames_u8, masks_u8, args) if native else comp
    if return_stages:
        stages = dict(flow_f=flow_f, flow_b=flow_b, done_f=done_f, done_b=done_b, mask_gradient=mask_gradient,
                      frame_blends=np.stack(frame_blends), mask=mask)
        if native:
            stages["comp"] = np.stack(comp)
        return out, stages
    return out


# ------------------------------------------------------------------------------------------------ visualisations
def _write_flow_sets(outroot, sub, sets, backend):
    """One directory pair per flow set, as the driver names them: {sub}/{mode}_flo/%05d.flo (Middlebury) and
    {sub}/{mode}_png/%05d.png (flow_viz colours, RGB, written by PIL). sets: [(mode, flows [H,W,2,n])]. Each set is
    coloured in one batched backend call; the files are encoded on the host pool."""
    from . import io as IO
    from PIL import Image
    written = []
    for mode, flows in sets:
        fl = np.ascontiguousarray(np.moveaxis(np.asarray(flows, dtype=np.float32), -1, 0))     # [n,H,W,2]
        fdir, pdir = os.path.join(outroot, sub, mode + "_flo"), os.path.join(outroot, sub, mode + "_png")
        os.makedirs(fdir, exist_ok=True)
        os.makedirs(pdir, exist_ok=True)
        if not fl.shape[0]:
            continue
        imgs = backend.flow_images(fl)

        def one(i):
            IO.write_flo(os.path.join(fdir, "%05d.flo" % i), fl[i])
            Image.fromarray(imgs[i]).save(os.path.join(pdir, "%05d.png" % i))
            return [os.path.join(fdir, "%05d.flo" % i), os.path.join(pdir, "%05d.png" % i)]

        written += sum(_per_frame(one, fl.shape[0]), [])
    return written


def _write_prop(outroot, frames, masks):
    """save_fgcp (:157-177): prop_frames/ and masks_left/ PNGs through cv2.imwrite of the float arrays times 255 (cv2
    rounds them), and the same arrays as .npy files in prop_frames_npy/ and masks_left_npy/."""
    dirs = [os.path.join(outroot, d) for d in ("prop_frames", "masks_left", "prop_frames_npy", "masks_left_npy")]
    for d in dirs:
        os.makedirs(d, exist_ok=True)
    if len(frames) != masks.shape[2]:
        raise ValueError(f"{len(frames)} propagated frames but {masks.shape[2]} masks")

    def one(i):
        fr, mk = frames[i] * 255.0, masks[:, :, i] * 255.0
        paths = [os.path.join(dirs[0], "%05d.png" % i), os.path.join(dirs[1], "%05d.png" % i),
                 os.path.join(dirs[2], "%05d.npy" % i), os.path.join(dirs[3], "%05d.npy" % i)]
        for ok in (cv2.imwrite(paths[0], fr), cv2.imwrite(paths[1], mk)):
            if not ok:
                raise OSError(f"cv2.imwrite could not write {paths[0]} / {paths[1]}")
        np.save(paths[2], fr)
        np.save(paths[3], mk)
        return paths

    return sum(_per_frame(one, len(frames)), [])


def write_visualisations(outroot, vis, backend, vis_flows=False, vis_completed_flows=False, vis_prop=False):
    """The driver's visualisation outputs under `outroot`, from the dict `vis` that video_inpainting(..., vis_out=vis)
    filled: --vis_flows (calculate_flow :241-287) flow/{forward,backward}_{flo,png}/; --vis_completed_flows
    (save_flows :120-155) completed_flow/{forward,backward}_{flo,png}/, coloured like --vis_flows where the driver
    uses cvbase.flow2rgb; --vis_prop (save_fgcp :157-177) prop_frames/, masks_left/ and their _npy twins. The flow
    colours come from backend.flow_images. Returns the paths written."""
    written = []
    if vis_flows:
        written += _write_flow_sets(outroot, "flow", [("forward", vis["flow_f"]), ("backward", vis["flow_b"])], backend)
    if vis_completed_flows:
        written += _write_flow_sets(outroot, "completed_flow", [("forward", vis["done_f"]), ("backward", vis["done_b"])],
                                    backend)
    if vis_prop:
        written += _write_prop(outroot, vis["prop_frames"], vis["masks_left"])
    return written


# ------------------------------------------------------------------------------------------------ command line
def load_ckpt_dir(d):
    """A checkpoint directory of the reference (FGT/train.py:45-50): one *.tar holding `model_state_dict` and one
    *.yaml config. Returns (state_dict, config)."""
    import glob
    import os

    import yaml

    tars, yamls = glob.glob(os.path.join(d, "*.tar")), glob.glob(os.path.join(d, "*.yaml"))
    if len(tars) != 1 or len(yamls) != 1:
        raise FileNotFoundError(f"{d}: expected exactly one *.tar and one *.yaml (found {len(tars)}, {len(yamls)})")
    with open(yamls[0]) as fh:
        return torch.load(tars[0], map_location="cpu")["model_state_dict"], yaml.full_load(fh)


def load_models(raft_model, lafc_ckpts, fgt_ckpts, device, mixed_precision=False, fgt_mixed_precision=False,
                lafc_mixed_precision=False, small=False):
    """initialize_RAFT / initialize_LAFC / initialize_FGT (:186-230) with the drop-in modules: the same checkpoint
    layout (a `module.`-prefixed RAFT state dict; directories holding one *.tar with `model_state_dict` and one
    *.yaml config). mixed_precision: RAFT's fp16 mode (the reference's --mixed_precision, RAFT only).
    fgt_mixed_precision: the FGT generator's fp16 mode (FGT.enable_mixed_precision). lafc_mixed_precision: the LAFC
    flow-completion network's fp16 mode (P3DNet.enable_mixed_precision). The three are independent. small: RAFT's
    small model (the reference's --small; raft_small.SmallRAFT, fp32 only), from a checkpoint of that model. Returns
    (GpuBackend, lafc_config)."""
    from . import raft_small
    from .fgt_model import Model as FGTModel
    from .lafc_model import Model as LAFCModel

    raft = torch.nn.DataParallel(raft_small.make_raft(argparse.Namespace(
        small=bool(small), mixed_precision=bool(mixed_precision), alternate_corr=False)))
    raft.load_state_dict(torch.load(raft_model, map_location="cpu"))
    raft = raft.module.to(device).eval()
    lafc_sd, lafc_cfg = load_ckpt_dir(lafc_ckpts)
    lafc = LAFCModel(lafc_cfg)
    lafc.load_state_dict(lafc_sd)
    lafc.net.enable_mixed_precision(bool(lafc_mixed_precision))
    fgt_sd, fgt_cfg = load_ckpt_dir(fgt_ckpts)
    fgt = FGTModel(fgt_cfg)
    fgt.load_state_dict(fgt_sd)
    fgt.net.enable_mixed_precision(bool(fgt_mixed_precision))
    # inference only: no BatchNorm / dropout in LAFC or FGT (the driver never calls .eval() on them), but be explicit
    return GpuBackend(raft, lafc.to(device).eval(), fgt.to(device).eval(), device=device), lafc_cfg


def arg_parser():
    """The command line of main()."""
    ap = argparse.ArgumentParser(description=main.__doc__)
    ap.add_argument("--path", required=True, help="directory of *.png / *.jpg frames")
    ap.add_argument("--path_mask", default=None, help="directory of masks (non-zero = remove); not needed for video_extrapolation")
    ap.add_argument("--outroot", required=True, help="output directory (frames/%%05d.png, result.mp4)")
    ap.add_argument("--raft_model", default="../LAFC/flowCheckPoint/raft-things.pth")
    ap.add_argument("--lafc_ckpts", default="../LAFC/checkpoint")
    ap.add_argument("--fgt_ckpts", default="../FGT/checkpoint")
    ap.add_argument("--gpu", type=int, default=0)
    ap.add_argument("--native", action="store_true",
                    help="write the frames at the input size: the result is upscaled and pasted into the input frames "
                         "around the mask (object_removal, watermark_removal)")
    ap.add_argument("--mixed_precision", action="store_true",
                    help="run RAFT with fp16 tensor-core operands, as the reference's autocast mode (faster, not "
                         "fp32-accurate)")
    ap.add_argument("--small", action="store_true",
                    help="run RAFT's small model (RAFT-S; --raft_model must then be a small-model checkpoint such as "
                         "raft-small.pth): faster, coarser flow")
    ap.add_argument("--fgt_mixed_precision", action="store_true",
                    help="run the FGT generator with fp16 tensor-core operands, as the reference under CUDA autocast "
                         "(faster, not fp32-accurate; independent of --mixed_precision)")
    ap.add_argument("--lafc_mixed_precision", action="store_true",
                    help="run the LAFC flow-completion network with fp16 tensor-core operands, as the reference under "
                         "CUDA autocast (faster, not fp32-accurate; independent of the other two switches)")
    ap.add_argument("--vis_flows", action="store_true",
                    help="write the RAFT flows as flow/{forward,backward}_flo/*.flo and, coloured on the GPU, "
                         "flow/{forward,backward}_png/*.png")
    ap.add_argument("--vis_completed_flows", action="store_true",
                    help="write the completed flows as completed_flow/{forward,backward}_{flo,png}/")
    ap.add_argument("--vis_prop", action="store_true",
                    help="write the frames after flow-guided propagation (prop_frames/, green where it could not "
                         "fill) and what is left to fill (masks_left/), as PNG and .npy")
    ap.add_argument("--vis_frame", action="store_true",
                    help="accepted for the driver's command line; frames/ is always written")
    for k, v in DEFAULTS.items():
        if k == "mode":
            ap.add_argument("--mode", default=v, choices=list(MODES))
        elif k not in ("Nonlocal", "raft_iters"):
            ap.add_argument("--" + k, type=type(v), default=v)
    return ap


def main(argv=None):
    """`python -m fgt_b200.pipeline --path frames/ --path_mask masks/ --outroot out/ [--mode ...] ...` — the driver's
    command line (:764-855), visualisation switches included (write_visualisations)."""
    from . import io as IO
    ap = arg_parser()
    ns = ap.parse_args(argv)
    if ns.native and ns.mode == "video_extrapolation":
        ap.error("--native: video_extrapolation has no original frame to paste the result into")
    dev = torch.device("cuda", ns.gpu)
    fgt_kw = dict(fgt_mixed_precision=True) if ns.fgt_mixed_precision else {}
    if ns.lafc_mixed_precision:
        fgt_kw["lafc_mixed_precision"] = True
    if ns.small:
        fgt_kw["small"] = True
    backend, lafc_cfg = load_models(ns.raft_model, ns.lafc_ckpts, ns.fgt_ckpts, dev, ns.mixed_precision, **fgt_kw)
    args = make_args(**{k: getattr(ns, k) for k in DEFAULTS if hasattr(ns, k)})
    frames = IO.read_frames(ns.path)
    masks = IO.read_masks(ns.path_mask, rgb=ns.mode == "watermark_removal") if ns.mode != "video_extrapolation" else [None] * len(frames)
    if len(frames) != len(masks):
        raise ValueError(f"{len(frames)} frames but {len(masks)} masks")
    vis = {} if ns.vis_flows or ns.vis_completed_flows or ns.vis_prop else None
    comp = video_inpainting(frames, masks, backend, args, lafc_cfg["num_flows"], lafc_cfg["flow_interval"],
                            native=ns.native, vis_out=vis)
    if vis is not None:
        write_visualisations(ns.outroot, vis, backend, ns.vis_flows, ns.vis_completed_flows, ns.vis_prop)
    written = IO.write_frames(ns.outroot, comp)
    print(f"Done, {len(comp)} frames written to {ns.outroot} ({len(written)} files)")
    return comp


if __name__ == "__main__":
    main()
