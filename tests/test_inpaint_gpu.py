"""TELEA inpainting on the device (fgt_b200/inpaint.py, csrc/inpaint.cu) against cv2.inpaint(..., INPAINT_TELEA), the
host entry of the same routines and the host pipeline stages it replaces: byte for byte everywhere."""
import argparse

import cv2
import numpy as np
import pytest
import torch

from fgt_b200 import inpaint
from fgt_b200 import pipeline as PL
from fgt_b200 import synth

pytestmark = pytest.mark.gpu


def _frames(g, B, H, W, C=3):
    base = cv2.GaussianBlur(g.integers(0, 256, (H, W, C), dtype=np.uint8), (0, 0), 3).reshape(H, W, C)
    noise = g.integers(-20, 21, (B, H, W, C))
    return np.clip(base[None].astype(int) + noise, 0, 255).astype(np.uint8)


def _object_masks(g, B, H, W):
    m = np.zeros((B, H, W), np.uint8)
    for b in range(B):
        cx, cy = int(W * (0.3 + 0.4 * b / max(B, 1))), int(H * g.uniform(0.3, 0.7))
        cv2.ellipse(m[b], (cx, cy), (int(W * 0.12), int(H * 0.15)), float(g.uniform(0, 180)), 0, 360, 1, -1)
        m[b] = cv2.dilate(m[b], np.ones((9, 9), np.uint8))
    return m


def _cv2_all(frames, masks):
    return np.stack([cv2.inpaint(f, masks[i] if masks.ndim == 3 else masks, 3, cv2.INPAINT_TELEA)
                     for i, f in enumerate(frames)])


@pytest.mark.parametrize("B", [1, 7, 80])
def test_batches_per_frame_masks_256x432(B):
    g = np.random.default_rng(B)
    fr, mk = _frames(g, B, 256, 432), _object_masks(g, B, 256, 432)
    got = inpaint.inpaint_telea(fr, mk).cpu().numpy()
    assert np.array_equal(got, _cv2_all(fr, mk))


@pytest.mark.parametrize("B", [1, 80])
def test_shared_extrapolation_mask_256x432(B):
    g = np.random.default_rng(100 + B)
    ring = np.ones((256, 432), np.uint8)
    ring[64:192, 108:324] = 0
    fr = _frames(g, B, 256, 432)
    got = inpaint.inpaint_telea(fr, ring).cpu().numpy()
    assert np.array_equal(got, _cv2_all(fr, ring))


def test_1280x720_hole_at_the_bottom_edge():
    g = np.random.default_rng(9)
    fr = _frames(g, 2, 720, 1280)
    mk = np.zeros((2, 720, 1280), np.uint8)
    cv2.ellipse(mk[0], (640, 690), (160, 100), 0, 0, 360, 1, -1)
    cv2.ellipse(mk[1], (300, 300), (120, 90), 30, 0, 360, 1, -1)
    assert np.array_equal(inpaint.inpaint_telea(fr, mk).cpu().numpy(), _cv2_all(fr, mk))


def test_mixed_empty_and_full_masks_gray_and_single_images():
    g = np.random.default_rng(4)
    fr = _frames(g, 5, 60, 70)
    mk = _object_masks(g, 5, 60, 70)
    mk[1] = 0
    mk[3] = 1
    got = inpaint.inpaint_telea(fr, mk).cpu().numpy()
    assert np.array_equal(got, _cv2_all(fr, mk))
    assert np.array_equal(got[1], fr[1]) and np.array_equal(got[3], fr[3])
    gray = fr[..., 0]
    got1 = inpaint.inpaint_telea(gray[..., None], mk).cpu().numpy()
    assert np.array_equal(got1[..., 0], _cv2_all(gray, mk))
    assert np.array_equal(inpaint.inpaint_telea(fr[2], mk[2]).cpu().numpy(), cv2.inpaint(fr[2], mk[2], 3, cv2.INPAINT_TELEA))
    assert np.array_equal(inpaint.inpaint_telea(gray[2], mk[2]).cpu().numpy(), cv2.inpaint(gray[2], mk[2], 3, cv2.INPAINT_TELEA))


@pytest.mark.parametrize("masks", ["blobs", "speckle"])
def test_kernel_equals_host_entry_and_cv2(masks):
    g = np.random.default_rng(0 if masks == "blobs" else 1)
    fr = _frames(g, 16, 48, 64)
    if masks == "blobs":
        mk = (cv2.GaussianBlur(g.random((16, 48, 64)).transpose(1, 2, 0), (0, 0), 2) > 0.52).astype(np.uint8).transpose(2, 0, 1)
    else:
        mk = (g.random((16, 48, 64)) < 0.3).astype(np.uint8)
    mk = np.ascontiguousarray(mk)
    got = inpaint.inpaint_telea(fr, mk, 3).cpu().numpy()
    for i in range(16):
        assert np.array_equal(got[i], inpaint.inpaint_telea_host(fr[i], mk[i], 3))
        assert np.array_equal(got[i], cv2.inpaint(fr[i], mk[i], 3, cv2.INPAINT_TELEA))


def test_argument_errors():
    fr = np.zeros((2, 10, 12, 3), np.uint8)
    with pytest.raises(ValueError):
        inpaint.inpaint_telea(fr, np.zeros((3, 10, 12), np.uint8))
    with pytest.raises(TypeError):
        inpaint.inpaint_telea(fr.astype(np.float32), np.zeros((10, 12), np.uint8))
    with pytest.raises(RuntimeError, match="only radius 3"):
        inpaint.inpaint_telea(fr, np.zeros((10, 12), np.uint8), 5)
    with pytest.raises(RuntimeError, match="1 or 3 channels"):
        inpaint.inpaint_telea(np.zeros((2, 10, 12, 2), np.uint8), np.zeros((10, 12), np.uint8))


def _video(g, N, H, W):
    v = (_frames(g, N, H, W).astype(np.float32) / 255.0)
    out = PL._frame_major(N, H, W, 3)
    out[...] = np.moveaxis(v, 0, -1)
    return out


def test_prepare_gradients_matches_host_stage():
    g = np.random.default_rng(12)
    N, H, W = 6, 256, 432
    mk = np.moveaxis(_object_masks(g, N, H, W).astype(bool), 0, -1)
    md = np.moveaxis(np.stack([PL.gradient_mask(mk[..., i]) for i in range(N)]), 0, -1)
    v_host = _video(g, N, H, W)
    v_dev = v_host.copy()
    gx_h, gy_h = PL.prepare_gradients(v_host, mk, md)
    gx_d, gy_d = inpaint.prepare_gradients(v_dev, mk, md)
    assert gx_d.dtype == np.float32 and gx_d.shape == gx_h.shape
    assert np.array_equal(gx_d.view(np.uint32), gx_h.view(np.uint32))
    assert np.array_equal(gy_d.view(np.uint32), gy_h.view(np.uint32))
    assert np.array_equal(v_dev.view(np.uint32), v_host.view(np.uint32))          # the hole zeroed in place


def _backend(host_inpaint, H, W):
    from fgt_b200.fgt_model import Model as FGTModel
    from fgt_b200.lafc_model import Model as LAFCModel
    from fgt_b200.raft_model import RAFT
    dev = torch.device("cuda:0")
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (H, W)
    fgt = FGTModel(cfg); fgt.load_state_dict(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=31)); fgt = fgt.to(dev)
    lafc = LAFCModel(dict(synth.CFG_LAFC))
    lafc.load_state_dict(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=32)); lafc = lafc.to(dev)
    raft = RAFT(argparse.Namespace(small=False, mixed_precision=False, alternate_corr=False))
    raft.load_state_dict(synth.raft_state_dict(seed=33)); raft = raft.to(dev).eval()
    return PL.GpuBackend(raft, lafc, fgt, device=dev, host_inpaint=host_inpaint)


class _PoissonReplay:
    """The batched Poisson solve is not bit-reproducible from run to run (two runs of the same backend differ in a few
    blended values), so the first run records its inputs and results and the second run asserts that its inputs are
    bit-identical and gets the recorded results. Everything else runs for real."""

    def __init__(self, inner, tape):
        self.inner, self.tape = inner, tape

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def poisson_frames(self, *lists):
        if "in" not in self.tape:
            self.tape["in"] = [[np.array(x) for x in xs] for xs in lists]
            self.tape["out"] = self.inner.poisson_frames(*lists)
        else:
            for rec, xs in zip(self.tape["in"], lists):
                assert len(rec) == len(xs) and all(np.array_equal(a, np.asarray(b)) for a, b in zip(rec, xs))
        return [(b.copy(), u.copy()) for b, u in self.tape["out"]]


@pytest.mark.parametrize("mode", ["object_removal", "video_extrapolation"])
def test_pipeline_output_unchanged_by_device_inpaint(mode):
    frames, masks = synth.pipeline_clip(seed=5, N=7, H=64, W=96)
    kw = dict(imgH=64, imgW=96, flow_mask_dilates=3, frame_dilates=1, mode=mode)
    if mode == "video_extrapolation":
        kw.update(H_scale=1.5, W_scale=1.5)
    args = PL.make_args(**kw)
    dev_be, host_be = _backend(False, 64, 96), _backend(True, 64, 96)
    assert hasattr(dev_be, "inpaint_telea") and not hasattr(host_be, "inpaint_telea")
    tape = {}
    b, sb = PL.video_inpainting(frames, masks, _PoissonReplay(host_be, tape), args, return_stages=True)
    a, sa = PL.video_inpainting(frames, masks, _PoissonReplay(dev_be, tape), args, return_stages=True)
    a, b = np.stack(a), np.stack(b)
    assert np.array_equal(sa["frame_blends"].view(np.uint8), sb["frame_blends"].view(np.uint8))
    assert a.dtype == np.uint8 and np.array_equal(a, b)


def test_gpu_backend_default_keeps_the_host_inpaint():
    be = _backend(PL.HOST_INPAINT_DEFAULT, 64, 96)
    assert PL.HOST_INPAINT_DEFAULT and not hasattr(be, "inpaint_telea") and not hasattr(be, "prepare_gradients")
