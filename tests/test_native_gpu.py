"""Native-resolution output on the device (fgt_b200/native.py, csrc/native.cu) against its definition
(oracle/native_oracle.py): byte for byte everywhere, since every step is integer arithmetic."""
import argparse

import cv2
import numpy as np
import pytest
import torch

from fgt_b200 import lib, native
from fgt_b200 import pipeline as PL
from fgt_b200 import synth
from oracle import native_oracle as NO

pytestmark = pytest.mark.gpu


def _inputs(g, B, h, w, imgH, imgW):
    comp = g.integers(0, 256, (B, imgH, imgW, 3), dtype=np.uint8)
    base = cv2.GaussianBlur(g.integers(0, 256, (h, w, 3), dtype=np.uint8), (0, 0), 3)
    frames = np.clip(base[None].astype(np.int16) + g.integers(-20, 21, (B, h, w, 3)), 0, 255).astype(np.uint8)
    return comp, frames


def _object_masks(g, B, h, w):
    m = np.zeros((B, h, w), np.uint8)
    for b in range(B):
        cx, cy = int(w * (0.2 + 0.6 * b / max(B, 1))), int(h * g.uniform(0.3, 0.7))
        cv2.ellipse(m[b], (cx, cy), (int(w * 0.08), int(h * 0.12)), float(g.uniform(0, 180)), 0, 360, 255, -1)
    return m


def _oracle(comp, frames, masks, fd):
    """The definition, frame by frame (its int64 intermediates of a whole 1080p batch would not fit comfortably)."""
    if masks.ndim == 2 or (masks.ndim == 3 and masks.shape != frames.shape[:3]):
        return NO.composite_native(comp, frames, masks, fd)
    return np.concatenate([NO.composite_native(comp[i:i + 1], frames[i:i + 1], masks[i:i + 1], fd)
                           for i in range(len(frames))])


def _same(comp, frames, masks, fd):
    got = native.composite_native(comp, frames, masks, fd).cpu().numpy()
    want = _oracle(comp, frames, masks, fd)
    assert got.shape == want.shape and got.dtype == np.uint8
    assert np.array_equal(got, want), f"{int((got != want).sum())} values differ"
    return got


@pytest.mark.parametrize("B", [1, 7])
@pytest.mark.parametrize("fd", [0, 3])
def test_1080p_from_256x432_per_frame_masks(B, fd):
    g = np.random.default_rng(10 * B + fd)
    comp, frames = _inputs(g, B, 1080, 1920, 256, 432)
    _same(comp, frames, _object_masks(g, B, 1080, 1920), fd)


def test_batch_of_80_per_frame_and_shared_masks():
    g = np.random.default_rng(80)
    comp, frames = _inputs(g, 80, 360, 640, 128, 216)
    masks = _object_masks(g, 80, 360, 640)
    _same(comp, frames, masks, 0)
    _same(comp, frames, masks[17], 3)                                   # one mask for the whole batch, counted once


def test_1080p_shared_mask():
    g = np.random.default_rng(2)
    comp, frames = _inputs(g, 7, 1080, 1920, 256, 432)
    _same(comp, frames, _object_masks(g, 1, 1080, 1920)[0], 0)


@pytest.mark.parametrize("fd", [0, 3])
def test_same_size_s_equals_1(fd):
    g = np.random.default_rng(3 + fd)
    comp, frames = _inputs(g, 3, 720, 1280, 720, 1280)
    masks = _object_masks(g, 3, 720, 1280)
    got = _same(comp, frames, masks, fd)
    hole = masks != 0
    assert np.array_equal(got[hole], comp[hole])                         # at s = 1 the hole is comp itself


def test_empty_full_border_and_single_pixel_masks():
    g = np.random.default_rng(4)
    B, h, w = 8, 200, 300
    comp, frames = _inputs(g, B, h, w, 64, 96)
    m = np.zeros((B, h, w), np.uint8)
    m[1] = 1                                                             # full
    m[2, :12, 100:140] = 1                                               # touching each border
    m[3, -5:, 10:60] = 1
    m[4, 50:90, :3] = 1
    m[5, 120:150, -1:] = 1
    m[6, 77, 133] = 1                                                    # single pixels
    m[7, 0, 0] = m[7, h - 1, w - 1] = m[7, 100, 150] = 1
    got = _same(comp, frames, m, 0)
    assert np.array_equal(got[0], frames[0])                             # empty: the frame unchanged
    assert np.array_equal(got[1], NO.upscale(comp[1], h, w))             # full: the upscaled result
    for fd in (0, 3):
        _same(comp[:3], frames[:3], m[:3], fd)


def test_rgb_watermark_masks():
    g = np.random.default_rng(5)
    comp, frames = _inputs(g, 4, 270, 480, 128, 216)
    m = np.zeros((4, 270, 480, 3), np.uint8)
    for b in range(4):
        m[b, 30 + 10 * b:90 + 10 * b, 40:200, b % 3] = 255                # one colour channel marks the hole
    m[3, 200:230, 300:400] = 128
    _same(comp, frames, m, 0)
    _same(comp, frames, m[2], 3)                                         # one colour mask for every frame


def test_argument_errors_surface_the_library_text_through_lib_call():
    g = np.random.default_rng(6)
    comp, frames = _inputs(g, 2, 60, 80, 30, 40)
    masks = np.zeros((2, 60, 80), np.uint8)
    with pytest.raises(RuntimeError, match="3 channels"):
        native.composite_native(np.zeros((2, 30, 40, 4), np.uint8), np.zeros((2, 60, 80, 4), np.uint8), masks, 0)
    with pytest.raises(RuntimeError, match="uint16 count"):
        native.composite_native(np.zeros((1, 1, 1, 3), np.uint8), np.zeros((1, 300, 300, 3), np.uint8),
                                np.zeros((300, 300), np.uint8), 0)
    with pytest.raises(ValueError):
        native.composite_native(comp, frames, np.zeros((2, 60, 81), np.uint8), 0)
    dev = torch.device("cuda:0")
    c, f = torch.from_numpy(comp).to(dev), torch.from_numpy(frames).to(dev)
    ws = torch.zeros(lib.call("fgt_native_workspace", 2, 60, 80, 2), dtype=torch.uint8, device=dev)
    out = torch.empty_like(f)
    with pytest.raises(RuntimeError, match="not the working size"):            # counts built for k = 3, comp gives k = 2
        lib.call("fgt_native_composite", c, 2, 30, 40, f, 60, 80, 3, 0, 3, ws, ws.numel(), out)
    with pytest.raises(RuntimeError, match="workspace of"):
        lib.call("fgt_native_count", f, 2, 60, 80, 2, ws, ws.numel() - 1)
    with pytest.raises(RuntimeError, match="empty size"):
        lib.call("fgt_native_composite", c, 0, 30, 40, f, 60, 80, 3, 0, 2, ws, ws.numel(), out)
    with pytest.raises(RuntimeError, match="alias"):
        lib.call("fgt_native_composite", c, 2, 30, 40, f, 60, 80, 3, 0, 2, ws, ws.numel(), f)


def _backend(H, W):
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
    return PL.GpuBackend(raft, lafc, fgt, device=dev)


def test_command_line_native_writes_input_size_frames(tmp_path):
    import os

    from fgt_b200 import io as IO
    from tests.test_pipeline import _write_ckpts
    frames, masks = synth.pipeline_clip(seed=5, N=5, H=128, W=192)
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    sds = dict(fgt=synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=31),
               lafc=synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=32),
               raft=synth.raft_state_dict(seed=33))
    tmp = str(tmp_path)
    _write_ckpts(tmp, cfg, sds)
    IO.write_frames(os.path.join(tmp, "in"), frames, mp4=False)
    IO.write_frames(os.path.join(tmp, "msk"), [np.repeat(m[..., None], 3, -1) for m in masks], mp4=False)
    out = PL.main(["--path", os.path.join(tmp, "in", "frames"), "--path_mask", os.path.join(tmp, "msk", "frames"),
                   "--outroot", os.path.join(tmp, "out"), "--raft_model", os.path.join(tmp, "raft.pth"),
                   "--lafc_ckpts", os.path.join(tmp, "lafc"), "--fgt_ckpts", os.path.join(tmp, "fgt"),
                   "--imgH", "64", "--imgW", "96", "--flow_mask_dilates", "3", "--frame_dilates", "1", "--native"])
    back = IO.read_frames(os.path.join(tmp, "out", "frames"))
    assert len(back) == 5 and all(b.shape == (128, 192, 3) and np.array_equal(a, b) for a, b in zip(out, back))
    c, _ = NO.counts(np.stack(masks) != 0, 128, 192, 64, 96, 1)
    assert np.array_equal(np.stack(back)[c == 0], np.stack(frames)[c == 0])


@pytest.mark.parametrize("mode", ["object_removal", "watermark_removal"])
def test_pipeline_native_on_gpu_backend_equals_oracle_composite(mode):
    frames, masks = synth.pipeline_clip(seed=5, N=7, H=128, W=192)
    if mode == "watermark_removal":
        masks = [np.repeat(m[..., None], 3, -1) for m in masks]
    args = PL.make_args(imgH=64, imgW=96, flow_mask_dilates=3, frame_dilates=1, mode=mode)
    be = _backend(64, 96)
    out, st = PL.video_inpainting(frames, masks, be, args, return_stages=True, native=True)
    out = np.stack(out)
    assert out.shape == (7, 128, 192, 3) and st["comp"].shape == (7, 64, 96, 3)
    assert np.array_equal(out, NO.composite_native(st["comp"], np.stack(frames), np.stack(masks), 1))
