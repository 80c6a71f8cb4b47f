"""Native-resolution output (oracle/native_oracle.py, fgt_b200/native.py, pipeline.video_inpainting(native=True)) on the
CPU: the fixed-point upscale against cv2.resize, the properties the blend window's constants promise, the pipeline glue
with the CPU oracle backend, and the errors."""
import cv2
import numpy as np
import pytest
import scipy.ndimage

from fgt_b200 import pipeline as PL
from fgt_b200 import synth
from oracle import native_oracle as NO


def _sizes(g, n):
    """(H, W, h, w) source / destination pairs: random up- and downscales, one axis at a time, exact integer factors."""
    out = []
    for t in range(n):
        H, W = (int(v) for v in g.integers(2, 80, 2))
        kind = t % 4
        if kind == 0:
            h, w = (int(v) for v in g.integers(2, 240, 2))
        elif kind == 1:
            h, w = (int(g.integers(2, 240)), W) if t % 8 == 1 else (H, int(g.integers(2, 240)))
        elif kind == 2:
            fy, fx = (int(v) for v in g.integers(1, 6, 2))
            h, w = H * fy, W * fx
        else:
            h, w = max(1, H // int(g.integers(1, 4))), max(1, W // int(g.integers(1, 4)))
        out.append((H, W, h, w))
    return out


def test_upscale_within_one_level_of_cv2_resize():
    g = np.random.default_rng(0)
    fractions = []
    for H, W, h, w in _sizes(g, 320):
        comp = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
        got = NO.upscale(comp, h, w)
        want = cv2.resize(comp, (w, h), interpolation=cv2.INTER_LINEAR)
        d = np.abs(got.astype(np.int16) - want)
        assert got.shape == want.shape and d.max() <= 1, (H, W, h, w, int(d.max()))
        fractions.append(float((d != 0).mean()))
    print(f"values off by one level: mean {np.mean(fractions):.2%}, max {np.max(fractions):.2%}, "
          f"{sum(f > 0 for f in fractions)} of {len(fractions)} size pairs")


def test_upscale_at_the_same_size_is_the_identity():
    comp = np.random.default_rng(1).integers(0, 256, (17, 23, 3), dtype=np.uint8)
    assert np.array_equal(NO.upscale(comp, 17, 23), comp)


def _random_hole(g, h, w):
    m = np.zeros((h, w), bool)
    for _ in range(int(g.integers(1, 4))):
        y, x = int(g.integers(-3, h)), int(g.integers(-3, w))
        m[max(y, 0):y + int(g.integers(1, h // 3 + 2)), max(x, 0):x + int(g.integers(1, w // 3 + 2))] = True
    return m


def test_window_is_full_within_r_and_empty_beyond_r_plus_4k():
    g = np.random.default_rng(2)
    for t in range(40):
        h, w = (int(v) for v in g.integers(20, 160, 2))
        imgH, imgW = (int(v) for v in g.integers(8, 64, 2))
        fd = int(g.integers(0, 4))
        hole = _random_hole(g, h, w)
        k, r = NO.native_window(h, w, imgH, imgW, fd)
        c, A = NO.counts(hole[None], h, w, imgH, imgW, fd)
        dist = scipy.ndimage.distance_transform_cdt(~hole, metric="taxicab")      # L1 distance to the hole
        assert (c[0][dist <= r] == A).all() and (c[0][dist > r + 4 * k] == 0).all(), (h, w, imgH, imgW, fd)
        assert c.min() >= 0 and c.max() <= A


def test_working_hole_footprint_is_pure_upscale():
    """Every native pixel whose cv2-nearest working pixel is in the pipeline's working hole (the INTER_NEAREST resize of
    the mask, dilated frame_dilates times) gets out == up."""
    g = np.random.default_rng(3)
    for t in range(60):
        h, w = (int(v) for v in g.integers(16, 300, 2))
        imgH, imgW = (int(v) for v in g.integers(8, 120, 2))
        fd = int(g.integers(0, 4))
        mask = _random_hole(g, h, w).astype(np.uint8) * 255
        if t % 5 == 0:                                          # single-pixel holes are the worst case for nearest
            mask[:] = 0
            mask[int(g.integers(0, h)), int(g.integers(0, w))] = 255
        work = cv2.resize(mask, (imgW, imgH), interpolation=cv2.INTER_NEAREST) != 0
        if fd > 0:
            work = scipy.ndimage.binary_dilation(work, iterations=fd)
        foot = cv2.resize(work.astype(np.uint8), (w, h), interpolation=cv2.INTER_NEAREST) != 0
        comp = g.integers(0, 256, (1, imgH, imgW, 3), dtype=np.uint8)
        frames = g.integers(0, 256, (1, h, w, 3), dtype=np.uint8)
        out = NO.composite_native(comp, frames, mask, fd)[0]
        up = NO.upscale(comp[0], h, w)
        assert np.array_equal(out[foot], up[foot]), (h, w, imgH, imgW, fd)


def test_composite_blends_in_integers():
    g = np.random.default_rng(4)
    comp = g.integers(0, 256, (2, 8, 12, 3), dtype=np.uint8)
    frames = g.integers(0, 256, (2, 30, 40, 3), dtype=np.uint8)
    masks = np.zeros((2, 30, 40), np.uint8)
    masks[0, 10:14, 18:22] = 1
    out = NO.composite_native(comp, frames, masks, 0)
    c, A = NO.counts(masks != 0, 30, 40, 8, 12, 0)
    up = NO.upscale(comp, 30, 40).astype(np.int64)
    want = (c[..., None] * up + (A - c[..., None]) * frames + A // 2) // A
    assert np.array_equal(out, want) and np.array_equal(out[1], frames[1])       # an empty mask returns the frame
    rgb = np.zeros((30, 40, 3), np.uint8)
    rgb[10:14, 18:22, 1] = 7                                                     # one colour channel marks the hole
    assert np.array_equal(NO.composite_native(comp[:1], frames[:1], rgb, 0), out[:1])


class _NativeOracleBackend:
    """The CPU oracle backend with the oracle's composite as its composite_native."""

    def __init__(self, inner):
        self.inner = inner

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def composite_native(self, comp, frames, masks, frame_dilates):
        return NO.composite_native(comp, frames, masks, frame_dilates)


def _oracle_backend(H, W):
    from oracle import fgt_oracle as O
    from oracle.pipeline_oracle import OracleBackend
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (H, W)
    return OracleBackend(synth.raft_state_dict(seed=33),
                         O.strip_net(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=32)),
                         O.strip_net(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=31)))


def test_pipeline_native_output_with_oracle_backend():
    frames, masks = synth.pipeline_clip(seed=5, N=5, H=128, W=192)
    args = PL.make_args(imgH=64, imgW=96, flow_mask_dilates=3, frame_dilates=1)
    be = _NativeOracleBackend(_oracle_backend(64, 96))
    out, st = PL.video_inpainting(frames, masks, be, args, return_stages=True, native=True)
    out = np.stack(out)
    assert out.shape == (5, 128, 192, 3) and out.dtype == np.uint8
    assert st["comp"].shape == (5, 64, 96, 3)
    c, A = NO.counts(np.stack(masks) != 0, 128, 192, 64, 96, 1)
    far = c == 0
    assert far.mean() > 0.5 and np.array_equal(out[far], np.stack(frames)[far])
    assert np.array_equal(out, NO.composite_native(st["comp"], np.stack(frames), np.stack(masks), 1))
    plain = PL.video_inpainting(frames, masks, be, args)
    assert np.array_equal(np.stack(plain), st["comp"])


def test_native_errors():
    frames, masks = synth.pipeline_clip(seed=5, N=3, H=32, W=48)
    be = _NativeOracleBackend(object())
    with pytest.raises(ValueError, match="video_extrapolation"):
        PL.video_inpainting(frames, None, be, PL.make_args(mode="video_extrapolation", imgH=32, imgW=48), native=True)
    with pytest.raises(ValueError, match="mask sizes"):
        PL.video_inpainting(frames, [m[:-1] for m in masks], be, PL.make_args(imgH=32, imgW=48), native=True)
    with pytest.raises(ValueError, match="one size"):
        PL.video_inpainting([frames[0], frames[1][:-2]], masks[:2], be, PL.make_args(imgH=32, imgW=48), native=True)
    with pytest.raises(TypeError, match="composite_native"):
        PL.video_inpainting(frames, masks, object(), PL.make_args(imgH=32, imgW=48), native=True)
    with pytest.raises(SystemExit):
        PL.main(["--path", "x", "--outroot", "y", "--mode", "video_extrapolation", "--native"])
    from fgt_b200 import native
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        native.composite_native(np.zeros((1, 4, 4, 3), np.uint8), np.zeros((1, 8, 8, 3), np.uint8),
                                np.zeros((8, 8), np.uint8), 0, device="cpu")


def test_window_constants_match_the_oracle_and_the_count_limit():
    from fgt_b200 import lib, native
    for h, w, H, W, fd in [(1080, 1920, 256, 432, 0), (1080, 1920, 256, 432, 3), (720, 1280, 720, 1280, 0),
                           (100, 50, 200, 400, 2), (257, 432, 256, 432, 1)]:
        assert native.native_window(h, w, H, W, fd) == NO.native_window(h, w, H, W, fd)
    assert native.native_window(1080, 1920, 256, 432, 0) == (5, 11)
    L = lib.load()
    assert L.fgt_native_workspace(2, 30, 40, 127) == 3 * 2 * 30 * 40
    assert L.fgt_native_workspace(1, 30, 40, 128) < 0
    assert "uint16" in L.fgt_last_error().decode()
    assert L.fgt_native_workspace(0, 30, 40, 1) < 0 and "empty" in L.fgt_last_error().decode()


def test_sharded_backend_delegates_composite_native():
    class Inner:
        def composite_native(self, comp, frames, masks, frame_dilates):
            return "native"

    sb = PL.ShardedBackend.__new__(PL.ShardedBackend)     # the delegation alone; no process group needed
    sb.inner = Inner()
    assert sb.composite_native(None, None, None, 0) == "native"
    sb.inner = object()
    assert not hasattr(sb, "composite_native")
