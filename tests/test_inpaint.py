"""TELEA inpainting (csrc/inpaint.cu) on the CPU: fgt_inpaint_telea_host runs the kernels' plan and level-by-level
fill through the same __host__ __device__ routines, and must equal cv2.inpaint(..., cv2.INPAINT_TELEA) byte for byte.
Needs only the built library."""
import cv2
import numpy as np
import pytest

from fgt_b200 import inpaint


def _image(g, H, W, C, kind):
    shp = (H, W, C) if C == 3 else (H, W)
    if kind == "random":
        return g.integers(0, 256, shp, dtype=np.uint8)
    if kind == "blurred":
        return cv2.GaussianBlur(g.integers(0, 256, shp, dtype=np.uint8), (0, 0), float(g.uniform(1, 6)))
    yy, xx = np.mgrid[:H, :W]
    ramp = (yy * g.uniform(0.5, 4) + xx * g.uniform(0.5, 4)) % 256
    img = np.stack([ramp + 40 * c for c in range(C)], -1) if C == 3 else ramp
    return (np.asarray(img) % 256).astype(np.uint8)


def _blobs(g, H, W):
    return (cv2.GaussianBlur(g.random((H, W)), (0, 0), 2) > g.uniform(0.5, 0.56)).astype(np.uint8)


def _rects(g, H, W):
    m = np.zeros((H, W), np.uint8)
    for _ in range(int(g.integers(1, 4))):                  # several components, some touching the borders
        y0, x0 = int(g.integers(-3, H)), int(g.integers(-3, W))
        m[max(y0, 0):y0 + int(g.integers(1, 15)), max(x0, 0):x0 + int(g.integers(1, 15))] = 255
    return m


def _same(img, m, r):
    want = cv2.inpaint(img, m, r, cv2.INPAINT_TELEA)
    got = inpaint.inpaint_telea_host(img, m, r)
    assert got.shape == want.shape and got.dtype == np.uint8
    assert np.array_equal(got, want), f"{int((got != want).sum())} bytes differ (radius {r}, hole {int((m != 0).sum())} px)"


@pytest.mark.parametrize("kind", ["random", "blurred", "gradient"])
@pytest.mark.parametrize("masks", ["rects", "blobs"])
def test_random_cases_match_cv2(kind, masks):
    g = np.random.default_rng(10 * ("random", "blurred", "gradient").index(kind) + ("rects", "blobs").index(masks))
    for t in range(60):
        H, W = (int(v) for v in g.integers(8, 70, 2))
        C = 3 if t % 3 else 1
        m = _rects(g, H, W) if masks == "rects" else _blobs(g, H, W)
        _same(_image(g, H, W, C, kind), m, 3)


@pytest.mark.parametrize("seed", range(4))
def test_speckle_sweep_radius_3(seed):
    # small images with speckled masks reach the most border and tie cases per pixel; 2000 cases per seed
    g = np.random.default_rng(1000 + seed)
    for t in range(2000):
        H, W = (int(v) for v in g.integers(2, 40, 2))
        img = g.integers(0, 256, (H, W), dtype=np.uint8) if t % 2 else _image(g, H, W, 3, "blurred")
        m = (g.random((H, W)) < g.uniform(0.05, 0.6)).astype(np.uint8)
        _same(img, m, 3)


def test_radius_is_rounded_like_cv2_and_only_3_is_accepted():
    g = np.random.default_rng(5)
    img, m = _image(g, 30, 40, 3, "blurred"), _rects(g, 30, 40)
    for r in (2.51, 3.0, 3.49):                              # cvRound -> 3
        assert np.array_equal(inpaint.inpaint_telea_host(img, m, r), cv2.inpaint(img, m, r, cv2.INPAINT_TELEA)), r
    for r in (0.2, 1, 2, 2.5, 3.5, 4, 5, 12, 100, 150.0, -4.0):   # rounds (and clamps) to another radius
        with pytest.raises(RuntimeError, match="only radius 3 is supported"):
            inpaint.inpaint_telea_host(img, m, r)


def test_holes_at_and_near_every_border():
    g = np.random.default_rng(11)
    img = _image(g, 20, 24, 3, "blurred")
    for d in range(4):                                       # at the border, next to it, two and three pixels away
        for side in range(4):
            m = np.zeros((20, 24), np.uint8)
            if side == 0:
                m[d:d + 4, 8:14] = 1
            elif side == 1:
                m[16 - d:20 - d, 8:14] = 1
            elif side == 2:
                m[7:12, d:d + 4] = 1
            else:
                m[7:12, 20 - d:24 - d] = 1
            _same(img, m, 3)


def test_degenerate_masks_return_the_image():
    g = np.random.default_rng(2)
    img = _image(g, 20, 24, 3, "random")
    for m in (np.zeros((20, 24), np.uint8), np.ones((20, 24), np.uint8)):
        out = inpaint.inpaint_telea_host(img, m, 3)
        assert np.array_equal(out, img)
        _same(img, m, 3)
    one = np.zeros((20, 24), np.uint8)
    one[9, 13] = 1
    _same(img, one, 3)


def test_extrapolation_ring_and_object_hole_256x432():
    g = np.random.default_rng(3)
    img = _image(g, 256, 432, 3, "blurred")
    ring = np.ones((256, 432), np.uint8)
    ring[64:192, 108:324] = 0
    _same(img, ring, 3)
    obj = np.zeros((256, 432), np.uint8)
    cv2.ellipse(obj, (200, 130), (70, 50), 20, 0, 360, 1, -1)
    _same(img, cv2.dilate(obj, np.ones((9, 9), np.uint8)), 3)


def test_hole_pixels_keep_their_own_values_until_filled():
    # the hole is not zeroed: pixels read before they are filled must be read from the input
    g = np.random.default_rng(4)
    for t in range(20):
        img = _image(g, 40, 50, 3, "random")
        _same(img, _blobs(g, 40, 50), 3)


def test_argument_errors():
    img = np.zeros((10, 12, 3), np.uint8)
    m = np.zeros((10, 12), np.uint8)
    with pytest.raises(RuntimeError, match="1 or 3 channels"):
        inpaint.inpaint_telea_host(np.zeros((10, 12, 2), np.uint8), m)
    with pytest.raises(RuntimeError, match="at least 2x2"):
        inpaint.inpaint_telea_host(np.zeros((1, 12, 3), np.uint8), np.zeros((1, 12), np.uint8))
    with pytest.raises(RuntimeError, match="NaN"):
        inpaint.inpaint_telea_host(img, m, float("nan"))
    with pytest.raises(ValueError):
        inpaint.inpaint_telea_host(img, np.zeros((10, 11), np.uint8))


def test_sharded_backend_delegates_the_inpaint_calls():
    from fgt_b200 import pipeline as PL

    class Inner:
        def inpaint_telea(self, images, masks):
            return "telea"

        def prepare_gradients(self, video, mask, mask_dilated):
            return "grads"

    sb = PL.ShardedBackend.__new__(PL.ShardedBackend)     # the delegation alone; no process group needed
    sb.inner = Inner()
    assert sb.inpaint_telea(None, None) == "telea" and sb.prepare_gradients(None, None, None) == "grads"
    sb.inner = object()
    assert not hasattr(sb, "inpaint_telea") and not hasattr(sb, "prepare_gradients")
