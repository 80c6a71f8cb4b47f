"""GPU parity of the driver's mask / resize glue kernels (fgt_b200/morph.py, csrc/morph.cu) against the library calls
they replace, evaluated on the same seeded inputs: scipy.ndimage.binary_dilation / binary_fill_holes and cv2.resize
(bit-exact for masks), cv2.resize INTER_LINEAR of two-channel flows and F.interpolate bilinear (bit-exact as well)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _masks(seed, B=6, H=240, W=432):
    g = np.random.default_rng(seed)
    m = np.zeros((B, H, W), np.uint8)
    for b in range(B):
        for _ in range(4):  # rectangles, rings (holes to fill), border-touching blobs, speckles
            y0, x0 = g.integers(0, H - 40), g.integers(0, W - 60)
            h, w = g.integers(10, 40), g.integers(10, 60)
            m[b, y0:y0 + h, x0:x0 + w] = 255
            if g.random() < 0.6:
                m[b, y0 + 3:y0 + h - 3, x0 + 3:x0 + w - 3] = 0
        m[b, :5, 100:140] = 1
        m[b, H - 30:, W - 8:] = 7
        ys, xs = g.integers(0, H, 50), g.integers(0, W, 50)
        m[b, ys, xs] = 1
    m[0] = 0
    # a spiral: background path that needs many propagation passes
    sp = np.ones((H, W), np.uint8)
    y, x, k = 2, 2, 0
    for r in range(2, 60, 4):
        sp[r, r:W - r] = 0; sp[r:H - r, W - r - 1] = 0; sp[H - r - 1, r + 4:W - r] = 0; sp[r + 4:H - r, r + 4] = 0
    m[1] = sp
    return m


@pytest.mark.parametrize("iters", [1, 4, 12])
def test_binary_dilation_bit_exact(iters):
    import scipy.ndimage
    from fgt_b200 import morph
    m = _masks(1)
    got = morph.binary_dilation(m, iterations=iters).cpu().numpy()
    ref = np.stack([scipy.ndimage.binary_dilation(x, iterations=iters) for x in m])
    assert got.dtype == bool and (got == ref).all()


def test_binary_fill_holes_bit_exact():
    import scipy.ndimage
    from fgt_b200 import morph
    m = _masks(2)
    got = morph.binary_fill_holes(m).cpu().numpy()
    ref = np.stack([scipy.ndimage.binary_fill_holes(x) for x in m])
    assert (got == ref).all()
    assert got[1].sum() == ref[1].sum()


@pytest.mark.parametrize("src,dst", [((480, 864), (240, 432)), ((270, 480), (240, 432)), ((120, 200), (256, 432))])
def test_resize_nearest_and_bilinear(src, dst):
    import cv2
    import torch.nn.functional as F
    from fgt_b200 import morph
    g = np.random.default_rng(3)
    m = (g.random((3,) + src) < 0.3).astype(np.uint8) * 255
    got = morph.resize_nearest(m, dst).cpu().numpy()
    ref = np.stack([cv2.resize(x, dsize=(dst[1], dst[0]), interpolation=cv2.INTER_NEAREST) for x in m])
    assert (got == ref).all()
    fl = (g.standard_normal((3,) + src + (2,)) * 5).astype(np.float32)
    sx, sy = dst[1] / src[1], dst[0] / src[0]
    got = morph.resize_bilinear(fl, dst, channel_scale=(sx, sy)).cpu().numpy()
    ref = np.stack([cv2.resize(x, (dst[1], dst[0]), interpolation=cv2.INTER_LINEAR) for x in fl])
    ref[..., 0] *= sx
    ref[..., 1] *= sy
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))     # cv2's INTER_AREA at the exact 2x as well
    img = torch.from_numpy((g.random((2, 3) + src) * 255).astype(np.float32))
    got = morph.resize_bilinear(img, dst, layout="nchw").cpu()
    ref = F.interpolate(img, size=dst, mode="bilinear", align_corners=False)
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32))    # ATen's CPU arithmetic, FMAs included
