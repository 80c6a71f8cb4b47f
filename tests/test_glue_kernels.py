"""The driver-glue interpreter (tests/glue_emulator.py) against the library calls the glue kernels replace, on the CPU:
scipy.ndimage.binary_dilation / binary_fill_holes, cv2.resize (INTER_NEAREST, INTER_LINEAR), torch.max, and the
reference driver's numpy float32 window compositing and gradient preparation. Bit for bit, on hand-built inputs that
take each decision both ways: 1-pixel-wide images, foreground on the border and on the boundary between batch images,
holes joined to the outside only diagonally, mask values 1 / 7 / 255, nearest-neighbour ratios where the double step
`1 / (OW / W)` and exact integer division disagree, bilinear coordinates that land on integers, cv2's exact-2x
INTER_AREA switch and its unclamped vertical fraction at the first and last rows, NaN / +-0 / +-inf planes, frames on
every k / 255 and model outputs one ulp either side of every uint8 boundary.

cv2 INTER_LINEAR is stated for two-channel images (the driver's flows) and other channel counts but 1, 3 and 4, which
cv2 hands to IPP: there its outputs differ from the statement in most pixels (pinned below as a divergence).
tests/test_glue_kernels_gpu.py replays the CUDA kernels against the same interpreter.
"""
import numpy as np
import pytest
import torch

from tests import glue_emulator as G

F32 = np.float32


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    return np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ------------------------------------------------------------------------------------------------------- masks
def _edge_masks():
    """[B,H,W] uint8 batches: every image touches the border and the next image's first row."""
    out = []
    g = np.random.default_rng(11)
    for H, W in ((1, 1), (1, 9), (9, 1), (2, 2), (7, 11), (33, 40)):
        m = (g.random((3, H, W)) < 0.35).astype(np.uint8)
        m[:, -1, :] = np.array([1, 7, 255], np.uint8)[:, None]        # last row set, next image's first row clear
        m[1, 0, :] = 0
        out.append(m)
    # a hole joined to the outside only diagonally, a closed ring, a ring open by one pixel; values 1 / 7 / 255
    d = np.zeros((3, 9, 9), np.uint8)
    d[0, 2:7, 2:7] = 1
    d[0, 3:6, 3:6] = 0
    d[0, 2, 2] = 0                                                    # corner hole cell touches (1, 1) diagonally
    d[0, 3, 3] = 0
    d[1, 1:8, 1:8] = 7
    d[1, 2:7, 2:7] = 0
    d[2, 0:5, 0:5] = 255
    d[2, 1:4, 1:4] = 0
    d[2, 0, 2] = 0                                                    # hole open to the top border
    d[2, 8, :] = 255
    out.append(d)
    out.append(_spiral(40, 64)[None])
    return out


def _spiral(H, W):
    """tests/test_morph.py's spiral, opened to the top border: a background path that needs many propagation passes."""
    sp = np.ones((H, W), np.uint8)
    sp[:2, W // 2] = 0
    for r in range(2, min(H, W) // 2 - 4, 4):
        sp[r, r:W - r] = 0
        sp[r:H - r, W - r - 1] = 0
        sp[H - r - 1, r + 4:W - r] = 0
        sp[r + 4:H - r, r + 4] = 0
    return sp


@pytest.mark.parametrize("iters", [1, 2, 12])
def test_dilation_equals_scipy(iters):
    import scipy.ndimage
    for m in _edge_masks():
        B, H, W = m.shape
        src, tmp, out = torch.from_numpy(m), torch.full((B, H, W), 0xA5, dtype=torch.uint8), torch.zeros(B, H, W,
                                                                                                         dtype=torch.uint8)
        emu = G.call("fgt_binary_dilate", src, B, H, W, iters, tmp, out)
        ref = np.stack([scipy.ndimage.binary_dilation(x, iterations=iters) for x in m])
        assert np.array_equal(out.numpy(), ref.astype(np.uint8)), (m.shape, iters)
        assert bool(emu.written_mask(tmp).all()) == (iters > 1)


def _fill(m, passes=3):
    B, H, W = m.shape
    fg, reach = torch.from_numpy(m), torch.full((B, H, W), 0xA5, dtype=torch.uint8)
    changed = torch.full((1,), -7, dtype=torch.int32)
    G.call("fgt_fill_holes_init", fg, B, H, W, reach)
    flags = []
    for _ in range(H * W + 1):
        G.call("fgt_fill_holes_pass", fg, B, H, W, reach, changed, passes)
        flags.append(int(changed))
        if not flags[-1]:
            break
    out = torch.full((B, H, W), 0xA5, dtype=torch.uint8)
    G.call("fgt_fill_holes_finish", reach, B, H, W, out)
    return out.numpy(), flags


def test_fill_holes_equals_scipy():
    import scipy.ndimage
    for m in _edge_masks():
        for passes in (1, 3):
            got, flags = _fill(m, passes)
            ref = np.stack([scipy.ndimage.binary_fill_holes(x) for x in m]).astype(np.uint8)
            assert np.array_equal(got, ref), (m.shape, passes)
            assert flags[-1] == 0 and all(flags[:-1])
    got, flags = _fill(_spiral(40, 64)[None], 1)
    assert len(flags) > 4                         # the spiral takes several launches; the last one changes nothing


def test_fill_pass_is_per_line_sequential():
    """One pass reaches along the border rows, then down a whole column run, but not along the row the column run
    turns into: that takes the next pass's row sweep."""
    m = np.ones((1, 6, 6), np.uint8)
    m[0, 0, 1] = 0                                 # border opening
    m[0, 1:5, 1] = 0                               # column run down from it
    m[0, 4, 2:5] = 0                               # row run from its end
    r = G.fill_pass(m != 0, np.zeros((1, 6, 6), bool))
    assert r[0, 0, 1] and r[0, 1:5, 1].all() and not r[0, 4, 2:5].any()
    r = G.fill_pass(m != 0, r)
    assert r[0, 4, 2:5].all()


# ----------------------------------------------------------------------------------------------------- nearest
def _nearest_disagreements(limit=64):
    """(src, dst) sizes up to `limit` where floor(d * (1 / (dst / src))) in double differs from d * src // dst."""
    out = []
    for s in range(1, limit):
        for d in range(1, limit):
            dd = np.arange(d)
            if not np.array_equal(np.floor(dd * (1.0 / (d / s))).astype(np.int64), dd * s // d):
                out.append((s, d))
    return out


def test_nearest_double_step_equals_cv2_where_integer_division_does_not():
    import cv2
    bad = _nearest_disagreements()
    assert bad, "no size pair separates the double step from integer division"
    print(f"\n{len(bad)} size pairs, first {bad[:12]}")
    g = np.random.default_rng(12)
    checked = 0
    for s, d in bad[:40] + [(1, 5), (5, 1), (7, 3), (9, 3), (3, 9)]:
        for C in (1, 3):
            x = g.integers(0, 256, (2, s + 1, s, C), dtype=np.uint8)     # W = s, H = s + 1
            OH, OW = d + 1, d
            out = torch.zeros(2, OH, OW, C, dtype=torch.uint8)
            G.call("fgt_resize_nearest_u8", torch.from_numpy(x), 2, s + 1, s, C, OH, OW, out)
            ref = np.stack([cv2.resize(im, (OW, OH), interpolation=cv2.INTER_NEAREST) for im in x])
            assert np.array_equal(out.numpy(), ref.reshape(out.shape)), (s, d, C)
            checked += 1
    assert checked > 40


# ---------------------------------------------------------------------------------------------------- bilinear
RESIZES = [((270, 480), (240, 432)), ((240, 432), (480, 864)), ((720, 1280), (240, 432)), ((120, 200), (256, 432)),
           ((100, 100), (300, 300)), ((480, 864), (240, 432)), ((2, 2), (1, 1)), ((1, 1), (5, 7)), ((1, 7), (5, 3)),
           ((3, 1), (8, 1)), ((7, 9), (3, 4)), ((4, 8), (8, 16)), ((6, 10), (3, 5))]


def _flows(src, C, seed):
    g = np.random.default_rng(seed)
    x = (g.standard_normal((2,) + src + (C,)) * 5).astype(F32)
    edge = F32([-0.0, 0.0, -0.0, -0.0, 1e-38, -1e30])
    x.reshape(-1)[:min(6, x.size)] = edge[:min(6, x.size)]
    return x


def _bilinear(x, dst, nchw=False, scale=(1.0, 1.0)):
    B = x.shape[0]
    H, W, C = (x.shape[2], x.shape[3], x.shape[1]) if nchw else x.shape[1:]
    out = torch.zeros((B, C) + dst if nchw else (B,) + dst + (C,), dtype=torch.float32)
    G.call("fgt_resize_bilinear_f32", torch.from_numpy(np.ascontiguousarray(x)), B, H, W, C, dst[0], dst[1],
           int(nchw), float(scale[0]), float(scale[1]), out)
    return out.numpy()


@pytest.mark.parametrize("src,dst", RESIZES)
def test_bilinear_equals_cv2_with_the_drivers_channel_scales(src, dst):
    """cv2.resize INTER_LINEAR of [H,W,2] flows, then flow[..., 0] *= W' / W and flow[..., 1] *= H' / H in float32
    (video_inpainting.py:264-270), bit for bit; also with five channels."""
    import cv2
    for C in (2, 5):
        x = _flows(src, C, 13)
        sx, sy = float(dst[1]) / float(src[1]), float(dst[0]) / float(src[0])
        got = _bilinear(x, dst, scale=(sx, sy))
        ref = np.stack([cv2.resize(im, (dst[1], dst[0]), interpolation=cv2.INTER_LINEAR) for im in x])
        ref = ref.reshape(got.shape)
        ref[..., 0] *= sx
        ref[..., 1] *= sy
        assert _bits_equal(got, ref), (src, dst, C, int((got.view(np.uint32) != ref.view(np.uint32)).sum()))


def test_bilinear_exact_2x_is_cv2s_area_path_and_its_edge_rows_keep_the_fraction():
    """The two places where plain bilinear arithmetic is not cv2: exactly 2x smaller (cv2 runs INTER_AREA) and, on
    upscales, the first and last output rows, where cv2 keeps the vertical fraction and reads the edge row twice
    (r * (1 - f) + r * f, not r). The statement reproduces both; clamping the fraction would miss exactly those rows."""
    import cv2
    x = _flows((120, 200), 2, 14)
    ref = np.stack([cv2.resize(im, (432, 256), interpolation=cv2.INTER_LINEAR) for im in x])
    got = G.resize_linear(x, 256, 432)
    assert _bits_equal(got, ref)
    clamped = G._interp(x, G._cv_x(432, 200), G._cv_x(256, 120))
    diff = np.nonzero((clamped.view(np.uint32) != ref.view(np.uint32)).any(axis=(0, 2, 3)))[0]
    assert len(diff) and set(diff.tolist()) <= {0, 255}, diff
    x = _flows((480, 864), 2, 15)
    ref = np.stack([cv2.resize(im, (432, 240), interpolation=cv2.INTER_LINEAR) for im in x])
    assert _bits_equal(G.resize_linear(x, 240, 432), ref)
    plain = G._interp(x, G._cv_x(432, 864), G._cv_y(240, 480))
    assert (plain.view(np.uint32) != ref.view(np.uint32)).mean() > 0.05


def test_bilinear_coordinates_on_integers_and_one_pixel_sources():
    """Integer-ratio upscales put every coordinate on k + 0.25 / 0.75 and downscales by 3 on integers (fraction 0: the
    right tap weighs 0); one-pixel sources in either direction broadcast their pixel."""
    import cv2
    for src, dst in (((4, 6), (4, 18)), ((9, 12), (3, 4)), ((1, 1), (3, 3)), ((1, 5), (4, 5)), ((5, 1), (5, 4))):
        x = _flows(src, 2, 16)
        ref = np.stack([cv2.resize(im, (dst[1], dst[0]), interpolation=cv2.INTER_LINEAR) for im in x])
        assert _bits_equal(_bilinear(x, dst), ref), (src, dst)
    assert np.array_equal(G._cv_x(4, 12)[2], np.zeros(4, F32))


def test_bilinear_ipp_channel_counts_diverge_from_the_statement():
    """For C = 1, 3 and 4 cv2 does not run its own arithmetic (it defers to IPP): the statement, and the kernel, are
    cv2's for other channel counts only. Pinned so that a change in cv2's dispatch is noticed."""
    import cv2
    for C in (1, 3, 4):
        x = _flows((270, 480), C, 17)
        ref = np.stack([cv2.resize(im, (432, 240), interpolation=cv2.INTER_LINEAR) for im in x]).reshape(2, 240, 432, C)
        assert (G.resize_linear(x, 240, 432).view(np.uint32) != ref.view(np.uint32)).mean() > 0.2, C


def test_bilinear_nchw_equals_f_interpolate():
    """The nchw form is ATen's vectorised CPU kernel: FMA coordinates and FMA interpolation, bit for bit with
    F.interpolate at the driver's sizes. On small images ATen takes a scalar path that rounds differently (pinned at
    within 1e-7 of the largest value). fma32 is checked against exact rational arithmetic."""
    import fractions
    import torch.nn.functional as F
    g = np.random.default_rng(18)
    a, b, c = (g.standard_normal(2000).astype(F32) * F32(2.0) ** g.integers(-30, 30, 2000).astype(F32) for _ in range(3))
    Q = fractions.Fraction

    def round32(v):   # the exact value v to the nearest fp32, ties to even
        f = F32(float(v))
        cands = sorted({f, np.nextafter(f, F32(-np.inf)), np.nextafter(f, F32(np.inf))},
                       key=lambda y: (abs(Q(float(y)) - v), int(np.array(y).view(np.uint32)) & 1))
        return cands[0]

    want = [round32(Q(float(p)) * Q(float(q)) + Q(float(r))) for p, q, r in zip(a, b, c)]
    assert _bits_equal(G.fma32(a, b, c), np.array(want, F32))
    for src, dst in (((270, 480), (240, 432)), ((120, 200), (256, 432)), ((480, 864), (240, 432)), ((1, 1), (3, 5)),
                     ((7, 9), (3, 4))):
        x = (g.random((2, 3) + src) * 255).astype(F32)
        got = _bilinear(x, dst, nchw=True)
        ref = F.interpolate(torch.from_numpy(x), size=dst, mode="bilinear", align_corners=False).numpy()
        if src[0] * src[1] > 1000:
            assert _bits_equal(got, ref), (src, dst)
        assert np.abs(got - ref).max() <= 1e-7 * np.abs(ref).max(), (src, dst)


# --------------------------------------------------------------------------------------------------- plane max
def _plane_max(x):
    x = np.ascontiguousarray(x, dtype=F32)
    out = torch.zeros(x.shape[0], dtype=torch.float32)
    G.call("fgt_plane_max", torch.from_numpy(x), x.shape[0], x.shape[1], out)
    return out.numpy()


@pytest.mark.parametrize("n", [1, 255, 256, 257])
def test_plane_max_equals_torch_max(n):
    g = np.random.default_rng(19 + n)
    P = 8
    x = g.standard_normal((P, n)).astype(F32)
    x[0] = -np.abs(x[0]) - 1                           # all negative
    x[1] = -0.0
    x[1, n // 2] = 0.0                                 # -0 and +0
    x[2] = -np.abs(x[2])
    x[2, -1] = -0.0                                    # only -0 at the top
    x[3, n // 3] = np.nan                              # NaN: torch.max propagates it
    x[4, -1] = np.inf
    x[5] = -np.inf
    x[6, 0] = -np.inf
    got = _plane_max(x)
    ref = torch.from_numpy(x).max(dim=1).values.numpy()
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan) and nan[3]
    assert np.array_equal(got[~nan], ref[~nan])       # torch's sign of a zero maximum depends on its order
    assert not np.signbit(got[1]) and (n == 1 or np.signbit(got[2])) and got[4] == np.inf and got[5] == -np.inf


# ------------------------------------------------------------------------------------ window gather / compose
def _ulp_neighbours_of_u8_boundaries():
    """Model outputs o one fp32 ulp either side of, and on, each o with (o + 1) / 2 * 255 = k, and -1 / +1."""
    k = np.arange(256, dtype=np.float64)
    o = (k / 255 * 2 - 1).astype(F32)
    vals = np.concatenate([o, np.nextafter(o, F32(-2)), np.nextafter(o, F32(2)), F32([-1, 1])]).astype(F32)
    return np.clip(vals, F32(-1), F32(1))


def _window_case(H=16, W=24, N=4, seed=20):
    g = np.random.default_rng(seed)
    HW = H * W
    frames = g.random((N, 3, HW)).astype(F32)
    k255 = (np.arange(256) / 255).astype(F32)
    frames.reshape(-1)[:2 * 256] = np.concatenate([k255, np.nextafter(k255, F32(2))])   # every k / 255 and above
    masks = (g.random((N, HW)) < 0.5).astype(np.uint8) * np.array([1, 7, 255, 1], np.uint8)[:N, None]
    flows = g.standard_normal((N, 2, HW)).astype(F32)
    fmax = g.standard_normal((N, 2)).astype(F32)
    fmax[0] = (0.0, -0.0)                              # x / 0: IEEE inf / NaN, as numpy divides
    fmax[1, 0] = -2.5
    filled = g.uniform(-1, 1, (N, 3, HW)).astype(F32)
    b = _ulp_neighbours_of_u8_boundaries()
    filled.reshape(-1)[:b.size] = b
    return frames, masks, flows, fmax, filled, H, W


def test_window_gather_equals_reference_arithmetic():
    frames, masks, flows, fmax, filled, H, W = _window_case()
    N, HW = masks.shape
    ids = np.array([2, 0, 3], np.int32)
    t = len(ids)
    of, ofl, om = (torch.full((t, c, HW), np.nan, dtype=torch.float32) for c in (3, 2, 1))
    G.call("fgt_window_gather", torch.from_numpy(frames), torch.from_numpy(masks), torch.from_numpy(flows),
           torch.from_numpy(fmax), torch.from_numpy(ids), t, H, W, of, ofl, om)
    m = torch.from_numpy((masks[ids] != 0).astype(F32))[:, None]
    # the reference in torch float32 (:695, :719-722, norm_flows :402-407)
    normed = torch.from_numpy(frames[ids]) * 2 - 1
    assert _bits_equal(of.numpy(), (normed * (1 - m)).numpy())
    assert _bits_equal(ofl.numpy(), (torch.from_numpy(flows[ids]) / torch.from_numpy(fmax[ids])[:, :, None]).numpy())
    assert _bits_equal(om.numpy(), m.numpy())
    assert np.isinf(ofl.numpy()[1, 0]).any() and np.isnan(ofl.numpy()[1]).sum() == 0


def test_window_compose_and_u8_equal_reference_arithmetic():
    """First and later visits of the same frames, as the driver composes them (:725-745) in numpy float32; the u8
    conversions truncate at every k / 255 frame value and every model-output boundary, and the 0.5 / 0.5 averages of
    odd sums land on .5, which the final astype(uint8) truncates."""
    frames, masks, flows, fmax, filled, H, W = _window_case()
    N, HW = masks.shape
    comp = torch.full((N, H, W, 3), np.nan, dtype=torch.float32)
    want = [None] * N
    visits = [([1, 3], [1, 1]), ([3, 0], [0, 1]), ([1, 3, 0], [0, 0, 0])]
    g = np.random.default_rng(21)
    for ids, first in visits:
        k = len(ids)
        out = filled[g.permutation(N)[:k]].copy() if ids != visits[0][0] else filled[:k].copy()
        G.call("fgt_window_compose", torch.from_numpy(out), torch.from_numpy(frames), torch.from_numpy(masks),
               torch.tensor(ids, dtype=torch.int32), torch.tensor(first, dtype=torch.uint8), k, H, W, comp)
        f = (out.transpose(0, 2, 1).reshape(k, H, W, 3) + F32(1)) / F32(2) * F32(255)    # filled_frames (:725-726)
        for i, idx in enumerate(ids):
            valid_frame = frames[idx].T.reshape(H, W, 3) * F32(255.0)
            valid_mask = (masks[idx] != 0).astype(F32).reshape(H, W, 1)
            c = f[i].astype(np.uint8) * valid_mask + valid_frame.astype(np.uint8) * (1 - valid_mask)
            want[idx] = c if want[idx] is None else want[idx].astype(F32) * F32(0.5) + c.astype(F32) * F32(0.5)
    for idx in (0, 1, 3):
        assert _bits_equal(comp.numpy()[idx], np.ascontiguousarray(want[idx], dtype=F32)), idx
    u8 = torch.zeros(N * HW * 3, dtype=torch.uint8)
    sel = comp[[0, 1, 3]].contiguous()
    G.call("fgt_comp_to_u8", sel, sel.numel(), u8)
    ref = np.stack([want[i] for i in (0, 1, 3)]).astype(np.uint8).reshape(-1)
    assert np.array_equal(u8.numpy()[:ref.size], ref)
    assert (np.modf(sel.numpy())[0] == 0.5).any()
    a = (_ulp_neighbours_of_u8_boundaries() + F32(1)) / F32(2) * F32(255)
    assert len(np.unique(a.astype(np.uint8))) == 256 and (a != np.trunc(a)).any()


# ---------------------------------------------------------------------------------------------- gradient prep
def test_grad_prep_equals_reference_arithmetic():
    """All 256 levels through *255 -> uint8 -> /255, k / 255 and the next float down; forward differences at the last
    row and column; pixels inside and outside mask_dilated (video_inpainting.py:588-615)."""
    g = np.random.default_rng(22)
    B, H, W = 2, 12, 32
    v = g.random((B, H, W, 3)).astype(F32)
    k255 = (np.arange(256) / 255).astype(F32)
    v.reshape(-1)[:512] = np.concatenate([k255, np.nextafter(k255, F32(-1))]).clip(0, 1)
    hole = g.random((B, H, W)) < 0.2
    md = hole | (g.random((B, H, W)) < 0.2)
    md[:, -1, ::2] = True
    md[:, ::3, -1] = True
    u8 = torch.zeros(B, H, W, 3, dtype=torch.uint8)
    G.call("fgt_grad_prep_pre", torch.from_numpy(v), torch.from_numpy(hole.astype(np.uint8)), B, H, W, u8)
    gx, gy = (torch.full((B, H, W, 3), np.nan, dtype=torch.float32) for _ in range(2))
    filled = torch.from_numpy(g.integers(0, 256, (B, H, W, 3), dtype=np.uint8))   # stands in for the TELEA output
    filled.view(-1)[:256] = torch.arange(256, dtype=torch.uint8)
    G.call("fgt_grad_prep_post", filled, torch.from_numpy(md.astype(np.uint8)), B, H, W, gx, gy)
    for b in range(B):
        img = v[b].copy()
        img[hole[b], :] = 0
        assert np.array_equal(u8.numpy()[b], (img * 255).astype(np.uint8))
        img = filled.numpy()[b].astype(np.float32) / 255.0
        rx = np.concatenate((np.diff(img, axis=1), np.zeros((H, 1, 3), dtype=np.float32)), axis=1)
        ry = np.concatenate((np.diff(img, axis=0), np.zeros((1, W, 3), dtype=np.float32)), axis=0)
        rx[md[b], :] = 0
        ry[md[b], :] = 0
        assert _bits_equal(gx.numpy()[b], rx) and _bits_equal(gy.numpy()[b], ry)
    levels = np.unique(u8.numpy())
    assert len(levels) == 256
