"""A numpy interpreter of the driver-glue entries of include/fgt_b200.h (mask, resize, window and gradient kernels), for
CPU tensors.

`GlueEmulator` stands in for the ctypes library the way tests/prop_emulator.py's `PropEmulator` does: the entries of
`GLUE_ENTRIES` run here on the CPU storages behind their pointer arguments, every other entry is refused, and every
store is recorded (`records`, `written_bytes`) so that a replay can check the bytes a launch must leave alone.

Semantics are restated from the header and the library calls the entries replace (scipy.ndimage, cv2.resize, torch.max
and the reference driver's numpy float32 arithmetic, tool/video_inpainting.py), not from the kernels' code. Every
float32 operation is a separate numpy float32 operation in the library's order, so each product and sum is rounded once.
- fgt_binary_dilate: `iterations` passes of the 3x3 cross, border 0, into `out` (0 / 1); `tmp` is scratch: addressed
  when iterations > 1, its contents not specified.
- fgt_fill_holes_init: reach = 0. fgt_fill_holes_pass: changed = 0, then `passes` times: every row swept left to right
  (a background pixel becomes reached if it is on the image border or its left neighbour is a reached background
  pixel) and right to left, then every column top-down and bottom-up; changed = 1 if any pixel became reached.
  One thread owns one row or column, so each sweep is sequential along its line and the launch is deterministic.
  fgt_fill_holes_finish: out = 1 where reach == 0.
- fgt_resize_nearest_u8: cv2 INTER_NEAREST, sx = min(floor(dx * (1 / (OW / W))), W - 1) in double, likewise sy.
- fgt_resize_bilinear_f32: `resize_linear` below (cv2 INTER_LINEAR, with cv2's exact-2x switch to INTER_AREA) or, with
  nchw, `resize_aten` (ATen's CPU bilinear kernel, whose FMAs are part of its arithmetic); then channels 0 / 1 times
  fp32 scale_c0 / scale_c1.
- fgt_plane_max: torch.max of every plane; NaN if the plane holds one; a zero maximum is +0 if the plane holds a +0.
- fgt_window_gather / fgt_window_compose / fgt_comp_to_u8: oracle/clip_oracle.py's window arithmetic on one window.
- fgt_grad_prep_pre: u8 = trunc(fp32((hole ? 0 : v) * 255)). fgt_grad_prep_post: fp32(u8 / 255), forward
  differences in float32 (last column / row 0), 0 under mask_dilated.
"""
import numpy as np
import torch

from fgt_b200 import lib
from tests.gemm_emulator import _Refused
from tests.kernel_emulator import KernelEmulator, _raw

GLUE_ENTRIES = ("fgt_binary_dilate", "fgt_fill_holes_init", "fgt_fill_holes_pass", "fgt_fill_holes_finish",
                "fgt_resize_nearest_u8", "fgt_resize_bilinear_f32", "fgt_plane_max", "fgt_window_gather",
                "fgt_window_compose", "fgt_comp_to_u8", "fgt_grad_prep_pre", "fgt_grad_prep_post")
F32 = np.float32


# ------------------------------------------------------------------------------------------- library statements
def dilate_cross(m):
    """One pass of scipy.ndimage.binary_dilation with the 3x3 cross, border 0, of bool images [..., H, W]."""
    o = m.copy()
    o[..., 1:, :] |= m[..., :-1, :]
    o[..., :-1, :] |= m[..., 1:, :]
    o[..., :, 1:] |= m[..., :, :-1]
    o[..., :, :-1] |= m[..., :, 1:]
    return o


def _sweep(bg, reach, seed):
    """One sequential sweep along the last axis, towards higher indices: a background pixel becomes reached if it is
    reached or seeded, or its predecessor (after the update) is a reached background pixel."""
    pos = np.broadcast_to(np.arange(bg.shape[-1]), bg.shape)
    last_fg = np.maximum.accumulate(np.where(~bg, pos, -1), axis=-1)
    last_seed = np.maximum.accumulate(np.where(bg & (reach | seed), pos, -1), axis=-1)
    return bg & (last_seed > last_fg)


def fill_pass(fg, reach):
    """One pass of the hole-filling propagation on bool [B,H,W]: rows left to right (seeded on the image border) and
    right to left, then columns top-down and bottom-up. Returns the new reach."""
    bg = ~fg
    border = np.zeros(fg.shape[-2:], dtype=bool)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
    none = False
    r = _sweep(bg, reach, np.broadcast_to(border, fg.shape))
    r = _sweep(bg[..., ::-1], r[..., ::-1], none)[..., ::-1]
    bt, rt = np.swapaxes(bg, -1, -2), np.swapaxes(r, -1, -2)
    rt = _sweep(bt, rt, none)
    rt = _sweep(bt[..., ::-1], rt[..., ::-1], none)[..., ::-1]
    return np.ascontiguousarray(np.swapaxes(rt, -1, -2))


def nearest_index(d, s):
    """cv2 INTER_NEAREST source indices of d outputs from s inputs."""
    return np.minimum(np.floor(np.arange(d) * (1.0 / (d / s))).astype(np.int64), s - 1)


def _cv_x(d, s):
    """cv2 resizeGeneric_ INTER_LINEAR along x: (left index, right index, fraction), the weight collapsing onto the edge
    sample outside [0, s - 1)."""
    f = ((np.arange(d) + 0.5) * (1.0 / (d / s)) - 0.5).astype(F32)
    i = np.floor(f).astype(np.int64)
    f = f - i.astype(F32)
    lo, hi = i < 0, i >= s - 1
    f[lo | hi] = 0
    i[lo], i[hi] = 0, s - 1
    return i, np.minimum(i + 1, s - 1), f


def _cv_y(d, s):
    """Along y the fraction is kept and only the two rows are clamped (cv2 clips the ring-buffer rows)."""
    f = ((np.arange(d) + 0.5) * (1.0 / (d / s)) - 0.5).astype(F32)
    i = np.floor(f).astype(np.int64)
    f = f - i.astype(F32)
    return np.clip(i, 0, s - 1), np.clip(i + 1, 0, s - 1), f


def fma32(a, b, c):
    """fp32 fma(a, b, c), correctly rounded: a * b is exact in float64, the sum is formed with its exact error
    (two-sum) and rounded to odd in float64, which then rounds to fp32 as the exact value would."""
    a, b, c = (np.asarray(v, dtype=F32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    z = s - p
    e = (p - (s - z)) + (c - z)
    bits = s.view(np.int64).copy()
    fix = (e != 0) & ((bits & 1) == 0)
    bits[fix] += np.where((e[fix] > 0) == (s[fix] > 0), 1, -1)
    return bits.view(np.float64).astype(F32)


def _aten(d, s):
    """ATen area_pixel_compute_source_index (align_corners = False) as built with FMA: fp32 fma(scale, d + 0.5, -0.5),
    negative -> 0, truncated index."""
    sc = F32(s) / F32(d)
    f = np.maximum(fma32(sc, np.arange(d).astype(F32) + F32(0.5), F32(-0.5)), F32(0))
    i = np.minimum(f.astype(np.int64), s - 1)
    return i, np.minimum(i + 1, s - 1), f - i.astype(F32)


def _interp_fma(x, xs, ys):
    """ATen's CPU order with FMA: rows fma(a0, left, a1 * right), then fma(1 - fy, r0, fy * r1)."""
    (x0, x1, fx), (y0, y1, fy) = xs, ys
    a0, a1 = (F32(1) - fx)[:, None], fx[:, None]
    left, right = x[:, :, x0], x[:, :, x1]
    rows = fma32(left, np.broadcast_to(a0, left.shape), right * a1)
    b0, b1 = (F32(1) - fy)[:, None, None], fy[:, None, None]
    r0, r1 = rows[:, y0], rows[:, y1]
    return fma32(r0, np.broadcast_to(b0, r0.shape), r1 * b1)


def _interp(x, xs, ys):
    """Bilinear interpolation of fp32 [B,H,W,C] with per-axis (i0, i1, f): rows a0 * left + a1 * right, then
    (1 - fy) * r0 + fy * r1, every operation in float32."""
    (x0, x1, fx), (y0, y1, fy) = xs, ys
    a0, a1 = (F32(1) - fx)[:, None], fx[:, None]
    rows = x[:, :, x0] * a0 + x[:, :, x1] * a1
    b0, b1 = (F32(1) - fy)[:, None, None], fy[:, None, None]
    return rows[:, y0] * b0 + rows[:, y1] * b1


def resize_linear(x, OH, OW):
    """cv2.resize(x, (OW, OH), interpolation=INTER_LINEAR) of fp32 [B,H,W,C], as cv2 computes it for C = 2 (and any C
    but 1, 3 and 4, which cv2 hands to IPP). Exactly 2x smaller in both directions: INTER_AREA's
    (0 + (((a + b) + c) + d)) * 0.25 of each 2x2 block, a b the upper row."""
    x = np.asarray(x, dtype=F32)
    H, W = x.shape[1:3]
    if H == 2 * OH and W == 2 * OW:
        s = ((x[:, 0::2, 0::2] + x[:, 0::2, 1::2]) + x[:, 1::2, 0::2]) + x[:, 1::2, 1::2]
        return (F32(0) + s) * F32(0.25)
    return _interp(x, _cv_x(OW, W), _cv_y(OH, H))


def resize_aten(x, OH, OW):
    """The nchw form on fp32 [B,H,W,C]: F.interpolate(mode="bilinear", align_corners=False) as ATen's vectorised CPU
    kernel computes it with FMA."""
    x = np.asarray(x, dtype=F32)
    H, W = x.shape[1:3]
    return _interp_fma(x, _aten(OW, W), _aten(OH, H))


def plane_max(x):
    """[P, n] fp32 -> [P]: the maximum; NaN where a plane holds one; +0 over -0."""
    x = np.asarray(x, dtype=F32)
    with np.errstate(invalid="ignore"):
        m = x.max(axis=1)
    plus_zero = ((x == 0) & ~np.signbit(x)).any(axis=1)
    m = np.where(m == 0, np.where(plus_zero, F32(0.0), F32(-0.0)), m)
    m[np.isnan(x).any(axis=1)] = np.nan
    return m


def as_u8(v):
    """numpy's float32 -> uint8 of in-range values: truncation toward zero."""
    return np.trunc(v).astype(np.int64).astype(np.uint8)


# ------------------------------------------------------------------------------------------------------ emulator
class _GlueEntry:
    def __init__(self, emu, name):
        self.emu, self.name, self.argtypes, self.restype = emu, name, None, None

    def __call__(self, *args):
        assert self.argtypes is not None and len(args) == len(self.argtypes), self.name
        a = {k: _raw(v, t) for k, v, t in zip(lib.PROTOS[self.name].names, args, self.argtypes)}
        getattr(self.emu, "_" + self.name[4:])(a)
        return 0


_DT = {"u8": torch.uint8, "i32": torch.int32, "f32": torch.float32}


class GlueEmulator(KernelEmulator):
    """Stands in for the ctypes library: the glue entries run in numpy on the CPU."""

    def __getattr__(self, name):
        if not name.startswith("fgt_"):
            raise AttributeError(name)
        e = _GlueEntry(self, name) if name in GLUE_ENTRIES else _Refused(name)
        setattr(self, name, e)
        return e

    def load(self, p, kind, n):
        """numpy copy of the first n elements at address p."""
        return self.flat(p, _DT[kind])[:n].numpy().copy()

    def store(self, p, kind, v, idx=None):
        """Writes v (flat) at elements idx (default: the first v.size) of the buffer at p and records the store.
        kind "addr": addressed, contents unspecified (nothing written here)."""
        fl = self.flat(p, torch.uint8 if kind == "addr" else _DT[kind])
        v = np.asarray(v).reshape(-1)
        idx = np.arange(v.size) if idx is None else np.asarray(idx, dtype=np.int64).reshape(-1)
        t = torch.from_numpy(idx)
        if kind != "addr":
            fl[t] = torch.from_numpy(np.ascontiguousarray(v.astype(fl.numpy().dtype)))
        self._rec(kind, fl, t)

    # ---------------------------------------------------------------------------------------------------- morph
    def _binary_dilate(self, a):
        B, H, W, n = a["B"], a["H"], a["W"], a["iterations"]
        m = self.load(a["in"], "u8", B * H * W).reshape(B, H, W) != 0
        for _ in range(n):
            m = dilate_cross(m)
        self.store(a["out"], "u8", m.astype(np.uint8))
        if n > 1:
            self.store(a["tmp"], "addr", np.zeros(B * H * W, np.uint8))

    def _fill_holes_init(self, a):
        self.store(a["reach"], "u8", np.zeros(a["B"] * a["H"] * a["W"], np.uint8))

    def _fill_holes_pass(self, a):
        B, H, W = a["B"], a["H"], a["W"]
        fg = self.load(a["fg"], "u8", B * H * W).reshape(B, H, W) != 0
        reach0 = self.load(a["reach"], "u8", B * H * W).reshape(B, H, W)
        r = reach0 != 0
        for _ in range(a["passes"]):
            r = fill_pass(fg, r)
        new = np.where(r & (reach0 == 0), np.uint8(1), reach0)   # newly reached pixels become 1, nothing else moves
        self.store(a["reach"], "u8", new)
        self.store(a["changed"], "i32", np.array([int((r != (reach0 != 0)).any())], np.int32))

    def _fill_holes_finish(self, a):
        n = a["B"] * a["H"] * a["W"]
        self.store(a["out"], "u8", (self.load(a["reach"], "u8", n) == 0).astype(np.uint8))

    def _resize_nearest_u8(self, a):
        B, H, W, C, OH, OW = (a[k] for k in ("B", "H", "W", "C", "OH", "OW"))
        x = self.load(a["in"], "u8", B * H * W * C).reshape(B, H, W, C)
        self.store(a["out"], "u8", x[:, nearest_index(OH, H)][:, :, nearest_index(OW, W)])

    def _resize_bilinear_f32(self, a):
        B, H, W, C, OH, OW = (a[k] for k in ("B", "H", "W", "C", "OH", "OW"))
        x = self.load(a["in"], "f32", B * H * W * C)
        if a["nchw"]:
            y = resize_aten(x.reshape(B, C, H, W).transpose(0, 2, 3, 1), OH, OW)
        else:
            y = resize_linear(x.reshape(B, H, W, C), OH, OW)
        y = y.copy()
        for c, s in ((0, a["scale_c0"]), (1, a["scale_c1"])):
            if c < C:
                y[..., c] = y[..., c] * F32(s)
        self.store(a["out"], "f32", y.transpose(0, 3, 1, 2) if a["nchw"] else y)

    # ----------------------------------------------------------------------------------------------------- clip
    def _plane_max(self, a):
        P, n = a["planes"], a["plane_size"]
        self.store(a["out"], "f32", plane_max(self.load(a["x"], "f32", P * n).reshape(P, n)))

    def _window_gather(self, a):
        t, HW = a["t"], a["H"] * a["W"]
        ids = self.load(a["ids"], "i32", t).astype(np.int64)
        N = int(ids.max()) + 1
        m = (self.load(a["masks"], "u8", N * HW).reshape(N, HW)[ids] != 0).astype(F32)
        fr = self.load(a["frames"], "f32", N * 3 * HW).reshape(N, 3, HW)[ids]
        fl = self.load(a["flows"], "f32", N * 2 * HW).reshape(N, 2, HW)[ids]
        fmax = self.load(a["fmax"], "f32", N * 2).reshape(N, 2)[ids]
        with np.errstate(divide="ignore", invalid="ignore"):
            self.store(a["out_frames"], "f32", (fr * F32(2) - F32(1)) * (F32(1) - m)[:, None])
            self.store(a["out_flows"], "f32", fl / fmax[:, :, None])
        self.store(a["out_masks"], "f32", m)

    def _window_compose(self, a):
        k, HW = a["k"], a["H"] * a["W"]
        ids = self.load(a["ids"], "i32", k).astype(np.int64)
        N = int(ids.max()) + 1
        first = self.load(a["first"], "u8", k)
        o = self.load(a["filled"], "f32", k * 3 * HW).reshape(k, 3, HW).transpose(0, 2, 1)
        fr = self.load(a["frames"], "f32", N * 3 * HW).reshape(N, 3, HW)[ids].transpose(0, 2, 1)
        m = (self.load(a["masks"], "u8", N * HW).reshape(N, HW)[ids] != 0).astype(F32)[:, :, None]
        comp = self.flat(a["comp"], torch.float32)[:N * HW * 3].numpy().reshape(N, HW, 3)
        fa = as_u8((o + F32(1)) * F32(0.5) * F32(255)).astype(F32)          # (out + 1) / 2 * 255 (:725-726)
        fb = as_u8(fr * F32(255)).astype(F32)                                # frame * 255 (:729)
        v = fa * m + fb * (F32(1) - m)                                       # (:731-733)
        idx = []
        for j in range(k):                                                   # a frame appears once among neighbours
            i = ids[j]
            comp[i] = v[j] if first[j] else comp[i] * F32(0.5) + v[j] * F32(0.5)
            idx.append(np.arange(i * HW * 3, (i + 1) * HW * 3))
        self._rec("f32", self.flat(a["comp"], torch.float32), torch.from_numpy(np.concatenate(idx)))

    def _comp_to_u8(self, a):
        self.store(a["out"], "u8", as_u8(self.load(a["comp"], "f32", a["total"])))

    # ------------------------------------------------------------------------------------------------ gradients
    def _grad_prep_pre(self, a):
        n = a["B"] * a["H"] * a["W"]
        v = self.load(a["video"], "f32", n * 3).reshape(n, 3)
        hole = self.load(a["mask"], "u8", n) != 0
        v[hole] = 0
        self.store(a["u8"], "u8", as_u8(v * F32(255)))

    def _grad_prep_post(self, a):
        B, H, W = a["B"], a["H"], a["W"]
        img = self.load(a["u8"], "u8", B * H * W * 3).reshape(B, H, W, 3).astype(F32) / F32(255)
        gx, gy = np.zeros_like(img), np.zeros_like(img)
        gx[:, :, :-1] = img[:, :, 1:] - img[:, :, :-1]
        gy[:, :-1] = img[:, 1:] - img[:, :-1]
        md = self.load(a["mask_dilated"], "u8", B * H * W).reshape(B, H, W) != 0
        gx[md] = 0
        gy[md] = 0
        self.store(a["gx"], "f32", gx)
        self.store(a["gy"], "f32", gy)


def call(name, *args):
    """Runs entry `name` of a fresh GlueEmulator on CPU tensors (passed as addresses, like lib.call). Returns the
    emulator (its records)."""
    emu = GlueEmulator()
    p = lib.PROTOS[name]
    e = getattr(emu, name)
    e.argtypes = p.argtypes
    for x in args:
        if isinstance(x, torch.Tensor):
            st = x.untyped_storage()
            emu._storages.append([st.data_ptr(), st.data_ptr() + st.nbytes(), x])
    args = [x.data_ptr() if isinstance(x, torch.Tensor) else x for x in args]
    e(*(args + (["stream"] if p.stream else [])))
    return emu
