"""A numpy / float64 interpreter of the three flow-propagation entries of include/fgt_b200.h, for CPU tensors.

`PropEmulator` stands in for the ctypes library the way tests/kernel_emulator.py's `KernelEmulator` does (it extends
it for pointer resolution and store records): `fgt_prop_step`, `fgt_prop_gather` and `fgt_prop_fuse` are served, every
other entry is refused. Each entry takes the C-ABI arguments and works on the CPU storages behind them, in the kernels'
layouts: mask uint8 [N,H,W] (nonzero = hole), one frame pair's flows float32 [H,W,2] = (u, v), gradients float32
[N,H,W,3], and per NN slot nn_y / nn_x float64, nn_t int32, have uint8 and cuv float64 [N,H,W,2].

Semantics are restated from the header and oracle/prop_oracle.py (the reference's get_flowNN_gradient and
common_utils.interp / consistCheck), not from prop.cu:
- remap(img, x, y): cv2.remap INTER_LINEAR with a zero border. sx = rint(fp32(x * 32)) (half to even), tap column
  sx >> 5 (floor), fraction (sx & 31) / 32, likewise in y; weights (1 - fy)(1 - fx), (1 - fy) fx, fy (1 - fx), fy fx
  and the four products summed in that order, all in fp32. A non-finite coordinate samples nothing (0).
- fgt_prop_step, frame t, neighbour frame tn: for every hole pixel (y, x) of frame t, ny = fp32(y + v), nx = fp32(x + u)
  from flow_step; (iy, ix) = np.round (half to even). Round trip ry = fp32(ny + remap(back_v)), rx likewise; diff =
  sqrt((ry - y)^2 + (rx - x)^2) in float64; the pixel is consistent iff diff < thres (so NaN and inf never are).
  Neighbour cell (tn, iy, ix) must satisfy 0 <= iy < H - 1 and 0 <= ix < W - 1. Case 1 (the cell is known):
  nn = (ny, nx, tn), have = 1, cuv = (|fp32(rx - x)|, |fp32(ry - y)|). Case 2 (the cell is a hole with have == 1):
  nn = nn(cell) + (ny - iy, nx - ix) in float64, kept only if its np.round lies inside the same bounds; nn_t = nn_t(cell),
  have = 1, cuv = max(own, |cuv(cell)|) per component. Otherwise nothing is written.
- fgt_prop_gather, source frame s: every hole pixel whose nn_t equals s gets remap(gradients of frame s,
  fp32(nn_x), fp32(nn_y)) for the three channels of gx and of gy (the source frame as it was before the launch).
- fgt_prop_fuse: tofill = hole and no slot has have == 1 (written everywhere). Where some slot has have == 1,
  c_k = exp(-sqrt(cuv_k0^2 + cuv_k1^2) / alpha) for the slots that do (0 otherwise), den = c0 + c1, weights c_k / den
  or, where den == 0, equal weights over those slots; output fp32(g_b w0 + g_f w1) in float64.

Every store is recorded as in KernelEmulator (`records`, `written_bytes`). `counts` tallies, over all calls, the
decisions each pixel took (see `_prop_step` / `_prop_fuse` for the keys). `fuse` keeps the last fusion's written
elements (flat indices into gx / gy), their float64 values, magnitudes, exactness of weights and smaller confidence, for
the GPU bars (`fuse_ulps`).
"""
import collections

import numpy as np
import torch

from fgt_b200 import lib
from tests.gemm_emulator import _Refused
from tests.kernel_emulator import KernelEmulator, _raw

PROP_ENTRIES = ("fgt_prop_step", "fgt_prop_gather", "fgt_prop_fuse")
F32 = np.float32


def remap(img, x, y):
    """cv2.remap(img, x, y, INTER_LINEAR, BORDER_CONSTANT 0) of fp32 img [H,W] or [H,W,C] at fp32 coordinates."""
    img = np.asarray(img, dtype=F32)
    H, W = img.shape[:2]
    x, y = np.asarray(x, dtype=F32), np.asarray(y, dtype=F32)
    ok = np.isfinite(x) & np.isfinite(y)
    with np.errstate(invalid="ignore", over="ignore"):
        sx = np.rint(np.where(ok, x, F32(0)) * F32(32)).astype(np.float64)
        sy = np.rint(np.where(ok, y, F32(0)) * F32(32)).astype(np.float64)
    # beyond a few image sizes every tap is outside; clamping keeps the integers exact and in range
    lim = 32.0 * (max(H, W) + 4)
    sx, sy = np.clip(sx, -lim, lim).astype(np.int64), np.clip(sy, -lim, lim).astype(np.int64)
    ix, iy = sx >> 5, sy >> 5
    fx, fy = (sx & 31).astype(F32) / F32(32), (sy & 31).astype(F32) / F32(32)

    def tap(yy, xx):
        inside = ok & (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        v = img[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)]
        return np.where(inside[..., None] if img.ndim == 3 else inside, v, F32(0))

    ws = ((F32(1) - fy) * (F32(1) - fx), (F32(1) - fy) * fx, fy * (F32(1) - fx), fy * fx)
    if img.ndim == 3:
        ws = tuple(w[..., None] for w in ws)
    acc = tap(iy, ix) * ws[0]
    acc = acc + tap(iy, ix + 1) * ws[1]
    acc = acc + tap(iy + 1, ix) * ws[2]
    acc = acc + tap(iy + 1, ix + 1) * ws[3]
    return acc.astype(F32)


def _in_bounds(r, n):
    """0 <= r < n - 1 for rounded float64 values r (NaN and inf are outside)."""
    with np.errstate(invalid="ignore"):
        return np.isfinite(r) & (r >= 0) & (r < n - 1)


class _PropEntry:
    def __init__(self, emu, name):
        self.emu, self.name, self.argtypes, self.restype = emu, name, None, None

    def __call__(self, *args):
        assert self.argtypes is not None and len(args) == len(self.argtypes), self.name
        a = {k: _raw(v, t) for k, v, t in zip(lib.PROTOS[self.name].names, args, self.argtypes)}
        getattr(self.emu, "_" + self.name[4:])(a)
        return 0


class PropEmulator(KernelEmulator):
    """Stands in for the ctypes library: the three propagation entries run in numpy on the CPU."""

    def __init__(self):
        super().__init__()
        self.counts = collections.Counter()
        self.fuse = None

    def __getattr__(self, name):
        if not name.startswith("fgt_"):
            raise AttributeError(name)
        e = _PropEntry(self, name) if name in PROP_ENTRIES else _Refused(name)
        setattr(self, name, e)
        return e

    # numpy views of the storage behind an address (writes go to the storage)
    def arr(self, p, dtype, shape):
        fl = self.flat(p, dtype)
        return fl[:int(np.prod(shape))].numpy().reshape(shape), fl

    def _store(self, fl, idx, kind):
        self._rec(kind, fl, torch.from_numpy(np.asarray(idx, dtype=np.int64).reshape(-1)))

    def _prop_step(self, a):
        H, W, t, tn, thres = a["H"], a["W"], a["t"], a["tn"], a["thres"]
        HW = H * W
        mask_fl = self.flat(a["mask"], torch.uint8).numpy()
        step, _ = self.arr(a["flow_step"], torch.float32, (H, W, 2))
        back, _ = self.arr(a["flow_back"], torch.float32, (H, W, 2))
        ny_fl, nx_fl = (self.flat(a[k], torch.float64) for k in ("nn_y", "nn_x"))
        nt_fl, hv_fl, cuv_fl = (self.flat(a["nn_t"], torch.int32), self.flat(a["have"], torch.uint8),
                                self.flat(a["cuv"], torch.float64))
        nn_y, nn_x, nn_t, have, cuv = ny_fl.numpy(), nx_fl.numpy(), nt_fl.numpy(), hv_fl.numpy(), cuv_fl.numpy()
        c = self.counts
        p = np.nonzero(mask_fl[t * HW:(t + 1) * HW])[0]
        ys, xs = p // W, p % W
        with np.errstate(invalid="ignore", over="ignore"):
            ny = ys.astype(F32) + step[ys, xs, 1]
            nx = xs.astype(F32) + step[ys, xs, 0]
            ry = ny + remap(back[:, :, 1], nx, ny)
            rx = nx + remap(back[:, :, 0], nx, ny)
            dy, dx = ry.astype(np.float64) - ys, rx.astype(np.float64) - xs
            diff = np.sqrt(dy * dy + dx * dx)
            consist = diff < thres
            rny, rnx = np.round(ny).astype(np.float64), np.round(nx).astype(np.float64)
        finite = np.isfinite(ny) & np.isfinite(nx)
        c["step_nonfinite_position"] += int((~finite).sum())
        c["step_consistent"] += int(consist.sum())
        c["step_inconsistent"] += int((~consist).sum())
        c["step_diff_eq_thres"] += int((diff == thres).sum())
        c["step_diff_below_thres_by_under_1e-6"] += int(((diff < thres) & (diff > thres - 1e-6)).sum())
        inb = _in_bounds(rny, H) & _in_bounds(rnx, W)
        c["step_consistent_out_of_bounds"] += int((consist & ~inb).sum())
        for name, r, n in (("row", rny, H), ("col", rnx, W)):
            for off in (2, 1):
                c[f"step_consistent_{name}_{n - off}"] += int((consist & (r == n - off)).sum())
            c[f"step_consistent_{name}_negative"] += int((consist & (r < 0)).sum())
        for name, v in (("y", ny), ("x", nx)):
            with np.errstate(invalid="ignore"):
                half = consist & (v - np.floor(v) == 0.5)
                c[f"step_tie_{name}_to_even_below"] += int((half & (np.round(v) < v)).sum())
                c[f"step_tie_{name}_to_even_above"] += int((half & (np.round(v) > v)).sum())
        sel = consist & inb
        p, ys, xs, ny, nx, ry, rx = p[sel], ys[sel], xs[sel], ny[sel], nx[sel], ry[sel], rx[sel]
        iy, ix = rny[sel].astype(np.int64), rnx[sel].astype(np.int64)
        ua = np.abs(rx - xs.astype(F32)).astype(np.float64)
        va = np.abs(ry - ys.astype(F32)).astype(np.float64)
        q = tn * HW + iy * W + ix
        o = t * HW + p
        known = mask_fl[q] == 0
        chain = ~known & (have[q] == 1)
        c["step_case1"] += int(known.sum())
        c["step_hole_without_neighbour"] += int((~known & ~chain).sum())
        ty = nn_y[q] + (ny.astype(np.float64) - iy)
        tx = nn_x[q] + (nx.astype(np.float64) - ix)
        with np.errstate(invalid="ignore"):
            tin = _in_bounds(np.round(ty), H) & _in_bounds(np.round(tx), W)
        c2 = chain & tin
        c["step_case2"] += int(c2.sum())
        c["step_case2_out_of_bounds"] += int((chain & ~tin).sum())
        c["step_case2_out_of_bounds_at_last_row"] += int((chain & (np.round(ty) == H - 1)).sum())
        prev_u, prev_v = np.abs(cuv[2 * q]), np.abs(cuv[2 * q + 1])
        c["step_case2_own_residual_larger"] += int((c2 & (ua > prev_u)).sum())
        c["step_case2_chained_residual_larger"] += int((c2 & (ua < prev_u)).sum())
        w1, w2 = o[known], o[c2]
        old_t = nn_t[q[c2]].copy()   # frame tn is read, frame t written: no overlap, but copy before any store
        nn_y[w1], nn_x[w1], nn_t[w1], have[w1] = ny[known], nx[known], tn, 1
        cuv[2 * w1], cuv[2 * w1 + 1] = ua[known], va[known]
        nn_y[w2], nn_x[w2], nn_t[w2], have[w2] = ty[c2], tx[c2], old_t, 1
        cuv[2 * w2], cuv[2 * w2 + 1] = np.maximum(ua[c2], prev_u[c2]), np.maximum(va[c2], prev_v[c2])
        w = np.concatenate([w1, w2])
        for fl, kind in ((ny_fl, "f64"), (nx_fl, "f64"), (nt_fl, "i32"), (hv_fl, "u8")):
            self._store(fl, w, kind)
        self._store(cuv_fl, np.concatenate([2 * w, 2 * w + 1]), "f64")

    def _prop_gather(self, a):
        N, H, W, s = a["N"], a["H"], a["W"], a["s"]
        total = N * H * W
        mask = self.flat(a["mask"], torch.uint8).numpy()[:total]
        nn_y, nn_x = (self.flat(a[k], torch.float64).numpy()[:total] for k in ("nn_y", "nn_x"))
        nn_t = self.flat(a["nn_t"], torch.int32).numpy()[:total]
        o = np.nonzero((mask != 0) & (nn_t == s))[0]
        self.counts["gather_pixels"] += len(o)
        px, py = nn_x[o].astype(F32), nn_y[o].astype(F32)
        for k in ("gx", "gy"):
            g, fl = self.arr(a[k], torch.float32, (N, H, W, 3))
            src = g[s].copy()
            g.reshape(-1, 3)[o] = remap(src, px, py)
            self._store(fl, (3 * o[:, None] + np.arange(3)).reshape(-1), "f32")

    def _prop_fuse(self, a):
        N, H, W, alpha = a["N"], a["H"], a["W"], a["alpha"]
        total = N * H * W
        mask = self.flat(a["mask"], torch.uint8).numpy()[:total] != 0
        h = [mask & (self.flat(a[k], torch.uint8).numpy()[:total] == 1) for k in ("have0", "have1")]
        cuv = [self.flat(a[k], torch.float64).numpy()[:2 * total].reshape(total, 2) for k in ("cuv0", "cuv1")]
        tofill = mask & ~h[0] & ~h[1]
        t_arr, t_fl = self.arr(a["tofill"], torch.uint8, (total,))
        t_arr[:] = tofill
        self._store(t_fl, np.arange(total), "u8")
        o = np.nonzero(h[0] | h[1])[0]
        h0, h1 = h[0][o], h[1][o]
        with np.errstate(over="ignore", under="ignore", invalid="ignore"):
            conf = [np.where(hk, np.exp(-np.sqrt(ck[o, 0] * ck[o, 0] + ck[o, 1] * ck[o, 1]) / alpha), 0.0)
                    for hk, ck in ((h0, cuv[0]), (h1, cuv[1]))]
        den = conf[0] + conf[1]
        zero = den == 0
        cnt = h0.astype(np.float64) + h1
        with np.errstate(invalid="ignore", divide="ignore"):
            w0 = np.where(zero, h0 / cnt, conf[0] / np.where(zero, 1.0, den))
            w1 = np.where(zero, h1 / cnt, conf[1] / np.where(zero, 1.0, den))
        both = h0 & h1
        tiny = 2.0 ** -1022
        c = self.counts
        c["fuse_one_candidate"] += int((~both).sum())
        c["fuse_two_candidates"] += int((both & ~zero).sum())
        c["fuse_den_zero"] += int(zero.sum())
        c["fuse_subnormal_confidence"] += int(sum(((ck > 0) & (ck < tiny)).sum() for ck in conf))
        c["fuse_two_candidates_both_subnormal"] += int((both & (conf[0] > 0) & (conf[0] < tiny) & (conf[1] > 0)
                                                        & (conf[1] < tiny)).sum())
        c["fuse_tofill"] += int(tofill.sum())
        vals, mags = {}, {}
        for kb, kf, ko in (("gx_bn", "gx_fn", "gx"), ("gy_bn", "gy_fn", "gy")):
            gb = self.flat(a[kb], torch.float32).numpy()[:3 * total].reshape(total, 3)[o].astype(np.float64)
            gf = self.flat(a[kf], torch.float32).numpy()[:3 * total].reshape(total, 3)[o].astype(np.float64)
            v = gb * w0[:, None] + gf * w1[:, None]
            out, fl = self.arr(a[ko], torch.float32, (total, 3))
            out[o] = v.astype(F32)
            self._store(fl, (3 * o[:, None] + np.arange(3)).reshape(-1), "f32")
            vals[ko], mags[ko] = v.reshape(-1), (np.abs(gb * w0[:, None]) + np.abs(gf * w1[:, None])).reshape(-1)
        exact = np.repeat(~both | zero, 3)
        cmin = np.repeat(np.where(both, np.minimum(conf[0], conf[1]), 1.0), 3)
        self.fuse = dict(idx=(3 * o[:, None] + np.arange(3)).reshape(-1), v=vals, mag=mags, exact=exact, cmin=cmin)


def emulate(gx, gy, mask, ff, fb, thres, alpha, states=None):
    """propagation.propagate's launch sequence (2(N-1) steps, 2N gathers, one fusion) through the interpreter, on CPU
    tensors made from reference-layout inputs (gradients [H,W,3,N], mask [H,W,N], flows [H,W,2,N-1]). Returns the fused
    gradients and mask_tofill in the reference layouts and the emulator; `states`, if a list, receives both slots'
    final state."""
    from fgt_b200 import propagation
    from tests.test_launch_trace import recording

    def t(a, perm, dtype):
        return torch.from_numpy(np.ascontiguousarray(a.astype(dtype).transpose(perm)))

    m = t(mask, (2, 0, 1), np.uint8)
    f, b = t(ff, (3, 0, 1, 2), F32), t(fb, (3, 0, 1, 2), F32)
    x, y = t(gx, (3, 0, 1, 2), F32), t(gy, (3, 0, 1, 2), F32)
    emu, make = PropEmulator(), propagation.slot_state

    def keep(*args):
        s = make(*args)
        if states is not None:
            states.append(s)
        return s

    propagation.slot_state = keep
    try:
        with recording(emu):
            tofill = propagation.propagate(m, f, b, x, y, float(thres), float(alpha))
    finally:
        propagation.slot_state = make
    return x.permute(1, 2, 3, 0).numpy(), y.permute(1, 2, 3, 0).numpy(), tofill.permute(1, 2, 0).numpy() != 0, emu


def fuse_ulps(got, v, mag, exact, cmin):
    """Distance in fp32 ulps of the fused values `got` (fp32) from fp32(v), v the interpreter's float64 values, and
    whether each element was exempt from bit identity. Elements with exact weights (one candidate, or den == 0) must be
    fp32(v) bit for bit. Elsewhere device `exp` and numpy's may differ by an ulp, which moves v by a few double ulps:
    fp32(v) is required unless fp32(v - e m) != fp32(v + e m), with e = 8 * 2^-53 and m = |g_b w0| + |g_f w1| (|v|
    without cancellation); where a confidence is subnormal its ulp is 2^-1074 absolute, so e grows by 2^-1072 / cmin.
    Outside the exemption the distance is reported as infinite unless it is 0."""
    got = np.asarray(got, dtype=F32)
    want = v.astype(F32)
    e = 8 * 2.0 ** -53 + np.where(cmin < 2.0 ** -1022, 2.0 ** -1072 / np.maximum(cmin, 2.0 ** -1074), 0.0)
    lo, hi = (v - e * mag).astype(F32), (v + e * mag).astype(F32)
    exempt = ~exact & (lo != hi)
    same = got.view(np.uint32) == want.view(np.uint32)
    ulp = np.spacing(np.maximum(np.abs(want), np.abs(got)).astype(F32)).astype(np.float64)
    dist = np.abs(got.astype(np.float64) - want) / ulp
    inside = exempt & (got >= np.minimum(lo, hi)) & (got <= np.maximum(lo, hi))
    return np.where(same, 0.0, np.where(inside, dist, np.inf)), exempt
