"""Float64 interpreters of the solver entries of include/fgt_b200.h: region fill's conjugate gradients
(fgt_regionfill_*) and Poisson blending's LSQR (fgt_poisson_*), for CPU tensors.

`SolverEmulator` stands in for the ctypes library the way tests/glue_emulator.py's `GlueEmulator` does: the entries of
`SOLVER_ENTRIES` run here on the CPU storages behind their pointer arguments, every other entry is refused, and every
store is recorded (`records`, `written_bytes`) so that a replay can check the bytes a launch must leave alone.
`fgt_poisson_graph_create` remembers its arguments under the handle it returns; each `fgt_poisson_graph_launch` of that
handle runs `iters` iterations on them.

Semantics come from the header and from the operations it names, not from the kernels' code: the operators and
right-hand sides are oracle/poisson_oracle.py's (`equation_codes`, `rhs`, `matvec`, `rmatvec`, `unfilled_sweeps`)
and oracle/regionfill_oracle.py's (`system`); LSQR's scalar step is `lsqr_step` below, one pass of `PO.lsqr`'s loop in
Python float64 on the header's state slots, with `PO._sym_ortho`; CG is the header's recurrence.

Each store also appends a check to `checks`: (buffer label, kind, flat view, element indices, wanted values, bar,
system of each element or None). Kinds:
- "exact": bit for bit (codes, counts, u after set-up, kctr, clr, unf, both finish kernels, region fill's x = 0 and
  the stopped / istop / itn state slots);
- "multiset": the set-up's pixel list, compared per frame as a sorted multiset (blocks append in arrival order);
- "bar": |got - want| <= bar per element, want computed in extended precision (np.longdouble) so it stands for the
  exact value. Vector updates: bar = u * n * sum|terms| (u = 2^-53, n roundings in the element's formula, the sums of
  up to 8 neighbour terms in any order, FMA contraction allowed), plus the bar of any operand produced earlier in the
  same launch times its coefficient. Atomically accumulated sums of N terms: u * N * sum|terms| plus the propagated
  bars of the terms, for any summation order. Every rounding also carries 2^-1074 for the subnormal range;
- "state": LSQR's floating-point state slots, within 1e-12 relative.
Where a stop test's quantity lies within 1e-12 relative of its threshold the system goes into `near` (with the
iteration); a replay then accepts either decision for that system and counts it.
"""
import contextlib
import math

import numpy as np
import torch

from fgt_b200 import lib
from oracle import poisson_oracle as PO
from oracle import regionfill_oracle as RO
from tests.gemm_emulator import _Refused
from tests.kernel_emulator import KernelEmulator, _raw

SOLVER_ENTRIES = ("fgt_regionfill_init", "fgt_regionfill_iters", "fgt_regionfill_finish", "fgt_poisson_setup",
                  "fgt_poisson_iters", "fgt_poisson_graph_create", "fgt_poisson_graph_launch",
                  "fgt_poisson_graph_destroy", "fgt_poisson_unfilled", "fgt_poisson_finish")
U = 2.0 ** -53                 # unit roundoff of float64
SUB = 2.0 ** -1074             # absolute rounding error bound of one operation in the subnormal range
HP = np.longdouble             # extended precision for the wanted values
NEAR = 1e-12                   # relative distance of a stop test from its threshold that accepts either decision
ROUND_T1, ROUND_T2 = 14, 13    # roundings from the state and the slot sums to LSQR's t1 = phi / rho, t2 = -theta / rho
DONE, ISTOP, ITN = 12, 13, 14
_DT = {"u8": torch.uint8, "i32": torch.int32, "f64": torch.float64}


def lsqr_step(prev, k, bbk, aak, wwk, atol, btol, ctol, iter_lim):
    """One pass of PO.lsqr's loop (k >= 1) or its set-up (k == 0) on the header's 16 state slots, from the sums
    bb[k] = beta_k^2, aa[k] = alfa_k^2 and ww[k] = |w|^2. Returns (state, (t1, t2, vscale, au), skip_all, skip_u,
    near): au = alfa_k / beta_k; near = some stop test within NEAR of its threshold."""
    cur = [0.0] * 16
    if k == 0:
        beta, alfa = math.sqrt(bbk), math.sqrt(aak)
        cur[0], cur[1], cur[2], cur[7] = alfa, alfa, beta, -1.0
        cur[9] = 1.0 / alfa if alfa > 0 else 1.0
        cur[10] = 1.0 / beta if beta > 0 else 1.0
        cur[11], cur[15] = beta, beta
        cur[DONE] = 1.0 if alfa * beta == 0 else 0.0      # "the exact solution is x = 0": istop 0, itn 0
        return cur, (0.0, 0.0, cur[9], alfa * cur[10]), cur[DONE] != 0, cur[DONE] != 0, False
    if prev[DONE] != 0:
        return list(prev), (0.0, 0.0, 1.0, 0.0), True, True, False
    alfa, anorm, vscale, uscale = prev[0], prev[3], prev[9], 1.0
    beta = math.sqrt(bbk)
    if beta > 0:
        anorm = math.sqrt(anorm * anorm + alfa * alfa + beta * beta)
        alfa = math.sqrt(aak)
        vscale = 1.0 / alfa if alfa > 0 else 1.0
        uscale = 1.0 / beta
    cs, sn, rho = (float(t) for t in PO._sym_ortho(prev[1], beta))
    theta = sn * alfa
    rhobar = -cs * alfa
    phi = cs * prev[2]
    phibar = sn * prev[2]
    tau = sn * phi
    t1, t2 = phi / rho, -theta / rho
    ddnorm = prev[4] + wwk / (rho * rho)                  # ddnorm += |w / rho|^2
    delta = prev[8] * rho
    gambar = -prev[7] * rho
    rhs = phi - delta * prev[6]
    zbar = rhs / gambar
    xnorm = math.sqrt(prev[5] + zbar * zbar)
    gamma = math.sqrt(gambar * gambar + theta * theta)
    z = rhs / gamma
    bnorm = prev[11]
    acond = anorm * math.sqrt(ddnorm)
    rnorm = abs(phibar)
    arnorm = alfa * abs(tau)
    test1 = rnorm / bnorm
    test2 = arnorm / (anorm * rnorm + PO.EPS)
    test3 = 1.0 / (acond + PO.EPS)
    t1_ = test1 / (1 + anorm * xnorm / bnorm)
    rtol = btol + atol * anorm * xnorm / bnorm
    istop = 0
    if k >= iter_lim:
        istop = 7
    if 1 + test3 <= 1:
        istop = 6
    if 1 + test2 <= 1:
        istop = 5
    if 1 + t1_ <= 1:
        istop = 4
    if test3 <= ctol:
        istop = 3
    if test2 <= atol:
        istop = 2
    if test1 <= rtol:
        istop = 1
    # 1 + t <= 1 holds exactly for t <= 2^-53 (ties to even)
    pairs = [(test3, U), (test2, U), (t1_, U), (test3, ctol), (test2, atol), (test1, rtol)]
    near = any(thr > 0 and abs(q - thr) <= NEAR * thr for q, thr in pairs)
    cur[0], cur[1], cur[2], cur[3], cur[4] = alfa, rhobar, phibar, anorm, ddnorm
    cur[5], cur[6], cur[7], cur[8] = prev[5] + z * z, z, gambar / gamma, theta / gamma
    cur[9], cur[10], cur[11], cur[15] = vscale, uscale, bnorm, beta
    cur[DONE], cur[ISTOP], cur[ITN] = (1.0 if istop else 0.0), float(istop), float(k)
    return cur, (t1, t2, vscale, alfa * uscale), False, istop != 0, near


def sum_bar(t, et, old=0.0):
    """Bar of old + sum(t) accumulated in any order: N terms with their roundings, plus the terms' own bars et."""
    n = t.size + (old != 0)
    return float(U * n * (np.abs(t).sum() + abs(old)) + et.sum() + n * SUB)


def _abs_op(op, code, a):
    """sum of |terms| of op(code, a) for op = PO.matvec / PO.rmatvec and a >= 0: own terms + neighbour terms."""
    return 2 * op(code & 15, a) - op(code, a)


def _pop(c):
    return sum((c >> i) & 1 for i in range(8)).astype(np.int64)


_SYSTEMS = {}


def _system(mask):
    key = (mask.shape, mask.tobytes())
    if key not in _SYSTEMS:
        if len(_SYSTEMS) > 64:
            _SYSTEMS.clear()
        A, R = RO.system(mask)
        _SYSTEMS[key] = (A.astype(HP), abs(A).astype(HP), R.astype(HP), np.diff(A.indptr) - 1)
    return _SYSTEMS[key]


class _SolverEntry:
    def __init__(self, emu, name):
        self.emu, self.name, self.argtypes, self.restype = emu, name, None, None

    def __call__(self, *args):
        assert self.argtypes is not None and len(args) == len(self.argtypes), self.name
        a = {k: (v if type(v).__name__ == "CArgObject" else _raw(v, t))
             for k, v, t in zip(lib.PROTOS[self.name].names, args, self.argtypes)}
        getattr(self.emu, "_" + self.name[4:])(a)
        return 0


class SolverEmulator(KernelEmulator):
    """Stands in for the ctypes library: the solver entries run in numpy on the CPU. `bars = False` skips the
    extended-precision wanted values and bars (whole solves chained on the CPU need only the stored results)."""

    def __init__(self):
        super().__init__()
        self.checks, self.near, self.graphs, self.bars = [], [], {}, True
        self._next_graph = 0x5000

    def __getattr__(self, name):
        if not name.startswith("fgt_"):
            raise AttributeError(name)
        e = _SolverEntry(self, name) if name in SOLVER_ENTRIES else _Refused(name)
        setattr(self, name, e)
        return e

    # ------------------------------------------------------------------------------------------- loads / stores
    def arr(self, p, kind, n):
        """numpy view (shared) of the first n elements at address p, None for NULL."""
        return None if p is None else self.flat(p, _DT[kind])[:n].numpy()

    def store(self, label, p, kind, idx, want, check="exact", bar=None, sys=None):
        """Stores float64(want) (or want as is) at elements idx of the buffer at p, records the store and its check."""
        fl = self.flat(p, _DT[kind])
        idx = np.asarray(idx, dtype=np.int64).reshape(-1)
        want = np.asarray(want).reshape(-1)
        fl.numpy()[idx] = want.astype(fl.numpy().dtype)
        t = torch.from_numpy(idx)
        self._rec(kind, fl, t)
        if self.bars:
            bar = None if bar is None else np.asarray(bar, np.float64).reshape(-1)
            self.checks.append((label, check, fl, t, want, bar,
                                None if sys is None else np.broadcast_to(np.asarray(sys), idx.shape).copy()))

    # ------------------------------------------------------------------------------------------------ region fill
    def _regionfill_init(self, a):
        B, H, W = a["B"], a["H"], a["W"]
        n = H * W
        img = self.arr(a["img"], "f64", B * n).reshape(B, n)
        mask = self.arr(a["mask"], "u8", B * n).reshape(B, H, W) != 0
        self.store("x", a["x"], "f64", np.arange(B * n), np.zeros(B * n))
        rr = self.arr(a["rr"], "f64", B)
        for b in range(B):
            m = mask[b].reshape(-1)
            pix = np.nonzero(m)[0] + b * n
            rhs, e = np.zeros(0, HP), np.zeros(0)
            if m.any():
                _, _, R, _ = _system(mask[b])
                rhs = R @ img[b].astype(HP)
                nb = np.diff(R.indptr)
                e = U * np.maximum(nb - 1, 0) * (abs(R) @ np.abs(img[b]).astype(HP)) + nb * SUB
            for lab, p in (("r", a["r"]), ("p0", a["p0"])):
                out = np.full(n, HP(0))
                out[m] = rhs
                eb = np.zeros(n)
                eb[m] = e
                self.store(lab, p, "f64", np.arange(n) + b * n, out, "bar", eb)
            if pix.size:
                self.store("rr", a["rr"], "f64", [b], rr[b] + (rhs * rhs).sum(), "bar",
                           sum_bar(rhs * rhs, 2 * np.abs(rhs) * e + e * e, rr[b]))

    def _regionfill_iters(self, a):
        for k in range(a["k0"], a["k0"] + a["iters"]):
            self._cg_iteration(a, k)

    def _cg_iteration(self, a, k):
        B, H, W = a["B"], a["H"], a["W"]
        n = H * W
        mask = self.arr(a["mask"], "u8", B * n).reshape(B, H, W) != 0
        x, r = self.arr(a["x"], "f64", B * n), self.arr(a["r"], "f64", B * n)
        pold_p, pnew_p = (a["p0"], a["p1"]) if k % 2 == 0 else (a["p1"], a["p0"])
        p_old = self.arr(pold_p, "f64", B * n)
        rr, pap = self.arr(a["rr"], "f64", (k + 2) * B), self.arr(a["pap"], "f64", (k + 1) * B)
        for b in range(B):
            m = mask[b].reshape(-1)
            if not m.any():
                continue
            A, absA, _, off = _system(mask[b])
            sel = np.nonzero(m)[0] + b * n
            beta = 0.0
            if k > 0 and rr[(k - 1) * B + b] > 0:
                beta = rr[k * B + b] / rr[(k - 1) * B + b]
            rv, po = r[sel].astype(HP), p_old[sel].astype(HP)
            p = rv + HP(beta) * po
            M = np.abs(rv) + np.abs(HP(beta) * po)
            e_p = (2 * U * M + 2 * SUB).astype(np.float64)
            ap = A @ p
            n_ap = 3 + off
            e_ap = (U * n_ap * (absA @ M) + n_ap * SUB).astype(np.float64)
            self.store("p", pnew_p, "f64", sel, p, "bar", e_p)
            self.store("ap", a["ap"], "f64", sel, ap, "bar", e_ap)
            t = p * ap
            s_pap = pap[k * B + b] + t.sum()
            bar_pap = sum_bar(t, np.abs(p) * e_ap + np.abs(ap) * e_p + e_p * e_ap, pap[k * B + b])
            self.store("pap", a["pap"], "f64", [k * B + b], s_pap, "bar", bar_pap)
            alpha, rel = 0.0, 0.0
            if float(s_pap) > 0:
                alpha = rr[k * B + b] / float(s_pap)
                rel = bar_pap / float(s_pap) + U
            xv = x[sel].astype(HP)
            xa, ra = HP(alpha) * p, HP(alpha) * ap
            xn, rn = xv + xa, rv - ra
            e_x = 2 * U * (np.abs(xv) + np.abs(xa)) + abs(alpha) * e_p + np.abs(xa) * rel + 2 * SUB
            e_r = 2 * U * (np.abs(rv) + np.abs(ra)) + abs(alpha) * e_ap + np.abs(ra) * rel + 2 * SUB
            self.store("x", a["x"], "f64", sel, xn, "bar", e_x)
            self.store("r", a["r"], "f64", sel, rn, "bar", e_r)
            e_r = e_r.astype(np.float64)
            o = (k + 1) * B + b
            self.store("rr", a["rr"], "f64", [o], rr[o] + (rn * rn).sum(), "bar",
                       sum_bar(rn * rn, 2 * np.abs(rn) * e_r + e_r * e_r, rr[o]))

    def _regionfill_finish(self, a):
        N = a["total"]
        img, x = self.arr(a["img"], "f64", N), self.arr(a["x"], "f64", N)
        m = self.arr(a["mask"], "u8", N) != 0
        self.store("out", a["out"], "f64", np.arange(N), np.where(m, x, img))

    # --------------------------------------------------------------------------------------------------- poisson
    def _poisson_setup(self, a):
        F, H, W = a["F"], a["H"], a["W"]
        n = H * W
        trg = self.arr(a["trg"], "f64", F * n * 3).reshape(F, H, W, 3)
        gx = self.arr(a["gx"], "f64", F * H * (W - 1) * 3).reshape(F, H, W - 1, 3)
        gy = self.arr(a["gy"], "f64", F * (H - 1) * W * 3).reshape(F, H - 1, W, 3)
        hole = self.arr(a["hole"], "u8", F * n).reshape(F, H, W)
        gm, ed = (self.arr(a[k], "u8", F * n) for k in ("gmask", "edge"))
        zero = np.zeros((H, W), np.uint8)
        cnt, bb = self.arr(a["cnt"], "i32", F), self.arr(a["bb"], "f64", 3 * F)
        for f in range(F):
            code = PO.equation_codes(hole[f], zero if gm is None else gm.reshape(F, H, W)[f],
                                     zero if ed is None else ed.reshape(F, H, W)[f])
            b = PO.rhs(code, trg[f], gx[f], gy[f])                                        # [4, H, W, 3]
            self.store("code", a["code"], "u8", np.arange(n) + f * n, code)
            nn, yy, xx = np.nonzero((code[None] >> np.arange(4)[:, None, None]) & 1)
            eq = (((f * 4 + nn) * n + yy * W + xx) * 3)[:, None] + np.arange(3)
            self.store("u", a["u"], "f64", eq, b[nn, yy, xx])
            own = np.nonzero((code.reshape(-1) & 15) != 0)[0]
            c0 = int(cnt[f])
            self.store("list", a["list"], "i32", f * n + c0 + np.arange(own.size),
                       (own | (code.reshape(-1)[own].astype(np.int64) << 24)).astype(np.uint32).view(np.int32),
                       "multiset")
            self.store("cnt", a["cnt"], "i32", [f], np.int32(c0 + own.size))
            for c in range(3):
                t = b[nn, yy, xx, c].astype(HP) ** 2
                if t.size:
                    self.store("bb", a["bb"], "f64", [3 * f + c], bb[3 * f + c] + t.sum(), "bar",
                               sum_bar(t, np.zeros(t.size), bb[3 * f + c]))

    def _poisson_unfilled(self, a):
        F, H, W = a["F"], a["H"], a["W"]
        n = H * W
        hole = self.arr(a["hole"], "u8", F * n).reshape(F, H, W)
        gm = self.arr(a["gmask"], "u8", F * n)
        out = np.zeros((2, F, H, W), np.uint8)
        for f in range(F):
            tl, br = PO.unfilled_sweeps(hole[f], np.zeros((H, W), np.uint8) if gm is None else gm.reshape(F, H, W)[f])
            out[0, f], out[1, f] = ~tl, ~br
        self.store("clr", a["clr"], "u8", np.arange(out.size), out)

    def _poisson_finish(self, a):
        F, H, W = a["F"], a["H"], a["W"]
        N = F * H * W
        trg, x = self.arr(a["trg"], "f64", N * 3).reshape(N, 3), self.arr(a["x"], "f64", N * 3).reshape(N, 3)
        h = self.arr(a["hole"], "u8", N) != 0
        self.x_final = x.copy()
        self.store("out", a["out"], "f64", np.arange(N * 3),
                   np.where(h[:, None], x.astype(np.float32).astype(np.float64), trg))
        if a["unf"] is not None:
            clr = self.arr(a["clr"], "u8", 2 * N).reshape(2, N)
            self.store("unf", a["unf"], "u8", np.arange(N), (h & (clr[0] == 0) & (clr[1] == 0)).astype(np.uint8))

    def _poisson_iters(self, a):
        for _ in range(a["iters"]):
            self._lsqr_iteration(a)

    def _poisson_graph_create(self, a):
        h = self._next_graph
        self._next_graph += 16
        self.graphs[h] = {k: v for k, v in a.items() if k != "exec_out"}
        a["exec_out"]._obj.value = h

    def _poisson_graph_launch(self, a):
        self._poisson_iters(self.graphs[a["exec"]])

    def _poisson_graph_destroy(self, a):
        self.graphs.pop(a["exec"], None)

    def _lsqr_iteration(self, a):
        F, H, W = a["F"], a["H"], a["W"]
        n, S = H * W, 3 * F
        kctr = self.arr(a["kctr"], "i32", 2)
        k = int(kctr[0])
        self.store("kctr", a["kctr"], "i32", [1, 0], np.array([k, k + 1], np.int32))
        lst = self.arr(a["list"], "i32", F * n).reshape(F, n).view(np.uint32)[:, :a["max_cnt"]]
        u = self.arr(a["u"], "f64", F * 4 * n * 3).reshape(F, 4, n, 3)
        v, w, x = (self.arr(a[q], "f64", F * n * 3).reshape(F, n, 3) for q in "vwx")
        slots = (k + 2) * S
        bb, aa, ww = (self.arr(a[q], "f64", slots) for q in ("bb", "aa", "ww"))
        state = self.arr(a["state"], "f64", 2 * S * 16).reshape(2, S, 16)
        ctol = 1.0 / a["conlim"] if a["conlim"] > 0 else 0.0
        hp = HP if self.bars else np.float64
        for f in range(F):
            code = np.zeros(n, np.uint8)
            ent = lst[f][((lst[f] >> 24) & 15) != 0]
            code[(ent & 0xFFFFFF).astype(np.int64)] = (ent >> 24).astype(np.uint8)
            code = code.reshape(H, W)
            own = np.nonzero((code.reshape(-1) & 15) != 0)[0]
            nt = _pop(code.reshape(-1)[own])                         # u terms of (A^T u)[p]
            eqn, eqp = np.nonzero(((code.reshape(-1)[None] >> np.arange(4)[:, None]) & 1) != 0)
            for c in range(3):
                s = 3 * f + c
                prev = state[(k + 1) & 1, s].tolist()
                done = k >= 1 and prev[DONE] != 0
                beta = math.sqrt(bb[k * S + s])
                vo = v[f, :, c].astype(hp)
                vk, e_v, rel_a = vo, np.zeros(n), 0.0
                if not done and beta > 0:                         # v = A^T u / beta - beta P[9] v
                    inv = 1.0 / beta
                    coef = beta * prev[9] if k >= 1 else 0.0
                    uh = u[f, :, :, c].reshape(4, H, W).astype(hp)
                    vk = (PO.rmatvec(code, uh) * hp(inv)).reshape(-1) - hp(coef) * vo
                    vk = np.where((code.reshape(-1) & 15) != 0, vk, vo)
                    if self.bars:
                        mag = _abs_op(PO.rmatvec, code, np.abs(uh)).reshape(-1)[own] * inv + np.abs(coef * vo[own])
                        e_v[own] = (U * (nt + 2) * mag + (nt + 2) * SUB).astype(np.float64)
                    self.store("v", a["v"], "f64", (f * n + own) * 3 + c, vk[own], "bar", e_v[own], s)
                    t = vk[own] ** 2
                    a_new = aa[k * S + s] + t.sum()
                    bar_aa = sum_bar(t, 2 * np.abs(vk[own]) * e_v[own] + e_v[own] ** 2, aa[k * S + s]) \
                        if self.bars else 0.0
                    self.store("aa", a["aa"], "f64", [k * S + s], a_new, "bar", bar_aa, s)
                    rel_a = bar_aa / (2 * float(a_new)) if float(a_new) > 0 else 0.0
                    aak = float(a_new)
                else:
                    aak = aa[k * S + s]
                cur, (t1, t2, vscale, au), skip_all, skip_u, near = lsqr_step(
                    prev, k, bb[k * S + s], aak, ww[k * S + s], a["atol"], a["btol"], ctol, a["iter_lim"])
                if near:
                    self.near.append((s, k))
                self.store("state", a["state"], "f64", ((k & 1) * S + s) * 16 + np.arange(16), np.array(cur), "state",
                           sys=np.full(16, s))
                if skip_all:
                    continue
                wo, xo = w[f, own, c].astype(hp), x[f, own, c].astype(hp)
                vn = vk * hp(vscale)
                e_vn = abs(vscale) * e_v + np.abs(vn).astype(np.float64) * (rel_a + U)
                xa, wa = hp(t1) * wo, hp(t2) * wo
                xn, wn = xo + xa, vn[own] + wa
                e_x = 2 * U * (np.abs(xo) + np.abs(xa)) + ROUND_T1 * U * np.abs(xa) + 2 * SUB
                e_w = (e_vn[own] + 2 * U * (np.abs(vn[own]) + np.abs(wa)) + (rel_a + ROUND_T2 * U) * np.abs(wa)
                       + 3 * SUB).astype(np.float64)
                self.store("x", a["x"], "f64", (f * n + own) * 3 + c, xn, "bar", e_x, s)
                self.store("w", a["w"], "f64", (f * n + own) * 3 + c, wn, "bar", e_w, s)
                o = (k + 1) * S + s
                self.store("ww", a["ww"], "f64", [o], ww[o] + (wn * wn).sum(), "bar",
                           sum_bar(wn * wn, 2 * np.abs(wn) * e_w + e_w * e_w, ww[o]) if self.bars else 0.0, s)
                if skip_u:
                    continue
                uo = u[f, eqn, eqp, c].astype(hp)
                av = PO.matvec(code, vn.reshape(H, W)).reshape(4, n)[eqn, eqp]
                ua = hp(au) * uo
                un = av - ua
                e_u = np.zeros(eqn.size)
                if self.bars:
                    mag_av = _abs_op(PO.matvec, code, np.abs(vn).reshape(H, W)).reshape(4, n)[eqn, eqp]
                    e_av = _abs_op(PO.matvec, code, e_vn.reshape(H, W)).reshape(4, n)[eqn, eqp] + U * mag_av
                    e_u = (e_av + (rel_a + U) * np.abs(ua) + 2 * U * (mag_av + np.abs(ua)) + 4 * SUB).astype(np.float64)
                self.store("u", a["u"], "f64", ((f * 4 + eqn) * n + eqp) * 3 + c, un, "bar", e_u, s)
                self.store("bb", a["bb"], "f64", [o], bb[o] + (un * un).sum(), "bar",
                           sum_bar(un * un, 2 * np.abs(un) * e_u + e_u * e_u, bb[o]) if self.bars else 0.0, s)


@contextlib.contextmanager
def emulating(monkeypatch, bars=False):
    """`with emulating(monkeypatch) as emu:` runs poisson_blend_batch / regionfill_batch on CPU tensors with every
    launch interpreted (`bars` as in SolverEmulator)."""
    from fgt_b200 import poisson, regionfill
    from tests.test_launch_trace import recording
    emu = SolverEmulator()
    emu.bars = bars
    cpu = lambda device=None: torch.device("cpu")
    monkeypatch.setattr(poisson, "_dev", cpu)
    monkeypatch.setattr(regionfill, "_dev", cpu)
    with recording(emu):
        yield emu
