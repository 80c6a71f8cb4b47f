"""CPU oracle for gradient-domain (Poisson) blending (TEST INFRASTRUCTURE — see oracle/fgt_oracle.py).

Restates /root/reference/tool/utils/Poisson_blend_img.py:19-270 (`Poisson_blend_img`, `solvePoisson`,
`constructEquation`), the driver's call at tool/video_inpainting.py:645-656, matrix-free:

* Unknowns: the pixels of `holeMask`. For every hole pixel p and each of its 4 neighbours q = p + d_n
  (n = 0 right, 1 down, 2 left, 3 up; :91-99) there is one equation when q is inside the image (:131),
  neither p nor q is an edge pixel (:189) and the gradient between them is known (`gradientMask` == 0 at the
  pixel that owns the forward difference: p for n = 0/1, the left / upper neighbour for n = 2/3; :192-199):
      q outside the hole:  x_p        = s_n * g + imgTrg[q]      (:201-227)
      q inside the hole:   x_p - x_q  = s_n * g                  (:235-266)
  with g = imgSrc_gx[p] (n=0), imgSrc_gx[left of p] (n=2), imgSrc_gy[p] (n=1), imgSrc_gy[above p] (n=3) and
  s_n = -1 for n = 0/1, +1 for n = 2/3. Every in-hole edge therefore appears twice (once from each end).
* The over-determined system is solved per colour channel by scipy's `lsqr` with its DEFAULT tolerances
  (atol = btol = 1e-6, conlim = 1e8, iter_lim = 2·H·W; :38) starting from x = 0 — i.e. the result is the LSQR
  iterate at which the stopping rule fires, not the converged least-squares solution (they differ by up to
  ~1e-4 on [0,1] images). `lsqr()` below restates Paige & Saunders' algorithm as scipy 1.18.1 implements it
  (scipy/sparse/linalg/_isolve/lsqr.py; third-party, not under /root/reference), including every stopping
  test, in float64. The reference feeds float32 `A`/`b`, so scipy runs the bidiagonalisation in float32;
  float64 iterates stop at the same iteration and agree to ~1e-6 (tests/golden/poisson_*.npz pin this).
* The reconstruction is stored in a float32 image (:29,40) and blended in float64:
  out = hole ? float64(float32(x)) : imgTrg (:43-44).
* `UnfilledMask` (:139-172): hole pixels that cannot be reached from outside the hole through known
  gradients, as the product of a forward raster sweep (from the up / left neighbour) and a backward sweep
  (from the down / right neighbour). Restated as the same two sweeps, vectorised per row.
"""
import math

import numpy as np

EPS = np.finfo(np.float64).eps
DY = (0, 1, 0, -1)
DX = (1, 0, -1, 0)


def equation_codes(hole, gmask, edge):
    """uint8 [H,W]: bit n = equation (p, n) exists, bit 4+n = its neighbour lies inside the hole."""
    hole = np.asarray(hole).astype(bool)
    gm = np.asarray(gmask) != 0
    ed = np.asarray(edge) != 0
    H, W = hole.shape
    code = np.zeros((H, W), dtype=np.uint8)
    ys, xs = np.nonzero(hole)
    for n in range(4):
        qy, qx = ys + DY[n], xs + DX[n]
        inside = (qy >= 0) & (qy < H) & (qx >= 0) & (qx < W)
        qyc, qxc = np.where(inside, qy, 0), np.where(inside, qx, 0)
        not_edge = ~ed[ys, xs] & ~ed[qyc, qxc]
        if n in (0, 1):
            have = ~gm[ys, xs]
        elif n == 2:
            have = ~gm[ys, np.where(inside, xs - 1, 0)]
        else:
            have = ~gm[np.where(inside, ys - 1, 0), xs]
        valid = inside & not_edge & have
        inh = valid & hole[qyc, qxc]
        code[ys, xs] |= (valid.astype(np.uint8) << n) | (inh.astype(np.uint8) << (4 + n))
    return code


def rhs(code, trg, gx, gy):
    """b [4,H,W,C] float64 (zero where no equation). gx [H,W-1,C], gy [H-1,W,C] forward differences."""
    H, W = code.shape
    C = trg.shape[2]
    trg = np.asarray(trg, dtype=np.float64)
    gxp = np.zeros((H, W, C)); gxp[:, :W - 1] = gx
    gyp = np.zeros((H, W, C)); gyp[:H - 1] = gy
    b = np.zeros((4, H, W, C))
    ys, xs = np.nonzero(code & 15)
    for n in range(4):
        sel = ((code[ys, xs] >> n) & 1).astype(bool)
        y, x = ys[sel], xs[sel]
        qy, qx = y + DY[n], x + DX[n]
        g = (-gxp[y, x], -gyp[y, x], gxp[y, x - 1], gyp[y - 1, x])[n]
        bnd = ~((code[y, x] >> (4 + n)) & 1).astype(bool)
        b[n, y, x] = g + np.where(bnd[:, None], trg[qy, qx], 0.0)
    return b


def _shift(a, n):
    """a[q] sampled at p, q = p + d_n, zero outside the image."""
    out = np.zeros_like(a)
    if n == 0:
        out[:, :-1] = a[:, 1:]
    elif n == 1:
        out[:-1] = a[1:]
    elif n == 2:
        out[:, 1:] = a[:, :-1]
    else:
        out[1:] = a[:-1]
    return out


def matvec(code, v):
    """(A v)[n,p] = v_p - [q in hole] v_q for the equations that exist. v [H,W] (any float dtype, kept)."""
    u = np.zeros((4,) + v.shape, dtype=v.dtype)
    for n in range(4):
        valid = ((code >> n) & 1).astype(bool)
        inh = ((code >> (4 + n)) & 1).astype(bool)
        u[n] = np.where(valid, v - np.where(inh, _shift(v, n), 0.0), 0.0)
    return u


def rmatvec(code, u):
    """(A^T u)[p] = sum_n u[n,p] - sum_n u[(n+2)%4, q_n] over neighbours q_n whose equation towards p is in-hole."""
    out = np.zeros(u.shape[1:], dtype=u.dtype)
    for n in range(4):
        out += np.where(((code >> n) & 1).astype(bool), u[n], 0.0)
        m = (n + 2) % 4
        contrib = np.where(((code >> (4 + m)) & 1).astype(bool), u[m], 0.0)   # lives at q, addressed to q + d_m = p
        out -= _shift(contrib, n)
    return out


def _sym_ortho(a, b):
    """scipy/sparse/linalg/_isolve/lsqr.py:_sym_ortho (stable Givens rotation)."""
    if b == 0:
        return np.sign(a), 0.0, abs(a)
    if a == 0:
        return 0.0, np.sign(b), abs(b)
    if abs(b) > abs(a):
        tau = a / b
        s = np.sign(b) / math.sqrt(1 + tau * tau)
        c = s * tau
        r = b / s
    else:
        tau = b / a
        c = np.sign(a) / math.sqrt(1 + tau * tau)
        s = c * tau
        r = a / c
    return c, s, r


def lsqr(code, b, atol=1e-6, btol=1e-6, conlim=1e8, iter_lim=None):
    """LSQR on the matrix-free operator, x0 = 0, damp = 0. b [4,H,W] -> (x [H,W], istop, itn)."""
    H, W = code.shape
    if iter_lim is None:
        iter_lim = 2 * H * W
    ctol = 1.0 / conlim if conlim > 0 else 0.0
    x = np.zeros((H, W))
    bnorm = float(np.linalg.norm(b))
    beta = bnorm
    if beta > 0:
        u = b / beta
        v = rmatvec(code, u)
        alfa = float(np.linalg.norm(v))
    else:
        u = b.copy()
        v = np.zeros((H, W))
        alfa = 0.0
    if alfa > 0:
        v = v / alfa
    w = v.copy()
    rhobar, phibar = alfa, beta
    anorm = ddnorm = xxnorm = z = 0.0
    cs2, sn2 = -1.0, 0.0
    itn = istop = 0
    if alfa * beta == 0:
        return x, 0, 0
    while itn < iter_lim:
        itn += 1
        u = matvec(code, v) - alfa * u
        beta = float(np.linalg.norm(u))
        if beta > 0:
            u = u / beta
            anorm = math.sqrt(anorm * anorm + alfa * alfa + beta * beta)
            v = rmatvec(code, u) - beta * v
            alfa = float(np.linalg.norm(v))
            if alfa > 0:
                v = v / alfa
        cs, sn, rho = _sym_ortho(rhobar, beta)
        theta = sn * alfa
        rhobar = -cs * alfa
        phi = cs * phibar
        phibar = sn * phibar
        tau = sn * phi
        t1 = phi / rho
        t2 = -theta / rho
        ddnorm += float(np.linalg.norm(w / rho)) ** 2
        x = x + t1 * w
        w = v + t2 * w
        delta = sn2 * rho
        gambar = -cs2 * rho
        rhs_ = phi - delta * z
        zbar = rhs_ / gambar
        xnorm = math.sqrt(xxnorm + zbar * zbar)
        gamma = math.sqrt(gambar * gambar + theta * theta)
        cs2 = gambar / gamma
        sn2 = theta / gamma
        z = rhs_ / gamma
        xxnorm += z * z
        acond = anorm * math.sqrt(ddnorm)
        rnorm = abs(phibar)
        arnorm = alfa * abs(tau)
        test1 = rnorm / bnorm
        test2 = arnorm / (anorm * rnorm + EPS)
        test3 = 1.0 / (acond + EPS)
        t1_ = test1 / (1 + anorm * xnorm / bnorm)
        rtol = btol + atol * anorm * xnorm / bnorm
        if itn >= iter_lim:
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
        if istop:
            break
    return x, istop, itn


def unfilled_mask(hole, gmask):
    """Poisson_blend_img.py:139-172 / getUnfilledMask :270-309. hole, gmask [H,W] -> bool [H,W]."""
    tl, br = unfilled_sweeps(hole, gmask)
    return tl & br


def unfilled_sweeps(hole, gmask):
    """The two sweeps of unfilled_mask: (forward, backward) bool [H,W], True = hole pixel the sweep leaves unfilled."""
    hole = np.asarray(hole).astype(bool)
    gm = np.asarray(gmask) != 0
    H, W = hole.shape
    ok = ~gm                                   # a cleared pixel with a known gradient lets its successor clear
    tl = hole.copy()                           # 1 = still unfilled
    for i in range(H):
        up = np.zeros(W, bool) if i == 0 else (~tl[i - 1] & ok[i - 1])
        row = tl[i] & ~up
        for j in range(1, W):                  # left-to-right dependency inside the row
            if row[j] and not row[j - 1] and ok[i, j - 1]:
                row[j] = False
        tl[i] = row
    br = hole.copy()
    for i in range(H - 1, -1, -1):
        down = np.zeros(W, bool) if i == H - 1 else (~br[i + 1] & ok[i])
        row = br[i] & ~down
        for j in range(W - 2, -1, -1):
            if row[j] and not row[j + 1] and ok[i, j]:
                row[j] = False
        br[i] = row
    return tl, br


def poisson_blend(trg, gx, gy, hole, gmask=None, edge=None, return_info=False):
    """Poisson_blend_img.py:19-44. trg [H,W,3], gx [H,W-1,3], gy [H-1,W,3], hole [H,W] -> (blend float64 [H,W,3],
    UnfilledMask bool [H,W])."""
    trg = np.asarray(trg)
    hole = np.asarray(hole).astype(bool)
    H, W, C = trg.shape
    gmask = np.zeros((H, W), bool) if gmask is None else np.asarray(gmask)
    edge = np.zeros((H, W), bool) if edge is None else np.asarray(edge)
    code = equation_codes(hole, gmask, edge)
    b = rhs(code, trg, np.asarray(gx, dtype=np.float64), np.asarray(gy, dtype=np.float64))
    out = np.asarray(trg, dtype=np.float64).copy()
    info = []
    for c in range(C):
        x, istop, itn = lsqr(code, b[..., c])
        info.append((istop, itn))
        out[..., c][hole] = x.astype(np.float32).astype(np.float64)[hole]
    unf = unfilled_mask(hole, gmask)
    return (out, unf, info) if return_info else (out, unf)
