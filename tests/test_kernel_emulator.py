"""The float64 interpreters of tests/kernel_emulator.py against independent float64 statements of the reference
operations, at the argument forms the forwards use and at the edges where such kernels go wrong; whole forwards run
through them on the CPU against the reference goldens and oracles.

- Coverage: every entry of the launch-trace golden has an interpreter, and every form (`kernel_emulator.form`: the
  discrete options of one call) that occurs in the seven golden traces has a case here. A forward that starts calling a
  new kernel, or a kernel with a new option, fails `test_every_trace_form_has_a_case`.
- Cases: each launches the production launcher (`lib.*`) under `emulating_all()` and compares the interpreter's float64
  values with `F.layer_norm`, `F.fold` / `F.unfold`, `F.conv2d` (depthwise and 3x3), `F.instance_norm`,
  `F.avg_pool2d`, `F.interpolate` (nearest, and bilinear for upflow8), `oracle.raft_oracle.corr_lookup` /
  `upsample_flow`, or a float64 softmax attention written per zone and per window. Bar EXACT (1e-12 of the largest
  value): the reference is fed the operands as stored. The stored elements must be exactly the operation's own (rows
  past nl + G of swin_prep, columns past the lookup values of the lookup rows, the channels outside the flow slice,
  dropped attention rows are not), each the float64 value in its output format, and every other element keeps its
  sentinel bit for bit. upflow8 is compared on its fp32 output at 1e-6 of (1 + the largest value).
- Whole forwards in float64 on CPU tensors, bars rel-L2 and max/max <= 1e-4 (rel-L2 / max-over-max observed): FGT fp32
  at 64 x 96, t = 3, 1.55e-5 / 2.13e-5 against both its golden and the oracle (its flow branch is 1-term fp16 by
  design); LAFC at 64 x 96 5.6e-6 / 1.0e-5 (flow) and 4.1e-7 / 1.9e-6 (edge); RAFT at 128 x 160, 3 iterations, against
  the oracle 1.9e-5 / 2.2e-5 (low) and 1.1e-5 / 1.6e-5 (up). What is left is the rounding of stored activations to
  split-bf16 (and fp16 in FGT's flow branch).
- The 1-pixel pyramid level: at 64 x 96 RAFT's coarsest correlation level is 1 x 1. The reference sampler divides by
  W - 1 and H - 1 there and returns NaN; the interpreter (and the kernel) sample it bilinearly with zero padding.
"""
import argparse
import functools
import gzip
import json

import pytest
import torch
import torch.nn.functional as F

from fgt_b200 import lib, synth
from oracle import raft_oracle as RO
from tests.kernel_emulator import ENTRIES, emulating_all, form
from tests.test_launch_trace import GOLDEN
from tests.util import load_golden, max_over_max, rel_l2

EXACT = 1e-12
SENTINEL = -1234.5
FWD_TOL = 1e-4


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(*shape, seed, scale=1.0, shift=0.0):
    return torch.randn(*shape, generator=_gen(seed)) * scale + shift


def _buf(shape, fmt):
    """A sentinel-filled output: "f32" [*shape], "f16" [*shape] or "split" [2, *shape]."""
    if fmt == "split":
        return torch.full((2,) + tuple(shape), SENTINEL, dtype=torch.bfloat16)
    return torch.full(tuple(shape), SENTINEL, dtype=torch.float16 if fmt == "f16" else torch.float32)


def _act16(x, fmt):
    """x stored in a 16-bit format and the float64 value of what is stored."""
    t = x.half() if fmt == "f16" else lib.to_split(x)
    return t, _val(t)


def _val(t):
    if t.dtype == torch.bfloat16:
        return t[0].double() + t[1].double()
    return t.double()


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32 if t.element_size() == 4 else torch.int64)


def _check(emu, out, before, ref, what, ref_f32=False):
    """The interpreter stored exactly the elements where ref (float64, out's logical shape) is not NaN, with float64
    values within EXACT of ref, each stored in out's format; every other element of out kept its bits. ref_f32: the
    reference rounds its result to fp32 (oracle.raft_oracle.corr_lookup), so each element may also differ by that
    rounding, 2^-24 of its magnitude."""
    got = emu.stored(out)
    want = ~torch.isnan(ref)
    assert torch.equal(~torch.isnan(got), want), f"{what}: stored elements differ from the operation's own"
    if want.any():
        g, r = got[want], ref[want]
        slack = 2.0 ** -24 * r.abs() if ref_f32 else 0.0
        err = (((g - r).abs() - slack).clamp_min(0).max() / r.abs().max().clamp_min(1e-300)).item()
        assert err <= EXACT, f"{what}: interpreter vs reference {err:.3e}"
        g = got[want]
        if out.dtype == torch.bfloat16:
            assert torch.equal(out[:, want], lib.to_split(g.float())), f"{what}: split store"
        else:
            assert torch.equal(out[want], g.to(out.dtype)), f"{what}: store rounding"
    mask = emu.written_mask(out)
    assert torch.equal(_bits(out)[~mask], _bits(before)[~mask]), f"{what}: elements outside the operation written"
    return got


def _run(fn):
    """fn() under the interpreter; returns the emulator."""
    with torch.no_grad(), emulating_all() as emu:
        fn()
    return emu


CASES = {}


def case(*forms_params, ids=None):
    """Registers a case function for each parameter tuple (name: function name + id)."""
    def deco(fn):
        for i, p in enumerate(forms_params):
            key = fn.__name__[1:] + ("" if not forms_params[1:] and ids is None else f"[{ids[i] if ids else i}]")
            CASES[key] = functools.partial(fn, *p)
        return fn
    return deco


# ------------------------------------------------------------------------------------------------------ im2col_nchw
IM2COL = [  # fmt, two sources, replicate, k, stride, scaled: the forms of the traces, at odd sizes
    ("split", True, False, 3, 2, False), ("f16", True, False, 3, 2, False), ("f16", False, True, 5, 1, False),
    ("split", False, True, 5, 1, False), ("split", False, False, 3, 1, False), ("split", False, False, 7, 1, False),
    ("f16", False, False, 7, 1, False), ("split", False, False, 7, 2, True), ("f16", False, False, 7, 2, True),
    ("f16", False, False, 3, 1, False), ("split", True, True, 5, 1, False),
]


@case(*IM2COL, ids=["-".join(map(str, p)) for p in IM2COL])
def _im2col(fmt, two, replicate, k, stride, scaled):
    n, H, W, c0, c1 = 2, 13, 17, 2 if two else 3, 1 if two else 0
    pad = k // 2
    s0, s1 = _randn(n, c0, H, W, seed=1), (_randn(n, c1, H, W, seed=2) if two else None)
    cin = c0 + c1
    cpad = (k * k * cin + 7) // 8 * 8 + 8
    OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    scale, shift = (2.0 / 255.0, -1.0) if scaled else (1.0, 0.0)
    if scaled:
        s0 = torch.randint(0, 256, s0.shape, generator=_gen(3)).float()
    out = _buf((n, OH, OW, cpad), fmt)
    before = out.clone()
    emu = _run(lambda: lib.im2col_nchw(s0, s1, out, k=k, stride=stride, pad=pad, replicate=replicate, OH=OH, OW=OW,
                                       scale=scale, shift=shift))
    x = torch.cat([s0, s1], 1).double() if two else s0.double()
    sc = torch.tensor(scale, dtype=torch.float32).item()
    x = x * sc + torch.tensor(shift, dtype=torch.float32).item()
    x = F.pad(x, (pad,) * 4, mode="replicate" if replicate else "constant")
    u = F.unfold(x, k, stride=stride).view(n, cin, k * k, OH, OW).permute(0, 3, 4, 2, 1).reshape(n, OH, OW, -1)
    ref = torch.zeros(n, OH, OW, cpad, dtype=torch.float64)
    ref[..., :k * k * cin] = u
    _check(emu, out, before, ref, "im2col")
    return emu.forms


# ---------------------------------------------------------------------------------------------------------- rownorm
ROWNORM = [  # fmt, gather, affine, two sources, destination remap
    ("split", False, False, False, False), ("f16", False, False, False, False), ("split", True, True, False, False),
    ("f16", True, True, False, False), ("split", True, False, True, True), ("f16", False, True, True, True),
]


@case(*ROWNORM, ids=["-".join(map(str, p)) for p in ROWNORM])
def _rownorm(fmt, gather, affine, two, remap):
    rpb, nb = 19, 3                               # odd rows per batch
    total = rpb * nb
    ca, cb, nsrc = 20, (12 if two else 0), (45 if gather else total)
    C = ca + cb
    a = _randn(nsrc, ca, seed=4, scale=2.0, shift=3.0)
    a[:3] = 0.75                                  # constant rows: eps alone sets the scale
    a[3:8] = _randn(5, ca, seed=41, scale=1e-3, shift=0.5)   # spread 1e-3, below sqrt(eps)
    b = _randn(nsrc, cb, seed=5) if two else None
    g = torch.randint(-1, nsrc, (total,), generator=_gen(6), dtype=torch.int32) if gather else None
    dbr, r0 = (rpb + 5, 2) if remap else (rpb, 0)
    gm, bt = (_randn(C, seed=7), _randn(C, seed=8)) if affine else (None, None)
    out = _buf((nb * dbr + 3, C), fmt)
    before = out.clone()
    emu = _run(lambda: lib.rownorm(a, b, out, gather=g, rows_per_batch=rpb, total_rows=total, dst_batch_rows=dbr,
                                   dst_row0=r0, eps=1e-5, gamma=gm, beta=bt))
    X = torch.cat([a, b], 1).double() if two else a.double()
    src = g.long() if gather else torch.arange(total)
    eps = torch.tensor(1e-5, dtype=torch.float32).item()
    y = F.layer_norm(X[src.clamp_min(0)], (C,), gm.double() if affine else None, bt.double() if affine else None, eps)
    y[src < 0] = 0.0
    ref = torch.full((nb * dbr + 3, C), float("nan"), dtype=torch.float64)
    d = torch.arange(total)
    ref[(d // rpb) * dbr + r0 + d % rpb] = y
    _check(emu, out, before, ref, "rownorm")
    return emu.forms


# -------------------------------------------------------------------------------------------------------- attention
ATTN = [  # f16, mode, row map, Lq < Lk (dense)
    (False, 0, True, False), (True, 0, True, False), (False, 1, True, False), (True, 1, True, False),
    (False, 0, True, True), (False, 0, False, False), (False, 1, False, False),
]


@case(*ATTN, ids=["-".join(map(str, p)) for p in ATTN])
def _attention(f16, mode, rowmap, short_q):
    heads, B = 2, 3
    C = heads * 128
    fmt = "f16" if f16 else "split"
    if mode == 0:
        Lk = 100                                   # a partial last key tile
        Lq = 70 if short_q else Lk
        R = Lk
    else:
        Lq, G = 256, 45                            # four 64-token windows, an odd number of pooled keys
        Lk = R = Lq + G + 3                        # padding rows after the pooled ones
    qkv, val = _act16(_randn(B * R, 3 * C, seed=9, scale=0.35), fmt)
    rows_out = B * Lq + 5
    m = None
    if rowmap:
        m = torch.randperm(rows_out, generator=_gen(10))[:B * Lq].to(torch.int32)
        m[torch.randperm(B * Lq, generator=_gen(11))[:B * Lq // 7]] = -1
    out = _buf((rows_out, C), fmt)
    before = out.clone()
    kw = dict(glob_start=Lq, glob_count=G) if mode == 1 else {}
    emu = _run(lambda: lib.attention(qkv, qkv, qkv, out, batches=B, heads=heads, Lq=Lq, Lk=Lk, Lk_rows=R, q_ld=3 * C,
                                     k_ld=3 * C, v_ld=3 * C, out_ld=C, q_batch_stride=R * 3 * C,
                                     k_batch_stride=R * 3 * C, v_batch_stride=R * 3 * C, out_batch_stride=Lq * C,
                                     scale=1.0 / 128 ** 0.5, mode=mode, k_off=C, v_off=2 * C, out_rowmap=m, **kw))
    sc = torch.tensor(1.0 / 128 ** 0.5, dtype=torch.float32).item()
    v = val.view(B, R, 3, heads, 128)
    res = torch.empty(B, Lq, heads, 128, dtype=torch.float64)
    for b in range(B):
        for h in range(heads):
            q, k, vv = v[b, :, 0, h], v[b, :, 1, h], v[b, :, 2, h]
            if mode == 0:                      # a zone: every query sees the zone's Lk keys
                res[b, :, h] = torch.softmax(q[:Lq] @ k[:Lk].t() * sc, -1) @ vv[:Lk]
            else:                              # a window: its own 64 keys and the pooled ones
                for w in range(Lq // 64):
                    keys = torch.cat([torch.arange(w * 64, w * 64 + 64), torch.arange(Lq, Lq + G)])
                    res[b, w * 64:w * 64 + 64, h] = torch.softmax(q[w * 64:w * 64 + 64] @ k[keys].t() * sc,
                                                                  -1) @ vv[keys]
    res = res.reshape(B * Lq, C)
    ref = torch.full((rows_out, C), float("nan"), dtype=torch.float64)
    if rowmap:
        keep = m >= 0
        ref[m[keep].long()] = res[keep]
    else:
        ref[:B * Lq] = res
    _check(emu, out, before, ref, "attention")
    return emu.forms


# ------------------------------------------------------------------------------------------------- fold / fold_unfold
def _fold_geo():
    bt, C, k, s, p, OH, OW = 2, 8, 7, 3, 3, 20, 23
    return bt, C, k, s, p, OH, OW, (OH + 2 * p - k) // s + 1, (OW + 2 * p - k) // s + 1


def _torch_patches(hid, bt, th, tw, C, k):    # position-major [bt*L, P*C] -> nn.Fold's [bt, C*P, L]
    return hid.view(bt, th * tw, k * k, C).permute(0, 3, 2, 1).reshape(bt, C * k * k, th * tw)


@case(("split",), ("f16",), ids=["split", "f16"])
def _fold_unfold(fmt):
    bt, C, k, s, p, OH, OW, th, tw = _fold_geo()
    hid = _randn(bt * th * tw, k * k * C, seed=12)
    out = _buf((bt * th * tw, k * k * C), fmt)
    before = out.clone()
    emu = _run(lambda: lib.fold_unfold(hid, bt, th, tw, C, k, k, s, p, OH, OW, out, relu=True))
    x = _torch_patches(hid.double(), bt, th, tw, C, k)
    img = F.fold(x, (OH, OW), k, padding=p, stride=s)
    img = F.relu(img / F.fold(torch.ones_like(x), (OH, OW), k, padding=p, stride=s))
    u = F.unfold(img, k, padding=p, stride=s).view(bt, C, k * k, th * tw).permute(0, 3, 2, 1)
    _check(emu, out, before, u.reshape(bt * th * tw, k * k * C), "fold_unfold")
    return emu.forms


@case(("split", False), ("f16", False), ("f16", True), ids=["split", "f16", "f16-f32-normalize"])
def _fold(fmt, normalize):
    bt, C, k, s, p, OH, OW, th, tw = _fold_geo()
    hid = _randn(bt * th * tw, k * k * C, seed=13)
    add = _randn(bt, OH, OW, C, seed=14)
    out = _buf((bt, OH, OW, C), fmt)
    o32 = _buf((bt, OH, OW, C), "f32") if normalize else None
    before = out.clone()
    emu = _run(lambda: lib.fold(hid, bt, th, tw, C, k, k, s, p, OH, OW, normalize=normalize, add=add, out=o32,
                                out_split=out))
    x = _torch_patches(hid.double(), bt, th, tw, C, k)
    img = F.fold(x, (OH, OW), k, padding=p, stride=s)
    if normalize:
        img = img / F.fold(torch.ones_like(x), (OH, OW), k, padding=p, stride=s)
    ref = img.permute(0, 2, 3, 1) + add.double()
    _check(emu, out, before, ref, "fold")
    if normalize:
        _check(emu, o32, _buf(o32.shape, "f32"), ref, "fold fp32")
    return emu.forms


# ---------------------------------------------------------------------------------------------------- dwconv3x3_res
@case(("split",), ("f16",), (None,), ids=["split", "f16", "f32"])
def _dwconv3x3_res(fmt):
    bt, h, w, C = 2, 7, 11, 12
    x = _randn(bt, h, w, C, seed=15)
    wt, bias = _randn(C, 1, 3, 3, seed=16), _randn(C, seed=17)
    out = _buf((bt, h, w, C), "f32")
    o16 = _buf((bt, h, w, C), fmt) if fmt else None
    b16 = o16.clone() if fmt else None
    emu = _run(lambda: lib.dwconv3x3_res(x, bt, h, w, C, wt, bias, out, o16))
    xn = x.double().permute(0, 3, 1, 2)
    ref = (xn + F.conv2d(xn, wt.double(), bias.double(), padding=1, groups=C)).permute(0, 2, 3, 1)
    _check(emu, out, _buf(out.shape, "f32"), ref, "dwconv3x3_res fp32")
    if fmt:
        _check(emu, o16, b16, ref, "dwconv3x3_res 16-bit")
    return emu.forms


# -------------------------------------------------------------------------------------------------------- swin_prep
@case(("split",), ("f16",), ids=["split", "f16"])
def _swin_prep(fmt):
    """Three 8x8 windows over a 7 x 20 grid (padded to 8 x 24) and the dummy fourth window that makes the query tiles
    whole; pooled grid 2 x 5 with gd = 4 (the last pooled row and column are partly padding)."""
    bt, h, w, d, df, gd = 2, 7, 20, 16, 8, 4
    C = d + df
    nwin, ws = 4, 8
    nl = nwin * ws * ws
    gh, gw = -(-h // gd), -(-w // gd)
    G = gh * gw
    R = nl + G + 6
    x = _randn(bt * h * w, d, seed=18, shift=0.5)
    fp = _randn(bt * h * w, df, seed=19, scale=2.0)
    wm = torch.full((bt, nwin, ws, ws), -1, dtype=torch.int32)
    for f in range(bt):
        for wi in range(3):
            for py in range(ws):
                for px in range(ws):
                    y, xx = py, wi * ws + px
                    if y < h and xx < w:
                        wm[f, wi, py, px] = f * h * w + y * w + xx
    wm = wm.reshape(-1)
    gk_w, gk_b = _randn(gd * gd, C, seed=20, scale=0.3), _randn(C, seed=21)
    gv_w, gv_b = _randn(gd * gd, d, seed=22, scale=0.3), _randn(d, seed=23)
    qkn, vn = _buf((bt * R, C), fmt), _buf((bt * R, d), fmt)
    b_qkn, b_vn = qkn.clone(), vn.clone()
    emu = _run(lambda: lib.swin_prep(x, fp, bt, h, w, wm, nl, R, gd, gh, gw, gk_w, gk_b, gv_w, gv_b, qkn, vn, eps=1e-5))
    eps = torch.tensor(1e-5, dtype=torch.float32).item()
    xf = torch.cat([x, fp], 1).double()

    def rows(t, wt, bias, c):
        idx = wm.long()
        win = F.layer_norm(t[idx.clamp_min(0)], (c,), eps=eps)
        win[idx < 0] = 0.0
        img = F.pad(t.view(bt, h, w, c).permute(0, 3, 1, 2), (0, gw * gd - w, 0, gh * gd - h))
        pooled = F.conv2d(img, wt.double().t().reshape(c, 1, gd, gd), bias.double(), stride=gd, groups=c)
        pooled = F.layer_norm(pooled.permute(0, 2, 3, 1).reshape(bt, G, c), (c,), eps=eps)
        ref = torch.full((bt, R, c), float("nan"), dtype=torch.float64)
        ref[:, :nl] = win.view(bt, nl, c)
        ref[:, nl:nl + G] = pooled
        return ref.view(bt * R, c)

    _check(emu, qkn, b_qkn, rows(xf, gk_w, gk_b, C), "swin_prep qkn")
    _check(emu, vn, b_vn, rows(x.double(), gv_w, gv_b, d), "swin_prep vn")
    return emu.forms


# -------------------------------------------------------------------------------------------------------- conv_tail
@case(("split", True), ("f16", True), ("split", False), ("f16", False), ids=["split", "f16", "split-nhwc", "f16-nhwc"])
def _conv_tail(fmt, nchw):
    """FGT's decoder tail (64 -> 3, tanh, NCHW output) and RAFT's flow head tail (256 -> 2, no activation, NHWC)."""
    n, H, W = 2, 9, 21
    cin, cout, act = (64, 3, lib.ACT_TANH) if nchw else (256, 2, lib.ACT_NONE)
    x, xv = _act16(_randn(n, H, W, cin, seed=24), fmt)
    w = _randn(cout, cin, 3, 3, seed=25, scale=0.1)
    wp = lib.pack_taps_as_n(w).view(32, cin)
    wt, wv = _act16(wp, fmt)
    bias = _randn(cout, seed=26)
    out = _buf((n, cout, H, W) if nchw else (n, H, W, cout), "f32")
    emu = _run(lambda: lib.conv_tail(x, n, H, W, cin, wt, cout, bias, act, out, nchw=nchw))
    wref = wv[:9 * cout].view(3, 3, cout, cin).permute(2, 3, 0, 1)
    ref = F.conv2d(xv.permute(0, 3, 1, 2), wref, bias.double(), padding=1)
    ref = torch.tanh(ref) if nchw else ref.permute(0, 2, 3, 1)
    _check(emu, out, _buf(out.shape, "f32"), ref, "conv_tail")
    return emu.forms


# ------------------------------------------------------------------------------------------------------ upsample2x
@case(())
def _upsample2x():
    n, H, W, C = 2, 5, 7, 16
    x = lib.to_split(_randn(n, H, W, C, seed=29))
    out = _buf((n, 2 * H, 2 * W, C), "split")
    emu = _run(lambda: lib.upsample2x(x, n, H, W, C, out))
    ref = F.interpolate(x.double().view(2 * n, H, W, C).permute(0, 3, 1, 2), scale_factor=2, mode="nearest")
    assert torch.equal(out.double(), ref.permute(0, 2, 3, 1).reshape(out.shape)), "upsample2x"
    assert emu.written_mask(out).all()
    return emu.forms


# ------------------------------------------------------------------------------------------ chan_stats / instnorm_act
INORM = [  # 16-bit output, fp32 output, relu, residual: the forms of the traces
    ("split", False, True, False), ("split", True, True, False), ("split", True, True, True), (None, True, False, False),
    ("f16", False, True, False), ("f16", True, False, False), ("f16", True, True, False), ("f16", True, True, True),
]


@case(*INORM, ids=["-".join(map(str, p)) for p in INORM])
def _instnorm(fmt, f32, relu, res):
    """Channels whose mean is 30 times their spread (and some at mean 0): the variance from the sums cancels."""
    n, HW, C = 2, 37, 12
    shift = torch.where(torch.arange(C) % 2 == 0, 30.0, 0.0)
    x = _randn(n, HW, C, seed=30) + shift
    r = F.relu(_randn(n, HW, C, seed=31)) if res else None
    stats = torch.full((n * C * 2,), SENTINEL, dtype=torch.float64)
    out = _buf((n, HW, C), "f32") if f32 else None
    o16 = _buf((n, HW, C), fmt) if fmt else None
    b16 = o16.clone() if fmt else None
    emu = _run(lambda: (lib.chan_stats(x, n, HW, C, stats),
                        lib.instnorm_act(x, stats, n, HW, C, relu=relu, res=r, out=out, out_split=o16)))
    xd = x.double()
    _check(emu, stats, torch.full_like(stats, SENTINEL),
           torch.stack([xd.sum(1), (xd * xd).sum(1)], -1).reshape(-1), "chan_stats")
    eps = torch.tensor(1e-5, dtype=torch.float32).item()
    y = F.instance_norm(xd.permute(0, 2, 1), eps=eps).permute(0, 2, 1)
    if relu:
        y = F.relu(y)
    if res:
        if fmt == "f16":
            y = y.half().double()
        y = F.relu(y + r.double())
    if fmt == "f16":
        y = y.half().double()
    if out is not None:
        _check(emu, out, _buf(out.shape, "f32"), y, "instnorm_act fp32")
    if o16 is not None:
        _check(emu, o16, b16, y, "instnorm_act 16-bit")
    return emu.forms


@case(())
def _avgpool2():
    rows, h, w = 6, 15, 27                           # odd sizes: the last row and column are dropped
    x = _randn(rows, h, w, seed=32)
    out = _buf((rows, h // 2, w // 2), "f32")
    emu = _run(lambda: lib.avgpool2(x, rows, h, w, out))
    _check(emu, out, _buf(out.shape, "f32"), F.avg_pool2d(x.double()[:, None], 2, stride=2)[:, 0], "avgpool2")
    return emu.forms


# ------------------------------------------------------------------------------------------------------- corr_lookup
def _pyramid(h, w, seed):
    lv = [_randn(h * w, h, w, seed=seed)]
    for _ in range(3):
        lv.append(F.avg_pool2d(lv[-1][:, None], 2, stride=2)[:, 0].contiguous())
    return lv


def _edge_coords(h, w, seed):
    """Lookup centres at the edges: on integers, at w - 1 / h - 1, one pixel outside, half a pixel outside, far
    outside (beyond the +-1e6 clamp) and random."""
    g = _gen(seed)
    n = h * w
    xs = torch.rand(n, generator=g) * (w + 8) - 4
    ys = torch.rand(n, generator=g) * (h + 8) - 4
    special = [(0.0, 0.0), (w - 1.0, h - 1.0), (-1.0, -1.0), (float(w), float(h)), (w - 0.5, -0.5), (3.0, h - 1.0),
               (w - 1.0, 2.0), (-0.5, h - 0.5), (1e7, 2.0), (-1e7, -3e7), (2.5e6, 1.0), (5.0, -2e6), (8.0, 4.0)]
    for i, (a, b) in enumerate(special):
        xs[i * 7], ys[i * 7] = a, b
    ints = torch.arange(n) % 5 == 1
    xs[ints], ys[ints] = xs[ints].round(), ys[ints].round()
    return torch.stack([xs, ys], 1).contiguous()


@case(("split", 4, 384), ("f16", 4, 384), ("split", 3, 200), ids=["split", "f16", "split-r3-200"])
def _corr_lookup(fmt, r, pitch):
    """Radius 4 into the basic model's 384-wide rows, radius 3 into the small model's 200-wide rows."""
    h, w = 16, 24                                    # coarsest level 2 x 3
    pyr = _pyramid(h, w, 33)
    co = _edge_coords(h, w, 34)
    out = _buf((h * w, pitch), fmt)
    before = out.clone()
    emu = _run(lambda: lib.corr_lookup(pyr, co, h * w, r, out))
    nv = 4 * (2 * r + 1) ** 2
    ref = RO.corr_lookup([t[:, None].double() for t in pyr], co.double().t().reshape(1, 2, h, w), r)
    full = torch.full((h * w, pitch), float("nan"), dtype=torch.float64)
    full[:, :nv] = ref[0].reshape(nv, h * w).t()
    _check(emu, out, before, full, "corr_lookup", ref_f32=True)
    return emu.forms


# -------------------------------------------------------------------------------------------------- raft_flow_update
FLOW_UPDATE = [("split", False, False), ("split", True, False), ("f16", False, False), ("f16", True, True),
               ("split", True, True), ("f16", True, False)]


@case(*FLOW_UPDATE, ids=["-".join(map(str, p)) for p in FLOW_UPDATE])
def _raft_flow_update(fmt, delta, delta_f16):
    """Exactly defined: fp32 coords + delta (fp16-rounded first when delta_f16), fp32 flow, its 16-bit copy in channels
    254 and 255 of a 256-wide GRU input whose other channels are untouched."""
    n, h, w = 2, 5, 9
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    grid = torch.stack([xs, ys], -1).float().reshape(1, h * w, 2)
    coords = (grid + _randn(n, h * w, 2, seed=35, scale=3.0)).reshape(-1, 2).contiguous()
    dl = _randn(n * h * w, 2, seed=36, scale=2.0) if delta else None
    c0 = coords.clone()
    flow = _buf((n, 2, h, w), "f32")
    xb = _buf((n * h * w, 256), fmt)
    before = xb.clone()
    emu = _run(lambda: lib.raft_flow_update(coords, dl, h, w, flow, xb, 254, n=n, delta_f16=delta_f16))
    c1 = c0 + (dl.half().float() if delta_f16 else dl) if delta else c0
    assert torch.equal(coords, c1), "coords"
    fl = (c1.view(n, h * w, 2) - grid).view(n, h, w, 2)
    _check(emu, flow, _buf(flow.shape, "f32"), fl.permute(0, 3, 1, 2).double(), "flow_nchw")
    ref = torch.full((n * h * w, 256), float("nan"), dtype=torch.float64)
    ref[:, 254:] = fl.reshape(-1, 2).double()
    _check(emu, xb, before, ref, "GRU input")
    return emu.forms


# ---------------------------------------------------------------------------------------------------- convex_upsample
@case(())
def _convex_upsample():
    n, h, w = 2, 5, 7
    g = _gen(37)
    mask = (torch.randint(0, 2, (n * h * w, 576), generator=g) * 120 - 60).float()   # logits of +-60
    mask[::3] = _randn(mask[::3].shape[0], 576, seed=38, scale=20.0)
    flow = _randn(n, 2, h, w, seed=39, scale=4.0)
    out = _buf((n, 2, 8 * h, 8 * w), "f32")
    emu = _run(lambda: lib.convex_upsample(mask, flow, h, w, out, n=n))
    ref = RO.upsample_flow(flow.double(), mask.double().view(n, h, w, 576).permute(0, 3, 1, 2))
    _check(emu, out, _buf(out.shape, "f32"), ref, "convex_upsample")
    return emu.forms


# ------------------------------------------------------------------------------------------------------ f16_to_split
@case(())
def _f16_to_split():
    """Every finite fp16 bit pattern: hi + lo is the fp16 value exactly, hi its bf16 rounding."""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    src = bits.view(torch.float16)
    fin = torch.isfinite(src)
    out = _buf((65536,), "split")
    emu = _run(lambda: lib.f16_to_split(src, out))
    assert torch.equal(out[0, fin].double() + out[1, fin].double(), src[fin].double()), "hi + lo != value"
    assert torch.equal(out[0, fin], src[fin].float().to(torch.bfloat16)), "hi"
    assert torch.equal(emu.stored(out)[fin], src[fin].double())
    return emu.forms


# ---------------------------------------------------------------------------------------------------------- upflow8
@case(())
def _upflow8():
    """1-pixel sides included: align_corners maps every output of such a side to its one input."""
    forms = set()
    for h, w in ((3, 5), (1, 4), (4, 1), (1, 1)):
        flow = torch.randn(2, 2, h, w, generator=_gen(h * 10 + w))
        out = _buf((2, 2, 8 * h, 8 * w), "f32")
        emu = _run(lambda: lib.upflow8(flow, h, w, out, n=2))
        ref = 8 * F.interpolate(flow.double(), size=(8 * h, 8 * w), mode="bilinear", align_corners=True)
        assert (out.double() - ref).abs().max() <= 1e-6 * (1 + ref.abs().max()), (h, w)
        forms |= emu.forms
    return forms


# --------------------------------------------------------------------------------------------------------- the tests
@pytest.mark.parametrize("name", sorted(CASES))
def test_interpreter_matches_reference(name):
    _cached(name)


@functools.lru_cache(maxsize=None)
def _cached(name):
    return CASES[name]()


def _trace_forms():
    with gzip.open(GOLDEN, "rt") as f:
        g = json.load(f)
    out = {}
    for case_name, calls in g.items():
        for name, args in calls:
            if name != "fgt_gemm_tc":
                out.setdefault((name, form(name, dict(zip(lib.PROTOS[name].names, args)))), case_name)
    return out


def test_rownorm_gather_all_dropped():
    """A gather that drops every row writes zero rows only (the header's F.pad rows)."""
    a = _randn(4, 8, seed=46)
    out = _buf((6, 8), "split")
    before = out.clone()
    g = torch.full((5,), -1, dtype=torch.int32)
    emu = _run(lambda: lib.rownorm(a, None, out, gather=g, rows_per_batch=5, total_rows=5, dst_batch_rows=5))
    ref = torch.full((6, 8), float("nan"), dtype=torch.float64)
    ref[:5] = 0.0
    _check(emu, out, before, ref, "rownorm, every row dropped")


def test_every_trace_form_has_a_case():
    """Every entry of the traces has an interpreter and every (entry, form) of the traces has a case above. The GEMM
    engine's layer forms are covered by tests/test_gemm_layers.py."""
    traced = _trace_forms()
    assert {n for n, _ in traced} <= set(ENTRIES)
    covered = set()
    for name in CASES:
        covered |= _cached(name)
    missing = {k: v for k, v in traced.items() if k not in covered}
    assert not missing, f"trace forms without a case: {missing}"


# ------------------------------------------------------------------------------------------------- whole forwards
def _close(got, ref, what, tol=FWD_TOL):
    got, ref = torch.as_tensor(got).double(), torch.as_tensor(ref).double()
    assert torch.isfinite(got).all(), f"{what}: non-finite"
    r, m = rel_l2(got, ref), max_over_max(got, ref)
    assert r <= tol and m <= tol, f"{what}: rel_l2={r:.3e} max/max={m:.3e} (tol {tol:g})"


def test_fgt_forward_in_float64():
    from fgt_b200.fgt_model import Model
    from oracle import fgt_oracle as O
    g = load_golden("fgt_small_default")
    meta = g["meta"]
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = tuple(meta["res"])
    sd = synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=meta["seed"], regime=meta["regime"])
    m = Model(cfg)
    m.load_state_dict(sd)
    fr, fl, mk = synth.fgt_inputs(seed=meta["seed"] + 2, t=meta["t"], H=meta["H"], W=meta["W"])
    with torch.no_grad(), emulating_all():
        out = m.net._forward_impl(fr, fl, mk)
    _close(out.reshape(g["out"].shape), torch.from_numpy(g["out"]), "FGT vs reference golden")
    with torch.no_grad():
        ref = O.fgt_forward(O.strip_net(sd), fr, fl, mk)
    _close(out.reshape(ref.shape), ref, "FGT vs oracle")


def test_lafc_forward_in_float64():
    from fgt_b200.lafc_model import Model
    from oracle import lafc_oracle as LO
    g = load_golden("lafc_small_scaled")
    meta = g["meta"]
    sd = synth.make_state_dict(synth.lafc_param_shapes(), seed=meta["seed"], regime=meta["regime"])
    fl, mk = synth.lafc_inputs(seed=meta["seed"] + 1, H=meta["H"], W=meta["W"])
    m = Model(synth.CFG_LAFC)
    m.load_state_dict(sd)
    with torch.no_grad(), emulating_all():
        flow, edge = m.net._forward_impl(fl, mk)
    _close(flow, torch.from_numpy(g["flow"]), "LAFC flow vs reference golden")
    _close(edge, torch.from_numpy(g["edge"]), "LAFC edge vs reference golden")
    with torch.no_grad():
        rf, re_ = LO.lafc_forward({k[4:]: v for k, v in sd.items()}, fl, mk)
    _close(flow, rf, "LAFC flow vs oracle")
    _close(edge, re_, "LAFC edge vs oracle")


def _raft_model(seed=3):
    from fgt_b200.raft_model import RAFT
    m = RAFT(argparse.Namespace(small=False, mixed_precision=False, alternate_corr=False))
    sd = synth.raft_state_dict(seed=seed)
    m.load_state_dict(sd)
    return m, sd


def test_raft_forward_in_float64():
    """128 x 160: the coarsest correlation level is 2 x 2 (at 64 x 96 it is 1 x 1, see the next test)."""
    m, sd = _raft_model()
    im1, im2 = synth.raft_inputs(seed=4, H=128, W=160)
    with torch.no_grad(), emulating_all():
        lo, up = m._forward_impl(im1, im2, 3, None, True, False)
    with torch.no_grad():
        olo, oup = RO.raft_forward(sd, im1, im2, iters=3)
    _close(lo, olo, "RAFT low vs oracle")
    _close(up, oup, "RAFT up vs oracle")


def test_one_pixel_pyramid_level_diverges_from_reference():
    """At 64 x 96 the correlation pyramid is 8x12, 4x6, 2x3, 1x1. The reference sampler divides by W - 1 = 0 and
    H - 1 = 0 at the 1 x 1 level, so all its level-3 samples are NaN (and so is its whole flow); the interpreter, like
    the kernel, samples that level bilinearly with zero padding and is finite. Deliberate: the 1 x 1 level then holds
    the mean correlation, which is what the reference computes for every other size."""
    h, w = 8, 12
    pyr = _pyramid(h, w, 40)
    assert tuple(pyr[3].shape[1:]) == (1, 1)
    co = _edge_coords(h, w, 41)
    out = _buf((h * w, 384), "split")
    emu = _run(lambda: lib.corr_lookup(pyr, co, h * w, 4, out))
    ref = RO.corr_lookup([t[:, None].double() for t in pyr], co.double().t().reshape(1, 2, h, w))[0]
    ref = ref.reshape(324, h * w).t()
    got = emu.stored(out)[:, :324]
    assert torch.isnan(ref[:, 243:]).all(), "the reference sampler is finite on the 1 x 1 level"
    assert torch.isfinite(got).all()
    assert ((got[:, :243] - ref[:, :243]).abs() - 2.0 ** -24 * ref[:, :243].abs()).max() <= EXACT * ref[:, :243].abs().max()
    # the 1 x 1 level: the level's one value at the (81) window points whose bilinear footprint covers pixel (0, 0)
    c = (co.double() / 8.0).clamp(-1e6, 1e6)
    d = torch.arange(-4, 5, dtype=torch.float64)
    wx = (1 - (c[:, 0:1] + d).abs()).clamp_min(0)     # hat weight of pixel 0 along x, window index a
    wy = (1 - (c[:, 1:2] + d).abs()).clamp_min(0)
    lvl = pyr[3].double().reshape(-1, 1, 1)
    assert (got[:, 243:].view(-1, 9, 9) - wx[:, :, None] * wy[:, None, :] * lvl).abs().max() <= EXACT
