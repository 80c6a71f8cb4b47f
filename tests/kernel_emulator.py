"""Float64 interpreters of the C-ABI entries the three networks launch besides the GEMM engine, for CPU tensors.

`emulating_all()` installs a `KernelEmulator` as the library `lib.load()` returns, the way tests/gemm_emulator.py
installs its `fgt_gemm_tc` interpreter (which this class extends), so the production launchers fill their arguments as
they do on the GPU and every launch of a forward is executed here instead: the 17 entries of `ENTRIES` and
`fgt_gemm_tc`. Any other entry is refused. `gemm_emulator.emulating()` stays strict (GEMM only).

Semantics are restated from include/fgt_b200.h and from the reference operations the header names (through oracle/),
not from the kernels' code paths:
- fgt_im2col_nchw: row (n, oy, ox), channel (ky*k + kx)*cin + c = v*scale + shift of input (oy*stride + ky - pad,
  ox*stride + kx - pad), zero outside (replicate = 0) or clamped to the edge (replicate = 1); channels up to cpad are 0.
- fgt_rownorm: LayerNorm (biased variance) of [a ; b] row gather[d] (or d) into row (d / rpb) * dst_batch_rows +
  dst_row0 + d % rpb of a (ca + cb)-wide buffer; gather[d] < 0 writes a zero row; optional affine.
- fgt_attention: softmax(scale * Q K^T) V per batch and head; dense: keys [0, Lk); windowed: query window r / 64 sees
  key rows [64 (r / 64), + 64) and [glob_start, + glob_count); output rows through out_rowmap (< 0 not written).
- fgt_fold / fgt_fold_unfold: nn.Fold of position-major patches (sum of the entries covering a pixel, divided by their
  count when normalised, + add); fold_unfold writes back to every patch entry the (ReLU'd) mean of its pixel, zero for
  entries in the padding ring (nn.Unfold).
- fgt_dwconv3x3_res: x + depthwise 3x3 (zero padding 1) + bias. fgt_upsample2x: nearest x2 copy of both bf16 planes.
- fgt_swin_prep: window rows through win_map (< 0: zero rows) and pooled rows (depthwise gd x gd / stride gd + bias over
  the zero-padded grid, weights tap-major), LayerNorm of [x ; f'] into qkn and of x into vn; rows [nl + G, R) of each
  frame are not written.
- fgt_conv_tail: act(bias + 3x3 convolution with zero padding) at arbitrary output strides.
- fgt_chan_stats: per (image, channel) sum and sum of squares. fgt_instnorm_act: (x - mean) / sqrt(var + eps) with the
  biased variance from those sums, ReLU, residual relu(y + res); an fp16 output rounds y before the residual add and
  again after it, and the fp32 copy holds the fp16 value.
- fgt_avgpool2: 2x2 mean (floor sizes). fgt_corr_lookup: bilinear samples (align_corners pixel coordinates, zero
  padding) of level l at coords / 2^l (clamped to +-1e6) + (a - r, b - r), channel l (2r+1)^2 + a (2r+1) + b.
- fgt_raft_flow_update: coords += delta (delta rounded to fp16 first when delta_f16), stored fp32; flow = coords - grid
  (fp32) into NCHW and into channels x_chan, x_chan + 1 of the GRU input.
- fgt_convex_upsample: RAFT.upsample_flow. fgt_f16_to_split: hi = bf16(v), lo = bf16(v - hi).
- fgt_upflow8: 8 * bilinear x8 with align_corners=True, source index scale * dst with scale = (in - 1) / (out - 1)
  (0 for a 1-pixel side), as ATen's upsample_bilinear2d.
Arithmetic is float64 on the operands as stored (hi + lo for split-bf16, the fp16 value for fp16); each output is
stored once in its format: fp32 rounded once, split-bf16 as `lib.to_split`, fp16 rounded to nearest. Scalar float
arguments are taken at the fp32 value the C ABI receives.

Every store is recorded in `emu.records` as (kind, flat view, element indices, plane, float64 values before the store
rounding): kind "f32", "f64", "f16", "split" (hi at idx, lo at idx + plane), "raw" (a bit copy) or "addr" (addressed,
value not computed: attention rows skipped under `attn_budget`). `written_mask(t)` gives the elements of a buffer the
stores addressed, `written_bytes` the bytes of a storage, `stored(t)` the float64 values. `emu.forms` collects
(entry, form) of every call, `form()` being the discrete options of one call.
"""
import contextlib
import ctypes

import torch
import torch.nn.functional as F

from fgt_b200 import lib
from tests.gemm_emulator import GemmEmulator, _act, _GemmEntry, _r16, _Refused
from tests.test_launch_trace import recording

ENTRIES = ("fgt_im2col_nchw", "fgt_rownorm", "fgt_attention", "fgt_fold_unfold", "fgt_fold", "fgt_dwconv3x3_res",
           "fgt_swin_prep", "fgt_conv_tail", "fgt_upsample2x", "fgt_chan_stats", "fgt_instnorm_act", "fgt_avgpool2",
           "fgt_corr_lookup", "fgt_raft_flow_update", "fgt_convex_upsample", "fgt_f16_to_split", "fgt_upflow8")


def _k16(p, plane):
    """Output format of a 16-bit destination: None (absent), "f16" (plane 0) or "split"."""
    return None if p is None else ("f16" if plane == 0 else "split")


def _on(p):
    return p is not None


def form(name, a):
    """The discrete options of one call of entry `name`, args `a` (a dict by parameter name; a descriptor as a dict).
    Works on live arguments and on the launch-trace golden's JSON arguments alike (pointers only tested for None)."""
    if name == "fgt_im2col_nchw":
        return (_k16(a["out_hi"], a["out_plane"]), _on(a["src1"]), bool(a["replicate"]), a["k"], a["stride"],
                (a["scale"], a["shift"]) != (1.0, 0.0))
    if name == "fgt_rownorm":
        return (_k16(a["out_hi"], a["out_plane"]), _on(a["gather"]), _on(a["gamma"]), _on(a["b"]),
                a["dst_row0"] != 0 or a["dst_batch_rows"] != a["rows_per_batch"])
    if name == "fgt_attention":
        d = a["desc"]
        return (bool(d["f16"]), d["mode"], _on(d["out_rowmap"]), d["mode"] == 0 and d["Lq"] != d["Lk"])
    if name == "fgt_fold_unfold":
        return (_k16(a["out_hi"], a["out_plane"]), bool(a["relu"]))
    if name == "fgt_fold":
        return (_k16(a["out_hi"], a["out_plane"]), _on(a["out"]), bool(a["normalize"]), _on(a["add"]))
    if name == "fgt_dwconv3x3_res":
        return (_k16(a["out_hi"], a["out_plane"]),)
    if name == "fgt_swin_prep":
        return (_k16(a["qkn_hi"], a["qkn_plane"]),)
    if name == "fgt_conv_tail":
        return (a["x_plane"] == 0, a["act"], a["os_x"] == 1)
    if name == "fgt_instnorm_act":
        return (_k16(a["out_hi"], a["out_plane"]), _on(a["out"]), bool(a["relu"]), _on(a["res"]))
    if name == "fgt_corr_lookup":
        return (_k16(a["out_hi"], a["out_plane"]), a["levels"], a["radius"])
    if name == "fgt_raft_flow_update":
        return (_on(a["delta"]), bool(a["delta_f16"]), _k16(a["x_hi"], a["x_plane"]))
    assert name in ENTRIES, name
    return ()


def _raw(v, t):
    """Plain Python value of ctypes argument v declared as t (pointers -> int or None, c_float -> its fp32 value)."""
    if isinstance(v, ctypes.c_void_p):
        return v.value
    if isinstance(v, ctypes.Array):
        return [_raw(x, None) for x in v]
    if type(v).__name__ == "CArgObject":
        return struct_dict(v._obj)
    if t is ctypes.c_float:
        return ctypes.c_float(v).value
    return v


def struct_dict(s):
    """A descriptor struct as {field: plain value} (the launch-trace golden's shape, with raw pointers)."""
    out = {}
    for f, _ in s._fields_:
        v = getattr(s, f)
        out[f] = [struct_dict(x) for x in v] if isinstance(v, ctypes.Array) else v
    return out


class _KernelEntry:
    def __init__(self, emu, name):
        self.emu, self.name, self.argtypes, self.restype = emu, name, None, None

    def __call__(self, *args):
        assert self.argtypes is not None and len(args) == len(self.argtypes), self.name
        a = {k: _raw(v, t) for k, v, t in zip(lib.PROTOS[self.name].names, args, self.argtypes)}
        self.emu.forms.add((self.name, form(self.name, a)))
        getattr(self.emu, "_" + self.name[4:])(a)
        return 0


def _ln(x, eps):
    m = x.mean(-1, keepdim=True)
    v = ((x - m) ** 2).mean(-1, keepdim=True)
    return (x - m) / torch.sqrt(v + eps)


class KernelEmulator(GemmEmulator):
    """Stands in for the ctypes library: the entries of ENTRIES and fgt_gemm_tc run in float64 on the CPU."""

    def __init__(self):
        super().__init__()
        self.records = []
        self.forms = set()
        self.attn_budget = None

    def __getattr__(self, name):
        if not name.startswith("fgt_"):
            raise AttributeError(name)
        if name == "fgt_gemm_tc":
            e = _GemmEntry(self)
        elif name in ENTRIES:
            e = _KernelEntry(self, name)
        else:
            e = _Refused(name)
        setattr(self, name, e)
        return e

    # ------------------------------------------------------------------------------------------------ loads / stores
    def f32(self, p, n=None):
        fl = self.flat(p, torch.float32)
        return (fl if n is None else fl[:n]).double()

    def i32(self, p, n):
        return self.flat(p, torch.int32)[:n].long()

    def v16(self, p, plane, shape, strides, f16):
        return self._plane_pair(p, plane, shape, strides, f16)

    def _rec(self, kind, fl, idx, plane=None, v=None):
        self.records.append((kind, fl, idx, plane, v))
        self.written.append((fl, idx))
        if kind == "split":
            self.written.append((fl, idx + plane))

    def st32(self, p, idx, v):
        fl = self.flat(p, torch.float32)
        idx = idx.reshape(-1)
        fl[idx] = v.reshape(-1).float()
        self._rec("f32", fl, idx, v=v.reshape(-1))

    def st16(self, p, plane, idx, v):
        idx, v = idx.reshape(-1), v.reshape(-1)
        if plane == 0:
            fl = self.flat(p, torch.float16)
            fl[idx] = v.half()
            self._rec("f16", fl, idx, v=v)
        else:
            sp = lib.to_split(v.float())
            fl = self.flat(p, torch.bfloat16)
            fl[idx] = sp[0]
            fl[idx + plane] = sp[1]
            self._rec("split", fl, idx, plane, v)

    def _store(self, d, v32, o32, v16, o16):   # fgt_gemm_tc's stores, recorded like the others
        if d.out_f32 and v32 is not None:
            self.st32(d.out_f32, o32, v32)
        if d.out_hi and v16 is not None:
            self.st16(d.out_hi, 0 if d.out_half else d.out_plane, o16, v16)

    def written_bytes(self, t):
        """Boolean mask over the bytes of the uint8 tensor `t` (one whole storage) that the recorded stores cover."""
        mask = torch.zeros(t.numel(), dtype=torch.bool)
        base = t.untyped_storage().data_ptr()
        for kind, fl, idx, plane, _ in self.records:
            if fl.untyped_storage().data_ptr() != base:
                continue
            es = fl.element_size()
            for i in ((idx,) if not plane else (idx, idx + plane)):
                b = (fl.storage_offset() + i)[:, None] * es + torch.arange(es)[None, :]
                mask[b.reshape(-1)] = True
        return mask

    def stored(self, t):
        """float64 values (before the store rounding) the recorded stores gave the elements of contiguous tensor `t`
        (a split-bf16 tensor [2, ...] counts as its logical shape), NaN where nothing was stored."""
        split = t.dtype == torch.bfloat16
        hi = t[0] if split else t
        out = torch.full((hi.numel(),), float("nan"), dtype=torch.float64)
        base = t.untyped_storage().data_ptr()
        for kind, fl, idx, plane, v in self.records:
            if fl.untyped_storage().data_ptr() != base or fl.dtype != t.dtype or v is None:
                continue
            pos = fl.storage_offset() + idx - hi.storage_offset()
            ok = (pos >= 0) & (pos < hi.numel())
            out[pos[ok]] = v.reshape(-1)[ok]
        return out.view(hi.shape)

    # ------------------------------------------------------------------------------------------------------ entries
    def _im2col_nchw(self, a):
        n, H, W, k, s, pad, OH, OW, cpad = (a[x] for x in "n H W k stride pad OH OW cpad".split())
        cin = a["c0"] + a["c1"]
        src = self.f32(a["src0"], n * a["c0"] * H * W).view(n, a["c0"], H, W)
        if a["c1"]:
            src = torch.cat([src, self.f32(a["src1"], n * a["c1"] * H * W).view(n, a["c1"], H, W)], 1)
        t = torch.arange(k)
        y = torch.arange(OH)[:, None] * s + t[None, :] - pad      # [OH, ky]
        x = torch.arange(OW)[:, None] * s + t[None, :] - pad      # [OW, kx]
        oky = torch.ones_like(y, dtype=torch.bool) if a["replicate"] else (y >= 0) & (y < H)
        okx = torch.ones_like(x, dtype=torch.bool) if a["replicate"] else (x >= 0) & (x < W)
        v = src[:, :, y.clamp(0, H - 1)[:, :, None, None], x.clamp(0, W - 1)[None, None, :, :]]  # [n,cin,OH,ky,OW,kx]
        v = torch.where(oky[:, :, None, None] & okx[None, None, :, :], v * a["scale"] + a["shift"], 0.0)
        out = torch.zeros(n, OH, OW, cpad, dtype=torch.float64)
        out[..., :k * k * cin] = v.permute(0, 2, 4, 3, 5, 1).reshape(n, OH, OW, k * k * cin)
        self.st16(a["out_hi"], a["out_plane"], torch.arange(out.numel()), out)

    def _rownorm(self, a):
        ca, cb, rpb, total = a["ca"], a["cb"], a["rows_per_batch"], a["total_rows"]
        C = ca + cb
        d = torch.arange(total)
        drow = (d // rpb) * a["dst_batch_rows"] + a["dst_row0"] + d % rpb
        src = self.i32(a["gather"], total) if a["gather"] else d
        nsrc = max(int(src.max()), 0) + 1
        fa = self.flat(a["a"], torch.float32)
        X = fa.as_strided((nsrc, ca), (a["lda"], 1), fa.storage_offset()).double()
        if cb:
            fb = self.flat(a["b"], torch.float32)
            X = torch.cat([X, fb.as_strided((nsrc, cb), (a["ldb"], 1), fb.storage_offset()).double()], 1)
        y = _ln(X[src.clamp_min(0)], a["eps"])
        if a["gamma"]:
            y = y * self.f32(a["gamma"], C) + self.f32(a["beta"], C)
        y[src < 0] = 0.0
        self.st16(a["out_hi"], a["out_plane"], drow[:, None] * C + torch.arange(C)[None, :], y)

    def _attention(self, a):
        """With `attn_budget` set, only every s-th 64-row query window is computed (s chosen so that the float64 work
        stays within the budget, in multiply-adds); the rows of the others are recorded as addressed ("addr")."""
        d = a["desc"]
        f16, B, Hh, Lq = bool(d["f16"]), d["batches"], d["heads"], d["Lq"]
        assert d["head_dim"] == 128
        C = Hh * 128

        def rows(p, plane, bstride, ld, n):   # [B, heads, n, 128]
            v = self.v16(p, 0 if f16 else plane, (B, n, C), (bstride, ld, 1), f16)
            return v.view(B, n, Hh, 128).permute(0, 2, 1, 3)

        nk = d["Lk_rows"]
        Q = rows(d["q_hi"], d["q_plane"], d["q_batch_stride"], d["q_ld"], Lq)
        K = rows(d["k_hi"], d["k_plane"], d["k_batch_stride"], d["k_ld"], nk)
        V = rows(d["v_hi"], d["v_plane"], d["v_batch_stride"], d["v_ld"], nk)
        sc = ctypes.c_float(d["scale"]).value
        nw = -(-Lq // 64)
        keys_per_row = d["Lk"] if d["mode"] == 0 else 64 + d["glob_count"]
        step = 1
        if self.attn_budget:
            step = max(1, -(-2 * B * Lq * keys_per_row * C // int(self.attn_budget)))
        win = torch.arange(0, nw, step)
        qsel = (win[:, None] * 64 + torch.arange(64)[None, :]).reshape(-1)
        qsel = qsel[qsel < Lq]
        O = torch.empty(B, Hh, qsel.numel(), 128, dtype=torch.float64)
        if d["mode"] == 0:
            assert d["Lk"] <= nk
            for b in range(B):
                for h in range(Hh):
                    S = (Q[b, h, qsel] @ K[b, h, :d["Lk"]].t()) * sc
                    O[b, h] = torch.softmax(S, -1) @ V[b, h, :d["Lk"]]
        else:
            assert d["mode"] == 1 and Lq % 64 == 0
            g0, gc = d["glob_start"], d["glob_count"]
            keys = torch.cat([torch.arange(g0, g0 + gc)[None, :].expand(win.numel(), gc),
                              (win[:, None] * 64 + torch.arange(64)[None, :])], 1)   # [windows, gc + 64]
            assert int(keys.max()) < nk
            for b in range(B):
                Kw, Vw = K[b][:, keys], V[b][:, keys]                 # [heads, windows, gc + 64, 128]
                Qw = Q[b][:, qsel].reshape(Hh, win.numel(), 64, 128)
                S = (Qw @ Kw.transpose(-1, -2)) * sc
                O[b] = (torch.softmax(S, -1) @ Vw).reshape(Hh, -1, 128)
        O = O.permute(0, 2, 1, 3).reshape(-1, C)
        r = torch.arange(B * Lq)
        if d["out_rowmap"]:
            m = self.i32(d["out_rowmap"], B * Lq)
            keep, off = m >= 0, m * d["out_ld"]
        else:
            keep, off = torch.ones(B * Lq, dtype=torch.bool), (r // Lq) * d["out_batch_stride"] + (r % Lq) * d["out_ld"]
        kc, oc = keep.view(B, Lq)[:, qsel].reshape(-1), off.view(B, Lq)[:, qsel].reshape(-1)
        plane = 0 if f16 else d["out_plane"]
        cols = torch.arange(C)[None, :]
        self.st16(d["out_hi"], plane, oc[kc][:, None] + cols, O[kc])
        computed = torch.zeros(B, Lq, dtype=torch.bool)
        computed[:, qsel] = True
        rest = (off[keep & ~computed.view(-1)][:, None] + cols).reshape(-1)
        if rest.numel():
            self.records.append(("addr", self.flat(d["out_hi"], torch.int16), rest, plane, None))

    def _patches(self, a):
        """(hid [bt, L*P, C], pixel of every patch entry [L*P], inside mask [L*P]) of a fold geometry."""
        bt, th, tw, C, kh, kw, s, pad, OW = (a[x] for x in "bt th tw C kh kw stride pad OW".split())
        OH = a["OH"]
        hid = self.f32(a["hid"], bt * th * tw * kh * kw * C).view(bt, th * tw * kh * kw, C)
        y = (torch.arange(th)[:, None, None, None] * s + torch.arange(kh)[None, None, :, None] - pad)
        x = (torch.arange(tw)[None, :, None, None] * s + torch.arange(kw)[None, None, None, :] - pad)
        y, x = y.expand(th, tw, kh, kw).reshape(-1), x.expand(th, tw, kh, kw).reshape(-1)
        inside = (y >= 0) & (y < OH) & (x >= 0) & (x < OW)
        return hid, (y * OW + x), inside

    def _fold_sum(self, a):
        hid, pix, inside = self._patches(a)
        npx = a["OH"] * a["OW"]
        img = torch.zeros(a["bt"], npx, a["C"], dtype=torch.float64)
        img.index_add_(1, pix[inside], hid[:, inside])
        cnt = torch.zeros(npx, dtype=torch.float64).index_add_(0, pix[inside], torch.ones(int(inside.sum()),
                                                                                           dtype=torch.float64))
        return img, cnt, pix, inside

    def _fold(self, a):
        img, cnt, _, _ = self._fold_sum(a)
        if a["normalize"]:
            assert bool((cnt > 0).all())
            img = img / cnt[None, :, None]
        if a["add"]:
            img = img + self.f32(a["add"], img.numel()).view(img.shape)
        idx = torch.arange(img.numel())
        if a["out"]:
            self.st32(a["out"], idx, img)
        if a["out_hi"]:
            self.st16(a["out_hi"], a["out_plane"], idx, img)

    def _fold_unfold(self, a):
        img, cnt, pix, inside = self._fold_sum(a)
        img = img / cnt.clamp_min(1)[None, :, None]
        if a["relu"]:
            img = img.clamp_min(0.0)
        out = torch.zeros(a["bt"], pix.numel(), a["C"], dtype=torch.float64)
        out[:, inside] = img[:, pix[inside]]
        self.st16(a["out_hi"], a["out_plane"], torch.arange(out.numel()), out)

    def _dwconv3x3_res(self, a):
        bt, h, w, C = a["bt"], a["h"], a["w"], a["C"]
        x = self.f32(a["x"], bt * h * w * C).view(bt, h, w, C)
        wt = self.f32(a["weight"], C * 9).view(C, 9)
        xp = F.pad(x, (0, 0, 1, 1, 1, 1))
        v = self.f32(a["bias"], C).expand(bt, h, w, C).clone()
        for ty in range(3):
            for tx in range(3):
                v += wt[:, ty * 3 + tx] * xp[:, ty:ty + h, tx:tx + w, :]
        v = v + x
        idx = torch.arange(v.numel())
        self.st32(a["out"], idx, v)
        if a["out_hi"]:
            self.st16(a["out_hi"], a["out_plane"], idx, v)

    def _swin_prep(self, a):
        d, df, bt, h, w, nl, R, gd, gh, gw = (a[x] for x in "d df bt h w nl R gd gh gw".split())
        C, G, eps = d + df, gh * gw, a["eps"]
        x = self.f32(a["x"], bt * h * w * d).view(bt * h * w, d)
        xf = torch.cat([x, self.f32(a["fp"], bt * h * w * df).view(bt * h * w, df)], 1)
        wm = self.i32(a["win_map"], bt * nl)
        qk, vv = _ln(xf[wm.clamp_min(0)], eps), _ln(x[wm.clamp_min(0)], eps)
        qk[wm < 0], vv[wm < 0] = 0.0, 0.0
        win_rows = (torch.arange(bt * nl) // nl) * R + torch.arange(bt * nl) % nl

        def pool(t, wgt, bias, c):   # depthwise gd x gd / stride gd over the zero-padded grid, weights [gd*gd, c]
            g = torch.zeros(bt, gh * gd, gw * gd, c, dtype=torch.float64)
            hh, ww = min(h, gh * gd), min(w, gw * gd)
            g[:, :hh, :ww] = t.view(bt, h, w, c)[:, :hh, :ww]
            g = g.view(bt, gh, gd, gw, gd, c) * self.f32(wgt, gd * gd * c).view(1, 1, gd, 1, gd, c)
            return (g.sum((2, 4)) + self.f32(bias, c)).reshape(bt * G, c)

        pk, pv = _ln(pool(xf, a["gk_w"], a["gk_b"], C), eps), _ln(pool(x, a["gv_w"], a["gv_b"], d), eps)
        pool_rows = (torch.arange(bt * G) // G) * R + nl + torch.arange(bt * G) % G
        rows = torch.cat([win_rows, pool_rows])
        self.st16(a["qkn_hi"], a["qkn_plane"], rows[:, None] * C + torch.arange(C), torch.cat([qk, pk]))
        self.st16(a["vn_hi"], a["vn_plane"], rows[:, None] * d + torch.arange(d), torch.cat([vv, pv]))

    def _conv_tail(self, a):
        n, H, W, cin, cout = a["n"], a["H"], a["W"], a["cin"], a["cout"]
        f16 = a["x_plane"] == 0 and a["w_plane"] == 0
        x = self.v16(a["x_hi"], a["x_plane"], (n, H, W, cin), (H * W * cin, W * cin, cin, 1), f16)
        wt = self.v16(a["w_hi"], a["w_plane"], (9 * cout, cin), (a["k_pad"], 1), f16)
        xp = F.pad(x, (0, 0, 1, 1, 1, 1))
        v = torch.zeros(n, H, W, cout, dtype=torch.float64)
        if a["bias"]:
            v += self.f32(a["bias"], cout)
        for ty in range(3):
            for tx in range(3):
                t = ty * 3 + tx
                v += xp[:, ty:ty + H, tx:tx + W, :] @ wt[t * cout:(t + 1) * cout].t()
        v = _act(v, a["act"])
        idx = (torch.arange(n)[:, None, None, None] * a["os_n"] + torch.arange(H)[None, :, None, None] * a["os_y"]
               + torch.arange(W)[None, None, :, None] * a["os_x"] + torch.arange(cout)[None, None, None, :] * a["os_c"])
        self.st32(a["out"], idx, v)

    def _upsample2x(self, a):
        n, H, W, C = a["n"], a["H"], a["W"], a["C"]
        fi, fo = self.flat(a["in_hi"], torch.bfloat16), self.flat(a["out_hi"], torch.bfloat16)
        y, x = torch.arange(2 * H), torch.arange(2 * W)
        src = ((torch.arange(n)[:, None, None, None] * H + (y // 2)[None, :, None, None]) * W
               + (x // 2)[None, None, :, None]) * C + torch.arange(C)
        dst = torch.arange(n * 4 * H * W * C).view(src.shape)
        for ip, op in ((0, 0), (a["in_plane"], a["out_plane"])):
            fo[dst.reshape(-1) + op] = fi[src.reshape(-1) + ip]
            self._rec("raw", fo, dst.reshape(-1) + op)

    def _chan_stats(self, a):
        n, HW, C = a["n"], a["HW"], a["C"]
        x = self.f32(a["x"], n * HW * C).view(n, HW, C)
        st = torch.stack([x.sum(1), (x * x).sum(1)], -1)   # [n, C, 2]
        fl = self.flat(a["stats"], torch.float64)
        idx = torch.arange(n * C * 2)
        fl[idx] = st.reshape(-1)
        self._rec("f64", fl, idx, v=st.reshape(-1))

    def _instnorm_act(self, a):
        n, HW, C = a["n"], a["HW"], a["C"]
        st = self.flat(a["stats"], torch.float64)[:n * C * 2].view(n, 1, C, 2)
        mean = st[..., 0] / HW
        var = (st[..., 1] / HW - mean * mean).clamp_min(0.0)
        y = (self.f32(a["x"], n * HW * C).view(n, HW, C) - mean) / torch.sqrt(var + a["eps"])
        if a["relu"]:
            y = y.clamp_min(0.0)
        f16 = a["out_hi"] is not None and a["out_plane"] == 0
        if a["res"]:
            if f16:
                y = _r16(y)
            y = (y + self.f32(a["res"], n * HW * C).view(n, HW, C)).clamp_min(0.0)
        if f16:
            y = _r16(y)
        idx = torch.arange(y.numel())
        if a["out"]:
            self.st32(a["out"], idx, y)
        if a["out_hi"]:
            self.st16(a["out_hi"], a["out_plane"], idx, y)

    def _avgpool2(self, a):
        rows, h, w = a["rows"], a["h"], a["w"]
        x = self.f32(a["in"], rows * h * w).view(rows, h, w)[:, :h // 2 * 2, :w // 2 * 2]
        v = x.reshape(rows, h // 2, 2, w // 2, 2).sum((2, 4)) * 0.25
        self.st32(a["out"], torch.arange(v.numel()), v)

    def _corr_lookup(self, a):
        r, n_pix, L = a["radius"], a["n_pix"], a["levels"]
        win = 2 * r + 1
        co = self.f32(a["coords"], 2 * n_pix).view(n_pix, 2)
        dd = torch.arange(-r, r + 1, dtype=torch.float64)
        p = torch.arange(n_pix)
        out = torch.empty(n_pix, L, win, win, dtype=torch.float64)
        for l in range(L):
            hl, wl = a["level_h_host"][l], a["level_w_host"][l]
            vol = self.f32(a["level_ptrs_host"][l], n_pix * hl * wl)
            c = (co / 2.0 ** l).clamp(-1e6, 1e6)
            X = c[:, 0:1] + dd            # [p, a]: window index a offsets x
            Y = c[:, 1:2] + dd            # [p, b]: window index b offsets y
            x0, y0 = torch.floor(X), torch.floor(Y)
            fx, fy = (X - x0)[:, :, None], (Y - y0)[:, None, :]
            x0, y0 = x0.long()[:, :, None], y0.long()[:, None, :]

            def at(yy, xx):
                ok = (yy >= 0) & (yy < hl) & (xx >= 0) & (xx < wl)
                i = p[:, None, None] * hl * wl + yy.clamp(0, hl - 1) * wl + xx.clamp(0, wl - 1)
                return torch.where(ok, vol[i], 0.0)

            out[:, l] = ((1 - fx) * (1 - fy) * at(y0, x0) + fx * (1 - fy) * at(y0, x0 + 1)
                         + (1 - fx) * fy * at(y0 + 1, x0) + fx * fy * at(y0 + 1, x0 + 1))
        idx = p[:, None] * a["out_pitch"] + torch.arange(L * win * win)[None, :]
        self.st16(a["out_hi"], a["out_plane"], idx, out.reshape(n_pix, -1))

    def _raft_flow_update(self, a):
        n, h, w = a["n"], a["h"], a["w"]
        N = n * h * w
        co = self.f32(a["coords"], 2 * N).view(N, 2)
        if a["delta"]:
            dl = self.f32(a["delta"], 2 * N).view(N, 2)
            if a["delta_f16"]:
                dl = _r16(dl)
            co = (co + dl).float().double()
            self.st32(a["coords"], torch.arange(2 * N), co)
        q = torch.arange(N) % (h * w)
        img = torch.arange(N) // (h * w)
        fx, fy = (co[:, 0] - (q % w)).float().double(), (co[:, 1] - (q // w)).float().double()
        self.st32(a["flow_nchw"], torch.cat([img * 2 * h * w + q, img * 2 * h * w + h * w + q]), torch.cat([fx, fy]))
        if a["x_hi"]:
            o = torch.arange(N)[:, None] * a["x_pitch"] + a["x_chan"] + torch.arange(2)[None, :]
            self.st16(a["x_hi"], a["x_plane"], o, torch.stack([fx, fy], 1))

    def _convex_upsample(self, a):
        n, h, w = a["n"], a["h"], a["w"]
        m = torch.softmax(self.f32(a["mask"], n * h * w * 576).view(n, h, w, 9, 8, 8), 3)
        fp = F.pad(self.f32(a["flow_nchw"], n * 2 * h * w).view(n, 2, h, w), (1, 1, 1, 1))
        nb = torch.stack([8.0 * fp[:, :, k // 3:k // 3 + h, k % 3:k % 3 + w] for k in range(9)], -1)   # [n,2,h,w,9]
        up = torch.einsum("nyxkij,ncyxk->ncyixj", m, nb).reshape(n, 2, 8 * h, 8 * w)
        self.st32(a["out"], torch.arange(up.numel()), up)

    def _f16_to_split(self, a):
        v = self.flat(a["src"], torch.float16)[:a["n"]].double()
        self.st16(a["out_hi"], a["out_plane"], torch.arange(a["n"]), v)

    def _upflow8(self, a):
        n, h, w = a["n"], a["h"], a["w"]
        f = self.f32(a["flow_nchw"], n * 2 * h * w).view(n, 2, h, w)

        def axis(size):
            dst = torch.arange(8 * size, dtype=torch.float64)
            src = dst * ((size - 1) / (8 * size - 1))
            i0 = src.long()
            return i0, (i0 + 1).clamp(max=size - 1), src - i0

        y0, y1, ly = axis(h)
        x0, x1, lx = axis(w)
        ly, lx = ly[:, None], lx[None, :]
        top = (1 - lx) * f[:, :, y0][:, :, :, x0] + lx * f[:, :, y0][:, :, :, x1]
        bot = (1 - lx) * f[:, :, y1][:, :, :, x0] + lx * f[:, :, y1][:, :, :, x1]
        up = 8.0 * ((1 - ly) * top + ly * bot)
        self.st32(a["out"], torch.arange(up.numel()), up)


@contextlib.contextmanager
def emulating_all():
    """`with emulating_all() as emu:` runs every launch of the block (ENTRIES and fgt_gemm_tc) in float64."""
    emu = KernelEmulator()
    with recording(emu):
        yield emu
