"""Every GEMM layer form the three networks launch, run through the float64 interpreter of `fgt_gemm_tc`
(tests/gemm_emulator.py) and compared with a float64 restatement of the reference layer.

Each case packs its weights with the production `_pack` of its network (synth state dicts) and issues the same
`ops.conv` / `ops.linear` / `lib.gemm_tc` call, with the same arguments, that the forward issues
(tests/test_launch_trace.py pins the forward to those descriptors). The reference side is the layer as the reference
states it: `F.conv2d` / `F.conv3d` with the reference's `groups`, the per-group concatenation of the encoder's skip
inputs (FGT model.py:61-64), nearest x2 upsampling followed by the 3x3 conv for the decoder's deconvs, and the ConvGRU
formula of RAFT's update.py:45-60.

Bars:
- EXACT (1e-12 of the largest value) where the reference layer is fed the operands as packed (split-bf16 hi + lo, or
  fp16): this checks the host decomposition itself (grouped segments, block-diagonal enc14, 3-D and dilated taps,
  strided A operands, channel and row addressing). Observed: <= 4.4e-16. The fp16 deconv is restated with the host's
  phase kernels (fp16 taps summed, rounded once): EXACT, observed 0; against the reference's upsample + 3x3 conv with
  per-tap fp16 weights it is a sanity bound, 2.3e-4 observed, bar 1e-3.
- KTOL for the fp32 deconv, whose host sums the phase taps in fp32 before splitting them. Observed: 2.7e-6.
- The mixed GRU halves: both sides round at the same points, but a float64 value on an fp16 rounding boundary may land
  one fp16 ulp apart (the restatement's conv sums in another order) and carry into the state update: 2.6e-4 observed,
  bar 2^-10.
- Stored outputs: exactly the elements of the layer's slice are stored (the interpreter's record of its stores against
  the case's own statement of the slice), each within its format's rounding of the float64 value, and every other
  element keeps the sentinel the buffer was filled with (channel slices, RAFT's channels 254-255, the rows of a fused
  Q|K|V buffer, the upper half of RAFT's GRU input).

The same cases run on the GPU against this interpreter in tests/test_gemm_layers_gpu.py.
"""
import argparse
import functools

import pytest
import torch
import torch.nn.functional as F

from fgt_b200 import lib, synth
from tests.gemm_emulator import emulating

KTOL = 1e-4
EXACT = 1e-12
SENTINEL = -1234.5


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _act16(shape, f16, seed, scale=1.0):
    """A 16-bit activation tensor (split-bf16 [2, *shape] or fp16 [*shape]) and its float64 value."""
    x = torch.randn(*shape, generator=_gen(seed)) * scale
    t = x.half() if f16 else lib.to_split(x)
    return t, _val(t)


def _val(t):
    """float64 value of a 16-bit activation tensor (or of an fp32 one)."""
    if t.dtype == torch.bfloat16:
        return t[0].double() + t[1].double()
    return t.double()


def _wval(w, f16):
    """float64 value of a weight as the packing stores it (elementwise: fp16, or hi + lo of its split)."""
    return w.half().double() if f16 else _val(lib.to_split(w.float()))


def _sentinel(shape, dtype, dev):
    if dtype == torch.bfloat16:
        shape = (2,) + tuple(shape)
    return torch.full(shape, SENTINEL, dtype=dtype, device=dev)


def _nhwc(x):   # [n, C, H, W] -> [n, H, W, C]
    return x.permute(0, 2, 3, 1)


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _leaky(x, s=0.2):
    return torch.where(x > 0, x, s * x)


# ---------------------------------------------------------------------------------------------------------- models
@functools.lru_cache(maxsize=None)
def _fgt():
    from fgt_b200.fgt_model import Model
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    m = Model(cfg)
    m.load_state_dict(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=1))
    return m.net


@functools.lru_cache(maxsize=None)
def _lafc():
    from fgt_b200.lafc_model import Model
    m = Model(synth.CFG_LAFC)
    m.load_state_dict(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=5))
    return m.net


@functools.lru_cache(maxsize=None)
def _raft():
    from fgt_b200.raft_model import RAFT
    m = RAFT(argparse.Namespace(small=False, mixed_precision=False, alternate_corr=False))
    m.load_state_dict(synth.raft_state_dict(seed=3))
    return m


_PACKED = {}


def _packed(net, dev, half=False):
    """The production pack of `net` on `dev` (cached per device and precision)."""
    key = (id(net), str(dev), half)
    if key not in _PACKED:
        _PACKED[key] = net._pack(dev, half) if half else net._pack(dev)
    return _PACKED[key]


def _sd(net):
    return {k: v.detach().double() for k, v in net.state_dict().items() if v.dtype.is_floating_point}


# ---------------------------------------------------------------------------------------------------------- cases
# A case builder takes (dev, big) and returns a dict:
#   run():   issues the production call(s) on `dev`
#   bufs:    {name: output tensor}, pre-filled with SENTINEL (or with the contents the forward leaves there)
#   ref():   float64 reference values of each launch, [out_z, out_h, out_w, N] (the emulator's `v` layout)
#   place:   {name: (decode, fn)}: decode(buf) -> float64 logical view of the buffer, fn(ref values) -> (mask, want):
#            the elements the launches address and their reference values, in the decoded layout
#   bar:     EXACT or KTOL (emulator values against ref)
#   f16:     1-term layer
# `big` selects the production-sized geometry the GPU tests use.

def _fgt_grouped(name, segs_in, groups, seg_counts, ref_groups, mixed, dev, big):
    """enc10 / enc12 / enc14 / enc16: NHWC 3x3 convs over [x0 ; previous output] with grouped segments."""
    net, f16 = _fgt(), mixed
    P = _packed(net, dev, mixed)
    bt, H, W = (2, 60, 108) if big else (2, 10, 13)
    xs, vals = [], []
    for i, c in enumerate(segs_in):
        t, v = _act16((bt, H, W, c), f16, seed=10 + i)
        xs.append((t.to(dev), c))
        vals.append(v)
    N = P[name]["N"]
    out = _sentinel((bt, H, W, N), torch.float16 if f16 else torch.bfloat16, dev)
    bufs = dict(out=out)
    key = {"enc10": "10", "enc12": "12", "enc14": "14", "enc16": "16"}[name]
    sd = _sd(net)
    w = sd[f"frame_endoder.layers.{key}.weight"]
    b = sd[f"frame_endoder.layers.{key}.bias"]
    if mixed:
        b = b.half().double()

    def run():
        from fgt_b200.fgt_model import conv
        kw = dict(kx=3, ky=3, pad_x=1, pad_y=1)
        if name == "enc14":
            kw["alg_k"] = 9 * (32 + 48)
        conv(xs, P[name], out_split=bufs["out"], groups=groups, seg_counts=seg_counts, **kw)

    def ref():
        # model.py:61-64: per reference group, cat(x0 group slice, previous output group slice), then the conv
        G = ref_groups
        c0, c1 = segs_in[0] // G, segs_in[1] // G
        x = torch.cat([torch.cat([_nchw(vals[0])[:, g * c0:(g + 1) * c0], _nchw(vals[1])[:, g * c1:(g + 1) * c1]], 1)
                       for g in range(G)], 1) if G > 1 else torch.cat([_nchw(vals[0]), _nchw(vals[1])], 1)
        y = F.conv2d(x, _wval(w, f16), b, padding=1, groups=G)
        return [_leaky(_nhwc(y))]

    place = dict(out=(_val, lambda r: (torch.ones(bt, H, W, N, dtype=torch.bool), r[0])))
    return dict(run=run, bufs=bufs, ref=ref, place=place, bar=EXACT, f16=f16)


def case_enc10(dev, big=False, mixed=False):
    return _fgt_grouped("enc10", (256, 384), 2, [128, 192], 2, mixed, dev, big)


def case_enc12(dev, big=False, mixed=False):
    return _fgt_grouped("enc12", (256, 512), 4, [64, 128], 4, mixed, dev, big)


def case_enc14(dev, big=False, mixed=False):
    return _fgt_grouped("enc14", (256, 384), 2, [128, 192], 8, mixed, dev, big)


def case_enc16(dev, big=False, mixed=False):
    return _fgt_grouped("enc16", (256, 256), 1, [256, 256], 1, mixed, dev, big)


def case_deconv(dev, big=False, mixed=False):
    """dec1: nearest x2 + 3x3 conv as four 2x2 phase convs writing the interleaved output (out_phase)."""
    from fgt_b200.fgt_model import FGT
    net, f16 = _fgt(), mixed
    P = _packed(net, dev, mixed)
    bt, h, w, C = (2, 60, 108, 128) if big else (2, 7, 11, 128)
    x, xv = _act16((bt, h, w, C), f16, seed=20)
    x = x.to(dev)
    out = _sentinel((bt, 2 * h, 2 * w, C), torch.float16 if f16 else torch.bfloat16, dev)
    bufs = dict(out=out)
    sd = _sd(net)
    wt, b = sd["decoder.layer1.conv.featureConv.weight"], sd["decoder.layer1.conv.featureConv.bias"]
    if mixed:
        b = b.half().double()

    def run():
        FGT._deconv(x, C, P, "dec1", bufs["out"])

    def full():
        wr = wt.half().double() if mixed else wt
        up = F.interpolate(_nchw(xv), scale_factor=2, mode="nearest")
        return _leaky(_nhwc(F.conv2d(up, wr, b, padding=1)))

    def upsampled():
        y = full()
        return [y[:, py::2, px::2] for py in (0, 1) for px in (0, 1)]

    def phases():
        # the host's phase kernels: fp16 taps of the 3x3 filter summed (in float64: exact for <= 4 fp16 values) and
        # rounded to fp16 once; output (2i+py, 2j+px) reads rows i-1+py, i+py and columns j-1+px, j+px
        rows = {0: ([0], [1, 2]), 1: ([0, 1], [2])}
        wr, xp = wt.half().double(), F.pad(_nchw(xv), (1, 1, 1, 1))
        out = []
        for py in (0, 1):
            for px in (0, 1):
                w2 = torch.stack([torch.stack([wr[:, :, rows[py][a], :][:, :, :, rows[px][c]].sum((2, 3))
                                               for c in (0, 1)], -1) for a in (0, 1)], -2).half().double()
                y = F.conv2d(xp, w2, b)[:, :, py:py + h, px:px + w]
                out.append(_leaky(_nhwc(y)))
        return out

    def at(r):
        y = torch.empty(bt, 2 * h, 2 * w, C, dtype=torch.float64)
        for i, (py, px) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
            y[:, py::2, px::2] = r[i]
        return torch.ones(y.shape, dtype=torch.bool), y

    if mixed:   # EXACT against the packed phase kernels; the reference's upsample + 3x3 conv as a sanity bound
        return dict(run=run, bufs=bufs, ref=phases, place=dict(out=(_val, at)), bar=EXACT, f16=f16,
                    sanity=(upsampled, 1e-3))
    return dict(run=run, bufs=bufs, ref=upsampled, place=dict(out=(_val, at)), bar=KTOL, f16=f16)


def case_qkv_slice(dev, big=False, mixed=False):
    """SWMHSA's V projection into columns [2d, 3d) of the fused [rows, 3d] Q|K|V buffer (os_x = 3d, out_elem_offset)."""
    from fgt_b200.fgt_model import linear
    net, f16 = _fgt(), mixed
    P = _packed(net, dev, mixed)
    d = net.d
    rows = 2 * 3 * 64 + 40 if big else 136   # not a multiple of the 128-row tile
    vn, vv = _act16((rows, d), f16, seed=30)
    vn = vn.to(dev)
    qkv = _sentinel((rows, 3 * d), torch.float16 if f16 else torch.bfloat16, dev)
    bufs = dict(qkv=qkv)
    wp = P["s0.v"]

    def run():
        linear([(vn, d)], wp, rows, out_split=bufs["qkv"], os_x=3 * d, out_elem_offset=2 * d)

    def ref():
        w = wp["w"].cpu()
        wv = w.double() if f16 else w[0].double() + w[1].double()
        return [(vv @ wv.t() + wp["b"].cpu().double()).reshape(1, 1, rows, d)]

    def at(r):
        mask = torch.zeros(rows, 3 * d, dtype=torch.bool)
        mask[:, 2 * d:] = True
        want = torch.zeros(rows, 3 * d, dtype=torch.float64)
        want[:, 2 * d:] = r[0].reshape(rows, d)
        return mask, want

    return dict(run=run, bufs=bufs, ref=ref, place=dict(qkv=(_val, at)), bar=EXACT, f16=f16)


def _lafc_case(dev, big, name, key, in_c, out_c, conv_kw, ref_fn, T=3, out_z=None, aux=None, nchw=False,
               act=lib.ACT_LEAKY02, aux_mode=lib.AUX_NONE, f32_out=False, in_place=False):
    """One LAFC conv over a [T, H, W, C] split input."""
    from fgt_b200 import ops
    net = _lafc()
    P = _packed(net, dev)
    H, W = (60, 108) if big else (9, 13)
    x, xv = _act16((T, H, W, in_c), False, seed=40)
    x = x.to(dev)
    oz = T if out_z is None else out_z
    sd = _sd(net)
    w, b = sd[key + ".featureConv.weight"], sd[key + ".featureConv.bias"]
    auxv = None
    bufs = {}
    if aux is not None:
        auxv = torch.randn(oz, H, W, out_c, generator=_gen(41)) if aux == "rand" else None
    if nchw:
        bufs["out"] = torch.full((oz, out_c, H, W), SENTINEL, device=dev)
    elif in_place:   # res2: e4 (split) and e4f (fp32, also the residual) written in place
        bufs["out"] = _sentinel((oz, H, W, out_c), torch.bfloat16, dev)
        bufs["outf"] = auxv.float().to(dev)
    else:
        bufs["out"] = _sentinel((oz, H, W, out_c), torch.bfloat16, dev)
        if f32_out:
            bufs["outf"] = torch.full((oz, H, W, out_c), SENTINEL, device=dev)
    aux_t = auxv.float().to(dev) if auxv is not None and not in_place else None
    auxv64 = auxv.float().double() if auxv is not None else None

    def run():
        kw = dict(conv_kw, act=act, aux_mode=aux_mode)
        if out_z is not None:
            kw["out_z"] = out_z
        if nchw:
            ops.conv([(x, in_c)], P[name], out_f32=bufs["out"], nchw_out=True, **kw)
        elif in_place:
            ops.conv([(x, in_c)], P[name], out_split=bufs["out"], out_f32=bufs["outf"], aux=bufs["outf"], **kw)
        else:
            ops.conv([(x, in_c)], P[name], out_split=bufs["out"], out_f32=bufs.get("outf"), aux=aux_t, **kw)

    def ref():
        return [ref_fn(xv, _wval(w, False), b, auxv64)]

    def whole(r):
        y = r[0]
        return torch.ones(y.shape, dtype=torch.bool), y

    place = dict(out=(_val, whole))
    if nchw:
        place = dict(out=(_val, lambda r: (torch.ones(oz, out_c, H, W, dtype=torch.bool), _nchw(r[0]))))
    if "outf" in bufs:
        place["outf"] = (_val, whole)
    return dict(run=run, bufs=bufs, ref=ref, place=place, bar=EXACT, f16=False)


def _conv3d(xv, w, b, pad):   # xv [T, H, W, C] -> [T', H, W, N]
    y = F.conv3d(xv.permute(3, 0, 1, 2)[None], w, b, padding=pad)[0]
    return y.permute(1, 2, 3, 0)


def case_lafc_ztaps(dev, big=False, mixed=False):
    """e2a2: (3,1,1) temporal conv as z-taps with zero fill at both ends (kz=3, pad_z=1)."""
    c = _lafc().c
    return _lafc_case(dev, big, "e2a2", "encoder2.1.conv2", c, c, dict(kz=3, pad_z=1),
                      lambda x, w, b, a: _leaky(_conv3d(x, w, b, (1, 0, 0))))


def case_lafc_ztaps_residual(dev, big=False, mixed=False):
    """res2: z-taps with the fp32 output updated in place as the residual (aux == out_f32) and its split copy."""
    c = _lafc().c
    return _lafc_case(dev, big, "res2", "res_blocks.0.conv2", 4 * c, 4 * c, dict(kz=3, pad_z=1),
                      lambda x, w, b, a: _leaky(_conv3d(x, w, b, (1, 0, 0))) + a, aux="rand",
                      aux_mode=lib.AUX_ADD, in_place=True)


def case_lafc_collapse(dev, big=False, mixed=False):
    """cond2: temporal collapse, a (T,1,1) conv to one output frame (kz=T, out_z=1)."""
    c = _lafc().c
    return _lafc_case(dev, big, "cond2", "condense2", 2 * c, 2 * c, dict(kz=3, pad_z=0), out_z=1,
                      ref_fn=lambda x, w, b, a: _leaky(_conv3d(x, w, b, 0)))


def _lafc_dilated(d):
    def case(dev, big=False, mixed=False):
        c = _lafc().c
        return _lafc_case(dev, big, f"mid{(8, 4, 2, 1).index(d)}", f"middle.{(8, 4, 2, 1).index(d)}", 4 * c, 4 * c,
                          dict(kx=3, ky=3, dil=d, pad_x=d, pad_y=d), T=1,
                          ref_fn=lambda x, w, b, a: _leaky(_nhwc(F.conv2d(_nchw(x), w, b, padding=d, dilation=d))))
    case.__doc__ = f"mid: 3x3 conv with dilation {d} (padding {d}) on one frame (LAFC's dilated middle, 8/4/2/1)."
    return case


def case_lafc_nchw(dev, big=False, mixed=False):
    """dec_2: 3x3 conv to 2 channels stored NCHW fp32 (os_c != 1, per-element stores, N tail of a 16-wide tile)."""
    c = _lafc().c
    return _lafc_case(dev, big, "dec_2", "decoder.2", c // 2, 2, dict(kx=3, ky=3, pad_x=1, pad_y=1), T=1,
                      act=lib.ACT_NONE, nchw=True,
                      ref_fn=lambda x, w, b, a: _nhwc(F.conv2d(_nchw(x), w, b, padding=1)))


def case_lafc_edge(dev, big=False, mixed=False):
    """edge_2: LeakyReLU(0.01) of (conv + residual), the residual added before the activation, 16 channels."""
    return _lafc_case(dev, big, "edge_2", "edgeDetector.mid_layer_2", 16, 16, dict(kx=3, ky=3, pad_x=1, pad_y=1),
                      T=1, act=lib.ACT_LEAKY001, aux_mode=lib.AUX_ADD_PRE, aux="rand",
                      ref_fn=lambda x, w, b, a: _leaky(_nhwc(F.conv2d(_nchw(x), w, b, padding=1)) + a, 0.01))


def _raft_geo(big):
    return (1, 60, 108) if big else (1, 7, 10)


def case_raft_mconv(dev, big=False, mixed=False):
    """mconv: N = 126 channels into channels [128, 254) of the GRU input x; channels 254-255 hold the flow."""
    from fgt_b200 import ops
    net, f16 = _raft(), mixed
    P = _packed(net, dev, mixed)
    n, h, w = _raft_geo(big)
    x, xv = _act16((n, h, w, 256), f16, seed=50)
    x = x.to(dev)
    x4 = _sentinel((n, h, w, 256), torch.float16 if f16 else torch.bfloat16, dev)
    flow, _ = _act16((n, h, w, 2), f16, seed=51)
    x4[..., 254:] = flow.to(dev)   # written earlier by raft_flow_update
    bufs = dict(x4=x4)
    sd = _sd(net)
    wt, b = sd["update_block.encoder.conv.weight"], sd["update_block.encoder.conv.bias"]
    if mixed:
        b = b.half().double()

    def run():
        ops.conv([(x, 256)], P["mconv"], kx=3, ky=3, pad_x=1, pad_y=1, act=lib.ACT_RELU, out_c_total=256,
                 out_c_offset=128, out_split=bufs["x4"])

    def ref():
        return [_nhwc(F.conv2d(_nchw(xv), _wval(wt, f16), b, padding=1)).clamp_min(0)]

    def at(r):
        mask = torch.zeros(n, h, w, 256, dtype=torch.bool)
        mask[..., 128:254] = True
        want = torch.zeros(n, h, w, 256, dtype=torch.float64)
        want[..., 128:254] = r[0]
        return mask, want

    return dict(run=run, bufs=bufs, ref=ref, place=dict(x4=(_val, at)), bar=EXACT, f16=f16)


def case_raft_gru(dev, big=False, mixed=False, half="1"):
    """One SepConvGRU half (1: the 1x5 taps, 2: the 5x1 ones): z | r*h as one N=256 GEMM (AUX_GRU_ZR), then q with the
    state update (AUX_GRU), two A segments [h ; x] each, as update.py:45-60 (under autocast when mixed)."""
    from fgt_b200 import ops
    net, f16 = _raft(), mixed
    P = _packed(net, dev, mixed)
    n, h, w = _raft_geo(big)
    tot = n * h * w
    a16 = torch.float16 if f16 else torch.bfloat16
    hf0 = torch.tanh(torch.randn(tot, 128, generator=_gen(60)))
    if f16:
        hf0 = hf0.half().float()   # the mixed path's state is fp16-valued
    h16 = hf0.half() if f16 else lib.to_split(hf0)
    x4, xv = _act16((n, h, w, 256), f16, seed=61)
    bufs = dict(z=torch.full((tot, 128), SENTINEL, device=dev), rh=_sentinel((n, h, w, 128), a16, dev),
                hf=hf0.to(dev), h4=lib.view16(h16, n, h, w, 128).clone().to(dev))
    x4 = x4.to(dev)
    hv = _val(h16).view(n, h, w, 128)    # h as the conv operand
    hfv = hf0.double().view(n, h, w, 128)  # h as the fp32 state the epilogue reads
    sd = _sd(net)
    u = "update_block.gru."
    kx, ky = (5, 1) if half == "1" else (1, 5)
    pad = (ky // 2, kx // 2)

    def wb(g):
        wt, b = sd[u + f"conv{g}{half}.weight"], sd[u + f"conv{g}{half}.bias"]
        return _wval(wt, f16), (b.half().double() if f16 else b)

    def run():
        kw = dict(kx=kx, ky=ky, pad_x=kx // 2, pad_y=ky // 2, seg_counts=[128, 256])
        ops.conv([(bufs["h4"], 128), (x4, 256)], P[f"gru.zr{half}"], act=lib.ACT_SIGMOID, aux=bufs["hf"],
                 aux_mode=lib.AUX_GRU_ZR, out_f32=bufs["z"].view(n, h, w, 128), out_c_total=128, out_split=bufs["rh"],
                 **kw)
        ops.conv([(bufs["rh"], 128), (x4, 256)], P[f"gru.q{half}"], act=lib.ACT_TANH, aux=bufs["hf"], aux2=bufs["z"],
                 aux_mode=lib.AUX_GRU, out_f32=bufs["hf"].view(n, h, w, 128), out_split=bufs["h4"], **kw)

    r16 = (lambda t: t.half().double()) if f16 else (lambda t: t)   # noqa: E731

    def ref():
        # update.py:45-52: hx = cat(h, x); z = sigmoid(convz1(hx)); r = sigmoid(convr1(hx));
        # q = tanh(convq1(cat(r*h, x))); h = (1-z)*h + z*q  -- every tensor op rounded to fp16 under autocast
        hx = torch.cat([_nchw(hv), _nchw(xv)], 1)
        (wz, bz), (wr, br), (wq, bq) = wb("z"), wb("r"), wb("q")
        z = r16(torch.sigmoid(r16(F.conv2d(hx, wz, bz, padding=pad))))
        r = r16(torch.sigmoid(r16(F.conv2d(hx, wr, br, padding=pad))))
        rh = r16(r * _nchw(hfv))
        # the q launch reads z and r*h as stored: z in fp32, r*h as its split-bf16 (or fp16) operand
        zs = z.float().double()
        rhs = rh if f16 else _nchw(_val(lib.to_split(_nhwc(rh).float())))
        q = r16(torch.tanh(r16(F.conv2d(torch.cat([rhs, _nchw(xv)], 1), wq, bq, padding=pad))))
        if f16:
            hn = r16(r16(r16(1 - zs) * _nchw(hfv)) + r16(zs * q))
        else:
            hn = (1 - zs) * _nchw(hfv) + zs * q
        return [torch.cat([_nhwc(z), _nhwc(rh)], -1), _nhwc(hn)]

    full = lambda r: torch.ones(r.shape, dtype=torch.bool)   # noqa: E731
    place = dict(z=(_val, lambda r: (full(r[0][..., :128]).view(tot, 128), r[0][..., :128].reshape(tot, 128))),
                 rh=(_val, lambda r: (full(r[0][..., 128:]), r[0][..., 128:])),
                 hf=(_val, lambda r: (full(r[1]).view(tot, 128), r[1].reshape(tot, 128))),
                 h4=(_val, lambda r: (full(r[1]), r[1])))
    # fp32: the emulator and the restatement share the GRU formula in float64; mixed: the fp16 roundings of both are
    # at the same points, so a value near an fp16 rounding boundary can land one fp16 ulp apart (rare at these sizes)
    return dict(run=run, bufs=bufs, ref=ref, place=place, bar=EXACT if not f16 else 2.0 ** -10, f16=f16)


def case_raft_corr(dev, big=False, mixed=False):
    """All-pairs correlation: image-1 rows as A, image-2 rows as the weight operand [N = npx, K = 256], alpha = 1/16."""
    n, h, w = _raft_geo(big)
    npx = h * w
    fmap, fv = _act16((2 * npx, 256), False, seed=70)
    fmap = fmap.to(dev)
    bufs = dict(corr=torch.full((npx, npx), SENTINEL, device=dev))

    def run():
        lib.gemm_tc([lib.ASeg(fmap[:, :npx], 256, npx)], fmap[:, npx:], npx, out_w=npx, bn=128, alpha=1.0 / 16.0,
                    out_f32=bufs["corr"], tag="corr")

    def ref():
        return [(fv[:npx] @ fv[npx:].t() / 16.0).reshape(1, 1, npx, npx)]

    place = dict(corr=(_val, lambda r: (torch.ones(npx, npx, dtype=torch.bool), r[0].reshape(npx, npx))))
    return dict(run=run, bufs=bufs, ref=ref, place=place, bar=EXACT, f16=False)


def case_raft_mask(dev, big=False, mixed=False):
    """Mask head: 0.25 * conv1x1(m0) as alpha = 0.25 with the bias pre-scaled, fp32 rows of 576."""
    from fgt_b200 import ops
    net, f16 = _raft(), mixed
    P = _packed(net, dev, mixed)
    n, h, w = _raft_geo(big)
    tot = n * h * w
    m0, mv = _act16((tot, 256), f16, seed=80)
    m0 = m0.to(dev)
    bufs = dict(mask=torch.full((tot, 576), SENTINEL, device=dev))
    sd = _sd(net)
    wt, b = sd["update_block.mask.2.weight"], sd["update_block.mask.2.bias"]
    if f16:
        b = b.half().double()

    def run():
        ops.linear([(m0, 256)], P["mask2"], tot, alpha=0.25, out_f32=bufs["mask"])

    def ref():
        return [(0.25 * (mv @ _wval(wt[:, :, 0, 0], f16).t() + b)).reshape(1, 1, tot, 576)]

    place = dict(mask=(_val, lambda r: (torch.ones(tot, 576, dtype=torch.bool), r[0].reshape(tot, 576))))
    return dict(run=run, bufs=bufs, ref=ref, place=place, bar=EXACT, f16=f16)


def case_gate(dev, big=False, mixed=False):
    """SWMHSA's flow gate f' = f * sigmoid(W [x ; f] + b): a two-segment ungrouped linear, SIGMOID + AUX_MUL, fp32 out
    (attention_flow.py:126-128)."""
    from fgt_b200.fgt_model import linear
    net, f16 = _fgt(), mixed
    P = _packed(net, dev, mixed)
    d, df = net.d, net.df
    rows = 2 * 22 * 36 if big else 136
    xs, xv = _act16((rows, d), f16, seed=90)
    fs, fv = _act16((rows, df), f16, seed=91)
    f = torch.randn(rows, df, generator=_gen(92))
    xs, fs = xs.to(dev), fs.to(dev)
    bufs = dict(fp=torch.full((rows, df), SENTINEL, device=dev))
    f_dev = f.to(dev)
    sd = _sd(net)
    a = "first_s_transformer.attention.reweightFlow.0."
    w, b = sd[a + "weight"], sd[a + "bias"]
    if f16:
        b = b.half().double()

    def run():
        linear([(xs, d), (fs, df)], P["s0.gate"], rows, act=lib.ACT_SIGMOID, aux=f_dev, aux_mode=lib.AUX_MUL,
               out_f32=bufs["fp"], bn=64 if rows <= 128 * 66 else None)

    def ref():
        return [(torch.sigmoid(torch.cat([xv, fv], 1) @ _wval(w, f16).t() + b) * f.double()).reshape(1, 1, rows, df)]

    place = dict(fp=(_val, lambda r: (torch.ones(rows, df, dtype=torch.bool), r[0].reshape(rows, df))))
    return dict(run=run, bufs=bufs, ref=ref, place=place, bar=EXACT, f16=f16)


def case_q_sharded(dev, big=False, mixed=False):
    """Frame-sharded TMHSA's Q projection: a strided 2-D A operand (rows of this rank's frame inside every zone of the
    all-gathered [zones * Lz, d] buffer: elem_offset, sy = Lz * d) with the output box over (tokens x zones)."""
    from fgt_b200 import ops
    from fgt_b200.fgt_model import _pick_bn
    net = _fgt()
    P = dict(_packed(net, dev))
    net._split_qkv(P, "t0")
    d = net.d
    zones, T, off = 4, 3, 1
    zl = 11 * 18 if big else 3 * 5
    Lz = T * zl
    s_all, sv = _act16((zones * Lz, d), False, seed=95)
    s_all = s_all.to(dev)
    bufs = dict(q=_sentinel((zones * zl, d), torch.bfloat16, dev))
    wq = P["t0.q"]
    sd = _sd(net)
    a = "first_t_transformer.attention.query_embedding."

    def run():
        bw, bh = ops.pick_box(zl, zones)
        lib.gemm_tc([lib.ASeg(s_all, d, zl, zones, 1, sx=d, sy=Lz * d, elem_offset=off * zl * d)], wq["w"], d,
                    out_w=zl, out_h=zones, box_w=bw, box_h=bh, bn=_pick_bn(d), bias=wq["b"], out_split=bufs["q"],
                    os_x=d, os_y=zl * d, tag=wq["name"])

    def ref():
        x = sv.view(zones, Lz, d)[:, off * zl:(off + 1) * zl]
        return [(x @ _wval(sd[a + "weight"], False).t() + sd[a + "bias"]).reshape(1, zones, zl, d)]

    place = dict(q=(_val, lambda r: (torch.ones(zones * zl, d, dtype=torch.bool), r[0].reshape(zones * zl, d))))
    return dict(run=run, bufs=bufs, ref=ref, place=place, bar=EXACT, f16=False)


def case_lafc_twoseg(dev, big=False, mixed=False):
    """decoder2.0: 3x3 conv over the upsampled [filled ; pre] pair as two ungrouped A segments (lafc.py:64-71)."""
    from fgt_b200 import ops
    net = _lafc()
    P = _packed(net, dev)
    c = net.c
    H, W = (60, 108) if big else (9, 13)
    u1, v1 = _act16((1, H, W, 4 * c), False, seed=96)
    u2, v2 = _act16((1, H, W, 4 * c), False, seed=97)
    u1, u2 = u1.to(dev), u2.to(dev)
    bufs = dict(out=_sentinel((1, H, W, 2 * c), torch.bfloat16, dev))
    sd = _sd(net)
    w, b = sd["decoder2.0.conv.featureConv.weight"], sd["decoder2.0.conv.featureConv.bias"]

    def run():
        ops.conv([(u1, 4 * c), (u2, 4 * c)], P["dec2_0"], kx=3, ky=3, pad_x=1, pad_y=1, out_split=bufs["out"],
                 seg_counts=[4 * c, 4 * c])

    def ref():
        x = torch.cat([_nchw(v1), _nchw(v2)], 1)
        return [_leaky(_nhwc(F.conv2d(x, _wval(w, False), b, padding=1)))]

    place = dict(out=(_val, lambda r: (torch.ones(r[0].shape, dtype=torch.bool), r[0])))
    return dict(run=run, bufs=bufs, ref=ref, place=place, bar=EXACT, f16=False)


def case_raft_add_relu(dev, big=False, mixed=False):
    """The context net's residual conv: relu(relu(BN(conv(y))) + x) with eval BatchNorm folded into the weights, as
    AUX_ADD_RELU with fp32 + 16-bit outputs (extractor.py:47-56); fp16 under autocast when mixed. The reference folds
    BN as the host does (float64, rounded once to fp32 or fp16), so it is fed the operands as packed."""
    from fgt_b200 import ops
    net, f16 = _raft(), mixed
    P = _packed(net, dev, mixed)
    n, H, W = (1, 240, 432) if big else (1, 9, 13)
    k = "cnet.layer1.0"
    y, yv = _act16((n, H, W, 64), f16, seed=98)
    res = torch.randn(n, H, W, 64, generator=_gen(99))
    if f16:
        res = res.half().float()
    y, res_d = y.to(dev), res.to(dev)
    bufs = dict(outf=torch.full((n, H, W, 64), SENTINEL, device=dev),
                out=_sentinel((n, H, W, 64), torch.float16 if f16 else torch.bfloat16, dev))
    sd = _sd(net)
    g, be, mu, var = (sd[f"{k}.norm2.{x}"] for x in ("weight", "bias", "running_mean", "running_var"))
    sc = g / torch.sqrt(var + 1e-5)
    wf = sd[f"{k}.conv2.weight"] * sc[:, None, None, None]
    bf = (sd[f"{k}.conv2.bias"] - mu) * sc + be
    bf = bf.half().double() if f16 else bf.float().double()
    r16 = (lambda t: t.half().double()) if f16 else (lambda t: t)   # noqa: E731

    def run():
        ops.conv([(y, 64)], P[f"{k}.conv2"], kx=3, ky=3, pad_x=1, pad_y=1, act=lib.ACT_RELU, aux=res_d,
                 aux_mode=lib.AUX_ADD_RELU, out_f32=bufs["outf"], out_split=bufs["out"])

    def ref():
        c = r16(_nhwc(F.conv2d(_nchw(yv), _wval(wf, f16), bf, padding=1)).clamp_min(0))
        return [r16((c + res.double()).clamp_min(0))]

    whole = lambda r: (torch.ones(r[0].shape, dtype=torch.bool), r[0])   # noqa: E731
    return dict(run=run, bufs=bufs, ref=ref, place=dict(outf=(_val, whole), out=(_val, whole)), bar=EXACT, f16=f16)


def case_raft_cnet_inp(dev, big=False, mixed=False):
    """inp = relu(context net output channels 128-255) as a linear into columns [0, 128) of the 256-wide GRU input x
    (os_x = 256); columns 128-255 must stay untouched (raft.py:112-115)."""
    from fgt_b200 import ops
    net, f16 = _raft(), mixed
    P = _packed(net, dev, mixed)
    n, h, w = _raft_geo(big)
    tot = n * h * w
    c, cv = _act16((tot, 128), f16, seed=100)
    c = c.to(dev)
    bufs = dict(x=_sentinel((tot, 256), torch.float16 if f16 else torch.bfloat16, dev))
    sd = _sd(net)
    wt, b = sd["cnet.conv2.weight"][128:, :, 0, 0], sd["cnet.conv2.bias"][128:]
    if f16:
        b = b.half().double()

    def run():
        ops.linear([(c, 128)], P["cnet.inp"], tot, act=lib.ACT_RELU, os_x=256, out_split=bufs["x"])

    def ref():
        return [(cv @ _wval(wt, f16).t() + b).clamp_min(0).reshape(1, 1, tot, 128)]

    def at(r):
        mask = torch.zeros(tot, 256, dtype=torch.bool)
        mask[:, :128] = True
        want = torch.zeros(tot, 256, dtype=torch.float64)
        want[:, :128] = r[0].reshape(tot, 128)
        return mask, want

    return dict(run=run, bufs=bufs, ref=ref, place=dict(x=(_val, at)), bar=EXACT, f16=f16)


CASES = {
    "enc10": case_enc10, "enc12": case_enc12, "enc14": case_enc14, "enc16": case_enc16, "deconv": case_deconv,
    "qkv_slice": case_qkv_slice, "gate": case_gate, "q_sharded": case_q_sharded,
    "lafc_ztaps": case_lafc_ztaps, "lafc_ztaps_residual": case_lafc_ztaps_residual,
    "lafc_collapse": case_lafc_collapse, "lafc_dilated8": _lafc_dilated(8), "lafc_dilated4": _lafc_dilated(4),
    "lafc_dilated2": _lafc_dilated(2), "lafc_dilated1": _lafc_dilated(1), "lafc_twoseg": case_lafc_twoseg,
    "lafc_nchw": case_lafc_nchw, "lafc_edge": case_lafc_edge,
    "raft_mconv": case_raft_mconv, "raft_gru_1x5": case_raft_gru,
    "raft_gru_5x1": functools.partial(case_raft_gru, half="2"), "raft_add_relu": case_raft_add_relu,
    "raft_cnet_inp": case_raft_cnet_inp, "raft_corr": case_raft_corr, "raft_mask": case_raft_mask,
}
MIXED = ("enc10", "enc12", "enc14", "enc16", "deconv", "qkv_slice", "gate", "raft_mconv", "raft_gru_1x5",
         "raft_gru_5x1", "raft_add_relu", "raft_cnet_inp", "raft_mask")
PARAMS = [(name, False) for name in CASES] + [(name, True) for name in MIXED]


def emulate(case):
    """Runs a CPU case through the interpreter; returns the float64 values of its launches and the interpreter."""
    with torch.no_grad(), emulating() as emu:
        case["run"]()
    return [e["v"] for e in emu.launches], emu


def check_placement(case, before, what, tol):
    """Addressed elements within `tol` (of the largest) of the reference, every other element bit-identical."""
    refs = case["ref"]()
    for name, (decode, at) in case["place"].items():
        buf = case["bufs"][name].cpu()
        mask, want = at(refs)
        got = decode(buf)
        assert got.shape == mask.shape, (name, got.shape, mask.shape)
        raw_mask = mask.expand(buf.shape) if buf.dim() > mask.dim() else mask
        assert torch.equal(buf[~raw_mask], before[name][~raw_mask]), f"{what}: {name} written outside its slice"
        err = (got[mask] - want[mask]).abs().max().item() / (want[mask].abs().max().item() + 1e-30)
        assert err <= tol, f"{what}: {name} stored values off by {err:.3e} (tol {tol:g})"


def store_tol(case):
    """Rounding of the stored format: split-bf16 hi + lo of an fp32 value (~2^-17), fp16 (2^-11)."""
    return 2.0 ** -10 if case["f16"] else 2.0 ** -15


@pytest.mark.parametrize("name,mixed", PARAMS)
def test_layer_form_matches_reference(name, mixed):
    """The emulated launch(es) against the float64 reference layer (EXACT, or KTOL / the case's bar for weights the
    host transforms), then the stored outputs: addressed elements within the format's rounding, the rest untouched."""
    case = CASES[name](torch.device("cpu"), mixed=mixed)
    before = {k: v.clone() for k, v in case["bufs"].items()}
    vs, emu = emulate(case)
    refs = case["ref"]()
    for bname, (_, at) in case["place"].items():   # the elements stored are exactly the layer's slice
        raw = emu.written_mask(case["bufs"][bname])
        written = raw.any(0) if case["bufs"][bname].dtype == torch.bfloat16 else raw
        assert torch.equal(written, at(refs)[0]), f"{name}: {bname}: stored elements differ from the layer's slice"
    assert len(vs) == len(refs), f"{len(vs)} launches, {len(refs)} reference values"
    for i, (v, r) in enumerate(zip(vs, refs)):
        r = r.reshape(v.shape)
        err = (v - r).abs().max().item() / (r.abs().max().item() + 1e-30)
        assert err <= case["bar"], f"{name} launch {i}: {err:.3e} (bar {case['bar']:g})"
    if "sanity" in case:   # a second, looser restatement (the reference layer before the host's weight transform)
        sref, sbar = case["sanity"]
        for i, (v, r) in enumerate(zip(vs, sref())):
            r = r.reshape(v.shape)
            err = (v - r).abs().max().item() / (r.abs().max().item() + 1e-30)
            assert err <= sbar, f"{name} launch {i} vs the reference layer: {err:.3e} (bar {sbar:g})"
    check_placement(case, before, name, max(store_tol(case), case["bar"]))


def test_emulator_refuses_other_entries():
    """Only fgt_gemm_tc is emulated: another entry called while the interpreter is installed is an error."""
    with emulating():
        with pytest.raises(AssertionError, match="fgt_attention"):
            lib.load().fgt_attention(None, None)
