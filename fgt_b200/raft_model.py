"""H100-native RAFT (basic model) behind the reference's nn.Module interface, and the host forward it shares with the
small model (raft_small.SmallRAFT).

Drop-in for the reference's RAFT/raft.py: `RAFT(args).forward(image1, image2, iters=12, flow_init=None, upsample=True,
test_mode=False)` with the reference's state_dict keys (179 tensors of raft-things.pth; survives the driver's
DataParallel wrap/unwrap, tool/video_inpainting.py:186-197, call site :263). Parameter holders only; arithmetic runs in
libfgt_sm90a.so:

  * feature / context encoders: implicit-GEMM convs; InstanceNorm = fgt_chan_stats + fgt_instnorm_act,
    eval-mode BatchNorm folded into the conv weights at pack time;
  * all-pairs correlation: one wgmma GEMM fmap1 x fmap2^T (alpha = 1/sqrt(256)) + fgt_avgpool2 pyramid;
  * per iteration: fgt_corr_lookup -> motion encoder convs -> SepConvGRU (z, r*h, and the
    (1-z)h+zq update fused in GEMM epilogues) -> flow head -> fgt_raft_flow_update;
  * mask head + fgt_convex_upsample only where the result is consumed (last iteration in test_mode;
    the reference computes and discards the other 19, RAFT/raft.py:134-143).

Precision follows `args.mixed_precision`, read on every forward like the reference (raft.py:100,111,128):
  * False (default): every conv is a 3-term split-bf16 GEMM (fp32-grade).
  * True: the convs of the three autocast regions (feature net, context net, update block) are 1-term fp16 GEMMs on
    fp16 weights and fp16 activation rows; the correlation volume and its lookup stay fp32 (raft.py:103-104), and the
    coordinates are fp32 (DESIGN.md section 2 lists where the rounding points differ from autocast).
The two paths keep separate packed weights, workspaces and CUDA graphs.

`_RAFTBase` is the host side both models share: `forward`, the weight packing, the encoders' stem and residual stages,
the correlation pyramid, the context split and the iteration loop with its GRU and flow head. A model class gives its
widths as class attributes, and its motion encoder and upsampling in `_update_heads`.
"""
import math

import torch
import torch.nn as nn

from . import lib, ops
from .graphs import NativeNet

C3 = dict(kx=3, ky=3, pad_x=1, pad_y=1)


class _ResBlock(nn.Module):
    def __init__(self, cin, planes, norm, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, planes, 3, padding=1, stride=stride)
        self.conv2 = nn.Conv2d(planes, planes, 3, padding=1)
        mk = (lambda: nn.BatchNorm2d(planes)) if norm == "batch" else (lambda: nn.InstanceNorm2d(planes))
        self.norm1, self.norm2 = mk(), mk()
        self.stride = stride
        if stride != 1:
            self.norm3 = mk()
            self.downsample = nn.Sequential(nn.Conv2d(cin, planes, 1, stride=stride), self.norm3)


class _Encoder(nn.Module):
    def __init__(self, out_dim, norm):
        super().__init__()
        self.norm_fn = norm
        self.norm1 = nn.BatchNorm2d(64) if norm == "batch" else nn.InstanceNorm2d(64)
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3)
        self.layer1 = nn.Sequential(_ResBlock(64, 64, norm, 1), _ResBlock(64, 64, norm, 1))
        self.layer2 = nn.Sequential(_ResBlock(64, 96, norm, 2), _ResBlock(96, 96, norm, 1))
        self.layer3 = nn.Sequential(_ResBlock(96, 128, norm, 2), _ResBlock(128, 128, norm, 1))
        self.conv2 = nn.Conv2d(128, out_dim, 1)


class _MotionEncoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.convc1 = nn.Conv2d(324, 256, 1)
        self.convc2 = nn.Conv2d(256, 192, 3, padding=1)
        self.convf1 = nn.Conv2d(2, 128, 7, padding=3)
        self.convf2 = nn.Conv2d(128, 64, 3, padding=1)
        self.conv = nn.Conv2d(256, 126, 3, padding=1)


class _GRU(nn.Module):
    def __init__(self):
        super().__init__()
        for g in "zrq":
            setattr(self, f"conv{g}1", nn.Conv2d(384, 128, (1, 5), padding=(0, 2)))
        for g in "zrq":
            setattr(self, f"conv{g}2", nn.Conv2d(384, 128, (5, 1), padding=(2, 0)))


class _FlowHead(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(128, 256, 3, padding=1)
        self.conv2 = nn.Conv2d(256, 2, 3, padding=1)


class _UpdateBlock(nn.Module):
    def __init__(self):
        super().__init__()
        self.encoder = _MotionEncoder()
        self.gru = _GRU()
        self.flow_head = _FlowHead()
        self.mask = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(), nn.Conv2d(256, 576, 1))


class _RAFTBase(NativeNet):
    """RAFT.forward (raft.py:86-148) on n image pairs at once: every kernel of the update loop covers the n*h*w
    positions of all pairs, which is what fills the 132 SMs (one 1/8-resolution pair is 51 tiles).

    Widths of a model: FDIM feature dim, STEM stem width, STAGES (width, stride) of the three residual stages, BLOCK
    the convs of a block as (name, width divisor, kernel, strided), HDIM / CDIM hidden / context dims, RADIUS lookup
    radius, LOOK lookup row pitch, XW GRU-input row pitch (x = [inp | motion features | flow]), FLOW_CH the flow's
    channel in x, GRU the GRU's convs as (suffix, kx, ky)."""

    def __init__(self, args):
        super().__init__()
        self.args = args
        if getattr(args, "alternate_corr", False):
            raise ValueError("alternate_corr is unreachable in the reference (RAFT/raft.py:106) and unsupported")
        self._mixed()
        self.hidden_dim, self.context_dim = self.HDIM, self.CDIM
        args.corr_levels, args.corr_radius = 4, self.RADIUS

    def _mixed(self):
        return bool(getattr(self.args, "mixed_precision", False))

    # ------------------------------------------------------------------ weight packing
    def _pack(self, dev, half=False):
        """half: the mixed-precision set, every conv as a 1-term fp16 layer with fp16-rounded weights and biases (the
        casts autocast applies to a conv's parameters)."""
        sd = {k: v.detach().float() for k, v in self.state_dict().items() if v.dtype.is_floating_point}
        P = {}
        rnd = (lambda t: t.half()) if half else (lambda t: t.float())  # noqa: E731

        def wb(key, bn=None):
            w, b = sd[key + ".weight"], sd[key + ".bias"]
            if bn is not None:  # eval-mode BatchNorm folded into the conv (raft.py:55, model.eval())
                g, be = sd[bn + ".weight"].double(), sd[bn + ".bias"].double()
                mu, var = sd[bn + ".running_mean"].double(), sd[bn + ".running_var"].double()
                s = g / torch.sqrt(var + 1e-5)
                w = rnd(w.double() * s[:, None, None, None])  # folded in fp64, rounded once
                b = rnd((b.double() - mu) * s + be)
            elif half:
                w, b = w.half(), b.half()
            return w, b

        def put(name, key, bn=None, segs=None, im2col=None):
            w, b = wb(key, bn)
            P[name] = ops.packed(name, w, b, dev, segs, im2col, half=half)

        def norm(prefix, i):  # the BatchNorm after a block's i-th conv, where the encoder has one (basic context net)
            return f"{prefix}.norm{i}" if f"{prefix}.norm{i}.running_mean" in sd else None

        for net in ("fnet", "cnet"):
            put(f"{net}.conv1", f"{net}.conv1", norm(net, 1), im2col=192)
            for li in (1, 2, 3):
                for bi in (0, 1):
                    k = f"{net}.layer{li}.{bi}"
                    for i, (c, *_) in enumerate(self.BLOCK, start=1):
                        put(f"{k}.{c}", f"{k}.{c}", norm(k, i))
                    if li > 1 and bi == 0:
                        put(k + ".down", k + ".downsample.0", norm(k, len(self.BLOCK) + 1))
            put(f"{net}.conv2", f"{net}.conv2")
        u = "update_block."
        w, b = wb(u + "encoder.convc1")
        w = torch.nn.functional.pad(w, (0, 0, 0, 0, 0, self.LOOK - w.shape[1]))  # lookup rows: values + zero pad
        P["convc1"] = ops.packed("convc1", w, b, dev, half=half)
        put("convf1", u + "encoder.convf1", im2col=128)
        put("convf2", u + "encoder.convf2")
        put("mconv", u + "encoder.conv")
        segs = [self.HDIM, self.FLOW_CH + 2]
        for s, _, _ in self.GRU:
            put(f"gru.q{s}", u + f"gru.convq{s}", segs=segs)
            (wz, bz), (wr, br) = wb(u + f"gru.convz{s}"), wb(u + f"gru.convr{s}")
            P[f"gru.zr{s}"] = ops.packed(f"gru.zr{s}", torch.cat([wz, wr], 0), torch.cat([bz, br], 0), dev, segs,
                                         half=half)
        put("fh1", u + "flow_head.conv1")
        w2, b2 = wb(u + "flow_head.conv2")  # 2-output conv for fgt_conv_tail: the taps as the N of its GEMM
        P["fh2"] = ops.packed("fh2", lib.pack_taps_as_n(w2), b2, dev, half=half)
        self._pack_heads(put, P)
        cw, hd = P["cnet.conv2"], self.HDIM  # net | inp halves of the context net's output conv (raft.py:112-113)
        P["cnet.net"] = dict(cw, w=cw["w"][..., :hd, :].contiguous(), b=cw["b"][:hd].contiguous(), N=hd,
                             name="cnet.net")
        P["cnet.inp"] = dict(cw, w=cw["w"][..., hd:, :].contiguous(), b=cw["b"][hd:].contiguous(), N=self.CDIM,
                             name="cnet.inp")
        self._packed[half] = P
        return P

    def _pack_heads(self, put, P):
        """Packs the model's own update-block convs with put(name, state-dict key)."""

    # ------------------------------------------------------------------ encoders
    def _encoder(self, img, net, P, dev, n, mixed=False):
        """BasicEncoder / SmallEncoder.forward (extractor.py:168-192,244-267) on `n` raw [0,255] images [n,3,H,W] ->
        NHWC features before the output conv (split-bf16, or fp16 rows when mixed)."""
        _, _, H, W = img.shape
        inst = net == "fnet"
        B, A = self._allocators((net, n, H, W, mixed), dev, mixed)
        RELU, NONE = lib.ACT_RELU, lib.ACT_NONE
        H2, W2, C0 = H // 2, W // 2, self.STEM
        col = A("col", (n, H2, W2, 192))
        # 2*(x/255)-1 applied to in-bounds taps (raft.py:90-91); zero padding stays zero
        lib.im2col_nchw(img, None, col, k=7, stride=2, pad=3, replicate=False, OH=H2, OW=W2, scale=2.0 / 255.0,
                        shift=-1.0, tag=net + ".conv1")
        stats = B("stats", (n * self.STAGES[-1][0] * 2,), dtype=torch.float64)
        # largest pre-norm conv output, reused. mixed: left unrounded (autocast rounds it to fp16 before the norm);
        # rounding it through an fp16 side output costs the half-resolution convs the batched GEMM epilogue
        # (DESIGN.md section 2)
        raw = B("raw", (n * H2 * W2 * C0,))

        def conv_norm_act(xs, name, hh, ww, c_out, k, stride, out_split, out_f32=None, res=None, relu=True):
            """conv (+folded BN) + norm (feature net) + relu [+ residual relu]; writes out_split / out_f32."""
            oh, ow = (hh + 2 * (k // 2) - k) // stride + 1, (ww + 2 * (k // 2) - k) // stride + 1
            kw = dict(kx=k, ky=k, stride=stride, pad_x=k // 2, pad_y=k // 2)
            if inst:
                r = raw[:n * oh * ow * c_out].view(n, oh, ow, c_out)
                ops.conv(xs, P[name], act=NONE, out_f32=r, **kw)
                lib.chan_stats(r, n, oh * ow, c_out, stats)
                lib.instnorm_act(r, stats, n, oh * ow, c_out, relu=relu, res=res, out=out_f32, out_split=out_split)
            elif res is not None:
                ops.conv(xs, P[name], act=RELU, aux=res, aux_mode=lib.AUX_ADD_RELU, out_f32=out_f32,
                         out_split=out_split, **kw)
            else:
                ops.conv(xs, P[name], act=RELU if relu else NONE, out_f32=out_f32, out_split=out_split, **kw)

        x = A("x0", (n, H2, W2, C0))
        xf = B("x0f", (n, H2, W2, C0))
        col16 = lib.view16(col, n * H2 * W2, 192)
        if inst:
            r = raw.view(n, H2, W2, C0)
            ops.linear([(col16, 192)], P[net + ".conv1"], n * H2 * W2, out_f32=r)
            lib.chan_stats(r, n, H2 * W2, C0, stats)
            lib.instnorm_act(r, stats, n, H2 * W2, C0, relu=True, out=xf, out_split=x)
        else:
            ops.linear([(col16, 192)], P[net + ".conv1"], n * H2 * W2, act=RELU, out_f32=xf, out_split=x)
        hh, ww, cin = H2, W2, C0
        for li, (dim, stride) in enumerate(self.STAGES, start=1):
            for bi in (0, 1):
                st = stride if bi == 0 else 1
                k = f"{net}.layer{li}.{bi}"
                oh, ow = hh // st, ww // st
                y, c, yh, yw = x, cin, hh, ww
                for i, (conv, div, ks, strided) in enumerate(self.BLOCK[:-1], start=1):
                    s = st if strided else 1
                    yo = A(f"{k}.y{i}", (n, yh // s, yw // s, dim // div))
                    conv_norm_act([(y, c)], f"{k}.{conv}", yh, yw, dim // div, ks, s, yo)
                    y, c, yh, yw = yo, dim // div, yh // s, yw // s
                if st != 1:  # x = norm(conv1x1_s2(x)), no ReLU (extractor.py:52-53,102-104)
                    res = B(f"{k}.ds", (n, oh, ow, dim))
                    ds16 = A(f"{k}.ds16", (n, oh, ow, dim)) if mixed else None  # makes `res` fp16-valued; never read
                    conv_norm_act([(x, cin)], k + ".down", hh, ww, dim, 1, st, ds16, out_f32=res, relu=False)
                else:
                    res = xf
                xo = A(f"{k}.out", (n, oh, ow, dim))
                xof = B(f"{k}.outf", (n, oh, ow, dim))
                conv, _, ks, _ = self.BLOCK[-1]
                conv_norm_act([(y, c)], f"{k}.{conv}", oh, ow, dim, ks, 1, xo, out_f32=xof, res=res)
                x, xf, hh, ww, cin = xo, xof, oh, ow, dim
        return x

    # ------------------------------------------------------------------ forward
    def _forward_batch(self, im1, im2, iters, flow_init, test_mode, P, dev, mixed=False):
        n, _, H, W = im1.shape
        if H % 8 or W % 8:
            raise ValueError(f"RAFT input {H}x{W} must be divisible by 8 (the reference crashes otherwise, "
                             "RAFT/raft.py:64-71 vs extractor.py)")
        h, w = H // 8, W // 8
        npx = h * w
        tot = n * npx
        B, A = self._allocators(("iter", n, H, W, mixed), dev, mixed)
        RELU, SIG, TANH, NONE = lib.ACT_RELU, lib.ACT_SIGMOID, lib.ACT_TANH, lib.ACT_NONE
        E, D, HD, XW = self.STAGES[-1][0], self.FDIM, self.HDIM, self.XW
        # ---- feature net on all 2n images, 1x1 output conv -> fmaps [2, 2n*npx, D] (split)
        f = lib.view16(self._encoder(torch.cat([im1, im2], 0), "fnet", P, dev, 2 * n, mixed), 2 * tot, E)
        fmap = B("fmap", (2 * tot, D), dtype=torch.bfloat16)
        if mixed:
            # fp16 output (autocast), then exactly to split-bf16: the 3-term correlation below is the reference's fp32
            # correlation of fmap.float() (raft.py:103-104)
            fmap16 = A("fmap16", (2 * tot, D))
            ops.linear([(f, E)], P["fnet.conv2"], 2 * tot, out_split=fmap16)
            lib.f16_to_split(fmap16, fmap)
        else:
            ops.linear([(f, E)], P["fnet.conv2"], 2 * tot, out_split=fmap)
        # ---- all-pairs correlation (corr.py:52-60): corr[i,j] = <f1_i, f2_j> / sqrt(D) per pair, then the pyramid
        pyr = [B("corr0", (tot, h, w))]
        for i in range(n):
            f1 = lib.ASeg(fmap[:, i * npx:(i + 1) * npx], D, npx)
            f2 = fmap[:, (n + i) * npx:(n + i + 1) * npx]  # rows of image 2 as the "weight" operand [N=npx, K=D]
            lib.gemm_tc([f1], f2, npx, out_w=npx, bn=128, alpha=1.0 / math.sqrt(D),
                        out_f32=pyr[0][i * npx:(i + 1) * npx], tag="corr")
        hh, ww = h, w
        for i in range(1, 4):
            nxt = B(f"corr{i}", (tot, hh // 2, ww // 2))
            lib.avgpool2(pyr[-1], tot, hh, ww, nxt)
            pyr.append(nxt)
            hh, ww = hh // 2, ww // 2
        # ---- context net: net = tanh(c[:HDIM]), inp = relu(c[HDIM:]) (raft.py:112-115)
        c = lib.view16(self._encoder(im1, "cnet", P, dev, n, mixed), tot, E)
        hsp = A("h", (tot, HD))
        hf = B("hf", (tot, HD))
        xbuf = A("x", (tot, XW), zero=XW != self.FLOW_CH + 2)  # pad channels after the flow are zeroed once
        ops.linear([(c, E)], P["cnet.net"], tot, act=TANH, out_f32=hf, out_split=hsp)
        ops.linear([(c, E)], P["cnet.inp"], tot, act=RELU, os_x=XW, out_split=xbuf)
        # ---- iterations
        coords = B("coords", (tot, 2))
        ys, xs = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
        coords.view(n, npx, 2).copy_(torch.stack([xs, ys], -1).reshape(1, npx, 2).float().expand(n, npx, 2))
        if flow_init is not None:
            coords.add_(flow_init.permute(0, 2, 3, 1).reshape(tot, 2).float())
        flow_nchw = B("flow", (n, 2, h, w))
        lib.raft_flow_update(coords, None, h, w, flow_nchw, xbuf, self.FLOW_CH, n=n)
        look = A("look", (tot, self.LOOK), zero=True)  # lookup values + zero pad channels
        h4 = lib.view16(hsp, n, h, w, HD)
        x4 = lib.view16(xbuf, n, h, w, XW)
        motion, upsample = self._update_heads(P, B, A, n, h, w, look, flow_nchw, h4, x4)
        z = B("z", (tot, HD))
        rh = A("rh", (n, h, w, HD))
        fh = A("fh", (n, h, w, P["fh1"]["N"]))
        delta = B("delta", (tot, 2))
        ups = []
        for it in range(iters):
            lib.corr_lookup(pyr, coords, tot, self.RADIUS, look)
            motion()
            # SepConvGRU / ConvGRU (update.py:23-31,45-60): z = sigmoid(convz(hx)) and r*h = sigmoid(convr(hx)) * h as
            # ONE GEMM of N = 2 HDIM over the shared input, then the (1-z)h + zq update in the q conv's epilogue
            for s, kx, ky in self.GRU:
                kw = dict(kx=kx, ky=ky, pad_x=kx // 2, pad_y=ky // 2, seg_counts=[HD, self.FLOW_CH + 2])
                ops.conv([(h4, HD), (x4, XW)], P[f"gru.zr{s}"], act=SIG, aux=hf, aux_mode=lib.AUX_GRU_ZR,
                         out_f32=z.view(n, h, w, HD), out_c_total=HD, out_split=rh, **kw)
                ops.conv([(rh, HD), (x4, XW)], P[f"gru.q{s}"], act=TANH, aux=hf, aux2=z, aux_mode=lib.AUX_GRU,
                         out_f32=hf.view(n, h, w, HD), out_split=h4, **kw)
            # flow head (update.py:13-14); its 2-output conv: taps-as-N tensor-core GEMM and the 9-tap sum in one kernel
            ops.conv([(h4, HD)], P["fh1"], act=RELU, out_split=fh, **C3)
            lib.conv_tail(fh, n, h, w, P["fh1"]["N"], P["fh2"]["w"], 2, P["fh2"]["b"], NONE, delta, nchw=False,
                          tag="fh2")
            lib.raft_flow_update(coords, delta, h, w, flow_nchw, xbuf, self.FLOW_CH, n=n, delta_f16=mixed)
            if not test_mode or it == iters - 1:
                up = torch.empty(n, 2, 8 * h, 8 * w, device=dev)
                upsample(up)
                ups.append(up)
        return flow_nchw.clone(), ups

    def forward(self, image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False):
        mixed = self._mixed()  # read on every call, as the reference reads self.args.mixed_precision
        if not image1.is_cuda:
            raise RuntimeError("fgt_b200 RAFT runs on a CUDA (sm_90a) device only; there is no CPU fallback")
        if self._graphs is not None and flow_init is None:
            out = self._graphed((iters, bool(test_mode), mixed),
                                lambda a, b: self._forward_impl(a, b, iters, None, test_mode, mixed),
                                image1.float().contiguous(), image2.float().contiguous())
            return list(out) if not test_mode else out
        return self._forward_impl(image1, image2, iters, flow_init, test_mode, mixed)

    def _forward_impl(self, image1, image2, iters, flow_init, test_mode, mixed=False):
        dev = image1.device
        P = self._packed.get(mixed) or self._pack(dev, mixed)
        image1, image2 = image1.float().contiguous(), image2.float().contiguous()
        lo, ups = self._forward_batch(image1, image2, iters, flow_init, test_mode, P, dev, mixed)
        if test_mode:
            return lo, ups[-1]
        return ups


class RAFT(_RAFTBase):
    FDIM, STEM, STAGES = 256, 64, ((64, 1), (96, 2), (128, 2))
    BLOCK = (("conv1", 1, 3, True), ("conv2", 1, 3, False))   # residual block (extractor.py:9-56)
    HDIM = CDIM = 128
    RADIUS, LOOK = 4, 384   # 4 levels x 9 x 9 = 324 values, zero-padded
    XW, FLOW_CH = 256, 254  # x = [inp(128) | motion features(126) | flow(2)]
    GRU = (("1", 5, 1), ("2", 1, 5))  # SepConvGRU: horizontal (1x5) then vertical (5x1)

    def __init__(self, args):
        if getattr(args, "small", False):
            raise ValueError("fgt_b200.raft_model.RAFT is the basic model; the small model (small=True) is "
                             "fgt_b200.raft_small.SmallRAFT, and fgt_b200.raft_small.make_raft(args) chooses by args.small")
        super().__init__(args)
        self.fnet = _Encoder(256, "instance")
        self.cnet = _Encoder(256, "batch")
        self.update_block = _UpdateBlock()
        for net in (self.fnet, self.cnet):  # extractor.py:146-153
            for m in net.modules():
                if isinstance(m, nn.Conv2d):
                    nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')

    def _pack_heads(self, put, P):
        u = "update_block."
        put("convc2", u + "encoder.convc2")
        put("mask0", u + "mask.0")
        put("mask2", u + "mask.2")
        P["mask2"]["b"] = P["mask2"]["b"] * 0.25  # mask = 0.25 * conv(x) (update.py:135): alpha scales W x

    def _update_heads(self, P, B, A, n, h, w, look, flow, h4, x4):
        """(motion encoder, upsampling) of one iteration: BasicMotionEncoder (update.py:89-97) into x4's channels
        [128, 254), and mask head scaled by 0.25 (update.py:122-125,135) + convex upsampling (raft.py:73-84)."""
        tot = n * h * w
        RELU = lib.ACT_RELU
        cor1 = A("cor1", (n, h, w, 256))
        corflo = A("corflo", (n, h, w, 256))  # [cor(192) | flo(64)]
        fcol = A("fcol", (n, h, w, 128))
        flo1 = A("flo1", (n, h, w, 128))
        m0 = A("m0", (n, h, w, 256))
        mask = B("mask", (tot, 576))

        def motion():
            ops.linear([(look, 384)], P["convc1"], tot, act=RELU, out_split=lib.view16(cor1, tot, 256))
            ops.conv([(cor1, 256)], P["convc2"], act=RELU, out_c_total=256, out_c_offset=0, out_split=corflo, **C3)
            lib.im2col_nchw(flow, None, fcol, k=7, stride=1, pad=3, replicate=False, OH=h, OW=w)
            ops.linear([(lib.view16(fcol, tot, 128), 128)], P["convf1"], tot, act=RELU,
                       out_split=lib.view16(flo1, tot, 128))
            ops.conv([(flo1, 128)], P["convf2"], act=RELU, out_c_total=256, out_c_offset=192, out_split=corflo, **C3)
            ops.conv([(corflo, 256)], P["mconv"], act=RELU, out_c_total=256, out_c_offset=128, out_split=x4, **C3)

        def upsample(up):
            ops.conv([(h4, 128)], P["mask0"], act=RELU, out_split=m0, **C3)
            ops.linear([(lib.view16(m0, tot, 256), 256)], P["mask2"], tot, alpha=0.25, out_f32=mask)
            lib.convex_upsample(mask, flow, h, w, up, n=n)

        return motion, upsample
