"""H100-native small RAFT (the reference's --small, RAFT-S) behind the reference's nn.Module interface, and the
reference's model constructor.

`SmallRAFT(args).forward(image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False)` takes the
reference's state_dict keys for RAFT(small=True) (106 tensors; survives the driver's DataParallel wrap/unwrap) and runs
on libfgt_sm90a.so like raft_model.RAFT:

  * feature / context encoders (SmallEncoder of BottleneckBlocks, extractor.py:60-116,195-267): implicit-GEMM convs;
    the feature net's InstanceNorm = fgt_chan_stats + fgt_instnorm_act, the context net has no norm layer;
  * all-pairs correlation over 128-dimensional features (alpha = 1/sqrt(128)) + fgt_avgpool2 pyramid, 4 levels;
  * per iteration: fgt_corr_lookup (radius 3, 196 values) -> SmallMotionEncoder convs -> ConvGRU (3x3 convs, z | r and
    the (1-z)h+zq update fused in GEMM epilogues) -> flow head -> fgt_raft_flow_update;
  * fgt_upflow8 (8 * bilinear x8, align_corners=True, utils.py:80-82) only where the result is consumed (last
    iteration in test_mode).

fp32 only (3-term split-bf16 GEMMs): the small model under mixed_precision is not implemented and is refused.
"""
import math

import torch
import torch.nn as nn

from . import lib, ops
from .graphs import NativeNet
from .raft_model import RAFT as _BasicRAFT

HDIM, CDIM = 96, 64
LOOK = 200   # lookup rows: 4 levels x 7 x 7 = 196 values, zero-padded to a multiple of 8 channels
XW = 152     # GRU input rows x = [inp(64) | motion features(80) | flow(2)] = 146 channels, zero-padded
FLOW_CH = CDIM + 80


class _Bottleneck(nn.Module):
    def __init__(self, cin, planes, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, planes // 4, 1)
        self.conv2 = nn.Conv2d(planes // 4, planes // 4, 3, padding=1, stride=stride)
        self.conv3 = nn.Conv2d(planes // 4, planes, 1)
        if stride != 1:
            self.downsample = nn.Sequential(nn.Conv2d(cin, planes, 1, stride=stride))


class _SmallEncoder(nn.Module):
    def __init__(self, out_dim):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 32, 7, stride=2, padding=3)
        self.layer1 = nn.Sequential(_Bottleneck(32, 32, 1), _Bottleneck(32, 32, 1))
        self.layer2 = nn.Sequential(_Bottleneck(32, 64, 2), _Bottleneck(64, 64, 1))
        self.layer3 = nn.Sequential(_Bottleneck(64, 96, 2), _Bottleneck(96, 96, 1))
        self.conv2 = nn.Conv2d(96, out_dim, 1)
        for m in self.modules():  # extractor.py:226-228
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')


class _MotionEncoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.convc1 = nn.Conv2d(196, 96, 1)
        self.convf1 = nn.Conv2d(2, 64, 7, padding=3)
        self.convf2 = nn.Conv2d(64, 32, 3, padding=1)
        self.conv = nn.Conv2d(128, 80, 3, padding=1)


class _GRU(nn.Module):
    def __init__(self):
        super().__init__()
        for g in "zrq":
            setattr(self, f"conv{g}", nn.Conv2d(HDIM + 146, HDIM, 3, padding=1))


class _FlowHead(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(HDIM, 128, 3, padding=1)
        self.conv2 = nn.Conv2d(128, 2, 3, padding=1)


class _UpdateBlock(nn.Module):
    def __init__(self):
        super().__init__()
        self.encoder = _MotionEncoder()
        self.gru = _GRU()
        self.flow_head = _FlowHead()


def _refuse_mixed(args):
    if getattr(args, "mixed_precision", False):
        raise ValueError("fgt_b200 small RAFT: mixed_precision is not implemented for the small model "
                         "(use the basic model, or small=True with mixed_precision=False)")


class SmallRAFT(NativeNet):
    def __init__(self, args):
        super().__init__()
        self.args = args
        if getattr(args, "alternate_corr", False):
            raise ValueError("alternate_corr is unreachable in the reference (RAFT/raft.py:106) and unsupported")
        _refuse_mixed(args)
        self.hidden_dim, self.context_dim = HDIM, CDIM
        args.corr_levels, args.corr_radius = 4, 3
        self.fnet = _SmallEncoder(128)
        self.cnet = _SmallEncoder(HDIM + CDIM)
        self.update_block = _UpdateBlock()

    _allocators = _BasicRAFT._allocators

    # ------------------------------------------------------------------ weight packing
    def _pack(self, dev):
        sd = {k: v.detach().float() for k, v in self.state_dict().items()}
        P = {}

        def put(name, key, segs=None, im2col=None, w=None):
            P[name] = ops.packed(name, sd[key + ".weight"] if w is None else w, sd[key + ".bias"], dev, segs, im2col)

        for net in ("fnet", "cnet"):
            put(f"{net}.conv1", f"{net}.conv1", im2col=192)
            for li in (1, 2, 3):
                for bi in (0, 1):
                    k = f"{net}.layer{li}.{bi}"
                    for c in ("conv1", "conv2", "conv3"):
                        put(f"{k}.{c}", f"{k}.{c}")
                    if li > 1 and bi == 0:
                        put(k + ".down", k + ".downsample.0")
            put(f"{net}.conv2", f"{net}.conv2")
        u = "update_block."
        e = u + "encoder."
        put("convc1", e + "convc1", w=torch.nn.functional.pad(sd[e + "convc1.weight"], (0, 0, 0, 0, 0, LOOK - 196)))
        put("convf1", e + "convf1", im2col=128)
        put("convf2", e + "convf2")
        put("mconv", e + "conv")
        g = u + "gru.conv"
        P["gru.zr"] = ops.packed("gru.zr", torch.cat([sd[g + "z.weight"], sd[g + "r.weight"]], 0),
                                 torch.cat([sd[g + "z.bias"], sd[g + "r.bias"]], 0), dev, [HDIM, 146])
        put("gru.q", g + "q", segs=[HDIM, 146])
        put("fh1", u + "flow_head.conv1")
        put("fh2", u + "flow_head.conv2", w=lib.pack_taps_as_n(sd[u + "flow_head.conv2.weight"]))
        cw = P["cnet.conv2"]  # net | inp halves of the context net's output conv (raft.py:112-113)
        P["cnet.net"] = dict(cw, w=cw["w"][..., :HDIM, :].contiguous(), b=cw["b"][:HDIM].contiguous(), N=HDIM,
                             name="cnet.net")
        P["cnet.inp"] = dict(cw, w=cw["w"][..., HDIM:, :].contiguous(), b=cw["b"][HDIM:].contiguous(), N=CDIM,
                             name="cnet.inp")
        self._packed[False] = P
        return P

    # ------------------------------------------------------------------ encoders
    def _encoder(self, img, net, P, dev, n):
        """SmallEncoder.forward (extractor.py:244-267) on `n` raw [0,255] images [n,3,H,W] -> NHWC split-bf16
        features [2, n, H/8, W/8, 96] before the output conv."""
        _, _, H, W = img.shape
        inst = net == "fnet"
        B, A = self._allocators((net, n, H, W, False), dev, False)
        RELU, NONE = lib.ACT_RELU, lib.ACT_NONE
        H2, W2 = H // 2, W // 2
        col = A("col", (n, H2, W2, 192))
        # 2*(x/255)-1 applied to in-bounds taps (raft.py:90-91); zero padding stays zero
        lib.im2col_nchw(img, None, col, k=7, stride=2, pad=3, replicate=False, OH=H2, OW=W2, scale=2.0 / 255.0,
                        shift=-1.0, tag=net + ".conv1")
        stats = B("stats", (n * 96 * 2,), dtype=torch.float64)
        raw = B("raw", (n * H2 * W2 * 32,))  # largest pre-norm conv output (32 channels at 1/2), reused

        def conv_norm_act(xs, name, hh, ww, c_out, stride, out_split, out_f32=None, res=None, relu=True, k=1):
            """conv + norm (feature net) + relu [+ residual relu]; writes out_split / out_f32."""
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

        x = A("x0", (n, H2, W2, 32))
        xf = B("x0f", (n, H2, W2, 32))
        if inst:
            r = raw.view(n, H2, W2, 32)
            ops.linear([(lib.view16(col, n * H2 * W2, 192), 192)], P[net + ".conv1"], n * H2 * W2, out_f32=r)
            lib.chan_stats(r, n, H2 * W2, 32, stats)
            lib.instnorm_act(r, stats, n, H2 * W2, 32, relu=True, out=xf, out_split=x)
        else:
            ops.linear([(lib.view16(col, n * H2 * W2, 192), 192)], P[net + ".conv1"], n * H2 * W2, act=RELU, out_f32=xf,
                       out_split=x)
        hh, ww, cin = H2, W2, 32
        for li, (dim, stride) in enumerate(((32, 1), (64, 2), (96, 2)), start=1):
            for bi in (0, 1):
                st = stride if bi == 0 else 1
                k = f"{net}.layer{li}.{bi}"
                q = dim // 4
                oh, ow = hh // st, ww // st
                y1 = A(f"{k}.y1", (n, hh, ww, q))
                conv_norm_act([(x, cin)], k + ".conv1", hh, ww, q, 1, y1)
                y2 = A(f"{k}.y2", (n, oh, ow, q))
                conv_norm_act([(y1, q)], k + ".conv2", hh, ww, q, st, y2, k=3)
                if st != 1:  # x = norm4(conv1x1_s2(x)), no ReLU (extractor.py:102-104,113-114)
                    res = B(f"{k}.ds", (n, oh, ow, dim))
                    conv_norm_act([(x, cin)], k + ".down", hh, ww, dim, st, None, out_f32=res, relu=False)
                else:
                    res = xf
                xo = A(f"{k}.out", (n, oh, ow, dim))
                xof = B(f"{k}.outf", (n, oh, ow, dim))
                conv_norm_act([(y2, q)], k + ".conv3", oh, ow, dim, 1, xo, out_f32=xof, res=res)
                x, xf, hh, ww, cin = xo, xof, oh, ow, dim
        return x

    # ------------------------------------------------------------------ forward
    def _forward_batch(self, im1, im2, iters, flow_init, test_mode, P, dev):
        """RAFT.forward (raft.py:86-148) of the small model on n image pairs at once."""
        n, _, H, W = im1.shape
        if H % 8 or W % 8:
            raise ValueError(f"RAFT input {H}x{W} must be divisible by 8 (the reference crashes otherwise, "
                             "RAFT/raft.py:64-71 vs extractor.py)")
        h, w = H // 8, W // 8
        npx = h * w
        tot = n * npx
        B, A = self._allocators(("iter", n, H, W, False), dev, False)
        RELU, SIG, TANH, NONE = lib.ACT_RELU, lib.ACT_SIGMOID, lib.ACT_TANH, lib.ACT_NONE
        # ---- feature net on all 2n images, 1x1 output conv -> fmaps [2, 2n*npx, 128] (split)
        f96 = self._encoder(torch.cat([im1, im2], 0), "fnet", P, dev, 2 * n)
        fmap = B("fmap", (2 * tot, 128), dtype=torch.bfloat16)
        ops.linear([(f96.view(2, 2 * tot, 96), 96)], P["fnet.conv2"], 2 * tot, out_split=fmap)
        # ---- all-pairs correlation (corr.py:52-60): <f1_i, f2_j> / sqrt(128) per pair, then the pyramid
        pyr = [B("corr0", (tot, h, w))]
        for i in range(n):
            f1 = lib.ASeg(fmap[:, i * npx:(i + 1) * npx], 128, npx)
            f2 = fmap[:, (n + i) * npx:(n + i + 1) * npx]
            lib.gemm_tc([f1], f2, npx, out_w=npx, bn=128, alpha=1.0 / math.sqrt(128.0),
                        out_f32=pyr[0][i * npx:(i + 1) * npx], tag="corr")
        hh, ww = h, w
        for i in range(1, 4):
            nxt = B(f"corr{i}", (tot, hh // 2, ww // 2))
            lib.avgpool2(pyr[-1], tot, hh, ww, nxt)
            pyr.append(nxt)
            hh, ww = hh // 2, ww // 2
        # ---- context net: net = tanh(c[:96]), inp = relu(c[96:]) (raft.py:112-115)
        c96 = self._encoder(im1, "cnet", P, dev, n)
        hsp = A("h", (tot, HDIM))
        hf = B("hf", (tot, HDIM))
        xbuf = A("x", (tot, XW), zero=True)
        ops.linear([(lib.view16(c96, tot, 96), 96)], P["cnet.net"], tot, act=TANH, out_f32=hf, out_split=hsp)
        ops.linear([(lib.view16(c96, tot, 96), 96)], P["cnet.inp"], tot, act=RELU, os_x=XW, out_split=xbuf)
        # ---- iterations
        coords = B("coords", (tot, 2))
        ys, xs = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing="ij")
        coords.view(n, npx, 2).copy_(torch.stack([xs, ys], -1).reshape(1, npx, 2).float().expand(n, npx, 2))
        if flow_init is not None:
            coords.add_(flow_init.permute(0, 2, 3, 1).reshape(tot, 2).float())
        flow_nchw = B("flow", (n, 2, h, w))
        lib.raft_flow_update(coords, None, h, w, flow_nchw, xbuf, FLOW_CH, n=n)
        look = A("look", (tot, LOOK), zero=True)
        corflo = A("corflo", (n, h, w, 128))  # [cor(96) | flo(32)]
        fcol = A("fcol", (n, h, w, 128))
        flo1 = A("flo1", (n, h, w, 64))
        z = B("z", (tot, HDIM))
        rh = A("rh", (n, h, w, HDIM))
        fh = A("fh", (n, h, w, 128))
        delta = B("delta", (tot, 2))
        h4 = lib.view16(hsp, n, h, w, HDIM)
        x4 = lib.view16(xbuf, n, h, w, XW)
        c3 = dict(kx=3, ky=3, pad_x=1, pad_y=1)
        ups = []
        for it in range(iters):
            lib.corr_lookup(pyr, coords, tot, 3, look)
            # motion encoder (update.py:71-77)
            ops.linear([(look, LOOK)], P["convc1"], tot, act=RELU, os_x=128, out_split=lib.view16(corflo, tot, 128))
            lib.im2col_nchw(flow_nchw, None, fcol, k=7, stride=1, pad=3, replicate=False, OH=h, OW=w)
            ops.linear([(lib.view16(fcol, tot, 128), 128)], P["convf1"], tot, act=RELU, out_split=lib.view16(flo1, tot, 64))
            ops.conv([(flo1, 64)], P["convf2"], act=RELU, out_c_total=128, out_c_offset=96, out_split=corflo, **c3)
            ops.conv([(corflo, 128)], P["mconv"], act=RELU, out_c_total=XW, out_c_offset=CDIM, out_split=x4, **c3)
            # ConvGRU (update.py:23-31): z = sigmoid(convz(hx)) and r*h = sigmoid(convr(hx)) * h as ONE N=192 GEMM
            kw = dict(seg_counts=[HDIM, 146], **c3)
            ops.conv([(h4, HDIM), (x4, XW)], P["gru.zr"], act=SIG, aux=hf, aux_mode=lib.AUX_GRU_ZR,
                     out_f32=z.view(n, h, w, HDIM), out_c_total=HDIM, out_split=rh, **kw)
            ops.conv([(rh, HDIM), (x4, XW)], P["gru.q"], act=TANH, aux=hf, aux2=z, aux_mode=lib.AUX_GRU,
                     out_f32=hf.view(n, h, w, HDIM), out_split=h4, **kw)
            # flow head (update.py:13-14): 96 -> 128 conv, then the 128 -> 2 conv in fgt_conv_tail
            ops.conv([(h4, HDIM)], P["fh1"], act=RELU, out_split=fh, **c3)
            lib.conv_tail(fh, n, h, w, 128, P["fh2"]["w"], 2, P["fh2"]["b"], NONE, delta, nchw=False, tag="fh2")
            lib.raft_flow_update(coords, delta, h, w, flow_nchw, xbuf, FLOW_CH, n=n)
            if not test_mode or it == iters - 1:
                up = torch.empty(n, 2, 8 * h, 8 * w, device=dev)
                lib.upflow8(flow_nchw, h, w, up, n=n)
                ups.append(up)
        return flow_nchw.clone(), ups

    def forward(self, image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False):
        _refuse_mixed(self.args)  # read on every call, as the reference reads self.args.mixed_precision
        if not image1.is_cuda:
            raise RuntimeError("fgt_b200 RAFT runs on a CUDA (sm_90a) device only; there is no CPU fallback")
        if self._graphs is not None and flow_init is None:
            out = self._graphed((iters, bool(test_mode)),
                                lambda a, b: self._forward_impl(a, b, iters, None, test_mode),
                                image1.float().contiguous(), image2.float().contiguous())
            return list(out) if not test_mode else out
        return self._forward_impl(image1, image2, iters, flow_init, test_mode)

    def _forward_impl(self, image1, image2, iters, flow_init, test_mode):
        dev = image1.device
        P = self._packed.get(False) or self._pack(dev)
        image1, image2 = image1.float().contiguous(), image2.float().contiguous()
        lo, ups = self._forward_batch(image1, image2, iters, flow_init, test_mode, P, dev)
        if test_mode:
            return lo, ups[-1]
        return ups


def make_raft(args):
    """The reference's model constructor RAFT(args) (RAFT/raft.py:25-56): SmallRAFT when args.small is set, else the
    basic model, raft_model.RAFT."""
    from . import raft_model
    return SmallRAFT(args) if getattr(args, "small", False) else raft_model.RAFT(args)
