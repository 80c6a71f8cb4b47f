"""H100-native FGT generator behind the reference's nn.Module interface.

Drop-in for /root/reference/FGT/models/model.py: `Model(config).forward(frames, flows, masks)`
with the same constructor dict, forward signature, output shape ([b*t,3,H,W]) and state_dict
keys/shapes (SURVEY.md Appendix B), so `load_state_dict(state["model_state_dict"])` of a reference
checkpoint works (tool/video_inpainting.py:217-230, call site :724).

The nn.Modules below only HOLD parameters under the reference's names; forward() never calls
them. All arithmetic runs in libfgt_sm90a.so (wgmma implicit-GEMM engine, fused flash
attention, HBM-bound helpers) through fgt_b200.lib. There is no CPU / PyTorch fallback.
"""
import functools
import math

import torch
import torch.nn as nn

from . import lib, ops
from .graphs import NativeNet, workspace
from .packing import fold_layernorm

LN_EPS = 1e-5


# ----------------------------------------------------------------------------------------------
# parameter holders (names mirror the reference so state_dict keys match)
# ----------------------------------------------------------------------------------------------
class _ConvHolder(nn.Module):
    """Stands in for VanillaConv (network_blocks_2d.py:7-43): key '<name>.featureConv.*'."""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.featureConv = nn.Conv2d(cin, cout, k)


class _DeconvHolder(nn.Module):
    """Stands in for VanillaDeconv (network_blocks_2d.py:46-60): key '<name>.conv.featureConv.*'."""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.conv = _ConvHolder(cin, cout, k)


class _Encoder(nn.Module):
    def __init__(self, cin):
        super().__init__()
        spec = [(cin, 64, 1), (64, 64, 1), (64, 128, 1), (128, 256, 1), (256, 384, 1), (640, 512, 2), (768, 384, 4),
                (640, 256, 8), (512, 128, 1)]
        layers = []
        for ci, co, g in spec:
            layers += [nn.Conv2d(ci, co, 3, groups=g), nn.LeakyReLU(0.2)]
        self.layers = nn.ModuleList(layers)


class _FFN(nn.Module):
    def __init__(self, d, hidden):
        super().__init__()
        self.conv1 = nn.Linear(d, hidden)
        self.conv2 = nn.Sequential(nn.ReLU(), nn.Dropout(0.0), nn.Linear(hidden, d), nn.Dropout(0.0))


class _TAttn(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.query_embedding = nn.Linear(d, d)
        self.key_embedding = nn.Linear(d, d)
        self.value_embedding = nn.Linear(d, d)
        self.output_linear = nn.Linear(d, d)


class _SAttn(nn.Module):
    def __init__(self, d, df, gd):
        super().__init__()
        self.query_embedding = nn.Linear(d + df, d)
        self.key_embedding = nn.Linear(d + df, d)
        self.value_embedding = nn.Linear(d, d)
        self.output_linear = nn.Linear(d, d)
        self.global_extract_v = nn.Conv2d(d, d, gd, stride=gd, groups=d)
        self.global_extract_k = nn.Conv2d(d + df, d + df, gd, stride=gd, groups=d + df)
        self.q_norm = nn.LayerNorm(d + df)
        self.k_norm = nn.LayerNorm(d + df)
        self.v_norm = nn.LayerNorm(d)
        self.reweightFlow = nn.Sequential(nn.Linear(d + df, df), nn.Sigmoid())


class _TBlock(nn.Module):
    def __init__(self, d, hidden):
        super().__init__()
        self.attention = _TAttn(d)
        self.ffn = _FFN(d, hidden)
        self.norm1 = nn.LayerNorm(d)
        self.norm2 = nn.LayerNorm(d)


class _SBlock(nn.Module):
    def __init__(self, d, df, gd, hidden):
        super().__init__()
        self.attention = _SAttn(d, df, gd)
        self.ffn = _FFN(d, hidden)
        self.norm = nn.LayerNorm(d)


class _TSBlock(nn.Module):
    def __init__(self, d, df, gd, hidden):
        super().__init__()
        self.t_transformer = _TBlock(d, hidden)
        self.s_transformer = _SBlock(d, df, gd, hidden)


class _PosEmb(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.proj = nn.Conv2d(d, d, 3, padding=1, groups=d)


class _Vec2Patch(nn.Module):
    def __init__(self, d, cout):
        super().__init__()
        self.embedding = nn.Linear(d, cout)


class _Decoder(nn.Module):
    def __init__(self, c, cout):
        super().__init__()
        self.layer1 = _DeconvHolder(c, c, 3)
        self.layer2 = _ConvHolder(c, c // 2, 3)
        self.layer3 = _DeconvHolder(c // 2, c // 2, 3)
        self.final = _ConvHolder(c // 2, cout, 3)


def _pick_bn(n_per_group, groups=1):
    if n_per_group % 128 == 0:
        return 128
    if n_per_group <= 128:
        return (n_per_group + 15) // 16 * 16 if groups == 1 else n_per_group
    if groups > 1:
        for bn in (96, 80, 64, 48, 32, 16):
            if n_per_group % bn == 0:
                return bn
    return 128


def _fill_sms(bn, n_total, m_positions, groups=1, n_sms=132):
    """Short windows (a frame-sharded rank's 1-3 frames, the driver's t = 6 window) leave most SMs without a tile when
    the channel tile is 128 wide, and a sub-wave GEMM takes as long as its one tile: halve the tile while the launch
    covers at most half a wave (down to 64)."""
    m_tiles = -(-m_positions // 128)
    while (bn > 64 and bn % 32 == 0 and 2 * m_tiles * -(-n_total // bn) <= n_sms   # at most half a wave
           and (groups == 1 or (n_total // groups) % (bn // 2) == 0)):
        bn //= 2
    return bn


def _tile(n_total, groups, m_positions):
    """FGT's channel-tile policy (ops.conv_tile is the conv networks')."""
    return _fill_sms(_pick_bn(n_total // groups, groups), n_total, m_positions, groups)


# every GEMM of the generator takes its channel tile from FGT's policy
conv = functools.partial(ops.conv, tile=_tile)
linear = functools.partial(ops.linear, tile=_tile)


class FGT(NativeNet):
    """Parameter layout of FGT (model.py:196-246) + the sm_90a forward schedule (model.py:249-283)."""

    def __init__(self, t_groupSize, s_windowSize, g_downSize, input_resolution, in_channels, cnum, flow_inChannel,
                 flow_cnum, frame_hidden, flow_hidden, passmask, numBlocks, kernel_size, stride, padding, num_heads,
                 conv_type, norm, use_bias, ape, mlp_ratio=4, drop=0, init_weights=True):
        super().__init__()
        if conv_type != 'vanilla':
            raise ValueError("fgt_b200 implements conv_type='vanilla' only (the only type any shipped config selects)")
        if frame_hidden // num_heads != 128:
            raise ValueError("fgt_b200 attention kernels require head_dim == 128")
        if not passmask or not ape or not use_bias:
            raise ValueError("fgt_b200 implements PASSMASK=1, ape=1, use_bias=1 (the shipped configuration)")
        if drop != 0:
            raise ValueError("dropout must be 0 at inference")
        self.tw, self.sw, self.gd = t_groupSize, s_windowSize, g_downSize
        if self.sw != 8:
            raise ValueError("fgt_b200 spatial attention assumes 8x8 windows (64-token key tiles)")
        self.in_channels = in_channels
        self.d, self.df, self.heads = frame_hidden, flow_hidden, num_heads
        self.ksz, self.stride, self.padding = tuple(kernel_size), tuple(stride), tuple(padding)
        assert self.ksz[0] == self.ksz[1] and self.stride[0] == self.stride[1] and self.padding[0] == self.padding[1]
        self.cnum = cnum
        self.mlp_c = mlp_ratio
        hidden = self.ksz[0] * self.ksz[1] * mlp_ratio
        self.frame_endoder = _Encoder(in_channels)
        self.flow_encoder = nn.Sequential(nn.ReplicationPad2d(2), _ConvHolder(flow_inChannel, flow_cnum, 5),
                                          _ConvHolder(flow_cnum, flow_cnum * 2, 3),
                                          _ConvHolder(flow_cnum * 2, flow_cnum * 2, 3),
                                          _ConvHolder(flow_cnum * 2, flow_cnum * 2, 3))
        self.patch2vec = nn.Conv2d(cnum * 2, frame_hidden, kernel_size, stride, padding)
        self.f_patch2vec = nn.Conv2d(flow_cnum * 2, flow_hidden, kernel_size, stride, padding)
        self.add_pos_emb = _PosEmb(frame_hidden)
        out_shape = (input_resolution[0] // 4, input_resolution[1] // 4)
        self.token_size = [int((out_shape[i] + 2 * padding[i] - kernel_size[i]) / stride[i] + 1) for i in range(2)]
        self.first_t_transformer = _TBlock(frame_hidden, hidden)
        self.first_s_transformer = _SBlock(frame_hidden, flow_hidden, g_downSize, hidden)
        self.transformer = nn.Sequential(*[_TSBlock(frame_hidden, flow_hidden, g_downSize, hidden)
                                           for _ in range(numBlocks // 2 - 1)])
        self.vec2patch = _Vec2Patch(frame_hidden, self.ksz[0] * self.ksz[1] * cnum * 2)
        self.decoder = _Decoder(cnum * 2, 3)
        if init_weights:
            self.init_weights()
        self._mixed = False
        self.capture = None  # set to a dict to record intermediate activations (tests)

    def _cap(self, name, t):
        if self.capture is not None:
            self.capture[name] = t.detach().clone()

    def init_weights(self, gain=0.02):
        """BaseNetwork.init_weights (BaseNetwork.py:20-46): N(0, gain) conv/linear weights, zero bias."""
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                nn.init.normal_(m.weight.data, 0.0, gain)
                if m.bias is not None:
                    nn.init.constant_(m.bias.data, 0.0)

    # ------------------------------------------------------------------ weight packing (one-time)
    def _perm_hidden(self, c):
        """hidden index c*P + p (torch fold layout) -> p*c_count + c (position-major)."""
        P = self.ksz[0] * self.ksz[1]
        idx = torch.arange(P * c).reshape(c, P).t().reshape(-1)  # new[p*c + ci] = old[ci*P + p]
        return idx

    def _pack(self, dev, half=False):
        """half: the mixed-precision set. Every layer of the generator is a 1-term fp16 layer: weights and biases are
        rounded to fp16 once (the casts autocast applies to a Linear's / conv's parameters), LayerNorm affines folded
        into a Linear are folded in fp64 first. LayerNorm affines applied by the norm kernel stay fp32 (autocast runs
        layer_norm in fp32)."""
        sd = {k: v.detach().float() for k, v in self.state_dict().items()}
        P = {}
        rnd = (lambda t: t.half().float()) if half else (lambda t: t)  # noqa: E731

        def put(name, w, b, segs=None):
            P[name] = ops.packed(name, rnd(w), rnd(b), dev, segs, half=half)

        def layer(name, key, segs=None):
            put(name, sd[key + ".weight"], sd[key + ".bias"], segs)

        enc = "frame_endoder.layers."
        for i in (2, 4, 6, 8):
            layer(f"enc{i}", enc + str(i))
        # The flow branch (flow encoder + f_patch2vec) has fp16 weights in both sets: single-plane fp16 operands and
        # activations, one MMA per K step instead of three and half the activation bytes. The flow features only steer
        # the spatial attention's gate and Q/K; the flow tokens stay within 1e-3 of the fp32 reference (fp16 has three
        # more mantissa bits than bf16) and the end-to-end error of the whole branch in fp16 is < 1e-4
        # (tools/precision_study.py, DESIGN.md 2). Every other layer class of the fp32 set needs the 3-term split
        # product: each costs 2e-4..7e-4 end to end on its own even in fp16.
        # Tiny-channel first layers consume im2col rows (fgt_im2col_nchw): one K=64 GEMM each.
        for name, key, h16 in (("enc0", enc + "0", half), ("fenc1", "flow_encoder.1.featureConv", True)):
            P[name] = ops.packed(name, sd[key + ".weight"], rnd(sd[key + ".bias"]), dev, im2col_pad=64, half=h16)
        layer("enc10", enc + "10", [128, 192])
        layer("enc12", enc + "12", [64, 128])
        # enc14 (8 groups of 32+48 -> 32 channels) as 2 super-groups of 4 with block-diagonal weights: the engine then
        # works on 128-wide tiles and full 64-channel chunks (5 per tap for 4 groups instead of 2 half-empty ones per
        # group), which cuts its operand traffic by 3/8 at the price of multiplying exact zeros
        w14, G14 = sd[enc + "14.weight"], 4
        co_g, c0_g, c1_g = w14.shape[0] // 8, 32, 48
        wbd = torch.zeros(w14.shape[0], G14 * (c0_g + c1_g), 3, 3, dtype=w14.dtype, device=w14.device)
        for gi in range(8):
            j, rows_o = gi % G14, slice(gi * co_g, (gi + 1) * co_g)
            wbd[rows_o, j * c0_g:(j + 1) * c0_g] = w14[rows_o, :c0_g]
            wbd[rows_o, G14 * c0_g + j * c1_g:G14 * c0_g + (j + 1) * c1_g] = w14[rows_o, c0_g:]
        put("enc14", wbd, sd[enc + "14.bias"], [G14 * c0_g, G14 * c1_g])
        layer("enc16", enc + "16", [256, 256])
        for name, key in (("fenc2", "flow_encoder.2.featureConv"), ("fenc3", "flow_encoder.3.featureConv"),
                          ("fenc4", "flow_encoder.4.featureConv"), ("f_patch2vec", "f_patch2vec")):
            P[name] = ops.packed(name, sd[key + ".weight"], rnd(sd[key + ".bias"]), dev, half=True)
        layer("patch2vec", "patch2vec")
        P["pos_w"] = rnd(sd["add_pos_emb.proj.weight"]).reshape(-1).contiguous().to(dev)
        P["pos_b"] = rnd(sd["add_pos_emb.proj.bias"]).contiguous().to(dev)
        perm_ffn = self._perm_hidden(self.mlp_c).to(sd["patch2vec.weight"].device)

        def ffn(pre, name, gamma, beta):
            w1, b1 = fold_layernorm(sd[pre + "ffn.conv1.weight"], sd[pre + "ffn.conv1.bias"], gamma, beta, half=half)
            put(name + ".ffn1", w1[perm_ffn], b1[perm_ffn])
            put(name + ".ffn2", sd[pre + "ffn.conv2.2.weight"][:, perm_ffn], sd[pre + "ffn.conv2.2.bias"])

        def tblock(pre, name):
            # norm1 is NOT folded: TMHSA zero-pads the LayerNorm OUTPUT (attention_base.py:86-89), so padded
            # rows must be exact zeros after the affine; rownorm applies gamma/beta itself here.
            a = pre + "attention."
            P[name + ".ln_g"] = sd[pre + "norm1.weight"].contiguous().to(dev)
            P[name + ".ln_b"] = sd[pre + "norm1.bias"].contiguous().to(dev)
            put(name + ".qkv", torch.cat([sd[a + n + "_embedding.weight"] for n in ("query", "key", "value")], 0),
                torch.cat([sd[a + n + "_embedding.bias"] for n in ("query", "key", "value")], 0))
            put(name + ".o", sd[a + "output_linear.weight"], sd[a + "output_linear.bias"])
            ffn(pre, name, sd[pre + "norm2.weight"], sd[pre + "norm2.bias"])

        def sblock(pre, name):
            a = pre + "attention."
            put(name + ".gate", sd[a + "reweightFlow.0.weight"], sd[a + "reweightFlow.0.bias"], [self.d, self.df])
            wq, bq = fold_layernorm(sd[a + "query_embedding.weight"], sd[a + "query_embedding.bias"],
                                    sd[a + "q_norm.weight"], sd[a + "q_norm.bias"], half=half)
            wk, bk = fold_layernorm(sd[a + "key_embedding.weight"], sd[a + "key_embedding.bias"],
                                    sd[a + "k_norm.weight"], sd[a + "k_norm.bias"], half=half)
            wv, bv = fold_layernorm(sd[a + "value_embedding.weight"], sd[a + "value_embedding.bias"],
                                    sd[a + "v_norm.weight"], sd[a + "v_norm.bias"], half=half)
            put(name + ".qk", torch.cat([wq, wk], 0), torch.cat([bq, bk], 0))
            put(name + ".v", wv, bv)
            put(name + ".o", sd[a + "output_linear.weight"], sd[a + "output_linear.bias"])
            # depthwise pooling weights tap-major [gd*gd, C] (fgt_swin_prep reads one coalesced row per tap)
            P[name + ".gk_w"] = rnd(sd[a + "global_extract_k.weight"]).reshape(self.d + self.df, -1).t().contiguous().to(dev)
            P[name + ".gk_b"] = rnd(sd[a + "global_extract_k.bias"]).contiguous().to(dev)
            P[name + ".gv_w"] = rnd(sd[a + "global_extract_v.weight"]).reshape(self.d, -1).t().contiguous().to(dev)
            P[name + ".gv_b"] = rnd(sd[a + "global_extract_v.bias"]).contiguous().to(dev)
            ffn(pre, name, sd[pre + "norm.weight"], sd[pre + "norm.bias"])

        tblock("first_t_transformer.", "t0")
        sblock("first_s_transformer.", "s0")
        for i in range(len(self.transformer)):
            tblock(f"transformer.{i}.t_transformer.", f"t{i + 1}")
            sblock(f"transformer.{i}.s_transformer.", f"s{i + 1}")
        perm_v2p = self._perm_hidden(self.cnum * 2).to(perm_ffn.device)
        put("vec2patch", sd["vec2patch.embedding.weight"][perm_v2p], sd["vec2patch.embedding.bias"][perm_v2p])
        # VanillaDeconv = nearest x2 then 3x3 conv (network_blocks_2d.py:58-60). Output pixel (2i+py, 2j+px)
        # only sees 2x2 low-res inputs, so each deconv becomes four 2x2 "phase" convs on the low-res map with
        # pre-summed taps (2.25x fewer MACs, no upsampled intermediate): rows {i-1,i} for py=0, {i,i+1} for py=1.
        def deconv(name, key):
            w, b = rnd(sd[key + ".weight"]), sd[key + ".bias"]  # mixed: the fp16 taps are summed, then rounded once
            rows = {0: ([0], [1, 2]), 1: ([0, 1], [2])}  # phase -> 3x3 tap indices merged into each of the 2 taps
            for py in (0, 1):
                for px in (0, 1):
                    w2 = torch.stack([torch.stack([w[:, :, rows[py][a], :][:, :, :, rows[px][c]].sum((2, 3))
                                                   for c in (0, 1)], -1) for a in (0, 1)], -2)  # [co, ci, 2, 2]
                    put(f"{name}.p{py}{px}", w2, b)

        deconv("dec1", "decoder.layer1.conv.featureConv")
        layer("dec2", "decoder.layer2.featureConv")
        deconv("dec3", "decoder.layer3.conv.featureConv")
        # final 64->3 conv for fgt_conv_tail: the taps as the N of its GEMM (9*3 rows, zero-padded to 32)
        put("dec4", lib.pack_taps_as_n(sd["decoder.final.featureConv.weight"]), sd["decoder.final.featureConv.bias"])
        self._packed[half] = P
        return P

    # ------------------------------------------------------------------ geometry / workspaces
    def _geometry(self, b, t, H, W, dev, mixed=False):
        key = (b, t, H, W, str(dev), mixed)
        if key in self._geo:
            return self._geo[key]
        if H % 4 or W % 4:
            raise ValueError(f"FGT input {H}x{W} must be divisible by 4 (model.py:55-63 views features as H//4 x W//4)")
        g = type("Geo", (), {})()
        g.a16 = lib.act16_dtype(mixed)
        bt = b * t
        g.b, g.t, g.bt, g.H, g.W = b, t, bt, H, W
        g.OH, g.OW = H // 4, W // 4
        k, s, p = self.ksz[0], self.stride[0], self.padding[0]
        g.h = (g.OH + 2 * p - k) // s + 1
        g.w = (g.OW + 2 * p - k) // s + 1
        g.n = g.h * g.w
        h, w = g.h, g.w
        # --- temporal zones (attention_base.py:29-34 / 46-50)
        gs = self.tw
        wh, ww = math.ceil(h / gs), math.ceil(w / gs)
        g.tHn, g.tWn = h + (wh - h % wh) % wh, w + (ww - w % ww) % ww
        g.zh, g.zw = g.tHn // gs, g.tWn // gs
        g.Lz = t * g.zh * g.zw
        g.Lzp = (g.Lz + 7) // 8 * 8
        g.zones = b * gs * gs
        bi, zy, zx, ti, yy, xx = torch.meshgrid(torch.arange(b), torch.arange(gs), torch.arange(gs), torch.arange(t),
                                                torch.arange(g.zh), torch.arange(g.zw), indexing="ij")
        Y, X = zy * g.zh + yy, zx * g.zw + xx
        tok = ((bi * t + ti) * h + Y) * w + X
        tok = torch.where((Y < h) & (X < w), tok, torch.full_like(tok, -1))
        g.zone_map = tok.reshape(-1).to(torch.int32).to(dev)
        # --- spatial windows (attention_flow.py:39-43 / 58-61)
        ws = self.sw
        g.sHn, g.sWn = h + (ws - h % ws) % ws, w + (ws - w % ws) % ws
        g.nwin = (g.sHn // ws) * (g.sWn // ws)
        g.nwp = (g.nwin + 1) // 2 * 2
        g.gh, g.gw = g.sHn // self.gd, g.sWn // self.gd
        g.G = g.gh * g.gw
        g.glr = (g.G + 63) // 64 * 64
        g.R = g.nwp * 64 + g.glr
        f, wy, wx, py, px = torch.meshgrid(torch.arange(bt), torch.arange(g.sHn // ws), torch.arange(g.sWn // ws),
                                           torch.arange(ws), torch.arange(ws), indexing="ij")
        Y, X = wy * ws + py, wx * ws + px
        tok = (f * h + Y) * w + X
        tok = torch.where((Y < h) & (X < w), tok, torch.full_like(tok, -1)).reshape(bt, g.nwin * 64)
        full = torch.full((bt, g.nwp * 64), -1, dtype=tok.dtype)
        full[:, :g.nwin * 64] = tok
        g.win_map = full.reshape(-1).to(torch.int32).to(dev)
        g.bufs = {}
        self._geo[key] = g
        return g

    @staticmethod
    def _buf(g, name, shape, dev, dtype=torch.float32, zero=False):
        return workspace(g.bufs, name, shape, dev, dtype, zero)

    # ------------------------------------------------------------------ op helpers
    @staticmethod
    def _deconv(x, cin, P, name, out_split):
        """nearest-x2 + 3x3 conv + LeakyReLU as four 2x2 phase convs writing the interleaved [n,2h,2w,N] output."""
        for py in (0, 1):
            for px in (0, 1):
                wp = P[f"{name}.p{py}{px}"]
                ops.conv([(x, cin)], wp, kx=2, ky=2, pad_x=1 - px, pad_y=1 - py, out_phase=(py, px),
                         bn=_pick_bn(wp["N"]), out_split=out_split)

    def _ffn(self, g, P, name, x, xs, dev, need_split=True):
        """x += FusionFeedForward(LN(x)) (ffn_base.py:53-77, model.py:128-129 / 147-148). need_split: whether the next
        consumer reads the split-bf16 copy of x (a spatial block's gate GEMM, vec2patch); when it does not (a temporal
        block or the positional embedding follows: they read the fp32 x), the second GEMM writes the fp32 x alone."""
        with lib.scope("ffn"):
            self._ffn_impl(g, P, name, x, xs if need_split else None, dev)

    def _ffn_impl(self, g, P, name, x, xs, dev):
        rows, d = g.bt * g.n, self.d
        k, s, p = self.ksz[0], self.stride[0], self.padding[0]
        hidden = k * k * self.mlp_c
        y = self._buf(g, "ffn_y", (rows, d), dev, g.a16)
        hid = self._buf(g, "ffn_hid", (rows, hidden), dev)
        hid2 = self._buf(g, "ffn_hid2", (rows, hidden), dev, g.a16)
        lib.rownorm(x, None, y, rows_per_batch=rows, total_rows=rows, dst_batch_rows=rows, eps=LN_EPS)
        linear([(y, d)], P[name + ".ffn1"], rows, out_f32=hid)
        # fold / coverage division / unfold / ReLU (ffn_base.py:57-75) in one launch, no image round trip
        lib.fold_unfold(hid, g.bt, g.h, g.w, self.mlp_c, k, k, s, p, g.OH, g.OW, hid2, relu=True)
        linear([(hid2, hidden)], P[name + ".ffn2"], rows, aux=x, aux_mode=lib.AUX_ADD, out_f32=x, out_split=xs)

    def enable_frame_sharding(self, total_frames, group=None, rank=None, world=None, exchange="p2p"):
        """Frame-sharded execution of ONE clip window over the ranks of `group` (SURVEY §8e): this rank's
        forward() then takes only its contiguous frames [1, t_local, ...] (parallel.shard_items(total_frames,
        rank, world)) and returns their inpainted frames. Everything is per frame except TMHSA, which needs
        the LayerNorm'd zone rows of all frames once per temporal layer:
          exchange="p2p"  — the LayerNorm kernel stores its rows straight into every peer's K/V-input buffer
                            over NVLink (fgt_rownorm_bcast) and a device-side barrier orders them
                            (fgt_peer_barrier); no collective call, CUDA-graph replayable;
          exchange="nccl" — torch.distributed all-gather of the rows + re-ordering copies (the baseline).
        total_frames=None switches sharding off. Collective: every rank of the group must call it."""
        if total_frames is None:
            self._fshard = None
            return
        if self._mixed:
            raise ValueError("frame sharding runs the fp32 path only: call enable_mixed_precision(False) first")
        import torch.distributed as dist
        from . import parallel
        if exchange not in ("p2p", "nccl"):
            raise ValueError(f"exchange={exchange!r}")
        if world is None:
            world = dist.get_world_size(group) if dist.is_initialized() else 1
            rank = dist.get_rank(group) if dist.is_initialized() else 0
        self._fshard = dict(T=total_frames, group=group, rank=rank, counts=parallel.frame_counts(total_frames, world),
                            work={}, exchange=exchange, layer=0)
        if exchange == "p2p":
            if getattr(self, "_peer", None) is None:
                from .peer import PeerGroup
                self._peer = PeerGroup(group, rank, world)
            self._fshard["peer"] = self._peer

    def _temporal_sharded_p2p(self, g, P, name, x, xs, dev):
        """Frame-sharded TMHSA with the exchange fused into the LayerNorm: rows go to all peers by P2P stores."""
        fs = self._fshard
        counts, rank, pg = fs["counts"], fs["rank"], fs["peer"]
        d, zl = self.d, g.zh * g.zw
        T, off = sum(counts), sum(counts[:rank])
        Lzl, Lz = g.Lz, T * zl
        plane = g.zones * Lz * d
        key = ("s_all", g.zones, Lz, d)
        if key not in fs["work"]:
            bufs = []
            for _ in range(2):  # double-buffered by layer parity: a peer may still read layer i while i+1 is written
                ptrs, view = pg.alloc(2 * plane * 2)
                bufs.append((ptrs, view.view(torch.bfloat16).view(2, g.zones * Lz, d)))
            fs["work"][key] = bufs
        ptrs, s_all = fs["work"][key][fs["layer"] % 2]
        fs["layer"] += 1
        self._split_qkv(P, name)
        q = self._buf(g, f"tp_q{T}", (g.zones * Lzl, d), dev, g.a16)
        kv = self._buf(g, f"tp_kv{T}", (g.zones * Lz, 2 * d), dev, g.a16)
        att = self._buf(g, "att_tok", (g.bt * g.n, d), dev, g.a16)   # attention output in token order
        lib.rownorm_bcast(x, ptrs, plane, gather=g.zone_map, rows_per_batch=Lzl, total_rows=g.zones * Lzl,
                          dst_batch_rows=Lz, dst_row0=off * zl, eps=LN_EPS, gamma=P[name + ".ln_g"],
                          beta=P[name + ".ln_b"])
        # Q only for this rank's frames: rows [off*zl, off*zl + Lzl) of every zone, read in place (strided view). These
        # rows were written by this rank's own LayerNorm launch (stream order), so the Q projection runs BEFORE the
        # barrier and hides the time the peers' rows need to arrive over NVLink.
        wq = P[name + ".q"]
        bw, bh = ops.pick_box(Lzl, g.zones)
        lib.gemm_tc([lib.ASeg(s_all, d, Lzl, g.zones, 1, sx=d, sy=Lz * d, elem_offset=off * zl * d)], wq["w"], d,
                    out_w=Lzl, out_h=g.zones, box_w=bw, box_h=bh, bn=_pick_bn(d), bias=wq["b"],
                    out_split=q, os_x=d, os_y=Lzl * d, tag=wq["name"])
        pg.barrier()  # every peer's rows of this layer are in s_all
        linear([(s_all, d)], P[name + ".kv"], g.zones * Lz, out_split=kv)
        lib.attention(q, kv, kv, att, batches=g.zones, heads=self.heads, Lq=Lzl, Lk=Lz, q_ld=d, k_ld=2 * d, v_ld=2 * d,
                      out_ld=d, q_batch_stride=Lzl * d, k_batch_stride=Lz * 2 * d, v_batch_stride=Lz * 2 * d,
                      out_batch_stride=Lzl * d, scale=1.0 / math.sqrt(d // self.heads), v_off=d, out_rowmap=g.zone_map,
                      tag=name)
        self._out_proj(g, P, name, att, x)

    def _out_proj(self, g, P, name, att, x):
        """x += output_linear(att) (attention_base.py:105, attention_flow.py:170; residual of model.py:127 / 146). The
        attention kernel has already undone the zone / window regrouping in its store (out_rowmap), so this is a plain
        row-major GEMM over the real tokens with the residual in its epilogue."""
        rows = g.bt * g.n
        linear([(att, self.d)], P[name + ".o"], rows, aux=x, aux_mode=lib.AUX_ADD, out_f32=x)

    def _split_qkv(self, P, name):
        """Q-only and K|V-only slices of the fused temporal projection (frame-sharded TMHSA: Q for the local
        frames, K|V for the rows of every frame)."""
        if name + ".q" not in P:
            d, w = self.d, P[name + ".qkv"]
            P[name + ".q"] = dict(w, w=w["w"][:, :d].contiguous(), b=w["b"][:d].contiguous(), N=d, name=name + ".q")
            P[name + ".kv"] = dict(w, w=w["w"][:, d:].contiguous(), b=w["b"][d:].contiguous(), N=2 * d,
                                   name=name + ".kv")

    def _temporal_sharded(self, g, P, name, x, xs, dev):
        """TMHSA over all T frames of the window with this rank holding g.t of them: queries = own frames,
        keys / values = every frame (projected locally from the all-gathered LayerNorm output)."""
        from . import parallel
        fs = self._fshard
        if fs["exchange"] == "p2p":
            return self._temporal_sharded_p2p(g, P, name, x, xs, dev)
        counts = fs["counts"]
        d, zl = self.d, g.zh * g.zw
        T, tmax = sum(counts), max(counts)
        Lzl, Lz, Lqp = g.Lz, T * zl, tmax * zl
        self._split_qkv(P, name)
        s_loc = self._buf(g, f"ts_s{T}", (g.zones * Lqp, d), dev, g.a16, zero=True)
        q = self._buf(g, f"ts_q{T}", (g.zones * Lqp, d), dev, g.a16)
        kv = self._buf(g, f"ts_kv{T}", (g.zones * Lz, 2 * d), dev, g.a16)
        att = self._buf(g, "att_tok", (g.bt * g.n, d), dev, g.a16)   # attention output in token order
        lib.rownorm(x, None, s_loc, gather=g.zone_map, rows_per_batch=Lzl, total_rows=g.zones * Lzl,
                    dst_batch_rows=Lqp, eps=LN_EPS, gamma=P[name + ".ln_g"], beta=P[name + ".ln_b"])
        s_all = parallel.allgather_zone_rows(s_loc.view(2, g.zones, Lqp, d), counts, zl, fs["group"], fs["work"])
        s_all = s_all.view(2, g.zones * Lz, d)
        linear([(s_loc, d)], P[name + ".q"], g.zones * Lqp, out_split=q)
        linear([(s_all, d)], P[name + ".kv"], g.zones * Lz, out_split=kv)
        lib.attention(q, kv, kv, att, batches=g.zones, heads=self.heads, Lq=Lzl, Lk=Lz, q_ld=d, k_ld=2 * d, v_ld=2 * d,
                      out_ld=d, q_batch_stride=Lqp * d, k_batch_stride=Lz * 2 * d, v_batch_stride=Lz * 2 * d,
                      out_batch_stride=Lzl * d, scale=1.0 / math.sqrt(d // self.heads), v_off=d, out_rowmap=g.zone_map,
                      tag=name)
        self._out_proj(g, P, name, att, x)

    def _temporal(self, g, P, name, x, xs, dev, need_split=True):
        """TemporalTransformer.forward (model.py:124-130) with TMHSA (attention_base.py:76-106)."""
        with lib.scope("tmhsa"):
            if getattr(self, "_fshard", None) is not None:
                self._temporal_sharded(g, P, name, x, xs, dev)
            else:
                self._tmhsa(g, P, name, x, dev)
        self._ffn(g, P, name, x, xs, dev, need_split)

    def _tmhsa(self, g, P, name, x, dev):
        """x += TMHSA(LN(x)): LayerNorm + zone gather, fused QKV GEMM, dense flash attention, out-projection."""
        d, rows_z = self.d, g.zones * g.Lz
        s_zm = self._buf(g, "t_s", (rows_z, d), dev, g.a16)
        qkv = self._buf(g, "t_qkv", (rows_z, 3 * d), dev, g.a16)
        att = self._buf(g, "att_tok", (g.bt * g.n, d), dev, g.a16)   # attention output in token order
        lib.rownorm(x, None, s_zm, gather=g.zone_map, rows_per_batch=rows_z, total_rows=rows_z,
                    dst_batch_rows=rows_z, eps=LN_EPS, gamma=P[name + ".ln_g"], beta=P[name + ".ln_b"])
        linear([(s_zm, d)], P[name + ".qkv"], rows_z, out_split=qkv)  # one N=1536 GEMM: Q | K | V, all row-major
        lib.attention(qkv, qkv, qkv, att, batches=g.zones, heads=self.heads, Lq=g.Lz, Lk=g.Lz, q_ld=3 * d, k_ld=3 * d,
                      v_ld=3 * d, out_ld=d, q_batch_stride=g.Lz * 3 * d, k_batch_stride=g.Lz * 3 * d,
                      v_batch_stride=g.Lz * 3 * d, out_batch_stride=g.Lz * d, scale=1.0 / math.sqrt(d // self.heads),
                      k_off=d, v_off=2 * d, out_rowmap=g.zone_map, tag=name)
        self._out_proj(g, P, name, att, x)

    def _spatial(self, g, P, name, x, xs, f, fs, dev, need_split=True):
        """SpatialTransformer.forward (model.py:144-149) with SWMHSA (attention_flow.py:115-171)."""
        with lib.scope("swmhsa"):
            self._swmhsa(g, P, name, x, xs, f, fs, dev)
        self._ffn(g, P, name, x, xs, dev, need_split)

    def _swmhsa(self, g, P, name, x, xs, f, fs, dev):
        """x += SWMHSA(x, f): flow gate, pooled global tokens, LayerNorms, Q|K and V GEMMs, windowed flash attention,
        out-projection."""
        d, df, bt = self.d, self.df, g.bt
        rows = bt * g.n
        fp = self._buf(g, "s_fp", (rows, df), dev)
        qkn = self._buf(g, "s_qkn", (bt * g.R, d + df), dev, g.a16, zero=True)
        vn = self._buf(g, "s_vn", (bt * g.R, d), dev, g.a16, zero=True)
        qkv = self._buf(g, "s_qkv", (bt * g.R, 3 * d), dev, g.a16)
        att = self._buf(g, "att_tok", (rows, d), dev, g.a16)         # attention output in token order
        # flow re-weighting gate: f' = f * sigmoid(W_r [x; f] + b_r)   (attention_flow.py:126-128)
        linear([(xs, d), (fs, df)], P[name + ".gate"], rows, act=lib.ACT_SIGMOID, aux=f, aux_mode=lib.AUX_MUL,
               out_f32=fp, bn=64 if rows <= 128 * 66 else None)  # <= half a wave of 128-wide tiles -> 64 wide
        # pooled global tokens (attention_flow.py:135,145) and the LayerNorm statistics of window rows and pooled
        # rows (attention_flow.py:142-143,154): one launch
        nl = g.nwp * 64
        lib.swin_prep(x, fp, bt, g.h, g.w, g.win_map, nl, g.R, self.gd, g.gh, g.gw, P[name + ".gk_w"],
                      P[name + ".gk_b"], P[name + ".gv_w"], P[name + ".gv_b"], qkn, vn, eps=LN_EPS, tag=name)
        # Q | K from the 768-wide normalised rows, V from the 512-wide ones: two GEMMs into one [rows, 3d] buffer
        linear([(qkn, d + df)], P[name + ".qk"], bt * g.R, out_split=qkv, os_x=3 * d)
        linear([(vn, d)], P[name + ".v"], bt * g.R, out_split=qkv, os_x=3 * d, out_elem_offset=2 * d)
        lib.attention(qkv, qkv, qkv, att, batches=bt, heads=self.heads, Lq=nl, Lk=g.R, Lk_rows=g.R, q_ld=3 * d,
                      k_ld=3 * d, v_ld=3 * d, out_ld=d, q_batch_stride=g.R * 3 * d, k_batch_stride=g.R * 3 * d,
                      v_batch_stride=g.R * 3 * d, out_batch_stride=nl * d, scale=1.0 / math.sqrt(d // self.heads),
                      mode=1, glob_start=nl, glob_count=g.G, k_off=d, v_off=2 * d, out_rowmap=g.win_map, tag=name)
        self._out_proj(g, P, name, att, x)

    # ------------------------------------------------------------------ forward
    def enable_mixed_precision(self, on=True):
        """Mixed precision, opt-in: the generator runs as the reference does under
        torch.autocast("cuda", dtype=torch.float16). Every Linear / conv is a 1-term fp16 tensor-core GEMM (fp16
        weights and activation rows, fp32 accumulation), the attention takes fp16 Q, K, V with its scores and softmax
        in fp32, LayerNorm statistics stay fp32. The fp16 weights, workspaces and CUDA graphs are kept apart from the
        fp32 path's, so the flag may change between calls; off (the default) gives the fp32 path's outputs bit for
        bit. Not available with frame sharding. DESIGN.md section 2 lists where the rounding points differ from
        autocast."""
        if on and getattr(self, "_fshard", None) is not None:
            raise ValueError("mixed precision is not available with frame sharding: call enable_frame_sharding(None) "
                             "first")
        self._mixed = bool(on)

    def forward(self, masked_frames, flows, masks):
        if not masked_frames.is_cuda:
            raise RuntimeError("fgt_b200.FGT runs on a CUDA (sm_90a) device only; there is no CPU fallback")
        fs = getattr(self, "_fshard", None)
        graph_ok = fs is None or fs["exchange"] == "p2p"  # NCCL calls are not captured; the P2P exchange is kernels only
        mixed = self._mixed
        if self._graphs is not None and self.capture is None and graph_ok:
            return self._graphed((mixed,), lambda *a: self._forward_impl(*a, mixed=mixed),
                                 masked_frames.float().contiguous(), flows.float().contiguous(), masks.float().contiguous())
        return self._forward_impl(masked_frames, flows, masks, mixed=mixed)

    def _forward_impl(self, masked_frames, flows, masks, mixed=False):
        dev = masked_frames.device
        b, t, c, H, W = masked_frames.shape
        bt = b * t
        fs = getattr(self, "_fshard", None)
        if fs is not None and (b != 1 or t != fs["counts"][fs["rank"]]):
            raise ValueError(f"frame sharding: rank {fs['rank']} expects [1, {fs['counts'][fs['rank']]}, ...] frames "
                             f"of the {fs['T']}-frame window, got [{b}, {t}, ...]")
        if fs is not None and fs["exchange"] == "p2p":
            fs["layer"] = 0
            fs["peer"].barrier()  # every peer has finished reading the exchange buffers of the previous forward
        P = self._packed.get(mixed) or self._pack(dev, mixed)
        g = self._geometry(b, t, H, W, dev, mixed)
        B = lambda name, shape, dtype=torch.float32: self._buf(g, name, shape, dev, dtype)  # noqa: E731
        A = lambda name, shape: self._buf(g, name, shape, dev, g.a16)  # noqa: E731
        frames = masked_frames.reshape(bt, c, H, W).float().contiguous()
        mk = masks.reshape(bt, 1, H, W).float().contiguous()
        fl = flows.reshape(bt, flows.shape[2], H, W).float().contiguous()
        H2, W2, OH, OW = H // 2, W // 2, g.OH, g.OW

        # ---- frame encoder (model.py:53-66)
        lib._scope[1:] = ["encoder"]  # module labels for the per-launch profiler (bench.py "modules")
        incol = A("in_col", (bt, H2, W2, 64))
        lib.im2col_nchw(frames, mk, incol, k=3, stride=2, pad=1, replicate=False, OH=H2, OW=W2, tag="enc0")
        e0 = A("e0", (bt, H2, W2, 64))
        e2 = A("e2", (bt, H2, W2, 64))
        e4 = A("e4", (bt, OH, OW, 128))
        x0 = A("e6", (bt, OH, OW, 256))
        e8 = A("e8", (bt, OH, OW, 384))
        e10 = A("e10", (bt, OH, OW, 512))
        e12 = A("e12", (bt, OH, OW, 384))
        e14 = A("e14", (bt, OH, OW, 256))
        enc = A("enc", (bt, OH, OW, 128))
        enc_f = B("enc_f", (bt, OH, OW, 128))
        k3 = dict(kx=3, ky=3, pad_x=1, pad_y=1)
        linear([(incol, 64)], P["enc0"], bt * H2 * W2, act=lib.ACT_LEAKY02, out_split=e0)
        conv([(e0, 64)], P["enc2"], out_split=e2, **k3)
        conv([(e2, 64)], P["enc4"], stride=2, out_split=e4, **k3)
        conv([(e4, 128)], P["enc6"], out_split=x0, **k3)
        conv([(x0, 256)], P["enc8"], out_split=e8, **k3)
        conv([(x0, 256), (e8, 384)], P["enc10"], out_split=e10, groups=2, seg_counts=[128, 192], **k3)
        conv([(x0, 256), (e10, 512)], P["enc12"], out_split=e12, groups=4, seg_counts=[64, 128], **k3)
        conv([(x0, 256), (e12, 384)], P["enc14"], out_split=e14, groups=2, seg_counts=[128, 192],
             alg_k=9 * (32 + 48), **k3)  # roofline accounting: the reference's 8-group conv
        conv([(x0, 256), (e14, 256)], P["enc16"], out_split=enc, out_f32=enc_f, seg_counts=[256, 256], **k3)
        # ---- flow encoder (model.py:206-212): fp16 weights and activations in both precisions (see _pack)
        lib._scope[-1] = "flow_encoder"
        fcol = B("f_col", (bt, H, W, 64), torch.float16)
        lib.im2col_nchw(fl, None, fcol, k=5, stride=1, pad=2, replicate=True, OH=H, OW=W, tag="fenc1")
        f1 = B("f1", (bt, H, W, 64), torch.float16)
        f2 = B("f2", (bt, H2, W2, 128), torch.float16)
        f3 = B("f3", (bt, H2, W2, 128), torch.float16)
        f4 = B("f4", (bt, OH, OW, 128), torch.float16)
        linear([(fcol, 64)], P["fenc1"], bt * H * W, act=lib.ACT_LEAKY02, out_split=f1)
        conv([(f1, 64)], P["fenc2"], stride=2, out_split=f2, **k3)
        conv([(f2, 128)], P["fenc3"], out_split=f3, **k3)
        conv([(f3, 128)], P["fenc4"], stride=2, out_split=f4, **k3)
        # ---- patch embedding (model.py:261-262,270-271): conv output NHWC == token-major
        lib._scope[-1] = "patch_embed"
        rows = bt * g.n
        xa = B("x_a", (rows, self.d))
        xb = B("x_b", (rows, self.d))
        xs = A("x_s", (rows, self.d))
        f = B("f", (rows, self.df))
        fs = A("f_s", (rows, self.df))
        k, s, p = self.ksz[0], self.stride[0], self.padding[0]
        kp = dict(kx=k, ky=k, stride=s, pad_x=p, pad_y=p, act=lib.ACT_NONE)
        conv([(enc, 128)], P["patch2vec"], out_f32=xa, **kp)
        conv([(f4, 128)], P["f_patch2vec"], out_f32=f, out_split=fs, **kp)
        self._cap("enc", enc_f)
        self._cap("tok0", xa)
        self._cap("ftok", f)
        # ---- transformer (model.py:272-277)
        lib._scope[-1] = "pos_emb"
        self._temporal(g, P, "t0", xa, xs, dev, need_split=False)   # the positional embedding re-creates the split copy
        self._cap("t0", xa)
        lib.dwconv3x3_res(xa, bt, g.h, g.w, self.d, P["pos_w"], P["pos_b"], xb, xs)
        x = xb
        nb = len(self.transformer)
        self._spatial(g, P, "s0", x, xs, f, fs, dev, need_split=nb == 0)   # a temporal block follows: it reads fp32 x
        self._cap("s0", x)
        for i in range(nb):
            self._temporal(g, P, f"t{i + 1}", x, xs, dev)                  # the spatial block's gate GEMM reads xs
            self._spatial(g, P, f"s{i + 1}", x, xs, f, fs, dev, need_split=i == nb - 1)   # last: vec2patch reads xs
        self._cap("tok_final", x)
        # ---- vec2patch + skip (model.py:278-279)
        lib._scope[-1] = "vec2patch"
        v2p = B("v2p", (rows, k * k * self.cnum * 2))
        feat = A("feat", (bt, OH, OW, self.cnum * 2))
        linear([(xs, self.d)], P["vec2patch"], rows, out_f32=v2p)
        lib.fold(v2p, bt, g.h, g.w, self.cnum * 2, k, k, s, p, OH, OW, normalize=False, add=enc_f, out_split=feat)
        # ---- decoder (model.py:188-193,281-282)
        lib._scope[-1] = "decoder"
        c2 = self.cnum * 2
        d1 = A("d1", (bt, H2, W2, c2))
        d2 = A("d2", (bt, H2, W2, c2 // 2))
        d3 = A("d3", (bt, H, W, c2 // 2))
        out = torch.empty(bt, 3, H, W, device=dev, dtype=torch.float32)
        self._deconv(feat, c2, P, "dec1", d1)
        conv([(d1, c2)], P["dec2"], out_split=d2, **k3)
        self._deconv(d2, c2 // 2, P, "dec3", d3)
        # final 64 -> 3 conv + tanh: taps-as-N tensor-core GEMM and the 9-tap sum in one kernel (no HBM intermediate)
        lib.conv_tail(d3, bt, H, W, c2 // 2, P["dec4"]["w"], 3, P["dec4"]["b"], lib.ACT_TANH, out, nchw=True, tag="dec4")
        lib._scope[1:] = []
        return out


class Model(nn.Module):
    """Same constructor/forward as FGT.models.model.Model (model.py:12-25)."""

    def __init__(self, config):
        super().__init__()
        self.net = FGT(config['tw'], config['sw'], config['gd'], config['input_resolution'], config['in_channel'],
                       config['cnum'], config['flow_inChannel'], config['flow_cnum'], config['frame_hidden'],
                       config['flow_hidden'], config['PASSMASK'], config['numBlocks'], config['kernel_size'],
                       config['stride'], config['padding'], config['num_head'], config['conv_type'], config['norm'],
                       config['use_bias'], config['ape'], config['mlp_ratio'], config['drop'], config['init_weights'])

    def forward(self, frames, flows, masks):
        return self.net(frames, flows, masks)
