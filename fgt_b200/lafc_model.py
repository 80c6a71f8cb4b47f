"""H100-native LAFC flow-completion network behind the reference's nn.Module interface.

Drop-in for /root/reference/LAFC/models/lafc.py: `Model(config).forward(flows, masks, edges=None)`
-> (flow [b,2,H,W], edge [b,1,H,W]) with the same constructor dict and state_dict keys
(tool/video_inpainting.py:200-214, call site :378). The nn.Modules only hold parameters; every
convolution runs on the wgmma implicit-GEMM engine (P3D (1,k,k) convs as per-frame 2-D taps,
(3,1,1) temporal convs as z-taps with TMA zero fill, dilated convs as tap offsets, skip concats as
K-segments), the input gather and nearest upsampling on HBM-bound helper kernels. No CPU fallback.

Opt-in mixed precision (`P3DNet.enable_mixed_precision()`): the reference module under
torch.autocast("cuda", dtype=torch.float16), with every conv a 1-term fp16 GEMM (oracle/lafc_mixed_oracle.py is the
definition; DESIGN.md section 2 the rounding points).
"""
import torch
import torch.nn as nn

from . import lib, ops
from .graphs import NativeNet, workspace


class _C3(nn.Module):
    def __init__(self, ci, co, k):
        super().__init__()
        self.featureConv = nn.Conv3d(ci, co, k)


class _C2(nn.Module):
    def __init__(self, ci, co, k):
        super().__init__()
        self.featureConv = nn.Conv2d(ci, co, k)


class _D2(nn.Module):
    def __init__(self, ci, co, k):
        super().__init__()
        self.conv = _C2(ci, co, k)


class _P3D(nn.Module):
    def __init__(self, ci, co, k):
        super().__init__()
        self.conv1 = _C3(ci, co, (1, k, k))
        self.conv2 = _C3(co, co, (3, 1, 1))


class _Edge(nn.Module):
    def __init__(self, mid=16):
        super().__init__()
        self.projection = _C2(2, mid, 3)
        self.mid_layer_1 = _C2(mid, mid, 3)
        self.mid_layer_2 = _C2(mid, mid, 3)
        self.out_layer = _C2(mid, 1, 1)


class P3DNet(NativeNet):
    def __init__(self, num_flows, num_feats, in_channels, passmask, use_residual, res_blocks, use_bias, conv_type,
                 init_weights):
        super().__init__()
        if conv_type != 'vanilla' or not passmask or not use_bias:
            raise ValueError("fgt_b200 LAFC implements conv_type='vanilla', PASSMASK=1, use_bias=1 (shipped config)")
        if in_channels != 3:
            raise ValueError("fgt_b200 LAFC expects flows(2)+mask(1) input channels")
        c = num_feats
        self.c, self.T, self.use_residual, self.resNums = c, num_flows, use_residual, res_blocks
        self._mixed = False
        self.encoder2 = nn.Sequential(nn.ReplicationPad3d((2, 2, 2, 2, 0, 0)), _P3D(in_channels, c, 5), _P3D(c, 2 * c, 3))
        self.encoder4 = nn.Sequential(_P3D(2 * c, 2 * c, 3), _P3D(2 * c, 4 * c, 3))
        base = _P3D(4 * c, 4 * c, 3)
        self.res_blocks = nn.Sequential(*[base for _ in range(res_blocks)])
        self.condense2 = _C3(2 * c, 2 * c, (num_flows, 1, 1))
        self.condense4_pre = _C3(4 * c, 4 * c, (num_flows, 1, 1))
        self.condense4_post = _C3(4 * c, 4 * c, (num_flows, 1, 1))
        self.middle = nn.Sequential(*[_C2(4 * c, 4 * c, 3) for _ in range(4)])
        self.decoder2 = nn.Sequential(_D2(8 * c, 2 * c, 3), _C2(2 * c, 2 * c, 3), _C2(2 * c, 2 * c, 3))
        self.decoder = nn.Sequential(_D2(4 * c, c, 3), _C2(c, c // 2, 3), _C2(c // 2, 2, 3))
        self.edgeDetector = _Edge()
        if init_weights:
            for m in self.modules():  # BaseNetwork.init_weights('kaiming'), LAFC/models/BaseNetwork.py:25-51
                if isinstance(m, (nn.Conv2d, nn.Conv3d)):
                    nn.init.kaiming_normal_(m.weight.data, a=0, mode='fan_in')
                    nn.init.constant_(m.bias.data, 0.0)

    def _pack(self, dev, half=False):
        """half: the mixed-precision set, every conv a 1-term fp16 layer whose weight and bias are rounded to fp16 once
        (autocast's casts of the conv's parameters)."""
        sd = {k: v.detach().float() for k, v in self.state_dict().items()}
        if half:
            sd = {k: v.half().float() for k, v in sd.items()}
        c = self.c
        P = {}

        def put(name, key, segs=None, im2col=None):
            P[name] = ops.packed(name, sd[key + ".featureConv.weight"], sd[key + ".featureConv.bias"], dev, segs, im2col,
                                 half=half)

        w = sd["encoder2.1.conv1.featureConv.weight"]  # [c,3,1,5,5] -> 2-D filter for the im2col path
        P["e2a1"] = ops.packed("e2a1", w[:, :, 0], sd["encoder2.1.conv1.featureConv.bias"], dev, im2col_pad=128,
                               half=half)
        put("e2a2", "encoder2.1.conv2")
        put("e2b1", "encoder2.2.conv1")
        put("e2b2", "encoder2.2.conv2")
        put("e4a1", "encoder4.0.conv1")
        put("e4a2", "encoder4.0.conv2")
        put("e4b1", "encoder4.1.conv1")
        put("e4b2", "encoder4.1.conv2")
        if self.resNums > 0:
            put("res1", "res_blocks.0.conv1")
            put("res2", "res_blocks.0.conv2")
        put("cond2", "condense2")
        put("cond4pre", "condense4_pre")
        put("cond4post", "condense4_post")
        for i in range(4):
            put(f"mid{i}", f"middle.{i}")
        put("dec2_0", "decoder2.0.conv", [4 * c, 4 * c])
        put("dec2_1", "decoder2.1")
        put("dec2_2", "decoder2.2")
        put("dec_0", "decoder.0.conv", [2 * c, 2 * c])
        put("dec_1", "decoder.1")
        put("dec_2", "decoder.2")
        put("edge_p", "edgeDetector.projection", im2col=64)
        put("edge_1", "edgeDetector.mid_layer_1")
        put("edge_2", "edgeDetector.mid_layer_2")
        put("edge_o", "edgeDetector.out_layer")
        self._packed[half] = P
        return P

    def _forward_one(self, x, P, dev, mixed=False):
        """x: [T, 3, H, W] fp32 (flows + mask per candidate frame) -> (flow [2,H,W], edge [1,H,W]). mixed: fp16
        activation buffers, fp16 packed weights P, and every GEMM rounds where autocast makes an fp16 tensor."""
        T, _, H, W = x.shape
        c = self.c
        H2, W2, H4, W4 = H // 2, W // 2, H // 4, W // 4
        bufs = self._geo.setdefault((T, H, W, mixed), {})
        a16 = torch.float16 if mixed else torch.bfloat16  # 16-bit activations: fp16 (mixed) or split-bf16
        B = lambda n, s, split=True: workspace(bufs, n, s, dev, a16 if split else torch.float32)  # noqa: E731
        conv = (lambda *a, **k: ops.conv(*a, autocast=True, **k)) if mixed else ops.conv  # noqa: E731
        linear = (lambda *a, **k: ops.linear(*a, autocast=True, **k)) if mixed else ops.linear  # noqa: E731
        L = lib.ACT_LEAKY02
        # encoder2 (lafc.py:23-30): ReplicationPad + (1,5,5) conv via im2col, then the (3,1,1) conv
        col = B("col", (T, H, W, 128))
        lib.im2col_nchw(x, None, col, k=5, stride=1, pad=2, replicate=True, OH=H, OW=W, tag="e2a1")
        a1 = B("a1", (T, H, W, c))
        linear([(lib.view16(col, T * H * W, 128), 128)], P["e2a1"], T * H * W, act=L, out_split=a1)
        a2 = B("a2", (T, H, W, c))
        conv([(a1, c)], P["e2a2"], kz=3, pad_z=1, out_split=a2)
        a3 = B("a3", (T, H2, W2, 2 * c))
        conv([(a2, c)], P["e2b1"], kx=3, ky=3, stride=2, pad_x=1, pad_y=1, out_split=a3)
        e2 = B("e2", (T, H2, W2, 2 * c))
        e2f = B("e2f", (T, H2, W2, 2 * c), split=False)
        conv([(a3, 2 * c)], P["e2b2"], kz=3, pad_z=1, out_split=e2, out_f32=e2f)
        ce2 = B("ce2", (1, H2, W2, 2 * c))
        conv([(e2, 2 * c)], P["cond2"], kz=T, pad_z=0, out_z=1, out_split=ce2)
        # encoder4 (lafc.py:31-36)
        t1 = B("t1", (T, H2, W2, 2 * c))
        conv([(e2, 2 * c)], P["e4a1"], kx=3, ky=3, pad_x=1, pad_y=1, out_split=t1)
        e4a = B("e4a", (T, H2, W2, 2 * c))
        if self.use_residual:
            conv([(t1, 2 * c)], P["e4a2"], kz=3, pad_z=1, out_split=e4a, aux=e2f, aux_mode=lib.AUX_ADD)
        else:
            conv([(t1, 2 * c)], P["e4a2"], kz=3, pad_z=1, out_split=e4a)
        t2 = B("t2", (T, H4, W4, 4 * c))
        conv([(e4a, 2 * c)], P["e4b1"], kx=3, ky=3, stride=2, pad_x=1, pad_y=1, out_split=t2)
        e4 = B("e4", (T, H4, W4, 4 * c))
        e4f = B("e4f", (T, H4, W4, 4 * c), split=False)
        conv([(t2, 4 * c)], P["e4b2"], kz=3, pad_z=1, out_split=e4, out_f32=e4f)
        ce4 = B("ce4", (1, H4, W4, 4 * c))
        conv([(e4, 4 * c)], P["cond4pre"], kz=T, pad_z=0, out_z=1, out_split=ce4)
        # residual blocks: one shared block applied resNums times (lafc.py:38-43,94-95)
        t3 = B("t3", (T, H4, W4, 4 * c))
        for _ in range(self.resNums):
            conv([(e4, 4 * c)], P["res1"], kx=3, ky=3, pad_x=1, pad_y=1, out_split=t3)
            conv([(t3, 4 * c)], P["res2"], kz=3, pad_z=1, out_split=e4, out_f32=e4f, aux=e4f, aux_mode=lib.AUX_ADD)
        y0 = B("y0", (1, H4, W4, 4 * c))
        y1 = B("y1", (1, H4, W4, 4 * c))
        conv([(e4, 4 * c)], P["cond4post"], kz=T, pad_z=0, out_z=1, out_split=y0)
        # dilated middle (lafc.py:54-63)
        src, dst = y0, y1
        for i, d in enumerate((8, 4, 2, 1)):
            conv([(src, 4 * c)], P[f"mid{i}"], kx=3, ky=3, dil=d, pad_x=d, pad_y=d, out_split=dst)
            src, dst = dst, src
        # decoder2 (lafc.py:64-71): nearest x2 of [filled ; pre] then conv
        u1 = B("u1", (1, H2, W2, 4 * c))
        u2 = B("u2", (1, H2, W2, 4 * c))
        lib.upsample2x(src, 1, H4, W4, 4 * c, u1)
        lib.upsample2x(ce4, 1, H4, W4, 4 * c, u2)
        d20 = B("d20", (1, H2, W2, 2 * c))
        d21 = B("d21", (1, H2, W2, 2 * c))
        conv([(u1, 4 * c), (u2, 4 * c)], P["dec2_0"], kx=3, ky=3, pad_x=1, pad_y=1, out_split=d20,
             seg_counts=[4 * c, 4 * c])
        conv([(d20, 2 * c)], P["dec2_1"], kx=3, ky=3, pad_x=1, pad_y=1, out_split=d21)
        conv([(d21, 2 * c)], P["dec2_2"], kx=3, ky=3, pad_x=1, pad_y=1, out_split=d20)
        # decoder (lafc.py:72-79)
        u3 = B("u3", (1, H, W, 2 * c))
        u4 = B("u4", (1, H, W, 2 * c))
        lib.upsample2x(d20, 1, H2, W2, 2 * c, u3)
        lib.upsample2x(ce2, 1, H2, W2, 2 * c, u4)
        d0 = B("d0", (1, H, W, c))
        d1 = B("d1", (1, H, W, c // 2))
        conv([(u3, 2 * c), (u4, 2 * c)], P["dec_0"], kx=3, ky=3, pad_x=1, pad_y=1, out_split=d0,
             seg_counts=[2 * c, 2 * c])
        conv([(d0, c)], P["dec_1"], kx=3, ky=3, pad_x=1, pad_y=1, out_split=d1)
        flow = torch.empty(1, 2, H, W, device=dev, dtype=torch.float32)
        conv([(d1, c // 2)], P["dec_2"], kx=3, ky=3, pad_x=1, pad_y=1, act=lib.ACT_NONE, out_f32=flow, nchw_out=True)
        # edge head (lafc.py:141-148)
        ecol = B("ecol", (1, H, W, 64))
        lib.im2col_nchw(flow, None, ecol, k=3, stride=1, pad=1, replicate=False, OH=H, OW=W, tag="edge_p")
        ep = B("ep", (1, H, W, 16))
        epf = B("epf", (1, H, W, 16), split=False)
        linear([(lib.view16(ecol, H * W, 64), 64)], P["edge_p"], H * W, act=L, out_split=ep, out_f32=epf)
        e1 = B("e1", (1, H, W, 16))
        e2_ = B("e2_", (1, H, W, 16))
        conv([(ep, 16)], P["edge_1"], kx=3, ky=3, pad_x=1, pad_y=1, out_split=e1)
        conv([(e1, 16)], P["edge_2"], kx=3, ky=3, pad_x=1, pad_y=1, act=lib.ACT_LEAKY001, aux=epf,
             aux_mode=lib.AUX_ADD_PRE, out_split=e2_)
        edge = torch.empty(1, 1, H, W, device=dev, dtype=torch.float32)
        conv([(e2_, 16)], P["edge_o"], act=lib.ACT_SIGMOID, out_f32=edge, nchw_out=True)
        return flow, edge

    def enable_mixed_precision(self, on=True):
        """Mixed precision, opt-in: the network runs as the reference does under
        torch.autocast("cuda", dtype=torch.float16). Every conv is a 1-term fp16 tensor-core GEMM (fp16 weights, biases
        and activation rows, fp32 accumulation) that rounds to fp16 wherever autocast makes an fp16 tensor. Autocast's
        outputs are fp16; these stay fp32 tensors holding the fp16-rounded values, so callers keep their dtypes. The
        fp16 weights, workspaces and CUDA graphs are kept apart from the fp32 path's, so the flag may change between
        calls; off (the default) gives the fp32 path's outputs bit for bit. DESIGN.md section 2 lists where the
        rounding points differ from autocast."""
        self._mixed = bool(on)

    def forward(self, flows, masks, edges=None):
        if edges is not None:
            raise ValueError("fgt_b200 LAFC: the `edges` input is unused by the shipped driver (always None)")
        if not flows.is_cuda:
            raise RuntimeError("fgt_b200 LAFC runs on a CUDA (sm_90a) device only; there is no CPU fallback")
        mixed = self._mixed
        if self._graphs is not None:
            fn = (lambda *a: self._forward_impl(*a, mixed=True)) if mixed else self._forward_impl
            return self._graphed((True,) if mixed else (), fn, flows.float().contiguous(), masks.float().contiguous())
        return self._forward_impl(flows, masks, mixed=mixed)

    def _forward_impl(self, flows, masks, mixed=False):
        b, _, T, H, W = flows.shape
        if T != self.T or H % 4 or W % 4:
            raise ValueError(f"LAFC input [T={T},{H}x{W}]: T must be {self.T} and H, W divisible by 4")
        dev = flows.device
        P = self._packed.get(mixed) or self._pack(dev, mixed)
        x = torch.cat([flows.float(), masks.float()], 1).permute(0, 2, 1, 3, 4).contiguous()  # [b,T,3,H,W]
        outs = [self._forward_one(x[i], P, dev, mixed) for i in range(b)]
        return torch.cat([o[0] for o in outs], 0), torch.cat([o[1] for o in outs], 0)


class Model(nn.Module):
    """Same constructor/forward as LAFC.models.lafc.Model (lafc.py:6-15)."""

    def __init__(self, config):
        super().__init__()
        self.net = P3DNet(config['num_flows'], config['cnum'], config['in_channel'], config['PASSMASK'],
                          config['use_residual'], config['resBlocks'], config['use_bias'], config['conv_type'],
                          config['init_weights'])

    def forward(self, flows, masks, edges=None):
        return self.net(flows, masks, edges)
