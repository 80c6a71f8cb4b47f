"""H100-native single-frame ("2D") LAFC behind the reference's nn.Module interface.

Drop-in for /root/reference/FGT/models/lafc_single.py, the flow-completion network FGT's validation
(FGT/networks/network.py:258-352) runs before the transformer: `Model(config).forward(flows, masks, edges=None)`
-> (flow [n,2,H,W], edge [n,1,H,W]) with the same constructor dict and state_dict keys. Every frame is completed on
its own, so the n frames of a call are the batch of every launch. The nn.Modules only hold parameters; every
convolution runs on the wgmma implicit-GEMM engine (the replicate-padded 5x5 input conv through the im2col gather of
[flow | mask], dilated convs as tap offsets, skip concatenations as K-segments), the nearest x2 upsampling on the
helper kernel. fp32 only (split-bf16 operands, 3-term MMAs): the validation it serves has no autocast mode.

Reference quirks kept: the last decoder conv (24 -> 2 channels) keeps VanillaConv's default LeakyReLU(0.2), so the
completed flow is leaky-rectified; the edge head adds its projection back before a LeakyReLU of slope 0.01.
"""
import torch
import torch.nn as nn

from . import lib, ops
from .graphs import NativeNet, workspace
from .lafc_model import _C2, _D2, _Edge


class _Res(nn.Module):
    """ResidualBlock_noBN (FGT/models/utils/reconstructionLayers.py:34-61): bare nn.Conv2d keys."""

    def __init__(self, nf):
        super().__init__()
        self.conv1 = nn.Conv2d(nf, nf, 3, padding=1)
        self.conv2 = nn.Conv2d(nf, nf, 3, padding=1)


class P3DNet(NativeNet):
    def __init__(self, num_flows, num_feats, in_channels, passmask, use_residual, res_blocks, use_bias, conv_type,
                 init_weights):
        super().__init__()
        if conv_type != 'vanilla' or not passmask or not use_bias:
            raise ValueError("fgt_b200 2D LAFC implements conv_type='vanilla', PASSMASK=1, use_bias=1 (shipped config)")
        if in_channels != 3:
            raise ValueError("fgt_b200 2D LAFC expects flow(2)+mask(1) input channels")
        c = num_feats
        if c % 2:
            raise ValueError("fgt_b200 2D LAFC expects an even cnum")
        self.c, self.resNums = c, res_blocks
        self.encoder2 = nn.Sequential(nn.ReplicationPad2d(2), _C2(in_channels, c, 5), _C2(c, 2 * c, 3))
        self.encoder4 = nn.Sequential(_C2(2 * c, 2 * c, 3), _C2(2 * c, 4 * c, 3))
        self.res_blocks = nn.Sequential(*[_Res(4 * c) for _ in range(res_blocks)])
        self.middle = nn.Sequential(*[_C2(4 * c, 4 * c, 3) for _ in range(4)])
        self.decoder2 = nn.Sequential(_D2(8 * c, 2 * c, 3), _C2(2 * c, 2 * c, 3), _C2(2 * c, 2 * c, 3))
        self.decoder = nn.Sequential(_D2(4 * c, c, 3), _C2(c, c // 2, 3), _C2(c // 2, 2, 3))
        self.edgeDetector = _Edge()
        if init_weights:
            for m in self.modules():  # BaseNetwork.init_weights('normal', 0.02), FGT/models/BaseNetwork.py:20-46
                if isinstance(m, nn.Conv2d):
                    nn.init.normal_(m.weight.data, 0.0, 0.02)
                    nn.init.constant_(m.bias.data, 0.0)

    def _pack(self, dev):
        sd = {k: v.detach().float() for k, v in self.state_dict().items()}
        c = self.c
        P = {}

        def put(name, key, segs=None, im2col=None):
            P[name] = ops.packed(name, sd[key + ".weight"], sd[key + ".bias"], dev, segs, im2col)

        put("e2a", "encoder2.1.featureConv", im2col=128)   # 5x5x3 = 75 gathered inputs per row
        put("e2b", "encoder2.2.featureConv")
        put("e4a", "encoder4.0.featureConv")
        put("e4b", "encoder4.1.featureConv")
        for i in range(self.resNums):
            put(f"res{i}_1", f"res_blocks.{i}.conv1")
            put(f"res{i}_2", f"res_blocks.{i}.conv2")
        for i in range(4):
            put(f"mid{i}", f"middle.{i}.featureConv")
        put("dec2_0", "decoder2.0.conv.featureConv", [4 * c, 4 * c])
        put("dec2_1", "decoder2.1.featureConv")
        put("dec2_2", "decoder2.2.featureConv")
        put("dec_0", "decoder.0.conv.featureConv", [2 * c, 2 * c])
        put("dec_1", "decoder.1.featureConv")
        put("dec_2", "decoder.2.featureConv")
        put("edge_p", "edgeDetector.projection.featureConv", im2col=64)
        put("edge_1", "edgeDetector.mid_layer_1.featureConv")
        put("edge_2", "edgeDetector.mid_layer_2.featureConv")
        put("edge_o", "edgeDetector.out_layer.featureConv")
        self._packed[False] = P
        return P

    def forward(self, flows, masks, edges=None):
        if edges is not None:
            raise ValueError("fgt_b200 2D LAFC: the `edges` input is not implemented (FGT's validation passes None)")
        if not flows.is_cuda:
            raise RuntimeError("fgt_b200 2D LAFC runs on a CUDA (sm_90a) device only; there is no CPU fallback")
        flows, masks = flows.float().contiguous(), masks.float().contiguous()
        if self._graphs is not None:
            return self._graphed((), self._forward_impl, flows, masks)
        return self._forward_impl(flows, masks)

    def _forward_impl(self, flows, masks):
        """flows [n,2,H,W], masks [n,1,H,W] fp32 contiguous -> (flow [n,2,H,W], edge [n,1,H,W]);
        P3DNet.forward, lafc_single.py:70-89."""
        n, cf, H, W = flows.shape
        if cf != 2 or tuple(masks.shape) != (n, 1, H, W):
            raise ValueError(f"2D LAFC inputs: flows [n,2,H,W] and masks [n,1,H,W], got {tuple(flows.shape)} and "
                             f"{tuple(masks.shape)}")
        if H % 4 or W % 4:
            raise ValueError(f"2D LAFC input {H}x{W}: H and W must be divisible by 4 (the skip concatenations)")
        dev = flows.device
        P = self._packed.get(False) or self._pack(dev)
        c = self.c
        H2, W2, H4, W4 = H // 2, W // 2, H // 4, W // 4
        bufs = self._geo.setdefault((n, H, W), {})
        B = lambda name, s, split=True: workspace(bufs, name, s, dev, torch.bfloat16 if split else torch.float32)  # noqa: E731
        conv3 = lambda *a, **k: ops.conv(*a, kx=3, ky=3, **k)  # noqa: E731
        L = lib.ACT_LEAKY02
        # encoder2 (lafc_single.py:26-30): ReplicationPad2d(2) + 5x5 conv through the im2col gather, stride-2 conv
        col = B("col", (n, H, W, 128))
        lib.im2col_nchw(flows, masks, col, k=5, stride=1, pad=2, replicate=True, OH=H, OW=W, tag="e2a")
        a1 = B("a1", (n, H, W, c))
        ops.linear([(lib.view16(col, n * H * W, 128), 128)], P["e2a"], n * H * W, act=L, out_split=a1)
        e2 = B("e2", (n, H2, W2, 2 * c))
        conv3([(a1, c)], P["e2b"], stride=2, pad_x=1, pad_y=1, out_split=e2)
        # encoder4 (:31-35)
        t1 = B("t1", (n, H2, W2, 2 * c))
        conv3([(e2, 2 * c)], P["e4a"], pad_x=1, pad_y=1, out_split=t1)
        e4 = B("e4", (n, H4, W4, 4 * c))
        e4f = B("e4f", (n, H4, W4, 4 * c), split=False) if self.resNums else None
        conv3([(t1, 2 * c)], P["e4b"], stride=2, pad_x=1, pad_y=1, out_split=e4, out_f32=e4f)
        # residual blocks without BN (:36-38, 79-82): conv, LeakyReLU(0.2), conv, + identity in fp32, no activation
        src, srcf = e4, e4f
        t3 = B("t3", (n, H4, W4, 4 * c))
        for i in range(self.resNums):
            last = i == self.resNums - 1
            r = B(f"r{i % 2}", (n, H4, W4, 4 * c))
            rf = None if last else B(f"r{i % 2}f", (n, H4, W4, 4 * c), split=False)
            conv3([(src, 4 * c)], P[f"res{i}_1"], pad_x=1, pad_y=1, out_split=t3)
            conv3([(t3, 4 * c)], P[f"res{i}_2"], pad_x=1, pad_y=1, act=lib.ACT_NONE, aux=srcf, aux_mode=lib.AUX_ADD,
                  out_split=r, out_f32=rf)
            src, srcf = r, rf
        # dilated middle (:40-49)
        y = (B("y0", (n, H4, W4, 4 * c)), B("y1", (n, H4, W4, 4 * c)))
        for i, d in enumerate((8, 4, 2, 1)):
            conv3([(src, 4 * c)], P[f"mid{i}"], dil=d, pad_x=d, pad_y=d, out_split=y[i % 2])
            src = y[i % 2]
        # decoder2 (:50-57, 84-85): nearest x2 of [middle ; e4] then conv
        u1 = B("u1", (n, H2, W2, 4 * c))
        u2 = B("u2", (n, H2, W2, 4 * c))
        lib.upsample2x(src, n, H4, W4, 4 * c, u1)
        lib.upsample2x(e4, n, H4, W4, 4 * c, u2)
        d20 = B("d20", (n, H2, W2, 2 * c))
        d21 = B("d21", (n, H2, W2, 2 * c))
        conv3([(u1, 4 * c), (u2, 4 * c)], P["dec2_0"], pad_x=1, pad_y=1, out_split=d20, seg_counts=[4 * c, 4 * c])
        conv3([(d20, 2 * c)], P["dec2_1"], pad_x=1, pad_y=1, out_split=d21)
        conv3([(d21, 2 * c)], P["dec2_2"], pad_x=1, pad_y=1, out_split=d20)
        # decoder (:58-65, 86-87): nearest x2 of [decoder2 ; e2], then conv, conv, and the 24 -> 2 conv whose
        # LeakyReLU(0.2) the reference keeps
        u3 = B("u3", (n, H, W, 2 * c))
        u4 = B("u4", (n, H, W, 2 * c))
        lib.upsample2x(d20, n, H2, W2, 2 * c, u3)
        lib.upsample2x(e2, n, H2, W2, 2 * c, u4)
        d0 = B("d0", (n, H, W, c))
        d1 = B("d1", (n, H, W, c // 2))
        conv3([(u3, 2 * c), (u4, 2 * c)], P["dec_0"], pad_x=1, pad_y=1, out_split=d0, seg_counts=[2 * c, 2 * c])
        conv3([(d0, c)], P["dec_1"], pad_x=1, pad_y=1, out_split=d1)
        flow = torch.empty(n, 2, H, W, device=dev, dtype=torch.float32)
        conv3([(d1, c // 2)], P["dec_2"], pad_x=1, pad_y=1, act=L, out_f32=flow, nchw_out=True)
        # edge head (:92-112)
        ecol = B("ecol", (n, H, W, 64))
        lib.im2col_nchw(flow, None, ecol, k=3, stride=1, pad=1, replicate=False, OH=H, OW=W, tag="edge_p")
        ep = B("ep", (n, H, W, 16))
        epf = B("epf", (n, H, W, 16), split=False)
        ops.linear([(lib.view16(ecol, n * H * W, 64), 64)], P["edge_p"], n * H * W, act=L, out_split=ep, out_f32=epf)
        e1 = B("e1", (n, H, W, 16))
        e2_ = B("e2_", (n, H, W, 16))
        conv3([(ep, 16)], P["edge_1"], pad_x=1, pad_y=1, out_split=e1)
        conv3([(e1, 16)], P["edge_2"], pad_x=1, pad_y=1, act=lib.ACT_LEAKY001, aux=epf, aux_mode=lib.AUX_ADD_PRE,
              out_split=e2_)
        edge = torch.empty(n, 1, H, W, device=dev, dtype=torch.float32)
        ops.conv([(e2_, 16)], P["edge_o"], act=lib.ACT_SIGMOID, out_f32=edge, nchw_out=True)
        return flow, edge


class Model(nn.Module):
    """Same constructor/forward as FGT.models.lafc_single.Model (lafc_single.py:9-18)."""

    def __init__(self, config):
        super().__init__()
        self.net = P3DNet(config['num_flows'], config['cnum'], config['in_channel'], config['PASSMASK'],
                          config['use_residual'], config['resBlocks'], config['use_bias'], config['conv_type'],
                          config['init_weights'])

    def forward(self, flows, masks, edges=None):
        return self.net(flows, masks, edges)
