"""H100-native single-frame ("2D") LAFC behind the reference's nn.Module interface.

Drop-in for /root/reference/FGT/models/lafc_single.py, the flow-completion network FGT's validation
(FGT/networks/network.py:258-352) runs before the transformer: `Model(config).forward(flows, masks, edges=None)`
-> (flow [n,2,H,W], edge [n,1,H,W]) with the same constructor dict and state_dict keys. Every frame is completed on
its own, so the n frames of a call are the batch of every launch. The nn.Modules only hold parameters; every
convolution runs on the wgmma implicit-GEMM engine (the replicate-padded 5x5 input conv through the im2col gather of
[flow | mask], dilated convs as tap offsets, skip concatenations as K-segments), the nearest x2 upsampling on the
helper kernel. fp32 only (split-bf16 operands, 3-term MMAs): the validation it serves has no autocast mode. The
network after the residual blocks, `forward` and the weight packing are lafc_model._LAFCBase's.

Reference quirks kept: the last decoder conv (24 -> 2 channels) keeps VanillaConv's default LeakyReLU(0.2), so the
completed flow is leaky-rectified; the edge head adds its projection back before a LeakyReLU of slope 0.01.
"""
import torch.nn as nn

from . import lib, ops
from .lafc_model import C3, _C2, _LAFCBase


class _Res(nn.Module):
    """ResidualBlock_noBN (FGT/models/utils/reconstructionLayers.py:34-61): bare nn.Conv2d keys."""

    def __init__(self, nf):
        super().__init__()
        self.conv1 = nn.Conv2d(nf, nf, 3, padding=1)
        self.conv2 = nn.Conv2d(nf, nf, 3, padding=1)


class P3DNet(_LAFCBase):
    NAME, FLOWS, EDGES = "2D LAFC", "flow(2)", "not implemented (FGT's validation passes None)"

    def __init__(self, num_flows, num_feats, in_channels, passmask, use_residual, res_blocks, use_bias, conv_type,
                 init_weights):
        super().__init__(in_channels, passmask, use_bias, conv_type)
        c = num_feats
        if c % 2:
            raise ValueError("fgt_b200 2D LAFC expects an even cnum")
        self.c, self.resNums = c, res_blocks
        self.encoder2 = nn.Sequential(nn.ReplicationPad2d(2), _C2(in_channels, c, 5), _C2(c, 2 * c, 3))
        self.encoder4 = nn.Sequential(_C2(2 * c, 2 * c, 3), _C2(2 * c, 4 * c, 3))
        self.res_blocks = nn.Sequential(*[_Res(4 * c) for _ in range(res_blocks)])
        self._build_tail()
        if init_weights:
            for m in self.modules():  # BaseNetwork.init_weights('normal', 0.02), FGT/models/BaseNetwork.py:20-46
                if isinstance(m, nn.Conv2d):
                    nn.init.normal_(m.weight.data, 0.0, 0.02)
                    nn.init.constant_(m.bias.data, 0.0)

    def _pack_encoder(self, put, sd):
        put("e2a", "encoder2.1.featureConv", im2col=128)   # 5x5x3 = 75 gathered inputs per row
        put("e2b", "encoder2.2.featureConv")
        put("e4a", "encoder4.0.featureConv")
        put("e4b", "encoder4.1.featureConv")
        for i in range(self.resNums):
            put(f"res{i}_1", f"res_blocks.{i}.conv1")
            put(f"res{i}_2", f"res_blocks.{i}.conv2")

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
        B, A = self._allocators((n, H, W), dev, False)
        # encoder2 (lafc_single.py:26-30): ReplicationPad2d(2) + 5x5 conv through the im2col gather, stride-2 conv
        col = A("col", (n, H, W, 128))
        lib.im2col_nchw(flows, masks, col, k=5, stride=1, pad=2, replicate=True, OH=H, OW=W, tag="e2a")
        a1 = A("a1", (n, H, W, c))
        ops.linear([(lib.view16(col, n * H * W, 128), 128)], P["e2a"], n * H * W, act=lib.ACT_LEAKY02, out_split=a1)
        e2 = A("e2", (n, H2, W2, 2 * c))
        ops.conv([(a1, c)], P["e2b"], stride=2, out_split=e2, **C3)
        # encoder4 (:31-35)
        t1 = A("t1", (n, H2, W2, 2 * c))
        ops.conv([(e2, 2 * c)], P["e4a"], out_split=t1, **C3)
        e4 = A("e4", (n, H4, W4, 4 * c))
        e4f = B("e4f", (n, H4, W4, 4 * c)) if self.resNums else None
        ops.conv([(t1, 2 * c)], P["e4b"], stride=2, out_split=e4, out_f32=e4f, **C3)
        # residual blocks without BN (:36-38, 79-82): conv, LeakyReLU(0.2), conv, + identity in fp32, no activation
        src, srcf = e4, e4f
        t3 = A("t3", (n, H4, W4, 4 * c))
        for i in range(self.resNums):
            last = i == self.resNums - 1
            r = A(f"r{i % 2}", (n, H4, W4, 4 * c))
            rf = None if last else B(f"r{i % 2}f", (n, H4, W4, 4 * c))
            ops.conv([(src, 4 * c)], P[f"res{i}_1"], out_split=t3, **C3)
            ops.conv([(t3, 4 * c)], P[f"res{i}_2"], act=lib.ACT_NONE, aux=srcf, aux_mode=lib.AUX_ADD, out_split=r,
                     out_f32=rf, **C3)
            src, srcf = r, rf
        # dilated middle, decoders (skips: the encoder outputs) and edge head (:40-65, 84-112); the flow's conv keeps
        # the reference's LeakyReLU(0.2)
        y = (A("y0", (n, H4, W4, 4 * c)), A("y1", (n, H4, W4, 4 * c)))
        return self._tail(P, B, A, n, H, W, src, y, e4, e2, lib.ACT_LEAKY02)


class Model(nn.Module):
    """Same constructor/forward as FGT.models.lafc_single.Model (lafc_single.py:9-18)."""

    def __init__(self, config):
        super().__init__()
        self.net = P3DNet(config['num_flows'], config['cnum'], config['in_channel'], config['PASSMASK'],
                          config['use_residual'], config['resBlocks'], config['use_bias'], config['conv_type'],
                          config['init_weights'])

    def forward(self, flows, masks, edges=None):
        return self.net(flows, masks, edges)
