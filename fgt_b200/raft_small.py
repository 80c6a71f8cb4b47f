"""H100-native small RAFT (the reference's --small, RAFT-S) behind the reference's nn.Module interface, and the
reference's model constructor.

`SmallRAFT(args).forward(image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False)` takes the
reference's state_dict keys for RAFT(small=True) (106 tensors; survives the driver's DataParallel wrap/unwrap) and runs
on the host forward it shares with the basic model (raft_model._RAFTBase). What is its own:

  * feature / context encoders (SmallEncoder of BottleneckBlocks, extractor.py:60-116,195-267): implicit-GEMM convs;
    the feature net's InstanceNorm = fgt_chan_stats + fgt_instnorm_act, the context net has no norm layer;
  * all-pairs correlation over 128-dimensional features (alpha = 1/sqrt(128)) + fgt_avgpool2 pyramid, 4 levels;
  * per iteration: fgt_corr_lookup (radius 3, 196 values) -> SmallMotionEncoder convs -> ConvGRU (3x3 convs, z | r and
    the (1-z)h+zq update fused in GEMM epilogues) -> flow head -> fgt_raft_flow_update;
  * fgt_upflow8 (8 * bilinear x8, align_corners=True, utils.py:80-82) only where the result is consumed (last
    iteration in test_mode).

fp32 only (3-term split-bf16 GEMMs): the small model under mixed_precision is not implemented and is refused.
"""
import torch.nn as nn

from . import lib, ops, raft_model
from .raft_model import C3


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
            setattr(self, f"conv{g}", nn.Conv2d(96 + 146, 96, 3, padding=1))


class _FlowHead(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(96, 128, 3, padding=1)
        self.conv2 = nn.Conv2d(128, 2, 3, padding=1)


class _UpdateBlock(nn.Module):
    def __init__(self):
        super().__init__()
        self.encoder = _MotionEncoder()
        self.gru = _GRU()
        self.flow_head = _FlowHead()


class SmallRAFT(raft_model._RAFTBase):
    FDIM, STEM, STAGES = 128, 32, ((32, 1), (64, 2), (96, 2))
    BLOCK = (("conv1", 4, 1, False), ("conv2", 4, 3, True), ("conv3", 1, 1, False))   # bottleneck (extractor.py:60-116)
    HDIM, CDIM = 96, 64
    RADIUS, LOOK = 3, 200   # 4 levels x 7 x 7 = 196 values, zero-padded to a multiple of 8 channels
    XW, FLOW_CH = 152, 144  # x = [inp(64) | motion features(80) | flow(2)] = 146 channels, zero-padded
    GRU = (("", 3, 3),)

    def __init__(self, args):
        super().__init__(args)
        self.fnet = _SmallEncoder(128)
        self.cnet = _SmallEncoder(self.HDIM + self.CDIM)
        self.update_block = _UpdateBlock()

    def _mixed(self):
        if getattr(self.args, "mixed_precision", False):
            raise ValueError("fgt_b200 small RAFT: mixed_precision is not implemented for the small model "
                             "(use the basic model, or small=True with mixed_precision=False)")
        return False

    def _update_heads(self, P, B, A, n, h, w, look, flow, h4, x4):
        """(motion encoder, upsampling) of one iteration: SmallMotionEncoder (update.py:71-77) into x4's channels
        [64, 144), and upflow8."""
        tot = n * h * w
        RELU = lib.ACT_RELU
        corflo = A("corflo", (n, h, w, 128))  # [cor(96) | flo(32)]
        fcol = A("fcol", (n, h, w, 128))
        flo1 = A("flo1", (n, h, w, 64))

        def motion():
            ops.linear([(look, self.LOOK)], P["convc1"], tot, act=RELU, os_x=128,
                       out_split=lib.view16(corflo, tot, 128))
            lib.im2col_nchw(flow, None, fcol, k=7, stride=1, pad=3, replicate=False, OH=h, OW=w)
            ops.linear([(lib.view16(fcol, tot, 128), 128)], P["convf1"], tot, act=RELU,
                       out_split=lib.view16(flo1, tot, 64))
            ops.conv([(flo1, 64)], P["convf2"], act=RELU, out_c_total=128, out_c_offset=96, out_split=corflo, **C3)
            ops.conv([(corflo, 128)], P["mconv"], act=RELU, out_c_total=self.XW, out_c_offset=self.CDIM, out_split=x4,
                     **C3)

        def upsample(up):
            lib.upflow8(flow, h, w, up, n=n)

        return motion, upsample


def make_raft(args):
    """The reference's model constructor RAFT(args) (RAFT/raft.py:25-56): SmallRAFT when args.small is set, else the
    basic model, raft_model.RAFT."""
    return SmallRAFT(args) if getattr(args, "small", False) else raft_model.RAFT(args)
