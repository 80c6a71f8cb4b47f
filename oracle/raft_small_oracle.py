"""CPU oracle for the small RAFT model, the reference's --small (TEST INFRASTRUCTURE — see oracle/fgt_oracle.py header).

Functional PyTorch-CPU restatement of /root/reference/RAFT/raft.py:87-145 with args.small (hidden 96, context 64,
4 correlation levels of radius 3, raft.py:29-33,48-51), RAFT/extractor.py:60-116,195-267 (BottleneckBlock /
SmallEncoder), RAFT/update.py (SmallMotionEncoder :62-77, ConvGRU :16-31, FlowHead :6-14, SmallUpdateBlock :99-112)
and RAFT/utils/utils.py:80-82 (upflow8). The correlation pyramid and lookup are raft_oracle's. Pinned by
tests/golden/raft_s_*.npz (outputs of the unmodified reference).
"""
import torch
import torch.nn.functional as F

from oracle import raft_oracle as RO
from oracle.raft_oracle import _conv


def _norm(x, kind):
    # fnet: nn.InstanceNorm2d (no affine, per-image statistics); cnet: norm_fn='none' (nn.Sequential(), identity)
    return F.instance_norm(x, eps=1e-5) if kind == "instance" else x


def bottleneck(x, sd, key, kind, stride):
    """BottleneckBlock.forward, extractor.py:107-116."""
    y = F.relu(_norm(_conv(x, sd, key + ".conv1"), kind))
    y = F.relu(_norm(_conv(y, sd, key + ".conv2", stride, 1), kind))
    y = F.relu(_norm(_conv(y, sd, key + ".conv3"), kind))
    if stride != 1:
        x = _norm(_conv(x, sd, key + ".downsample.0", stride, 0), kind)
    return F.relu(x + y)


def small_encoder(x, sd, key, kind):
    """SmallEncoder.forward, extractor.py:244-267."""
    x = F.relu(_norm(_conv(x, sd, key + ".conv1", 2, 3), kind))
    for name, stride in (("layer1", 1), ("layer2", 2), ("layer3", 2)):
        x = bottleneck(x, sd, f"{key}.{name}.0", kind, stride)
        x = bottleneck(x, sd, f"{key}.{name}.1", kind, 1)
    return _conv(x, sd, key + ".conv2")


def motion_encoder(flow, corr, sd, key="update_block.encoder"):
    """SmallMotionEncoder.forward, update.py:71-77."""
    cor = F.relu(_conv(corr, sd, key + ".convc1"))
    flo = F.relu(_conv(flow, sd, key + ".convf1", 1, 3))
    flo = F.relu(_conv(flo, sd, key + ".convf2", 1, 1))
    out = F.relu(_conv(torch.cat([cor, flo], 1), sd, key + ".conv", 1, 1))
    return torch.cat([out, flow], 1)


def conv_gru(h, x, sd, key="update_block.gru"):
    """ConvGRU.forward, update.py:23-31."""
    hx = torch.cat([h, x], 1)
    z = torch.sigmoid(_conv(hx, sd, key + ".convz", 1, 1))
    r = torch.sigmoid(_conv(hx, sd, key + ".convr", 1, 1))
    q = torch.tanh(_conv(torch.cat([r * h, x], 1), sd, key + ".convq", 1, 1))
    return (1 - z) * h + z * q


def upflow8(flow):
    """utils/utils.py:80-82."""
    return 8 * F.interpolate(flow, size=(8 * flow.shape[2], 8 * flow.shape[3]), mode="bilinear", align_corners=True)


def raft_small_forward(sd, image1, image2, iters=20, flow_init=None, all_iters=False):
    """RAFT.forward(test_mode=True) of the small model, raft.py:87-145. sd: state_dict without the 'module.' prefix.
    Returns (flow_low [n,2,H/8,W/8], flow_up [n,2,H,W]); with all_iters also every iteration's upsampled flow."""
    hdim, cdim = 96, 64
    im1 = (2 * (image1 / 255.0) - 1.0).contiguous()
    im2 = (2 * (image2 / 255.0) - 1.0).contiguous()
    fm = small_encoder(torch.cat([im1, im2], 0), sd, "fnet", "instance")
    n = im1.shape[0]
    pyr = RO.corr_pyramid(fm[:n].float(), fm[n:].float())
    c = small_encoder(im1, sd, "cnet", "none")
    net, inp = torch.tanh(c[:, :hdim]), torch.relu(c[:, hdim:hdim + cdim])
    _, _, H, W = im1.shape
    ys, xs = torch.meshgrid(torch.arange(H // 8), torch.arange(W // 8), indexing="ij")
    coords0 = torch.stack([xs, ys], 0).to(im1.dtype)[None].repeat(n, 1, 1, 1)
    coords1 = coords0.clone()
    if flow_init is not None:
        coords1 = coords1 + flow_init
    ups = []
    for _ in range(iters):
        corr = RO.corr_lookup(pyr, coords1, r=3).to(im1.dtype)
        flow = coords1 - coords0
        net = conv_gru(net, torch.cat([inp, motion_encoder(flow, corr, sd)], 1), sd)
        delta = _conv(F.relu(_conv(net, sd, "update_block.flow_head.conv1", 1, 1)), sd,
                      "update_block.flow_head.conv2", 1, 1)
        coords1 = coords1 + delta
        ups.append(upflow8(coords1 - coords0))
    if all_iters:
        return coords1 - coords0, ups[-1], ups
    return coords1 - coords0, ups[-1]
