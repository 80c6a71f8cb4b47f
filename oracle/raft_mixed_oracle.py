"""RAFT oracle with the reference's mixed-precision mode (TEST INFRASTRUCTURE — see oracle/fgt_oracle.py header).

The same functional restatement as oracle/raft_oracle.py (RAFT/raft.py:87-145, extractor.py, corr.py, update.py,
utils/utils.py), device-agnostic, with a precision switch. With mixed_precision=False it computes exactly what
raft_oracle.raft_forward computes (tests/test_raft_mixed.py checks torch.equal); raft_oracle.py itself is left as the
golden-pinned fp32 definition.

Mixed precision (`raft_forward(..., mixed_precision=True)`, the reference's `--mixed_precision`): the feature net, the
context net and the update block run under CUDA autocast (raft.py:100,111,128). On CUDA tensors the oracle runs the same
three regions under torch.autocast("cuda", torch.float16). On CPU tensors it emulates those casts explicitly: every
function below takes `q`, the rounding to fp16 (values stay fp32 tensors holding fp16 numbers; q=None is fp32). The rules, each mirroring what autocast does to the reference's code:
  * a conv casts its input, weight and bias to fp16, accumulates in fp32 and gives an fp16 output (`_conv`; every
    nn.Conv2d in extractor.py and update.py);
  * elementwise ops on fp16 tensors give fp16, each rounded once: the residual add and ReLU (extractor.py:56),
    tanh / relu of the context split (raft.py:114-115), sigmoid / tanh / r*h and each op of (1-z)*h + z*q
    (update.py:48-58), and mask = .25 * conv (update.py:135);
  * instance and batch norm take the fp16 conv output, keep fp32 statistics and give fp16 (`_norm`,
    extractor.py:29-33,131-132: neither is on autocast's fp32 list);
  * fmap.float() precedes the correlation (raft.py:103-104); the correlation volume, its pyramid and the lookup are fp32
    outside the regions (corr.py);
  * torch.cat of an fp16 and an fp32 tensor promotes to fp32 (update.py:97,129 with the fp32 flow), and the next conv
    rounds it back to fp16;
  * coords1 + delta promotes the fp16 delta to fp32 (raft.py:132);
  * upsample_flow gets the fp16 mask: softmax of fp16 gives fp16, the weighted sum with the fp32 flow is fp32
    (raft.py:73-84,138);
  * the hidden state `net` stays fp16 between iterations (raft.py:128, update.py:58).
"""
import torch
import torch.nn.functional as F

from .raft_oracle import corr_pyramid, sample  # noqa: F401  (device-agnostic, no fp16 rule applies)


def _id(t):
    return t


def round_f16(t):
    """fp32 tensor -> the nearest fp16 values, kept as fp32 (the CPU emulation's rounding)."""
    return t.half().float()


def _norm(x, sd, key, kind, q=None):
    q = q or _id
    if kind == "instance":  # nn.InstanceNorm2d: no affine, per-image statistics (extractor.py:29-33)
        return q(F.instance_norm(x, eps=1e-5))
    return q(F.batch_norm(x, sd[key + ".running_mean"], sd[key + ".running_var"], sd[key + ".weight"],
                          sd[key + ".bias"], training=False, eps=1e-5))  # eval-mode BatchNorm2d


def _conv(x, sd, key, stride=1, pad=0, q=None):
    if q is None:
        return F.conv2d(x, sd[key + ".weight"], sd[key + ".bias"], stride=stride, padding=pad)
    return q(F.conv2d(q(x), q(sd[key + ".weight"]), q(sd[key + ".bias"]), stride=stride, padding=pad))


def res_block(x, sd, key, kind, stride, q=None):
    """ResidualBlock.forward, extractor.py:47-56."""
    y = F.relu(_norm(_conv(x, sd, key + ".conv1", stride, 1, q), sd, key + ".norm1", kind, q))
    y = F.relu(_norm(_conv(y, sd, key + ".conv2", 1, 1, q), sd, key + ".norm2", kind, q))
    if stride != 1:
        x = _norm(_conv(x, sd, key + ".downsample.0", stride, 0, q), sd, key + ".norm3", kind, q)
    return F.relu((q or _id)(x + y))


def encoder(x, sd, key, kind, q=None):
    """BasicEncoder.forward, extractor.py:168-192."""
    x = F.relu(_norm(_conv(x, sd, key + ".conv1", 2, 3, q), sd, key + ".norm1", kind, q))
    for name, stride in (("layer1", 1), ("layer2", 2), ("layer3", 2)):
        x = res_block(x, sd, f"{key}.{name}.0", kind, stride, q)
        x = res_block(x, sd, f"{key}.{name}.1", kind, 1, q)
    return _conv(x, sd, key + ".conv2", q=q)


def corr_lookup(pyr, coords, r=4):
    """CorrBlock.__call__, corr.py:29-50."""
    coords = coords.permute(0, 2, 3, 1)
    b, h, w, _ = coords.shape
    out = []
    d = torch.linspace(-r, r, 2 * r + 1, device=coords.device)
    delta = torch.stack(torch.meshgrid(d, d, indexing="ij"), dim=-1).view(1, 2 * r + 1, 2 * r + 1, 2)
    for i, corr in enumerate(pyr):
        c = coords.reshape(b * h * w, 1, 1, 2) / 2 ** i + delta
        out.append(sample(corr, c).view(b, h, w, -1))
    return torch.cat(out, dim=-1).permute(0, 3, 1, 2).contiguous().float()


def motion_encoder(flow, corr, sd, key="update_block.encoder", q=None):
    """BasicMotionEncoder.forward, update.py:89-97."""
    cor = F.relu(_conv(corr, sd, key + ".convc1", q=q))
    cor = F.relu(_conv(cor, sd, key + ".convc2", 1, 1, q))
    flo = F.relu(_conv(flow, sd, key + ".convf1", 1, 3, q))
    flo = F.relu(_conv(flo, sd, key + ".convf2", 1, 1, q))
    out = F.relu(_conv(torch.cat([cor, flo], 1), sd, key + ".conv", 1, 1, q))
    return torch.cat([out, flow], 1)


def sep_conv_gru(h, x, sd, key="update_block.gru", q=None):
    """SepConvGRU.forward, update.py:45-60."""
    Q = q or _id
    for sfx, pad in (("1", (0, 2)), ("2", (2, 0))):
        hx = torch.cat([h, x], 1)
        z = Q(torch.sigmoid(_conv(hx, sd, f"{key}.convz{sfx}", 1, pad, q)))
        r = Q(torch.sigmoid(_conv(hx, sd, f"{key}.convr{sfx}", 1, pad, q)))
        qq = Q(torch.tanh(_conv(torch.cat([Q(r * h), x], 1), sd, f"{key}.convq{sfx}", 1, pad, q)))
        h = Q(Q(Q(1 - z) * h) + Q(z * qq))
    return h


def upsample_flow(flow, mask, q=None):
    """RAFT.upsample_flow, raft.py:73-84."""
    n, _, h, w = flow.shape
    mask = (q or _id)(torch.softmax(mask.view(n, 1, 9, 8, 8, h, w), dim=2))
    up = F.unfold(8 * flow, [3, 3], padding=1).view(n, 2, 9, 1, 1, h, w)
    up = torch.sum(mask * up, dim=2).permute(0, 1, 4, 2, 5, 3)
    return up.reshape(n, 2, 8 * h, 8 * w)


def update_block(net, inp, corr, flow, sd, q=None):
    """BasicUpdateBlock.forward, update.py:127-136: (net, mask, delta_flow)."""
    mf = motion_encoder(flow, corr, sd, q=q)
    net = sep_conv_gru(net, torch.cat([inp, mf], 1), sd, q=q)
    delta = _conv(F.relu(_conv(net, sd, "update_block.flow_head.conv1", 1, 1, q)), sd,
                  "update_block.flow_head.conv2", 1, 1, q)
    mask = (q or _id)(0.25 * _conv(F.relu(_conv(net, sd, "update_block.mask.0", 1, 1, q)), sd,
                                   "update_block.mask.2", q=q))
    return net, mask, delta


def context(im1, sd, hdim=128, cdim=128, q=None):
    """The context net and its split, raft.py:111-115: (net, inp)."""
    c = encoder(im1, sd, "cnet", "batch", q)
    return (q or _id)(torch.tanh(c[:, :hdim])), torch.relu(c[:, hdim:hdim + cdim])


def _region(mixed, device):
    """The reference's `with autocast(enabled=self.args.mixed_precision)` (raft.py:100,111,128) on CUDA tensors."""
    return torch.autocast("cuda", torch.float16, enabled=mixed and device.type == "cuda")


def raft_forward(sd, image1, image2, iters=20, hdim=128, cdim=128, all_iters=False, mixed_precision=False):
    """RAFT.forward(test_mode=True), raft.py:87-145. sd: state_dict without the 'module.' prefix.
    Returns (flow_low [n,2,H/8,W/8], flow_up [n,2,H,W]); with all_iters also the per-iteration
    low-resolution flows. mixed_precision: autocast on CUDA tensors, the emulation above on CPU tensors."""
    dev = image1.device
    q = round_f16 if mixed_precision and dev.type != "cuda" else None
    im1 = (2 * (image1 / 255.0) - 1.0).contiguous()
    im2 = (2 * (image2 / 255.0) - 1.0).contiguous()
    with _region(mixed_precision, dev):
        fm = encoder(torch.cat([im1, im2], 0), sd, "fnet", "instance", q)
    n = im1.shape[0]
    f1, f2 = fm[:n].float(), fm[n:].float()
    pyr = corr_pyramid(f1, f2)
    with _region(mixed_precision, dev):
        net, inp = context(im1, sd, hdim, cdim, q)
    _, _, H, W = im1.shape
    ys, xs = torch.meshgrid(torch.arange(H // 8, device=dev), torch.arange(W // 8, device=dev), indexing="ij")
    coords0 = torch.stack([xs, ys], 0).float()[None].repeat(n, 1, 1, 1)
    coords1 = coords0.clone()
    lows = []
    flow_up = None
    for _ in range(iters):
        corr = corr_lookup(pyr, coords1)
        flow = coords1 - coords0
        with _region(mixed_precision, dev):
            net, mask, delta = update_block(net, inp, corr, flow, sd, q)
        coords1 = coords1 + delta
        flow_up = upsample_flow(coords1 - coords0, mask, q)
        lows.append(coords1 - coords0)
    if all_iters:
        return coords1 - coords0, flow_up, lows
    return coords1 - coords0, flow_up
