"""Seeded synthetic weights and inputs shared by tests, bench.py and tests/golden/make_golden.py.

There is no network, so FGT / LAFC checkpoints (Google-Drive downloads in the reference,
/root/reference/README.md:57) are replaced by seeded random weights of the same architecture, and
clips by seeded synthetic frames / masks / flows shaped like the driver's tensors
(/root/reference/tool/video_inpainting.py:689-708).
"""
import math
import zlib

import torch

CFG_A = dict(tw=2, sw=8, gd=4, input_resolution=(240, 432), in_channel=4, cnum=64, flow_inChannel=2,
             flow_cnum=64, frame_hidden=512, flow_hidden=256, PASSMASK=1, numBlocks=8, kernel_size=(7, 7),
             stride=(3, 3), padding=(3, 3), num_head=4, conv_type='vanilla', norm='None', use_bias=1, ape=1,
             mlp_ratio=40, drop=0, init_weights=1)


def fgt_param_shapes(cfg=CFG_A):
    """state_dict contract of FGT.models.model.Model (keys under 'net.'), SURVEY.md Appendix B;
    restates the constructors at /root/reference/FGT/models/model.py:28-50,196-246."""
    d, df = cfg['frame_hidden'], cfg['flow_hidden']
    cn, fcn = cfg['cnum'], cfg['flow_cnum']
    kh, kw = cfg['kernel_size']
    hid = kh * kw * cfg['mlp_ratio']
    gd = cfg['gd']
    s = {}

    def conv(name, co, ci, k1, k2=None):
        s[name + ".weight"] = (co, ci, k1, k1 if k2 is None else k2)
        s[name + ".bias"] = (co,)

    def lin(name, co, ci):
        s[name + ".weight"] = (co, ci)
        s[name + ".bias"] = (co,)

    def ln(name, c):
        s[name + ".weight"] = (c,)
        s[name + ".bias"] = (c,)

    enc = [(0, 64, cfg['in_channel']), (2, 64, 64), (4, 128, 64), (6, 256, 128), (8, 384, 256), (10, 512, 320),
           (12, 384, 192), (14, 256, 80), (16, 128, 512)]
    for i, co, ci in enc:
        conv(f"frame_endoder.layers.{i}", co, ci, 3)
    conv("flow_encoder.1.featureConv", fcn, cfg['flow_inChannel'], 5)
    conv("flow_encoder.2.featureConv", fcn * 2, fcn, 3)
    conv("flow_encoder.3.featureConv", fcn * 2, fcn * 2, 3)
    conv("flow_encoder.4.featureConv", fcn * 2, fcn * 2, 3)
    conv("patch2vec", d, cn * 2, kh, kw)
    conv("f_patch2vec", df, fcn * 2, kh, kw)
    conv("add_pos_emb.proj", d, 1, 3)

    def ffn(pre):
        lin(pre + "ffn.conv1", hid, d)
        lin(pre + "ffn.conv2.2", d, hid)

    def tblock(pre):
        for nm in ("query_embedding", "key_embedding", "value_embedding", "output_linear"):
            lin(pre + "attention." + nm, d, d)
        ffn(pre)
        ln(pre + "norm1", d)
        ln(pre + "norm2", d)

    def sblock(pre):
        lin(pre + "attention.query_embedding", d, d + df)
        lin(pre + "attention.key_embedding", d, d + df)
        lin(pre + "attention.value_embedding", d, d)
        lin(pre + "attention.output_linear", d, d)
        conv(pre + "attention.global_extract_v", d, 1, gd)
        conv(pre + "attention.global_extract_k", d + df, 1, gd)
        ln(pre + "attention.q_norm", d + df)
        ln(pre + "attention.k_norm", d + df)
        ln(pre + "attention.v_norm", d)
        lin(pre + "attention.reweightFlow.0", df, d + df)
        ffn(pre)
        ln(pre + "norm", d)

    for i in range(cfg['numBlocks'] // 2 - 1):
        tblock(f"transformer.{i}.t_transformer.")
        sblock(f"transformer.{i}.s_transformer.")
    tblock("first_t_transformer.")
    sblock("first_s_transformer.")
    lin("vec2patch.embedding", kh * kw * cn * 2, d)
    conv("decoder.layer1.conv.featureConv", cn * 2, cn * 2, 3)
    conv("decoder.layer2.featureConv", cn, cn * 2, 3)
    conv("decoder.layer3.conv.featureConv", cn, cn, 3)
    conv("decoder.final.featureConv", 3, cn, 3)
    return {"net." + k: v for k, v in s.items()}


def make_state_dict(shapes, seed=0, regime="scaled"):
    """Deterministic weights, independent of key order (each tensor seeded by crc32(key)).

    regime 'default': the reference init (normal(0, 0.02) weights, zero bias, LN = identity;
        /root/reference/FGT/models/BaseNetwork.py:20-46).
    regime 'scaled': variance-preserving weights (std = gain/sqrt(fan_in), gain 2 on Q/K projections), random biases and LN
        affines — keeps activations O(1) through the depth and makes softmax / LN non-degenerate
        (SURVEY.md §0: with the default init attention logits are ~0 and softmax bugs go unseen).
    """
    sd = {}
    for key, shape in shapes.items():
        g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(key.encode())) & 0x7FFFFFFF)
        is_norm = ("norm" in key.split(".")[-2]) if len(key.split(".")) >= 2 else False
        if key.endswith(".weight") and len(shape) >= 2:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            gain = 1.0
            if "query_embedding" in key or "key_embedding" in key:
                gain = 2.0  # attention logits std ~3: softmax clearly non-uniform
            elif "decoder.final" in key:
                gain = 0.5  # keep tanh out of saturation
            elif "vec2patch" in key:
                gain = 0.25
            if regime == "kaiming":  # LAFC's reference init (kaiming_normal fan_in, LAFC/models/BaseNetwork.py)
                gain = math.sqrt(2.0)
            std = 0.02 if regime == "default" else gain / math.sqrt(fan_in)
            sd[key] = torch.randn(shape, generator=g) * std
        elif key.endswith(".weight"):  # LayerNorm gamma
            sd[key] = torch.ones(shape) if regime == "default" else 1.0 + 0.2 * torch.randn(shape, generator=g)
        else:  # biases / LN beta
            if regime in ("default", "kaiming"):
                sd[key] = torch.zeros(shape)
            else:
                sd[key] = (0.1 if is_norm else 0.05) * torch.randn(shape, generator=g)
    return sd


def _smooth(noise, k=15):
    pad = k // 2
    ker = torch.ones(1, 1, k, k) / (k * k)
    n, c, h, w = noise.shape
    x = torch.nn.functional.pad(noise.reshape(n * c, 1, h, w), (pad, pad, pad, pad), mode="reflect")
    return torch.nn.functional.conv2d(x, ker).reshape(n, c, h, w)


def fgt_inputs(seed=0, t=10, H=240, W=432, b=1):
    """Synthetic clip shaped like the driver's FGT inputs (video_inpainting.py:689-708):
    frames in [-1,1] already multiplied by (1-mask), masks in {0,1} (seeded rectangles/ellipses
    covering roughly 10-30%), flows normalised per (frame, channel) by the signed max
    (video_inpainting.py:402-407)."""
    g = torch.Generator().manual_seed(seed)
    frames = torch.rand(b, t, 3, H, W, generator=g) * 2 - 1
    masks = torch.zeros(b, t, 1, H, W)
    ys = torch.arange(H).view(H, 1).float()
    xs = torch.arange(W).view(1, W).float()
    for bi in range(b):
        for ti in range(t):
            r = torch.rand(5, generator=g)
            hh = int(H * (0.3 + 0.25 * r[0].item()))
            ww = int(W * (0.3 + 0.25 * r[1].item()))
            y0 = int((H - hh) * r[2].item())
            x0 = int((W - ww) * r[3].item())
            if r[4].item() < 0.5:
                masks[bi, ti, 0, y0:y0 + hh, x0:x0 + ww] = 1.0
            else:
                cy, cx = y0 + hh / 2, x0 + ww / 2
                masks[bi, ti, 0] = ((((ys - cy) / (hh / 2)) ** 2 + ((xs - cx) / (ww / 2)) ** 2) <= 1.0).float()
    flows = _smooth(torch.randn(b * t, 2, H, W, generator=g)) * 3.0 * 15
    mx = flows.amax(dim=(2, 3), keepdim=True)
    flows = (flows / mx).reshape(b, t, 2, H, W)
    return frames * (1 - masks), flows, masks


# ----------------------------------------------------------------------------------------------
# LAFC (flow completion)
# ----------------------------------------------------------------------------------------------
CFG_LAFC = dict(num_flows=3, flow_interval=3, cnum=48, in_channel=3, PASSMASK=1, use_residual=1, resBlocks=1,
                use_bias=1, conv_type='vanilla', init_weights=1, model='lafc')


def lafc_param_shapes(cfg=CFG_LAFC):
    """state_dict contract of LAFC.models.lafc.Model (/root/reference/LAFC/models/lafc.py:18-82)."""
    c, T = cfg['cnum'], cfg['num_flows']
    s = {}

    def c3(name, co, ci, kt, k):
        s[name + ".featureConv.weight"] = (co, ci, kt, k, k)
        s[name + ".featureConv.bias"] = (co,)

    def c2(name, co, ci, k):
        s[name + ".featureConv.weight"] = (co, ci, k, k)
        s[name + ".featureConv.bias"] = (co,)

    def p3d(name, ci, co, k):
        c3(name + ".conv1", co, ci, 1, k)
        c3(name + ".conv2", co, co, 3, 1)

    p3d("encoder2.1", cfg['in_channel'], c, 5)
    p3d("encoder2.2", c, 2 * c, 3)
    p3d("encoder4.0", 2 * c, 2 * c, 3)
    p3d("encoder4.1", 2 * c, 4 * c, 3)
    p3d("res_blocks.0", 4 * c, 4 * c, 3)
    c3("condense2", 2 * c, 2 * c, T, 1)
    c3("condense4_pre", 4 * c, 4 * c, T, 1)
    c3("condense4_post", 4 * c, 4 * c, T, 1)
    for i in range(4):
        c2(f"middle.{i}", 4 * c, 4 * c, 3)
    c2("decoder2.0.conv", 2 * c, 8 * c, 3)
    c2("decoder2.1", 2 * c, 2 * c, 3)
    c2("decoder2.2", 2 * c, 2 * c, 3)
    c2("decoder.0.conv", c, 4 * c, 3)
    c2("decoder.1", c // 2, c, 3)
    c2("decoder.2", 2, c // 2, 3)
    c2("edgeDetector.projection", 16, 2, 3)
    c2("edgeDetector.mid_layer_1", 16, 16, 3)
    c2("edgeDetector.mid_layer_2", 16, 16, 3)
    c2("edgeDetector.out_layer", 1, 16, 1)
    return {"net." + k: v for k, v in s.items()}


def lafc_inputs(seed=0, T=3, H=240, W=432, b=1):
    """Diffused candidate flows (pixels) and hole masks shaped like complete_flow's call
    (/root/reference/tool/video_inpainting.py:369-378): flows [b,2,T,H,W], masks [b,1,T,H,W]."""
    g = torch.Generator().manual_seed(seed)
    flows = _smooth(torch.randn(b * T, 2, H, W, generator=g), k=21) * 60.0
    masks = torch.zeros(b, 1, T, H, W)
    for bi in range(b):
        for ti in range(T):
            r = torch.rand(4, generator=g)
            hh, ww = int(H * (0.2 + 0.3 * r[0].item())), int(W * (0.2 + 0.3 * r[1].item()))
            y0, x0 = int((H - hh) * r[2].item()), int((W - ww) * r[3].item())
            masks[bi, 0, ti, y0:y0 + hh, x0:x0 + ww] = 1.0
    flows = flows.reshape(b, T, 2, H, W).permute(0, 2, 1, 3, 4).contiguous()
    return flows, masks


# ----------------------------------------------------------------------------------------------
# single-frame ("2D") LAFC, FGT's validation flow completion (LAFC/config/train_single.yaml)
# ----------------------------------------------------------------------------------------------
CFG_LAFC_SINGLE = dict(num_flows=1, cnum=48, in_channel=3, PASSMASK=1, use_residual=1, resBlocks=1, use_bias=1,
                       conv_type='vanilla', init_weights=1, model='lafc_single')


def lafc_single_param_shapes(cfg=CFG_LAFC_SINGLE):
    """state_dict contract of FGT.models.lafc_single.Model (/root/reference/FGT/models/lafc_single.py:21-68)."""
    c = cfg['cnum']
    s = {}

    def c2(name, co, ci, k, bare=False):
        key = name if bare else name + ".featureConv"
        s[key + ".weight"] = (co, ci, k, k)
        s[key + ".bias"] = (co,)

    c2("encoder2.1", c, cfg['in_channel'], 5)
    c2("encoder2.2", 2 * c, c, 3)
    c2("encoder4.0", 2 * c, 2 * c, 3)
    c2("encoder4.1", 4 * c, 2 * c, 3)
    for i in range(cfg['resBlocks']):
        c2(f"res_blocks.{i}.conv1", 4 * c, 4 * c, 3, bare=True)
        c2(f"res_blocks.{i}.conv2", 4 * c, 4 * c, 3, bare=True)
    for i in range(4):
        c2(f"middle.{i}", 4 * c, 4 * c, 3)
    c2("decoder2.0.conv", 2 * c, 8 * c, 3)
    c2("decoder2.1", 2 * c, 2 * c, 3)
    c2("decoder2.2", 2 * c, 2 * c, 3)
    c2("decoder.0.conv", c, 4 * c, 3)
    c2("decoder.1", c // 2, c, 3)
    c2("decoder.2", 2, c // 2, 3)
    c2("edgeDetector.projection", 16, 2, 3)
    c2("edgeDetector.mid_layer_1", 16, 16, 3)
    c2("edgeDetector.mid_layer_2", 16, 16, 3)
    c2("edgeDetector.out_layer", 1, 16, 1)
    return {"net." + k: v for k, v in s.items()}


def lafc_single_state_dict(seed=0, regime="scaled", cfg=CFG_LAFC_SINGLE):
    """Seeded 2D-LAFC weights in LAFC's two golden regimes: 'scaled' (variance-preserving, random biases) or 'kaiming'
    (kaiming_normal fan_in, zero biases)."""
    return make_state_dict(lafc_single_param_shapes(cfg), seed=seed, regime=regime)


def lafc_single_inputs(seed=0, n=3, H=240, W=432):
    """Per-frame diffused flows (pixels) and hole masks as FGT's validation feeds the 2D LAFC
    (FGT/networks/network.py:299-304): flows [n,2,H,W], masks [n,1,H,W]."""
    flows, masks = lafc_inputs(seed=seed, T=n, H=H, W=W)
    return flows[0].transpose(0, 1).contiguous(), masks[0].transpose(0, 1).contiguous()


def validation_set(root, seed=0, videos=(("vid_a", 45), ("vid_b", 41), ("vid_short", 25)), H=90, W=150,
                   flow_hw=(72, 120), flow_ids=None):
    """Writes a seeded DAVIS-style validation set under `root` in the layout of FGT's valid_config.yaml:
    JPEGImages/<video>/%05d.jpg (smooth RGB frames, H x W), rectMask/<video>/%05d.png (one moving rectangle, 0 / 255)
    and flows/<video>/{forward,backward}_flo/%05d.flo (smooth flows of flow_hw, L - 1 per direction, or only the
    indices in flow_ids). Returns the three roots (frame_root, mask_root, flow_root)."""
    import os

    from PIL import Image

    from .io import write_flo
    roots = [os.path.join(root, d) for d in ("JPEGImages", "rectMask", "flows")]
    g = torch.Generator().manual_seed(seed)
    fh, fw = flow_hw
    for vi, (name, n) in enumerate(videos):
        for r in roots:
            os.makedirs(os.path.join(r, name), exist_ok=True)
        base = _smooth(torch.rand(1, 3, H, W, generator=g), k=9)[0]
        h0, w0 = int(H * (0.25 + 0.1 * vi)), int(W * (0.3 + 0.05 * vi))
        for i in range(n):
            shift = (i * 2) % W
            img = (torch.roll(base, shifts=shift, dims=2) * 255 + 20 * torch.rand(3, H, W, generator=g)).clamp(0, 255)
            Image.fromarray(img.permute(1, 2, 0).to(torch.uint8).numpy()).save(
                os.path.join(roots[0], name, f"{i:05d}.jpg"), quality=90)
            m = torch.zeros(H, W, dtype=torch.uint8)
            y0, x0 = (H - h0) // 2 + (i % 7) - 3, (i * 3) % (W - w0)
            m[y0:y0 + h0, x0:x0 + w0] = 255
            Image.fromarray(m.numpy()).save(os.path.join(roots[1], name, f"{i:05d}.png"))
        for sub in ("forward_flo", "backward_flo"):
            os.makedirs(os.path.join(roots[2], name, sub), exist_ok=True)
            for i in (range(n - 1) if flow_ids is None else sorted(set(flow_ids(n)))):
                f = _smooth(torch.randn(1, 2, fh, fw, generator=g), k=11)[0] * 40.0
                write_flo(os.path.join(roots[2], name, sub, f"{i:05d}.flo"), f.permute(1, 2, 0).numpy())
    return tuple(roots)


# ----------------------------------------------------------------------------------------------
# RAFT (basic model)
# ----------------------------------------------------------------------------------------------
def raft_param_shapes():
    """state_dict contract of RAFT.RAFT (basic), /root/reference/RAFT/{raft,extractor,update}.py; same
    179 keys as raft-things.pth minus the DataParallel 'module.' prefix."""
    s = {}

    def conv(name, co, ci, kh, kw=None):
        s[name + ".weight"] = (co, ci, kh, kh if kw is None else kw)
        s[name + ".bias"] = (co,)

    def bn(name, c):
        s[name + ".weight"] = (c,)
        s[name + ".bias"] = (c,)
        s[name + ".running_mean"] = (c,)
        s[name + ".running_var"] = (c,)
        s[name + ".num_batches_tracked"] = ()

    def enc(pre, out_dim, batch_norm):
        conv(pre + ".conv1", 64, 3, 7)
        if batch_norm:
            bn(pre + ".norm1", 64)
        cin = 64
        for li, (dim, stride) in enumerate(((64, 1), (96, 2), (128, 2)), start=1):
            for bi in range(2):
                k = f"{pre}.layer{li}.{bi}"
                st = stride if bi == 0 else 1
                conv(k + ".conv1", dim, cin if bi == 0 else dim, 3)
                conv(k + ".conv2", dim, dim, 3)
                if batch_norm:
                    bn(k + ".norm1", dim)
                    bn(k + ".norm2", dim)
                if st != 1:
                    conv(k + ".downsample.0", dim, cin, 1)
                    if batch_norm:
                        bn(k + ".norm3", dim)
                        bn(k + ".downsample.1", dim)  # alias of norm3 in the reference module
            cin = dim
        conv(pre + ".conv2", out_dim, 128, 1)

    enc("fnet", 256, False)
    enc("cnet", 256, True)
    u = "update_block."
    conv(u + "encoder.convc1", 256, 324, 1)
    conv(u + "encoder.convc2", 192, 256, 3)
    conv(u + "encoder.convf1", 128, 2, 7)
    conv(u + "encoder.convf2", 64, 128, 3)
    conv(u + "encoder.conv", 126, 256, 3)
    for g in "zrq":
        conv(u + f"gru.conv{g}1", 128, 384, 1, 5)
        conv(u + f"gru.conv{g}2", 128, 384, 5, 1)
    conv(u + "flow_head.conv1", 256, 128, 3)
    conv(u + "flow_head.conv2", 2, 256, 3)
    conv(u + "mask.0", 256, 128, 3)
    conv(u + "mask.2", 576, 256, 1)
    return s


def raft_state_dict(seed=0, flow_gain=0.5):
    """Seeded RAFT weights: He-style conv weights (std = gain/sqrt(fan_in)), small random biases,
    BatchNorm with random affine and running statistics; the flow head is damped (flow_gain) so the
    20-step recurrence stays in a sane flow range with random weights."""
    shapes = raft_param_shapes()
    sd = {}
    for key, shape in shapes.items():
        g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(key.encode())) & 0x7FFFFFFF)
        if key.endswith("num_batches_tracked"):
            sd[key] = torch.tensor(100, dtype=torch.int64)
        elif key.endswith("running_var"):
            sd[key] = 0.5 + torch.rand(shape, generator=g)
        elif key.endswith("running_mean"):
            sd[key] = 0.1 * torch.randn(shape, generator=g)
        elif len(shape) == 4:
            fan_in = shape[1] * shape[2] * shape[3]
            gain = 1.4
            if "flow_head.conv2" in key:
                gain = flow_gain
            elif "gru.conv" in key or "mask.2" in key:
                gain = 1.0
            sd[key] = torch.randn(shape, generator=g) * (gain / math.sqrt(fan_in))
        elif key.endswith(".weight"):  # BatchNorm gamma
            sd[key] = 1.0 + 0.2 * torch.randn(shape, generator=g)
        else:
            sd[key] = 0.05 * torch.randn(shape, generator=g)
    # the reference's downsample.1 IS norm3 (extractor.py:43-44): keep the aliases identical
    for k in list(sd):
        if ".downsample.1." in k:
            sd[k] = sd[k.replace(".downsample.1.", ".norm3.")].clone()
    return sd


def raft_inputs(seed=0, H=480, W=864, n=1, shift=3.0):
    """A smooth random image in [0,255] and a warped copy (global shift + smooth deformation)."""
    g = torch.Generator().manual_seed(seed)
    base = _smooth(torch.randn(n, 3, H + 32, W + 32, generator=g), k=9)
    base = base + 0.3 * _smooth(torch.randn(n, 3, H + 32, W + 32, generator=g), k=3)
    base = (base - base.amin()) / (base.amax() - base.amin()) * 255.0
    dx, dy = int(shift), int(-shift // 2)
    im1 = base[:, :, 16:16 + H, 16:16 + W].contiguous()
    im2 = base[:, :, 16 + dy:16 + dy + H, 16 + dx:16 + dx + W].contiguous()
    return im1, im2


# ----------------------------------------------------------------------------------------------
# RAFT (small model, the reference's --small)
# ----------------------------------------------------------------------------------------------
def raft_small_param_shapes():
    """state_dict contract of RAFT.RAFT(small=True), /root/reference/RAFT/{raft,extractor,update}.py: 106 keys, all
    conv weights and biases (InstanceNorm2d and the cnet's norm_fn='none' hold no parameters)."""
    s = {}

    def conv(name, co, ci, k):
        s[name + ".weight"] = (co, ci, k, k)
        s[name + ".bias"] = (co,)

    def enc(pre, out_dim):
        conv(pre + ".conv1", 32, 3, 7)
        cin = 32
        for li, (dim, stride) in enumerate(((32, 1), (64, 2), (96, 2)), start=1):
            for bi in range(2):
                k = f"{pre}.layer{li}.{bi}"
                ci = cin if bi == 0 else dim
                conv(k + ".conv1", dim // 4, ci, 1)
                conv(k + ".conv2", dim // 4, dim // 4, 3)
                conv(k + ".conv3", dim, dim // 4, 1)
                if bi == 0 and stride != 1:
                    conv(k + ".downsample.0", dim, ci, 1)
            cin = dim
        conv(pre + ".conv2", out_dim, 96, 1)

    enc("fnet", 128)
    enc("cnet", 96 + 64)
    u = "update_block."
    conv(u + "encoder.convc1", 96, 196, 1)
    conv(u + "encoder.convf1", 64, 2, 7)
    conv(u + "encoder.convf2", 32, 64, 3)
    conv(u + "encoder.conv", 80, 128, 3)
    for g in "zrq":
        conv(u + f"gru.conv{g}", 96, 96 + 146, 3)
    conv(u + "flow_head.conv1", 128, 96, 3)
    conv(u + "flow_head.conv2", 2, 128, 3)
    return s


def raft_small_state_dict(seed=0, flow_gain=0.5):
    """Seeded small-RAFT weights, drawn like raft_state_dict: He-style conv weights (gain 1.4, 1.0 for the GRU,
    flow_gain for the flow head's last conv) and small random biases."""
    sd = {}
    for key, shape in raft_small_param_shapes().items():
        g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(key.encode())) & 0x7FFFFFFF)
        if len(shape) == 4:
            gain = flow_gain if "flow_head.conv2" in key else 1.0 if "gru.conv" in key else 1.4
            sd[key] = torch.randn(shape, generator=g) * (gain / math.sqrt(shape[1] * shape[2] * shape[3]))
        else:
            sd[key] = 0.05 * torch.randn(shape, generator=g)
    return sd


# ----------------------------------------------------------------------------------------------
# flow-guided gradient propagation (get_flowNN_gradient)
# ----------------------------------------------------------------------------------------------
def prop_inputs(seed=0, H=64, W=96, N=6):
    """numpy inputs shaped like the driver's call (tool/video_inpainting.py:585-633): gradients
    [H,W,3,N] float32 (zero under the dilated mask), mask [H,W,N] bool (a moving box + a static blob),
    forward / backward flows [H,W,2,N-1] float32 that are approximately mutually consistent."""
    import numpy as np
    g = torch.Generator().manual_seed(seed)
    fl = _smooth(torch.randn(N - 1, 2, H, W, generator=g), k=11) * 25.0 + torch.tensor([1.5, -0.8]).view(1, 2, 1, 1)
    noise = _smooth(torch.randn(N - 1, 2, H, W, generator=g), k=5) * 1.5
    flow_f = fl.permute(2, 3, 1, 0).contiguous().numpy().astype(np.float32)
    flow_b = (-fl + noise).permute(2, 3, 1, 0).contiguous().numpy().astype(np.float32)
    mask = np.zeros((H, W, N), dtype=bool)
    for t in range(N):
        y0, x0 = H // 4 + t, W // 5 + 2 * t
        mask[y0:y0 + H // 3, x0:x0 + W // 3, t] = True
        mask[H - 14:H - 4, W - 20:W - 6, t] = True
    gx = torch.randn(H, W, 3, N, generator=g).numpy().astype(np.float32)
    gy = torch.randn(H, W, 3, N, generator=g).numpy().astype(np.float32)
    for t in range(N):
        gx[mask[:, :, t], :, t] = 0
        gy[mask[:, :, t], :, t] = 0
    return gx, gy, mask, flow_f, flow_b


def regionfill_inputs(seed=0, B=4, H=48, W=64):
    """Images [B,H,W] float32 (smooth flow-like fields) and hole masks [B,H,W] bool exercising the cases of
    tool/utils/region_fill.py: interior box, blob touching the image border and a corner (3- and 2-neighbour
    rows), several components, a one-pixel hole, an empty mask (last image when B >= 4)."""
    import numpy as np
    g = torch.Generator().manual_seed(seed)
    img = (_smooth(torch.randn(B, 1, H, W, generator=g), k=9)[:, 0] * 20.0).numpy().astype(np.float32)
    mask = np.zeros((B, H, W), dtype=bool)
    for b in range(B):
        if B >= 4 and b == B - 1:
            continue                                     # empty mask: image returned unchanged
        mask[b, H // 4 + b:H // 4 + b + H // 3, W // 5:W // 5 + W // 3 + 2 * b] = True
        if b % 3 == 0:
            mask[b, :H // 6, :W // 7] = True             # touches the top-left corner
            mask[b, H - 1, W // 2] = True                # single pixel on the bottom border
        if b % 3 == 1:
            mask[b, H - H // 5:, W - W // 4:] = True     # touches the bottom-right corner
            mask[b, 2, W - 1] = True
        if b % 3 == 2:
            mask[b, H // 2:H // 2 + 3, W - 6:] = True    # touches the right border only
        img[b][mask[b]] = 0.0                            # the driver zeroes the flow under the mask
    return img, mask


# ----------------------------------------------------------------------------------------------
# Poisson blending (Poisson_blend_img)
# ----------------------------------------------------------------------------------------------
def poisson_inputs(seed=0, F=3, H=64, W=96, with_edge=False):
    """numpy inputs shaped like the driver's per-frame call (tool/video_inpainting.py:645-656), stacked over F
    frames: target frames [F,H,W,3] float32 in [0,1] (zero inside the hole), forward-difference gradients
    gx [F,H,W-1,3] / gy [F,H-1,W,3] float32 (source gradients + noise, i.e. not integrable: the system is
    genuinely over-determined), hole masks [F,H,W] bool (interior box, a component touching the bottom-right
    corner, a one-pixel hole; the last frame of F >= 3 has an empty hole), gradient masks [F,H,W] bool (a solid
    block inside the box = gradients unknown there, plus one small component entirely without gradients) and,
    with_edge, an edge map [F,H,W] float32 (a line crossing the box)."""
    import numpy as np
    g = torch.Generator().manual_seed(seed)
    src = _smooth(torch.rand(F, 3, H, W, generator=g), k=9)
    src = (src - src.amin()) / (src.amax() - src.amin())
    src = (src.permute(0, 2, 3, 1) + 0.05 * torch.randn(F, H, W, 3, generator=g)).clamp(0, 1).numpy().astype(np.float32)
    hole = np.zeros((F, H, W), dtype=bool)
    gm = np.zeros((F, H, W), dtype=bool)
    for f in range(F):
        if F >= 3 and f == F - 1:
            continue
        y0, x0 = H // 4 + f, W // 5 + 2 * f
        hole[f, y0:y0 + H // 3, x0:x0 + W // 3] = True
        hole[f, H - H // 5:, W - W // 4:] = True
        hole[f, 2, W // 2] = True
        hole[f, H // 8:H // 8 + 3, W - 9:W - 5] = True
        gm[f, y0 + H // 8:y0 + H // 5, x0 + W // 8:x0 + W // 5] = True
        gm[f, H // 8 - 1:H // 8 + 4, W - 10:W - 4] = True       # this component has no usable gradient at all
    trg = src.copy()
    trg[hole] = 0
    gx = (np.diff(src, axis=2) + 0.02 * torch.randn(F, H, W - 1, 3, generator=g).numpy()).astype(np.float32)
    gy = (np.diff(src, axis=1) + 0.02 * torch.randn(F, H - 1, W, 3, generator=g).numpy()).astype(np.float32)
    if not with_edge:
        return trg, gx, gy, hole, gm
    edge = np.zeros((F, H, W), dtype=np.float32)
    edge[:, H // 3, :] = 1.0
    return trg, gx, gy, hole, gm, edge


# ----------------------------------------------------------------------------------------------
# whole driver pipeline (tool/video_inpainting.py::video_inpainting)
# ----------------------------------------------------------------------------------------------
def pipeline_clip(seed=5, N=7, H=64, W=96):
    """What the driver reads from disk: N uint8 RGB frames [H,W,3] (a smooth texture translating by (2, 1) px per
    frame) and N uint8 masks [H,W] (255 = remove; a box moving with the texture)."""
    import numpy as np
    g = torch.Generator().manual_seed(seed)
    big = _smooth(torch.rand(1, 3, H + 64, W + 64, generator=g), k=7)[0]
    big = (big - big.amin()) / (big.amax() - big.amin())
    frames, masks = [], []
    for i in range(N):
        y0, x0 = 16 + i, 16 + 2 * i
        frames.append((big[:, y0:y0 + H, x0:x0 + W].permute(1, 2, 0).numpy() * 255).astype(np.uint8))
        m = np.zeros((H, W), np.uint8)
        m[H // 3 + i:H // 3 + H // 4 + i, W // 3 + 2 * i:W // 3 + W // 4 + 2 * i] = 255
        masks.append(m)
    return frames, masks


# ----------------------------------------------------------------------------------------------
# clip scoring (fgt_b200/metrics.py)
# ----------------------------------------------------------------------------------------------
def _box(x, r):
    """Integer box sum of half-width r along axes 1 and 2 of an int64 [N,H,W,C] array (valid part only)."""
    import numpy as np
    for ax in (1, 2):
        c = np.cumsum(np.pad(x, [(1, 0) if a == ax else (0, 0) for a in range(4)]), axis=ax)
        n = x.shape[ax] - 2 * r
        x = np.take(c, range(2 * r + 1, 2 * r + 1 + n), axis=ax) - np.take(c, range(n), axis=ax)
    return x


def metric_pair(seed, N, H, W, C, kind, dtype):
    """(results, gts) [N,H,W,C] numpy arrays of `dtype` ('u8' or 'f32') on the 0..255 scale for scoring
    (fgt_b200/metrics.py): a smooth integer texture as the ground truth, and as the result the ground truth plus
    quarter-level noise (kind "noise"), its 3x3 box blur ("blur") or the ground truth itself ("same"). Integer
    arithmetic and exact float64 divisions only, so every machine regenerates the arrays bit for bit."""
    import numpy as np
    g = np.random.default_rng(seed)
    tex = _box(g.integers(0, 256, (N, H + 10, W + 10, C)), 4)[:, 1:-1, 1:-1]       # [N, H, W, C] box sums of 81
    lo, hi = tex.min(), tex.max()
    gt = (tex - lo) * 255 // max(hi - lo, 1)
    if kind == "noise":
        res = gt + g.integers(-48, 49, gt.shape) / 4.0
    elif kind == "blur":
        res = _box(np.pad(gt, [(0, 0), (1, 1), (1, 1), (0, 0)], mode="edge"), 1) / 9.0
    else:
        res = gt.astype(np.float64)
    res = np.clip(res, 0, 255)
    if dtype == "u8":
        return np.floor(res + 0.5).astype(np.uint8), gt.astype(np.uint8)
    return res.astype(np.float32), gt.astype(np.float32)


# ----------------------------------------------------------------------------------------------
# forward flow splatting (LAFC/models/utils/flow_warp.py)
# ----------------------------------------------------------------------------------------------
def flow_warp_inputs(seed=0, b=2, c=5, h=20, w=28):
    """Features [b,c,h,w] and a flow [b,2,h,w] with sub-pixel, exactly integer, negative and out-of-image targets."""
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(b, c, h, w, generator=g)
    flow = torch.randn(b, 2, h, w, generator=g) * 3.0
    flow[:, :, : h // 4] = torch.round(flow[:, :, : h // 4])          # integer displacements
    flow[:, :, :, -2:] += 40.0                                         # pushed out of the image
    flow[0, :, h // 2, : w // 2] = 0.0                                 # identity
    return feat, flow


# ----------------------------------------------------------------------------------------------
# flow colour coding (fgt_b200/flowviz.py)
# ----------------------------------------------------------------------------------------------
def vis_flows(seed, B, H, W, scale=8.0):
    """Flows [B,H,W,2] float32 shaped like RAFT's: per image a sum of three random plane waves of `scale` pixels
    (different in u and v), a constant drift and a little pixel noise, so every direction of the colour wheel occurs
    and each image has its own maximum."""
    import numpy as np
    g = np.random.default_rng(seed)
    ys, xs = np.arange(H, dtype=np.float32)[:, None], np.arange(W, dtype=np.float32)[None, :]
    out = np.empty((B, H, W, 2), np.float32)
    for b in range(B):
        s = np.float32(scale * g.uniform(0.25, 2.0))
        for c in range(2):
            acc = np.full((H, W), g.normal(0.0, 0.5) * s, np.float32)
            for _ in range(3):
                fy, fx, ph = g.uniform(-0.05, 0.05), g.uniform(-0.05, 0.05), g.uniform(0, 2 * np.pi)
                acc += s * np.float32(g.uniform(0.3, 1.0)) * np.sin(ys * np.float32(fy) + xs * np.float32(fx) +
                                                                    np.float32(ph))
            out[b, :, :, c] = acc + np.float32(0.05) * s * g.standard_normal((H, W), dtype=np.float32)
    return out
