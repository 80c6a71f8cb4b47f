"""LAFC oracle with autocast's mixed precision (TEST INFRASTRUCTURE — see oracle/fgt_oracle.py header).

The same functional restatement as oracle/lafc_oracle.py (LAFC/models/lafc.py P3DNet.forward :84-105, P3DBlock
:118-125, EdgeDetection :141-148), device-agnostic, with a precision switch. With mixed_precision=False it computes
exactly what lafc_oracle.lafc_forward computes (tests/test_lafc_mixed.py checks torch.equal); lafc_oracle.py itself is
left as the golden-pinned fp32 definition.

Mixed precision (`lafc_forward(..., mixed_precision=True)`) is the reference module run under
torch.autocast("cuda", dtype=torch.float16); the reference LAFC has no precision flag of its own. On CUDA tensors the
oracle runs the restatement under autocast. On CPU tensors it emulates autocast's casts explicitly: every function below
takes `q`, the rounding to fp16 (values stay fp32 tensors holding fp16 numbers; q=None is fp32). The rules, one per op
the network uses, each what autocast does to the reference's code:
  * Conv3d / Conv2d cast input, weight and bias to fp16, accumulate in fp32 and give an fp16 output (`_conv`; every
    VanillaConv / VanillaConv2d, network_blocks.py:33-39, network_blocks_2d.py:37-43);
  * LeakyReLU(0.2) after each conv, and the edge head's LeakyReLU(0.01) (lafc.py:138,146), on fp16 give fp16;
  * ReplicationPad3d runs on the fp32 input (no autocast rule; the first conv casts the padded tensor), nearest x2
    upsampling and torch.cat of fp16 tensors keep the dtype: no rounding;
  * the residual adds `feats + feat2` (lafc.py:122) and `flow + edge` (lafc.py:146) add two fp16 tensors into fp16;
  * torch.sigmoid (lafc.py:148) on fp16 gives fp16.
Autocast's outputs are fp16; the oracle returns them as fp32 tensors (the fp16 values), as the native module does.
"""
import torch
import torch.nn.functional as F

LEAK = 0.2


def _id(t):
    return t


def round_f16(t):
    """fp32 tensor -> the nearest fp16 values, kept as fp32 (the CPU emulation's rounding)."""
    return t.half().float()


def _conv(x, sd, key, q, **kw):
    w, b = sd[key + ".featureConv.weight"], sd[key + ".featureConv.bias"]
    conv = F.conv3d if w.dim() == 5 else F.conv2d
    if q is None:
        return conv(x, w, b, **kw)
    return q(conv(q(x), q(w), q(b), **kw))


def _c3(x, sd, key, q, stride=(1, 1, 1), pad=(0, 0, 0), act=True):
    """VanillaConv (3-D): Conv3d then LeakyReLU(0.2)."""
    y = _conv(x, sd, key, q, stride=stride, padding=pad)
    return (q or _id)(F.leaky_relu(y, LEAK)) if act else y


def _c2(x, sd, key, q, pad=1, dil=1, act=True):
    """VanillaConv2d: Conv2d then LeakyReLU(0.2)."""
    y = _conv(x, sd, key, q, padding=pad, dilation=dil)
    return (q or _id)(F.leaky_relu(y, LEAK)) if act else y


def p3d_block(x, sd, key, k, stride, pad, residual, q=None):
    """P3DBlock.forward: (1,k,k) conv then (3,1,1) conv, optional identity add."""
    y = _c3(x, sd, key + ".conv1", q, stride=(1, stride, stride), pad=(0, pad, pad))
    y = _c3(y, sd, key + ".conv2", q, pad=(1, 0, 0))
    return (q or _id)(x + y) if residual else y


def edge_head(flow, sd, q=None):
    """EdgeDetection.forward, lafc.py:141-148."""
    Q = q or _id
    p = _c2(flow, sd, "edgeDetector.projection", q)
    e = _c2(p, sd, "edgeDetector.mid_layer_1", q)
    e = _c2(e, sd, "edgeDetector.mid_layer_2", q, act=False)
    e = Q(F.leaky_relu(Q(p + e), 0.01))
    e = _c2(e, sd, "edgeDetector.out_layer", q, pad=0, act=False)
    return Q(torch.sigmoid(e))


def _forward(sd, flows, masks, use_residual, res_blocks, q):
    x = torch.cat([flows, masks], 1)
    x = F.pad(x, (2, 2, 2, 2, 0, 0), mode="replicate")
    e2 = p3d_block(x, sd, "encoder2.1", 5, 1, 0, False, q)
    e2 = p3d_block(e2, sd, "encoder2.2", 3, 2, 1, False, q)
    c_e2_pre = _c3(e2, sd, "condense2", q).squeeze(2)
    e4 = p3d_block(e2, sd, "encoder4.0", 3, 1, 1, bool(use_residual), q)
    e4 = p3d_block(e4, sd, "encoder4.1", 3, 2, 1, False, q)
    c_e4_pre = _c3(e4, sd, "condense4_pre", q).squeeze(2)
    for _ in range(res_blocks):
        e4 = p3d_block(e4, sd, "res_blocks.0", 3, 1, 1, True, q)
    y = _c3(e4, sd, "condense4_post", q).squeeze(2)
    for i, d in enumerate((8, 4, 2, 1)):
        y = _c2(y, sd, f"middle.{i}", q, pad=d, dil=d)
    y = torch.cat([y, c_e4_pre], 1)
    y = _c2(F.interpolate(y, scale_factor=2), sd, "decoder2.0.conv", q)
    y = _c2(y, sd, "decoder2.1", q)
    y = _c2(y, sd, "decoder2.2", q)
    y = torch.cat([y, c_e2_pre], 1)
    y = _c2(F.interpolate(y, scale_factor=2), sd, "decoder.0.conv", q)
    y = _c2(y, sd, "decoder.1", q)
    flow = _c2(y, sd, "decoder.2", q, act=False)
    return flow, edge_head(flow, sd, q)


def lafc_forward(sd, flows, masks, use_residual=1, res_blocks=1, mixed_precision=False):
    """P3DNet.forward. sd = Model.state_dict() with 'net.' stripped; flows [b,2,T,H,W], masks [b,1,T,H,W] ->
    (flow [b,2,H,W], edge [b,1,H,W]), fp32. mixed_precision: autocast on CUDA tensors, the emulation above on CPU
    tensors."""
    if not mixed_precision:
        return _forward(sd, flows, masks, use_residual, res_blocks, None)
    if flows.device.type == "cuda":
        with torch.autocast("cuda", torch.float16):
            flow, edge = _forward(sd, flows, masks, use_residual, res_blocks, None)
        return flow.float(), edge.float()
    return _forward(sd, flows, masks, use_residual, res_blocks, round_f16)
