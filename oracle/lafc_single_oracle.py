"""CPU oracle for the single-frame ("2D") LAFC (TEST INFRASTRUCTURE — see oracle/fgt_oracle.py header).

Functional PyTorch-CPU restatement of /root/reference/FGT/models/lafc_single.py (P3DNet.forward :70-89,
EdgeDetection.forward :105-112) with the blocks of FGT/models/utils/network_blocks_2d.py (VanillaConv :7-43: conv then
LeakyReLU(0.2) unless activation=None; VanillaDeconv :46-60: nearest x2 then VanillaConv) and
FGT/models/utils/reconstructionLayers.py:34-61 (ResidualBlock_noBN). Pinned by tests/golden/lafc_single_*.npz
(outputs of the unmodified reference, written by tests/golden/make_lafc_single_golden.py).
"""
import torch
import torch.nn.functional as F

LEAK = 0.2


def _c2(x, sd, key, pad=1, stride=1, dil=1, act=True):
    """VanillaConv.forward, network_blocks_2d.py:37-43."""
    y = F.conv2d(x, sd[key + ".featureConv.weight"], sd[key + ".featureConv.bias"], stride=stride, padding=pad,
                 dilation=dil)
    return F.leaky_relu(y, LEAK) if act else y


def _up(x):
    """VanillaDeconv's F.interpolate(scale_factor=2), nearest (network_blocks_2d.py:58-60)."""
    return F.interpolate(x, scale_factor=2)


def lafc_single_forward(sd, flows, masks, res_blocks=1):
    """P3DNet.forward, lafc_single.py:70-89, PASSMASK=1 and edges=None. sd = Model.state_dict() with 'net.' stripped.
    flows [n,2,H,W], masks [n,1,H,W] -> (flow [n,2,H,W], edge [n,1,H,W])."""
    x = F.pad(torch.cat([flows, masks], 1), (2, 2, 2, 2), mode="replicate")  # nn.ReplicationPad2d(2), :27
    e2 = _c2(x, sd, "encoder2.1", pad=0)
    e2 = _c2(e2, sd, "encoder2.2", stride=2)
    e4 = _c2(e2, sd, "encoder4.0")
    e4 = _c2(e4, sd, "encoder4.1", stride=2)
    y = e4
    for i in range(res_blocks):   # make_layer: res_blocks separate blocks (:36-38)
        k = f"res_blocks.{i}"
        r = F.leaky_relu(F.conv2d(y, sd[k + ".conv1.weight"], sd[k + ".conv1.bias"], padding=1), LEAK)
        y = y + F.conv2d(r, sd[k + ".conv2.weight"], sd[k + ".conv2.bias"], padding=1)   # no activation after the add
    for i, d in enumerate((8, 4, 2, 1)):
        y = _c2(y, sd, f"middle.{i}", pad=d, dil=d)
    y = torch.cat([y, e4], 1)                                   # :84
    y = _c2(_up(y), sd, "decoder2.0.conv")
    y = _c2(y, sd, "decoder2.1")
    y = _c2(y, sd, "decoder2.2")
    y = torch.cat([y, e2], 1)                                   # :86
    y = _c2(_up(y), sd, "decoder.0.conv")
    y = _c2(y, sd, "decoder.1")
    flow = _c2(y, sd, "decoder.2")   # the default LeakyReLU(0.2) is kept on the completed flow (:61-62)
    p = _c2(flow, sd, "edgeDetector.projection")
    e = _c2(p, sd, "edgeDetector.mid_layer_1")
    e = _c2(e, sd, "edgeDetector.mid_layer_2", act=False)
    e = F.leaky_relu(p + e, 0.01)  # nn.LeakyReLU() default slope, :109
    e = _c2(e, sd, "edgeDetector.out_layer", pad=0, act=False)
    return flow, torch.sigmoid(e)
