"""LAFC mixed precision on the H100: the reference flow-completion network under CUDA autocast
(oracle/lafc_mixed_oracle.py), with synthetic weights. The CPU emulation of autocast's casts is pinned to real autocast
op by op; our fp16 path is held to a multiple of the reference's own mixed-precision error E_ref (relative L2 of the
autocast oracle against the fp32 oracle on the same input), and to an absolute distance from our fp32 path."""
import argparse
import contextlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fgt_b200 import lib, synth
from oracle import lafc_mixed_oracle as LM
from tests.util import load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _strip(sd):
    return {k[4:]: v for k, v in sd.items()}


def _model(sd, mixed=True):
    from fgt_b200.lafc_model import Model
    m = Model(dict(synth.CFG_LAFC))
    m.load_state_dict(sd)
    m = m.to(DEV).eval()
    m.net.enable_mixed_precision(mixed)
    return m


@contextlib.contextmanager
def _no_tf32():
    """The fp32 oracle on CUDA: cuDNN's fp32 convolutions would otherwise run in TF32."""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _ulp16(a):
    return torch.exp2(torch.floor(torch.log2(a.abs().clamp_min(2.0 ** -14))) - 10)


def _agree(x, ref):
    """(fraction bit-equal, fraction within one fp16 ulp of ref) over the elements."""
    x, ref = x.float().cpu(), ref.float().cpu()
    return (x == ref).float().mean().item(), ((x - ref).abs() <= _ulp16(ref)).float().mean().item()


def _rel(a, b):
    a, b = a.double().cuda(), b.double().cuda()
    return ((a - b).norm() / b.norm()).item()


def test_emulation_rules_match_autocast():
    """Each rule of the CPU emulation against the same op under real CUDA autocast, on identical fp16-valued inputs, and
    the fp32 ops against the same reference. Convolutions: cuDNN's fp16 result is not always the correctly rounded one,
    so the rule is held to one fp16 ulp; the elementwise rules are held to bit equality. Measured on an H100 80GB HBM3:
    a conv lands bit-equal on 99.2-99.8 % of autocast's outputs and within one ulp on >= 99.87 % (fp32 convs: 78 %
    within one ulp); a residual P3D block and the edge head on 99.5 % / 99.7 %; LeakyReLU and sigmoid bit-equal
    everywhere. The bounds leave a margin of about 1 % of the outputs."""
    q = LM.round_f16
    g = torch.Generator().manual_seed(0)
    sd = _strip(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=7, regime="kaiming"))
    sdc = {k: v.cuda() for k, v in sd.items()}

    def check(name, f, args, min_equal=None, min_within=None):
        with torch.no_grad():
            with torch.autocast("cuda", torch.float16):
                ref = f(*[a.cuda().half() for a in args], sdc, None)   # inside the network every input is fp16
            eq, w1 = _agree(f(*args, sd, q), ref)
            eq32, w32 = _agree(f(*args, sd, None), ref)
        print(f"{name}: emulation equal {eq:.4f} within-1-ulp {w1:.4f}; fp32 equal {eq32:.4f} within-1-ulp {w32:.4f}")
        if min_equal is not None:
            assert eq >= min_equal and eq > eq32, (name, eq, eq32)
        if min_within is not None:
            assert w1 >= min_within and w1 > w32, (name, w1, w32)

    x5 = q(F.leaky_relu(torch.randn(1, 48, 3, 40, 56, generator=g), 0.2))
    x96 = q(F.leaky_relu(torch.randn(1, 96, 3, 20, 28, generator=g), 0.2))
    y192 = q(F.leaky_relu(torch.randn(1, 192, 20, 28, generator=g), 0.2))
    # conv + LeakyReLU(0.2): (1,3,3) stride 2, (3,1,1) with zero z-padding, the (T,1,1) condense, dilated 3x3
    check("P3D conv1 (1,3,3) s2", lambda x, s, q: LM._c3(x, s, "encoder2.2.conv1", q, stride=(1, 2, 2), pad=(0, 1, 1)),
          (x5,), min_within=0.99)
    check("P3D conv2 (3,1,1)", lambda x, s, q: LM._c3(x, s, "encoder4.0.conv2", q, pad=(1, 0, 0)), (x96,),
          min_within=0.99)
    check("condense (3,1,1)", lambda x, s, q: LM._c3(x, s, "condense2", q).squeeze(2), (x96,), min_within=0.99)
    check("middle dilation 8", lambda x, s, q: LM._c2(x, s, "middle.0", q, pad=8, dil=8), (y192,), min_within=0.99)
    # the whole residual P3D block (feats + feat2 in fp16)
    check("P3D residual block", lambda x, s, q: LM.p3d_block(x, s, "encoder4.0", 3, 1, 1, True, q), (x96,),
          min_within=0.98)
    # decoder conv on the nearest-upsampled skip concat; the final flow conv without activation
    d = q(torch.randn(1, 96, 20, 28, generator=g))
    check("decoder.0 upsample + cat + conv",
          lambda a, s, q: LM._c2(F.interpolate(torch.cat([a, a.flip(1)], 1), scale_factor=2), s, "decoder.0.conv", q),
          (d,), min_within=0.99)
    e = q(F.leaky_relu(torch.randn(1, 24, 40, 56, generator=g), 0.2))
    check("decoder.2 (flow)", lambda a, s, q: LM._c2(a, s, "decoder.2", q, act=False), (e,), min_within=0.99)
    # elementwise rules on fp16 inputs: LeakyReLU(0.2), LeakyReLU(0.01) of a residual sum, sigmoid
    a = q(torch.randn(1, 16, 40, 56, generator=g) * 4)
    b = q(torch.randn(1, 16, 40, 56, generator=g) * 4)
    Q = lambda q: q or (lambda t: t)  # noqa: E731
    check("LeakyReLU(0.2)", lambda a, s, q: Q(q)(F.leaky_relu(a, 0.2)), (a,), min_equal=0.999)
    check("LeakyReLU(0.01)(p + e)", lambda a, b, s, q: Q(q)(F.leaky_relu(Q(q)(a + b), 0.01)), (a, b), min_equal=0.999)
    check("sigmoid", lambda a, s, q: Q(q)(torch.sigmoid(a)), (a,), min_equal=0.999)
    # the edge head from the same fp16 flow
    fl = q(torch.randn(1, 2, 40, 56, generator=g) * 5)
    check("edge head", lambda f, s, q: LM.edge_head(f, s, q), (fl,), min_within=0.98)


def test_upsample2x_f16_is_an_exact_nearest_copy():
    """The single-plane fp16 form (both plane offsets 0): out[y, x] = in[y // 2, x // 2] bit for bit (the float64
    interpreter of a nearest x2 is this index map), and no byte outside the output changes."""
    g = torch.Generator().manual_seed(1)
    n, H, W, C = 2, 13, 21, 96
    x = (torch.randn(n, H, W, C, generator=g) * 100).half().to(DEV)
    x.view(-1)[::97] = float("inf")
    x.view(torch.int16).view(-1)[5::101] = 0x7E01        # NaN payloads travel as bits
    guard = 4096
    buf = torch.full((n * 2 * H * 2 * W * C + 2 * guard,), 12345, dtype=torch.int16, device=DEV)
    out = buf[guard:-guard].view(torch.float16).view(n, 2 * H, 2 * W, C)
    lib.upsample2x(x, n, H, W, C, out)
    torch.cuda.synchronize()
    want = x.view(torch.int16).repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert torch.equal(out.view(torch.int16), want)
    assert (buf[:guard] == 12345).all() and (buf[-guard:] == 12345).all()
    with pytest.raises(RuntimeError, match="plane offsets"):   # split input, fp16 output
        lib.upsample2x(lib.empty_split((n, H, W, C), DEV), n, H, W, C, out)


def _oracle(sd, fl, mk, mixed):
    sdc = {k: v.cuda() for k, v in _strip(sd).items()}
    with torch.no_grad(), _no_tf32():
        return LM.lafc_forward(sdc, fl.cuda(), mk.cuda(), mixed_precision=mixed)


# Bound on ours-mixed vs autocast, in E_ref: measured 0.68-1.05 E_ref (flow and edge, H100 80GB HBM3), where two
# independent fp16 roundings of one model are expected to differ by about sqrt(2) E_ref; the bound is twice that.
CASES = [  # name, H, W, regime, weight seed, input seed, bound on ours-vs-autocast in E_ref
    ("lafc_small_kaiming", 64, 96, "kaiming", 4, 5, 2.0),
    ("lafc_small_scaled", 64, 96, "scaled", 4, 5, 2.0),
    ("256x432", 256, 432, "scaled", 11, 12, 2.0),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_mixed_vs_autocast(case):
    name, H, W, regime, wseed, iseed, bound = case
    if name.startswith("lafc_small"):
        meta = load_golden(name)["meta"]   # the golden's own geometry and weight draw
        H, W, regime, wseed, iseed = meta["H"], meta["W"], meta["regime"], meta["seed"], meta["seed"] + 1
    sd = synth.make_state_dict(synth.lafc_param_shapes(), seed=wseed, regime=regime)
    fl, mk = synth.lafc_inputs(seed=iseed, H=H, W=W)
    ref32 = _oracle(sd, fl, mk, False)
    ref16 = _oracle(sd, fl, mk, True)
    m16 = _model(sd, True)
    m32 = _model(sd, False)
    with torch.no_grad():
        o16 = m16(fl.to(DEV), mk.to(DEV))
        o32 = m32(fl.to(DEV), mk.to(DEV))
    torch.cuda.synchronize()
    for what, a16, a32, r16, r32 in zip(("flow", "edge"), o16, o32, ref16, ref32):
        assert a16.dtype == torch.float32 and torch.isfinite(a16).all()
        assert torch.equal(a16, a16.half().float()), what   # fp16 values, returned as fp32
        e_ref = _rel(r16, r32)
        d_ac, d_32 = _rel(a16, r16), _rel(a16, a32)
        print(f"{name} {what}: E_ref {e_ref:.3e}; ours-mixed vs autocast {d_ac:.3e} ({d_ac / e_ref:.2f} E_ref); "
              f"vs ours-fp32 {d_32:.3e}; max |flow| diff {((a16 - a32).abs().max().item()):.4f}")
        assert d_ac <= bound * e_ref, (name, what, d_ac, e_ref)
    flow_err = (o16[0] - o32[0]).abs().max().item()
    assert flow_err <= 0.1, (name, flow_err)   # pixels; measured 0.0006-0.023 px (the largest with kaiming weights)


def test_graph_replay_and_switching():
    """fp16 graph replay equals fp16 eager; turning the mode on and off leaves the fp32 output bit-identical to a fresh
    fp32 model's."""
    sd = synth.make_state_dict(synth.lafc_param_shapes(), seed=21)
    fl, mk = [t.to(DEV) for t in synth.lafc_inputs(seed=22, H=64, W=96)]
    fresh = _model(sd, False)
    with torch.no_grad():
        want32 = fresh(fl, mk)
        m = _model(sd, True)
        eager16 = m(fl, mk)
        m.net.enable_cuda_graph(True)
        m(fl, mk)                       # eager call of the graph entry
        m(fl, mk)                       # capture + replay
        g16 = m(fl, mk)
        m.net.enable_mixed_precision(False)
        g32 = m(fl, mk)
        g32b = m(fl, mk)
        m.net.enable_mixed_precision(True)
        g16b = m(fl, mk)
        m.net.enable_cuda_graph(False)
        m.net.enable_mixed_precision(False)
        e32 = m(fl, mk)
    torch.cuda.synchronize()
    for a, b in zip(g16, eager16):
        assert torch.equal(a, b)
    for a, b in zip(g16b, eager16):
        assert torch.equal(a, b)
    for got in (g32, g32b, e32):
        for a, b in zip(got, want32):
            assert torch.equal(a, b)
    assert not torch.equal(eager16[0], want32[0])


def test_pipeline_with_all_three_mixed_modes():
    """One pipeline run on the pipeline_clip inputs with RAFT, LAFC and FGT in fp16, against the same run in fp32."""
    from fgt_b200 import pipeline as PL
    from fgt_b200.fgt_model import Model as FGTModel
    from fgt_b200.lafc_model import Model as LAFCModel
    from fgt_b200.raft_model import RAFT
    frames, masks = synth.pipeline_clip(seed=5, N=7, H=64, W=96)
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    outs = {}
    for mixed in (False, True):
        fgt = FGTModel(cfg)
        fgt.load_state_dict(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=31))
        fgt.net.enable_mixed_precision(mixed)
        lafc = LAFCModel(dict(synth.CFG_LAFC))
        lafc.load_state_dict(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=32))
        lafc.net.enable_mixed_precision(mixed)
        raft = RAFT(argparse.Namespace(small=False, mixed_precision=mixed, alternate_corr=False))
        raft.load_state_dict(synth.raft_state_dict(seed=33))
        be = PL.GpuBackend(raft.to(DEV).eval(), lafc.to(DEV), fgt.to(DEV), device=torch.device(DEV))
        args = PL.make_args(imgH=64, imgW=96, flow_mask_dilates=3, frame_dilates=1)
        outs[mixed] = PL.video_inpainting(frames, masks, be, args)
        assert lafc.net._mixed is mixed and (True in lafc.net._packed) is mixed
    a, b = (np.stack([np.asarray(f) for f in outs[k]]) for k in (True, False))
    assert a.shape == b.shape and len(outs[True]) == len(frames) and a.dtype == np.uint8
    diff = np.abs(a.astype(np.int16) - b.astype(np.int16))
    print(f"pipeline, all three fp16 modes vs fp32: max {diff.max()} grey levels, mean {diff.mean():.4f}, "
          f"{(diff > 0).mean() * 100:.2f} % of values differ")
    # measured: mean 0.058 grey levels, 3.6 % of the values differ (where a hole pixel's fill source flips, by up to
    # ~100 levels); bounds about 4x and 3x that
    assert diff.mean() <= 0.25 and (diff > 0).mean() <= 0.10


def test_batched_autocast_epilogue_equals_the_per_pair_one():
    """The autocast rounding runs in the batched epilogue (kExt = 2) wherever a tile allows it and in the per-pair one
    (epi_pair's r16 mode) elsewhere; with the previous tile schedule (`fgt_debug_gemm_serial_epilogue(1)`: same MMAs
    in the same order, per-pair epilogue only) the mixed forward gives the same bits."""
    import ctypes
    L = lib.load()
    L.fgt_debug_gemm_serial_epilogue.argtypes = [ctypes.c_int]
    sd = synth.make_state_dict(synth.lafc_param_shapes(), seed=23)
    fl, mk = [t.to(DEV) for t in synth.lafc_inputs(seed=24, H=96, W=160)]
    m = _model(sd, True)
    outs = []
    with torch.no_grad():
        for serial in (0, 1):
            L.fgt_debug_gemm_serial_epilogue(serial)
            try:
                outs.append(m(fl, mk))
                torch.cuda.synchronize()
            finally:
                L.fgt_debug_gemm_serial_epilogue(0)
    for a, b in zip(*outs):
        assert torch.equal(a, b)
