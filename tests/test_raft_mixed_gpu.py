"""RAFT mixed precision on the H100 (the reference's --mixed_precision: fnet, cnet and the update block under CUDA
autocast, RAFT/raft.py:100,111,128), with synthetic weights. The definition is the oracle under real CUDA autocast; the
CPU emulation of its casts is pinned to it here. Our fp16 path is held to twice the reference's own mixed-precision
error E_ref (mean end-point error of the autocast oracle against the fp32 oracle on the same input): two independent
fp16 roundings of the same model differ by about sqrt(2) E_ref."""
import argparse
import contextlib

import numpy as np
import pytest
import torch

from fgt_b200 import synth
from oracle import raft_mixed_oracle as RO
from tests.util import assert_close

pytestmark = pytest.mark.gpu


def _model(seed, mixed=True):
    from fgt_b200.raft_model import RAFT
    sd = synth.raft_state_dict(seed=seed)
    m = RAFT(argparse.Namespace(small=False, mixed_precision=mixed, alternate_corr=False))
    m.load_state_dict(sd)
    return m.cuda().eval(), sd


@contextlib.contextmanager
def _no_tf32():
    """The fp32 oracle on CUDA: cuDNN's fp32 convolutions would otherwise run in TF32."""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _oracle(sd, im1, im2, iters, mixed):
    sdc = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad(), _no_tf32():
        lo, up = RO.raft_forward(sdc, im1.cuda(), im2.cuda(), iters=iters, mixed_precision=mixed)
    return lo.float(), up.float()


def _epe(a, b):
    return (a.float().cuda() - b.float().cuda()).norm(dim=1).mean().item()


def _ulp16(a):
    return torch.exp2(torch.floor(torch.log2(a.abs().clamp_min(2.0 ** -14))) - 10)


def _agree(x, ref):
    """(fraction bit-equal, fraction within one fp16 ulp of ref) over the elements."""
    x, ref = x.float().cpu(), ref.float().cpu()
    return (x == ref).float().mean().item(), ((x - ref).abs() <= _ulp16(ref)).float().mean().item()


def test_emulation_rules_match_autocast():
    """Each rule of the CPU emulation against the same op under real CUDA autocast, on identical fp16-valued inputs, and
    the fp32 oracle against the same ops. Autocast's own fp16 convolutions (cuDNN) land on the correctly rounded value
    for about 72 % of the outputs and within one fp16 ulp for > 99 %; over several layers those one-ulp flips compound,
    which is why the rules are checked op by op (and one update-block step from the same state) rather than through the
    whole network."""
    q = RO.round_f16
    g = torch.Generator().manual_seed(0)
    sd = synth.raft_state_dict(seed=3)
    sdc = {k: v.cuda() for k, v in sd.items()}
    ac = torch.autocast("cuda", torch.float16)

    def check(name, f_ac, f_emu, f_32, min_equal=None, min_within=None, max_equal32=None, max_within32=None,
              region=True):
        with torch.no_grad():
            with torch.autocast("cuda", torch.float16, enabled=region):
                ref = f_ac()
            eq, w1 = _agree(f_emu(), ref)
            eq32, w32 = _agree(f_32(), ref)
        print(f"{name}: emulation equal {eq:.4f} within-1-ulp {w1:.4f}; fp32 equal {eq32:.4f} within-1-ulp {w32:.4f}")
        if min_equal is not None:
            assert eq >= min_equal and eq32 <= max_equal32, (name, eq, eq32)
        if min_within is not None:
            assert w1 >= min_within and w32 <= max_within32, (name, w1, w32)

    x = q(torch.relu(torch.randn(2, 64, 32, 40, generator=g)))
    xc = x.cuda()
    for key, stride, pad in (("cnet.layer1.0.conv1", 1, 1), ("fnet.layer2.0.downsample.0", 2, 0)):
        # a conv casts input, weight and bias to fp16, accumulates in fp32, gives fp16
        check(key, lambda: RO._conv(xc, sdc, key, stride, pad), lambda: RO._conv(x, sd, key, stride, pad, q),
              lambda: RO._conv(x, sd, key, stride, pad), min_within=0.98, max_within32=0.9)
    y = q(torch.randn(2, 64, 32, 40, generator=g) * 3 + 1)
    for key, kind in (("fnet.norm1", "instance"), ("cnet.norm1", "batch")):
        # instance / batch norm: fp16 in, fp32 statistics, fp16 out
        check(kind + " norm", lambda: RO._norm(y.cuda().half(), sdc, key, kind), lambda: RO._norm(y, sd, key, kind, q),
              lambda: RO._norm(y, sd, key, kind), min_equal=0.99, max_equal32=0.01)
    # the GRU: fp16 state, the fp32 flow channels promoted by the cat, fp16 gates and each op of (1-z)h + zq rounded
    h = q(torch.tanh(torch.randn(1, 128, 16, 20, generator=g)))
    xx = torch.cat([q(torch.relu(torch.randn(1, 254, 16, 20, generator=g))), torch.randn(1, 2, 16, 20, generator=g)], 1)
    check("sep_conv_gru", lambda: RO.sep_conv_gru(h.cuda().half(), xx.cuda(), sdc), lambda: RO.sep_conv_gru(h, xx, sd, q=q),
          lambda: RO.sep_conv_gru(h, xx, sd), min_equal=0.6, max_equal32=0.05, min_within=0.8, max_within32=0.7)
    # upsample_flow outside the regions: softmax of the fp16 mask gives fp16, the sum with the fp32 flow is fp32
    m = q(torch.randn(1, 576, 16, 20, generator=g) * 3)
    fl = torch.randn(1, 2, 16, 20, generator=g)
    check("upsample_flow", lambda: RO.upsample_flow(fl.cuda(), m.cuda().half()), lambda: RO.upsample_flow(fl, m, q),
          lambda: RO.upsample_flow(fl, m), min_equal=0.3, max_equal32=0.01, min_within=0.99, max_within32=0.97,
          region=False)
    # one update-block step (motion encoder, GRU, flow and mask heads) from the same fp16 state
    im1, _ = synth.raft_inputs(seed=4, H=128, W=160)
    pre = (2 * (im1 / 255.0) - 1.0).contiguous()
    with torch.no_grad(), ac:
        net, inp = RO.context(pre.cuda(), sdc)
    corr = torch.randn(1, 324, 16, 20, generator=g)
    flow = 0.7 * torch.randn(1, 2, 16, 20, generator=g)
    st = [t.float().cpu() for t in (net, inp)]
    with torch.no_grad():
        with ac:
            ub_ac = RO.update_block(net, inp, corr.cuda(), flow.cuda(), sdc)
        ub_em = RO.update_block(*st, corr, flow, sd, q)
        ub_32 = RO.update_block(*st, corr, flow, sd)
    for name, a, e, f in zip(("net", "mask", "delta"), ub_ac, ub_em, ub_32):
        (eq, w1), (eq32, w32) = _agree(e, a), _agree(f, a)
        print(f"update step {name}: emulation equal {eq:.4f} within-1-ulp {w1:.4f}; fp32 {eq32:.4f} / {w32:.4f}")
        assert eq >= eq32 + 0.2 and w1 >= w32 + 0.03, (name, eq, eq32, w1, w32)


def test_one_iteration_vs_autocast():
    """One update from the initial state. Autocast's own result after one iteration is about 2.5e-3 (relative L2) from
    fp32 on this input, and the CPU emulation, which applies every rounding rule of autocast but accumulates exactly,
    is as far from it (2.5e-3): cuDNN's fp16 convolutions miss the correctly rounded value by one ulp in about a quarter
    of their outputs, and one iteration compounds such one-ulp differences to the 2e-3 level. At this point no fp16
    implementation can be told apart from fp32 by its distance to autocast, so the bound is twice the reference's own
    error; the rules themselves are pinned op by op above, and the full recurrence below."""
    from tests.util import rel_l2
    model, sd = _model(3)
    fp32, _ = _model(3, mixed=False)
    im1, im2 = synth.raft_inputs(seed=4, H=128, W=160)
    with torch.no_grad():
        lo, up = model(im1.cuda(), im2.cuda(), iters=1, test_mode=True)
        lo32, up32 = fp32(im1.cuda(), im2.cuda(), iters=1, test_mode=True)
        elo, eup = RO.raft_forward(sd, im1, im2, iters=1, mixed_precision=True)
    olo, oup = _oracle(sd, im1, im2, 1, True)
    flo, fup = _oracle(sd, im1, im2, 1, False)
    for name, got, g32, emu, ref, f32 in (("low", lo, lo32, elo, olo, flo), ("up", up, up32, eup, oup, fup)):
        r_ref, r_ours = rel_l2(ref, f32), rel_l2(got, ref)
        r_emu16, r_emu32 = rel_l2(got, emu), rel_l2(g32, emu)
        print(f"one iteration {name}: ours vs autocast {r_ours:.3e}; autocast vs fp32 {r_ref:.3e}; emulation vs "
              f"autocast {rel_l2(emu, ref):.3e}; vs the emulation: ours mixed {r_emu16:.3e}, ours fp32 {r_emu32:.3e}")
        assert r_ours <= 2 * r_ref, (name, r_ours, r_ref)


@pytest.mark.parametrize("geo", [(3, 128, 160, 5), (1, 480, 864, 12)], ids=["128x160_b3", "480x864"])
def test_recurrence_within_reference_mixed_error(geo):
    n, H, W, seed = geo
    model, sd = _model(seed)
    fp32, _ = _model(seed, mixed=False)
    im1, im2 = synth.raft_inputs(seed=seed + 1, H=H, W=W, n=n)
    with torch.no_grad():
        lo, up = model(im1.cuda(), im2.cuda(), iters=20, test_mode=True)
        lo32, up32 = fp32(im1.cuda(), im2.cuda(), iters=20, test_mode=True)
    olo, _ = _oracle(sd, im1, im2, 20, True)
    flo, _ = _oracle(sd, im1, im2, 20, False)
    e_ref = _epe(olo, flo)
    e_ours = _epe(lo, olo)
    e_self = _epe(lo, lo32)
    print(f"{n}x{H}x{W}: E_ref {e_ref:.3e}, ours-mixed vs autocast {e_ours:.3e} ({e_ours / e_ref:.2f} E_ref), "
          f"ours-mixed vs ours-fp32 {e_self:.3e} ({e_self / e_ref:.2f} E_ref), |flow| {flo.norm(dim=1).mean():.3f}")
    assert torch.isfinite(lo).all() and torch.isfinite(up).all()
    assert not torch.equal(lo, lo32)  # the flag takes effect
    assert e_ours <= 2 * e_ref
    assert e_self <= 2 * e_ref


def test_batch_flow_init_sequence_and_graphs():
    model, _ = _model(3)
    im1, im2 = synth.raft_inputs(seed=13, H=128, W=160, n=3)
    a, b = im1.cuda(), im2.cuda()
    with torch.no_grad():
        lo, up = model(a, b, iters=5, test_mode=True)
        for i in range(3):  # instance-norm partial sums are split differently per batch: close, not bit-equal
            lo1, up1 = model(a[i:i + 1], b[i:i + 1], iters=5, test_mode=True)
            assert_close(lo[i:i + 1], lo1, 2e-3, f"batch vs single pair {i}")
        z0, zu = model(a, b, iters=2, flow_init=torch.zeros(3, 2, 16, 20, device="cuda"), test_mode=True)
        n0, nu = model(a, b, iters=2, test_mode=True)
        assert torch.equal(zu, nu) and torch.equal(z0, n0)
        f0 = 0.5 * torch.ones(3, 2, 16, 20, device="cuda")
        w0, _ = model(a, b, iters=2, flow_init=f0, test_mode=True)
        assert not torch.equal(w0, n0)
        seq = model(a, b, iters=3, test_mode=False)
        lo3, up3 = model(a, b, iters=3, test_mode=True)
        assert len(seq) == 3 and torch.equal(seq[-1], up3)
        model.enable_cuda_graph(True)
        try:
            g1 = model(a, b, iters=5, test_mode=True)
            g2 = model(a, b, iters=5, test_mode=True)  # replay
        finally:
            model.enable_cuda_graph(False)
    assert torch.equal(g1[0], lo) and torch.equal(g2[0], lo) and torch.equal(g2[1], up)


def test_toggling_the_flag_on_a_live_module():
    mixed, _ = _model(3, mixed=True)
    fp32, _ = _model(3, mixed=False)
    im1, im2 = synth.raft_inputs(seed=4, H=128, W=160)
    a, b = im1.cuda(), im2.cuda()
    with torch.no_grad():
        ref16 = mixed(a, b, iters=4, test_mode=True)[0]
        ref32 = fp32(a, b, iters=4, test_mode=True)[0]
        m = fp32  # one module, flag flipped between calls (the reference reads it on every forward)
        for graph in (False, True):
            m.enable_cuda_graph(graph)
            for flag, want in ((True, ref16), (False, ref32), (True, ref16)):
                m.args.mixed_precision = flag
                got = m(a, b, iters=4, test_mode=True)[0]
                assert torch.equal(got, want), (graph, flag)
        m.enable_cuda_graph(False)
        m.args.mixed_precision = False
    assert not torch.equal(ref16, ref32)


def test_video_inpainting_with_mixed_raft():
    from fgt_b200 import pipeline as PL
    from fgt_b200.fgt_model import Model as FGTModel
    from fgt_b200.lafc_model import Model as LAFCModel
    dev = torch.device("cuda:0")
    frames, masks = synth.pipeline_clip(seed=5, N=7, H=64, W=96)
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    fgt = FGTModel(cfg)
    fgt.load_state_dict(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=31))
    lafc = LAFCModel(dict(synth.CFG_LAFC))
    lafc.load_state_dict(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=32))
    raft, _ = _model(33, mixed=True)
    be = PL.GpuBackend(raft, lafc.to(dev), fgt.to(dev), device=dev)
    args = PL.make_args(imgH=64, imgW=96, flow_mask_dilates=3, frame_dilates=1)
    out = PL.video_inpainting(frames, masks, be, args)
    assert len(out) == len(frames)
    assert all(np.isfinite(np.asarray(f, dtype=np.float64)).all() for f in out)
