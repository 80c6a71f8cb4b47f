"""FGT's mixed-precision mode (FGT.enable_mixed_precision) on the GPU.

Definition: the reference FGT under torch.autocast("cuda", dtype=torch.float16), i.e. the oracle restatement run on
CUDA tensors inside autocast. Per kernel, each fp16 mode is checked against a torch restatement on the same fp16
inputs (or, for the CUDA-core producers, against the kernel's own split-bf16 mode rounded to fp16). End to end, the
mixed path must be no farther from autocast than 1.5x the reference's own mixed-precision error E_ref (autocast vs
the fp32 oracle)."""
import argparse
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fgt_b200 import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _f16_close(got, want, what, tol=1e-3):
    """got / want: fp16-valued tensors computed from the same fp32 values: within one fp16 rounding."""
    got, want = got.float(), want.float()
    err = (got - want).abs()
    bound = tol * want.abs() + 1e-4
    assert (err <= bound).all(), f"{what}: max err {err.max().item():.3e}"


# ------------------------------------------------------------------------------------------------ attention
def _attn_ref(q, k, v, scale):
    """softmax(q k^T scale) v per head in fp32 from fp16 operands; q [Lq, H*128], k / v [Lk, H*128]."""
    H = q.shape[-1] // 128
    qh = q.float().view(-1, H, 128).transpose(0, 1)
    kh = k.float().view(-1, H, 128).transpose(0, 1)
    vh = v.float().view(-1, H, 128).transpose(0, 1)
    p = torch.softmax(qh @ kh.transpose(1, 2) * scale, -1)
    return (p @ vh).transpose(0, 1).reshape(q.shape[0], -1)


@pytest.mark.parametrize("batches,L", [(3, 300), (1, 21000)])
def test_attention_dense_f16(batches, L):
    """Dense mode (temporal zones), including a 21 k-key zone (720p T=16 zones are of that size)."""
    from fgt_b200 import lib
    g = torch.Generator().manual_seed(L)
    H, d = 4, 512
    scale = 1.0 / math.sqrt(128)
    qkv = (torch.randn(batches, L, 3 * d, generator=g) * 1.5).half().to(DEV)
    out = torch.full((batches, L, d), float("nan"), dtype=torch.float16, device=DEV)
    lib.attention(qkv, qkv, qkv, out, batches=batches, heads=H, Lq=L, Lk=L, q_ld=3 * d, k_ld=3 * d, v_ld=3 * d,
                  out_ld=d, q_batch_stride=L * 3 * d, k_batch_stride=L * 3 * d, v_batch_stride=L * 3 * d,
                  out_batch_stride=L * d, scale=scale, k_off=d, v_off=2 * d)
    torch.cuda.synchronize()
    rows = torch.arange(L) if L <= 1024 else torch.cat([torch.arange(256), torch.arange(L - 256, L)])
    for b in range(batches):
        x = qkv[b]
        ref = _attn_ref(x[rows.to(DEV), :d], x[:, d:2 * d], x[:, 2 * d:], scale)
        got = out[b, rows.to(DEV)]
        assert torch.isfinite(got).all()
        assert _rel(got, ref) < 2e-3, (b, _rel(got, ref))


def test_attention_windowed_f16_720p_geometry():
    """Windowed mode (8x8 windows + pooled global tokens) at the padded 720p token grid: 60x107 tokens -> 64x112,
    112 windows, 448 pooled tokens (7 global key tiles); the output goes through the window row map."""
    from fgt_b200 import lib
    g = torch.Generator().manual_seed(7)
    H, d, bt = 4, 512, 2
    h, w, ws = 60, 107, 8
    nwin = (64 // ws) * (112 // ws)
    nl, G = nwin * 64, (64 // 4) * (112 // 4)
    R = nl + (G + 63) // 64 * 64
    scale = 1.0 / math.sqrt(128)
    qkv = (torch.randn(bt, R, 3 * d, generator=g)).half().to(DEV)
    # window row map as FGT builds it: window-major rows -> token index (-1 for the grid's padding)
    f, wy, wx, py, px = torch.meshgrid(torch.arange(bt), torch.arange(64 // ws), torch.arange(112 // ws),
                                       torch.arange(ws), torch.arange(ws), indexing="ij")
    Y, X = wy * ws + py, wx * ws + px
    tok = torch.where((Y < h) & (X < w), (f * h + Y) * w + X, torch.full_like(Y, -1)).reshape(-1)
    rowmap = tok.to(torch.int32).to(DEV)
    out = torch.zeros(bt * h * w, d, dtype=torch.float16, device=DEV)
    lib.attention(qkv, qkv, qkv, out, batches=bt, heads=H, Lq=nl, Lk=R, Lk_rows=R, q_ld=3 * d, k_ld=3 * d,
                  v_ld=3 * d, out_ld=d, q_batch_stride=R * 3 * d, k_batch_stride=R * 3 * d,
                  v_batch_stride=R * 3 * d, out_batch_stride=nl * d, scale=scale, mode=1, glob_start=nl,
                  glob_count=G, k_off=d, v_off=2 * d, out_rowmap=rowmap)
    torch.cuda.synchronize()
    for b in range(bt):
        x = qkv[b].float()
        q = x[:nl, :d].view(nwin, 64, H, 128)
        k = torch.cat([x[:nl, d:2 * d].view(nwin, 64, d), x[nl:nl + G, d:2 * d].expand(nwin, G, d)], 1)
        v = torch.cat([x[:nl, 2 * d:].view(nwin, 64, d), x[nl:nl + G, 2 * d:].expand(nwin, G, d)], 1)
        k, v = k.view(nwin, -1, H, 128), v.view(nwin, -1, H, 128)
        s = torch.einsum("wqhc,wkhc->whqk", q, k) * scale
        ref = torch.einsum("whqk,wkhc->wqhc", torch.softmax(s, -1), v).reshape(nl, d)
        m = tok[b * nl:(b + 1) * nl]
        keep = m >= 0
        got = out[m[keep].to(DEV)]
        assert _rel(got, ref[keep.to(DEV)]) < 2e-3


def test_attention_rejects_mixed_formats():
    from fgt_b200 import lib
    q = torch.zeros(128, 512, dtype=torch.float16, device=DEV)
    s = lib.empty_split((128, 512), DEV)
    with pytest.raises(RuntimeError, match="plane offsets must be 0"):
        lib.attention(q, s, s, q, batches=1, heads=4, Lq=128, Lk=128, q_ld=512, k_ld=512, v_ld=512, out_ld=512,
                      q_batch_stride=0, k_batch_stride=0, v_batch_stride=0, out_batch_stride=0, scale=0.1)


# ------------------------------------------------------------------------------------------------ CUDA-core producers
def test_rownorm_f16():
    from fgt_b200 import lib
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(333, 512, generator=g) * 3 + 1).to(DEV)
    gam, bet = torch.randn(512, generator=g).to(DEV), torch.randn(512, generator=g).to(DEV)
    gather = torch.arange(-1, 332, dtype=torch.int32, device=DEV)  # first row: a zero row
    out = torch.full((333, 512), float("nan"), dtype=torch.float16, device=DEV)
    lib.rownorm(x, None, out, gather=gather, rows_per_batch=333, total_rows=333, dst_batch_rows=333, eps=1e-5,
                gamma=gam, beta=bet)
    ref = F.layer_norm(x[:332], (512,), gam, bet, 1e-5).half()
    assert torch.equal(out[0], torch.zeros_like(out[0]))
    _f16_close(out[1:], ref, "rownorm")


def _both(fn, shape):
    """Runs fn(out16) into a split-bf16 and a single-plane fp16 buffer; returns (fp16 result, split result)."""
    from fgt_b200 import lib
    s = torch.zeros((2,) + shape, dtype=torch.bfloat16, device=DEV)
    h = torch.full(shape, float("nan"), dtype=torch.float16, device=DEV)
    fn(s)
    fn(h)
    torch.cuda.synchronize()
    return h, lib.from_split(s)


def test_fold_unfold_fold_dwconv_f16():
    from fgt_b200 import lib
    g = torch.Generator().manual_seed(2)
    bt, th, tw, C, k, st, p = 2, 12, 20, 40, 7, 3, 3
    OH, OW = (th - 1) * st + k - 2 * p, (tw - 1) * st + k - 2 * p
    hid = torch.randn(bt * th * tw, k * k * C, generator=g).to(DEV)
    h, s = _both(lambda o: lib.fold_unfold(hid, bt, th, tw, C, k, k, st, p, OH, OW, o, relu=True),
                 (bt * th * tw, k * k * C))
    _f16_close(h, s, "fold_unfold")
    C2 = 128
    hid2 = torch.randn(bt * th * tw, k * k * C2, generator=g).to(DEV)
    add = torch.randn(bt, OH, OW, C2, generator=g).to(DEV)
    h, s = _both(lambda o: lib.fold(hid2, bt, th, tw, C2, k, k, st, p, OH, OW, normalize=False, add=add, out_split=o),
                 (bt, OH, OW, C2))
    _f16_close(h, s, "fold+skip")
    x = torch.randn(bt * th * tw, 512, generator=g).to(DEV)
    wt, b = torch.randn(512 * 9, generator=g).to(DEV) * 0.1, torch.randn(512, generator=g).to(DEV)
    out32 = torch.empty_like(x)
    h, s = _both(lambda o: lib.dwconv3x3_res(x, bt, th, tw, 512, wt, b, out32, o), (bt * th * tw, 512))
    _f16_close(h, s, "dwconv3x3_res")
    ref = x.view(bt, th, tw, 512).permute(0, 3, 1, 2)
    ref = (F.conv2d(ref, wt.view(512, 1, 3, 3), b, padding=1, groups=512) + ref).permute(0, 2, 3, 1).reshape(-1, 512)
    _f16_close(h, ref.half(), "dwconv3x3_res vs torch", tol=2e-3)


def test_swin_prep_f16():
    from fgt_b200 import lib
    g = torch.Generator().manual_seed(3)
    bt, h, w, d, df, gd = 2, 10, 14, 512, 256, 4
    sH, sW = 16, 16
    nwin = (sH // 8) * (sW // 8)
    nl, gh, gw = nwin * 64, sH // gd, sW // gd
    R = nl + (gh * gw + 63) // 64 * 64
    x = torch.randn(bt * h * w, d, generator=g).to(DEV)
    fp = torch.randn(bt * h * w, df, generator=g).to(DEV)
    gk_w, gk_b = torch.randn(gd * gd, d + df, generator=g).to(DEV) * 0.2, torch.randn(d + df, generator=g).to(DEV)
    gv_w, gv_b = torch.randn(gd * gd, d, generator=g).to(DEV) * 0.2, torch.randn(d, generator=g).to(DEV)
    f, wy, wx, py, px = torch.meshgrid(torch.arange(bt), torch.arange(sH // 8), torch.arange(sW // 8),
                                       torch.arange(8), torch.arange(8), indexing="ij")
    Y, X = wy * 8 + py, wx * 8 + px
    win_map = torch.where((Y < h) & (X < w), (f * h + Y) * w + X, torch.full_like(Y, -1)).reshape(-1)
    win_map = win_map.to(torch.int32).to(DEV)
    outs = {}
    for mode in ("split", "f16"):
        if mode == "split":
            qkn, vn = lib.empty_split((bt * R, d + df), DEV).zero_(), lib.empty_split((bt * R, d), DEV).zero_()
        else:
            qkn = torch.zeros(bt * R, d + df, dtype=torch.float16, device=DEV)
            vn = torch.zeros(bt * R, d, dtype=torch.float16, device=DEV)
        lib.swin_prep(x, fp, bt, h, w, win_map, nl, R, gd, gh, gw, gk_w, gk_b, gv_w, gv_b, qkn, vn)
        outs[mode] = (qkn, vn)
    torch.cuda.synchronize()
    _f16_close(outs["f16"][0], lib.from_split(outs["split"][0]), "swin_prep qkn")
    _f16_close(outs["f16"][1], lib.from_split(outs["split"][1]), "swin_prep vn")


def test_conv_tail_f16():
    from fgt_b200 import lib
    g = torch.Generator().manual_seed(4)
    n, H, W, cin = 2, 37, 53, 64
    x = torch.randn(n, H, W, cin, generator=g).half().to(DEV)
    wt = (torch.randn(3, cin, 3, 3, generator=g) * 0.05).half().float()
    b = torch.randn(3, generator=g).half().float().to(DEV)
    from fgt_b200.packing import pack_weight
    wp = pack_weight(lib.pack_taps_as_n(wt), half=True).to(DEV)
    out = torch.empty(n, 3, H, W, device=DEV)
    lib.conv_tail(x, n, H, W, cin, wp, 3, b, lib.ACT_TANH, out, nchw=True)
    ref = torch.tanh(F.conv2d(x.float().permute(0, 3, 1, 2), wt.to(DEV), b, padding=1))
    assert _rel(out, ref) < 1e-4
    with pytest.raises(RuntimeError, match="both split-bf16"):
        lib.conv_tail(x, n, H, W, cin, pack_weight(lib.pack_taps_as_n(wt)).to(DEV), 3, b, lib.ACT_TANH, out, nchw=True)


# ------------------------------------------------------------------------------------------------ end to end
def _model(cfg, sd):
    from fgt_b200.fgt_model import Model
    m = Model(cfg)
    m.load_state_dict(sd)
    return m.to(DEV)


def _u8(x):
    return ((x.float().clamp(-1, 1) + 1) / 2 * 255).round().to(torch.int16).cpu()


CASES = [  # (name, config resolution, input H, W, b, t, regime, seed)
    ("64x96_scaled", (64, 96), 64, 96, 1, 3, "scaled", 1),
    ("64x96_default", (64, 96), 64, 96, 1, 3, "default", 2),
    ("432x240_t10", (240, 432), 240, 432, 1, 10, "scaled", 3),
    ("256x432_runtime_geo", (240, 432), 256, 432, 1, 6, "scaled", 4),
    ("b2_odd_t", (64, 96), 64, 96, 2, 3, "scaled", 5),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_mixed_end_to_end_vs_autocast(case):
    from oracle import fgt_oracle as O
    name, res, H, W, b, t, regime, seed = case
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = res
    sd = synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=seed, regime=regime)
    model = _model(cfg, sd)
    fr, fl, mk = (z.to(DEV) for z in synth.fgt_inputs(seed=seed + 10, t=t, H=H, W=W, b=b))
    sdc = {k: v.to(DEV) for k, v in O.strip_net(sd).items()}
    with torch.no_grad():
        out32 = model(fr, fl, mk)
        model.net.enable_mixed_precision(True)
        out16 = model(fr, fl, mk)
        ref32 = O.fgt_forward(sdc, fr, fl, mk)
        with torch.autocast("cuda", dtype=torch.float16):
            refac = O.fgt_forward(sdc, fr, fl, mk).float()
    assert torch.isfinite(out16).all()
    e_ref = _rel(refac, ref32)
    e_mixed = _rel(out16, refac)
    levels = (_u8(out16) - _u8(out32)).abs()
    hist = {int(v): int(c) for v, c in zip(*np.unique(levels.numpy(), return_counts=True))}
    print(f"\n{name}: E_ref={e_ref:.3e} mixed-vs-autocast={e_mixed:.3e} ratio={e_mixed / e_ref:.3f} "
          f"mixed-vs-fp32={_rel(out16, out32):.3e} uint8 |diff| histogram vs fp32 path {hist}")
    assert e_ref > 0
    assert e_mixed <= 1.5 * e_ref, (e_mixed, e_ref)
    # some weight draws overflow fp16 somewhere in the reference under autocast (E_ref ~0.6 at 432x240 seed 3, the
    # tanh output saturates); the mixed path keeps fp32 scores and residuals, so it must also stay near the fp32 path
    assert _rel(out16, out32) < 5e-3


# ------------------------------------------------------------------------------------------------ behaviour
def test_mixed_graph_replay_and_switching():
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    model = _model(cfg, synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=21))
    fr, fl, mk = (z.to(DEV) for z in synth.fgt_inputs(seed=22, t=3, H=64, W=96))
    net = model.net
    with torch.no_grad():
        ref32 = model(fr, fl, mk)
        net.enable_mixed_precision(True)
        ref16 = model(fr, fl, mk)
        net.enable_mixed_precision(False)
        assert torch.equal(model(fr, fl, mk), ref32)  # fp32 -> mixed -> fp32 on one model: the fp32 bits
        assert not torch.equal(ref16, ref32)
        net.enable_cuda_graph(True)
        for flag, want in ((True, ref16), (False, ref32), (True, ref16), (True, ref16), (False, ref32),
                           (False, ref32)):
            net.enable_mixed_precision(flag)
            assert torch.equal(model(fr, fl, mk), want), flag  # eager, capture, then replays
        net.enable_cuda_graph(False)
        net.enable_mixed_precision(False)


def test_pipeline_with_fgt_mixed_precision():
    from fgt_b200 import pipeline as PL
    from fgt_b200.fgt_model import Model as FGTModel
    from fgt_b200.lafc_model import Model as LAFCModel
    from fgt_b200.raft_model import RAFT
    frames, masks = synth.pipeline_clip(seed=5, N=7, H=64, W=96)
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    fgt = FGTModel(cfg)
    fgt.load_state_dict(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=31))
    fgt.net.enable_mixed_precision(True)
    lafc = LAFCModel(dict(synth.CFG_LAFC))
    lafc.load_state_dict(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=32))
    raft = RAFT(argparse.Namespace(small=False, mixed_precision=False, alternate_corr=False))
    raft.load_state_dict(synth.raft_state_dict(seed=33))
    be = PL.GpuBackend(raft.to(DEV).eval(), lafc.to(DEV), fgt.to(DEV), device=torch.device(DEV))
    args = PL.make_args(imgH=64, imgW=96, flow_mask_dilates=3, frame_dilates=1)
    out = PL.video_inpainting(frames, masks, be, args)
    assert len(out) == len(frames)
    assert all(np.isfinite(np.asarray(f, dtype=np.float64)).all() for f in out)
    assert fgt.net._mixed and True in fgt.net._packed
