"""GPU parity of the individual sm_90a kernels, called through the C-ABI (fgt_b200.lib), against
fp64 PyTorch restatements of the same op on the same seeded inputs."""

import pytest
import torch
import torch.nn.functional as F

from tests.util import assert_close

pytestmark = pytest.mark.gpu

KTOL = 1e-4  # split-bf16 3-term products: ~1e-5 observed, fp32-grade


def _lib():
    from fgt_b200 import lib
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    lib.load()
    return lib


@pytest.mark.parametrize("M,N,K,bn,act,aux,split", [
    (128, 128, 64, 128, 0, 0, False), (256, 256, 512, 128, 1, 0, True), (1000, 520, 1960, 128, 2, 0, True),
    (7200, 1536, 512, 256, 0, 1, False), (300, 48, 200, 48, 3, 2, False), (40000, 512, 512, 128, 4, 0, False),
])
def test_linear(M, N, K, bn, act, aux, split):
    from tools import diag_gemm as D
    assert D.linear_case(M, N, K, bn=bn, act=act, aux_mode=aux, split_out=split)


@pytest.mark.parametrize("kw", [
    dict(n=1, h=16, w=32, cin=64, cout=64, k=3), dict(n=2, h=60, w=108, cin=128, cout=256, k=3, bn=128),
    dict(n=2, h=61, w=107, cin=64, cout=128, k=3, stride=2, bn=128),
    dict(n=1, h=60, w=108, cin=128, cout=512, k=7, stride=3, pad=3, bn=128, act=0),
    dict(n=1, h=30, w=54, cin=192, cout=192, k=3, dil=4, bn=64),
    dict(n=2, h=24, w=40, cin=128, cout=256, k=3, groups=2, bn=128),
    dict(n=1, h=24, w=40, cin=8, cout=64, k=3, bn=64), dict(n=1, h=20, w=36, cin=64, cout=3, k=3, bn=16, act=0),
])
def test_conv(kw):
    from tools import diag_gemm as D
    assert D.conv_case(**kw)


@pytest.mark.parametrize("kw", [
    dict(M=7200, N=1960, K=512, bn=128),                                              # fp32 only, N tail (partial tile)
    dict(M=1000, N=520, K=1960, bn=128, act=2, split_only=True, aux_mode=1),          # split only, M and N tails, residual
    dict(M=7200, N=1536, K=512, bn=128, split_only=True),
    dict(M=333, N=256, K=320, bn=256, split_only=True, act=3, aux_mode=2),
    dict(M=7200, N=256, K=768, bn=128, terms=1, split_only=True),                     # fp16 operands, fp16 output
    dict(M=1000, N=192, K=576, bn=64, terms=1, act=1),                                # fp16 operands, fp32 output
    dict(M=2000, N=256, K=6272, bn=128, terms=1, split_out=True),                     # f_patch2vec: fp32 + split outputs
    dict(M=70000, N=64, K=64, bn=64, split_only=True, act=1),                         # one K iteration per tile
])
def test_linear_tails_and_one_term(kw):
    """Linear launches with M / N tails, one or two outputs, aux operands, a 256-wide tile and one K iteration per tile;
    terms=1 uses single-plane fp16 operands (the flow branch)."""
    from tools import diag_gemm as D
    assert D.linear_case(**kw)


@pytest.mark.parametrize("kw", [
    dict(n=2, h=61, w=107, cin=64, cout=128, k=3, stride=2, bn=128, split_only=True),  # partial output boxes at the right / bottom edges
    dict(n=2, h=60, w=108, cin=128, cout=128, k=3, bn=128, terms=1, split_only=True),
    dict(n=1, h=30, w=54, cin=192, cout=192, k=3, dil=4, bn=64, split_only=True),
])
def test_conv_edge_tiles_and_one_term(kw):
    from tools import diag_gemm as D
    assert D.conv_case(**kw)


def test_paired_epilogue_bit_equal_to_per_element_epilogue():
    """The paired-access epilogue (8-byte fp32 / 4-byte 16-bit stores and aux loads) and the per-element one run the same
    arithmetic: identical bits."""
    import ctypes
    lib = _lib()
    from fgt_b200 import packing
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    M, N, K = 1500, 712, 320
    a_s = lib.to_split(torch.randn(M, K, device=dev))
    w_s = packing.pack_weight(torch.randn(N, K, device=dev) / K ** 0.5).to(dev)
    b = torch.randn(N, device=dev)
    aux = torch.randn(M, N, device=dev)
    L = lib.load()
    L.fgt_debug_gemm_direct_epilogue.argtypes = [ctypes.c_int]
    outs = []
    for direct in (0, 1, 2):   # 0: paired stores + paired aux loads, 1: per-element stores and loads, 2: paired stores + per-element aux loads
        L.fgt_debug_gemm_direct_epilogue(direct)
        try:
            o32 = torch.zeros(M, N, device=dev)
            osp = torch.zeros(2, M, N, dtype=torch.bfloat16, device=dev)
            lib.gemm_tc([lib.ASeg(a_s, K, M)], w_s, N, out_w=M, bn=128, bias=b, act=lib.ACT_LEAKY02, out_f32=o32, aux=aux,
                        aux_mode=lib.AUX_ADD)
            lib.gemm_tc([lib.ASeg(a_s, K, M)], w_s, N, out_w=M, bn=128, bias=b, act=lib.ACT_LEAKY02, out_split=osp,
                        aux=aux, aux_mode=lib.AUX_ADD)
            torch.cuda.synchronize()
        finally:
            L.fgt_debug_gemm_direct_epilogue(0)
        outs.append((o32, osp))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert torch.equal(outs[0][0], outs[2][0]) and torch.equal(outs[0][1], outs[2][1])
    # in-place residual (aux == out), the out-projection / FFN pattern
    x0 = torch.randn(M, N, device=dev)
    res = []
    for direct in (0, 1):
        L.fgt_debug_gemm_direct_epilogue(direct)
        try:
            x = x0.clone()
            lib.gemm_tc([lib.ASeg(a_s, K, M)], w_s, N, out_w=M, bn=128, bias=b, out_f32=x, aux=x, aux_mode=lib.AUX_ADD)
            torch.cuda.synchronize()
        finally:
            L.fgt_debug_gemm_direct_epilogue(0)
        res.append(x)
    assert torch.equal(res[0], res[1])


def test_linear_rowmap_and_transposed_store():
    lib = _lib()
    from fgt_b200 import packing
    dev = torch.device("cuda:0")
    torch.manual_seed(1)
    M, N, K, Lb = 600, 256, 192, 150
    a = torch.randn(M, K, device=dev)
    w = torch.randn(N, K, device=dev) / K ** 0.5
    b = torch.randn(N, device=dev)
    ref = a.double() @ w.double().t() + b.double()
    a_s, w_s = lib.to_split(a), packing.pack_weight(w).to(dev)
    # row map: reverse order, drop every 7th row; residual add from the destination
    rowmap = torch.arange(M - 1, -1, -1, dtype=torch.int32, device=dev)
    rowmap[::7] = -1
    base = torch.randn(M, N, device=dev)
    out = base.clone()
    lib.gemm_tc([lib.ASeg(a_s, K, M)], w_s, N, out_w=M, bn=128, bias=b, out_f32=out, aux=out, aux_mode=lib.AUX_ADD,
                rowmap=rowmap)
    torch.cuda.synchronize()
    exp = base.double().clone()
    keep = rowmap >= 0
    exp[rowmap[keep].long()] += ref[keep]
    assert_close(out, exp, KTOL, "rowmap scatter + residual")
    # transposed, batched store: V^T[z, n, x] with pitch Lp
    Lp = 152
    vt = torch.zeros(2, M // Lb, N, Lp, dtype=torch.bfloat16, device=dev)
    lib.gemm_tc([lib.ASeg(a_s, K, M)], w_s, N, out_w=M, bn=128, bias=b, out_split=vt, lin_batch=Lb, os_z=N * Lp,
                os_x=1, os_c=Lp)
    torch.cuda.synchronize()
    got = lib.from_split(vt)[:, :, :Lb].permute(0, 2, 1).reshape(M, N)
    assert_close(got, ref, KTOL, "transposed store")


@pytest.mark.parametrize("batches,heads,L,qs", [(1, 1, 64, 1.0), (1, 2, 200, 1.0), (2, 4, 1800, 3.0), (4, 4, 37, 1.0),
                                                (1, 1, 21060, 2.0)])  # last: one 720p zone at T=13 (BASELINE config 5)
def test_attention_dense(batches, heads, L, qs):
    from tools import diag_attn as D
    assert D.dense_case(batches, heads, L, qscale=qs)


@pytest.mark.parametrize("frames,heads,nwin,nglob,qs", [(1, 1, 2, 60, 1.0), (3, 4, 15, 60, 3.0), (1, 4, 112, 448, 1.0)])
def test_attention_windowed(frames, heads, nwin, nglob, qs):
    from tools import diag_attn as D
    assert D.window_case(frames, heads, nwin, nglob, qscale=qs)


def _zone_rowmap(t, h, w, gs=2):
    """FGT's temporal-zone row map (fgt_model._geometry): zone-major rows (frame, y, x inside the zone) -> token index
    of a [t, h, w] grid, -1 for the rows of the zone padding past the grid."""
    zh, zw = -(-h // gs), -(-w // gs)
    zy, zx, ti, yy, xx = torch.meshgrid(torch.arange(gs), torch.arange(gs), torch.arange(t), torch.arange(zh),
                                        torch.arange(zw), indexing="ij")
    Y, X = zy * zh + yy, zx * zw + xx
    tok = torch.where((Y < h) & (X < w), (ti * h + Y) * w + X, torch.full_like(Y, -1))
    return tok.reshape(-1).to(torch.int32), zh * zw


@pytest.mark.parametrize("f16", (False, True))
@pytest.mark.parametrize("T,sharded", [(3, False), (5, False), (3, True)])
def test_attention_production_layouts(T, sharded, f16):
    """TMHSA as the FGT forward calls it: 4 zones of Lz = 11*18*T keys (odd T, not a multiple of the 64-key tile, so the
    last key tile of a zone runs into the next zone's rows), Q|K|V in one fused [rows, 3d] buffer read through k_off /
    v_off, the output scattered through the zone row map (-1 rows dropped). sharded: the frame-sharded call, Q of this
    rank's first frame only (Lq = Lz / T < Lk) from its own buffer, K|V from a [rows, 2d] buffer with v_off = d.
    The first 64 key rows of every zone (and the rows past the last zone) are scaled so that one of them would dominate
    the softmax of any query that wrongly saw it. Output rows no query row maps to keep their sentinel bit for bit.
    Bars: KTOL (split-bf16) or test_fgt_mixed_gpu's 2e-3 relative (fp16) against a float64 softmax of the operands."""
    import math
    lib = _lib()
    dev = torch.device("cuda:0")
    H, d, h, w = 4, 512, 21, 36
    g = torch.Generator().manual_seed(100 * T + sharded)
    zl = -(-h // 2) * -(-w // 2)
    zones, Lk = 4, T * zl
    t = 1 if sharded else T
    Lq = t * zl
    rowmap, _ = _zone_rowmap(t, h, w)
    kv_cols = 2 * d if sharded else 3 * d
    kv = torch.randn(zones * Lk + 64, kv_cols, generator=g)
    koff = 0 if sharded else d
    for z in range(zones + 1):   # dominating keys at the head of every zone's rows and past the last zone
        kv[z * Lk:z * Lk + 64, koff:koff + d] *= 6.0
    q_src = torch.randn(zones * Lq, d, generator=g) if sharded else None
    enc = (lambda x: x.half().contiguous()) if f16 else lib.to_split   # noqa: E731
    kv16 = enc(kv)
    q16 = enc(q_src) if sharded else kv16
    val = (lambda s: s.double()) if f16 else (lambda s: s[0].double() + s[1].double())   # noqa: E731
    kvv, qv = val(kv16), val(q16)
    rows_out = T * h * w + 37   # every token row of the window plus rows no query maps to
    sent = torch.full((rows_out, d), -1234.5, dtype=torch.float16) if f16 else \
        torch.full((2, rows_out, d), -1234.5, dtype=torch.bfloat16)
    out = sent.clone().to(dev)
    rm = rowmap.to(dev)
    scale = 1.0 / math.sqrt(128)
    if sharded:
        lib.attention(q16.to(dev), kv16.to(dev), kv16.to(dev), out, batches=zones, heads=H, Lq=Lq, Lk=Lk, q_ld=d,
                      k_ld=2 * d, v_ld=2 * d, out_ld=d, q_batch_stride=Lq * d, k_batch_stride=Lk * 2 * d,
                      v_batch_stride=Lk * 2 * d, out_batch_stride=Lq * d, scale=scale, v_off=d, out_rowmap=rm)
    else:
        x = kv16.to(dev)
        lib.attention(x, x, x, out, batches=zones, heads=H, Lq=Lq, Lk=Lk, q_ld=3 * d, k_ld=3 * d, v_ld=3 * d, out_ld=d,
                      q_batch_stride=Lk * 3 * d, k_batch_stride=Lk * 3 * d, v_batch_stride=Lk * 3 * d,
                      out_batch_stride=Lq * d, scale=scale, k_off=d, v_off=2 * d, out_rowmap=rm)
    torch.cuda.synchronize()
    out = out.cpu()
    want = torch.zeros(rows_out, d, dtype=torch.float64)
    hit = torch.zeros(rows_out, dtype=torch.bool)
    for z in range(zones):
        qz = qv[z * Lq:(z + 1) * Lq] if sharded else qv[z * Lk:z * Lk + Lq, :d]
        kz = kvv[z * Lk:(z + 1) * Lk, koff:koff + d]
        vz = kvv[z * Lk:(z + 1) * Lk, koff + d:koff + 2 * d]
        qh, kh, vh = (a.reshape(-1, H, 128).transpose(0, 1) for a in (qz, kz, vz))
        o = (torch.softmax(qh @ kh.transpose(1, 2) * scale, -1) @ vh).transpose(0, 1).reshape(Lq, d)
        m = rowmap[z * Lq:(z + 1) * Lq].long()
        keep = m >= 0
        want[m[keep]] = o[keep]
        hit[m[keep]] = True
    assert int(hit.sum()) == t * h * w
    if f16:
        assert torch.equal(out[~hit], sent[~hit]), "rows outside the row map written"
        got = out[hit].double()
        rel = ((got - want[hit]).norm() / want[hit].norm()).item()
        assert torch.isfinite(got).all() and rel < 2e-3, rel
    else:
        assert torch.equal(out[:, ~hit], sent[:, ~hit]), "rows outside the row map written"
        assert_close(out[0, hit].double() + out[1, hit].double(), want[hit], KTOL, "zone attention")


def test_rownorm_gather_affine():
    lib = _lib()
    dev = torch.device("cuda:0")
    torch.manual_seed(2)
    a = torch.randn(100, 512, device=dev) * 3 + 1
    b = torch.randn(100, 256, device=dev)
    gather = torch.randint(-1, 100, (2 * 70,), dtype=torch.int32, device=dev)
    out = torch.full((2, 2 * 80, 768), 7.0, dtype=torch.bfloat16, device=dev)
    gam, bet = torch.randn(768, device=dev), torch.randn(768, device=dev)
    lib.rownorm(a, b, out, gather=gather, rows_per_batch=70, total_rows=140, dst_batch_rows=80, dst_row0=5,
                gamma=gam, beta=bet)
    torch.cuda.synchronize()
    got = lib.from_split(out).reshape(2, 80, 768)[:, 5:75].reshape(140, 768)
    src = torch.cat([a, b], 1).double()
    ref = F.layer_norm(src[gather.clamp(min=0).long()], (768,), gam.double(), bet.double())
    ref[gather < 0] = 0
    assert_close(got, ref, KTOL, "rownorm")
    untouched = lib.from_split(out).reshape(2, 80, 768)[:, :5]
    assert (untouched == 14.0).all()


def test_fold_unfold_dwconv_dwpool_upsample_pack():
    lib = _lib()
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    bt, th, tw, C, OH, OW = 2, 6, 9, 40, 18, 25  # tokens of a 72x100 input
    hid = torch.randn(bt * th * tw, 49 * C, device=dev)
    # torch fold layout is channel-major (c*49+p); the kernels use position-major (p*C+c)
    cm = hid.reshape(bt, th * tw, 49, C).permute(0, 3, 2, 1).reshape(bt, C * 49, th * tw).double()
    img_ref = F.fold(cm, (OH, OW), (7, 7), stride=3, padding=3)
    cnt = F.fold(torch.ones_like(cm[:, :49]), (OH, OW), (7, 7), stride=3, padding=3)
    img = torch.empty(bt, OH, OW, C, device=dev)
    lib.fold(hid, bt, th, tw, C, 7, 7, 3, 3, OH, OW, normalize=True, out=img)
    torch.cuda.synchronize()
    assert_close(img.permute(0, 3, 1, 2), img_ref / cnt, KTOL, "fold normalised")
    add = torch.randn(bt, OH, OW, C, device=dev)
    sp = lib.empty_split((bt, OH, OW, C), dev)
    lib.fold(hid, bt, th, tw, C, 7, 7, 3, 3, OH, OW, normalize=False, add=add, out_split=sp)
    torch.cuda.synchronize()
    assert_close(lib.from_split(sp).permute(0, 3, 1, 2), img_ref + add.permute(0, 3, 1, 2).double(), KTOL, "fold+add")
    un = lib.empty_split((bt * th * tw, 49 * C), dev)
    lib.unfold(img, bt, th, tw, C, 7, 7, 3, 3, OH, OW, un, relu=True)
    torch.cuda.synchronize()
    ur = F.relu(F.unfold(img.permute(0, 3, 1, 2).double(), (7, 7), stride=3, padding=3))
    ur = ur.reshape(bt, C, 49, th * tw).permute(0, 3, 2, 1).reshape(bt * th * tw, 49 * C)
    assert_close(lib.from_split(un), ur, KTOL, "unfold+relu")
    # depthwise 3x3 + identity
    x = torch.randn(bt, th, tw, 64, device=dev)
    wt, bs = torch.randn(64, 1, 3, 3, device=dev), torch.randn(64, device=dev)
    o = torch.empty_like(x)
    osplit = lib.empty_split(x.shape, dev)
    lib.dwconv3x3_res(x, bt, th, tw, 64, wt.reshape(-1).contiguous(), bs, o, osplit)
    torch.cuda.synchronize()
    xr = x.permute(0, 3, 1, 2).double()
    ref = F.conv2d(xr, wt.double(), bs.double(), padding=1, groups=64) + xr
    assert_close(o.permute(0, 3, 1, 2), ref, KTOL, "dwconv3x3_res")
    assert_close(lib.from_split(osplit).permute(0, 3, 1, 2), ref, KTOL, "dwconv3x3_res split")
    # depthwise pooling over a zero-padded grid of [a ; b]
    a, b2 = torch.randn(bt, th, tw, 32, device=dev), torch.randn(bt, th, tw, 16, device=dev)
    wk, bk = torch.randn(48, 1, 4, 4, device=dev), torch.randn(48, device=dev)
    gh, gw = 2, 4  # padded grid 8 x 16
    po = torch.empty(bt, gh * gw, 48, device=dev)
    lib.dwpool(a, b2, bt, th, tw, 4, gh, gw, wk.reshape(-1).contiguous(), bk, po)
    torch.cuda.synchronize()
    cat = F.pad(torch.cat([a, b2], -1), (0, 0, 0, 16 - tw, 0, 8 - th)).permute(0, 3, 1, 2).double()
    pr = F.conv2d(cat, wk.double(), bk.double(), stride=4, groups=48).permute(0, 2, 3, 1).reshape(bt, gh * gw, 48)
    assert_close(po, pr, KTOL, "dwpool")
    # nearest x2
    s_in = lib.to_split(torch.randn(bt, 5, 7, 16, device=dev))
    s_out = lib.empty_split((bt, 10, 14, 16), dev)
    lib.upsample2x(s_in, bt, 5, 7, 16, s_out)
    torch.cuda.synchronize()
    ref = F.interpolate(lib.from_split(s_in).permute(0, 3, 1, 2), scale_factor=2).permute(0, 2, 3, 1)
    assert torch.equal(lib.from_split(s_out), ref)
    # NCHW pack with replication padding
    f0, f1 = torch.randn(bt, 3, 10, 12, device=dev), torch.randn(bt, 1, 10, 12, device=dev)
    pk = lib.empty_split((bt, 14, 16, 8), dev)
    lib.pack_nchw(f0, f1, pk, pad=2)
    torch.cuda.synchronize()
    ref = F.pad(torch.cat([f0, f1], 1), (2, 2, 2, 2), mode="replicate").permute(0, 2, 3, 1)
    got = lib.from_split(pk)
    assert_close(got[..., :4], ref, 1e-4, "pack_nchw")
    assert (got[..., 4:] == 0).all()


@pytest.mark.parametrize("bt,h,w", [(2, 20, 36), (1, 22, 36), (1, 7, 13)])
def test_swin_prep_vs_torch(bt, h, w):
    """fgt_swin_prep = zero-pad + window partition + depthwise pooling + the two LayerNorm statistics of SWMHSA's
    operand preparation (attention_flow.py:122-154), against an fp64 PyTorch restatement."""
    lib = _lib()
    dev = torch.device("cuda:0")
    torch.manual_seed(4)
    d, df, ws, gd = 512, 256, 8, 4
    x = torch.randn(bt * h * w, d, device=dev) * 2 + 0.3
    fp = torch.randn(bt * h * w, df, device=dev)
    Hn, Wn = h + (ws - h % ws) % ws, w + (ws - w % ws) % ws
    nwin = (Hn // ws) * (Wn // ws)
    nwp = (nwin + 1) // 2 * 2
    gh, gw = Hn // gd, Wn // gd
    G = gh * gw
    R = nwp * 64 + (G + 63) // 64 * 64
    nl = nwp * 64
    f, wy, wx, py, px = torch.meshgrid(torch.arange(bt), torch.arange(Hn // ws), torch.arange(Wn // ws), torch.arange(ws),
                                       torch.arange(ws), indexing="ij")
    Y, X = wy * ws + py, wx * ws + px
    tok = torch.where((Y < h) & (X < w), (f * h + Y) * w + X, torch.full_like(Y, -1)).reshape(bt, nwin * 64)
    full = torch.full((bt, nl), -1, dtype=tok.dtype)
    full[:, :nwin * 64] = tok
    win_map = full.reshape(-1).to(torch.int32).to(dev)
    gk_w, gk_b = torch.randn(d + df, 1, gd, gd, device=dev) * 0.3, torch.randn(d + df, device=dev)
    gv_w, gv_b = torch.randn(d, 1, gd, gd, device=dev) * 0.3, torch.randn(d, device=dev)
    qkn = torch.full((2, bt * R, d + df), 7.0, dtype=torch.bfloat16, device=dev)
    vn = torch.full((2, bt * R, d), 7.0, dtype=torch.bfloat16, device=dev)
    lib.swin_prep(x, fp, bt, h, w, win_map, nl, R, gd, gh, gw, gk_w.reshape(d + df, -1).t().contiguous(), gk_b,
                  gv_w.reshape(d, -1).t().contiguous(), gv_b, qkn, vn)
    torch.cuda.synchronize()
    # reference
    xg = F.pad(x.double().reshape(bt, h, w, d), (0, 0, 0, Wn - w, 0, Hn - h))
    qg = F.pad(torch.cat([x, fp], 1).double().reshape(bt, h, w, d + df), (0, 0, 0, Wn - w, 0, Hn - h))

    def windows(g):
        c = g.shape[-1]
        return g.reshape(bt, Hn // ws, ws, Wn // ws, ws, c).permute(0, 1, 3, 2, 4, 5).reshape(bt, nwin * 64, c)

    kg = F.conv2d(qg.permute(0, 3, 1, 2), gk_w.double(), gk_b.double(), stride=gd, groups=d + df).permute(0, 2, 3, 1)
    vg = F.conv2d(xg.permute(0, 3, 1, 2), gv_w.double(), gv_b.double(), stride=gd, groups=d).permute(0, 2, 3, 1)
    got_q = lib.from_split(qkn).reshape(bt, R, d + df)
    got_v = lib.from_split(vn).reshape(bt, R, d)
    valid = (tok >= 0).to(dev)
    ref_q = F.layer_norm(windows(qg), (d + df,)) * valid[..., None]   # rows of the zero padding are written as zeros
    ref_v = F.layer_norm(windows(xg), (d,)) * valid[..., None]
    assert_close(got_q[:, :nwin * 64], ref_q, KTOL, "swin_prep window rows (q|k)")
    assert_close(got_v[:, :nwin * 64], ref_v, KTOL, "swin_prep window rows (v)")
    assert_close(got_q[:, nl:nl + G], F.layer_norm(kg.reshape(bt, G, d + df), (d + df,)), KTOL, "swin_prep pooled rows (k)")
    assert_close(got_v[:, nl:nl + G], F.layer_norm(vg.reshape(bt, G, d), (d,)), KTOL, "swin_prep pooled rows (v)")
    assert (got_q[:, nwin * 64:nl] == 0).all() and (got_q[:, nl + G:] == 14.0).all()   # dummy window zeroed, pad rows untouched


@pytest.mark.parametrize("n,H,W,cin,cout,act", [(2, 24, 40, 64, 3, 4), (1, 21, 37, 128, 2, 0), (3, 240, 432, 64, 3, 4),
                                                  (2, 37, 53, 64, 3, 4), (3, 16, 20, 256, 2, 0), (1, 8, 40, 128, 3, 2)])
def test_conv_tail_vs_torch(n, H, W, cin, cout, act):
    """fgt_conv_tail (taps-as-N GEMM + in-SM tap sum + bias + activation) against F.conv2d in fp64, edge tiles included:
    FGT's decoder tail (64 -> 3, tanh), RAFT's flow head tail (256 -> 2, no activation) and a ReLU case."""
    lib = _lib()
    from fgt_b200 import packing
    dev = torch.device("cuda:0")
    torch.manual_seed(5)
    x = torch.randn(n, cin, H, W, device=dev)
    w = torch.randn(cout, cin, 3, 3, device=dev) / (cin * 9) ** 0.5
    b = torch.randn(cout, device=dev)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    ref = {0: lambda t: t, 2: torch.relu, 4: torch.tanh}[act](ref)
    xs = lib.to_split(x.permute(0, 2, 3, 1).contiguous())
    ws = packing.pack_weight(lib.pack_taps_as_n(w)).to(dev)
    out = torch.full((n, cout, H, W), float("nan"), device=dev)
    lib.conv_tail(xs, n, H, W, cin, ws, cout, b, act, out, nchw=True)
    torch.cuda.synchronize()
    assert_close(out, ref, KTOL, "conv_tail nchw")
    out2 = torch.full((n, H, W, cout), float("nan"), device=dev)
    lib.conv_tail(xs, n, H, W, cin, ws, cout, b, act, out2, nchw=False)
    torch.cuda.synchronize()
    assert_close(out2.permute(0, 3, 1, 2), ref, KTOL, "conv_tail nhwc")


@pytest.mark.parametrize("c0,c1,k,stride,pad,replicate,half", [(3, 1, 3, 2, 1, False, False), (2, 0, 5, 1, 2, True, True),
                                                               (3, 0, 7, 2, 3, False, False)])
def test_im2col_nchw_vs_torch(c0, c1, k, stride, pad, replicate, half):
    """fgt_im2col_nchw (rows of k*k*cin gathered inputs, (ky,kx)-major / channel-minor, zero or replication padding,
    optional affine on in-bounds samples, split-bf16 or fp16 rows) against F.unfold on the padded input."""
    lib = _lib()
    dev = torch.device("cuda:0")
    torch.manual_seed(6)
    n, H, W = 2, 37, 52
    a = torch.randn(n, c0, H, W, device=dev)
    b = torch.randn(n, c1, H, W, device=dev) if c1 else None
    x = torch.cat([a, b], 1) if c1 else a
    cin = c0 + c1
    OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    cpad = (k * k * cin + 63) // 64 * 64
    scale, shift = (2.0 / 255.0, -1.0) if k == 7 else (1.0, 0.0)
    out = (torch.full((n, OH, OW, cpad), 9.0, dtype=torch.float16, device=dev) if half
           else torch.full((2, n, OH, OW, cpad), 9.0, dtype=torch.bfloat16, device=dev))
    lib.im2col_nchw(a, b, out, k=k, stride=stride, pad=pad, replicate=replicate, OH=OH, OW=OW, scale=scale, shift=shift)
    torch.cuda.synchronize()
    xa = x.double() * scale + shift
    xp = F.pad(xa, (pad,) * 4, mode="replicate") if replicate else F.pad(xa, (pad,) * 4)
    cols = F.unfold(xp, k, stride=stride).reshape(n, cin, k * k, OH, OW)           # [n, c, tap, oy, ox]
    ref = cols.permute(0, 3, 4, 2, 1).reshape(n, OH, OW, k * k * cin)              # channel = tap*cin + c
    got = out.float() if half else lib.from_split(out)
    assert_close(got[..., :k * k * cin], ref, 1e-3 if half else KTOL, "im2col rows")
    assert (got[..., k * k * cin:] == 0).all()


@pytest.mark.parametrize("bt,OH,OW,C", [(2, 60, 108, 40), (1, 64, 108, 40), (1, 16, 24, 8), (1, 180, 320, 40)])
def test_fold_unfold_fused_equals_two_launches(bt, OH, OW, C):
    """fgt_fold_unfold == fgt_fold(normalize) -> fgt_unfold(relu), bit for bit (and both == nn.Fold / nn.Unfold, fp64),
    at the model's geometries (token grid = conv output size of the H/4 x W/4 map: the last rows of the padded map lie
    under no patch)."""
    lib = _lib()
    dev = torch.device("cuda:0")
    torch.manual_seed(7)
    k, s, p = 7, 3, 3
    th, tw = (OH + 2 * p - k) // s + 1, (OW + 2 * p - k) // s + 1
    hid = torch.randn(bt * th * tw, k * k * C, device=dev)
    img = torch.empty(bt, OH, OW, C, device=dev)
    two = torch.full((2, bt * th * tw, k * k * C), 3.0, dtype=torch.bfloat16, device=dev)
    one = torch.full_like(two, 5.0)
    lib.fold(hid, bt, th, tw, C, k, k, s, p, OH, OW, normalize=True, out=img)
    lib.unfold(img, bt, th, tw, C, k, k, s, p, OH, OW, two, relu=True)
    lib.fold_unfold(hid, bt, th, tw, C, k, k, s, p, OH, OW, one, relu=True)
    torch.cuda.synchronize()
    assert torch.equal(one, two)
    # fp64 reference through nn.Fold / nn.Unfold (hidden index is position-major here: p*C + c)
    cols = hid.double().reshape(bt, th * tw, k * k, C).permute(0, 3, 2, 1).reshape(bt, C * k * k, th * tw)
    im = F.fold(cols, (OH, OW), k, stride=s, padding=p) / F.fold(torch.ones_like(cols), (OH, OW), k, stride=s, padding=p)
    ref = F.relu(F.unfold(im, k, stride=s, padding=p)).reshape(bt, C, k * k, th * tw).permute(0, 3, 2, 1).reshape(bt * th * tw, -1)
    assert_close(lib.from_split(one), ref, KTOL, "fold_unfold vs nn.Fold/nn.Unfold")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_chain_on_two_devices_in_one_process():
    """The dynamic shared-memory limit the im2col, GEMM, attention and conv-tail kernels raise belongs to each kernel as
    loaded on one device: the chain run on cuda:0 and then on cuda:1 in one process gives the same bits on both."""
    lib = _lib()
    from fgt_b200 import packing
    g = torch.Generator().manual_seed(11)
    n, H, W, C = 1, 16, 24, 128
    M = n * H * W
    x = torch.randn(n, 3, H, W, generator=g)
    w1, b1 = torch.randn(C, 64, generator=g) / 8, torch.randn(C, generator=g)
    w2, b2 = torch.randn(3, C, 3, 3, generator=g) / 32, torch.randn(3, generator=g)
    outs = []
    for d in range(2):
        dev = torch.device("cuda", d)
        with torch.cuda.device(dev):
            cols = torch.empty(2, n, H, W, 64, dtype=torch.bfloat16, device=dev)
            lib.im2col_nchw(x.to(dev), None, cols, k=3, stride=1, pad=1, replicate=False, OH=H, OW=W)
            h = lib.empty_split((M, C), dev)
            lib.gemm_tc([lib.ASeg(cols, 64, M)], packing.pack_weight(w1).to(dev), C, out_w=M, bn=128, bias=b1.to(dev),
                        out_split=h)
            a = lib.empty_split((M, C), dev)
            lib.attention(h, h, h, a, batches=1, heads=1, Lq=M, Lk=M, q_ld=C, k_ld=C, v_ld=C, out_ld=C,
                          q_batch_stride=M * C, k_batch_stride=M * C, v_batch_stride=M * C, out_batch_stride=M * C,
                          scale=C ** -0.5)
            out = torch.full((n, 3, H, W), float("nan"), device=dev)
            lib.conv_tail(a, n, H, W, C, packing.pack_weight(lib.pack_taps_as_n(w2)).to(dev), 3, b2.to(dev),
                          lib.ACT_TANH, out, nchw=True)
            torch.cuda.synchronize(dev)
        outs.append(out.cpu())
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1])
