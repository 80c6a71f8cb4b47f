"""CPU: host-side logic (weight packing, LayerNorm folding, window/zone index maps, state_dict
contract) and the C-ABI surface (library loads, exports every symbol the header declares)."""
import ctypes
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

from fgt_b200 import lib, packing, synth
from fgt_b200.fgt_model import Model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _small_model():
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    return Model(cfg), cfg


def test_library_exports_header_symbols():
    from fgt_b200 import build
    build.build()
    cdll = ctypes.CDLL(lib.LIB_PATH)
    with open(os.path.join(ROOT, "include", "fgt_b200.h")) as fh:
        header = fh.read()
    names = set(re.findall(r"\b(fgt_[a-z0-9_]+)\s*\(", header))
    assert {"fgt_gemm_tc", "fgt_attention", "fgt_rownorm", "fgt_fold", "fgt_unfold"} <= names
    for n in sorted(names):
        assert hasattr(cdll, n), f"{n} declared in include/fgt_b200.h but not exported"
    assert lib.load().fgt_version() >= 100


def test_no_cpu_fallback():
    model, _ = _small_model()
    fr, fl, mk = synth.fgt_inputs(seed=0, t=2, H=64, W=96)
    with pytest.raises(RuntimeError):
        model(fr, fl, mk)


def test_state_dict_contract():
    model, cfg = _small_model()
    shapes = synth.fgt_param_shapes(cfg)
    sd = model.state_dict()
    assert set(sd.keys()) == set(shapes.keys())
    for k, s in shapes.items():
        assert tuple(sd[k].shape) == tuple(s), k
    assert "net.frame_endoder.layers.0.weight" in sd  # the reference's spelling (model.py:205)
    model.load_state_dict(synth.make_state_dict(shapes, seed=3))


def test_split_roundtrip():
    x = torch.randn(1000) * torch.logspace(-3, 3, 1000)
    s = lib.to_split(x)
    assert s.dtype == torch.bfloat16 and s.shape == (2, 1000)
    assert ((lib.from_split(s) - x).abs() / x.abs()).max() < 2 ** -15


def test_pack_weight_order():
    w = torch.randn(6, 10, 3, 3)
    p = lib.from_split(packing.pack_weight(w, [4, 6]))  # two segments -> each padded to 64
    assert p.shape == (6, 9 * 128)
    p = p.reshape(6, 9, 128)
    wt = w.reshape(6, 10, 9).permute(0, 2, 1)
    assert torch.allclose(p[:, :, 0:4], wt[:, :, 0:4], rtol=1e-4, atol=1e-6)
    assert torch.allclose(p[:, :, 64:70], wt[:, :, 4:10], rtol=1e-4, atol=1e-6)
    assert p[:, :, 4:64].abs().max() == 0 and p[:, :, 70:].abs().max() == 0


def test_fold_layernorm():
    torch.manual_seed(0)
    x = torch.randn(50, 32)
    w, b = torch.randn(16, 32), torch.randn(16)
    g, be = torch.randn(32), torch.randn(32)
    ref = F.linear(F.layer_norm(x, (32,), g, be), w, b)
    w2, b2 = packing.fold_layernorm(w, b, g, be)
    got = F.linear(F.layer_norm(x, (32,)), w2, b2)
    assert torch.allclose(got, ref, rtol=1e-4, atol=1e-4)
    # a zero row before LayerNorm becomes the LN bias (the reference's padded tokens)
    z = F.linear(F.layer_norm(torch.zeros(1, 32), (32,), g, be), w, b)
    assert torch.allclose(b2[None], z, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("b,t,H,W", [(1, 3, 64, 96), (1, 2, 72, 100), (2, 2, 80, 120), (1, 2, 720, 1280)])
def test_zone_and_window_maps(b, t, H, W):
    """The gather/scatter maps must reproduce the reference's pad + view + permute bookkeeping
    (attention_base.py:86-98, attention_flow.py:122-133)."""
    model, _ = _small_model()
    g = model.net._geometry(b, t, H, W, "cpu")
    h, w, n = g.h, g.w, g.n
    tok = torch.arange(b * t * n).reshape(b * t, h, w, 1).float()
    # temporal zones, as the reference does it
    gs = 2
    wh, ww = math.ceil(h / gs), math.ceil(w / gs)
    pad_r, pad_b = (ww - w % ww) % ww, (wh - h % wh) % wh
    x = F.pad(tok + 1, (0, 0, 0, pad_r, 0, pad_b)) - 1  # padded -> -1
    nh, nw = h + pad_b, w + pad_r
    x = x.view(b, t, gs, nh // gs, gs, nw // gs, 1, 1).permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(-1)
    assert torch.equal(x.to(torch.int32), g.zone_map)
    assert g.Lz == t * (nh // gs) * (nw // gs) and g.zones == b * 4
    # spatial windows
    ws = 8
    pad_r, pad_b = (ws - w % ws) % ws, (ws - h % ws) % ws
    x = F.pad(tok + 1, (0, 0, 0, pad_r, 0, pad_b)) - 1
    gh, gw = (h + pad_b) // ws, (w + pad_r) // ws
    x = x.reshape(b * t, gh, ws, gw, ws, 1).transpose(2, 3).reshape(b * t, gh * gw * ws * ws)
    wm = g.win_map.reshape(b * t, g.nwp * 64)
    assert torch.equal(x.to(torch.int32), wm[:, :g.nwin * 64])
    assert (wm[:, g.nwin * 64:] == -1).all()
    assert g.G == ((h + pad_b) // 4) * ((w + pad_r) // 4) and g.R % 64 == 0


def test_hidden_permutation_matches_fold():
    """Position-major hidden layout (p*C + c) is a pure re-indexing of nn.Fold's (c*P + p)."""
    model, _ = _small_model()
    perm = model.net._perm_hidden(40)
    hid = torch.randn(1, 35, 1960)  # 5x7 tokens
    ref = F.fold(hid.transpose(1, 2), (15, 21), (7, 7), stride=3, padding=3)
    hp = hid[:, :, perm].reshape(1, 5, 7, 49, 40)
    img = torch.zeros(1, 40, 15, 21)
    for ty in range(5):
        for tx in range(7):
            for p in range(49):
                y, x = ty * 3 + p // 7 - 3, tx * 3 + p % 7 - 3
                if 0 <= y < 15 and 0 <= x < 21:
                    img[0, :, y, x] += hp[0, ty, tx, p]
    assert torch.allclose(img, ref, atol=1e-5)


def test_c_abi_and_lib_call_reject_bad_arguments_without_touching_the_gpu(monkeypatch):
    """Error behaviour of the boundary (SURVEY 8b): a negative FGT_ERR_* code plus a thread-local message, checked
    before any CUDA call — so it can be exercised on a host without a device."""
    L = lib.load()
    L.fgt_last_error.restype = ctypes.c_char_p
    one = ctypes.c_void_p(8)                       # a non-null dummy; never dereferenced when validation fails first
    calls = [
        (L.fgt_poisson_setup, (None,) * 6 + (1, 4, 4) + (None,) * 6, "poisson_setup"),
        (L.fgt_poisson_setup, (one,) * 6 + (1, 1, 4) + (one,) * 6, "poisson_setup"),                    # H < 2
        (L.fgt_poisson_setup, (one,) * 6 + (1, 4096, 4096) + (one,) * 6, "2^24"),                      # H*W too large
        (L.fgt_poisson_iters, (None, 0, 1, 4, 4) + (None,) * 9 + (1, 1e-6, 1e-6, 1e8, 32, None), "poisson_iters"),
        (L.fgt_poisson_graph_launch, (None, None), "null graph"),
        (L.fgt_poisson_unfilled, (None, None, 1, 4, 4, None, None), "poisson_unfilled"),
        (L.fgt_poisson_finish, (None, None, None, 1, 4, 4, None, None, None, None), "poisson_finish"),
        (L.fgt_plane_max, (None, 1, 16, None, None), "plane_max"),
        (L.fgt_window_gather, (None,) * 5 + (1, 4, 4) + (None,) * 4, "window_gather"),
        (L.fgt_window_compose, (None,) * 5 + (1, 4, 4, None, None), "window_compose"),
        (L.fgt_comp_to_u8, (None, 16, None, None), "comp_to_u8"),
        (L.fgt_flow_splat, (None, None, 1, 1, 4, 4, 0, None, None, None), "flow_splat"),
        (L.fgt_regionfill_init, (None, None, 1, 4, 4, None, None, None, None, None), "regionfill_init"),
    ]
    for fn, args, needle in calls:
        rc = fn(*args)
        assert rc == -1, (fn.__name__, rc)          # FGT_ERR_ARG
        assert needle in L.fgt_last_error().decode(), (fn.__name__, L.fgt_last_error())
    assert L.fgt_poisson_graph_destroy(None) == 0   # destroying nothing is not an error
    monkeypatch.setattr(lib, "stream_ptr", lambda: None)
    with pytest.raises(RuntimeError, match="fgt_plane_max"):
        lib.call("fgt_plane_max", None, 1, 16, None)


# ------------------------------------------------------------------------------------------ round 2 host logic
def test_pack_weight_half_and_im2col():
    """1-term (fp16 single-plane) packing of the flow branch keeps pack_weight's K order; the im2col packing follows
    fgt_im2col_nchw's K index (ky*k + kx)*cin + c."""
    w = torch.randn(6, 10, 3, 3)
    h = packing.pack_weight(w, [4, 6], half=True)
    assert h.dtype == torch.float16 and h.shape == (6, 9 * 128)
    s = lib.from_split(packing.pack_weight(w, [4, 6]))
    assert torch.allclose(h.float(), s, rtol=2e-3, atol=1e-4)          # same layout, fp16 vs split-bf16 rounding
    w5 = torch.randn(8, 2, 5, 5)
    p = lib.from_split(packing.pack_weight_im2col(w5, cpad=64)).reshape(8, 64)
    for ky, kx, c in [(0, 0, 0), (0, 0, 1), (2, 3, 1), (4, 4, 0)]:
        assert torch.allclose(p[:, (ky * 5 + kx) * 2 + c], w5[:, c, ky, kx], rtol=1e-4, atol=1e-6)
    assert p[:, 50:].abs().max() == 0
    ph = packing.pack_weight_im2col(w5, cpad=64, half=True)
    assert ph.dtype == torch.float16 and ph.shape == (8, 64)


def test_fill_sms_tile_choice():
    """Channel-tile width by wave fill (fgt_model._fill_sms): 128 wide when the launch covers more than half a wave,
    halved (never below 64, never across a group boundary) when it does not."""
    from fgt_b200.fgt_model import _fill_sms
    assert _fill_sms(128, 512, 7200) == 128             # 57 x 4 = 228 tiles: > half a wave of 132 SMs
    assert _fill_sms(128, 512, 1440) == 64              # 12 x 4 = 48 tiles: 2 x 48 <= 132 -> 64 wide (96 tiles)
    assert _fill_sms(128, 512, 128) == 64               # a single row tile still stops at 64
    assert _fill_sms(64, 512, 128) == 64
    assert _fill_sms(128, 1536, 2160) == 128            # 17 x 12 = 204 tiles
    assert _fill_sms(128, 256, 720, groups=8) == 128    # 32 channels per group: a 64-wide tile must hold whole groups
    assert _fill_sms(128, 512, 720, groups=2) == 64


def test_bench_module_flops_match_survey():
    """bench.py's per-module denominators are SURVEY.md section 8(d)'s: 41.64 GFLOP per TMHSA layer, 3.091 GFLOP per
    frame per SWMHSA layer, 28.9 GFLOP per FFN layer at T = 10."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    f = bench.module_flops(10)
    assert abs(f["tmhsa"] / 1e9 - 41.64) < 0.01
    assert abs(f["swmhsa"] / 1e10 - 3.091) < 0.001
    assert abs(f["ffn"] / 1e9 - 28.9) < 0.01
    f2 = bench.module_flops(20)
    assert abs(f2["ffn"] / f["ffn"] - 2) < 1e-12 and f2["tmhsa"] / f["tmhsa"] > 2   # ∝ T and ∝ T + T^2
    # the arms of config 2 must describe the same workload (the driver compares the dicts)
    assert bench.config_dict(1).keys() == bench.config_dict(8).keys()
    assert bench.config_dict(1)["workload"] == bench.config_dict(8)["workload"]


def test_c_abi_rejects_bad_arguments_round2_entry_points():
    """Same contract for the entry points added in round 2 (include/fgt_b200.h): validation precedes any CUDA call."""
    L = lib.load()
    L.fgt_last_error.restype = ctypes.c_char_p
    one = ctypes.c_void_p(8)
    ll, f32 = ctypes.c_longlong, ctypes.c_float
    # fold_unfold: kernel smaller than the stride / patches that do not reach the map's last rows
    rc = L.fgt_fold_unfold(one, 1, 4, 4, 40, 2, 2, 3, 0, 12, 12, 1, one, ll(0), None)
    assert rc == -1 and "cover the stride" in L.fgt_last_error().decode()
    rc = L.fgt_fold_unfold(one, 1, 4, 4, 40, 7, 7, 3, 3, 60, 108, 1, one, ll(0), None)
    assert rc == -1 and "do not cover" in L.fgt_last_error().decode()
    rc = L.fgt_fold_unfold(None, 1, 20, 36, 40, 7, 7, 3, 3, 60, 108, 1, one, ll(0), None)
    assert rc == -1 and "fold_unfold" in L.fgt_last_error().decode()
    # dwconv / im2col argument checks
    rc = L.fgt_dwconv3x3_res(one, 1, 4, 4, 6, one, one, one, None, ll(0), None)
    assert rc == -1 and "multiple of 4" in L.fgt_last_error().decode()
    rc = L.fgt_im2col_nchw(one, 4, None, 0, 1, 8, 8, 3, 1, 1, 0, 8, 8, 32, f32(1), f32(0), one, ll(0), None)
    assert rc == -1 and "im2col_nchw" in L.fgt_last_error().decode()       # 3*3*4 = 36 > cpad 32
    rc = L.fgt_im2col_nchw(one, 4, None, 0, 1, 8, 4096, 7, 1, 3, 0, 8, 4096, 200, f32(1), f32(0), one, ll(0), None)
    assert rc == -1 and "staged input rows" in L.fgt_last_error().decode()  # 7 * 4 * 4102 floats > 160 KB
    # the fused SWMHSA operand preparation, the decoder tail and the device-side mask glue
    rc = L.fgt_swin_prep(one, one, 512, 256, 1, 20, 36, None, 960, 1024, 4, 6, 10, one, one, one, one, one, ll(0), one, ll(0),
                         f32(1e-5), None)
    assert rc == -1 and "swin_prep: null" in L.fgt_last_error().decode()
    rc = L.fgt_swin_prep(one, one, 512, 256, 1, 20, 36, one, 960, 1000, 4, 6, 10, one, one, one, one, one, ll(0), one, ll(0),
                         f32(1e-5), None)
    assert rc == -1 and "swin_prep" in L.fgt_last_error().decode()          # R = 1000 < 960 local + 60 pooled rows
    rc = L.fgt_conv_tail(one, ll(0), 1, 8, 8, 64, one, ll(0), 64, 4, one, 0, one, ll(0), ll(0), ll(0), ll(0), None)
    assert rc == -1 and "cout=4" in L.fgt_last_error().decode()
    rc = L.fgt_conv_tail(one, ll(0), 1, 8, 8, 48, one, ll(0), 48, 3, one, 0, one, ll(0), ll(0), ll(0), ll(0), None)
    assert rc == -1 and "conv_tail" in L.fgt_last_error().decode()          # cin must be a multiple of 64
    rc = L.fgt_conv_tail(one, ll(0), 1, 8, 8, 64, one, ll(0), 64, 3, one, 5, one, ll(0), ll(0), ll(0), ll(0), None)
    assert rc == -1 and "act=5" in L.fgt_last_error().decode()              # LeakyReLU(0.01) has no tail epilogue
    rc = L.fgt_binary_dilate(one, 1, 4, 4, 1, one, one, None)
    assert rc == -1 and "alias" in L.fgt_last_error().decode()
    rc = L.fgt_binary_dilate(one, 1, 4, 4, 0, ctypes.c_void_p(16), ctypes.c_void_p(24), None)
    assert rc == -1 and "binary_dilate" in L.fgt_last_error().decode()      # iterations >= 1
    rc = L.fgt_resize_nearest_u8(one, 1, 4, 4, 1, 0, 4, one, None)
    assert rc == -1 and "resize_nearest" in L.fgt_last_error().decode()
    rc = L.fgt_resize_bilinear_f32(None, 1, 4, 4, 1, 8, 8, 0, f32(1), f32(1), one, None)
    assert rc == -1 and "resize_bilinear" in L.fgt_last_error().decode()
    rc = L.fgt_fill_holes_pass(one, 1, 4, 4, one, None, 1, None)
    assert rc == -1 and "fill_holes" in L.fgt_last_error().decode()
