"""FGT's mixed-precision mode (FGT.enable_mixed_precision), CPU side: the switch and its guards, the fp16 weight
pack against the fp32 one, the command-line option, and the C-ABI's checks of the fp16 (single-plane) argument
forms. The numerics are defined by CUDA autocast and checked on the GPU (tests/test_fgt_mixed_gpu.py)."""
import ctypes

import pytest
import torch

from fgt_b200 import lib, synth


class _Stop(Exception):
    pass


def _model(seed=1):
    from fgt_b200.fgt_model import Model
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    m = Model(cfg)
    m.load_state_dict(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=seed))
    return m


def test_enable_and_disable():
    net = _model().net
    assert net._mixed is False
    net.enable_mixed_precision()
    assert net._mixed is True
    net.enable_mixed_precision(False)
    assert net._mixed is False
    with pytest.raises(RuntimeError, match="CUDA"):  # CPU tensors: no fallback in either mode
        net.enable_mixed_precision(True)
        net(*synth.fgt_inputs(seed=0, t=2, H=64, W=96))


def test_frame_sharding_is_rejected_in_either_order():
    net = _model().net
    net.enable_mixed_precision(True)
    with pytest.raises(ValueError, match="frame sharding"):
        net.enable_frame_sharding(4, rank=0, world=2, exchange="nccl")
    net.enable_mixed_precision(False)
    net.enable_frame_sharding(4, rank=0, world=2, exchange="nccl")
    with pytest.raises(ValueError, match="frame sharding"):
        net.enable_mixed_precision(True)
    net.enable_mixed_precision(False)  # turning it off is always allowed
    net.enable_frame_sharding(None)
    net.enable_mixed_precision(True)


def test_half_pack_is_the_rounded_fp32_pack():
    """Layer for layer, the fp16 pack holds the fp32 pack's values rounded to fp16 (LayerNorm folds in fp64, then one
    rounding), in the same layouts; the norm kernel's own affines stay fp32."""
    net = _model(seed=4).net
    cpu = torch.device("cpu")
    p32 = net._pack(cpu, half=False)
    p16 = net._pack(cpu, half=True)
    assert set(p32) == set(p16) and set(net._packed) == {False, True}

    def close16(a, b, what):
        a, b = a.double(), b.double()
        assert a.shape == b.shape, what
        assert ((a - b).abs() <= b.abs() * 2.0 ** -11 + 2.0 ** -24).all(), what  # half an fp16 ulp

    for k in p32:
        a, b = p16[k], p32[k]
        if isinstance(b, dict):
            want = lib.from_split(b["w"]) if b["w"].dtype == torch.bfloat16 else b["w"].float()
            assert a["w"].dtype == torch.float16, k
            if k.startswith(("dec1.p", "dec3.p")):  # sub-pixel phases: sums of fp16-rounded taps, then rounded once
                assert ((a["w"].double() - want.double()).abs() <= 2.0 ** -9 * want.abs().max()).all(), k
            else:
                close16(a["w"].float(), want, k + ".w")
            close16(a["b"], b["b"], k + ".b")
            assert torch.equal(a["b"], a["b"].half().float()), k   # biases are fp16 values
            assert a["N"] == b["N"]
        elif k.endswith((".ln_g", ".ln_b")):
            assert torch.equal(a, b), k
        else:
            close16(a, b, k)
            assert torch.equal(a, a.half().float()), k


def test_command_line_option_and_make_args(monkeypatch):
    from fgt_b200 import pipeline
    base = ["--path", "frames", "--path_mask", "masks", "--outroot", "out"]
    assert pipeline.arg_parser().parse_args(base).fgt_mixed_precision is False
    ns = pipeline.arg_parser().parse_args(base + ["--fgt_mixed_precision"])
    assert ns.fgt_mixed_precision is True and ns.mixed_precision is False  # independent of RAFT's switch
    seen = {}

    def fake_load(raft_model, lafc_ckpts, fgt_ckpts, device, mixed_precision=False, fgt_mixed_precision=False):
        seen.update(mp=mixed_precision, fmp=fgt_mixed_precision)
        raise _Stop

    monkeypatch.setattr(pipeline, "load_models", fake_load)
    for argv, want in (([], (False, False)), (["--fgt_mixed_precision"], (False, True)),
                       (["--mixed_precision"], (True, False))):
        with pytest.raises(_Stop):
            pipeline.main(base + argv)
        assert (seen.pop("mp"), seen.pop("fmp")) == want
    assert "fgt_mixed_precision" not in pipeline.DEFAULTS
    with pytest.raises(TypeError):
        pipeline.make_args(fgt_mixed_precision=True)


def test_c_abi_rejects_bad_fp16_arguments_without_touching_the_gpu():
    L = lib.load()
    one = ctypes.c_void_p(64)   # non-null dummies; never dereferenced when validation fails first
    odd = ctypes.c_void_p(66)
    ptrs = (ctypes.c_void_p * 2)(64, 128)

    def attn(f16, plane):
        d = lib.FgtAttnDesc()
        d.q_hi = d.k_hi = d.v_hi = d.out_hi = 64
        d.q_plane = d.k_plane = d.v_plane = d.out_plane = plane
        d.q_ld = d.k_ld = d.v_ld = d.out_ld = 512
        d.batches, d.heads, d.head_dim, d.Lq, d.Lk, d.Lk_rows = 1, 4, 128, 128, 128, 128
        d.f16 = f16
        return L.fgt_attention(ctypes.byref(d), None)

    calls = [
        (lambda: attn(1, 4096), "plane offsets must be 0"),
        (lambda: attn(2, 0), "f16=2"),
        (lambda: L.fgt_conv_tail(one, 0, 1, 8, 8, 64, one, 4096, 64, 3, one, 0, one, 0, 0, 0, 0, None),
         "both split-bf16"),
        (lambda: L.fgt_swin_prep(one, one, 512, 256, 1, 8, 8, one, 64, 128, 4, 2, 2, one, one, one, one, one, 0, one,
                                 4096, 1e-5, None), "both split-bf16"),
        (lambda: L.fgt_rownorm_bcast(one, 512, 512, None, 0, 0, None, 8, 8, 8, 0, None, None, ptrs, 2, 0, 1e-5, None),
         "one destination"),
        (lambda: L.fgt_rownorm(one, 512, 512, None, 0, 0, None, 8, 8, 8, 0, None, None, odd, 0, 1e-5, None),
         "misaligned"),
        (lambda: L.fgt_fold_unfold(one, 1, 4, 4, 64, 7, 7, 3, 3, 10, 10, 1, one, -4, None), "plane offset"),
        (lambda: L.fgt_fold(one, 1, 4, 4, 64, 7, 7, 3, 3, 10, 10, 0, None, None, odd, 0, None), "misaligned"),
        (lambda: L.fgt_dwconv3x3_res(one, 1, 4, 4, 64, one, one, one, one, 6, None), "plane offset"),
    ]
    for fn, needle in calls:
        assert fn() == -1, needle                   # FGT_ERR_ARG
        assert needle in L.fgt_last_error().decode(), (needle, L.fgt_last_error())
