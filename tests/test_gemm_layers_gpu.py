"""The GEMM engine on the layer forms of tests/test_gemm_layers.py at production geometries, against the float64
interpreter (tests/gemm_emulator.py) fed identical operands; and the extended (kExt = 1) epilogues replayed exactly on
the kernel's own accumulators.

Geometries: FGT's encoder at the 60 x 108 feature map (2 frames), its decoder deconv at 60 x 108 -> 120 x 216, the
fused Q|K|V rows of a 2-frame window; LAFC at 60 x 108 per frame; RAFT at 1/8 of 480 x 864 (60 x 108).
Bars (max error over the largest value): split-bf16 (3-term) layers KTOL; fp16 (1-term) layers with fp32 outputs 2e-4
as tools/diag_gemm.py's linear_case; 1-term layers whose outputs are fp16 (or fp32 copies of fp16 values) 2^-9: one
fp16 ulp of values in the largest value's binade, measured against a largest value that may sit just below that binade,
since the kernel's float32 and the interpreter's float64 values may round to neighbouring fp16 values (the mixed GRU
state showed 9.8e-4, one ulp at 1.0). Elements the descriptor does not address: bit-identical to the sentinel.
"""
import pytest
import torch

from fgt_b200 import lib
from tests import test_gemm_layers as L
from tests.gemm_emulator import emulating

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _tol(case):
    if not case["f16"]:
        return L.KTOL
    return 2.0 ** -9 if any(b.dtype == torch.float16 for b in case["bufs"].values()) else 2e-4


@pytest.mark.parametrize("name,mixed", L.PARAMS)
def test_kernel_matches_emulator_on_layer_forms(name, mixed):
    """The elements the kernel writes are the ones the interpreter writes (tests/test_gemm_layers.py checks those
    against the layer's own statement of its slice); the rest keep their sentinel bit for bit."""
    gpu = L.CASES[name](DEV, big=True, mixed=mixed)
    before = {k: v.cpu().clone() for k, v in gpu["bufs"].items()}
    with torch.no_grad():
        gpu["run"]()
    torch.cuda.synchronize()
    cpu = L.CASES[name](torch.device("cpu"), big=True, mixed=mixed)
    with torch.no_grad(), emulating() as emu:
        cpu["run"]()
    tol = _tol(gpu)
    for bname, (decode, _) in cpu["place"].items():
        got_raw, want_raw = gpu["bufs"][bname].cpu(), cpu["bufs"][bname]
        raw_mask = emu.written_mask(want_raw)
        written = raw_mask.any(0) if want_raw.dtype == torch.bfloat16 else raw_mask   # split: [2, ...] planes
        assert torch.equal(got_raw[~raw_mask], before[bname][~raw_mask]), f"{name}: {bname} written outside its slice"
        got, want = decode(got_raw)[written], decode(want_raw)[written]
        assert torch.isfinite(got).all(), f"{name}: {bname} non-finite"
        err = (got - want).abs().max().item() / (want.abs().max().item() + 1e-30)
        assert err <= tol, f"{name} mixed={mixed}: {bname} kernel vs emulator {err:.3e} (tol {tol:g})"


# ------------------------------------------------------------------------------------------ exact extended epilogues
M, N, K = 1000, 256, 192


def _ops(terms, seed=7):
    from fgt_b200 import packing
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(M, K, device=DEV, generator=g)
    w = torch.randn(N, K, device=DEV, generator=g) / K ** 0.5
    b = torch.randn(N, device=DEV, generator=g) * 0.5
    if terms == 1:
        return a.half().contiguous(), packing.pack_weight(w, half=True).to(DEV), b
    return lib.to_split(a), packing.pack_weight(w).to(DEV), b


def _launch(a, w, b, bn, n=N, **kw):
    lib.gemm_tc([lib.ASeg(a, K, M)], w, n, out_w=M, bn=bn, bias=b, **kw)


def _base(a, w, b, bn):
    """v = fmaf(acc, alpha, bias): the value every epilogue starts from (same operands, bn and box)."""
    v = torch.full((M, N), float("nan"), device=DEV)
    _launch(a, w, b, bn, out_f32=v)
    return v


def _r16(x):
    return x.half().float()


def _nan(shape=(M, N), dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


@pytest.mark.parametrize("bn", (64, 128))
@pytest.mark.parametrize("terms", (3, 1))
def test_extended_epilogues_bit_exact(terms, bn):
    """ADD_PRE, ADD_RELU, LEAKY001 and GRU_ZR (act none: z = v, r*h = v * h) in fp32 arithmetic, replayed on v in
    torch: bit-identical. Observed: identical."""
    a, w, b = _ops(terms)
    v = _base(a, w, b, bn)
    aux = torch.randn(M, N, device=DEV)
    out = _nan()
    _launch(a, w, b, bn, act=lib.ACT_LEAKY001, aux=aux, aux_mode=lib.AUX_ADD_PRE, out_f32=out)
    x = v + aux
    assert torch.equal(out, torch.where(x > 0, x, 0.01 * x)), "ADD_PRE + LEAKY001"
    out = _nan()
    _launch(a, w, b, bn, act=lib.ACT_LEAKY001, out_f32=out)
    assert torch.equal(out, torch.where(v > 0, v, 0.01 * v)), "LEAKY001"
    out = _nan()
    _launch(a, w, b, bn, act=lib.ACT_RELU, aux=aux, aux_mode=lib.AUX_ADD_RELU, out_f32=out)
    assert torch.equal(out, (v.clamp_min(0) + aux).clamp_min(0)), "ADD_RELU"
    h = torch.randn(M, N // 2, device=DEV)
    z = _nan((M, N // 2))
    rh = _nan((M, N // 2), torch.float16) if terms == 1 else lib.to_split(_nan((M, N // 2)))
    _launch(a, w, b, bn, aux=h, aux_mode=lib.AUX_GRU_ZR, out_f32=z, out_split=rh, os_x=N // 2)
    if terms == 1:   # out_half: v rounded to fp16 before the (identity) activation and after it
        assert torch.equal(z, _r16(v[:, :N // 2])), "GRU_ZR z (fp16)"
        assert torch.equal(rh, (_r16(v[:, N // 2:]) * h).half()), "GRU_ZR r*h (fp16)"
    else:
        assert torch.equal(z, v[:, :N // 2]), "GRU_ZR z"
        assert torch.equal(rh, lib.to_split(v[:, N // 2:] * h)), "GRU_ZR r*h"


@pytest.mark.parametrize("bn", (64, 128))
def test_fp16_output_epilogues_bit_exact(bn):
    """1-term launches with fp16 + fp32 outputs (mixed-precision RAFT): v rounded to fp16 before the activation and
    again after it; ADD_RELU rounds act(v) before the residual; the GRU update rounds (1 - z), (1 - z) h, z q and their
    sum. The fp32 copy equals the fp16 output. Replayed in torch fp32 with explicit fp16 roundings: bit-identical.
    Observed: identical."""
    a, w, b = _ops(1)
    v = _base(a, w, b, bn)
    aux = _r16(torch.randn(M, N, device=DEV))
    z = torch.sigmoid(torch.randn(M, N, device=DEV)).half().float()

    def both(**kw):
        o32, o16 = _nan(), _nan(dtype=torch.float16)
        _launch(a, w, b, bn, out_f32=o32, out_split=o16, **kw)
        assert torch.equal(o32, o16.float()), f"{kw}: fp32 copy != fp16 output"
        return o32

    x = _r16(v)
    assert torch.equal(both(act=lib.ACT_LEAKY02), _r16(torch.where(x > 0, x, 0.2 * x))), "out_half LeakyReLU"
    got = both(act=lib.ACT_RELU, aux=aux, aux_mode=lib.AUX_ADD_RELU)
    assert torch.equal(got, _r16((_r16(x.clamp_min(0)) + aux).clamp_min(0))), "out_half ADD_RELU"
    got = both(aux=aux, aux2=z, aux_mode=lib.AUX_GRU)
    q = _r16(x)
    assert torch.equal(got, _r16(_r16(_r16(_r16(1 - z) * aux) + _r16(z * q)))), "out_half GRU"


@pytest.mark.parametrize("bn", (64, 128))
def test_fp32_gru_update_within_two_ulps(bn):
    """fp32 GRU update h' = (1 - z) h + z q: nvcc may contract it into an FMA, so within 2 fp32 ulps of the float64
    formula on the kernel's own q, in ulps of |(1 - z) h| + |z q| (2 ulps of the result itself do not bound the
    rounding of the two terms where they cancel: that bound failed on H100)."""
    a, w, b = _ops(3)
    v = _base(a, w, b, bn)
    h = torch.randn(M, N, device=DEV)
    z = torch.rand(M, N, device=DEV)
    out = _nan()
    _launch(a, w, b, bn, aux=h, aux2=z, aux_mode=lib.AUX_GRU, out_f32=out)
    t0, t1 = (1 - z.double()) * h.double(), z.double() * v.double()
    want = t0 + t1
    # ulps of |t0| + |t1|: where the two terms cancel, the ulp of the sum understates the rounding of each term
    mag = (t0.abs() + t1.abs()).float()
    ulp = (torch.nextafter(mag, torch.tensor(float("inf"), device=DEV)) - mag).double()
    assert ((out.double() - want).abs() <= 2 * ulp).all(), "fp32 GRU beyond 2 ulps"


@pytest.mark.parametrize("act", (lib.ACT_SIGMOID, lib.ACT_TANH))
def test_sigmoid_tanh_within_1e6(act):
    """Sigmoid / tanh on v: within 1e-6 absolute of float64. After the fp16 rounding of a 1-term out_half launch,
    equal to the rounded float64 value except where that lies within 1e-6 of an fp16 rounding boundary.
    Observed on H100: both bars hold."""
    f64 = torch.sigmoid if act == lib.ACT_SIGMOID else torch.tanh
    a, w, b = _ops(3)
    v = _base(a, w, b, 128)
    out = _nan()
    _launch(a, w, b, 128, act=act, out_f32=out)
    assert (out.double() - f64(v.double())).abs().max().item() <= 1e-6
    a, w, b = _ops(1)
    v = _base(a, w, b, 128)
    o32, o16 = _nan(), _nan(dtype=torch.float16)
    _launch(a, w, b, 128, act=act, out_f32=o32, out_split=o16)
    y = f64(_r16(v).double())
    assert (y - o32.double()).abs().max().item() <= 1e-3   # fp16 rounding of values in [-1, 1]
    near = ((y + 1e-6).half() != (y - 1e-6).half())
    assert torch.equal(o16[~near], y[~near].half()), "fp16 sigmoid / tanh off a rounding boundary"
