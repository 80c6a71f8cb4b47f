"""The GEMM engine's tile schedule that issues the next tile's first K stage before a tile's epilogue, and its batched
epilogue (operand loads before the accumulators are final, 16-byte stores after a quad exchange), against the previous
schedule (`fgt_debug_gemm_serial_epilogue(1)`: no early stage, per-pair epilogue). Both run the same MMAs in the same
order and the same per-element arithmetic, so every output must be bit-identical: tiles per CTA of 1, 2, 3 (odd and
even), 1-9 K steps, bn 16/64/96/128, 1- and 3-term operands, in-place residual, gate multiply, activations, fp32 + split
and fp16 outputs, partial row tiles, N tails and a rowmap scatter."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

TILES = (1, 131, 132, 133, 264, 265, 3 * 132 + 1)


def _lib():
    from fgt_b200 import lib
    L = lib.load()
    L.fgt_debug_gemm_serial_epilogue.argtypes = [ctypes.c_int]
    return lib, L


def _both(run):
    """run() -> tuple of output tensors, once with each schedule."""
    _, L = _lib()
    res = []
    for serial in (1, 0):
        L.fgt_debug_gemm_serial_epilogue(serial)
        try:
            res.append(run())
            torch.cuda.synchronize()
        finally:
            L.fgt_debug_gemm_serial_epilogue(0)
    return res


def _operands(M, N, K, terms, seed):
    from fgt_b200 import lib, packing
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, K, device=dev, generator=g)
    w = torch.randn(N, K, device=dev, generator=g) / K ** 0.5
    b = torch.randn(N, device=dev, generator=g)
    if terms == 1:
        return a.half().contiguous(), packing.pack_weight(w, half=True).to(dev), b
    return lib.to_split(a), packing.pack_weight(w).to(dev), b


def _assert_equal(outs, what):
    old, new = outs
    for i, (o, n) in enumerate(zip(old, new)):
        assert torch.equal(o, n), f"{what}: output {i} differs between the schedules"


@pytest.mark.parametrize("terms", (3, 1))
@pytest.mark.parametrize("bn", (16, 64, 96, 128))
@pytest.mark.parametrize("tiles", TILES)
def test_schedules_bit_identical_tiles_and_k_steps(tiles, bn, terms):
    """1 to 9 K steps (the early stage is one of them), 1-4 tiles per CTA, the last row tile partial; x += A W^T + b in
    place with its split copy (the out-projection / ffn2 epilogue)."""
    lib, _ = _lib()
    dev = torch.device("cuda:0")
    N = bn
    M = 128 * tiles - 37
    for k_steps in range(1, 10):
        K = 64 * k_steps
        a_p, w_p, b = _operands(M, N, K, terms, seed=1000 * tiles + k_steps)
        x0 = torch.randn(M, N, device=dev)

        def run():
            x = x0.clone()
            xs = torch.full((2, M, N), float("nan"), dtype=torch.bfloat16, device=dev)
            lib.gemm_tc([lib.ASeg(a_p, K, M)], w_p, N, out_w=M, bn=bn, bias=b, aux=x, aux_mode=lib.AUX_ADD,
                        out_f32=x, out_split=xs, terms=terms)
            return x, xs

        _assert_equal(_both(run), f"tiles={tiles} bn={bn} terms={terms} K={K}")


@pytest.mark.parametrize("bn", (64, 128))
@pytest.mark.parametrize("act", ("none", "leaky02", "relu", "sigmoid", "tanh", "leaky001"))
# "half" is not an aux mode: aux NONE with 1-term operands and fp16 + fp32 outputs (the out_half rounding path)
@pytest.mark.parametrize("aux_mode", ("none", "add", "mul", "add_pre", "add_relu", "gru", "gru_zr", "half"))
def test_schedules_bit_identical_epilogues(aux_mode, act, bn):
    """Every kExt = 0 activation x aux mode, fp32 + split outputs, M tail (1500 rows) and an N tail (N = 712); and the
    kExt = 1 instantiation: LeakyReLU(0.01), pre-activation add, add + ReLU, the GRU update (aux2 = z), the fused z | r
    gates (N = 256, two C-channel outputs) and 1-term fp16 + fp32 outputs ("half", the mixed-precision rounding)."""
    lib, _ = _lib()
    dev = torch.device("cuda:0")
    M, K = 1500, 320
    N = 256 if aux_mode == "gru_zr" else 712
    terms = 1 if aux_mode == "half" else 3
    a_p, w_p, b = _operands(M, N, K, terms, seed=5)
    aux = torch.randn(M, N, device=dev)
    z = torch.rand(M, N, device=dev)
    acts = dict(none=lib.ACT_NONE, leaky02=lib.ACT_LEAKY02, relu=lib.ACT_RELU, sigmoid=lib.ACT_SIGMOID,
                tanh=lib.ACT_TANH, leaky001=lib.ACT_LEAKY001)
    modes = dict(none=lib.AUX_NONE, add=lib.AUX_ADD, mul=lib.AUX_MUL, add_pre=lib.AUX_ADD_PRE,
                 add_relu=lib.AUX_ADD_RELU, gru=lib.AUX_GRU, gru_zr=lib.AUX_GRU_ZR, half=lib.AUX_NONE)

    def run():
        if aux_mode == "gru_zr":   # z -> fp32 [M, N/2], r*h -> split [M, N/2], h = aux [M, N/2]
            zo = torch.full((M, N // 2), float("nan"), device=dev)
            rh = torch.full((2, M, N // 2), float("nan"), dtype=torch.bfloat16, device=dev)
            lib.gemm_tc([lib.ASeg(a_p, K, M)], w_p, N, out_w=M, bn=bn, bias=b, act=acts[act],
                        aux=aux[:, :N // 2].contiguous(), aux_mode=lib.AUX_GRU_ZR, out_f32=zo, out_split=rh, os_x=N // 2)
            return zo, rh
        o32 = torch.full((M, N), float("nan"), device=dev)
        if aux_mode == "half":
            osp = torch.full((M, N), float("nan"), dtype=torch.float16, device=dev)
        else:
            osp = torch.full((2, M, N), float("nan"), dtype=torch.bfloat16, device=dev)
        lib.gemm_tc([lib.ASeg(a_p, K, M)], w_p, N, out_w=M, bn=bn, bias=b, act=acts[act],
                    aux=aux if aux_mode not in ("none", "half") else None, aux_mode=modes[aux_mode],
                    aux2=z if aux_mode == "gru" else None, out_f32=o32, out_split=osp)
        return o32, osp

    _assert_equal(_both(run), f"aux={aux_mode} act={act} bn={bn}")


@pytest.mark.parametrize("bn", (16, 64, 96, 128))
def test_schedules_bit_identical_fp16_output_and_no_bias(bn):
    """1-term operands into a single fp16 plane (the flow branch), no bias, alpha != 1."""
    lib, _ = _lib()
    dev = torch.device("cuda:0")
    M, N, K = 7200 - 5, 2 * bn, 448
    a_p, w_p, _ = _operands(M, N, K, 1, seed=11)

    def run():
        o16 = torch.full((M, N), float("nan"), dtype=torch.float16, device=dev)
        lib.gemm_tc([lib.ASeg(a_p, K, M)], w_p, N, out_w=M, bn=bn, alpha=0.75, act=lib.ACT_LEAKY02, out_f16=o16,
                    terms=1)
        return (o16,)

    _assert_equal(_both(run), f"fp16 out bn={bn}")


@pytest.mark.parametrize("bn", (64, 128))
def test_schedules_bit_identical_rowmap_scatter(bn):
    """Rows scattered through a rowmap (reversed, every 7th dropped) with an in-place residual at the destination."""
    lib, _ = _lib()
    dev = torch.device("cuda:0")
    M, N, K = 5000, 256, 192
    a_p, w_p, b = _operands(M, N, K, 3, seed=13)
    rowmap = torch.arange(M - 1, -1, -1, dtype=torch.int32, device=dev)
    rowmap[::7] = -1
    x0 = torch.randn(M, N, device=dev)

    def run():
        x = x0.clone()
        lib.gemm_tc([lib.ASeg(a_p, K, M)], w_p, N, out_w=M, bn=bn, bias=b, out_f32=x, aux=x, aux_mode=lib.AUX_ADD,
                    rowmap=rowmap)
        return (x,)

    _assert_equal(_both(run), f"rowmap bn={bn}")


def test_schedules_bit_identical_conv_edge_boxes():
    """A 3x3 conv over NHWC with partial output boxes at the right / bottom edges (non-linear addressing)."""
    lib, _ = _lib()
    from fgt_b200 import packing
    dev = torch.device("cuda:0")
    n, h, w, cin, cout = 2, 61, 107, 64, 128
    g = torch.Generator(device=dev).manual_seed(17)
    x = lib.to_split(torch.randn(n, h, w, cin, device=dev, generator=g))
    wt = torch.randn(cout, cin, 3, 3, device=dev, generator=g) / (9 * cin) ** 0.5
    w_p = packing.pack_weight(wt).to(dev)
    b = torch.randn(cout, device=dev, generator=g)

    def run():
        o = torch.full((n, h, w, cout), float("nan"), device=dev)
        lib.gemm_tc([lib.ASeg(x, cin, w, h, n)], w_p, cout, kx=3, ky=3, pad_x=1, pad_y=1, out_w=w, out_h=h, out_z=n,
                    box_w=16, box_h=8, bn=128, bias=b, act=lib.ACT_LEAKY02, out_f32=o, os_z=h * w * cout,
                    os_y=w * cout, os_x=cout, os_c=1)
        return (o,)

    _assert_equal(_both(run), "conv 3x3 edge boxes")
