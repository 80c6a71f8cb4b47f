"""The GEMM engine's persistent schedule: one CTA per SM (132 on an H100 SXM) walks its tiles through one stage ring,
and a channel tile requested wider than 128 runs as narrower tiles. Launches with 1 tile, just under / at / just over
one and two waves, and 3 waves + 1 tile, with 1 to 9 K steps (more than the ring's 3-6 stages), are checked against a
float64 product of the rounded operands; and a tile computed in a many-tile launch must be bit-identical to the same
tile computed alone, whichever CTA ran it."""
import pytest
import torch

from tests.util import assert_close

pytestmark = pytest.mark.gpu

TILES = (1, 131, 132, 133, 264, 265, 3 * 132 + 1)
KTOL = 1e-4  # as tests/test_kernels_gpu.py: split-bf16 3-term products lose the lo x lo term (~2^-16)


def _operands(M, N, K, terms, seed):
    from fgt_b200 import lib, packing
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, K, device=dev, generator=g)
    w = torch.randn(N, K, device=dev, generator=g) / K ** 0.5
    b = torch.randn(N, device=dev, generator=g)
    if terms == 1:
        a_p, w_p = a.half().contiguous(), packing.pack_weight(w, half=True).to(dev)
        a_r, w_r = a_p.double(), w_p.double()
    else:
        a_p, w_p = lib.to_split(a), packing.pack_weight(w).to(dev)
        a_r, w_r = lib.from_split(a_p).double(), w_p[0].double() + w_p[1].double()
    return a_p, w_p, b, a_r, w_r


def _gemm(a_p, w_p, b, M, N, K, bn, terms):
    from fgt_b200 import lib
    out = torch.full((M, N), float("nan"), device=a_p.device)
    lib.gemm_tc([lib.ASeg(a_p, K, M)], w_p, N, out_w=M, bn=bn, bias=b, out_f32=out, terms=terms)
    return out


@pytest.mark.parametrize("terms", (3, 1))
@pytest.mark.parametrize("bn", (16, 64, 128, 256))
@pytest.mark.parametrize("tiles", TILES)
def test_tile_counts_and_k_steps(tiles, bn, terms):
    """bn=256 runs as two 128-wide tiles per 128 rows: N=256 and half as many row tiles (rounded up)."""
    from fgt_b200 import lib
    lib.load()
    N = bn
    m_tiles = tiles if bn <= 128 else -(-tiles // 2)
    M = 128 * m_tiles - 37  # the last row tile is partial
    for k_steps in range(1, 10):
        K = 64 * k_steps
        a_p, w_p, b, a_r, w_r = _operands(M, N, K, terms, seed=1000 * tiles + k_steps)
        out = _gemm(a_p, w_p, b, M, N, K, bn, terms)
        torch.cuda.synchronize()
        ref = a_r @ w_r.t() + b.double()
        assert_close(out, ref, tol=KTOL, what=f"tiles={tiles} bn={bn} terms={terms} K={K}")


@pytest.mark.parametrize("terms", (3, 1))
@pytest.mark.parametrize("bn", (64, 128))
def test_tile_bits_independent_of_schedule(bn, terms):
    """265 row tiles on 132 CTAs: CTA 0 runs tiles 0, 132 and 264, CTA 1 tiles 1 and 133, each at a different point of
    its stage ring. Each of those tiles, recomputed as a one-tile launch, gives the same bits."""
    from fgt_b200 import lib
    lib.load()
    M, N, K = 265 * 128, bn, 64 * 7
    a_p, w_p, b, _, _ = _operands(M, N, K, terms, seed=7)
    full = _gemm(a_p, w_p, b, M, N, K, bn, terms)
    for t in (0, 1, 132, 133, 264):
        rows = slice(128 * t, 128 * t + 128)
        a_t = a_p[rows] if terms == 1 else a_p[:, rows]
        alone = _gemm(a_t, w_p, b, 128, N, K, bn, terms)
        torch.cuda.synchronize()
        assert torch.equal(full[rows], alone), f"tile {t}: bits differ from the one-tile launch"
