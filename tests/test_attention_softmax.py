"""The designed attention cases of tests/attention_cases.py against the float64 model of flash_kernel's online-softmax
schedule, on the CPU: every case takes the branches it is named for (rescales per row and at which tiles, alpha
underflow, P near 2^8 in fp16, masked columns above the live maximum, the windowed key order), so a generator that
drifts stops passing here rather than silently covering less on the GPU; and the model equals torch.softmax in float64
(exactly up to 1e-12 with P unrounded, within its own P-rounding bar with P rounded)."""
import math

import pytest
import torch

from tests import attention_cases as A

CASES = {c.name: c for c in A.all_cases()}


def _groups(case, f16):
    """(b, h, rows, kidx, live, scores as loaded, Schedule) of every group."""
    for b, h, rows, kidx, live in case.groups():
        s, v = case.loaded(b, h, rows, kidx)
        yield b, h, rows, kidx, live, s, A.schedule(s, live, case.scale, f16, v)


def _steps(s, live, scale):
    """[rows, T - 1] fp32 steps between consecutive tile maxima, log2 units."""
    m = torch.where(live, s, torch.tensor(-math.inf)).amax(-1) * A.c32(scale)
    return (m[:, 1:] - m[:, :-1]).double()


def test_exact_scale_is_a_quarter_and_operands_are_16_bit_exact():
    assert float(A.c32(A.EXACT_SCALE)) == 0.25 and A.EXACT_SCALE > A.FGT_SCALE
    for c in CASES.values():
        for t in (c.q, c.k, c.v):
            assert torch.equal(t.bfloat16().double(), t) and torch.equal(t.half().double(), t), c.name
        assert c.v.abs().max() >= 61440, c.name   # V reaches +-6e4
        assert c.B > 1 and c.H > 1 and bool((c.rowmap < 0).any()), c.name
        if c.mode == 0:
            assert c.Lq % 128 != 0, c.name


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith("rise")])
def test_rising_maxima(name):
    c = CASES[name]
    d, T = c.intent["delta"], c.intent["tiles"]
    for f16 in (False, True):
        for b, h, rows, kidx, live, s, sch in _groups(c, f16):
            steps = _steps(s, live, c.scale)
            n = sch.rescales_after_first()
            if c.scale == A.EXACT_SCALE:
                assert bool((steps == d).all())
            else:
                assert bool(((steps - d).abs() < max(0.07, 0.01 * d)).all())   # bf16 S: 8 significant bits
            if d < 8 or (d == 8 and c.scale == A.EXACT_SCALE):   # every other tile; P reaches 2^d in between
                assert bool((n == (T - 1) // 2).all())
                assert bool((sch.grow[:, 1::2] == 0).all())
                assert sch.p16max.max() >= (256.0 if d == 8 else 128.0)
            elif d == 8:                                         # on the threshold: some step lands either side
                assert bool((n >= 2).all()) and bool(((steps > 8) & (steps < 8.07)).any())
            else:                                                # every tile, the newest maximum at P = 1
                assert bool((n == T - 1).all())
                assert sch.pmax[:, 1:].max() < 1.0 + 2.0 ** -16
                a = sch.alpha[:, 1:]
                if d == 140:                                     # alpha = 2^-140 flushed to 0
                    assert bool((a == 0).all())
                elif d == 40:
                    assert bool(((a > 0) & (a < 2.0 ** -39)).all())
                elif d == 16:
                    assert bool(((a > 2.0 ** -16.1) & (a < 2.0 ** -15.9)).all())


def test_falling_maxima_underflow():
    c = CASES["fall40"]
    for b, h, rows, kidx, live, s, sch in _groups(c, True):
        assert bool((sch.rescales_after_first() == 0).all())
        assert bool((sch.pmax[:, 4:] == 0).all())        # 2^-160 and below: flushed
        assert bool((sch.pmax[:, 3] > 0).all())          # 2^-120 .. 2^-127: still normal fp32 for the top key


def test_constant_scores_count_exactly():
    c = CASES["constant21k"]
    for b, h, rows, kidx, live, s, sch in _groups(c, False):
        assert bool((sch.l_run == c.Lk).all())
        assert bool((sch.rescales_after_first() == 0).all())
        mean = c.v[b, :c.Lk, h * 128:(h + 1) * 128].mean(0)
        assert torch.allclose(sch.out, mean.expand_as(sch.out), rtol=0, atol=1e-12 * float(mean.abs().max()))


def test_rows_rescale_at_different_tiles():
    c = CASES["rows_differ"]
    for b, h, rows, kidx, live, s, sch in _groups(c, True):
        i = rows % 128
        want = torch.zeros_like(sch.grow)
        want[:, 0] = True
        for r, ii in enumerate(i.tolist()):
            for t in A.RESCALE_TILES[(ii // 64, (ii % 16) // 8)]:
                want[r, t] = True
        assert torch.equal(sch.grow, want)
        g = sch.grow[:128]
        pair = torch.arange(128).view(8, 2, 8)          # [warp pair 16-row block, h, g]
        assert bool((g[pair[:, 0]] != g[pair[:, 1]]).any(-1).all())     # g vs g + 8: different tiles
        assert bool((g[:64] != g[64:]).any(-1).all())                    # warpgroup 0 vs 1


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith("partial")])
def test_partial_tile_masked_column_dominates(name):
    c = CASES[name]
    rem, inside = c.intent["rem"], c.intent["inside"]
    assert c.Lk % 64 == rem and (c.R > c.Lk) == inside
    for f16 in (False, True):
        for b, h, rows, kidx, live, s, sch in _groups(c, f16):
            last = s[:, -1]
            assert last[:, ~live[-1]].amax(1).gt(last[:, live[-1]].amax(1)).all()
            if not inside:
                assert bool((last[:, live[-1]] < 0).all()) and bool((kidx[-1, ~live[-1]] >= c.R).all())
            assert bool(sch.grow[:, -1].all())           # the partial tile rescales


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith("windowed")])
def test_windowed_own_window_last(name):
    c = CASES[name]
    assert c.G % 64 in (1, 63)
    Tg = c.intent["glob_tiles"]
    for f16 in (False, True):
        for b, h, rows, kidx, live, s, sch in _groups(c, f16):
            assert sch.grow.shape[1] == Tg + 1
            assert bool(sch.grow[:, -1].all())           # the own window, processed last, rescales
            assert bool((kidx[-1] // 64 == rows[0] // 64).all())
            top = torch.where(live, s, torch.tensor(-math.inf)).amax((1, 2))
            assert s[:, Tg - 1, ~live[Tg - 1]].amax(1).gt(top).all()   # padding rows after the pooled keys dominate
            wg = int(rows[0] % 128) // 64
            other = (rows[0] // 128) * 128 + (1 - wg) * 64 + torch.arange(64)
            ko = c.k[b, other][:, h * 128 + rows % 128].t()  # the other warpgroup's tile, in these rows' directions
            assert bool((ko.amin(1) > top.double()).all())


@pytest.mark.parametrize("f16", (None, False, True))
@pytest.mark.parametrize("name", list(CASES))
def test_model_is_the_softmax(name, f16):
    """The model's o / l_run equals the float64 softmax within its own bar: the fp32 roundings of the exponent (the
    model takes the kernel's scale_log2 and fma in fp32) and, with P rounded, P's 16-bit rounding."""
    c = CASES[name]
    for b, h, rows, kidx, live, s, sch in _groups(c, f16):
        want = A.softmax_rows(c, b, h, rows, kidx, live)
        err = (sch.out - want).abs()
        assert bool((err <= sch.err + sch.rel[:, None] * sch.mag + 1e-12 * sch.mag).all())
