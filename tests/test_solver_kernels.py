"""The solver interpreter (tests/solver_emulator.py) against the oracles on the CPU, and the bound of Poisson's host
loop.

- Chained through whole solves (poisson_blend_batch / regionfill_batch with the interpreter as the library), the
  interpreter stops every LSQR system where oracle/poisson_oracle.py's `lsqr` stops, with the same istop and itn, and
  its iterate agrees within 1e-11; its sweeps give `PO.unfilled_mask` exactly; region fill agrees with
  oracle/regionfill_oracle.py's direct solve within 1e-9. Cases: the goldens and the edge batches below. On the
  driver's seven Poisson calls (pipeline_poisson) LSQR loses orthogonality and no two float64 evaluations stop at the
  same iteration everywhere: there the stop rule, the iteration within one and the blend within 5e-6 are checked.
- Every stopping branch the settings reach (measured with `PO.lsqr` on synth.poisson_inputs(seed=3, F=1, H=24, W=40,
  with_edge=True), channel 0): istop 0 (b = 0), 1 / 2 (defaults, and the goldens), 3 (conlim = 10), 4 (a consistent
  b = A x0 with atol = btol = conlim = 0), 5 (atol = btol = conlim = 0) and 7 (max_iters = 5). Istop 6 (the condition
  estimate beyond 1 / eps) is not reached by any system of these operators and is not forced.
- max_iters: with a library whose tolerance tests never fire, every slot of bb / aa / ww an iteration can touch (it
  reads slot k and, while its system runs, adds into slot k + 1) lies inside the arrays poisson_blend_batch allocates.
tests/test_solver_kernels_gpu.py replays the CUDA kernels against the same interpreter, launch by launch.
"""
import numpy as np
import pytest
import torch

from fgt_b200 import poisson as P
from fgt_b200 import regionfill as RF
from fgt_b200 import synth
from oracle import poisson_oracle as PO
from oracle import regionfill_oracle as RO
from tests.solver_emulator import SolverEmulator, emulating
from tests.util import load_golden

POISSON_GOLDENS = {"poisson_small": (3, 64, 96, 7, False), "poisson_edge": (2, 48, 64, 8, True),
                   "poisson_mid": (2, 120, 216, 9, False)}
REGIONFILL_GOLDENS = {"regionfill_small": (4, 48, 64, 5), "regionfill_mid": (3, 120, 216, 6)}
BRANCH_INPUT = dict(seed=3, F=1, H=24, W=40, with_edge=True)


# ------------------------------------------------------------------------------------------------------- inputs
def poisson_golden(name):
    F, H, W, seed, with_edge = POISSON_GOLDENS[name]
    inp = synth.poisson_inputs(seed=seed, F=F, H=H, W=W, with_edge=with_edge)
    return inp[0], inp[1], inp[2], inp[3], inp[4], (inp[5] if with_edge else None)


def pipeline_poisson():
    g = load_golden("pipeline_poisson")
    trg = g["trg"]
    F, H, W = trg.shape[:3]
    bits = lambda k: np.unpackbits(g[k])[:F * H * W].reshape(F, H, W).astype(bool)
    return trg, g["gx"], g["gy"], bits("hole"), bits("gmask"), None


def _grads(img):
    return img[:, :, 1:] - img[:, :, :-1], img[:, 1:] - img[:, :-1]


def poisson_edge_batch(H, W, masks, seed):
    """F = 5 frames of H x W: 0 ragged holes through every border and corner, with one-pixel holes; 1 a hole whose
    equations gmask removes entirely (with masks; a run of hole pixels without); 2 no hole; 3 channel 1 with b = 0
    while channels 0 and 2 run; 4 half of the border ring. masks: real gmask / edge arrays, or None (NULL)."""
    g = np.random.default_rng(seed)
    F = 5
    img = (g.integers(0, 256, (F, H, W, 3)) / 256.0).astype(np.float32)
    hole = g.random((F, H, W)) < 0.35
    hole[0, [0, 0, -1, -1], [0, -1, 0, -1]] = True
    hole[1] = False
    hole[1, H // 2, W // 2:] = True
    hole[2] = False
    ring = np.ones((H, W), bool)
    ring[1:-1, 1:-1] = False
    hole[4] = ring & (g.random((H, W)) < 0.5)
    img[3, ..., 1] = 0
    gx, gy = _grads(img)
    trg = img.copy()
    trg[hole] = 0
    if not masks:
        return trg, gx, gy, hole, None, None
    gm = (g.random((F, H, W)) < 0.15) & hole
    gm[1] = False
    ys, xs = np.nonzero(hole[1])
    gm[1, ys, xs] = True                       # owners of frame 1's equations: the pixel, its left and upper neighbours
    gm[1, ys, np.maximum(xs - 1, 0)] = True
    gm[1, np.maximum(ys - 1, 0), xs] = True
    edge = g.random((F, H, W)) < 0.1
    return trg, gx, gy, hole, gm, edge


def poisson_block_boundary(seed=21):
    """Two 24 x 40 frames whose holes hold 256 and 257 pixels, each owning equations: one and two blocks of 256."""
    g = np.random.default_rng(seed)
    H, W = 24, 40
    img = (g.integers(0, 256, (2, H, W, 3)) / 256.0).astype(np.float32)
    hole = np.zeros((2, H, W), bool)
    for f, n in ((0, 256), (1, 257)):
        hole[f].reshape(-1)[g.permutation(H * W)[:n]] = True
    gx, gy = _grads(img)
    trg = img.copy()
    trg[hole] = 0
    return trg, gx, gy, hole, None, None


def poisson_edge_cases():
    out = {}
    for H in (2, 3):
        for W in (2, 31, 32, 33, 65):
            for masks in (False, True):
                out[f"{H}x{W}_{'masks' if masks else 'null'}"] = lambda H=H, W=W, m=masks: poisson_edge_batch(
                    H, W, m, 100 * H + W)
    out["block_boundary"] = poisson_block_boundary
    return out


def consistent_input():
    """BRANCH_INPUT with the gradients and boundary values of one image on a 1/256 grid, so every right-hand side is
    exactly A x0 (x0 = the image inside the hole)."""
    trg, _, _, hole, gm, edge = synth.poisson_inputs(**BRANCH_INPUT)
    img = (np.random.default_rng(4).integers(0, 256, trg.shape) / 256.0).astype(np.float32)
    gx, gy = _grads(img)
    trg = img.copy()
    trg[hole] = 0
    return trg, gx, gy, hole, gm, edge


def zero_channel_input():
    trg, gx, gy, hole, gm, edge = synth.poisson_inputs(**BRANCH_INPUT)
    trg, gx, gy = trg.copy(), gx.copy(), gy.copy()
    trg[..., 1] = gx[..., 1] = gy[..., 1] = 0
    return trg, gx, gy, hole, gm, edge


# (inputs, poisson_blend_batch settings, istop and itn of channel 0 as PO.lsqr gives them)
BRANCHES = {
    "defaults": (lambda: synth.poisson_inputs(**BRANCH_INPUT), {}, (2, 49)),
    "conlim_10": (lambda: synth.poisson_inputs(**BRANCH_INPUT), dict(conlim=10.0), (3, 6)),
    "zero_tolerances": (lambda: synth.poisson_inputs(**BRANCH_INPUT), dict(atol=0.0, btol=0.0, conlim=0.0), (5, 84)),
    "consistent": (consistent_input, dict(atol=0.0, btol=0.0, conlim=0.0), (4, None)),
    "max_iters_5": (lambda: synth.poisson_inputs(**BRANCH_INPUT), dict(max_iters=5), (7, 5)),
}


def oracle_lsqr(trg, gx, gy, hole, gm, edge, atol=1e-6, btol=1e-6, conlim=1e8, max_iters=None):
    """PO.lsqr per frame and channel: (x [F,H,W,3], istop [F,3], itn [F,3])."""
    F, H, W = hole.shape
    x = np.zeros((F, H, W, 3))
    istop, itn = np.zeros((F, 3), int), np.zeros((F, 3), int)
    zero = np.zeros((H, W), bool)
    for f in range(F):
        code = PO.equation_codes(hole[f], zero if gm is None else gm[f], zero if edge is None else edge[f])
        b = PO.rhs(code, trg[f], np.asarray(gx[f], np.float64), np.asarray(gy[f], np.float64))
        for c in range(3):
            x[f, ..., c], istop[f, c], itn[f, c] = PO.lsqr(code, b[..., c], atol, btol, conlim,
                                                         None if max_iters is None else min(max_iters, 2 * H * W))
    return x, istop, itn


def emulate_poisson(monkeypatch, inputs, **kw):
    trg, gx, gy, hole, gm, edge = inputs
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a))
    with emulating(monkeypatch) as emu:
        out, unf, istop, itn = P.poisson_blend_batch(t(trg), t(gx), t(gy), t(hole), t(gm), t(edge), return_info=True,
                                                     **kw)
    return out.numpy(), unf.numpy(), istop.numpy(), itn.numpy(), emu


def check_poisson(monkeypatch, inputs, **kw):
    out, unf, istop, itn, emu = emulate_poisson(monkeypatch, inputs, **kw)
    trg, gx, gy, hole, gm, edge = inputs
    x, ois, oit = oracle_lsqr(*inputs, **kw)
    assert np.array_equal(istop, ois) and np.array_equal(itn, oit), (istop.tolist(), ois.tolist(), itn.tolist(),
                                                                      oit.tolist())
    assert np.abs(emu.x_final.reshape(x.shape) - x * hole[..., None]).max() < 1e-11
    want = np.where(hole[..., None], emu.x_final.reshape(x.shape).astype(np.float32).astype(np.float64), trg)
    assert np.array_equal(out, want)
    zero = np.zeros(hole.shape[1:], bool)
    assert np.array_equal(unf, np.stack([PO.unfilled_mask(hole[f], zero if gm is None else gm[f])
                                         for f in range(hole.shape[0])]))
    return istop, itn


# ---------------------------------------------------------------------------------------------------- Poisson
@pytest.mark.parametrize("name", ["poisson_small", "poisson_edge"])
def test_poisson_interpreter_equals_oracle_lsqr_on_goldens(name, monkeypatch):
    istop, itn = check_poisson(monkeypatch, poisson_golden(name))
    assert set(istop.reshape(-1).tolist()) <= {0, 1, 2} and itn.max() > 10


def test_poisson_interpreter_on_the_drivers_calls(monkeypatch):
    """On the driver's calls the bidiagonalisation loses orthogonality: two float64 evaluations of LSQR (PO.lsqr's
    normalised vectors, the header's unnormalised ones) agree on alfa and beta to 1e-16 for the first iterations and
    differ in the first digit after ~70, so their stops can lie an iteration apart. Here the same stop rule (istop)
    fires within one iteration, and the blends agree within 5e-6, the bar the GPU path meets against the reference."""
    inputs = pipeline_poisson()
    out, unf, istop, itn, emu = emulate_poisson(monkeypatch, inputs)
    trg, gx, gy, hole, gm, _ = inputs
    x, ois, oit = oracle_lsqr(*inputs)
    assert np.array_equal(istop, ois) and np.abs(itn - oit).max() <= 1
    blend = np.where(hole[..., None], x.astype(np.float32).astype(np.float64), trg)
    assert np.abs(out - blend).max() < 5e-6
    assert np.array_equal(unf, np.stack([PO.unfilled_mask(hole[f], gm[f]) for f in range(hole.shape[0])]))


@pytest.mark.parametrize("case", sorted(poisson_edge_cases()))
def test_poisson_interpreter_equals_oracle_lsqr_on_edge_batches(case, monkeypatch):
    inputs = poisson_edge_cases()[case]()
    istop, itn = check_poisson(monkeypatch, inputs)
    if case != "block_boundary":
        assert (istop[2] == 0).all() and (itn[2] == 0).all()                       # no hole: x = 0
        assert not case.endswith("masks") or ((istop[1] == 0).all() and (itn[1] == 0).all())   # no equations
        assert istop[3, 1] == 0 and itn[3, 1] == 0 and (itn[3, [0, 2]] > 0).all()


@pytest.mark.parametrize("branch", sorted(BRANCHES))
def test_poisson_interpreter_reaches_every_stopping_branch(branch, monkeypatch):
    make, kw, (want_istop, want_itn) = BRANCHES[branch]
    istop, itn = check_poisson(monkeypatch, make(), **kw)
    assert istop[0, 0] == want_istop and (want_itn is None or itn[0, 0] == want_itn), (istop, itn)


def test_poisson_interpreter_b_zero_on_one_channel(monkeypatch):
    istop, itn = check_poisson(monkeypatch, zero_channel_input())
    assert istop[0, 1] == 0 and itn[0, 1] == 0 and (istop[0, [0, 2]] == 2).all()


def test_poisson_sweeps_equal_the_oracle(monkeypatch):
    """fgt_poisson_unfilled's two sweeps as the interpreter states them, through getUnfilledMask's call, on ragged
    holes with and without gradient masks at widths around the 32-column words."""
    rng = np.random.default_rng(5)
    for H, W in ((1, 1), (5, 31), (6, 32), (7, 33), (9, 70)):
        hole = rng.random((H, W)) < 0.6
        gm = (rng.random((H, W)) < 0.3) & hole
        with emulating(monkeypatch):
            got = P.getUnfilledMask(hole, gm)
        assert np.array_equal(got, PO.unfilled_mask(hole, gm))


# ----------------------------------------------------------------------------------------------- max_iters bound
class _NeverConverges(SolverEmulator):
    """LSQR kernels whose tolerance tests never fire: a system stops only at the device-side limit k >= iter_lim the
    kernels test, with istop 7 and itn k. Records the highest slot of bb / aa / ww any iteration touches: iteration k
    reads slot k and, while its system runs, adds into slot k + 1."""

    top = -1

    def _lsqr_iteration(self, a):
        S = 3 * a["F"]
        kctr = self.arr(a["kctr"], "i32", 2)
        k = int(kctr[0])
        kctr[0], kctr[1] = k + 1, k
        state = self.arr(a["state"], "f64", 2 * S * 16).reshape(2, S, 16)
        running = k == 0 or state[(k + 1) & 1, 0, 12] == 0
        self.slots = min(self.flat(a[q], torch.float64).numel() for q in ("bb", "aa", "ww")) // S
        self.top = max(self.top, k + 1 if running else k)
        cur = state[(k + 1) & 1].copy() if k else np.zeros((S, 16))
        if running and k >= a["iter_lim"]:
            cur[:, 12], cur[:, 13], cur[:, 14] = 1, 7, k
        state[k & 1] = cur


@pytest.mark.parametrize("use_graph", [True, False])
def test_max_iters_keeps_every_iteration_inside_the_slot_arrays(use_graph, monkeypatch):
    trg, gx, gy, hole, gm, edge = synth.poisson_inputs(**BRANCH_INPUT)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    stub = _NeverConverges()
    monkeypatch.setattr(P, "_dev", lambda device=None: torch.device("cpu"))
    from tests.test_launch_trace import recording
    for M in (5, P.CHUNK, 3 * P.CHUNK + 1):
        stub.top = -1
        info = None
        with recording(stub):
            try:
                info = P.poisson_blend_batch(t(trg), t(gx), t(gy), t(hole), t(gm), t(edge), return_info=True,
                                             max_iters=M, use_graph=use_graph)
            except RuntimeError:
                pass
        assert stub.top < stub.slots, f"max_iters={M}: an iteration touches slot {stub.top} of {stub.slots}"
        assert info is not None and (info[2] == 7).all() and (info[3] == M).all()
    with pytest.raises(ValueError):
        P.poisson_blend_batch(t(trg), t(gx), t(gy), t(hole), max_iters=0)


# ------------------------------------------------------------------------------------------------- region fill
def regionfill_golden(name):
    B, H, W, seed = REGIONFILL_GOLDENS[name]
    return synth.regionfill_inputs(seed=seed, B=B, H=H, W=W)


def regionfill_edge_batches():
    """Batches of one shape each: 1-pixel-high and -wide images (one-pixel holes at both ends, runs of holes);
    40 x 64 images with one-pixel holes in the four corners, a hole across the 2048-pixel block boundary, boundary
    values all 0 (rr0 = 0), an empty mask, and a one-pixel hole next to a large hole (it keeps iterating long after it
    has converged)."""
    g = np.random.default_rng(40)
    out = {}
    for name, (H, W) in (("row", (1, 64)), ("column", (64, 1))):
        img = g.standard_normal((3, H, W)) * 4
        m = np.zeros((3, H, W), bool)
        m[0].reshape(-1)[[0, -1]] = True
        m[1].reshape(-1)[5:40] = True
        m[2].reshape(-1)[::3] = True
        out[name] = (img, m)
    H, W = 40, 64
    img = g.standard_normal((6, H, W)) * 4
    m = np.zeros((6, H, W), bool)
    m[0, [0, 0, -1, -1], [0, -1, 0, -1]] = True
    m[1, 30:34, 10:50] = True                  # pixels 1930 .. 2161: across 2048
    img[2] = 0
    m[2, 5:20, 5:30] = True
    m[4, 17, 23] = True
    m[5, 2:38, 3:60] = True
    out["2d"] = (img, m)
    return out


def emulate_regionfill(monkeypatch, img, mask):
    with emulating(monkeypatch):
        out, k = RF.regionfill_batch(torch.from_numpy(np.ascontiguousarray(img)),
                                     torch.from_numpy(np.ascontiguousarray(mask)), return_iters=True)
    return out.numpy(), k


@pytest.mark.parametrize("case", sorted(REGIONFILL_GOLDENS) + sorted(regionfill_edge_batches()))
def test_regionfill_interpreter_equals_the_direct_solve(case, monkeypatch):
    img, mask = regionfill_golden(case) if case in REGIONFILL_GOLDENS else regionfill_edge_batches()[case]
    out, k = emulate_regionfill(monkeypatch, img, mask)
    want = np.stack([RO.regionfill(img[b], mask[b]) for b in range(img.shape[0])])
    assert np.abs(out - want).max() < 1e-9, np.abs(out - want).max()
    assert np.array_equal(out[~mask], np.asarray(img, np.float64)[~mask]) and 0 < k
