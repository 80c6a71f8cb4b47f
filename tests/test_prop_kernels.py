"""The flow-propagation interpreter (tests/prop_emulator.py) against the oracle and cv2.remap, on the CPU.

- Chained through propagation.propagate's launch sequence, the interpreter reproduces oracle/prop_oracle.py bit for bit
  (mask_tofill and both gradients) on the three golden clips and on the edge clips below.
- remap (the interpreter's and the oracle's) picks cv2.remap's taps and weights at the coordinates where its 1/32-pixel
  quantisation decides: odd multiples of 1/64, one fp32 ulp either side of them, (-1, 0) and [W - 1, W).
- The edge clips are built pixel by pixel so that every decision of fgt_prop_step and fgt_prop_fuse is taken both ways:
  half-integer neighbour positions for even and odd k and -0.5, the round trip at diff == thres (3-4-5) and just below,
  neighbours on rows and columns H - 2 / H - 1 / W - 2 / W - 1 and -1, case-2 chains over five frames (one rejected at
  row H - 1), NaN and +-inf flows, and fusion with one and two candidates, subnormal confidences and den == 0. The
  designed pixels' outcomes are asserted one by one, and the interpreter's decision counts on both sides.
tests/test_prop_kernels_gpu.py replays the CUDA kernels against the same interpreter on the same clips.
"""
import numpy as np
import pytest

from fgt_b200 import synth
from oracle import prop_oracle as PO
from tests.prop_emulator import emulate, remap
from tests.util import load_golden

GOLDEN_CLIPS = ["prop_small", "prop_thres1", "prop_mid"]
F32 = np.float32
ULP = float(np.spacing(F32(2.5)))   # fp32 ulp in [2, 4)


def golden_inputs(name):
    meta = load_golden(name)["meta"]
    return synth.prop_inputs(seed=meta["seed"], H=meta["H"], W=meta["W"], N=meta["N"]), meta["thres"], 0.1


# ------------------------------------------------------------------------------------------------------- edge clips
class _Clip:
    """A clip assembled pixel by pixel. `link` makes (t, y, x) a hole whose slot-`slot` step flow lands on (ny, nx) and
    sets the back flow on every tap the round trip reads with a nonzero weight to `-(u, v) + res`, so the round-trip
    residual is `res` where the arithmetic is exact. A flow cell is set once: a second, different value raises, so the
    designed pixels cannot disturb one another. Unset flows are 0; every other pixel is known."""

    def __init__(self, H, W, N, seed):
        self.H, self.W, self.N = H, W, N
        self.mask = np.zeros((H, W, N), dtype=bool)
        self.ff = np.zeros((H, W, 2, N - 1), dtype=F32)
        self.fb = np.zeros((H, W, 2, N - 1), dtype=F32)
        self.set_cells = {}
        self.seed = seed
        self.expect = []   # (slot, t, y, x, have expected, nn_y expected or None)

    def _set(self, name, k, y, x, uv):
        uv = tuple(F32(c) for c in uv)
        key = (name, k, y, x)
        old = self.set_cells.get(key)
        assert old is None or all(a.tobytes() == b.tobytes() for a, b in zip(old, uv)), f"flow cell {key} set twice"
        self.set_cells[key] = uv
        getattr(self, name)[y, x, :, k] = uv

    def link(self, slot, t, y, x, ny, nx, res=(0.0, 0.0), back=None, have=None, nn_y=None):
        ny, nx = F32(ny), F32(nx)
        u, v = F32(nx - F32(x)), F32(ny - F32(y))
        assert np.array_equal([F32(F32(x) + u), F32(F32(y) + v)], [nx, ny], equal_nan=True), "target not exact"
        self.mask[y, x, t] = True
        step, bk, k = ("fb", "ff", t - 1) if slot == 0 else ("ff", "fb", t)
        self._set(step, k, y, x, (u, v))
        if back is None:
            back = (F32(-u) + F32(res[0]), F32(-v) + F32(res[1]))
        if np.isfinite(nx) and np.isfinite(ny):
            sx, sy = int(np.rint(nx * F32(32))), int(np.rint(ny * F32(32)))
            for yy, wy in ((sy >> 5, 32 - (sy & 31)), ((sy >> 5) + 1, sy & 31)):
                for xx, wx in ((sx >> 5, 32 - (sx & 31)), ((sx >> 5) + 1, sx & 31)):
                    if wy and wx and 0 <= yy < self.H and 0 <= xx < self.W:
                        self._set(bk, k, yy, xx, back)
        if have is not None:
            self.expect.append((slot, t, y, x, have, nn_y))

    def inputs(self):
        g = np.random.default_rng(self.seed)
        gx = g.standard_normal((self.H, self.W, 3, self.N)).astype(F32)
        gy = g.standard_normal((self.H, self.W, 3, self.N)).astype(F32)
        for t in range(self.N):
            gx[self.mask[:, :, t], :, t] = 0
            gy[self.mask[:, :, t], :, t] = 0
        return gx, gy, self.mask.copy(), self.ff.copy(), self.fb.copy()


def _decisions_clip():
    """Slot-0 probes from frame 1 into frame 0 (whose holes never have a slot-0 neighbour), NaN / inf probes from frame
    2 into frame 1, and two chains through frames 1-5."""
    H, W, N = 10, 12, 6
    c = _Clip(H, W, N, seed=11)
    hole0 = c.mask[:, :, 0]
    # half-integer rows and columns, half to even: the other candidate cell is a hole without a neighbour
    c.link(0, 1, 5, 0, 2.5, 0, have=1, nn_y=2.5); hole0[3, 0] = True           # 2.5 -> 2
    c.link(0, 1, 6, 1, 3.5, 1, have=1, nn_y=3.5); hole0[3, 1] = True           # 3.5 -> 4 (truncation gives 3)
    c.link(0, 1, 7, 2, 7, 4.5, have=1); hole0[7, 5] = True                     # 4.5 -> 4
    c.link(0, 1, 8, 3, 8, 5.5, have=1); hole0[8, 5] = True                     # 5.5 -> 6
    c.link(0, 1, 2, 4, -0.5, 4, have=1, nn_y=-0.5)                             # -0.5 -> -0: row 0, in bounds
    c.link(0, 1, 6, 5, 6, -0.5, have=1)                                        # column -0.5 -> -0
    c.link(0, 1, 0, 7, np.nextafter(F32(-0.5), F32(-1)), 7, have=0)          # one ulp below -0.5 -> -1: outside
    c.link(0, 1, 2, 7, 2.5 + ULP, 7, have=1); hole0[2, 7] = True               # one ulp above the tie -> 3
    c.link(0, 1, 3, 8, 3.5 - ULP, 8, have=1); hole0[4, 8] = True               # one ulp below the tie -> 3
    # bounds: rows and columns H - 2 / H - 1 / W - 2 / W - 1 and -1 (each cell known, each round trip exact)
    c.link(0, 1, 5, 9, H - 1, 9, have=0)
    c.link(0, 1, 4, 10, H - 2, 10, have=1)
    c.link(0, 1, 1, 2, 1, W - 1, have=0)
    c.link(0, 1, 0, 6, 0, W - 2, have=1)
    c.link(0, 1, 1, 9, -1, 9, have=0)
    c.link(0, 1, 4, 1, 4, -1, have=0)
    # the round-trip test: diff == thres (3-4-5) fails, one fp32 ulp below it passes
    c.link(0, 1, 8, 8, 8, 8, res=(3, 4), have=0)
    c.link(0, 1, 3, 3, 3, 3, res=(-3, -4), have=0)
    c.link(0, 1, 0, 1, 0, 1, res=(3, np.nextafter(F32(4), F32(0))), have=1)
    c.link(0, 1, 1, 0, 1, 0, res=(0.5, -0.25), have=1)
    # non-finite flows and round trips write nothing (frame 2 -> frame 1, target cells known)
    c.link(0, 2, 1, 1, 1, np.nan, have=0)
    c.link(0, 2, 2, 2, np.inf, 2, have=0)
    c.link(0, 2, 3, 3, 3, -np.inf, have=0)
    c.link(0, 2, 4, 4, 4, 4, back=(np.nan, 0.0), have=0)
    c.link(0, 2, 5, 5, 5, 5, back=(0.0, np.inf), have=0)
    # chain A, row 5, column W - 2, frames 1-5: case 1 then case 2 four times, residue +0.25 a frame (5.5 -> 6 at
    # frame 2); the chained residual is the larger at frame 2, the pixel's own at frame 3
    for t, res in zip(range(1, 6), ((0.5, 0), (0.25, 0), (1.0, 0), (0.0, 0.5), (0.125, 0.25))):
        c.link(0, t, 5, W - 2, 5.25, W - 2, res=res, have=1, nn_y=5 + 0.25 * t)
    # chain B, row H - 2, column 0, frames 2-5: 8.25, 8.5 (-> 8, kept), 8.75 (-> 9 = H - 1, rejected), then the
    # next frame finds a hole without a neighbour
    for t, have, ny in ((2, 1, 8.25), (3, 1, 8.5), (4, 0, None), (5, 0, None)):
        c.link(0, t, H - 2, 0, H - 2 + 0.25, 0, have=have, nn_y=ny)
    return c


def _fuse_clip():
    """Frame 2 pixels with identity flows in both slots (frames 1 and 3 known there) and chosen residuals (r0, r1),
    so with alpha = 1e-3 the confidences exp(-1000 r) are normal, subnormal (r in (0.7084, 0.7444)) or 0."""
    H, W, N = 6, 8, 4
    c = _Clip(H, W, N, seed=12)
    pairs = [(0.0, 0.5), (0.25, 0.0), (0.71875, 0.7265625), (0.75, 0.8125), (0.71875, 0.75), (0.25, 0.75),
             (0.5, None), (0.71875, None), (None, 0.75), (0.0, 0.0)]
    for i, (r0, r1) in enumerate(pairs):
        y, x = 1 + i // 5, 1 + i % 5
        for slot, r in ((0, r0), (1, r1)):
            if r is None:
                c.link(slot, 2, y, x, y, np.nan, have=0)
            else:
                c.link(slot, 2, y, x, y, x, res=(r, 0.0), have=1)
    return c


def edge_clips():
    """[(name, inputs, thres, alpha)]: the decisions clip at the driver's settings and the fusion clip at alpha 0.1
    and 1e-3."""
    d, f = _decisions_clip(), _fuse_clip()
    return [("decisions", d.inputs(), 5.0, 0.1), ("fuse_alpha0.1", f.inputs(), 5.0, 0.1),
            ("fuse_alpha1e-3", f.inputs(), 5.0, 1e-3)]


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _vs_oracle(inputs, thres, alpha):
    gx, gy, mask, ff, fb = inputs
    states = []
    ex, ey, em, emu = emulate(gx, gy, mask, ff, fb, thres, alpha, states)
    with np.errstate(invalid="ignore", over="ignore"):
        ox, oy, om = PO.get_flownn_gradient(gx, gy, mask, ff, fb, thres, alpha)
    assert np.array_equal(em, om), "mask_tofill differs from the oracle"
    assert _bits_equal(ex, ox) and _bits_equal(ey, oy), "gradients differ from the oracle"
    N = mask.shape[2]
    assert len(emu.records) == 5 * 2 * (N - 1) + 2 * 2 * N + 3   # the launch sequence's stores
    return emu, states


@pytest.mark.parametrize("name", GOLDEN_CLIPS)
def test_chained_interpreter_equals_oracle_golden_clips(name):
    inputs, thres, alpha = golden_inputs(name)
    emu, _ = _vs_oracle(inputs, thres, alpha)
    assert emu.counts["step_case1"] > 0 and emu.counts["step_case2"] > 0


@pytest.mark.parametrize("case", range(3))
def test_chained_interpreter_equals_oracle_edge_clips(case):
    name, inputs, thres, alpha = edge_clips()[case]
    _vs_oracle(inputs, thres, alpha)


def _check_expectations(clip, states):
    for slot, t, y, x, have, nn_y in clip.expect:
        s = states[slot]
        got = int(s["have"][t, y, x])
        assert got == have, f"slot {slot} frame {t} ({y}, {x}): have {got}, expected {have}"
        if nn_y is not None:
            assert float(s["ny"][t, y, x]) == nn_y, f"slot {slot} frame {t} ({y}, {x}): nn_y {float(s['ny'][t, y, x])}"


def test_edge_clip_decisions_both_ways():
    """Every designed pixel's outcome, and each decision of fgt_prop_step taken both ways (counts over both passes)."""
    c = _decisions_clip()
    emu, states = _vs_oracle(c.inputs(), 5.0, 0.1)
    _check_expectations(c, states)
    k = emu.counts
    print("\n[decisions clip]", dict(sorted(k.items())))
    both_ways = [("step_consistent", "step_inconsistent"), ("step_diff_below_thres_by_under_1e-6",
                                                            "step_diff_eq_thres"),
                 ("step_case1", "step_hole_without_neighbour"), ("step_case2", "step_case2_out_of_bounds"),
                 ("step_case2_own_residual_larger", "step_case2_chained_residual_larger"),
                 ("step_tie_y_to_even_below", "step_tie_y_to_even_above"),
                 ("step_tie_x_to_even_below", "step_tie_x_to_even_above")]
    for a, b in both_ways:
        assert k[a] > 0 and k[b] > 0, (a, k[a], b, k[b])
    for key in ("step_nonfinite_position", "step_consistent_out_of_bounds", "step_consistent_row_8",
                "step_consistent_row_9", "step_consistent_col_10", "step_consistent_col_11",
                "step_consistent_row_negative", "step_consistent_col_negative", "step_case2_out_of_bounds_at_last_row"):
        assert k[key] > 0, key
    # chain A ends five frames from its source, in frame 0; chain B's accepted link keeps the source frame too
    assert int(states[0]["nt"][5, 5, 10]) == 0 and int(states[0]["nt"][3, 8, 0]) == 1
    assert float(states[0]["cuv"][2, 5, 10, 0]) == 0.5 and float(states[0]["cuv"][3, 5, 10, 0]) == 1.0


def test_fuse_clip_candidates_and_underflow():
    """One and two candidates, subnormal confidences (both, and beside a zero one), den == 0 with equal weights."""
    c = _fuse_clip()
    emu, states = _vs_oracle(c.inputs(), 5.0, 1e-3)
    _check_expectations(c, states)
    k = emu.counts
    print("\n[fuse clip, alpha 1e-3]", dict(sorted(k.items())))
    for key in ("fuse_one_candidate", "fuse_two_candidates", "fuse_den_zero", "fuse_subnormal_confidence",
                "fuse_two_candidates_both_subnormal"):
        assert k[key] > 0, key
    # den == 0: the two candidates' mean, exactly
    f = emu.fuse
    assert (f["exact"] & (f["cmin"] == 0)).any()


# ------------------------------------------------------------------------------------------------ remap tie choice
def _coords(W):
    """Odd multiples of 1/64 in [-1, W), one fp32 ulp either side, and points in (-1, 0) and [W - 1, W)."""
    ties = (np.arange(-64, 64 * W, 2) + 1).astype(F32) / F32(64)
    up, down = np.nextafter(ties, F32(np.inf)), np.nextafter(ties, F32(-np.inf))
    neg = np.array([-0.999, -0.75, -0.5, -0.3, -0.015625, -1e-7, -0.0], F32)
    last = np.array([W - 1, W - 1 + 1e-6, W - 0.75, W - 0.5, W - 0.0078125, np.nextafter(F32(W), F32(0))], F32)
    return np.concatenate([ties, up, down, neg, last]).astype(F32)


def _weights(fn, H, W, x, y):
    """[K, H*W]: the weight each coordinate gives every pixel, read through one-hot images."""
    out = np.zeros((x.size, H * W), F32)
    for j in range(H * W):
        img = np.zeros((H, W), F32)
        img.flat[j] = 1
        out[:, j] = fn(img, x, y).reshape(-1)
    return out


def test_remap_taps_and_weights_match_cv2():
    cv2 = pytest.importorskip("cv2")
    H, W = 5, 6
    c = _coords(max(H, W))
    mid = np.full_like(c, F32(2.3))
    for x, y in ((c, mid), (mid, c), (c, c[::-1].copy())):
        ref = _weights(lambda img, x, y: cv2.remap(img, x[None], y[None], cv2.INTER_LINEAR), H, W, x, y)
        for fn in (PO.remap_q32, remap):
            got = _weights(fn, H, W, x, y)
            bad = np.nonzero((got != ref).any(1))[0]
            assert bad.size == 0, f"{fn.__module__}: taps or weights differ at x={x[bad[:3]]}, y={y[bad[:3]]}"
        # a ramp decodes the quantised coordinate: value = rint(32 x) / 32 + 1 where both taps are in range
        ramp = np.tile(np.arange(W, dtype=F32) + 1, (H, 1))
        sx = np.rint(x * F32(32)) / 32
        ok = (sx >= -1) & (sx <= W - 1) & (np.rint(y * F32(32)) / 32 >= 0) & (np.rint(y * F32(32)) / 32 <= H - 1)
        got = remap(ramp, x, y)
        assert np.array_equal(got[ok], (sx + 1).astype(F32)[ok])
        assert np.array_equal(got, cv2.remap(ramp, x[None], y[None], cv2.INTER_LINEAR)[0])


def test_remap_ties_round_half_to_even():
    """x = k + 1/64 (32x = 32k + 0.5) keeps fraction 0 for even 32k; 32k + 1.5 rounds up to fraction 2/32."""
    img = np.tile(np.arange(8, dtype=F32) + 1, (3, 1))
    x = np.array([2 + 1 / 64, 2 + 3 / 64, -1 / 64, -3 / 64], F32)
    for fn in (remap, PO.remap_q32):
        got = fn(img, x, np.ones_like(x))
        assert np.array_equal(got, np.array([3.0, 3 + 2 / 32, 1.0, 30 / 32], F32))
