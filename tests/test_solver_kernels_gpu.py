"""Launch-by-launch replay of the solver kernels on the H100: every launch of the entries in
tests/solver_emulator.SOLVER_ENTRIES issued by real poisson_blend_batch / regionfill_batch calls runs on the GPU and
then, on CPU copies of the buffers it referenced as they were before the launch, through the interpreter of
tests/solver_emulator.py (the Replayer of tests/test_kernel_replay_gpu.py with that interpreter). A graph launch has no
pointer arguments: it is resolved through the arguments its fgt_poisson_graph_create call was given. CHUNK is 1, so
each replayed iteration call is one iteration, both paths are replayed (CUDA graph and direct launches), and before
each launch the buffers the entry only writes are filled with 0xA5 bytes, so a store the interpreter does not make
cannot hide behind a zero or an earlier result.

Bars, per launch (the interpreter's docstring derives them): every byte the interpreter does not write unchanged (a
stopped system's vectors and sums, pixels outside the mask, slots of other iterations); codes, counts, the pixel list
(as a multiset per frame), u after set-up, kctr, clr, unf, both finish kernels, region fill's initial x and the stop /
istop / itn state slots exact; vector updates and atomically accumulated sums within their per-element rounding bars;
the other state slots within 1e-12 relative. A stop decision other than the interpreter's is accepted only where a
stop test lies within 1e-12 relative of its threshold; such cases are counted.

Cases: the Poisson goldens and the driver's seven calls, every launch; Poisson edge batches (W 2 / 31 / 32 / 33 / 65,
H 2 / 3, holes on every border and corner, one-pixel holes, a hole gmask strips of all equations, an empty frame, a
channel with b = 0 beside running ones, gmask / edge NULL and real; frames of 256 and 257 equation-owning pixels);
every stopping branch of tests/test_solver_kernels.py; region fill's goldens and edge batches (1-pixel-high and -wide
images, corner pixels, a hole across the 2048-pixel block, rr0 = 0, an empty mask, a one-pixel hole iterating for
hundreds of iterations after it converged beside a large one); and production sizes, where set-up, sweep, finish and
the first, a middle and the last iteration call are replayed and the others run as they are: diffusion() of 10 frames
of 240 x 432, a border ring at 240 x 432, Poisson at 240 x 432 with F = 10, and set-up / sweep / finish at 720 x 1280.

Observed on an H100 80GB HBM3 (700 W power limit), largest error over all replayed launches in units of the bar:
exact everywhere it is required (0 differing values: codes, u after set-up, list, cnt, kctr, clr, unf, both finish
kernels, region fill's initial x, stop / istop / itn slots); Poisson iterations v 0.53, x 0.51, w 0.23, u 0.18, aa 0.20,
ww 0.17, bb 0.051 (set-up bb 0.0028), other state slots 0.0019 of 1e-12 relative; region fill init r and p0 0.95 (one
rounding per added boundary value, met almost exactly), rr 0.26; iterations ap 0.51, x 0.50, p 0.50, r 0.29, pap 0.12,
rr 0.051. Stop decisions accepted near a threshold: 0. The file's 18 tests take 152 s, 42 s of them replaying every
iteration of poisson_mid in the extended-precision interpreter.

Each of these changes fails a test here while the Poisson and region-fill tests of tests/test_poisson.py and
tests/test_regionfill.py still pass: psn_finish_kernel storing x without the float32 rounding (5658 of 55296 stored
values differ on poisson_small); lap_dir_kernel's beta taken from rr[k-1] / rr[k-2] (p off by 2.6e15 x its bar on
regionfill_small); psn_ux_kernel ignoring skip_u (bytes of a stopped system's u change, b = 0 channel).
"""
import collections
import ctypes
import time

import numpy as np
import pytest
import torch

from fgt_b200 import lib, synth
from fgt_b200 import poisson as P
from fgt_b200 import regionfill as RF
from tests.solver_emulator import DONE, ITN, NEAR, SOLVER_ENTRIES, SolverEmulator
from tests.test_kernel_replay_gpu import Replayer, _bytes
from tests.test_solver_kernels import (BRANCHES, BRANCH_INPUT, REGIONFILL_GOLDENS, oracle_lsqr, pipeline_poisson,
                                       poisson_edge_cases, poisson_golden, regionfill_edge_batches, regionfill_golden,
                                       zero_channel_input)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
ITERS = ("fgt_poisson_iters", "fgt_poisson_graph_launch", "fgt_regionfill_iters")
WRITE_ONLY = {"fgt_poisson_setup": ("code", "u"), "fgt_poisson_unfilled": ("clr",),
              "fgt_poisson_finish": ("out", "unf"), "fgt_regionfill_init": ("x", "r", "p0"),
              "fgt_regionfill_iters": ("ap",), "fgt_regionfill_finish": ("out",)}


@pytest.fixture(autouse=True)
def _one_cpu_thread():
    """Each replayed launch copies and compares a handful of sub-megabyte CPU tensors, where intra-op threads cost
    several times what they save."""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


class SolverReplayer(Replayer):
    """`select(name, i)`: replay the i-th call of entry `name` (default: every call). `near` counts stop decisions that
    differ from the interpreter's, accepted because a stop test lay within NEAR of its threshold; `x_final` is the
    LSQR iterate the last replayed finish launch read."""

    emulator = SolverEmulator

    def __init__(self, *args, select=None, **kw):
        super().__init__(*args, **kw)
        self.graphs, self.near, self.select = {}, 0, select
        self.calls = collections.Counter()
        self.x_final = None

    def _fill(self, p):
        p = p.value if hasattr(p, "value") else p
        if p is not None:
            _bytes(self._find(p)[1]).fill_(0xA5)

    def _replay(self, name, f, args):
        i = self.calls[name]
        self.calls[name] += 1
        if name == "fgt_poisson_graph_create":
            rc = f(*args)
            self.graphs[args[-1]._obj.value] = list(args[:-1])
            return rc
        if name == "fgt_poisson_graph_destroy" or (self.select is not None and not self.select(name, i)):
            return f(*args)
        names = lib.PROTOS[name].names
        a = dict(zip(names, args))
        if name == "fgt_poisson_graph_launch":
            h = a["exec"].value if isinstance(a["exec"], ctypes.c_void_p) else a["exec"]
            iargs = self.graphs[h] + [a["stream"]]
            assert iargs[lib.PROTOS["fgt_poisson_iters"].names.index("iters")] == 1, "replay one iteration per graph"
            run = lambda *_: f(*args)
            run.argtypes = lib.PROTOS["fgt_poisson_iters"].argtypes
            rc = super()._replay("fgt_poisson_iters", run, iargs)
            self.launches["fgt_poisson_iters"] -= 1
            self.launches[name] += 1
            return rc
        if name in ITERS:
            assert a["iters"] == 1, "replay one iteration per call"
        for k in WRITE_ONLY.get(name, ()):
            self._fill(a[k])
        if name == "fgt_regionfill_iters":
            self._fill(a["p1"] if a["k0"] % 2 == 0 else a["p0"])
        return super()._replay(name, f, args)

    @staticmethod
    def _check_untouched(name, emu, before, after, work):
        """Replayer._check_untouched with the written bytes of all storages marked in one pass over the records."""
        masks = {w.untyped_storage().data_ptr(): (b, torch.zeros(w.numel(), dtype=torch.bool)) for b, w in work.items()}
        for _, fl, idx, _, _ in emu.records:
            _, m = masks[fl.untyped_storage().data_ptr()]
            es = fl.element_size()
            m[((fl.storage_offset() + idx)[:, None] * es + torch.arange(es)).reshape(-1)] = True
        for b, m in masks.values():
            assert not bool(((after[b] != before[b]) & ~m).any()), f"{name}: bytes outside its outputs changed"

    def _compare(self, name, cargs, emu, before, after, work):
        key = {w.untyped_storage().data_ptr(): b for b, w in work.items()}

        def got_of(fl, idx):
            b = key[fl.untyped_storage().data_ptr()]
            g = torch.empty(0, dtype=fl.dtype).set_(after[b].untyped_storage(), fl.storage_offset(), fl.shape, (1,))
            return g[idx].numpy()

        stop = [DONE, DONE + 1, ITN]
        differ = {int(sys[0]) for _, kind, fl, idx, want, _, sys in emu.checks
                  if kind == "state" and not np.array_equal(got_of(fl, idx)[stop], want[stop])}
        near = {s for s, _ in emu.near}
        assert differ <= near, f"{name}: stop decisions of systems {sorted(differ - near)} differ from the interpreter"
        self.near += len(differ)                   # accepted: a stop test within NEAR of its threshold
        if not differ:
            self._check_untouched(name, emu, before, after, work)
        near = differ
        if name == "fgt_poisson_finish":
            self.x_final = emu.x_final
        a = dict(zip(lib.PROTOS[name].names, cargs))
        for label, kind, fl, idx, want, bar, sys in emu.checks:
            got = got_of(fl, idx)
            if got.size == 0:
                continue
            keep = np.ones(got.size, bool) if sys is None or not near else ~np.isin(sys, list(near))
            if kind == "exact":
                w = want.astype(got.dtype)
                same = (got.view(np.uint8).reshape(got.size, -1) == w.view(np.uint8).reshape(w.size, -1)).all(1)
                bad = int((~same)[keep].sum())
                err = float(bad)
                assert bad == 0, f"{name} {label}: {bad} of {got.size} values differ from the interpreter"
            elif kind == "multiset":
                n = a["H"] * a["W"]
                fr = idx.numpy() // n
                err = 0.0
                for f in np.unique(fr):
                    assert np.array_equal(np.sort(got[fr == f]), np.sort(want[fr == f])), f"{name} {label}: frame {f}"
            elif kind == "state":
                exact = np.zeros(16, bool)
                exact[[DONE, DONE + 1, ITN]] = True
                d = np.abs(got - want)
                assert np.array_equal(got[exact], want[exact]) or not keep.all(), f"{name}: stop slots {got[exact]}"
                rel = np.where(want != 0, d / np.abs(np.where(want != 0, want, 1)), np.where(d == 0, 0.0, np.inf))
                err = float(rel[~exact].max() / NEAR) if keep.all() else 0.0
                assert err <= 1.0, f"{name} state: {err:.3g} x 1e-12 relative"
            else:
                d = np.abs(got.astype(np.longdouble) - want)[keep]
                bb = bar[keep]
                r = np.where(bb > 0, d / np.where(bb > 0, bb, 1), np.where(d == 0, 0.0, np.inf)).astype(np.float64)
                err = float(r.max()) if r.size else 0.0
                assert np.isfinite(got[keep]).all(), f"{name} {label}: non-finite value"
                assert err <= 1.0, f"{name} {label}: error {err:.3g} x its bar"
            self.maxima[(name, label)] = max(self.maxima[(name, label)], err)


class replaying:
    def __init__(self, select=None):
        self.select = select

    def __enter__(self):
        self.saved = lib.load()
        self.rep = SolverReplayer(self.saved, SOLVER_ENTRIES, device_type=DEV.type, select=self.select)
        lib._lib = self.rep
        return self.rep

    def __exit__(self, *exc):
        lib._lib = self.saved
        self.rep._st.clear()
        return False


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _done(rep, what):
    rep.report(what)
    print(f"[{what}] stop decisions accepted near a threshold: {rep.near}")
    assert rep.near == 0


def _poisson(inputs, use_graph=True, select=None, **kw):
    trg, gx, gy, hole, gm, edge = inputs
    with replaying(select) as r:
        out = P.poisson_blend_batch(_t(trg), _t(gx), _t(gy), _t(hole), _t(gm), _t(edge), return_info=True,
                                    use_graph=use_graph, **kw)
    return r, [o.cpu().numpy() for o in out]


def _every_launch(monkeypatch, inputs, what, use_graph=True, **kw):
    monkeypatch.setattr(P, "CHUNK", 1)
    r, (out, unf, istop, itn) = _poisson(inputs, use_graph, **kw)
    _done(r, what)
    its = r.launches["fgt_poisson_graph_launch" if use_graph else "fgt_poisson_iters"]
    assert r.launches["fgt_poisson_setup"] == 1 and r.launches["fgt_poisson_finish"] == 1 and its == itn.max() + 1
    return out, istop, itn, r


# ---------------------------------------------------------------------------------------------------------- Poisson
@pytest.mark.parametrize("name", ["poisson_small", "poisson_edge", "poisson_mid", "pipeline_poisson"])
def test_replay_poisson_goldens(name, monkeypatch):
    inputs = pipeline_poisson() if name == "pipeline_poisson" else poisson_golden(name)
    _every_launch(monkeypatch, inputs, name, use_graph=name != "poisson_edge")


def test_replay_poisson_edge_batches(monkeypatch):
    for case, make in sorted(poisson_edge_cases().items()):
        inputs = make()
        out, istop, itn, _ = _every_launch(monkeypatch, inputs, case, use_graph=case.endswith("null"))
        _, ois, oit = oracle_lsqr(*inputs)
        assert np.array_equal(istop, ois) and np.array_equal(itn, oit), case


@pytest.mark.parametrize("branch", sorted(BRANCHES) + ["b_zero_channel"])
def test_replay_poisson_stopping_branches(branch, monkeypatch):
    if branch == "b_zero_channel":
        make, kw, want = zero_channel_input, {}, None
    else:
        make, kw, want = BRANCHES[branch]
    inputs = make()
    out, istop, itn, r = _every_launch(monkeypatch, inputs, branch, **kw)
    x, ois, oit = oracle_lsqr(*inputs, **kw)
    assert np.array_equal(istop, ois) and np.array_equal(itn, oit), (istop, ois, itn, oit)
    if want is None:
        assert istop[0, 1] == 0 and itn[0, 1] == 0
    else:
        assert istop[0, 0] == want[0] and (want[1] is None or itn[0, 0] == want[1])
    assert np.abs(r.x_final.reshape(x.shape) - x * inputs[3][..., None]).max() < 1e-11


def test_max_iters_stops_every_system_with_istop_7(monkeypatch):
    """max_iters = 5, inside the first chunk of 48 iterations: every system stops at iteration 5 with istop 7 and the
    iterate of PO.lsqr(iter_lim=5), on both paths with CHUNK as shipped (set-up, sweep and finish replayed)."""
    inputs = synth.poisson_inputs(**BRANCH_INPUT)
    x, _, _ = oracle_lsqr(*inputs, max_iters=5)
    for use_graph in (True, False):
        r, (out, unf, istop, itn) = _poisson(inputs, use_graph, select=lambda name, i: name not in ITERS, max_iters=5)
        assert (istop == 7).all() and (itn == 5).all()
        assert np.abs(r.x_final.reshape(x.shape) - x * inputs[3][..., None]).max() < 1e-11
        _done(r, f"max_iters=5 graph={use_graph}")


# ------------------------------------------------------------------------------------------------------ region fill
def _regionfill(img, mask, select=None):
    with replaying(select) as r:
        out, k = RF.regionfill_batch(_t(img), _t(mask), return_iters=True)
    return r, out.cpu().numpy(), k


@pytest.mark.parametrize("case", sorted(REGIONFILL_GOLDENS) + sorted(regionfill_edge_batches()))
def test_replay_regionfill(case, monkeypatch):
    monkeypatch.setattr(RF, "CHUNK", 1)
    img, mask = regionfill_golden(case) if case in REGIONFILL_GOLDENS else regionfill_edge_batches()[case]
    r, out, k = _regionfill(img, mask)
    _done(r, case)
    assert r.launches["fgt_regionfill_iters"] == k and np.isfinite(out).all()
    if case == "2d":
        assert k >= 200, "the one-pixel hole iterates for hundreds of iterations after converging"


# -------------------------------------------------------------------------------------------------- production sizes
def _first_middle_last(run):
    """Runs `run(select)` once unreplayed to count its iteration calls K, then replays every other launch and the
    iteration calls 0, K // 2 and K - 1."""
    counter = {}

    def none(name, i):
        counter[name] = i + 1
        return False

    run(none)
    pick = {n: {0, c // 2, c - 1} for n, c in counter.items() if n in ITERS}
    return run(lambda name, i: name not in ITERS or i in pick.get(name, ()))


def test_replay_production_sizes(monkeypatch):
    monkeypatch.setattr(P, "CHUNK", 1)
    monkeypatch.setattr(RF, "CHUNK", 1)
    t0 = time.time()
    H, W = 240, 432
    img, mask = synth.regionfill_inputs(seed=50, B=10, H=H, W=W)
    flows = np.stack([img, img[:, ::-1] * 0.5], -1)

    def diffusion(select):
        with replaying(select) as r:
            RF.diffusion(flows, mask[..., None])
        return r

    r = _first_middle_last(diffusion)
    _done(r, "diffusion 10 x 240 x 432")
    assert r.launches["fgt_regionfill_iters"] >= 3 and r.launches["fgt_regionfill_init"] == 1
    ring = np.ones((2, H, W), bool)
    ring[:, 12:-12, 16:-16] = False
    r = _first_middle_last(lambda s: _regionfill(img[:2], ring, s)[0])
    _done(r, "border ring 240 x 432")
    inputs = synth.poisson_inputs(seed=13, F=10, H=H, W=W) + (None,)
    r = _first_middle_last(lambda s: _poisson(inputs, True, s)[0])
    _done(r, "poisson 10 x 240 x 432")
    assert r.launches["fgt_poisson_graph_launch"] >= 3 and r.launches["fgt_poisson_setup"] == 1
    monkeypatch.setattr(P, "CHUNK", 48)
    big = synth.poisson_inputs(seed=14, F=1, H=720, W=1280) + (None,)
    r, _ = _poisson(big, True, lambda name, i: name not in ITERS)
    _done(r, "poisson 720 x 1280 set-up / sweep / finish")
    assert r.launches["fgt_poisson_setup"] == 1 and r.launches["fgt_poisson_unfilled"] == 1
    print(f"[production] {time.time() - t0:.1f} s")
