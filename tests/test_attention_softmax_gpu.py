"""fgt_attention on the designed cases of tests/attention_cases.py, in the split-bf16 and the fp16 build, replayed
against the float64 interpreter of tests/kernel_emulator.py (the Replayer of tests/test_kernel_replay_gpu.py): every
byte the interpreter does not write, the sentinel-filled output rows no query maps to included, must be unchanged, and
every written element must lie within its own bar.

The bar of output element (row r, column c). The operands are exact in both formats and every score is a single exact
product, so the error comes from the schedule's arithmetic alone. With P_k the weights of the documented schedule
(tests/attention_cases.schedule, in the frame of the row's reference maximum) and l = sum P_k:
- exponent: ex2.approx is within 2^-22 of 2^t, and t carries the fp32 roundings of scale_log2, of the fma, of m_tile and
  of each rescale's m_ref - m_tile, each at most 2^-24 |operand| with operands bounded by the key's distance below the
  final reference maximum plus 16: eps_k = 2^-21 + 2^-22 (m_final - x_k + 16) relative, on P_k;
- P's 16-bit form: |P16_k - P_k| exactly as the model rounds it (split-bf16 hi + lo of the fp32 P; fp16 to nearest,
  saturating). Taking the model's rounding rather than a 2^-11 bound keeps the bar tight where P16 is exact (every P a
  power of 2 at EXACT_SCALE), so a P that overflows fp16's range cannot hide in the bar;
- accumulation: each wgmma k-step and each rescale adds at most 17 addends into an fp32 accumulator, truncated at 2^-23
  of the largest: at most 2^-19 of sum P |V| per step, over steps = tiles * (4 * terms + 1) + 20 (terms 3 split, 1 fp16;
  the 20 cover l_run's per-thread and quad sums);
- the division by l_run, whose error (sum P eps / l plus the steps) scales sum P |V| / l;
- the output's own rounding: split-bf16 hi + lo within 2^-16 |o|; fp16 half an ulp of |o| plus 2^-22 |o|.
bar = [sum_k (P_k eps_k + |P16_k - P_k|) |V_kc| + (sum_k P_k eps_k + steps 2^-19) sum_k P_k |V_kc|] / l + rounding.
The kernel's own rule decides the rescales here, and the model reproduces it exactly on exact scores, so a bar built
from the model's weights is the bar of the kernel's arithmetic.

The contract for key rows the kernel reads but masks (dense [Lk, Lk_rows), windowed the padding after the pooled keys
in their last tile): K there may hold anything, NaN and Inf included, and the output is bit-identical to finite keys;
V there must be finite, since the masked key's P = 0 multiplies it and a NaN there is a NaN in every output row of the
batch (include/fgt_b200.h, `Lk_rows`).

test_rescale_census_at_production_geometry reports, without a bar, how often the lazy rescale runs on real activations:
the schedule model on the pre-launch operands of every attention launch of FGT's 432 x 240, T = 10 forward.
"""
import collections
import contextlib
import math

import pytest
import torch

from fgt_b200 import lib
from tests import attention_cases as A
from tests.kernel_emulator import KernelEmulator
from tests.test_kernel_replay_gpu import DEV, Replayer, _fgt, _ulp16

pytestmark = pytest.mark.gpu

CASES = {c.name: c for c in A.all_cases()}
SENTINEL = -1234.5


def _enc(x, f16):
    return x.half().contiguous() if f16 else lib.to_split(x.float())


def _out(case, f16):
    shape = (case.rows_out, case.C) if f16 else (2, case.rows_out, case.C)
    return torch.full(shape, SENTINEL, dtype=torch.float16 if f16 else torch.bfloat16, device=DEV)


def _bar_parts(case, f16):
    """Flat [rows_out * C] float64: the bar of every written output element before the output's own rounding."""
    terms = 1 if f16 else 3
    flat = torch.zeros(case.rows_out * case.C, dtype=torch.float64)
    for b, h, rows, sch in A.schedules(case, f16):
        steps = sch.grow.shape[1] * (4 * terms + 1) + 20
        bar = sch.err + (sch.rel + steps * 2.0 ** -19)[:, None] * sch.mag
        orow = case.rowmap[b * case.Lq + rows].long()
        keep = orow >= 0
        idx = orow[keep][:, None] * case.C + h * 128 + torch.arange(128)
        flat[idx.reshape(-1)] = bar[keep].reshape(-1)
    return flat


class _PerElement(Replayer):
    """Replays fgt_attention and holds each written element to its own bar (`self.bar`, flat over the output)."""

    bar = None
    worst = 0.0

    def _compare(self, name, cargs, emu, before, after, work):
        key = {w.untyped_storage().data_ptr(): b for b, w in work.items()}
        self._check_untouched(name, emu, before, after, work)
        n = 0
        for kind, fl, idx, plane, want in emu.records:
            assert kind in ("split", "f16"), kind
            g = torch.empty(0, dtype=fl.dtype).set_(after[key[fl.untyped_storage().data_ptr()]].untyped_storage(),
                                                    fl.storage_offset(), fl.shape, (1,))
            got = g[idx].double() + (g[idx + plane].double() if kind == "split" else 0.0)
            assert torch.isfinite(got).all(), f"{name}: non-finite output"
            w = want.abs()
            own = 2.0 ** -16 * w if kind == "split" else 0.5 * _ulp16(w) + 2.0 ** -22 * w
            ratio = (got - want).abs() / (self.bar[idx] + own + 1e-300)
            self.worst = max(self.worst, ratio.max().item())
            n += idx.numel()
        assert n > 0


@contextlib.contextmanager
def _replaying_per_element(bar):
    saved = lib.load()
    rep = _PerElement(saved, ("fgt_attention",), device_type=DEV.type)
    rep.bar = bar
    lib._lib = rep
    try:
        yield rep
    finally:
        lib._lib = saved
        rep._st.clear()


def _launch(case, f16, k=None, v=None, out=None):
    q = _enc(case.q.reshape(-1, case.C), f16).to(DEV)
    kk = _enc((case.k if k is None else k).reshape(-1, case.C), f16).to(DEV)
    vv = _enc((case.v if v is None else v).reshape(-1, case.C), f16).to(DEV)
    out = _out(case, f16) if out is None else out
    lib.attention(q, kk, vv, out, out_rowmap=case.rowmap.to(DEV), **case.launch_kwargs())
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("f16", (False, True), ids=("split", "fp16"))
@pytest.mark.parametrize("name", list(CASES))
def test_designed_scores_against_float64(name, f16):
    case = CASES[name]
    with _replaying_per_element(_bar_parts(case, f16)) as r:
        _launch(case, f16)
    assert r.launches["fgt_attention"] == 1
    print(f"\n[{name} {'fp16' if f16 else 'split'}] max error {r.worst:.3g} x bar")
    assert r.worst <= 1.0, f"{name}: error {r.worst:.3g} x its bar"


def _masked_rows(case):
    """Key rows the kernel reads but masks: [Lk, Lk_rows) dense, the padding after the pooled keys windowed."""
    if case.mode == 0:
        return torch.arange(case.Lk, case.R)
    end = case.Lq + -(-case.G // 64) * 64
    return torch.arange(case.Lq + case.G, end)


@pytest.mark.parametrize("f16", (False, True), ids=("split", "fp16"))
@pytest.mark.parametrize("name", ["partial1_inside", "windowed_g65"])
def test_masked_key_rows_contract(name, f16):
    """NaN, +Inf and -Inf in K's masked rows leave the output bit-identical; a NaN in V's masked rows of batch 0 makes
    every output of batch 0 NaN and leaves batch 1 bit-identical."""
    case = CASES[name]
    rows = _masked_rows(case)
    assert rows.numel() > 0
    base = _launch(case, f16).cpu()
    for bad in (math.nan, math.inf, -math.inf):
        k = case.k.clone()
        k[:, rows] = bad
        got = _launch(case, f16, k=k).cpu()
        assert torch.equal(got.view(torch.int16), base.view(torch.int16)), f"K = {bad} in a masked row changed the output"
    v = case.v.clone()
    v[0, rows[0]] = math.nan
    got = _launch(case, f16, v=v).cpu()
    m = case.rowmap.view(case.B, case.Lq).long()
    hi = (lambda t: t) if f16 else (lambda t: t[0])   # noqa: E731
    r0, r1 = m[0][m[0] >= 0], m[1][m[1] >= 0]
    assert torch.isnan(hi(got)[r0].float()).all(), "a NaN in a masked V row did not reach batch 0's outputs"
    assert torch.equal(hi(got)[r1].view(torch.int16), hi(base)[r1].view(torch.int16))


# ----------------------------------------------------------------------------------------- production census, report
class _Census(KernelEmulator):
    """Runs the schedule model on an attention launch's pre-launch operands instead of computing it; writes nothing."""

    rows_budget = 4e8   # sampled query rows x keys x 128 per launch
    seen = None

    def _attention(self, a):
        d = a["desc"]
        f16, B, H, Lq, R = bool(d["f16"]), d["batches"], d["heads"], d["Lq"], d["Lk_rows"]
        C = H * 128
        q = self.v16(d["q_hi"], 0 if f16 else d["q_plane"], (B, Lq, C), (d["q_batch_stride"], d["q_ld"], 1), f16)
        k = self.v16(d["k_hi"], 0 if f16 else d["k_plane"], (B, R, C), (d["k_batch_stride"], d["k_ld"], 1), f16)
        if d["mode"] == 1:
            assert d["glob_start"] == Lq
        case = A.Case("", d["mode"], B, H, Lq, d["Lk"], R, d["glob_count"], d["scale"], q, k, k, None, 0, {})
        keys = d["Lk"] if d["mode"] == 0 else 64 + d["glob_count"]
        groups = list(case.groups())
        per_group = groups[0][2].numel() * keys * 128
        step = max(1, int(len(groups) * per_group // self.rows_budget))
        for i, (b, h, rows, kidx, live) in enumerate(groups):
            if d["mode"] == 0:
                rows = rows[::max(1, int(per_group * len(groups) // self.rows_budget))]
            elif i % step:
                continue
            s, _ = case.loaded(b, h, rows, kidx)
            sch = A.schedule(s, live, d["scale"], f16)
            n = sch.rescales_after_first()
            st = self.seen[(("fp16" if f16 else "split"), ("dense", "windowed")[d["mode"]])]
            st["rows"] += n.numel()
            st["rescaling"] += int((n > 0).sum())
            st["last_tile"] += int((sch.grow[:, -1] & (n > 0)).sum())
            for j, c in zip(*torch.unique(n, return_counts=True)):
                st[f"n={int(j)}"] += int(c)


class _CensusReplayer(Replayer):
    emulator = _Census

    def _compare(self, name, cargs, emu, before, after, work):
        pass


@pytest.mark.parametrize("mixed", (False, True), ids=("split", "fp16"))
def test_rescale_census_at_production_geometry(mixed):
    """Report only: of the sampled query rows of every attention launch in FGT 432 x 240, T = 10, how many rescale after
    their first key tile, how many of those on the last tile, and the distribution of rescales per row."""
    run = _fgt((240, 432), 10, 240, 432, mixed=mixed)
    _Census.seen = collections.defaultdict(collections.Counter)
    with torch.no_grad():
        run()
        saved = lib.load()
        rep = _CensusReplayer(saved, ("fgt_attention",), device_type=DEV.type)
        lib._lib = rep
        try:
            run()
        finally:
            lib._lib = saved
            rep._st.clear()
    assert rep.launches["fgt_attention"] > 0
    for (prec, mode), st in sorted(_Census.seen.items()):
        dist = {k: v for k, v in sorted(st.items()) if k.startswith("n=")}
        print(f"\n[census {prec} {mode}] {rep.launches['fgt_attention']} launches, {st['rows']} rows sampled: "
              f"{100.0 * st['rescaling'] / st['rows']:.2f}% rescale after the first tile, "
              f"{100.0 * st['last_tile'] / st['rows']:.2f}% on the last tile; rescales per row {dist}")
