"""Launch-by-launch replay of real forwards on the H100: every replayed C-ABI call runs on the GPU and then, on CPU
copies of the buffers it referenced as they were before the launch, through the float64 interpreter of
tests/kernel_emulator.py. So the kernels are checked on real activations with every argument combination the forwards
use, and each launch is checked for the bytes it leaves alone.

Per replayed launch: every pointer argument (descriptor fields and pointer arrays included) is resolved to a live CUDA
storage; the storages are synchronised and copied to the CPU, the kernel runs, and they are copied again; the interpreter
runs on the pre-launch copies with the pointers translated to the same offsets. Every byte the interpreter does not
write must be bit-identical to the pre-launch copy; the elements it writes must agree within the entry's bar:
- exactly defined entries (upsample2x, f16_to_split, raft_flow_update, im2col_nchw without scale / shift): bit-identical;
- avgpool2: within 3 * 2^-24 of the mean of the four magnitudes (three fp32 roundings; the header fixes no sum order);
- attention: 1e-4 of the output's largest value (split-bf16), 2e-3 (fp16);
- fgt_gemm_tc: 2e-4 (split-bf16 layers), 2e-4 (fp16 layers with fp32 output) and 2^-9 (launches with an fp16 output,
  whose fp32 copy holds the same fp16 values), as tests/test_gemm_layers_gpu.py except the split-bf16 bar, 2e-4 here
  rather than 1e-4: the 3-term product's error scales with sum |a| |w| of each output, and on real activations
  cancellation leaves some outputs' largest value well below that sum (RAFT's fp32 64 x 96 forward showed 1.16e-4);
- other fp32, fp64 and split-bf16 outputs: 2e-5 of the output's largest value. Other fp16 outputs: at most one fp16 ulp
  from the interpreter's fp16 value, or within that 2e-5. The second clause is for small elements: these kernels' fp32
  error scales with their operands (LayerNorm's x - mean over the row, the up to 9 entries a fold sums, the four
  corners of a lookup), not with the element, so near zero it exceeds the element's own fp16 ulp;
- instnorm_act, split-bf16 / fp32: 2e-5 of the largest value plus each element's fp32 conditioning,
  s = 2^-22 (|x| + |mean|) rstd + 2^-23 |y| (x - mean, mean, rstd and the product rounded to fp32). With an fp16 output,
  the fp32 copy must hold the fp16 output's values bit for bit (the header's definition), and each fp16 value must lie
  in the interval the two roundings allow: y16 in [r16(relu(y - s)), r16(relu(y + s))] and, with a residual, the result
  in [r16(relu(lo(y16) + res - e)), r16(relu(hi(y16) + res + e))], e the fp32 rounding of the add. So a one-ulp flip of
  y16 before the add is accepted only where y lies within s of an fp16 rounding midpoint; elsewhere the result must be
  the interpreter's. (RAFT's downsample residual is negative: such a flip of a value near 1 survives in a result near 0.)
Forwards run eagerly, without CUDA graphs: the seven launch-trace cases at their geometries with every launch, the GEMMs
included (at 64 x 96 RAFT's coarsest correlation level is 1 x 1, where only the interpreter can serve as reference);
and the production geometries with every launch but the GEMMs (float64 CPU GEMMs at these sizes add minutes and no
coverage): FGT 432 x 240, T = 10, fp32 and mixed; RAFT on one 480 x 864 pair, 3 iterations, fp32 and mixed; LAFC at
the 240 x 432 clip's size. Production attention computes every k-th 64-row query window in float64 (k from a work
budget); the others are checked for their addresses only.

Observed on an H100 80GB HBM3, the largest error over all replayed launches in units of the entry's bar: bit-identical
for upsample2x, f16_to_split, raft_flow_update and unscaled im2col_nchw, and for scaled im2col_nchw (0); attention
0.20 (split) / 0.35 (fp16); gemm_tc 0.62 (split, fp32) / 0.41 (fp16); avgpool2 0.67; chan_stats 0.0018;
conv_tail 0.35 (0.29 in RAFT's flow head); convex_upsample 0.013; corr_lookup 0.56 (split); dwconv3x3_res 0.72;
fold 0.70; fold_unfold 0.35; instnorm_act 0.57 (split), and every fp16 value inside its interval; rownorm 0.69 (0.34
on the low-variance rows); swin_prep 0.64 (0.36); upflow8 0.013. The fp16 outputs of corr_lookup, dwconv3x3_res,
fold, fold_unfold, rownorm and swin_prep reach one fp16 ulp (1.0), never two.

Each of these changes to a kernel's arithmetic fails a test here: lookup windows a and b swapped (error 5e4 x the bar),
eps dropped from rownorm (non-finite on the constant rows; 58 x the bar in FGT's 64 x 96 forward), swin_prep writing a
padding row, raft_flow_update writing one channel lower (bytes outside its outputs changed), instnorm_act skipping
the fp16 rounding before the residual add or the one of its fp32 copy.
"""
import argparse
import collections
import ctypes
import gc
import weakref

import pytest
import torch
import torch.nn.functional as F

from fgt_b200 import lib, synth
from tests.kernel_emulator import ENTRIES, KernelEmulator
from tests.util import load_golden

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
EXACT_ENTRIES = {"fgt_upsample2x", "fgt_f16_to_split", "fgt_raft_flow_update"}
CUDA_CORE = 2e-5
GEMM_SPLIT = 2e-4


def _ptr_fields(s):
    """(struct, field) of every pointer field of a descriptor, nested arrays of structs included."""
    for f, t in s._fields_:
        if t is ctypes.c_void_p:
            yield s, f
        elif isinstance(getattr(s, f), ctypes.Array):
            for el in getattr(s, f):
                if isinstance(el, ctypes.Structure):
                    yield from _ptr_fields(el)


def _bytes(t):
    st = t.untyped_storage()
    return torch.empty(0, dtype=torch.uint8, device=t.device).set_(st, 0, (st.nbytes(),), (1,))


def _ulp16_dist(a, b):
    """fp16 ulp distance of two fp16 tensors (ordered bit patterns)."""
    def ordered(x):
        i = x.view(torch.int16).int()
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return (ordered(a) - ordered(b)).abs()


def _ulp16(v):
    """Spacing of fp16 values at magnitude v (float64)."""
    e = torch.floor(torch.log2(v.clamp_min(2.0 ** -14)))
    return torch.where(v < 2.0 ** -14, torch.full_like(v, 2.0 ** -24), torch.exp2(e - 10))


def _instnorm_y(emu, a, idx):
    """float64 (x - mean) * rstd at elements idx (from the statistics as stored) and its fp32 conditioning
    s = 2^-22 (|x| + |mean|) rstd + 2^-23 |y|: x - mean, mean, rstd and the product rounded to fp32. s dominates 2e-5
    of the largest output in channels whose spread is small against their mean."""
    n, HW, C = a["n"], a["HW"], a["C"]
    st = emu.flat(a["stats"], torch.float64)[:n * C * 2].view(n, C, 2)
    mean = st[..., 0] / HW
    rstd = 1.0 / torch.sqrt((st[..., 1] / HW - mean * mean).clamp_min(0) + a["eps"])
    img, c = idx // (HW * C), idx % C
    x, m, r = emu.f32(a["x"], n * HW * C)[idx], mean[img, c], rstd[img, c]
    y = (x - m) * r
    return y, 2.0 ** -22 * (x.abs() + m.abs()) * r + 2.0 ** -23 * y.abs()


def _r16(v):
    return v.float().half().double()


def _instnorm_f16_interval(emu, a, idx):
    """[lo, hi] of the fp16 values instnorm_act may store at elements idx: the kernel's fp32 y within s of the float64
    y, ReLU, rounded to fp16; with a residual, y16 + res (rounded to fp32), ReLU, rounded to fp16 again."""
    y, s = _instnorm_y(emu, a, idx)
    act = (lambda v: v.clamp_min(0.0)) if a["relu"] else (lambda v: v)
    lo, hi = _r16(act(y - s)), _r16(act(y + s))
    if a["res"]:
        r = emu.f32(a["res"], a["n"] * a["HW"] * a["C"])[idx]
        e = 2.0 ** -24 * (torch.maximum(lo.abs(), hi.abs()) + r.abs())
        lo, hi = _r16((lo + r - e).clamp_min(0.0)), _r16((hi + r + e).clamp_min(0.0))
    return lo, hi


class Replayer:
    """Stands in for the ctypes library: the entries in `entries` run on the GPU and are then replayed by the
    interpreter and compared; every other entry goes straight to the real library. `maxima[(entry, kind)]` holds the
    largest error seen, in the unit of the entry's bar. Subclasses replay other entries by naming another interpreter in
    `emulator` and overriding `_compare` (tests/test_prop_kernels_gpu.py)."""

    emulator = KernelEmulator

    def __init__(self, real, entries, attn_budget=None, device_type="cuda"):
        self.real, self.entries, self.attn_budget = real, set(entries), attn_budget
        self.device_type = device_type
        self._st = {}   # storage base -> (end, weak reference to a tensor on it): nothing is kept alive
        self.maxima = collections.defaultdict(float)
        self.launches = collections.Counter()

    def __getattr__(self, name):
        f = getattr(self.real, name)
        if name not in self.entries:
            return f
        return lambda *args: self._replay(name, f, args)

    def _find(self, p):
        """(storage base, a live tensor on that storage) of address p. Only storages that pointer arguments resolve to
        are remembered, by weak reference, so the replay keeps no buffer alive that the forward would free."""
        for base, (end, ref) in list(self._st.items()):
            t = ref()
            if t is None:
                del self._st[base]
            elif base <= p < end:
                return base, t
        for o in gc.get_objects():
            if isinstance(o, torch.Tensor) and o.device.type == self.device_type:
                st = o.untyped_storage()
                base = st.data_ptr()
                if st.nbytes() and base <= p < base + st.nbytes():
                    self._st[base] = (base + st.nbytes(), weakref.ref(o))
                    return base, o
        raise AssertionError(f"address {p:#x} is in no live {self.device_type} tensor")

    def _sync(self):
        if self.device_type == "cuda":
            torch.cuda.synchronize()

    def _pointers(self, args, argtypes):
        """(container, key) of every non-null pointer argument (the last argument, the stream, excluded)."""
        out = []
        for i, (a, t) in enumerate(zip(args[:-1], argtypes)):
            if type(a).__name__ == "CArgObject":
                for s, f in _ptr_fields(a._obj):
                    if getattr(s, f):
                        out.append((s, f))
            elif isinstance(a, ctypes.Array):
                if a._type_ is ctypes.c_void_p:
                    out += [(a, j) for j in range(len(a)) if a[j]]
            elif t is ctypes.c_void_p and a is not None:
                out.append((args, i))
        return out

    def _replay(self, name, f, args):
        args = list(args)
        # copies of descriptors and pointer arrays, so translating the interpreter's pointers leaves the real call alone
        cargs = []
        for a in args:
            if type(a).__name__ == "CArgObject":
                cargs.append(ctypes.byref(type(a._obj).from_buffer_copy(a._obj)))
            elif isinstance(a, ctypes.Array):
                cargs.append(type(a)(*a))
            else:
                cargs.append(a.value if isinstance(a, ctypes.c_void_p) else a)
        ptrs = self._pointers(cargs, f.argtypes)

        def get(h):
            v = getattr(h[0], h[1]) if isinstance(h[0], ctypes.Structure) else h[0][h[1]]
            return v.value if isinstance(v, ctypes.c_void_p) else v

        live = dict(self._find(get(h)) for h in ptrs)   # strong references for the duration of this launch
        bases = sorted(live)
        self._sync()
        before = {b: _bytes(live[b]).clone().cpu() for b in bases}
        rc = f(*args)
        if rc != 0:
            return rc
        self._sync()
        after = {b: _bytes(live[b]).clone().cpu() for b in bases}
        work = {b: before[b].clone() for b in bases}
        for h in ptrs:
            p = get(h)
            b = max(x for x in bases if x <= p)
            q = work[b].data_ptr() + (p - b)
            if isinstance(h[0], ctypes.Structure):
                setattr(h[0], h[1], q)
            else:
                h[0][h[1]] = q
        emu = self.emulator()
        emu.attn_budget = self.attn_budget
        emu._storages = [[w.data_ptr(), w.data_ptr() + w.numel(), w] for w in work.values()]
        entry = getattr(emu, name)
        entry.argtypes = f.argtypes
        entry(*cargs)
        self._compare(name, cargs, emu, before, after, work)
        self.launches[name] += 1
        return rc

    @staticmethod
    def _check_untouched(name, emu, before, after, work):
        for b, w in work.items():
            wb = emu.written_bytes(w)
            assert torch.equal(after[b][~wb], before[b][~wb]), f"{name}: bytes outside its outputs changed"

    def _compare(self, name, cargs, emu, before, after, work):
        key = {w.untyped_storage().data_ptr(): b for b, w in work.items()}
        self._check_untouched(name, emu, before, after, work)
        a = dict(zip(lib.PROTOS[name].names, cargs))
        exact = name in EXACT_ENTRIES or (name == "fgt_im2col_nchw" and (a["scale"], a["shift"]) == (1.0, 0.0))
        inorm16 = name == "fgt_instnorm_act" and a["out_hi"] and a["out_plane"] == 0
        stored = {}
        for kind, fl, idx, plane, _ in emu.records:
            if kind == "addr":
                continue
            b = key[fl.untyped_storage().data_ptr()]
            g = torch.empty(0, dtype=fl.dtype).set_(after[b].untyped_storage(), fl.storage_offset(), fl.shape, (1,))
            idxs = (idx,) if kind != "split" else (idx, idx + plane)
            if exact:   # bit for bit; a NaN only as a NaN (payloads are not specified)
                for i in idxs:
                    same = (g[i].view(torch.uint8).view(-1, g.element_size()) ==
                            fl[i].view(torch.uint8).view(-1, fl.element_size())).all(1)
                    assert bool((same | (torch.isnan(g[i].float()) & torch.isnan(fl[i].float()))).all()), \
                        f"{name}: not bit-identical"
                continue
            got, want = g[idx].double(), fl[idx].double()
            stored[kind] = got
            if kind == "split":
                got, want = got + g[idx + plane].double(), want + fl[idx + plane].double()
            assert torch.isfinite(got).all(), f"{name}: non-finite output"
            scale = want.abs().max().item() + 1e-30
            if name == "fgt_avgpool2":
                x = emu.f32(a["in"], a["rows"] * a["h"] * a["w"]).view(a["rows"], a["h"], a["w"]).abs()
                mag = F.avg_pool2d(x[:, None], 2, stride=2).reshape(-1)[idx]
                err = ((got - want).abs() / (3 * 2.0 ** -24 * mag + 1e-38)).max().item()
            elif name == "fgt_gemm_tc":
                d = cargs[0]._obj
                bar = GEMM_SPLIT if d.terms != 1 else (2.0 ** -9 if d.out_half else 2e-4)
                err = (got - want).abs().max().item() / scale / bar
            elif name == "fgt_attention":
                bar = 2e-3 if kind == "f16" else 1e-4
                err = (got - want).abs().max().item() / scale / bar
            elif inorm16:   # fp16 values, in the fp32 copy too: inside the interval the roundings allow
                lo, hi = _instnorm_f16_interval(emu, a, idx)
                assert bool(((lo <= want) & (want <= hi)).all()), "instnorm_act: interval misses the interpreter"
                out_by = (lo - got).clamp_min(0) + (got - hi).clamp_min(0)
                err = (out_by / _ulp16(want.abs())).max().item() + (1.0 if bool((out_by > 0).any()) else 0.0)
            elif kind == "f16":
                near = (got - want).abs() <= CUDA_CORE * scale
                d16 = _ulp16_dist(g[idx], fl[idx]).double()
                err = torch.where(near, torch.zeros_like(got), d16).max().item()
            elif name == "fgt_instnorm_act":
                slack = _instnorm_y(emu, a, idx)[1]
                err = (((got - want).abs() - slack).clamp_min(0).max().item()) / scale / CUDA_CORE
            else:
                err = (got - want).abs().max().item() / scale / CUDA_CORE
            self.maxima[(name, kind)] = max(self.maxima[(name, kind)], err)
            assert err <= 1.0, f"{name} ({kind}): error {err:.3g} x its bar"
        if inorm16 and "f32" in stored:
            assert torch.equal(stored["f32"], stored["f16"]), "instnorm_act: fp32 copy != fp16 output"

    def report(self, what):
        print(f"\n[{what}] launches {dict(self.launches)}")
        for (n, k), v in sorted(self.maxima.items()):
            print(f"[{what}] {n} {k}: max error {v:.3g} x bar")


class replaying:
    """`with replaying(entries) as r:` replays the launches of `entries` issued inside the block."""

    def __init__(self, entries=ENTRIES + ("fgt_gemm_tc",), attn_budget=None):
        self.entries, self.attn_budget = entries, attn_budget

    def __enter__(self):
        self.saved = lib.load()
        self.rep = Replayer(self.saved, self.entries, self.attn_budget, device_type=DEV.type)
        lib._lib = self.rep
        return self.rep

    def __exit__(self, *exc):
        lib._lib = self.saved
        self.rep._st.clear()
        return False


# ---------------------------------------------------------------------------------------------------------- forwards
def _fgt(res, t, H, W, mixed=False, sharded=False, seed=1, regime=None):
    from fgt_b200.fgt_model import Model
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = tuple(res)
    m = Model(cfg)
    kw = {} if regime is None else dict(regime=regime)
    m.load_state_dict(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=seed, **kw))
    m = m.to(DEV)
    if sharded:
        m.net.enable_frame_sharding(2, rank=0, world=1, exchange="nccl")
    fr, fl, mk = (x.to(DEV) for x in synth.fgt_inputs(seed=seed + 1, t=t, H=H, W=W))
    return lambda: m.net._forward_impl(fr, fl, mk, mixed=mixed)


def _raft(H, W, iters, mixed=False):
    from fgt_b200.raft_model import RAFT
    m = RAFT(argparse.Namespace(small=False, mixed_precision=mixed, alternate_corr=False))
    m.load_state_dict(synth.raft_state_dict(seed=3))
    m = m.to(DEV)
    im1, im2 = (x.to(DEV) for x in synth.raft_inputs(seed=4, H=H, W=W))
    return lambda: m._forward_impl(im1, im2, iters, None, True, mixed)


def _raft_small(H, W, iters):
    from fgt_b200.raft_small import SmallRAFT
    m = SmallRAFT(argparse.Namespace(small=True, mixed_precision=False, alternate_corr=False))
    m.load_state_dict(synth.raft_small_state_dict(seed=3))
    m = m.to(DEV)
    im1, im2 = (x.to(DEV) for x in synth.raft_inputs(seed=4, H=H, W=W))
    return lambda: m._forward_impl(im1, im2, iters, None, True)


def _lafc(H, W, T=None, mixed=False):
    from fgt_b200.lafc_model import Model
    m = Model(synth.CFG_LAFC)
    m.load_state_dict(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=5))
    m = m.to(DEV)
    kw = {} if T is None else dict(T=T)
    flows, masks = (x.to(DEV) for x in synth.lafc_inputs(seed=6, H=H, W=W, **kw))
    return lambda: m.net._forward_impl(flows, masks, mixed=mixed)


def _lafc_single(n, H, W):
    from fgt_b200.lafc_single import Model
    m = Model(synth.CFG_LAFC_SINGLE)
    m.load_state_dict(synth.lafc_single_state_dict(seed=5))
    m = m.to(DEV)
    flows, masks = (x.to(DEV) for x in synth.lafc_single_inputs(seed=6, n=n, H=H, W=W))
    return lambda: m.net._forward_impl(flows, masks)


TRACE_CASES = {   # the geometries of tests/test_launch_trace.py
    "fgt_fp32": lambda: _fgt((64, 96), 2, 64, 96),
    "fgt_mixed": lambda: _fgt((64, 96), 2, 64, 96, mixed=True),
    "fgt_sharded_nccl": lambda: _fgt((64, 96), 2, 64, 96, sharded=True),
    "raft_fp32": lambda: _raft(64, 96, 2),
    "raft_mixed": lambda: _raft(64, 96, 2, mixed=True),
    "raft_small": lambda: _raft_small(64, 96, 2),
    "lafc": lambda: _lafc(64, 96, T=3),
    "lafc_mixed": lambda: _lafc(64, 96, T=3, mixed=True),
    "lafc_single": lambda: _lafc_single(2, 64, 96),
}


def _lafc_full():
    m = load_golden("lafc_full")["meta"]
    return _lafc(m["H"], m["W"])


PRODUCTION = {
    "fgt_432x240_t10_fp32": lambda: _fgt((240, 432), 10, 240, 432),
    "fgt_432x240_t10_mixed": lambda: _fgt((240, 432), 10, 240, 432, mixed=True),
    "raft_480x864_fp32": lambda: _raft(480, 864, 3),
    "raft_480x864_mixed": lambda: _raft(480, 864, 3, mixed=True),
    "lafc_240x432_clip": _lafc_full,
}


def _replay_trace_case(case):
    run = TRACE_CASES[case]()
    with torch.no_grad():
        run()                       # packs the weights and allocates the workspaces outside the replay
        with replaying() as r:
            run()
    r.report(case)
    assert sum(r.launches.values()) > 0


def _replay_production_case(case):
    run = PRODUCTION[case]()
    with torch.no_grad():
        run()
        with replaying(ENTRIES, attn_budget=3e10) as r:
            run()
    r.report(case)
    assert sum(r.launches.values()) > 0


@pytest.mark.parametrize("case", sorted(c for c in TRACE_CASES if not c.startswith("raft")))
def test_replay_trace_cases_every_launch(case):
    _replay_trace_case(case)


@pytest.mark.parametrize("case", sorted(c for c in PRODUCTION if not c.startswith("raft")))
def test_replay_production_non_gemm_launches(case):
    _replay_production_case(case)


# RAFT's forwards pass fgt_corr_lookup's per-level host tables (device pointers, heights, widths): the replay resolves
# the pointer table element by element and passes the int tables through as they are.
@pytest.mark.parametrize("case", sorted(c for c in TRACE_CASES if c.startswith("raft")))
def test_replay_raft_trace_cases_with_host_level_tables(case):
    _replay_trace_case(case)


@pytest.mark.parametrize("case", sorted(c for c in PRODUCTION if c.startswith("raft")))
def test_replay_raft_production_non_gemm_launches_with_host_level_tables(case):
    _replay_production_case(case)


# ------------------------------------------------------------------------------------------------------- edge cases
def test_f16_to_split_every_pattern():
    """All 65536 fp16 patterns: for every finite value hi + lo == value exactly and hi = bf16(value); +-inf give hi =
    +-inf and a NaN lo (inf - inf); NaN gives NaN in both planes."""
    src = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16).to(DEV)
    out = torch.zeros(2, 65536, dtype=torch.bfloat16, device=DEV)
    with replaying(("fgt_f16_to_split",)) as r:
        lib.f16_to_split(src, out)
    assert r.launches["fgt_f16_to_split"] == 1
    s, o = src.cpu(), out.cpu()
    fin = torch.isfinite(s)
    assert torch.equal(o[0, fin].double() + o[1, fin].double(), s[fin].double())
    assert torch.equal(o[0, fin], s[fin].float().to(torch.bfloat16))
    inf = torch.isinf(s)
    assert torch.equal(o[0, inf].float(), s[inf].float()) and torch.isnan(o[1, inf]).all()
    nan = torch.isnan(s)
    assert torch.isnan(o[0, nan]).all() and torch.isnan(o[1, nan]).all()


def test_corr_lookup_edges_with_host_level_tables():
    """Lookup centres on integers, at w - 1 / h - 1, one pixel and half a pixel outside and beyond the +-1e6 clamp, into
    fp16 and split-bf16 rows of pitch 384 (columns 324-383 untouched), including a 1 x 1 coarsest level. The levels'
    pointers, heights and widths reach the entry as host tables."""
    from tests.test_kernel_emulator import _edge_coords, _pyramid
    for h, w in ((16, 24), (8, 12)):
        pyr = [t.to(DEV) for t in _pyramid(h, w, 42)]
        co = _edge_coords(h, w, 43).to(DEV)
        for out in (torch.full((h * w, 384), -7.0, dtype=torch.float16, device=DEV),
                    torch.full((2, h * w, 384), -7.0, dtype=torch.bfloat16, device=DEV)):
            with replaying(("fgt_corr_lookup",)) as r:
                lib.corr_lookup(pyr, co, h * w, 4, out)
            assert r.launches["fgt_corr_lookup"] == 1
            r.report(f"corr_lookup {h}x{w} {out.dtype}")


def test_raft_flow_update_four_modes_at_edges():
    """No delta / delta / fp16-rounded delta, into split-bf16 and fp16 GRU inputs: bit-identical to the interpreter
    at coordinates far outside the image, on fp16 rounding midpoints of the delta and at fractional pixel centres."""
    n, h, w = 2, 7, 11
    N = n * h * w
    g = torch.Generator().manual_seed(44)
    coords = torch.randn(N, 2, generator=g) * 5
    coords[:6] = torch.tensor([[-1e6, 1e6], [3e7, -2.5], [0.5, 0.5], [w - 1.0, h - 1.0], [-0.0, 0.0], [1e-30, 7.0]])
    delta = torch.randn(N, 2, generator=g) * 3
    mid = torch.tensor([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 2048.5, 65519.0, -1e-7, 3.0])   # fp16 midpoints / edges
    delta[:6, 0] = mid
    for delta_on, delta_f16 in ((False, False), (True, False), (True, True)):
        for x in (torch.zeros(2, N, 256, dtype=torch.bfloat16), torch.zeros(N, 256, dtype=torch.float16)):
            c, xb = coords.clone().to(DEV), x.to(DEV)
            flow = torch.zeros(n, 2, h, w, device=DEV)
            with replaying(("fgt_raft_flow_update",)) as r:
                lib.raft_flow_update(c, delta.to(DEV) if delta_on else None, h, w, flow, xb, 254, n=n,
                                     delta_f16=delta_f16)
            assert r.launches["fgt_raft_flow_update"] == 1


def _low_variance_rows(rows, C, seed):
    """Rows of spread 1e-3 (below sqrt(eps)), constant rows and ordinary rows: where eps sets the output scale."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, C, generator=g)
    x[0::3] = 0.5 + 1e-3 * torch.randn(x[0::3].shape, generator=g)
    x[1::6] = 0.75
    return x


def test_layernorm_low_variance_rows():
    """rownorm (with the zone gather, -1 rows and the affine, split-bf16 and fp16) and swin_prep (window, dummy and
    pooled rows) on rows whose variance is below eps or zero, replayed against the interpreter."""
    C, rows = 512, 300
    x = _low_variance_rows(rows, C, 47).to(DEV)
    g = torch.Generator().manual_seed(48)
    gather = torch.randint(-1, rows, (rows,), generator=g, dtype=torch.int32).to(DEV)
    gm, bt = torch.randn(C, generator=g).to(DEV), torch.randn(C, generator=g).to(DEV)
    for out in (torch.zeros(2, rows, C, dtype=torch.bfloat16, device=DEV),
                torch.zeros(rows, C, dtype=torch.float16, device=DEV)):
        with replaying(("fgt_rownorm",)) as r:
            lib.rownorm(x, None, out, gather=gather, rows_per_batch=rows, total_rows=rows, dst_batch_rows=rows,
                        eps=1e-5, gamma=gm, beta=bt)
            lib.rownorm(x, None, out, rows_per_batch=rows, total_rows=rows, dst_batch_rows=rows, eps=1e-5)
        assert r.launches["fgt_rownorm"] == 2
        r.report(f"rownorm low variance {out.dtype}")
    bt_, h, w, d, df, gd = 2, 8, 16, 512, 256, 4
    nl, G = 128 * 2, (h // gd) * (w // gd)
    R = nl + G + 8
    xs = _low_variance_rows(bt_ * h * w, d, 49).to(DEV)
    fp = _low_variance_rows(bt_ * h * w, df, 50).to(DEV)
    wm = torch.full((bt_, nl), -1, dtype=torch.int32)
    for f in range(bt_):
        wm[f, :h * w] = torch.arange(h * w, dtype=torch.int32) + f * h * w    # 2 windows of tokens, 2 dummy windows
    gk_w = torch.full((gd * gd, d + df), 1.0 / (gd * gd)).to(DEV)             # pooled rows keep the low spread
    gv_w = torch.full((gd * gd, d), 1.0 / (gd * gd)).to(DEV)
    gk_b, gv_b = torch.full((d + df,), 0.25).to(DEV), torch.full((d,), 0.25).to(DEV)
    for f16 in (False, True):
        qkn = (torch.zeros(bt_ * R, d + df, dtype=torch.float16) if f16
               else torch.zeros(2, bt_ * R, d + df, dtype=torch.bfloat16)).to(DEV)
        vn = (torch.zeros(bt_ * R, d, dtype=torch.float16) if f16
              else torch.zeros(2, bt_ * R, d, dtype=torch.bfloat16)).to(DEV)
        with replaying(("fgt_swin_prep",)) as r:
            lib.swin_prep(xs, fp, bt_, h, w, wm.reshape(-1).to(DEV), nl, R, gd, h // gd, w // gd, gk_w, gk_b, gv_w,
                          gv_b, qkn, vn, eps=1e-5)
        assert r.launches["fgt_swin_prep"] == 1
        r.report(f"swin_prep low variance f16={f16}")


def test_instance_norm_of_a_large_mean():
    """chan_stats + instnorm_act on channels whose mean is 30 times their spread, at RAFT's largest instance-norm
    geometry, against F.instance_norm in float64: 2e-5 of the largest value. Observed: 9.0e-6."""
    n, H, W, C = 2, 240, 432, 64
    g = torch.Generator().manual_seed(45)
    x = (torch.randn(n, H * W, C, generator=g) + torch.where(torch.arange(C) % 2 == 0, 30.0, 0.5)).to(DEV)
    stats = torch.empty(n * C * 2, dtype=torch.float64, device=DEV)
    out = torch.empty_like(x)
    lib.chan_stats(x, n, H * W, C, stats)
    lib.instnorm_act(x, stats, n, H * W, C, relu=False, out=out)
    ref = F.instance_norm(x.double().permute(0, 2, 1), eps=torch.tensor(1e-5).float().item()).permute(0, 2, 1)
    err = ((out.double() - ref).abs().max() / ref.abs().max()).item()
    print(f"\n[instance norm, mean 30 sigma] max error {err:.3g} of the largest value")
    assert err <= CUDA_CORE
