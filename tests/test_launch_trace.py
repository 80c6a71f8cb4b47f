"""The C-ABI call sequence of each network's forward, recorded on the CPU against a fixed golden.

The ctypes library is swapped for a recorder that returns success, so `_forward_impl` runs its whole host side on CPU
tensors: weight packing, workspace allocation, tile and box choice, descriptor filling. Every call is recorded with its
entry name and its arguments (descriptor structs field by field, pointer arrays element by element). A pointer is
recorded as (storage ordinal in order of first use, byte offset), so the trace pins which buffer and offset each
launch reads and writes, but not where the allocator put it. The golden (tests/golden/launch_trace.json.gz, written by
tests/golden/make_launch_trace.py) pins the launches to that schedule: a host-side change that alters any launch, its
order, a scalar argument or a buffer binding fails here.

Not covered: the P2P frame-sharded exchange (it needs CUDA IPC; tests/test_frame_shard_gpu.py runs it on the GPU).
"""
import argparse
import contextlib
import ctypes
import gc
import gzip
import json
import os

import pytest
import torch

from fgt_b200 import lib, synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "launch_trace.json.gz")


class _Entry:
    """One C-ABI entry of the recorder; `lib.load()` declares its argtypes as it does on the real library."""

    def __init__(self, rec, name):
        self.rec, self.name, self.argtypes = rec, name, None

    def __call__(self, *args):
        assert self.argtypes is not None and len(args) == len(self.argtypes), self.name
        self.rec.calls.append([self.name, [self.rec.value(a, t) for a, t in zip(args, self.argtypes)]])
        return 0


class _Recorder:
    """Stands in for the ctypes library: every `fgt_*` entry records its call and returns 0."""

    def __init__(self):
        self.calls = []
        self._storages = []   # [base, end, tensor]: kept alive so that no address is reused during the trace

    def __getattr__(self, name):
        if not name.startswith("fgt_"):
            raise AttributeError(name)
        e = _Entry(self, name)
        setattr(self, name, e)
        return e

    def _ptr(self, p):
        for i, (base, end, _) in enumerate(self._storages):
            if base <= p < end:
                return ["ptr", i, p - base]
        for o in gc.get_objects():
            if issubclass(type(o), torch.Tensor) and o.device.type == "cpu":
                st = o.untyped_storage()
                base = st.data_ptr()
                if st.nbytes() and base <= p < base + st.nbytes():
                    self._storages.append([base, base + st.nbytes(), o])
                    return ["ptr", len(self._storages) - 1, p - base]
        raise AssertionError(f"address {p:#x} is in no live tensor")

    def value(self, a, t):
        """JSON-ready value of argument or field `a` declared as ctypes type `t`."""
        if isinstance(a, ctypes.Array):
            return [self.value(x, a._type_) for x in a]
        if isinstance(a, ctypes.Structure):
            return {f: self.value(getattr(a, f), ft) for f, ft in a._fields_}
        if type(a).__name__ == "CArgObject":   # ctypes.byref(desc)
            return self.value(a._obj, None)
        if isinstance(a, ctypes.c_void_p):
            a = a.value
        if t is ctypes.c_void_p and isinstance(a, int):
            return self._ptr(a)
        assert a is None or isinstance(a, (int, float, str)), type(a)
        return a


@contextlib.contextmanager
def recording(rec=None):
    """Swaps the library `lib.load()` returns for a recorder (argument types declared by `lib.load()` itself) and
    the stream handle for a constant. `rec`: a stand-in other than a fresh _Recorder (tests/gemm_emulator.py)."""
    rec = _Recorder() if rec is None else rec
    saved = lib._lib, lib.LIB_PATH, lib.stream_ptr, ctypes.CDLL
    try:
        lib._lib, lib.LIB_PATH, ctypes.CDLL = None, __file__, (lambda path: rec)
        lib.load()
        ctypes.CDLL = saved[3]
        lib.stream_ptr = lambda: "stream"
        yield rec
    finally:
        lib._lib, lib.LIB_PATH, lib.stream_ptr, ctypes.CDLL = saved


def _fgt(mixed=False, sharded=False):
    from fgt_b200.fgt_model import Model
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    m = Model(cfg)
    m.load_state_dict(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=1))
    if sharded:   # one rank holding the whole window: the all-gather is a local copy
        m.net.enable_frame_sharding(2, rank=0, world=1, exchange="nccl")
    fr, fl, mk = synth.fgt_inputs(seed=2, t=2, H=64, W=96)
    return lambda: m.net._forward_impl(fr, fl, mk, mixed=mixed)


def _raft(mixed=False):
    from fgt_b200.raft_model import RAFT
    m = RAFT(argparse.Namespace(small=False, mixed_precision=mixed, alternate_corr=False))
    m.load_state_dict(synth.raft_state_dict(seed=3))
    im1, im2 = synth.raft_inputs(seed=4, H=64, W=96)
    return lambda: m._forward_impl(im1, im2, 2, None, True, mixed)


def _raft_small():
    from fgt_b200.raft_small import SmallRAFT
    m = SmallRAFT(argparse.Namespace(small=True, mixed_precision=False, alternate_corr=False))
    m.load_state_dict(synth.raft_small_state_dict(seed=3))
    im1, im2 = synth.raft_inputs(seed=4, H=64, W=96)
    return lambda: m._forward_impl(im1, im2, 2, None, True)


def _lafc(mixed=False):
    from fgt_b200.lafc_model import Model
    m = Model(synth.CFG_LAFC)
    m.load_state_dict(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=5))
    flows, masks = synth.lafc_inputs(seed=6, T=3, H=64, W=96)
    return lambda: m.net._forward_impl(flows, masks, mixed=mixed)


def _lafc_single():
    from fgt_b200.lafc_single import Model
    m = Model(synth.CFG_LAFC_SINGLE)
    m.load_state_dict(synth.lafc_single_state_dict(seed=5))
    flows, masks = synth.lafc_single_inputs(seed=6, n=2, H=64, W=96)
    return lambda: m.net._forward_impl(flows, masks)


CASES = {
    "fgt_fp32": lambda: _fgt(),
    "fgt_mixed": lambda: _fgt(mixed=True),
    "fgt_sharded_nccl": lambda: _fgt(sharded=True),
    "raft_fp32": lambda: _raft(),
    "raft_mixed": lambda: _raft(mixed=True),
    "raft_small": _raft_small,
    "lafc": lambda: _lafc(),
    "lafc_mixed": lambda: _lafc(mixed=True),
    "lafc_single": _lafc_single,
}


def trace(case):
    """The recorded C-ABI calls of one forward of `case` (JSON-ready lists)."""
    run = CASES[case]()
    with torch.no_grad(), recording() as rec:
        run()
    return rec.calls


def load_golden():
    with gzip.open(GOLDEN, "rt") as f:
        return json.load(f)


@pytest.mark.parametrize("case", sorted(CASES))
def test_launch_trace_matches_golden(case):
    want = load_golden()[case]
    got = json.loads(json.dumps(trace(case)))   # the golden's JSON types (tuples -> lists)
    assert [c[0] for c in got] == [c[0] for c in want], "entry sequence differs"
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"call {i} ({g[0]}) differs"
