"""The small RAFT model (the reference's --small) on the CPU: the oracle against goldens of the unmodified reference
(tests/golden/raft_s_*.npz), the module's state-dict contract and refusals, the constructor's choice of model, the whole
native forward through the float64 interpreters of its launches, and the --small switch of both command lines."""
import argparse

import pytest
import torch

from fgt_b200 import synth
from oracle import raft_small_oracle as RSO
from tests.kernel_emulator import emulating_all
from tests.util import assert_close, load_golden


def _args(**kw):
    return argparse.Namespace(**{**dict(small=True, mixed_precision=False, alternate_corr=False), **kw})


class _Stop(Exception):
    pass


@pytest.mark.parametrize("name", ["raft_s_i6", "raft_s_i20"])
def test_oracle_matches_reference_golden(name):
    g = load_golden(name)
    m = g["meta"]
    sd = synth.raft_small_state_dict(seed=m["seed"])
    im1, im2 = synth.raft_inputs(seed=m["seed"] + 1, H=m["H"], W=m["W"])
    with torch.no_grad():
        lo, up = RSO.raft_small_forward(sd, im1, im2, iters=m["iters"])
    assert_close(lo, g["lo"], 2e-5, name + " low-res flow")
    assert_close(up, g["up"], 2e-5, name + " upsampled flow")


def test_state_dict_contract_and_dataparallel_roundtrip():
    from fgt_b200.raft_small import SmallRAFT
    sd = synth.raft_small_state_dict(seed=3)
    dp = torch.nn.DataParallel(SmallRAFT(_args()))
    dp.load_state_dict({"module." + k: v for k, v in sd.items()})
    model = dp.module
    got = model.state_dict()
    assert set(got.keys()) == set(sd.keys()) and len(got) == 106
    for k, v in sd.items():
        assert torch.equal(got[k].cpu(), v), k
    assert (model.args.corr_levels, model.args.corr_radius) == (4, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        model(*synth.raft_inputs(seed=0, H=64, W=64), iters=1, test_mode=True)  # CPU tensors: no fallback


def test_constructor_chooses_the_model_and_refusals():
    from fgt_b200 import raft_model
    from fgt_b200.raft_small import SmallRAFT, make_raft
    assert type(make_raft(_args(small=False))) is raft_model.RAFT
    assert type(make_raft(_args())) is SmallRAFT
    with pytest.raises(ValueError, match="small"):
        raft_model.RAFT(_args())
    for build in (SmallRAFT, make_raft):
        with pytest.raises(ValueError, match="mixed_precision is not implemented for the small model"):
            build(_args(mixed_precision=True))
    m = SmallRAFT(_args())
    m.args.mixed_precision = True   # read on every forward, like the reference
    with pytest.raises(ValueError, match="not implemented"):
        m(*synth.raft_inputs(seed=0, H=64, W=64), iters=1, test_mode=True)


def test_upflow8_interpreter_matches_interpolate():
    """The fgt_upflow8 interpreter against F.interpolate, 1-pixel sides included: the interpreter suite's case."""
    from tests.test_kernel_emulator import CASES
    CASES["upflow8"]()


def test_small_forward_in_float64():
    """The whole native forward (every GEMM, lookup, norm and upflow8 launch) interpreted in float64, against the
    reference's golden and the oracle."""
    from fgt_b200.raft_small import SmallRAFT
    g = load_golden("raft_s_i6")
    meta = g["meta"]
    sd = synth.raft_small_state_dict(seed=meta["seed"])
    m = SmallRAFT(_args())
    m.load_state_dict(sd)
    im1, im2 = synth.raft_inputs(seed=meta["seed"] + 1, H=meta["H"], W=meta["W"])
    with torch.no_grad(), emulating_all() as emu:
        lo, up = m._forward_impl(im1, im2, meta["iters"], None, True)
    assert ("fgt_upflow8", ()) in emu.forms and ("fgt_corr_lookup", ("split", 4, 3)) in emu.forms
    assert_close(lo, g["lo"], 1e-4, "small RAFT low vs reference golden")
    assert_close(up, g["up"], 1e-4, "small RAFT up vs reference golden")
    with torch.no_grad():
        olo, oup = RSO.raft_small_forward(sd, im1, im2, iters=meta["iters"])
    assert_close(up, oup, 1e-4, "small RAFT up vs oracle")


# ------------------------------------------------------------------------------------------------ command lines
def test_pipeline_command_line_small(monkeypatch):
    from fgt_b200 import pipeline
    base = ["--path", "frames", "--path_mask", "masks", "--outroot", "out"]
    assert pipeline.arg_parser().parse_args(base).small is False
    seen = {}

    def fake_load(raft_model, lafc_ckpts, fgt_ckpts, device, mixed_precision=False, small=False):
        seen["small"] = small
        raise _Stop

    monkeypatch.setattr(pipeline, "load_models", fake_load)
    for argv, want in (([], False), (["--small"], True)):
        with pytest.raises(_Stop):
            pipeline.main(base + argv)
        assert seen.pop("small") is want


def _capture_constructor(monkeypatch):
    from fgt_b200 import raft_small
    seen = {}

    def fake(args):
        seen["args"] = args
        raise _Stop

    monkeypatch.setattr(raft_small, "make_raft", fake)
    return seen


def test_load_models_builds_the_small_model(monkeypatch):
    from fgt_b200 import pipeline
    seen = _capture_constructor(monkeypatch)
    for flag in (False, True):
        with pytest.raises(_Stop):
            pipeline.load_models("raft.pth", "lafc", "fgt", torch.device("cpu"), small=flag)
        assert seen.pop("args").small is flag
    with pytest.raises(_Stop):
        pipeline.load_models("raft.pth", "lafc", "fgt", torch.device("cpu"))
    assert seen.pop("args").small is False


def test_flow_extract_command_line_small(monkeypatch):
    from fgt_b200 import flow_extract
    seen = _capture_constructor(monkeypatch)
    for argv, want in (([], False), (["--small"], True)):
        with pytest.raises(_Stop):
            flow_extract.main(["--path", "videos", "--outroot", "flows"] + argv)
        assert seen.pop("args").small is want


def test_dropin_exports_the_constructor():
    import importlib
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "dropin"))
    try:
        sys.modules.pop("RAFT", None)
        R = importlib.import_module("RAFT")
        from fgt_b200.raft_small import make_raft
        assert R.RAFT is make_raft
    finally:
        sys.path.remove(os.path.join(root, "dropin"))
        sys.modules.pop("RAFT", None)
