"""RAFT mixed precision (the reference's --mixed_precision, RAFT/raft.py:100,111,128), CPU side: the mixed oracle's
fp32 mode equals the fp32 oracle, its fp16 emulation differs from fp32 and rounds every conv output to fp16, the command-line switches reach
the model, and the module keeps the reference's state-dict contract in either mode."""
import argparse

import pytest
import torch

from fgt_b200 import synth
from oracle import raft_mixed_oracle as RO
from oracle import raft_oracle

ARGS = dict(small=False, mixed_precision=True, alternate_corr=False)


class _Stop(Exception):
    pass


def _inputs():
    sd = synth.raft_state_dict(seed=3)
    im1, im2 = synth.raft_inputs(seed=4, H=128, W=160)  # 16x20 at 1/8: no 1-pixel pyramid level
    return sd, im1, im2


def test_oracle_fp32_mode_equals_the_fp32_oracle():
    sd, im1, im2 = _inputs()
    with torch.no_grad():
        lo, up, lows = RO.raft_forward(sd, im1, im2, iters=3, all_iters=True)
        lo_f, up_f = RO.raft_forward(sd, im1, im2, iters=3, mixed_precision=False)
        lo_o, up_o, lows_o = raft_oracle.raft_forward(sd, im1, im2, iters=3, all_iters=True)
    assert torch.equal(lo, lo_f) and torch.equal(up, up_f)
    assert torch.equal(lo, lo_o) and torch.equal(up, up_o)
    assert all(torch.equal(a, b) for a, b in zip(lows, lows_o))


def test_emulation_differs_from_fp32_and_rounds_every_conv(monkeypatch):
    sd, im1, im2 = _inputs()
    outs = []
    conv = RO._conv

    def rec(x, sd_, key, stride=1, pad=0, q=None):
        y = conv(x, sd_, key, stride, pad, q)
        outs.append((key, y))
        return y

    monkeypatch.setattr(RO, "_conv", rec)
    with torch.no_grad():
        lo_m, up_m = RO.raft_forward(sd, im1, im2, iters=2, mixed_precision=True)
    # 16 convs in each encoder and 15 in the update block per iteration
    assert len(outs) == 2 * 16 + 2 * 15
    for key, y in outs:
        assert y.dtype == torch.float32 and torch.equal(y, y.half().float()), f"{key}: output not fp16-representable"
    monkeypatch.setattr(RO, "_conv", conv)
    with torch.no_grad():
        lo, up = RO.raft_forward(sd, im1, im2, iters=2)
    assert torch.isfinite(lo_m).all() and torch.isfinite(up_m).all()
    assert not torch.equal(lo_m, lo) and not torch.equal(up_m, up)
    epe = (lo_m - lo).norm(dim=1).mean().item()
    assert 0 < epe < 0.05 * lo.norm(dim=1).mean().item()  # fp16 rounding, not a different model


def test_pipeline_command_line_flag(monkeypatch):
    from fgt_b200 import pipeline
    seen = {}

    def fake_load(raft_model, lafc_ckpts, fgt_ckpts, device, mixed_precision=False):
        seen["mp"] = mixed_precision
        raise _Stop

    monkeypatch.setattr(pipeline, "load_models", fake_load)
    for argv, want in (([], False), (["--mixed_precision"], True)):
        with pytest.raises(_Stop):
            pipeline.main(["--path", "frames", "--path_mask", "masks", "--outroot", "out"] + argv)
        assert seen.pop("mp") is want


def _capture_raft(monkeypatch):
    import fgt_b200.raft_model as RM
    seen = {}

    class Fake(RM.RAFT):
        def __init__(self, args):
            seen["mp"] = args.mixed_precision
            raise _Stop

    monkeypatch.setattr(RM, "RAFT", Fake)
    return seen


def test_load_models_passes_the_flag(monkeypatch):
    from fgt_b200 import pipeline
    seen = _capture_raft(monkeypatch)
    for flag in (False, True):
        with pytest.raises(_Stop):
            pipeline.load_models("raft.pth", "lafc", "fgt", torch.device("cpu"), mixed_precision=flag)
        assert seen.pop("mp") is flag
    with pytest.raises(_Stop):
        pipeline.load_models("raft.pth", "lafc", "fgt", torch.device("cpu"))
    assert seen.pop("mp") is False


def test_flow_extract_command_line_flag(monkeypatch):
    from fgt_b200 import flow_extract
    seen = _capture_raft(monkeypatch)
    for argv, want in (([], False), (["--mixed_precision"], True)):
        with pytest.raises(_Stop):
            flow_extract.main(["--path", "videos", "--outroot", "flows"] + argv)
        assert seen.pop("mp") is want


def test_mixed_module_keeps_state_dict_contract():
    from fgt_b200.raft_model import RAFT
    sd = synth.raft_state_dict(seed=3)
    dp = torch.nn.DataParallel(RAFT(argparse.Namespace(**ARGS)))
    dp.load_state_dict({"module." + k: v for k, v in sd.items()})
    model = dp.module
    got = model.state_dict()
    assert set(got.keys()) == set(sd.keys()) and len(got) == 179
    for k, v in sd.items():
        assert torch.equal(got[k].cpu(), v), k
    assert model._mixed() and model.args.mixed_precision is True
    with pytest.raises(RuntimeError):
        model(*synth.raft_inputs(seed=0, H=64, W=64), iters=1, test_mode=True)  # CPU tensors: no fallback
