"""LAFC's mixed-precision mode (P3DNet.enable_mixed_precision), CPU side: the autocast emulation of
oracle/lafc_mixed_oracle.py, the switch, the per-precision weight and workspace caches, the command-line option, and
the launch sequence of one fp16 forward against its case of the launch-trace golden. The numerics are defined by CUDA
autocast and checked on the GPU (tests/test_lafc_mixed_gpu.py)."""
import ctypes
import json
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from fgt_b200 import lib, synth
from oracle import lafc_mixed_oracle as LM
from oracle import lafc_oracle as LO
from tests.test_launch_trace import load_golden as load_trace_golden
from tests.test_launch_trace import recording


class _Stop(Exception):
    pass


def _sd(seed=5, regime="scaled"):
    return synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=seed, regime=regime)


def _strip(sd):
    return {k[4:]: v for k, v in sd.items()}


def _model(seed=5):
    from fgt_b200.lafc_model import Model
    m = Model(synth.CFG_LAFC)
    m.load_state_dict(_sd(seed))
    return m


def test_fp32_mode_is_the_pinned_oracle():
    sd = _strip(_sd(seed=4))
    fl, mk = synth.lafc_inputs(seed=5, H=32, W=48)
    with torch.no_grad():
        a = LO.lafc_forward(sd, fl, mk)
        b = LM.lafc_forward(sd, fl, mk, mixed_precision=False)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_emulation_is_the_pinned_oracle_with_autocast_casts_by_hand(monkeypatch):
    """The golden-pinned fp32 restatement with autocast's casts applied by hand to each op it calls (conv: fp16 input,
    weight, bias and output; LeakyReLU and sigmoid: fp16 in and out; padding, upsampling and cat untouched). Its
    residual sums stay fp32 until the next op rounds them, which is the same number: the sum of two fp16 values is
    rounded to fp32 and then to fp16 without a double-rounding error (24 >= 2 * 11 + 2 bits)."""
    q = LM.round_f16
    fl, mk = synth.lafc_inputs(seed=5, H=32, W=48)
    sds = {r: _strip(_sd(seed=4, regime=r)) for r in ("scaled", "kaiming")}
    with torch.no_grad():
        got = {r: LM.lafc_forward(sd, fl, mk, mixed_precision=True) for r, sd in sds.items()}
        fp32 = LO.lafc_forward(sds["scaled"], fl, mk)
        conv2d, conv3d, leaky, sigmoid = F.conv2d, F.conv3d, F.leaky_relu, torch.sigmoid
        monkeypatch.setattr(LO.F, "conv2d", lambda x, w, b, **k: q(conv2d(q(x), q(w), q(b), **k)))
        monkeypatch.setattr(LO.F, "conv3d", lambda x, w, b, **k: q(conv3d(q(x), q(w), q(b), **k)))
        monkeypatch.setattr(LO.F, "leaky_relu", lambda x, s: q(leaky(q(x), s)))
        monkeypatch.setattr(LO.torch, "sigmoid", lambda x: q(sigmoid(q(x))))
        want = {r: LO.lafc_forward(sd, fl, mk) for r, sd in sds.items()}
    for r in sds:
        for g, w in zip(got[r], want[r]):
            assert torch.equal(g, w), r
            assert torch.equal(g, q(g)), r   # fp16 values in fp32 tensors
    assert not torch.equal(fp32[0], got["scaled"][0])  # the emulation does round


def test_enable_and_disable():
    net = _model().net
    assert net._mixed is False
    net.enable_mixed_precision()
    assert net._mixed is True
    net.enable_mixed_precision(False)
    assert net._mixed is False
    net.enable_mixed_precision(True)
    with pytest.raises(RuntimeError, match="CUDA"):  # CPU tensors: no fallback in either mode
        net(*synth.lafc_inputs(seed=0, H=32, W=32))
    with pytest.raises(ValueError, match="edges"):   # the existing refusal stays
        net(*synth.lafc_inputs(seed=0, H=32, W=32), torch.zeros(1))


def test_half_pack_is_the_rounded_fp32_pack():
    net = _model(seed=4).net
    cpu = torch.device("cpu")
    p32 = net._pack(cpu, half=False)
    p16 = net._pack(cpu, half=True)
    assert set(p32) == set(p16) and set(net._packed) == {False, True}
    for k in p32:
        a, b = p16[k], p32[k]
        assert a["w"].dtype == torch.float16 and b["w"].dtype == torch.bfloat16, k
        w32 = lib.from_split(b["w"]).double()   # the fp32 weight to split-bf16's 16 bits: within 2^-16 relative
        assert ((a["w"].double() - w32).abs() <= w32.abs() * (2.0 ** -11 + 2.0 ** -15) + 2.0 ** -24).all(), k
        assert torch.equal(a["b"], b["b"].half().float()), k
        assert a["N"] == b["N"] and a["name"] == b["name"]


def _trace(mixed, m=None):
    m = m or _model()
    flows, masks = synth.lafc_inputs(seed=6, T=3, H=64, W=96)
    with torch.no_grad(), recording() as rec:
        m.net._forward_impl(flows, masks, mixed=mixed)
    return m, json.loads(json.dumps(rec.calls))


def test_weights_and_workspaces_are_kept_per_precision():
    m, _ = _trace(False)
    net = m.net
    p32 = net._packed[False]
    geo32 = dict(net._geo[(3, 64, 96, False)])
    _trace(True, m)
    assert net._packed[False] is p32 and set(net._packed) == {False, True}
    assert set(net._geo) == {(3, 64, 96, False), (3, 64, 96, True)}
    geo16 = net._geo[(3, 64, 96, True)]
    assert set(geo16) == set(geo32)
    for k, t in geo32.items():
        assert net._geo[(3, 64, 96, False)][k] is t, k
        if t.dtype == torch.bfloat16:      # split-bf16 [2, ...] -> single-plane fp16 [...]
            assert geo16[k].dtype == torch.float16 and geo16[k].shape == t.shape[1:], k
        else:                              # the fp32 residual operands stay fp32
            assert geo16[k].dtype == torch.float32 and geo16[k].shape == t.shape, k


def _gemms(calls):
    return [c[1][0] for c in calls if c[0] == "fgt_gemm_tc"]


def test_fp32_launch_sequence_is_unchanged():
    _, calls = _trace(False)
    assert calls == load_trace_golden()["lafc"]


def test_mixed_launch_sequence_matches_golden():
    _, calls = _trace(True)
    want = load_trace_golden()["lafc_mixed"]
    assert [c[0] for c in calls] == [c[0] for c in want], "entry sequence differs"
    for i, (g, w) in enumerate(zip(calls, want)):
        assert g == w, f"call {i} ({g[0]}) differs"


def test_mixed_launches_are_one_term_with_autocast_rounding():
    """Every GEMM of the fp16 forward is a 1-term layer with autocast's rounding; every 16-bit producer writes
    single-plane fp16; the fp32 forward has the same launches with split-bf16 operands."""
    _, c16 = _trace(True)
    _, c32 = _trace(False)
    assert [c[0] for c in c16] == [c[0] for c in c32]
    g16, g32 = _gemms(c16), _gemms(c32)
    assert len(g16) == 27
    for a, b in zip(g16, g32):
        assert (a["terms"], a["out_half"], a["w_plane"]) == (1, lib.OUT_HALF_AUTOCAST, 0)
        assert b["terms"] == 3 and b["out_half"] == 0
        assert all(s["plane"] == 0 for s in a["seg"][:a["num_segs"]])
        for f in ("kx", "ky", "kz", "stride", "dil", "pad_x", "pad_y", "pad_z", "N", "out_w", "out_h", "out_z", "box_w",
                  "box_h", "bn", "act", "aux_mode", "os_z", "os_y", "os_x", "os_c", "num_segs"):
            assert a[f] == b[f], f
        assert (a["out_hi"] is None) == (b["out_hi"] is None) and (a["out_f32"] is None) == (b["out_f32"] is None)
    for c in c16:
        if c[0] == "fgt_upsample2x":
            assert c[1][1] == 0 and c[1][7] == 0          # in_plane, out_plane: single-plane fp16
        if c[0] == "fgt_im2col_nchw":
            assert c[1][-2] == 0                          # out_plane
    assert sum(c[0] == "fgt_upsample2x" for c in c16) == 4
    assert [c[1][10] for c in c16 if c[0] == "fgt_im2col_nchw"] == [1, 0]   # replicate: e2a1 yes, edge_p no


def test_command_line_option_and_load_models(monkeypatch):
    from fgt_b200 import pipeline
    base = ["--path", "frames", "--path_mask", "masks", "--outroot", "out"]
    assert pipeline.arg_parser().parse_args(base).lafc_mixed_precision is False
    ns = pipeline.arg_parser().parse_args(base + ["--lafc_mixed_precision"])
    assert (ns.lafc_mixed_precision, ns.mixed_precision, ns.fgt_mixed_precision) == (True, False, False)
    seen = {}

    def fake_load(raft_model, lafc_ckpts, fgt_ckpts, device, mixed_precision=False, fgt_mixed_precision=False,
                  lafc_mixed_precision=False):
        seen.update(v=(mixed_precision, fgt_mixed_precision, lafc_mixed_precision))
        raise _Stop

    monkeypatch.setattr(pipeline, "load_models", fake_load)
    for argv, want in (([], (False, False, False)), (["--lafc_mixed_precision"], (False, False, True)),
                       (["--mixed_precision", "--fgt_mixed_precision", "--lafc_mixed_precision"], (True, True, True)),
                       (["--fgt_mixed_precision"], (False, True, False))):
        with pytest.raises(_Stop):
            pipeline.main(base + argv)
        assert seen.pop("v") == want
    assert "lafc_mixed_precision" not in pipeline.DEFAULTS
    with pytest.raises(TypeError):
        pipeline.make_args(lafc_mixed_precision=True)


def test_load_models_sets_the_switch(tmp_path, monkeypatch):
    """load_models(..., lafc_mixed_precision=...) reaches the LAFC module, and nothing else turns it on (the backend,
    which needs a GPU, is replaced by a record of the modules it receives)."""
    import yaml

    from fgt_b200 import pipeline
    lafc_dir, fgt_dir = tmp_path / "lafc", tmp_path / "fgt"
    lafc_dir.mkdir()
    fgt_dir.mkdir()
    torch.save({"model_state_dict": _sd()}, lafc_dir / "lafc.tar")
    (lafc_dir / "lafc.yaml").write_text(yaml.safe_dump(synth.CFG_LAFC))
    fcfg = dict(synth.CFG_A)
    fcfg["input_resolution"] = (64, 96)
    torch.save({"model_state_dict": synth.make_state_dict(synth.fgt_param_shapes(fcfg), seed=1)}, fgt_dir / "fgt.tar")
    (fgt_dir / "fgt.yaml").write_text(yaml.safe_dump({k: list(v) if isinstance(v, tuple) else v
                                                      for k, v in fcfg.items()}))
    raft_path = tmp_path / "raft.pth"
    torch.save({"module." + k: v for k, v in synth.raft_state_dict(seed=3).items()}, raft_path)
    monkeypatch.setattr(pipeline, "GpuBackend", lambda raft, lafc, fgt, device=None: SimpleNamespace(lafc=lafc, fgt=fgt))
    for flag in (False, True):
        backend, cfg = pipeline.load_models(str(raft_path), str(lafc_dir), str(fgt_dir), torch.device("cpu"),
                                            lafc_mixed_precision=flag)
        assert backend.lafc.net._mixed is flag and cfg["num_flows"] == 3
        assert backend.fgt.net._mixed is False
    backend, _ = pipeline.load_models(str(raft_path), str(lafc_dir), str(fgt_dir), torch.device("cpu"),
                                      fgt_mixed_precision=True)
    assert backend.lafc.net._mixed is False


def test_c_abi_rejects_mixed_upsample_planes_without_touching_the_gpu():
    L = lib.load()
    one = ctypes.c_void_p(64)
    for ip, op in ((0, 4096), (4096, 0), (-8, -8)):
        assert L.fgt_upsample2x(one, ip, 1, 4, 4, 16, one, op, None) == -1
        assert "plane offsets" in L.fgt_last_error().decode()
