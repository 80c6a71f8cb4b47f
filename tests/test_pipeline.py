"""Whole driver pipeline (tool/video_inpainting.py::video_inpainting, object removal) behind
fgt_b200.pipeline.video_inpainting — SURVEY §8f rank 3.

Goldens (tests/golden/pipeline_*.npz) come from ONE RUN OF THE UNMODIFIED REFERENCE DRIVER on the CPU
(tests/golden/make_pipeline_golden.py; seeded synthetic RAFT / LAFC / FGT weights, 7 frames of 64x96).
* CPU: the pipeline glue with the CPU oracle backend must reproduce the driver's stage outputs (flows to fp16
  storage precision, propagation mask exactly) and final frames (<= 1 level on < 0.1 % of the values).
* GPU: the same glue with the CUDA backend. The stages are chaotic in places (RAFT's 20 recurrent iterations with
  synthetic weights, hard consistency thresholds in the propagation), so 1e-4-level differences of the CUDA networks can
  move individual pixels across a threshold; the test therefore checks the stage outputs statistically (stated per
  assertion) and the final frames by mean absolute error and the fraction of values off by more than 2 levels."""
import os

import numpy as np
import pytest
import torch

from fgt_b200 import pipeline as PL
from fgt_b200 import synth
from oracle import fgt_oracle as O
from tests.util import load_golden


def _setup():
    g = load_golden("pipeline_clip")
    st = load_golden("pipeline_stages")
    m = g["meta"]
    frames, masks = synth.pipeline_clip(seed=m["clip_seed"], N=m["N"], H=m["H"], W=m["W"])
    args = PL.make_args(imgH=m["H"], imgW=m["W"], flow_mask_dilates=m["flow_mask_dilates"], frame_dilates=m["frame_dilates"])
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (m["H"], m["W"])
    sds = dict(fgt=synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=m["fgt_seed"]),
               lafc=synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=m["lafc_seed"]),
               raft=synth.raft_state_dict(seed=m["raft_seed"]))
    n = m["N"] * m["H"] * m["W"]
    st["mask_gradient"] = np.unpackbits(st["mask_gradient"])[:n].reshape(m["H"], m["W"], m["N"]).astype(bool)
    return g, st, frames, masks, args, cfg, sds


def test_helpers():
    assert PL.indices_gen(0, 3, 3, 6) == [3, 0, 3] and PL.indices_gen(5, 3, 3, 6) == [2, 5, 2]
    assert PL.indices_gen(2, 3, 3, 6) == [1, 2, 5]
    m = np.zeros((5, 6), bool); m[2, 3] = True
    gm = PL.gradient_mask(m)
    assert gm.sum() == 3 and gm[2, 3] and gm[1, 3] and gm[2, 2]
    with pytest.raises(TypeError):
        PL.make_args(bogus=1)


def test_pipeline_glue_with_oracle_backend_matches_reference_driver():
    from oracle.pipeline_oracle import OracleBackend
    g, st, frames, masks, args, cfg, sds = _setup()
    be = OracleBackend(sds["raft"], O.strip_net(sds["lafc"]), O.strip_net(sds["fgt"]))
    comp, stages = PL.video_inpainting(frames, masks, be, args, return_stages=True)
    for k in ("flow_f", "flow_b", "done_f", "done_b"):
        ref = st[k].astype(np.float32)
        assert np.abs(stages[k] - ref).max() <= 2e-2 + 1e-3 * np.abs(ref).max(), k      # fp16 storage of the golden
    assert np.abs(stages["done_f"] - np.moveaxis(g["flow_f"], 0, -1)).max() < 1e-3         # float32 golden of the FGT stage
    assert np.array_equal(np.asarray(stages["mask_gradient"], bool), st["mask_gradient"])
    assert np.abs(stages["frame_blends"][..., ::-1] - g["frames_rgb"]).max() < 1e-4
    comp = np.stack(comp)
    diff = np.abs(comp.astype(np.int16) - g["comp"].astype(np.int16))
    assert comp.dtype == np.uint8 and diff.max() <= 1 and (diff != 0).mean() < 1e-3, (diff.max(), (diff != 0).mean())


@pytest.mark.gpu
def test_gpu_pipeline_vs_reference_driver():
    from fgt_b200.fgt_model import Model as FGTModel
    from fgt_b200.lafc_model import Model as LAFCModel
    from fgt_b200.raft_model import RAFT
    import argparse
    g, st, frames, masks, args, cfg, sds = _setup()
    dev = torch.device("cuda:0")
    fgt = FGTModel(cfg); fgt.load_state_dict(sds["fgt"]); fgt = fgt.to(dev)
    lafc = LAFCModel(dict(synth.CFG_LAFC)); lafc.load_state_dict(sds["lafc"]); lafc = lafc.to(dev)
    raft = RAFT(argparse.Namespace(small=False, mixed_precision=False, alternate_corr=False))
    raft.load_state_dict(sds["raft"]); raft = raft.to(dev).eval()
    be = PL.GpuBackend(raft, lafc, fgt, device=dev)
    comp, stages = PL.video_inpainting(frames, masks, be, args, return_stages=True)
    rep = {}
    for k in ("flow_f", "flow_b", "done_f", "done_b"):
        ref = st[k].astype(np.float32)
        err = np.abs(stages[k] - ref)
        rep[k] = (float(err.mean()), float(err.max()), float(np.abs(ref).mean()))
    mg = np.asarray(stages["mask_gradient"], bool)
    rep["mask_gradient_mismatch"] = float((mg != st["mask_gradient"]).mean())
    comp = np.stack(comp)
    diff = np.abs(comp.astype(np.int16) - g["comp"].astype(np.int16))
    rep["comp"] = (float(diff.mean()), int(diff.max()), float((diff > 2).mean()))
    print("pipeline parity report:", rep)
    assert comp.shape == g["comp"].shape and comp.dtype == np.uint8
    hole0 = np.stack([np.asarray(m) != 0 for m in masks])                          # untouched where nothing was ever removed
    import scipy.ndimage
    far = ~np.stack([scipy.ndimage.binary_dilation(h, iterations=args.frame_dilates) for h in hole0])
    assert (comp[far] == g["comp"][far]).all()
    # bounds: flow error relative to the mean flow magnitude (incl. the golden's fp16 storage), propagation mask
    # identical, final frames within 1 level
    for k in ("flow_f", "flow_b", "done_f", "done_b"):
        assert rep[k][0] < 2e-3 * rep[k][2] and rep[k][1] < 1e-2 * rep[k][2], (k, rep[k])
    assert rep["mask_gradient_mismatch"] < 1e-3, rep
    assert rep["comp"][0] < 0.05 and rep["comp"][1] <= 8 and rep["comp"][2] < 1e-3, rep


def _write_ckpts(tmp, cfg, sds):
    import yaml
    os.makedirs(os.path.join(tmp, "fgt")); os.makedirs(os.path.join(tmp, "lafc"))
    torch.save({"model_state_dict": sds["fgt"]}, os.path.join(tmp, "fgt", "fgt.tar"))
    with open(os.path.join(tmp, "fgt", "config.yaml"), "w") as fh:
        yaml.safe_dump({**{k: (list(v) if isinstance(v, tuple) else v) for k, v in cfg.items()}, "model": "model"}, fh)
    torch.save({"model_state_dict": sds["lafc"]}, os.path.join(tmp, "lafc", "lafc.tar"))
    with open(os.path.join(tmp, "lafc", "config.yaml"), "w") as fh:
        yaml.safe_dump(dict(synth.CFG_LAFC), fh)
    torch.save({"module." + k: v for k, v in sds["raft"].items()}, os.path.join(tmp, "raft.pth"))


def test_cli_argument_and_checkpoint_errors(tmp_path):
    with pytest.raises(SystemExit):
        PL.main(["--path", "x"])                                        # required options missing
    os.makedirs(tmp_path / "empty")
    with pytest.raises(FileNotFoundError):
        PL.load_models(str(tmp_path / "nope.pth"), str(tmp_path / "empty"), str(tmp_path / "empty"), "cpu")


@pytest.mark.gpu
def test_gpu_command_line_end_to_end(tmp_path):
    """The driver's command line on directories of PNGs with checkpoints in the driver's layout; same frames as the
    array entry point (and therefore as the reference driver's golden)."""
    from fgt_b200 import io as IO
    g, st, frames, masks, args, cfg, sds = _setup()
    tmp = str(tmp_path)
    _write_ckpts(tmp, cfg, sds)
    IO.write_frames(os.path.join(tmp, "in"), frames, mp4=False)
    IO.write_frames(os.path.join(tmp, "msk"), [np.repeat(m[..., None], 3, -1) for m in masks], mp4=False)
    comp = PL.main(["--path", os.path.join(tmp, "in", "frames"), "--path_mask", os.path.join(tmp, "msk", "frames"),
                    "--outroot", os.path.join(tmp, "out"), "--raft_model", os.path.join(tmp, "raft.pth"),
                    "--lafc_ckpts", os.path.join(tmp, "lafc"), "--fgt_ckpts", os.path.join(tmp, "fgt"),
                    "--imgH", str(args.imgH), "--imgW", str(args.imgW), "--flow_mask_dilates", str(args.flow_mask_dilates),
                    "--frame_dilates", str(args.frame_dilates)])
    back = IO.read_frames(os.path.join(tmp, "out", "frames"))
    assert len(back) == len(frames) and all(np.array_equal(a, b) for a, b in zip(back, comp))
    diff = np.abs(np.stack(comp).astype(np.int16) - g["comp"].astype(np.int16))
    assert diff.max() <= 8 and diff.mean() < 0.05


# ------------------------------------------------------------------------------------------------ multi-rank (gloo)
def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist
    from oracle.pipeline_oracle import OracleBackend
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.set_num_threads(4)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g, st, frames, masks, args, cfg, sds = _setup()
        inner = OracleBackend(sds["raft"], O.strip_net(sds["lafc"]), O.strip_net(sds["fgt"]))
        be = PL.ShardedBackend(inner)
        calls = {"raft": 0, "fgt": 0}
        raft0, fgt0 = inner.raft_pairs, inner.fgt_model
        inner.raft_pairs = lambda a, b, it: (calls.__setitem__("raft", calls["raft"] + a.shape[0]), raft0(a, b, it))[1]
        inner.fgt_model = lambda a, b, c: (calls.__setitem__("fgt", calls["fgt"] + 1), fgt0(a, b, c))[1]
        comp, stages = PL.video_inpainting(frames, masks, be, args, return_stages=True)
        assert inner.fgt_model is not None
        q.put((rank, np.stack(comp), stages["done_f"], np.asarray(stages["mask_gradient"], bool), dict(calls)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_pipeline_gloo_matches_reference_driver(world):
    """SURVEY 8e on the CPU: 2 or 3 ranks, every stage's items sharded + all-gathered; all ranks end with the frames of
    the unmodified reference driver, and each rank evaluated only its share of the RAFT pairs and FGT windows (with
    three ranks one of them owns no window at all, and the 7 Poisson frames split 3 + 2 + 2)."""
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    g = load_golden("pipeline_clip")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in procs], key=lambda r: r[0])
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    comp0, done0, mg0 = res[0][1:4]
    for _, comp, done, mg, _calls in res[1:]:
        assert np.array_equal(comp0, comp) and np.array_equal(done0, done) and np.array_equal(mg0, mg)
    diff = np.abs(comp0.astype(np.int16) - g["comp"].astype(np.int16))
    assert diff.max() <= 1 and (diff != 0).mean() < 1e-3
    assert np.abs(done0 - np.moveaxis(g["flow_f"], 0, -1)).max() < 1e-3
    calls = [r[4] for r in res]
    assert sum(c["raft"] for c in calls) == 12 and sum(c["fgt"] for c in calls) == 2      # 6 + 6 pairs, 2 windows
    assert max(c["raft"] for c in calls) == 12 // world and sorted(c["fgt"] for c in calls) == [0] * (world - 2) + [1, 1]


def test_pipeline_glue_second_reference_run_12_frames():
    """A second full run of the unmodified reference driver (tests/golden/pipeline12.npz): 12 frames -> three windows,
    frames composed from up to three visits (0.25 / 0.25 / 0.5), a reference frame outside the neighbourhood, no frame
    dilation (the uint8-mask branch of the driver), different seeds for all three networks."""
    from oracle.pipeline_oracle import OracleBackend
    g = load_golden("pipeline12")
    m = g["meta"]
    from fgt_b200.parallel import window_schedule
    assert m["N"] == 12 and [len(n) + len(r) for _, n, r in window_schedule(12)] == [7, 11, 8]
    frames, masks = synth.pipeline_clip(seed=m["clip_seed"], N=m["N"], H=m["H"], W=m["W"])
    args = PL.make_args(imgH=m["H"], imgW=m["W"], flow_mask_dilates=m["flow_mask_dilates"], frame_dilates=m["frame_dilates"])
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (m["H"], m["W"])
    be = OracleBackend(synth.raft_state_dict(seed=m["raft_seed"]),
                       O.strip_net(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=m["lafc_seed"])),
                       O.strip_net(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=m["fgt_seed"])))
    comp, stages = PL.video_inpainting(frames, masks, be, args, return_stages=True)
    n = m["N"] * m["H"] * m["W"]
    bits = lambda k: np.unpackbits(g[k])[:n]
    assert np.array_equal(np.asarray(stages["mask_gradient"], bool).reshape(-1), bits("mask_gradient").astype(bool))
    assert np.array_equal(np.moveaxis(stages["mask"], -1, 0).reshape(-1), bits("mask_final").astype(bool))
    diff = np.abs(np.stack(comp).astype(np.int16) - g["comp"].astype(np.int16))
    assert diff.max() <= 1 and (diff != 0).mean() < 1e-3, (diff.max(), (diff != 0).mean())


@pytest.mark.parametrize("name", ["pipeline_watermark", "pipeline_extrapolation"])
def test_pipeline_other_driver_modes_match_reference_runs(name):
    """The driver's two other modes, each pinned by its own full run of the unmodified reference driver: watermark
    removal (RGB mask files multiplied into the frames before any resizing, consistencyThres 1) and video extrapolation
    (a 64x96 clip on an 80x120 canvas whose TELEA-initialised border is the hole; FGT runs at the canvas size)."""
    from oracle.pipeline_oracle import OracleBackend
    g = load_golden(name)
    m = g["meta"]
    frames, masks = synth.pipeline_clip(seed=m["clip_seed"], N=m["N"], H=m["H"], W=m["W"])
    if m["mode"] == "watermark_removal":
        masks = [np.repeat(x[..., None], 3, -1) for x in masks]           # colour mask files, as the driver expects there
    args = PL.make_args(mode=m["mode"], imgH=m["H"], imgW=m["W"], flow_mask_dilates=m["flow_mask_dilates"],
                        frame_dilates=m["frame_dilates"], consistencyThres=m["consistencyThres"], H_scale=m["scale"],
                        W_scale=m["scale"])
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = tuple(m["cfg_hw"])
    be = OracleBackend(synth.raft_state_dict(seed=m["raft_seed"]),
                       O.strip_net(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=m["lafc_seed"])),
                       O.strip_net(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=m["fgt_seed"])))
    comp, stages = PL.video_inpainting(frames, None if m["mode"] == "video_extrapolation" else masks, be, args,
                                       return_stages=True)
    comp = np.stack(comp)
    assert comp.shape == g["comp"].shape
    n = comp.shape[0] * comp.shape[1] * comp.shape[2]
    bits = lambda k: np.unpackbits(g[k])[:n].astype(bool)
    assert np.array_equal(np.asarray(stages["mask_gradient"], bool).reshape(-1), bits("mask_gradient"))
    assert np.array_equal(np.moveaxis(stages["mask"], -1, 0).reshape(-1), bits("mask_final"))
    diff = np.abs(comp.astype(np.int16) - g["comp"].astype(np.int16))
    assert diff.max() <= 1 and (diff != 0).mean() < 1e-3, (diff.max(), (diff != 0).mean())
    with pytest.raises(ValueError):
        PL.video_inpainting(frames, masks, be, PL.make_args(mode="colourise"))
