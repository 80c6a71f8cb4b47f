"""FGT's validation (fgt_b200.validate) on the CPU: the host steps of the module and of oracle/validate_oracle.py
against what the unmodified network.py methods returned on the seeded mini validation set
(tests/golden/validate_golden.npz) — bit for bit for the frame set, frames, masks and flows, at the regionfill tolerance
for the diffusion — and the command line: parsing, checkpoint directories, --limit and the report of skipped videos."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from fgt_b200 import synth
from fgt_b200 import validate as V
from oracle import validate_oracle as VO
from tests.util import load_golden


def digest(a):
    """Bit-for-bit fingerprint of an array: its dtype, shape and the SHA-256 of its bytes."""
    a = np.ascontiguousarray(a)
    return f"{a.dtype.str}{a.shape}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def sample_idx(n, k=4096):
    """The flat indices of the seeded samples validate_golden.npz stores of an n-element array."""
    return torch.randperm(n, generator=torch.Generator().manual_seed(1234))[:k]


def same(a, g, key):
    """a equals the array whose digest the golden stores under key + '_sha', bit for bit."""
    return digest(a) == str(g[key + "_sha"])


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    g = load_golden("validate_golden")
    root = tmp_path_factory.mktemp("valid")
    return g, synth.validation_set(str(root), seed=g["meta"]["seed"])


def _dirs(roots, name):
    return [os.path.join(r, name) for r in roots]


def test_frame_set_order_and_clamp(dataset):
    g, roots = dataset
    assert V.frame_ids(45) == list(g["vid_a_ids"]) == VO.ref_ids(45) == [0, 10, 30, 40, 18, 19, 20, 21]
    assert V.frame_ids(41) == list(g["vid_b_ids"])
    assert V.frame_ids(25) == [0, 10, 18, 19, 20, 21]
    assert V.frame_ids(19) == [0, 10, 18]                                # neighbours cut at the video's end
    fl = _dirs(roots, "vid_b")[2]
    names = [os.path.basename(p) for p in V.flow_files(fl, V.frame_ids(41), 41)]
    assert names[3] == "00039.flo"                                       # id 40 clamped to L - 2
    back = V.flow_files(fl, V.frame_ids(41), 41, "back")
    assert os.path.basename(back[0]) == "00000.flo" and "backward_flo" in back[0]
    with pytest.raises(NotImplementedError):
        V.flow_files(fl, [0], 41, "bi")
    with pytest.raises(ValueError, match="Unknown"):
        V.flow_files(fl, [0], 41, "sideways")


def test_frames_and_masks_bit_for_bit(dataset):
    g, roots = dataset
    fr, mk, _ = _dirs(roots, "vid_a")
    ids = list(g["vid_a_ids"])
    H, W = g["meta"]["H"], g["meta"]["W"]
    for frames in (V.read_frames(fr, W, H, ids), np.stack(VO.read_frames(fr, W, H, ids))):
        assert same(frames, g, "vid_a_frames")
    oracle_masks = np.stack(VO.read_masks(mk, W, H, ids))[..., 0]
    assert set(np.unique(oracle_masks)) <= {0.0, 1.0}
    for masks in (V.read_masks(mk, W, H, ids), oracle_masks.astype(np.uint8)):
        assert same(masks, g, "vid_a_masks")
    masks = V.read_masks(mk, W, H, ids)
    # the bilinear-then->0 mask is wider than a nearest resize of the same mask
    import cv2
    paths = sorted(os.listdir(mk))
    near = cv2.resize(cv2.imread(os.path.join(mk, paths[ids[0]]), 0), (W, H), interpolation=cv2.INTER_NEAREST) > 0
    assert masks[0].sum() > near.sum() and (masks[0] >= near).all()


def test_short_video_is_skipped(dataset):
    g, roots = dataset
    fr, mk, _ = _dirs(roots, "vid_short")
    assert int(g["short_frames_len"]) == 0 and VO.read_frames(fr, 96, 64, [0]) == []
    with pytest.raises(V.SkipVideo, match="30"):
        V.read_frames(fr, 96, 64, [0])
    with pytest.raises(V.SkipVideo, match="30"):
        V.read_masks(mk, 96, 64, [0])


@pytest.mark.parametrize("video,direction", [("vid_a", "for"), ("vid_b", "for"), ("vid_b", "back")])
def test_oracle_flows_bit_for_bit(dataset, video, direction):
    g, roots = dataset
    key = f"{video}_back_flows" if direction == "back" else f"{video}_flows"
    ids = list(g[f"{video}_ids"])
    L = {"vid_a": 45, "vid_b": 41}[video]
    got = np.stack(VO.read_flows(_dirs(roots, video)[2], g["meta"]["W"], g["meta"]["H"], ids, L - 1, direction))
    assert same(got, g, key)


def test_oracle_diffusion(dataset):
    """regionfill_oracle on the reference's flows and masks gives the reference's diffused flows (float32, as
    _validate hands them on) bit for bit."""
    g, roots = dataset
    fr, mk, fd = _dirs(roots, "vid_a")
    ids, H, W = list(g["vid_a_ids"]), g["meta"]["H"], g["meta"]["W"]
    fl = np.stack(VO.read_flows(fd, W, H, ids, 45 - 1))
    m = np.stack(VO.read_masks(mk, W, H, ids))[..., 0]
    assert same(fl, g, "vid_a_flows")
    from oracle import regionfill_oracle
    d = np.stack([np.stack([regionfill_oracle.regionfill(fl[i, :, :, c] * (1 - m[i]), m[i]) for c in range(2)], -1)
                  for i in range(len(fl))])
    assert same(d.astype(np.float32), g, "vid_a_diffused")
    val = d.transpose(0, 3, 1, 2).reshape(-1)[sample_idx(d.size).numpy()]
    assert np.abs(val - g["vid_a_diffused_val"]).max() <= 1e-6 * np.abs(val).max()


def test_as_png_u8_follows_imageio():
    c = np.zeros((2, 3, 3))
    c[0, 0] = 255.0
    c[1, 2] = 127.4
    u = V._as_png_u8(c)
    assert u[0, 0, 0] == 255 and u[1, 2, 0] == 127 and u[0, 1, 0] == 0
    assert np.array_equal(V._as_png_u8(np.full((2, 2, 3), 0.5)), np.full((2, 2, 3), 127, np.uint8))   # 127.5 + 0.499999999


def test_vis_canvas_layout_matches_reference(dataset):
    """vis_frames' canvas of the first frame of vid_a, rebuilt by write_vis from the reference's FGT output of that
    frame and the frames and masks as read here."""
    import tempfile
    from PIL import Image
    g, roots = dataset
    fdir, mdir, _ = _dirs(roots, "vid_a")
    ids, H, W = list(g["vid_a_ids"])[:1], g["meta"]["H"], g["meta"]["W"]
    fr = torch.from_numpy(V.read_frames(fdir, W, H, ids)).permute(0, 3, 1, 2).float() / 127.5 - 1
    m = torch.from_numpy(V.read_masks(mdir, W, H, ids)).float()[:, None]
    out = torch.from_numpy(g["vid_a_out0"])[None]
    with tempfile.TemporaryDirectory() as d:
        V.write_vis(d, out, m, fr, fr * (1 - m))
        got = np.asarray(Image.open(os.path.join(d, "result_compare_00000.png")))
    assert np.array_equal(got, V._as_png_u8(g["vid_a_vis0"].astype(np.float64)))


# ------------------------------------------------------------------------------------------------ command line
def test_command_line_parses():
    base = ["--frame_root", "f", "--mask_root", "m", "--flow_root", "fl", "--flow_ckpt", "a", "--fgt_ckpts", "b"]
    ns = V.arg_parser().parse_args(base)
    assert (ns.width, ns.height, ns.num_frames, ns.ref_length, ns.pivot, ns.flow_direction, ns.limit, ns.vis_dir,
            ns.gpu) == (432, 240, 5, 10, 20, "for", None, None, 0)
    ns = V.arg_parser().parse_args(base + ["--limit", "10", "--flow_direction", "back", "--gpu", "1"])
    assert (ns.limit, ns.flow_direction, ns.gpu) == (10, "back", 1)
    with pytest.raises(SystemExit):
        V.arg_parser().parse_args(base + ["--flow_direction", "sideways"])
    with pytest.raises(NotImplementedError):
        V.main(base + ["--flow_direction", "bi"])
    assert "--limit 10 reproduces" in " ".join(V.arg_parser().format_help().split())


def test_checkpoint_directories(tmp_path):
    import yaml
    from fgt_b200.pipeline import load_ckpt_dir
    d = tmp_path / "lafc"
    d.mkdir()
    sd = synth.lafc_single_state_dict(seed=2)
    torch.save({"model_state_dict": sd}, d / "lafc.pth.tar")
    (d / "train_single.yaml").write_text(yaml.safe_dump(synth.CFG_LAFC_SINGLE))
    got_sd, cfg = load_ckpt_dir(str(d))
    assert cfg == synth.CFG_LAFC_SINGLE and set(got_sd) == set(sd)
    from fgt_b200.lafc_single import Model
    Model(cfg).load_state_dict(got_sd)
    (d / "other.yaml").write_text("a: 1")
    with pytest.raises(FileNotFoundError, match="exactly one"):
        load_ckpt_dir(str(d))


def test_validate_applies_limit_and_reports_skipped(dataset, monkeypatch):
    g, roots = dataset
    seen = []

    def fake(lafc, fgt, frame_dir, mask_dir, flow_dir, **kw):
        seen.append(os.path.basename(flow_dir))
        V.read_frames(frame_dir, 96, 64, [0])
        V.read_masks(mask_dir, 96, 64, [0])
        return dict(l1=1.0, l2=2.0, psnr=30.0 + len(seen), ssim=0.5, frames=8)

    monkeypatch.setattr(V, "validate_video", fake)
    res = V.validate(None, None, *roots)
    assert seen == ["vid_a", "vid_b", "vid_short"]
    assert sorted(res["videos"]) == ["vid_a", "vid_b"] and list(res["skipped"]) == ["vid_short"]
    assert "30" in res["skipped"]["vid_short"] and res["mean"]["psnr"] == 31.5
    json.dumps(res)
    seen.clear()
    res = V.validate(None, None, *roots, limit=1)
    assert seen == ["vid_a"] and list(res["videos"]) == ["vid_a"] and res["skipped"] == {}
