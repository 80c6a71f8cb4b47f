"""Flow colour coding (RAFT/utils/flow_viz.py flow_to_image; fgt_b200/flowviz.py, csrc/flowviz.cu) and the driver's
visualisation switches of `python -m fgt_b200.pipeline` (CPU).

tests/golden/flowviz.npz holds the reference's own images of the flows below (tests/golden/make_flowviz_golden.py).
The oracle must equal them within one level, on at least 99.99 % of the values, and exactly on the cases whose angles
are exact (zero, axis-aligned and diagonal vectors): numpy's float32 arctan2 is SIMD code that depends on the host, and
an ulp of the angle can move a value by one level."""
import os

import cv2
import numpy as np
import pytest
from PIL import Image

from fgt_b200 import io as IO
from fgt_b200 import pipeline as PL
from fgt_b200 import synth
from oracle import flowviz_oracle as FO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flowviz.npz")
F = np.float32
# a vector whose radius, once divided by itself (+1e-5, lost in rounding above 256), rounds one ulp above 1
ULP_ABOVE = (F(2877.9478), F(3761.4875))


def _zero():
    return np.zeros((1, 5, 7, 2), F)


def _one_pixel():
    f = _zero()
    f[0, 2, 3] = (-2.5, 0.0)
    return f


def _signed_zeros():
    """The sign of a zero component picks the wheel's end: for u > 0, v = -0 gives entry 54 and v = +0 entry 0."""
    z, n = F(0.0), F(-0.0)
    vals = [(2, z), (1, z), (1, n), (-1, z), (-1, n), (z, 1), (n, 1), (z, -1), (n, -1), (z, z), (n, z), (z, n), (n, n),
            (F(0.5), n), (F(-0.5), n), (n, F(-0.5))]
    return np.array(vals, F).reshape(1, 4, 4, 2)


def _axis_diag():
    dirs = [(1, 0), (0, 1), (-1, 0), (0, -1), (1, 1), (-1, 1), (-1, -1), (1, -1)]
    mags = [0.25, 0.5, 1.0, 2.0]
    return np.array([[(m * dx, m * dy) for dx, dy in dirs] for m in mags], F)[None]


def _radius_one():
    """Image 0: (1024, 0) normalises to exactly (1, 0), radius 1 (the `rad <= 1` branch). Image 1: ULP_ABOVE normalises
    to radius 1 + 2^-23 (the `* 0.75` branch). Both images also hold a small vector."""
    f = np.array([[[(1024, 0), (3, 4)]], [[ULP_ABOVE, (0.5, 0.5)]]], F)
    for b, want in ((0, 1.0), (1, np.nextafter(F(1), F(2)))):
        r = np.sqrt(np.square(f[b, ..., 0]) + np.square(f[b, ..., 1]))
        d = r.max() + F(1e-5)
        u, v = f[b, 0, 0] / d
        assert np.sqrt(u * u + v * v) == want
    return f


def _huge():
    """Components of 1e30 square to Inf in float32: the maximum is Inf, every vector normalises to a signed zero."""
    return np.array([[(1e30, 0), (-1e30, 1e30), (3e38, -3e38), (1.0, -2.0)],
                     [(0.0, -1e30), (-7.0, 0.0), (1e-30, 5.0), (-0.0, -0.0)]], F)[None]


def _maxima():
    f = synth.vis_flows(21, 3, 9, 13)
    return f * np.array([0.01, 1.0, 300.0], F)[:, None, None, None]


CASES = {
    # name: (flows [B,H,W,2], exact angles)
    "synth": (lambda: synth.vis_flows(7, 4, 48, 64), False),
    "zero": (_zero, True),
    "one_pixel": (_one_pixel, True),
    "signed_zeros": (_signed_zeros, True),
    "axis_diag": (_axis_diag, True),
    "radius_one": (_radius_one, False),
    "huge": (_huge, False),
    "maxima": (_maxima, False),
    "shape_1x1": (lambda: synth.vis_flows(31, 2, 1, 1), False),
    "shape_1xW": (lambda: synth.vis_flows(32, 2, 1, 37), False),
    "shape_7x5": (lambda: synth.vis_flows(33, 2, 7, 5), False),
}


def golden():
    g = np.load(GOLDEN)
    return {name: (g[f"{name}/flows"], g[f"{name}/rgb"], g[f"{name}/bgr"]) for name in CASES}


def check_images(got, ref, exact, what):
    """Within one level everywhere, identical on >= 99.99 % of the values, identical everywhere when `exact`."""
    assert got.shape == ref.shape and got.dtype == np.uint8, (what, got.shape, ref.shape, got.dtype)
    d = np.abs(got.astype(np.int16) - ref.astype(np.int16))
    assert d.max() <= 1, (what, int(d.max()))
    assert (d != 0).mean() <= 1e-4, (what, int((d != 0).sum()), d.size)
    if exact:
        assert (d == 0).all(), (what, int((d != 0).sum()))


def test_golden_flows_are_the_cases():
    """The stored flows are what CASES generates here (so the GPU tests colour the same inputs)."""
    for name, (flows, rgb, bgr) in golden().items():
        assert np.array_equal(flows.view(np.uint32), CASES[name][0]().view(np.uint32)), name
        assert np.array_equal(bgr, rgb[..., ::-1]), name


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_golden(name):
    flows, rgb, bgr = golden()[name]
    exact = CASES[name][1]
    check_images(FO.flow_images(flows), rgb, exact, name)
    check_images(FO.flow_images(flows, convert_to_bgr=True), bgr, exact, name)


def test_oracle_edge_semantics():
    z = FO.flow_to_image(_zero()[0])
    assert (z == 255).all()                                   # radius 0 -> white
    sz = FO.flow_to_image(_signed_zeros()[0]).reshape(16, 3)
    # u > 0, v = +0 -> entry 0; v = -0 -> entry 54; both at radius 1 / (2 + 1e-5) (1 - rad * (1 - w / 255))
    rad = np.float64(F(1) / (F(2) + F(1e-5)))
    blend = lambda k: np.floor(255 * (1 - rad * (1 - FO.WHEEL[k] / 255.0))).astype(np.uint8)
    assert np.array_equal(sz[1], blend(0)) and np.array_equal(sz[2], blend(54)) and not np.array_equal(sz[1], sz[2])
    assert FO.WHEEL[54].tolist() == [255, 0, 43] and FO.WHEEL[0].tolist() == [255, 0, 0]
    with pytest.raises(ValueError, match="NaN or Inf"):
        FO.flow_to_image(np.array([[[np.nan, 0]]], F))
    with pytest.raises(ValueError, match="NaN or Inf"):
        FO.flow_to_image(np.array([[[1, np.inf]]], F))


def test_host_api_refusals_without_a_gpu():
    from fgt_b200 import flowviz
    with pytest.raises(TypeError, match="float32"):
        flowviz.flow_to_image(np.zeros((4, 4, 2)))
    with pytest.raises(ValueError, match=r"\[H,W,2\]"):
        flowviz.flow_to_image(np.zeros((4, 4, 3), F))
    with pytest.raises(ValueError, match="empty"):
        flowviz.flow_to_image(np.zeros((0, 4, 4, 2), F))
    with pytest.raises(RuntimeError, match="CUDA"):
        flowviz.flow_to_image(np.zeros((4, 4, 2), F), device="cpu")


# ------------------------------------------------------------------------------------------------ command line
class _OracleColours:
    """Backend stand-in: only what the visualisation writers use, coloured by the oracle; counts the calls."""

    def __init__(self):
        self.calls = []

    def flow_images(self, flows, convert_to_bgr=False):
        self.calls.append(flows.shape)
        return FO.flow_images(flows, convert_to_bgr)


def _stages(N=4, H=12, W=16):
    g = np.random.default_rng(5)
    fl = lambda seed: np.moveaxis(synth.vis_flows(seed, N - 1, H, W), 0, -1)            # [H,W,2,N-1]
    frames = [g.random((H, W, 3)) if i % 2 == 0 else g.random((H, W, 3)).astype(F) for i in range(N)]
    frames[0][0, 0] = [0.5 / 255, 1.5 / 255, 2.5 / 255]                                 # cv2's rounding ties
    masks = g.random((H, W, N)) < 0.2
    return dict(flow_f=fl(1), flow_b=fl(2), done_f=fl(3), done_b=fl(4), prop_frames=frames, masks_left=masks)


def _run_cli(monkeypatch, outroot, switches, vis, backend):
    comp = [np.full((12, 16, 3), 17 * i, np.uint8) for i in range(4)]

    def fake_video_inpainting(frames, masks, be, args, num_flows, flow_interval, native=False, vis_out=None):
        assert be is backend
        if vis_out is not None:
            vis_out.update(vis)
        return comp

    monkeypatch.setattr(PL, "load_models", lambda *a, **k: (backend, {"num_flows": 3, "flow_interval": 3}))
    monkeypatch.setattr(PL, "video_inpainting", fake_video_inpainting)
    monkeypatch.setattr(IO, "read_frames", lambda d: [np.zeros((12, 16, 3), np.uint8)] * 4)
    monkeypatch.setattr(IO, "read_masks", lambda d, rgb=False: [np.zeros((12, 16), np.uint8)] * 4)
    PL.main(["--path", "frames", "--path_mask", "masks", "--outroot", str(outroot)] + switches)


def _tree(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


def test_command_line_writes_the_driver_tree(tmp_path, monkeypatch):
    vis, be = _stages(), _OracleColours()
    out = tmp_path / "vis"
    _run_cli(monkeypatch, out, ["--vis_flows", "--vis_completed_flows", "--vis_prop", "--vis_frame"], vis, be)
    n = 3
    want = [f"frames/{i:05d}.png" for i in range(4)]
    for sub in ("flow", "completed_flow"):
        for mode in ("forward", "backward"):
            want += [f"{sub}/{mode}_flo/{i:05d}.flo" for i in range(n)] + [f"{sub}/{mode}_png/{i:05d}.png" for i in range(n)]
    for d, ext in (("prop_frames", "png"), ("masks_left", "png"), ("prop_frames_npy", "npy"), ("masks_left_npy", "npy")):
        want += [f"{d}/{i:05d}.{ext}" for i in range(4)]
    got = [p for p in _tree(out) if p != "result.mp4"]
    assert got == sorted(want)
    assert be.calls == [(n, 12, 16, 2)] * 4                  # one batched colouring per flow set
    for sub, (kf, kb) in (("flow", ("flow_f", "flow_b")), ("completed_flow", ("done_f", "done_b"))):
        for mode, key in (("forward", kf), ("backward", kb)):
            for i in range(n):
                flow = vis[key][..., i]
                back = IO.read_flo(str(out / sub / f"{mode}_flo" / f"{i:05d}.flo"))
                assert np.array_equal(back.view(np.uint32), np.ascontiguousarray(flow).view(np.uint32))
                png = Image.open(out / sub / f"{mode}_png" / f"{i:05d}.png")
                assert png.mode == "RGB" and np.array_equal(np.array(png), FO.flow_to_image(flow))
    for i, fr in enumerate(vis["prop_frames"]):
        for d, arr in (("prop_frames", fr * 255.0), ("masks_left", vis["masks_left"][:, :, i] * 255.0)):
            ok, enc = cv2.imencode(".png", arr)
            assert ok and (out / d / f"{i:05d}.png").read_bytes() == enc.tobytes()
            npy = np.load(out / f"{d}_npy" / f"{i:05d}.npy")
            assert npy.dtype == arr.dtype and np.array_equal(npy, arr)
        assert np.load(out / "prop_frames_npy" / f"{i:05d}.npy").dtype == (np.float64 if i % 2 == 0 else np.float32)
    assert cv2.imread(str(out / "prop_frames" / "00000.png"))[0, 0].tolist() == [0, 2, 2]   # half to even, as cv2 rounds


def test_command_line_without_switches_writes_what_it_always_wrote(tmp_path, monkeypatch):
    vis, be = _stages(), _OracleColours()
    _run_cli(monkeypatch, tmp_path / "plain", [], vis, be)
    _run_cli(monkeypatch, tmp_path / "frame", ["--vis_frame"], vis, be)
    ref = tmp_path / "ref"
    IO.write_frames(str(ref), [np.full((12, 16, 3), 17 * i, np.uint8) for i in range(4)])
    for d in ("plain", "frame"):
        assert _tree(tmp_path / d) == _tree(ref)
        for p in _tree(ref):
            assert (tmp_path / d / p).read_bytes() == (ref / p).read_bytes(), (d, p)
    assert be.calls == []


def test_switches_parse():
    base = ["--path", "f", "--outroot", "o"]
    ns = PL.arg_parser().parse_args(base)
    assert not (ns.vis_flows or ns.vis_completed_flows or ns.vis_prop or ns.vis_frame)
    ns = PL.arg_parser().parse_args(base + ["--vis_flows", "--vis_completed_flows", "--vis_prop", "--vis_frame"])
    assert ns.vis_flows and ns.vis_completed_flows and ns.vis_prop and ns.vis_frame


def test_vis_out_holds_the_driver_stages_with_per_frame_dtypes():
    """video_inpainting(..., vis_out=...) on the (deterministic) oracle backend: the flows and frames the switches
    write, the propagated frames with the driver's per-frame dtypes, and the same result as without it."""
    from oracle import fgt_oracle as O
    from oracle.pipeline_oracle import OracleBackend
    from tests.test_pipeline import _setup
    _, _, frames, masks, args, _, sds = _setup()
    masks = [np.asarray(m).copy() for m in masks]
    masks[1][:] = 0                                            # a frame without a hole is not blended
    be = OracleBackend(sds["raft"], O.strip_net(sds["lafc"]), O.strip_net(sds["fgt"]))
    vis = {}
    comp, st = PL.video_inpainting(frames, masks, be, args, return_stages=True, vis_out=vis)
    plain = PL.video_inpainting(frames, masks, be, args)
    assert all(np.array_equal(a, b) for a, b in zip(comp, plain)) and len(comp) == len(plain)
    for k in ("flow_f", "flow_b", "done_f", "done_b"):
        assert np.array_equal(vis[k], st[k]), k
    assert [f.dtype for f in vis["prop_frames"]] == [np.float64, np.float32] + [np.float64] * (len(frames) - 2)
    assert np.array_equal(np.stack(vis["prop_frames"]), st["frame_blends"])
    assert np.array_equal(vis["masks_left"], st["mask"])
