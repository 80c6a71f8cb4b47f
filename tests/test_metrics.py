"""Quality metrics (fgt_b200/metrics.py, oracle/metrics_oracle.py) on the CPU: the oracle against the reference's own
psnr.py / ssim.py outputs (tests/golden/metrics.npz), and the host API's and the command line's refusals."""
import os

import numpy as np
import pytest
import torch

from fgt_b200 import lib, synth
from fgt_b200 import metrics as M
from oracle import metrics_oracle as MO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz")

# name: synth.metric_pair's (seed, N, H, W, C, kind, dtype).
CASES = {
    "noise_64x96x3_u8": (1, 3, 64, 96, 3, "noise", "u8"),
    "blur_64x96x3_f32": (2, 3, 64, 96, 3, "blur", "f32"),
    "same_64x96x3_u8": (3, 2, 64, 96, 3, "same", "u8"),
    "same_40x30x1_f32": (4, 2, 40, 30, 1, "same", "f32"),
    "min_11x11x3_u8": (5, 4, 11, 11, 3, "noise", "u8"),
    "min_11x11x1_f32": (6, 3, 11, 11, 1, "noise", "f32"),
    "odd_37x53x1_u8": (7, 3, 37, 53, 1, "blur", "u8"),
    "odd_45x71x3_f32": (8, 2, 45, 71, 3, "noise", "f32"),
    "driver_256x432x3_u8": (9, 3, 256, 432, 3, "noise", "u8"),
    "driver_256x432x3_f32": (10, 2, 256, 432, 3, "blur", "f32"),
}
KEYS = ("l1", "l2", "psnr", "ssim", "ssim_channels")
# Bound on |oracle - golden| / |golden| over every case and key. Measured: at most 3.5e-14, on the single-position SSIM
# of the 11x11 frames (the oracle's direct 11x11 sum against cv2.filter2D in ssim.py; elsewhere below 8e-15); L1, L2
# and PSNR are equal to the last bit.
ORACLE_GOLDEN_GAP = 1e-13


def case_inputs(name):
    return synth.metric_pair(*CASES[name])


def rel_err(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float(np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-300)))


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def test_golden_covers_every_case(golden):
    assert {k.split("/")[0] for k in golden} == set(CASES)
    for name, (_, N, _, _, C, _, _) in CASES.items():
        assert golden[f"{name}/ssim"].shape == (N,) and golden[f"{name}/ssim_channels"].shape == (N, C)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_golden(golden, name):
    res, gts = case_inputs(name)
    got = MO.clip_metrics(res, gts)
    for k in KEYS:
        assert rel_err(got["per_frame"][k], golden[f"{name}/{k}"]) <= ORACLE_GOLDEN_GAP, k
    for k in KEYS[:4]:
        assert got[k] == pytest.approx(float(np.mean(golden[f"{name}/{k}"])), rel=ORACLE_GOLDEN_GAP)
    if CASES[name][5] == "same":
        assert np.all(golden[f"{name}/psnr"] == 100) and np.all(golden[f"{name}/ssim"] == 1.0)
        assert np.all(got["per_frame"]["psnr"] == 100) and np.all(got["per_frame"]["ssim"] == 1.0)
        assert np.all(got["per_frame"]["l1"] == 0) and np.all(got["per_frame"]["l2"] == 0)


def test_inputs_are_what_the_cases_say():
    res, gts = case_inputs("same_64x96x3_u8")
    assert res.dtype == np.uint8 and np.array_equal(res, gts) and gts.min() == 0 and gts.max() == 255
    res, gts = case_inputs("noise_64x96x3_u8")
    assert 0 < np.abs(res.astype(int) - gts).max() <= 12
    res, gts = case_inputs("blur_64x96x3_f32")
    assert res.dtype == np.float32 and res.shape == (3, 64, 96, 3) and not np.array_equal(res, gts)


def test_oracle_refuses_what_the_reference_cannot_score():
    a = np.zeros((10, 20, 3), np.uint8)
    with pytest.raises(ValueError, match="11x11"):
        MO.frame_metrics(a, a)
    with pytest.raises(ValueError, match="shape"):
        MO.frame_metrics(np.zeros((20, 20, 3)), np.zeros((20, 21, 3)))
    with pytest.raises(ValueError, match="C = 1 or 3"):
        MO.frame_metrics(np.zeros((20, 20, 2)), np.zeros((20, 20, 2)))


def test_oracle_converts_uint8_before_subtracting():
    a, b = np.full((12, 12, 1), 10, np.uint8), np.full((12, 12, 1), 20, np.uint8)
    l1, l2, psnr, _, _ = MO.frame_metrics(a, b)
    assert l1 == 10.0 and l2 == pytest.approx(10.0 / 12) and psnr == pytest.approx(20 * np.log10(25.5))


@pytest.mark.parametrize("shape_a, shape_b, match", [
    ((2, 20, 20, 3), (2, 20, 21, 3), "one shape"),
    ((2, 20, 20, 3), (3, 20, 20, 3), "one shape"),
    ((20, 20, 3), (20, 20, 3), "one shape"),
    ((2, 20, 20, 2), (2, 20, 20, 2), "C = 1 or 3"),
    ((0, 20, 20, 3), (0, 20, 20, 3), "N >= 1"),
    ((2, 10, 20, 3), (2, 10, 20, 3), "11x11"),
    ((2, 20, 10, 1), (2, 20, 10, 1), "11x11"),
])
def test_host_api_refuses_bad_shapes(shape_a, shape_b, match):
    with pytest.raises(ValueError, match=match):
        M.frame_metrics(np.zeros(shape_a, np.uint8), np.zeros(shape_b, np.uint8))


@pytest.mark.parametrize("dtype", [np.float64, np.int16, np.uint16, np.bool_])
def test_host_api_refuses_unsupported_dtypes(dtype):
    good = np.zeros((2, 20, 20, 3), np.uint8)
    with pytest.raises(TypeError, match="uint8 or float32"):
        M.frame_metrics(np.zeros((2, 20, 20, 3), dtype), good)
    with pytest.raises(TypeError, match="uint8 or float32"):
        M.frame_metrics(good, np.zeros((2, 20, 20, 3), dtype))


def test_cpu_tensors_raise():
    a = torch.zeros(2, 20, 20, 3, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        M.frame_metrics(a, a, device="cpu")
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            M.frame_metrics(a, a)


def test_workspace_query_refuses_bad_sizes():
    assert lib.call("fgt_metrics_workspace", 2, 64, 96, 3) == 2 * 3 * (2 * 3) * 3 * 8     # 2x3 tiles of 32x32
    assert lib.call("fgt_metrics_workspace", 1, 11, 11, 1) == 3 * 8
    for args, match in [((0, 64, 96, 3), "no frames"), ((2, 10, 96, 3), "11x11"), ((2, 64, 10, 1), "11x11"),
                        ((2, 64, 96, 2), "channels"), ((30000, 64, 96, 3), "65535")]:
        with pytest.raises(RuntimeError, match=match):
            lib.call("fgt_metrics_workspace", *args)


def _write(d, frames):
    from fgt_b200 import io
    return os.path.join(os.path.dirname(io.write_frames(d, frames, mp4=False)[0]))


def test_command_line_reports_mismatched_directories(tmp_path, capsys):
    res, gts = case_inputs("noise_64x96x3_u8")
    r = _write(str(tmp_path / "res"), list(res))
    g2 = _write(str(tmp_path / "g2"), list(gts[:2]))
    with pytest.raises(SystemExit):
        M.main(["--result", r, "--gt", g2])
    assert "3 frames" in capsys.readouterr().err
    g_small = _write(str(tmp_path / "gs"), [f[:60] for f in gts])
    with pytest.raises(SystemExit):
        M.main(["--result", r, "--gt", g_small])
    assert "differ in size" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        M.main(["--result", r])                                       # --gt is required
    with pytest.raises(FileNotFoundError):
        M.main(["--result", r, "--gt", str(tmp_path / "missing")])


def test_command_line_parses():
    a = M._parser().parse_args(["--result", "x", "--gt", "y", "--gpu", "2"])
    assert (a.result, a.gt, a.gpu) == ("x", "y", 2)
    assert M._parser().parse_args(["--result", "x", "--gt", "y"]).gpu == 0
