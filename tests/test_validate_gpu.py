"""FGT's validation (fgt_b200.validate) on the H100, on the seeded mini validation set of tests/golden/validate_golden.npz:
each stage against what the unmodified network.py recorded (bit for bit through the golden's digests, or at a
tolerance on its seeded samples), the per-video metrics against oracle/validate_oracle.py run
on the same bytes, and the glue kernels of csrc/validate.cu bit for bit against their numpy / torch definitions."""
import numpy as np
import pytest
import torch

from fgt_b200 import lib, synth
from fgt_b200 import validate as V
from oracle import validate_oracle as VO
from oracle.fgt_oracle import strip_net
from tests.test_validate import same, sample_idx
from tests.util import REL_TOL, assert_close, load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    from fgt_b200.fgt_model import Model as FGTModel
    from fgt_b200.lafc_single import Model as LAFCSingle
    g = load_golden("validate_golden")
    meta = g["meta"]
    roots = synth.validation_set(str(tmp_path_factory.mktemp("valid")), seed=meta["seed"])
    fgt_cfg = dict(synth.CFG_A, input_resolution=(meta["H"], meta["W"]))
    fgt_sd = synth.make_state_dict(synth.fgt_param_shapes(fgt_cfg), seed=meta["seed"] + 1)
    lafc_sd = synth.lafc_single_state_dict(seed=meta["seed"] + 2, regime="scaled")
    fgt, lafc = FGTModel(fgt_cfg), LAFCSingle(synth.CFG_LAFC_SINGLE)
    fgt.load_state_dict(fgt_sd)
    lafc.load_state_dict(lafc_sd)
    return g, roots, lafc.cuda().eval(), fgt.cuda().eval(), strip_net(lafc_sd), strip_net(fgt_sd)


def _video(roots, name):
    return [r + "/" + name for r in roots]


def test_stages_against_reference(setup):
    g, roots, lafc, fgt, _, _ = setup
    H, W = g["meta"]["H"], g["meta"]["W"]
    st = {}
    res = V.validate_video(lafc, fgt, *_video(roots, "vid_a"), width=W, height=H, stages=st)
    assert res["frames"] == 8 and st["ids"] == list(g["vid_a_ids"])
    assert same(st["frames"], g, "vid_a_frames") and same(st["masks"], g, "vid_a_masks")
    assert same(st["flows"].cpu().numpy(), g, "vid_a_flows")                       # the bit-exact cv2 resize

    def sampled(x, key, tol, what):
        x = x.cpu()
        assert_close(x.reshape(-1)[sample_idx(x.numel())], g[key + "_val"], tol, what)
        assert abs(x.double().norm().item() - float(g[key + "_l2"])) <= tol * float(g[key + "_l2"]), what

    sampled(st["diffused"], "vid_a_diffused", 1e-6, "diffused flows")             # CG at 1e-12, rounded to fp32
    sampled(st["completed"], "vid_a_completed", REL_TOL, "completed flows")
    comp = st["completed"].cpu()
    normed = comp / comp.flatten(2).max(-1, keepdim=True)[0].unsqueeze(-1)
    assert_close(st["normed"], normed, REL_TOL, "normalised flows")
    sampled(st["out"], "vid_a_out", REL_TOL, "FGT output")
    # the frames' uint8 copy is exact; the composite's within one level where FGT's output differs at the 1e-4 level
    assert same(st["frames_u8"].cpu().numpy(), g, "vid_a_frames_u8")
    d = np.abs(st["comp_u8"].cpu().numpy().astype(int) - g["vid_a_comp_u8"].astype(int))
    print(f"\ncomposite uint8 vs reference: {int((d > 0).sum())} of {d.size} values differ, max {int(d.max())}")
    assert d.max() <= 1


def test_validate_against_oracle_on_the_same_bytes(setup):
    g, roots, lafc, fgt, lafc_sd, fgt_sd = setup
    H, W = g["meta"]["H"], g["meta"]["W"]
    res = V.validate(lafc, fgt, *roots, width=W, height=H)
    assert sorted(res["videos"]) == ["vid_a", "vid_b"] and list(res["skipped"]) == ["vid_short"]
    for name, got in res["videos"].items():
        want, _ = VO.validate_video(lafc_sd, fgt_sd, *_video(roots, name), W, H)
        gaps = {k: abs(got[k] - want[k]) for k in ("psnr", "ssim", "l1", "l2")}
        print(f"\n{name}: psnr {got['psnr']:.4f} dB (oracle {want['psnr']:.4f}), ssim {got['ssim']:.6f} "
              f"(oracle {want['ssim']:.6f}), gaps {gaps}")
        assert gaps["psnr"] <= 0.05 and gaps["ssim"] <= 1e-3 and got["frames"] == want["frames"] == 8
    assert abs(res["mean"]["psnr"] - np.mean([v["psnr"] for v in res["videos"].values()])) < 1e-12


def test_back_direction_reads_the_shifted_flows(setup):
    g, roots, _, _, _, _ = setup
    ids = list(g["vid_b_back_ids"])
    paths = V.flow_files(_video(roots, "vid_b")[2], ids, 41, "back")
    got = V.read_flows(paths, g["meta"]["W"], g["meta"]["H"], torch.device("cuda"))
    assert same(got.cpu().numpy(), g, "vid_b_back_flows")
    paths = V.flow_files(_video(roots, "vid_b")[2], list(g["vid_b_ids"]), 41)
    got = V.read_flows(paths, g["meta"]["W"], g["meta"]["H"], torch.device("cuda"))
    assert same(got.cpu().numpy(), g, "vid_b_flows")


def test_glue_kernels_bit_for_bit():
    gen = torch.Generator().manual_seed(3)
    t, H, W = 3, 17, 29
    frames = torch.randint(0, 256, (t, H, W, 3), generator=gen, dtype=torch.uint8)
    masks = (torch.rand(t, H, W, generator=gen) < 0.3).to(torch.uint8)
    fr = torch.empty(t, 3, H, W, device="cuda")
    masked, mk = torch.empty_like(fr), torch.empty(t, 1, H, W, device="cuda")
    lib.call("fgt_valid_inputs", frames.cuda(), masks.cuda(), t, H, W, fr, masked, mk)
    want = frames.permute(0, 3, 1, 2).contiguous().float() / 127.5 - 1
    m = masks.float()[:, None]
    assert torch.equal(fr.cpu(), want) and torch.equal(mk.cpu(), m) and torch.equal(masked.cpu(), want * (1 - m))
    # score: out values around the rounding points of the quantisation, and outside [-1, 1]
    out = torch.rand(t, 3, H, W, generator=gen) * 2.4 - 1.2
    out[0, 0, 0, :20] = (torch.arange(20) / 127.5 - 1).float()
    cu, fu = torch.empty(t, H, W, 3, dtype=torch.uint8, device="cuda"), torch.empty(t, H, W, 3, dtype=torch.uint8,
                                                                                       device="cuda")
    lib.call("fgt_valid_score", out.cuda(), want.cuda(), m.cuda(), t, H, W, cu, fu)
    comp = (out * m + want * (1 - m)).permute(0, 2, 3, 1).numpy()
    q = lambda x: np.clip((x + 1) / 2 * 255, 0, 255).astype(np.uint8)  # noqa: E731
    assert np.array_equal(cu.cpu().numpy(), q(comp))
    assert np.array_equal(fu.cpu().numpy(), q(want.permute(0, 2, 3, 1).numpy()))
    # flow scaling (numpy float32: u / pre_w * w) and the per-plane normalisation (torch: x / max)
    fl = (torch.randn(2, H, W, 2, generator=gen) * 30).numpy()
    d = torch.from_numpy(fl).cuda()
    lib.call("fgt_valid_flow_scale", d, 2 * H * W, 150.0, 432.0, 90.0, 240.0)
    ref = fl.copy()
    ref[..., 0] = ref[..., 0] / 150 * 432
    ref[..., 1] = ref[..., 1] / 90 * 240
    assert np.array_equal(d.cpu().numpy(), ref)
    x = torch.randn(t, 2, H, W, generator=gen).cuda()
    fmax = torch.empty(t * 2, device="cuda")
    lib.call("fgt_plane_max", x, t * 2, H * W, fmax)
    y = torch.empty_like(x)
    lib.call("fgt_valid_norm_flows", x, fmax, t * 2, H * W, y)
    assert torch.equal(y, x / x.flatten(2).max(-1, keepdim=True)[0].unsqueeze(-1))
