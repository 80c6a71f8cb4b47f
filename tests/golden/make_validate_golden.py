"""Runs the UNMODIFIED reference validation `FGT/networks/network.py::Network._validate` on the CPU over a seeded
mini validation set (synth.validation_set: two videos of 45 and 41 frames and one of 25, 90 x 150 frames, 72 x 120
flows, evaluated at 64 x 96, so every resize runs) and records what each step hands on -> validate_golden.npz:
every step of the first video (the diffused flows rounded to float32), the frame set and flows of the second. What the
tests match bit for bit (frames, masks, flows, the float32 diffused flows, the frames' uint8 copy) is stored as a
SHA-256 digest of its bytes, what they match at a tolerance (diffused and completed flows, FGT output) as 4096 seeded
samples and its L2 norm, and the composite's uint8 values in full. The first frame's vis_frames canvas is stored
with the FGT output it shows.

    python tests/golden/make_validate_golden.py

Only available in the build container (/root/reference). `_validate` runs on a stub `self` (a subclass of Network
whose Trainer base is stubbed) with the seeded synthetic 2D-LAFC and FGT weights of fgt_b200.synth. Modules that are
not in this image are stubbed in sys.modules: cvbase (read_flow: a Middlebury reader), imageio (imread: Pillow;
imwrite: captures the vis_frames canvases), skimage (canny, unused), data.util's __init__ (matplotlib) and metrics (calculate_metrics: captures the uint8
arrays it is handed; skimage's PSNR / SSIM are not run). Every data-loading method is wrapped to record its output,
and both networks to record their inputs and outputs. The dataset is regenerated from the seed by the tests; only
the recorded arrays are stored. A second pass of the data-loading methods with flow_direction 'back' records the
shifted flows.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch
from PIL import Image

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from fgt_b200 import synth  # noqa: E402
from tests.test_validate import digest, sample_idx  # noqa: E402

SEED, H, W = 21, 64, 96
CAP = {}


def _read_flo(path):
    with open(path, "rb") as f:
        assert np.fromfile(f, np.float32, 1)[0] == 202021.25
        w, h = np.fromfile(f, np.int32, 2)
        return np.fromfile(f, np.float32, 2 * w * h).reshape(h, w, 2)


def _stubs():
    for m in ("cvbase", "imageio", "skimage", "skimage.feature", "metrics", "trainer"):
        sys.modules[m] = types.ModuleType(m)
    sys.modules["cvbase"].read_flow = _read_flo
    sys.modules["imageio"].imread = lambda p: np.asarray(Image.open(p))
    sys.modules["imageio"].imwrite = lambda p, im: CAP.setdefault("vis", {}).__setitem__(p, np.array(im))
    sys.modules["skimage.feature"].canny = None
    sys.modules["metrics"].calculate_metrics = lambda r, g: (CAP["scored"].append((r.copy(), g.copy())),
                                                             dict(psnr=0.0, ssim=0.0, l1=0.0, l2=0.0))[1]
    sys.modules["trainer"].Trainer = object
    sys.path[:0] = [os.path.join(REF, "FGT")]
    util = types.ModuleType("data.util")      # the real package, without its __init__ (it needs matplotlib)
    util.__path__ = [os.path.join(REF, "FGT", "data", "util")]
    sys.modules["data.util"] = util


def main():
    _stubs()
    from models.lafc_single import Model as LAFCSingle
    from models.model import Model as FGTModel
    from networks.network import Network

    fgt_cfg = dict(synth.CFG_A, input_resolution=(H, W))
    fgt_sd = synth.make_state_dict(synth.fgt_param_shapes(fgt_cfg), seed=SEED + 1)
    lafc_sd = synth.lafc_single_state_dict(seed=SEED + 2, regime="scaled")
    fgt = FGTModel(fgt_cfg)
    fgt.load_state_dict(fgt_sd)
    lafc = LAFCSingle(synth.CFG_LAFC_SINGLE)
    lafc.load_state_dict(lafc_sd)
    rec = {}

    def wrap(name, fn):
        def run(*a):
            out = fn(*a)
            rec.setdefault(name, []).append(out)
            return out
        return run

    class Stub(Network):
        def __init__(self, root, direction="for"):
            fr, mr, fl = synth.validation_set(root, seed=SEED)
            self.valInfo = dict(frame_root=fr, mask_root=mr, flow_root=fl, flow_width=W, flow_height=H)
            self.opt = dict(num_frames=5, ref_length=10, flow_direction=direction, use_tb_logger=False,
                            device="cpu", path=dict(VAL_IMAGES=os.path.join(root, "vis")))
            self.rank = 0
            self.logger = types.SimpleNamespace(info=lambda *a: None)
            self.model = wrap("fgt", fgt)
            self.model.eval = fgt.eval
            self.model.train = fgt.train
            self.flow_model = wrap("lafc", lambda f, m: lafc(f, m))
            for k in ("read_frames", "read_masks", "read_flows", "diffusion_flows", "norm_flows", "get_ref_index"):
                setattr(self, k, wrap(k, getattr(super(), k)))

        def save_checkpoint(self, epoch):
            pass

    CAP["scored"] = []
    with tempfile.TemporaryDirectory() as root, torch.no_grad():
        stub = Stub(root)
        order = sorted(os.listdir(stub.valInfo["flow_root"]))
        orig = os.listdir
        os.listdir = lambda p: sorted(orig(p))            # one fixed video order for the recording
        try:
            stub._validate(0)
        finally:
            os.listdir = orig
        back = Stub(root + "_back", "back")
        fl_dir = os.path.join(back.valInfo["flow_root"], "vid_b")
        ids_b = list(rec["get_ref_index"][1])      # _validate extends the returned list by the neighbours
        back_flows = back.read_flows(fl_dir, W, H, ids_b, 41 - 1)
    scored = [n for n in order if n != "vid_short"]
    arrs = dict(meta=np.array(repr(dict(seed=SEED, H=H, W=W, videos=order, scored=scored, torch=torch.__version__,
                                        numpy=np.__version__))))
    # vid_a: every step; vid_b: the frame set and the flows read (its last reference frame's flow index is clamped).
    # Steps the tests match bit for bit are stored as digests; the ones matched at a tolerance as seeded samples and
    # L2 norms; the composite in full (its uint8 values are compared level by level).
    masks = np.stack(rec["read_masks"][0])[..., 0]
    assert set(np.unique(masks)) <= {0.0, 1.0}
    diffused = np.stack(rec["diffusion_flows"][0]).astype(np.float32)       # [t,h,w,2], rounded as _validate does
    exact = dict(vid_a_frames=np.stack(rec["read_frames"][0]), vid_a_masks=masks.astype(np.uint8),
                 vid_a_flows=np.stack(rec["read_flows"][0]), vid_a_diffused=diffused,
                 vid_a_frames_u8=CAP["scored"][0][1], vid_b_flows=np.stack(rec["read_flows"][1]),
                 vid_b_back_flows=np.stack(back_flows))
    arrs.update({k + "_sha": np.array(digest(v)) for k, v in exact.items()})
    near = dict(diffused=diffused.transpose(0, 3, 1, 2), completed=rec["lafc"][0][0].numpy(), out=rec["fgt"][0].numpy())
    for k, v in near.items():
        arrs[f"vid_a_{k}_val"] = v.reshape(-1)[sample_idx(v.size).numpy()]
        arrs[f"vid_a_{k}_l2"] = np.float64(np.linalg.norm(v.astype(np.float64)))
    arrs["vid_a_comp_u8"] = CAP["scored"][0][0]
    arrs["vid_a_ids"] = np.array(rec["get_ref_index"][0])
    arrs["vid_b_ids"] = np.array(rec["get_ref_index"][1])
    arrs["vid_b_back_ids"] = np.array(ids_b)
    # the short video: read_frames / read_masks returned [] (it is skipped); rec holds one entry per video processed
    arrs["short_frames_len"] = np.int64(len(rec["read_frames"][order.index("vid_short")]))
    vis = sorted(k for k in CAP["vis"] if "vid_a" in k)
    arrs["vid_a_vis0"] = CAP["vis"][vis[0]].astype(np.float32)   # float32 values (the canvas is float64)
    arrs["vid_a_out0"] = rec["fgt"][0][0].numpy()                  # the FGT output that canvas shows
    np.savez_compressed(os.path.join(HERE, "validate_golden.npz"), **arrs)
    print("saved", {k: v.shape for k, v in arrs.items()})


if __name__ == "__main__":
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    main()
