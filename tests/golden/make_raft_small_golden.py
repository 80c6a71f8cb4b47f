"""Generates the small-RAFT goldens (raft_s_*.npz) by running the UNMODIFIED reference RAFT(small=True), the
reference's --small, on the CPU. `raft_s_` names the small model; the older raft_small_i*.npz hold the basic model on
a small image.

    python tests/golden/make_raft_small_golden.py

Weights (synth.raft_small_state_dict) and inputs (synth.raft_inputs) are seeded, so tests regenerate them anywhere and
only the reference outputs are stored. The two large geometries store the full low-resolution flow and 8192 sampled
values of the upsampled one, like raft_full_i20.npz.
"""
import argparse
import importlib
import os
import sys

import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [REF, ROOT]

from fgt_b200 import synth  # noqa: E402
from oracle import raft_small_oracle as RSO  # noqa: E402

VERSIONS = dict(torch=torch.__version__, numpy=np.__version__)


def case(name, H, W, iters, seed, sample=None):
    R = importlib.import_module("RAFT")
    model = R.RAFT(argparse.Namespace(small=True, mixed_precision=False, alternate_corr=False)).eval()
    sd = synth.raft_small_state_dict(seed=seed)
    model.load_state_dict(sd)
    assert len(model.state_dict()) == 106
    im1, im2 = synth.raft_inputs(seed=seed + 1, H=H, W=W)
    with torch.no_grad():
        lo, up = model(im1, im2, iters=iters, test_mode=True)
    if sample is None:   # the oracle restates the reference: pin it here too
        with torch.no_grad():
            olo, oup = RSO.raft_small_forward(sd, im1, im2, iters=iters)
        err = ((oup - up).norm() / up.norm()).item()
        assert err < 1e-5, err
        print(name, "oracle vs reference rel", err)
    meta = dict(H=H, W=W, iters=iters, seed=seed, model="small", **VERSIONS)
    arrs = dict(meta=np.array(repr(meta)), lo_l2=np.float64(lo.double().norm().item()),
                up_l2=np.float64(up.double().norm().item()), lo=lo.numpy().astype(np.float32))
    if sample is None:
        arrs["up"] = up.numpy().astype(np.float32)
    else:
        g = torch.Generator().manual_seed(1234)
        ui = torch.randperm(up.numel(), generator=g)[:sample]
        arrs.update(up_idx=ui.numpy(), up_val=up.reshape(-1)[ui].numpy())
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **arrs)
    print(name, "|flow|max", lo.abs().max().item(), "saved")


if __name__ == "__main__":
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    case("raft_s_i6", 128, 192, 6, seed=3)
    case("raft_s_i20", 128, 192, 20, seed=3)
    case("raft_s_full_i20", 480, 864, 20, seed=4, sample=8192)
    case("raft_s_720p_i20", 720, 1280, 20, seed=7, sample=8192)
