"""Generates the 2D-LAFC goldens (lafc_single_*.npz) by running the UNMODIFIED reference
FGT/models/lafc_single.Model on the CPU, with the shipped configuration (LAFC/config/train_single.yaml).

    python tests/golden/make_lafc_single_golden.py

Weights (synth.lafc_single_state_dict) and inputs (synth.lafc_single_inputs) are seeded, so tests regenerate them
anywhere and only the reference outputs are stored: in full for the small and the odd geometry, as 8192 sampled
values and the L2 norms for 240x432 with t = 13 (the validation's frame count). Every file also records the
reference's state-dict keys and shapes.
"""
import importlib
import os
import sys

import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(REF, "FGT"), ROOT]

from fgt_b200 import synth  # noqa: E402
from oracle import lafc_single_oracle as LSO  # noqa: E402

VERSIONS = dict(torch=torch.__version__, numpy=np.__version__)


def case(name, n, H, W, regime, seed, sample=None):
    M = importlib.import_module("models.lafc_single")
    model = M.Model(synth.CFG_LAFC_SINGLE).eval()
    sd = synth.lafc_single_state_dict(seed=seed, regime=regime)
    model.load_state_dict(sd)
    ref_sd = model.state_dict()
    assert list(ref_sd) == list(sd), "synth key order differs from the reference"
    fl, mk = synth.lafc_single_inputs(seed=seed + 1, n=n, H=H, W=W)
    with torch.no_grad():
        flow, edge = model(fl, mk)
        oflow, oedge = LSO.lafc_single_forward({k[4:]: v for k, v in sd.items()}, fl, mk)
    err = max(((oflow - flow).norm() / flow.norm()).item(), ((oedge - edge).norm() / edge.norm()).item())
    assert err < 1e-5, err
    meta = dict(n=n, H=H, W=W, regime=regime, seed=seed, **VERSIONS)
    arrs = dict(meta=np.array(repr(meta)), keys=np.array(list(ref_sd)),
                shapes=np.array([repr(tuple(v.shape)) for v in ref_sd.values()]),
                flow_l2=np.float64(flow.double().norm().item()), edge_l2=np.float64(edge.double().norm().item()))
    if sample is None:
        arrs["flow"] = flow.numpy().astype(np.float32)
        arrs["edge"] = edge.numpy().astype(np.float32)
    else:
        g = torch.Generator().manual_seed(1234)
        fi = torch.randperm(flow.numel(), generator=g)[:sample]
        ei = torch.randperm(edge.numel(), generator=g)[:sample]
        arrs.update(flow_idx=fi.numpy(), flow_val=flow.reshape(-1)[fi].numpy(), edge_idx=ei.numpy(),
                    edge_val=edge.reshape(-1)[ei].numpy())
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **arrs)
    print(name, "oracle vs reference rel", err, "flow std", flow.std().item(), "saved")


if __name__ == "__main__":
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    case("lafc_single_scaled", 3, 64, 96, "scaled", seed=11)
    case("lafc_single_kaiming", 3, 64, 96, "kaiming", seed=11)
    case("lafc_single_odd", 2, 68, 124, "scaled", seed=12)
    case("lafc_single_full_scaled", 13, 240, 432, "scaled", seed=13, sample=8192)
    case("lafc_single_full_kaiming", 13, 240, 432, "kaiming", seed=13, sample=8192)
