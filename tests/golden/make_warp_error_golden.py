"""Writes warp_error.npz: the reference's own image_warp and fbConsistencyCheck outputs on the seeded cases of
tests/test_warp_error.py, and the pads of its InputPadder.

    python tests/golden/make_warp_error_golden.py

Runs the UNMODIFIED FGT/models/utils/fbConsistencyCheck.py and RAFT/utils/utils.py of a reference checkout (REF, as in
make_golden.py), loaded by file path, on the CPU, with torch.nn.functional.grid_sample bound to align_corners=True for
the calls (the project's one departure from the reference; see fgt_b200/warp_error.py). Stores, per CASES entry, the
image [b,c,h,w] (float32 on 0..1), the flows F and B [b,2,h,w], image_warp(image, F) and the first output of
fbConsistencyCheck(F, B) as uint8; per LARGE entry only those outputs at the seeded sample positions (its inputs are
regenerated from its seed); and under 'pads' InputPadder((h, w))._pad for each of PAD_SIZES.
"""
import functools
import importlib.util
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.test_warp_error import CASES, GOLDEN, LARGE, PAD_SIZES, case_inputs, sample_positions  # noqa: E402


def _load(package, path, name):
    pkg = types.ModuleType(package)                   # the module imports its sibling sobel2 relatively
    pkg.__path__ = [os.path.dirname(path)]
    sys.modules[package] = pkg
    spec = importlib.util.spec_from_file_location(f"{package}.{name}", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod


def reference(fbc, img, f, b):
    orig = F.grid_sample
    F.grid_sample = functools.partial(orig, align_corners=True)
    try:
        img, f, b = (torch.from_numpy(x) for x in (img, f, b))
        return fbc.image_warp(img, f).numpy(), fbc.fbConsistencyCheck(f, b)[0].numpy().astype(np.uint8)
    finally:
        F.grid_sample = orig


if __name__ == "__main__":
    fbc = _load("ref_fgt_utils", os.path.join(REF, "FGT/models/utils/fbConsistencyCheck.py"), "fbConsistencyCheck")
    utils = _load("ref_raft_utils", os.path.join(REF, "RAFT/utils/utils.py"), "utils")
    arrs = {}
    for name in CASES:
        img, f, b = case_inputs(name)
        warped, occ = reference(fbc, img, f, b)
        arrs.update({f"{name}/image": img, f"{name}/flow_fw": f, f"{name}/flow_bw": b, f"{name}/warped": warped,
                     f"{name}/occ": occ})
        print(name, img.shape, "occluded", occ.mean())
    for name in LARGE:
        warped, occ = reference(fbc, *case_inputs(name))
        arrs[f"{name}/warped"] = warped.reshape(-1)[sample_positions(name, warped.shape)]
        arrs[f"{name}/occ"] = occ.reshape(-1)[sample_positions(name, occ.shape)]
        print(name, warped.shape, "occluded", occ.mean())
    arrs["pads"] = np.array([utils.InputPadder((h, w))._pad for h, w in PAD_SIZES], np.int64)
    np.savez_compressed(GOLDEN, **arrs)
