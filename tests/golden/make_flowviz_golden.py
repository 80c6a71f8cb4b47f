"""Writes flowviz.npz: the reference's own colour images of the flows of tests/test_flowviz.py CASES.

    python tests/golden/make_flowviz_golden.py

Runs the UNMODIFIED RAFT/utils/flow_viz.py of a reference checkout (REF, as in make_golden.py), loaded by file path,
under the host's numpy (2.x, NEP 50 promotion), on float32 flows as the driver hands them over (calculate_flow,
tool/video_inpainting.py:264-276). Stores, per case, the flows [B,H,W,2] and flow_to_image of each in RGB and in BGR
order. The reference raises IndexError on NaN or Inf, so no such case is stored.
"""
import importlib.util
import os
import sys

import numpy as np

REF = "/root/reference/RAFT/utils/flow_viz.py"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.test_flowviz import CASES, GOLDEN  # noqa: E402


def _flow_viz():
    spec = importlib.util.spec_from_file_location("ref_flow_viz", REF)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    fv = _flow_viz()
    arrs = {}
    for name, (make, _) in CASES.items():
        flows = make()
        with np.errstate(over="ignore"):
            rgb = np.stack([fv.flow_to_image(f) for f in flows])
            bgr = np.stack([fv.flow_to_image(f, convert_to_bgr=True) for f in flows])
        arrs.update({f"{name}/flows": flows, f"{name}/rgb": rgb, f"{name}/bgr": bgr})
        print(name, flows.shape, np.bincount(rgb.reshape(-1), minlength=256).nonzero()[0].size, "distinct levels")
    np.savez_compressed(GOLDEN, **arrs)
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")
