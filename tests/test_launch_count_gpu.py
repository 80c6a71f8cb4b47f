"""COUNTERS["launches"] (bench.py's gpu_launches) against the kernels torch.profiler records, per entry point.

Each entry point runs once under the profiler; the change of the counter must equal the number of the library's kernels
(namespace fgt) the profiler saw. Torch's own kernels (input conversions, workspace fills) and memsets are not launches
of the library, so they are not counted on either side.
"""
import argparse

import numpy as np
import pytest
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

from fgt_b200 import clip, flow_warp, inpaint, lib, morph, native, poisson, regionfill, synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _launches(fn):
    """(change of COUNTERS["launches"], library kernels recorded by the profiler) over one fn()."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        l0 = lib.COUNTERS["launches"]
        fn()
        torch.cuda.synchronize()
        counted = lib.COUNTERS["launches"] - l0
    names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
    return counted, sum(1 for n in names if "fgt::" in n or "_ZN3fgt" in n)


def _clip():
    frames, masks = synth.pipeline_clip(seed=5, N=12, H=64, W=96)
    fr = torch.from_numpy(np.stack(frames)).to(DEV).permute(0, 3, 1, 2).float().div(255).contiguous()
    mk = (torch.from_numpy(np.stack(masks)).to(DEV) != 0).to(torch.uint8)
    fl = torch.randn(12, 2, 64, 96, device=DEV)
    filled = torch.rand(24, 3, 64, 96, device=DEV)   # the stub model's output: no kernel of its own
    return lambda: clip.inpaint_clip_device(lambda f, _fl, _m: filled[:f.shape[1]], fr, mk, fl)


def _poisson():
    trg, gx, gy, hole, gm = synth.poisson_inputs(seed=1, F=3, H=48, W=64)
    return lambda: (poisson.poisson_blend_batch(trg, gx, gy, hole, gm, use_graph=False),
                    poisson.getUnfilledMask(hole[0], gm[0]))


def _morph():
    m = torch.zeros(3, 40, 56, dtype=torch.uint8, device=DEV)
    m[:, 10:30, 12:40] = 1
    m[:, 18:22, 20:30] = 0
    x = torch.rand(2, 40, 56, 2, device=DEV)
    return lambda: (morph.binary_dilation(m, 4), morph.binary_fill_holes(m), morph.resize_nearest(m, (20, 28)),
                    morph.resize_bilinear(x, (80, 112), channel_scale=(2.0, 2.0)))


def _regionfill():
    img, mask = synth.regionfill_inputs(seed=2, B=4, H=48, W=64)
    flows = np.stack([img[:2], img[2:]], -1)
    return lambda: regionfill.diffusion(flows, mask[:2, ..., None])


def _flow_warp():
    feat, flow = (t.to(DEV) for t in synth.flow_warp_inputs(seed=3))
    return lambda: flow_warp.flow_prop(feat, flow)


def _inpaint():
    g = torch.Generator().manual_seed(4)
    img = torch.randint(0, 256, (3, 40, 56, 3), dtype=torch.uint8, generator=g)
    m = torch.zeros(3, 40, 56, dtype=torch.uint8)
    m[:, 12:24, 16:36] = 1
    video = torch.rand(40, 56, 3, 3, generator=g).numpy()
    mask = np.zeros((40, 56, 3), bool)
    mask[12:24, 16:36] = True
    dil = np.zeros_like(mask)
    dil[10:26, 14:38] = True
    return lambda: (inpaint.inpaint_telea(img, m), inpaint.prepare_gradients(video, mask, dil, device=DEV))


def _native():
    g = torch.Generator().manual_seed(5)
    comp = torch.randint(0, 256, (3, 30, 40, 3), dtype=torch.uint8, generator=g)
    frames = torch.randint(0, 256, (3, 60, 80, 3), dtype=torch.uint8, generator=g)
    masks = torch.zeros(3, 60, 80, dtype=torch.uint8)
    masks[:, 20:36, 30:50] = 255
    return lambda: native.composite_native(comp, frames, masks, 2, device=DEV)


def _fgt():
    from fgt_b200.fgt_model import Model
    cfg = dict(synth.CFG_A)
    cfg["input_resolution"] = (64, 96)
    m = Model(cfg)
    m.load_state_dict(synth.make_state_dict(synth.fgt_param_shapes(cfg), seed=1))
    m = m.to(DEV)
    fr, fl, mk = (x.to(DEV) for x in synth.fgt_inputs(seed=2, t=2, H=64, W=96))
    return lambda: m(fr, fl, mk)


def _raft():
    from fgt_b200.raft_model import RAFT
    m = RAFT(argparse.Namespace(small=False, mixed_precision=False, alternate_corr=False))
    m.load_state_dict(synth.raft_state_dict(seed=3))
    m = m.to(DEV)
    im1, im2 = (x.to(DEV) for x in synth.raft_inputs(seed=4, H=64, W=96))
    return lambda: m(im1, im2, iters=2, test_mode=True)


def _lafc():
    from fgt_b200.lafc_model import Model
    m = Model(synth.CFG_LAFC)
    m.load_state_dict(synth.make_state_dict(synth.lafc_param_shapes(synth.CFG_LAFC), seed=5))
    m = m.to(DEV)
    flows, masks = (x.to(DEV) for x in synth.lafc_inputs(seed=6, T=3, H=64, W=96))
    return lambda: m(flows, masks)


CASES = {"clip": _clip, "poisson": _poisson, "morph": _morph, "regionfill": _regionfill, "flow_warp": _flow_warp,
         "inpaint": _inpaint, "native": _native, "fgt": _fgt, "raft": _raft, "lafc": _lafc}


@pytest.mark.parametrize("case", sorted(CASES))
def test_launch_counter_matches_the_profiler(case):
    with torch.no_grad():
        counted, kernels = _launches(CASES[case]())
    print(f"[launches] {case}: counted {counted}, profiler {kernels}")
    assert kernels > 0
    assert counted == kernels
