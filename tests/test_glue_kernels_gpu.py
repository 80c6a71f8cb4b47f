"""Launch-by-launch replay of the driver-glue kernels on the H100: every launch of the entries in
tests/glue_emulator.GLUE_ENTRIES issued by real calls runs on the GPU and then, on CPU copies of the buffers it
referenced as they were before the launch, through the numpy interpreter of tests/glue_emulator.py (the Replayer of
tests/test_kernel_replay_gpu.py with that interpreter). Before each launch the buffers the entry only writes are filled
with 0xA5 bytes, so a store the interpreter does not make cannot hide behind a zero or an earlier result.

Bar, per launch: every stored element bit-identical to the interpreter (a NaN of fgt_plane_max only as a NaN: its
payload is not specified), and every byte the interpreter does not write unchanged. `tmp` of fgt_binary_dilate is
scratch: addressed, not compared.

Cases: the edge inputs of tests/test_glue_kernels.py (1-pixel images, batch boundaries, diagonal holes, the spiral,
nearest ratios where the double step and integer division disagree, exact 2x, one-pixel sources, NaN / +-0 / +-inf
planes, every k / 255 frame value and model outputs on every uint8 boundary); the glue calls of a GpuBackend on the
watermark and extrapolation goldens' clips (mask resize, dilation, hole filling and a flow resize from RAFT's size up
to the working size); clip.inpaint_clip on the pipeline_clip golden; inpaint.prepare_gradients on that clip; and a
1080 x 1920 batch, whose launches outnumber the capped grids (16 x SMs blocks of 256) so the grid-stride loops run.

Observed on an H100 80GB HBM3 (700 W power limit): every stored value of every entry bit-identical (0 differing values
in all 12 entries over every launch), no byte outside the interpreter's stores changed. The file's 8 tests take 39 s,
19 s of them the 1080 x 1920 batch.
"""
import time

import numpy as np
import pytest
import torch

from fgt_b200 import lib
from tests.glue_emulator import GLUE_ENTRIES, GlueEmulator
from tests.test_kernel_replay_gpu import Replayer, _bytes
from tests.test_glue_kernels import _edge_masks, _flows, _nearest_disagreements, _spiral, _window_case
from tests.util import load_golden

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
WRITE_ONLY = {"fgt_binary_dilate": ("tmp", "out"), "fgt_fill_holes_init": ("reach",), "fgt_fill_holes_pass": ("changed",),
              "fgt_fill_holes_finish": ("out",), "fgt_resize_nearest_u8": ("out",), "fgt_resize_bilinear_f32": ("out",),
              "fgt_plane_max": ("out",), "fgt_window_gather": ("out_frames", "out_flows", "out_masks"),
              "fgt_comp_to_u8": ("out",), "fgt_grad_prep_pre": ("u8",), "fgt_grad_prep_post": ("gx", "gy")}


class GlueReplayer(Replayer):
    emulator = GlueEmulator

    def _replay(self, name, f, args):
        names = lib.PROTOS[name].names
        for k in WRITE_ONLY.get(name, ()):
            p = args[names.index(k)]
            p = p.value if hasattr(p, "value") else p
            _, t = self._find(p)
            _bytes(t).fill_(0xA5)
        return super()._replay(name, f, args)

    def _compare(self, name, cargs, emu, before, after, work):
        self._check_untouched(name, emu, before, after, work)
        key = {w.untyped_storage().data_ptr(): b for b, w in work.items()}
        for kind, fl, idx, _, _ in emu.records:
            if kind == "addr":
                continue
            b = key[fl.untyped_storage().data_ptr()]
            g = torch.empty(0, dtype=fl.dtype).set_(after[b].untyped_storage(), fl.storage_offset(), fl.shape, (1,))
            got, want = g[idx], fl[idx]
            same = (got.view(torch.uint8).view(-1, got.element_size()) ==
                    want.view(torch.uint8).view(-1, want.element_size())).all(1)
            if got.dtype == torch.float32:
                same |= torch.isnan(got) & torch.isnan(want)
            bad = int((~same).sum())
            self.maxima[(name, kind)] = max(self.maxima[(name, kind)], float(bad))
            assert bad == 0, f"{name} ({kind}): {bad} of {len(idx)} stored values differ from the interpreter"


class replaying:
    def __enter__(self):
        self.saved = lib.load()
        self.rep = GlueReplayer(self.saved, GLUE_ENTRIES, device_type=DEV.type)
        lib._lib = self.rep
        return self.rep

    def __exit__(self, *exc):
        lib._lib = self.saved
        self.rep._st.clear()
        return False


def _done(rep, what, **expect):
    rep.report(what)
    for k, n in expect.items():
        assert rep.launches["fgt_" + k] >= n, (k, dict(rep.launches))
    assert all(v == 0 for v in rep.maxima.values())


# ------------------------------------------------------------------------------------------------------ edge inputs
def test_replay_mask_edges():
    from fgt_b200 import morph
    with replaying() as r:
        for m in _edge_masks():
            for iters in (1, 2, 12):
                morph.binary_dilation(m, iters, device=DEV)
            for passes in (1, 3):
                morph.binary_fill_holes(m, device=DEV, passes_per_check=passes)
        morph.binary_fill_holes(_spiral(40, 64)[None], device=DEV, passes_per_check=1)
    _done(r, "mask edges", binary_dilate=21, fill_holes_pass=20, fill_holes_finish=15)


def test_replay_resize_edges():
    from fgt_b200 import morph
    from tests.test_glue_kernels import RESIZES
    g = np.random.default_rng(30)
    with replaying() as r:
        for s, d in _nearest_disagreements()[:20] + [(1, 5), (5, 1), (7, 3), (9, 3), (3, 9)]:
            for C in (1, 3):
                x = g.integers(0, 256, (2, s + 1, s, C), dtype=np.uint8)
                morph.resize_nearest(x if C > 1 else x[..., 0], (d + 1, d), device=DEV)
        for src, dst in RESIZES + [((4, 6), (4, 18)), ((9, 12), (3, 4)), ((1, 5), (4, 5)), ((5, 1), (5, 4))]:
            for C in (2, 5):
                x = _flows(src, C, 31)
                morph.resize_bilinear(x, dst, channel_scale=(dst[1] / src[1], dst[0] / src[0]), device=DEV)
            x = _flows(src, 3, 32).transpose(0, 3, 1, 2).copy()
            morph.resize_bilinear(x, dst, layout="nchw", device=DEV)
    _done(r, "resize edges", resize_nearest_u8=50, resize_bilinear_f32=3 * 17)


def test_replay_plane_max_and_window_edges():
    frames, masks, flows, fmax, filled, H, W = _window_case()
    N, HW = masks.shape
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    with replaying() as r:
        for n in (1, 255, 256, 257):
            x = np.random.default_rng(n).standard_normal((6, n)).astype(np.float32)
            x[0] = -np.abs(x[0]) - 1
            x[1] = -0.0
            x[1, n // 2] = 0.0
            x[2, n // 3] = np.nan
            x[3, -1] = np.inf
            x[4] = -np.inf
            xd, out = d(x), torch.empty(6, dtype=torch.float32, device=DEV)   # live tensors: the replay resolves them
            lib.call("fgt_plane_max", xd, 6, n, out)
        fr, mk, fl, fm = d(frames), d(masks), d(flows), d(fmax)
        comp = torch.empty(N, H, W, 3, dtype=torch.float32, device=DEV)
        for ids, first in (([1, 3], [1, 1]), ([3, 0, 2], [0, 1, 1]), ([1, 3, 0, 2], [0, 0, 0, 0])):
            t = len(ids)
            di = torch.tensor(ids, dtype=torch.int32, device=DEV)
            of, ofl, om = (torch.empty(t, c, H, W, device=DEV) for c in (3, 2, 1))
            lib.call("fgt_window_gather", fr, mk, fl, fm, di, t, H, W, of, ofl, om)
            out_t, fi = d(filled[:t]), torch.tensor(first, dtype=torch.uint8, device=DEV)
            lib.call("fgt_window_compose", out_t, fr, mk, di, fi, t, H, W, comp)
        out = torch.empty(N * HW * 3, dtype=torch.uint8, device=DEV)
        lib.call("fgt_comp_to_u8", comp, comp.numel(), out)
    _done(r, "plane max / window edges", plane_max=4, window_gather=3, window_compose=3, comp_to_u8=1)


def test_replay_grad_prep_edges():
    from fgt_b200 import inpaint
    g = np.random.default_rng(33)
    H, W, N = 12, 32, 3
    v = g.random((H, W, 3, N)).astype(np.float32)
    k255 = (np.arange(256) / 255).astype(np.float32)
    v[..., 0].reshape(-1)[:512] = np.concatenate([k255, np.nextafter(k255, np.float32(-1))]).clip(0, 1)
    hole = g.random((H, W, N)) < 0.2
    md = hole | (g.random((H, W, N)) < 0.2)
    md[-1, ::2] = True
    md[::3, -1] = True
    with replaying() as r:
        inpaint.prepare_gradients(v, hole, md, device=DEV)
    _done(r, "grad prep edges", grad_prep_pre=1, grad_prep_post=1)


# ---------------------------------------------------------------------------------------------------- real calls
@pytest.mark.parametrize("name", ["pipeline_watermark", "pipeline_extrapolation"])
def test_replay_gpu_backend_glue_on_golden_clips(name):
    """The GpuBackend's glue calls at the mode's geometry: masks resized from the clip's size to the working size (the
    clip scaled by the mode's scale: 128 x 192, 80 x 120), dilated and hole-filled, and flows at the clip's size (where
    RAFT runs) resized up to the working size with their vectors rescaled."""
    from fgt_b200 import pipeline as PL, synth
    m = load_golden(name)["meta"]
    frames, masks = synth.pipeline_clip(seed=m["clip_seed"], N=m["N"], H=m["H"], W=m["W"])
    be = PL.GpuBackend(None, None, None, device=DEV)
    H, W = int(round(m["H"] * m["scale"])), int(round(m["W"] * m["scale"]))
    mk = np.stack([np.asarray(x) != 0 for x in masks]).astype(np.uint8) * 255
    g = np.random.default_rng(34)
    with replaying() as r:
        rm = be.resize_masks(mk, H, W)
        dm = be.dilate_masks(rm, max(1, m["flow_mask_dilates"]))
        be.fill_holes(dm)
        be.dilate_masks(rm, 4)
        be.resize_flows((g.standard_normal((m["N"] - 1, 2, m["H"], m["W"])) * 3).astype(np.float32), H, W)
    _done(r, name, resize_nearest_u8=1, resize_bilinear_f32=1, binary_dilate=2, fill_holes_finish=1)


def test_replay_inpaint_clip_and_prepare_gradients_on_pipeline_clip():
    from fgt_b200 import clip as C, inpaint
    from tests.test_clip import _exact_model, _golden
    g, frame_blends, mask, flow_f = _golden()
    with replaying() as r:
        C.inpaint_clip(_exact_model, frame_blends, mask, flow_f, device=DEV)
        video = np.ascontiguousarray(np.stack(frame_blends, -1).astype(np.float32))
        import scipy.ndimage
        md = np.stack([scipy.ndimage.binary_dilation(mask[..., i], iterations=2) for i in range(mask.shape[-1])], -1)
        inpaint.prepare_gradients(video, mask, md, device=DEV)
    _done(r, "pipeline_clip", plane_max=1, window_gather=1, window_compose=1, comp_to_u8=1, grad_prep_pre=1,
          grad_prep_post=1)


def test_replay_1080p_grid_stride():
    from fgt_b200 import inpaint, morph
    B, H, W = 2, 1080, 1920
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    assert B * H * W > sms * 16 * 256, "one grid stride covers the batch"
    g = np.random.default_rng(35)
    m = (g.random((B, H, W)) < 0.02).astype(np.uint8)
    m[:, 500:600, 800:1000] = 1
    m[:, 520:580, 850:950] = 0
    t0 = time.time()
    with replaying() as r:
        morph.binary_dilation(m, 2, device=DEV)
        morph.binary_fill_holes(m, device=DEV)
        morph.resize_nearest(m, (540, 960), device=DEV)
        morph.resize_bilinear(_flows((540, 960), 2, 36), (H, W), channel_scale=(2.0, 2.0), device=DEV)
        v = g.random((H, W, 3, B)).astype(np.float32)
        inpaint.prepare_gradients(v, np.moveaxis(m, 0, -1) != 0, np.moveaxis(m, 0, -1) != 0, device=DEV)
        vd, vmax = torch.from_numpy(np.ascontiguousarray(np.moveaxis(v, -1, 0))).to(DEV), torch.empty(2, device=DEV)
        lib.call("fgt_plane_max", vd, 2, H * W * 3, vmax)
    print(f"[1080x1920] replay {time.time() - t0:.1f} s")
    _done(r, "1080x1920", binary_dilate=1, fill_holes_pass=1, resize_nearest_u8=1, resize_bilinear_f32=1,
          grad_prep_pre=1, grad_prep_post=1, plane_max=1)
