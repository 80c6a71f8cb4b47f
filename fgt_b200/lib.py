"""ctypes binding of libfgt_sm90a.so (the C-ABI in include/fgt_b200.h).

PyTorch is used here only to own device memory and the CUDA stream; all arithmetic on the path
is done by the kernels in the shared library. There is no CPU fallback: if the library is missing
or a call fails, a RuntimeError is raised.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfgt_sm90a.so")

ACT_NONE, ACT_LEAKY02, ACT_RELU, ACT_SIGMOID, ACT_TANH, ACT_LEAKY001 = 0, 1, 2, 3, 4, 5
AUX_NONE, AUX_ADD, AUX_MUL, AUX_ADD_PRE, AUX_ADD_RELU, AUX_GRU, AUX_GRU_ZR = 0, 1, 2, 3, 4, 5, 6

_c_ll = ctypes.c_longlong
_c_p = ctypes.c_void_p


class FgtASeg(ctypes.Structure):
    _fields_ = [("hi", _c_p), ("plane", _c_ll), ("C", ctypes.c_int), ("DX", ctypes.c_int),
                ("DY", ctypes.c_int), ("DZ", ctypes.c_int), ("sx", _c_ll), ("sy", _c_ll), ("sz", _c_ll),
                ("c_base", ctypes.c_int), ("c_per_group", ctypes.c_int), ("c_count", ctypes.c_int)]


class FgtGemmDesc(ctypes.Structure):
    _fields_ = [("num_segs", ctypes.c_int), ("seg", FgtASeg * 2),
                ("kx", ctypes.c_int), ("ky", ctypes.c_int), ("kz", ctypes.c_int),
                ("stride", ctypes.c_int), ("dil", ctypes.c_int),
                ("pad_x", ctypes.c_int), ("pad_y", ctypes.c_int), ("pad_z", ctypes.c_int),
                ("w_hi", _c_p), ("w_plane", _c_ll), ("N", ctypes.c_int), ("k_pad", ctypes.c_int),
                ("groups", ctypes.c_int),
                ("out_w", ctypes.c_int), ("out_h", ctypes.c_int), ("out_z", ctypes.c_int),
                ("box_w", ctypes.c_int), ("box_h", ctypes.c_int), ("bn", ctypes.c_int),
                ("bias", _c_p), ("alpha", ctypes.c_float), ("act", ctypes.c_int),
                ("aux", _c_p), ("aux_mode", ctypes.c_int),
                ("out_f32", _c_p), ("out_hi", _c_p), ("out_plane", _c_ll),
                ("os_z", _c_ll), ("os_y", _c_ll), ("os_x", _c_ll), ("os_c", _c_ll),
                ("rowmap", _c_p), ("lin_batch", ctypes.c_int), ("aux2", _c_p), ("terms", ctypes.c_int),
                ("out_half", ctypes.c_int)]


class FgtAttnDesc(ctypes.Structure):
    _fields_ = [("q_hi", _c_p), ("q_plane", _c_ll), ("q_batch_stride", _c_ll), ("q_ld", ctypes.c_int),
                ("k_hi", _c_p), ("k_plane", _c_ll), ("k_batch_stride", _c_ll), ("k_ld", ctypes.c_int),
                ("v_hi", _c_p), ("v_plane", _c_ll), ("v_batch_stride", _c_ll), ("v_ld", ctypes.c_int),
                ("out_hi", _c_p), ("out_plane", _c_ll), ("out_batch_stride", _c_ll), ("out_ld", ctypes.c_int),
                ("batches", ctypes.c_int), ("heads", ctypes.c_int), ("head_dim", ctypes.c_int),
                ("Lq", ctypes.c_int), ("Lk", ctypes.c_int), ("Lk_rows", ctypes.c_int),
                ("scale", ctypes.c_float), ("mode", ctypes.c_int),
                ("glob_start", ctypes.c_int), ("glob_count", ctypes.c_int), ("out_rowmap", _c_p),
                ("f16", ctypes.c_int)]


_lib = None


def load():
    """Loads the shared library (fails loudly if it has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: run `python -m fgt_b200.build` (or __graft_entry__.build()). "
            "fgt_b200 has no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    lib.fgt_version.restype = ctypes.c_int
    lib.fgt_last_error.restype = ctypes.c_char_p
    lib.fgt_gemm_tc.argtypes = [ctypes.POINTER(FgtGemmDesc), _c_p]
    lib.fgt_gemm_tc.restype = ctypes.c_int
    lib.fgt_attention.argtypes = [ctypes.POINTER(FgtAttnDesc), _c_p]
    lib.fgt_attention.restype = ctypes.c_int
    ci, cf, cll, cd_ = ctypes.c_int, ctypes.c_float, _c_ll, ctypes.c_double
    lib.fgt_pack_nchw.argtypes = [_c_p, ci, _c_p, ci, ci, ci, ci, ci, ci, _c_p, cll, _c_p]
    lib.fgt_im2col_nchw.argtypes = [_c_p, ci, _c_p, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, cf, cf, _c_p, cll, _c_p]
    lib.fgt_im2col_nchw.restype = ctypes.c_int
    lib.fgt_rownorm.argtypes = [_c_p, ci, ci, _c_p, ci, ci, _c_p, ci, cll, ci, ci, _c_p, _c_p, _c_p, cll, cf, _c_p]
    lib.fgt_rownorm_bcast.argtypes = [_c_p, ci, ci, _c_p, ci, ci, _c_p, ci, cll, ci, ci, _c_p, _c_p, _c_p, ci, cll, cf, _c_p]
    lib.fgt_rownorm_bcast.restype = ctypes.c_int
    lib.fgt_peer_alloc.argtypes = [ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p)]
    lib.fgt_peer_free.argtypes = [_c_p]
    lib.fgt_peer_export.argtypes = [_c_p, ctypes.c_char_p]
    lib.fgt_peer_import.argtypes = [ctypes.c_char_p, ctypes.POINTER(ctypes.c_void_p)]
    lib.fgt_peer_unimport.argtypes = [_c_p]
    lib.fgt_peer_barrier.argtypes = [_c_p, ci, ci, _c_p, _c_p]
    for fn in (lib.fgt_peer_alloc, lib.fgt_peer_free, lib.fgt_peer_export, lib.fgt_peer_import, lib.fgt_peer_unimport,
               lib.fgt_peer_barrier):
        fn.restype = ctypes.c_int
    lib.fgt_regionfill_init.argtypes = [_c_p, _c_p, ci, ci, ci, _c_p, _c_p, _c_p, _c_p, _c_p]
    lib.fgt_regionfill_iters.argtypes = [_c_p, ci, ci, ci, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, ci, ci, _c_p]
    lib.fgt_regionfill_finish.argtypes = [_c_p, _c_p, cll, _c_p, _c_p, _c_p]
    for fn in (lib.fgt_regionfill_init, lib.fgt_regionfill_iters, lib.fgt_regionfill_finish):
        fn.restype = ctypes.c_int
    lib.fgt_poisson_setup.argtypes = [_c_p] * 6 + [ci, ci, ci, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p]
    lib.fgt_poisson_iters.argtypes = [_c_p, ci, ci, ci, ci] + [_c_p] * 9 + [ci, cd_, cd_, cd_, ci, _c_p]
    lib.fgt_poisson_graph_create.argtypes = [_c_p, ci, ci, ci, ci] + [_c_p] * 9 + [ci, cd_, cd_, cd_, ci, ctypes.POINTER(ctypes.c_void_p)]
    lib.fgt_poisson_graph_launch.argtypes = [_c_p, _c_p]
    lib.fgt_poisson_graph_destroy.argtypes = [_c_p]
    lib.fgt_poisson_unfilled.argtypes = [_c_p, _c_p, ci, ci, ci, _c_p, _c_p]
    lib.fgt_poisson_finish.argtypes = [_c_p, _c_p, _c_p, ci, ci, ci, _c_p, _c_p, _c_p, _c_p]
    lib.fgt_poisson_advance_host.argtypes = [_c_p, _c_p, _c_p, ci, cd_, cd_, cd_, cd_, cd_, cd_, ci]
    for fn in (lib.fgt_poisson_setup, lib.fgt_poisson_iters, lib.fgt_poisson_unfilled, lib.fgt_poisson_finish,
               lib.fgt_poisson_advance_host, lib.fgt_poisson_graph_create, lib.fgt_poisson_graph_launch,
               lib.fgt_poisson_graph_destroy):
        fn.restype = ctypes.c_int
    lib.fgt_plane_max.argtypes = [_c_p, ci, cll, _c_p, _c_p]
    lib.fgt_window_gather.argtypes = [_c_p, _c_p, _c_p, _c_p, _c_p, ci, ci, ci, _c_p, _c_p, _c_p, _c_p]
    lib.fgt_window_compose.argtypes = [_c_p, _c_p, _c_p, _c_p, _c_p, ci, ci, ci, _c_p, _c_p]
    lib.fgt_comp_to_u8.argtypes = [_c_p, cll, _c_p, _c_p]
    for fn in (lib.fgt_plane_max, lib.fgt_window_gather, lib.fgt_window_compose, lib.fgt_comp_to_u8):
        fn.restype = ctypes.c_int
    lib.fgt_flow_splat.argtypes = [_c_p, _c_p, ci, ci, ci, ci, ci, _c_p, _c_p, _c_p]
    lib.fgt_flow_splat.restype = ctypes.c_int
    lib.fgt_flow_splat_targets_host.argtypes = [cf, cf, ci, ci, ci, ci, ci, _c_p, _c_p, _c_p, _c_p]
    lib.fgt_flow_splat_targets_host.restype = ctypes.c_int
    lib.fgt_tapsum.argtypes = [_c_p, ci, ci, ci, ci, ci, ci, ci, ci, cll, _c_p, ci, _c_p, cll, cll, cll, cll, _c_p]
    lib.fgt_tapsum.restype = ctypes.c_int
    lib.fgt_dwpool.argtypes = [_c_p, ci, _c_p, ci, ci, ci, ci, ci, ci, ci, _c_p, _c_p, _c_p, _c_p]
    lib.fgt_binary_dilate.argtypes = [_c_p, ci, ci, ci, ci, _c_p, _c_p, _c_p]
    lib.fgt_fill_holes_init.argtypes = [_c_p, ci, ci, ci, _c_p, _c_p]
    lib.fgt_fill_holes_pass.argtypes = [_c_p, ci, ci, ci, _c_p, _c_p, ci, _c_p]
    lib.fgt_fill_holes_finish.argtypes = [_c_p, ci, ci, ci, _c_p, _c_p]
    lib.fgt_resize_nearest_u8.argtypes = [_c_p, ci, ci, ci, ci, ci, ci, _c_p, _c_p]
    lib.fgt_resize_bilinear_f32.argtypes = [_c_p, ci, ci, ci, ci, ci, ci, ci, cf, cf, _c_p, _c_p]
    for fn in (lib.fgt_binary_dilate, lib.fgt_fill_holes_init, lib.fgt_fill_holes_pass, lib.fgt_fill_holes_finish,
               lib.fgt_resize_nearest_u8, lib.fgt_resize_bilinear_f32):
        fn.restype = ctypes.c_int
    lib.fgt_inpaint_telea_workspace.argtypes = [ci, ci, ci]
    lib.fgt_inpaint_telea_workspace.restype = cll
    lib.fgt_inpaint_telea.argtypes = [_c_p, _c_p, ci, ci, ci, ci, cll, cd_, _c_p, cll, _c_p, _c_p]
    lib.fgt_inpaint_telea_plan.argtypes = [_c_p, ci, ci, ci, cd_, _c_p, cll, _c_p]
    lib.fgt_inpaint_telea_fill.argtypes = [_c_p, ci, ci, ci, ci, ci, cd_, _c_p, cll, _c_p, _c_p]
    lib.fgt_inpaint_telea_host.argtypes = [_c_p, _c_p, ci, ci, ci, cd_, _c_p]
    lib.fgt_grad_prep_pre.argtypes = [_c_p, _c_p, ci, ci, ci, _c_p, _c_p]
    lib.fgt_grad_prep_post.argtypes = [_c_p, _c_p, ci, ci, ci, _c_p, _c_p, _c_p]
    for fn in (lib.fgt_inpaint_telea, lib.fgt_inpaint_telea_plan, lib.fgt_inpaint_telea_fill, lib.fgt_inpaint_telea_host,
               lib.fgt_grad_prep_pre, lib.fgt_grad_prep_post):
        fn.restype = ctypes.c_int
    lib.fgt_native_workspace.argtypes = [ci, ci, ci, ci]
    lib.fgt_native_workspace.restype = cll
    lib.fgt_native_count.argtypes = [_c_p, ci, ci, ci, ci, _c_p, cll, _c_p]
    lib.fgt_native_composite.argtypes = [_c_p, ci, ci, ci, _c_p, ci, ci, ci, ci, ci, _c_p, cll, _c_p, _c_p]
    for fn in (lib.fgt_native_count, lib.fgt_native_composite):
        fn.restype = ctypes.c_int
    lib.fgt_conv_tail.argtypes = [_c_p, cll, ci, ci, ci, ci, _c_p, cll, ci, ci, _c_p, ci, _c_p, cll, cll, cll, cll, _c_p]
    lib.fgt_conv_tail.restype = ctypes.c_int
    lib.fgt_swin_prep.argtypes = [_c_p, _c_p, ci, ci, ci, ci, ci, _c_p, ci, ci, ci, ci, ci, _c_p, _c_p, _c_p, _c_p, _c_p,
                                  cll, _c_p, cll, cf, _c_p]
    lib.fgt_swin_prep.restype = ctypes.c_int
    lib.fgt_dwconv3x3_res.argtypes = [_c_p, ci, ci, ci, ci, _c_p, _c_p, _c_p, _c_p, cll, _c_p]
    lib.fgt_fold.argtypes = [_c_p, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, _c_p, _c_p, _c_p, cll, _c_p]
    lib.fgt_unfold.argtypes = [_c_p, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, _c_p, cll, _c_p]
    lib.fgt_fold_unfold.argtypes = [_c_p, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, _c_p, cll, _c_p]
    lib.fgt_fold_unfold.restype = ctypes.c_int
    lib.fgt_upsample2x.argtypes = [_c_p, cll, ci, ci, ci, ci, _c_p, cll, _c_p]
    for fn in (lib.fgt_pack_nchw, lib.fgt_rownorm, lib.fgt_dwpool, lib.fgt_dwconv3x3_res, lib.fgt_fold,
               lib.fgt_unfold, lib.fgt_upsample2x):
        fn.restype = ctypes.c_int
    cd = ctypes.c_double
    lib.fgt_chan_stats.argtypes = [_c_p, ci, ci, ci, _c_p, _c_p]
    lib.fgt_instnorm_act.argtypes = [_c_p, _c_p, ci, ci, ci, cf, ci, _c_p, _c_p, _c_p, cll, _c_p]
    lib.fgt_avgpool2.argtypes = [_c_p, cll, ci, ci, _c_p, _c_p]
    lib.fgt_corr_lookup.argtypes = [ctypes.POINTER(_c_p), ctypes.POINTER(ci), ctypes.POINTER(ci), ci, ci, _c_p, ci,
                                    ci, _c_p, cll, _c_p]
    lib.fgt_raft_flow_update.argtypes = [_c_p, _c_p, ci, ci, ci, ci, _c_p, _c_p, cll, ci, ci, _c_p]
    lib.fgt_convex_upsample.argtypes = [_c_p, _c_p, ci, ci, ci, _c_p, _c_p]
    lib.fgt_f16_to_split.argtypes = [_c_p, cll, _c_p, cll, _c_p]
    for fn in (lib.fgt_chan_stats, lib.fgt_instnorm_act, lib.fgt_avgpool2, lib.fgt_corr_lookup,
               lib.fgt_raft_flow_update, lib.fgt_convex_upsample, lib.fgt_f16_to_split):
        fn.restype = ctypes.c_int
    lib.fgt_prop_step.argtypes = [_c_p, _c_p, _c_p, ci, ci, ci, ci, cd, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p]
    lib.fgt_prop_gather.argtypes = [_c_p, _c_p, _c_p, _c_p, ci, ci, ci, ci, _c_p, _c_p, _c_p]
    lib.fgt_prop_fuse.argtypes = [_c_p, _c_p, _c_p, _c_p, _c_p, ci, ci, ci, cd, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p,
                                  _c_p, _c_p]
    for fn in (lib.fgt_prop_step, lib.fgt_prop_gather, lib.fgt_prop_fuse):
        fn.restype = ctypes.c_int
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().fgt_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")
    COUNTERS["launches"] += 1


def check_rc(rc, what):
    """check() for calls that launch no kernel (allocation, IPC)."""
    if rc != 0:
        msg = load().fgt_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")


# Kernel-launch counter (bench.py's "gpu_launches") and optional per-launch CUDA-event profiler.
COUNTERS = {"launches": 0}
_profile = None  # list of (kernel, tag, flops, bytes, ev_start, ev_end) when enabled
_scope = [""]    # module label of the launches being issued (bench.py's per-module roofline block)


class scope:
    """`with lib.scope("tmhsa"):` labels every launch recorded by the profiler inside the block."""

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        _scope.append(self.name)

    def __exit__(self, *exc):
        _scope.pop()
        return False


def profile_start():
    global _profile
    _profile = []


def profile_stop():
    """Returns [(kernel, tag, algorithmic_flops, algorithmic_bytes, milliseconds, module_scope)]; syncs the device."""
    global _profile
    recs, _profile = _profile, None
    torch.cuda.synchronize()
    return [(k, t, fl, by, e0.elapsed_time(e1), sc) for (k, t, fl, by, sc, e0, e1) in recs]


class _Prof:
    """Brackets one C-ABI launch with CUDA events on the launching stream when profiling is on."""

    def __init__(self, kernel, tag, flops=0.0, nbytes=0.0):
        self.meta = (kernel, tag, float(flops), float(nbytes))

    def __enter__(self):
        if _profile is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if _profile is not None and exc[0] is None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            _profile.append(self.meta + (_scope[-1], self.e0, e1))
        return False


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t, elem_offset=0):
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr() + elem_offset * t.element_size())


# ------------------------------------------------------------------------------------------
# split-bf16 tensors: a torch.bfloat16 tensor whose leading dimension (size 2) is the plane.
# ------------------------------------------------------------------------------------------
def to_split(x):
    """fp32 tensor [...] -> bf16 tensor [2, ...] with hi = bf16(x), lo = bf16(x - hi)."""
    x = x.float()
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return torch.stack([hi, lo], 0).contiguous()


def from_split(s):
    return s[0].float() + s[1].float()


def empty_split(shape, device):
    return torch.empty((2,) + tuple(shape), dtype=torch.bfloat16, device=device)


def view16(t, *shape):
    """A 16-bit activation tensor viewed as `shape`: [2, *shape] when split-bf16, [*shape] when fp16."""
    return t.view(*shape) if t.dtype == torch.float16 else t.view(2, *shape)


def plane_elems(s):
    """Element offset from the hi plane to the lo plane (works for row-sliced views too)."""
    return s.stride(0)


class ASeg:
    """One channel-contiguous A operand view: split tensor + logical (C, DX, DY, DZ) geometry."""

    def __init__(self, split, C, DX, DY=1, DZ=1, sx=None, sy=None, sz=None, c_base=0, c_per_group=0,
                 c_count=None, elem_offset=0):
        self.split = split
        self.C, self.DX, self.DY, self.DZ = C, DX, DY, DZ
        self.sx = C if sx is None else sx
        self.sy = self.sx * DX if sy is None else sy
        self.sz = self.sy * DY if sz is None else sz
        self.c_base, self.c_per_group = c_base, c_per_group
        self.c_count = C if c_count is None else c_count
        self.elem_offset = elem_offset


def gemm_tc(segs, w_split, N, *, kx=1, ky=1, kz=1, stride=1, dil=1, pad_x=0, pad_y=0, pad_z=0, groups=1,
            out_w, out_h=1, out_z=1, box_w=128, box_h=1, bn=128, bias=None, alpha=1.0, act=ACT_NONE,
            aux=None, aux_mode=AUX_NONE, out_f32=None, out_split=None, out_elem_offset=0,
            os_z=0, os_y=0, os_x=None, os_c=1, rowmap=None, lin_batch=0, aux2=None, terms=None, out_f16=None,
            alg_k=None, tag=""):
    """Generic launcher for fgt_gemm_tc. Output strides are in elements; see include/fgt_b200.h.
    The weight's dtype selects the MMA form: a split-bf16 weight takes split-bf16 A segments (3 terms), an fp16 weight
    plain fp16 ones (1 term). out_split, the optional 16-bit output, is split-bf16 or plain fp16. Optional checks of
    the caller's expectation: terms, the MMA form; out_f16, a 16-bit output that must be fp16."""
    lib = load()
    f16 = w_split.dtype == torch.float16
    assert terms is None or terms == (1 if f16 else 3), "terms=1 takes fp16 weights, terms=3 split-bf16 ones"
    if out_f16 is not None:
        assert out_split is None and out_f16.dtype == torch.float16
        out_split = out_f16
    d = FgtGemmDesc()
    d.num_segs = len(segs)
    k_real = 0
    for i, s in enumerate(segs):
        assert (s.split.dtype == torch.float16) == f16, "A segments and weight: both split-bf16 or both fp16"
        a = d.seg[i]
        a.hi = s.split.data_ptr() + 2 * s.elem_offset
        a.plane = 0 if f16 else plane_elems(s.split)
        a.C, a.DX, a.DY, a.DZ = s.C, s.DX, s.DY, s.DZ
        a.sx, a.sy, a.sz = s.sx, s.sy, s.sz
        a.c_base, a.c_per_group, a.c_count = s.c_base, s.c_per_group, s.c_count
        k_real += s.c_count
    d.kx, d.ky, d.kz, d.stride, d.dil = kx, ky, kz, stride, dil
    d.pad_x, d.pad_y, d.pad_z = pad_x, pad_y, pad_z
    d.w_hi = w_split.data_ptr()
    d.w_plane = 0 if f16 else plane_elems(w_split)
    d.N = N
    d.k_pad = w_split.shape[-1]
    d.groups = groups
    d.out_w, d.out_h, d.out_z = out_w, out_h, out_z
    d.box_w, d.box_h, d.bn = box_w, box_h, bn
    d.bias = bias.data_ptr() if bias is not None else None
    d.alpha = alpha
    d.act = act
    d.aux = (aux.data_ptr() + 4 * out_elem_offset) if aux is not None else None
    d.aux_mode = aux_mode
    d.aux2 = (aux2.data_ptr() + 4 * out_elem_offset) if aux2 is not None else None
    d.out_f32 = (out_f32.data_ptr() + 4 * out_elem_offset) if out_f32 is not None else None
    if out_split is not None:
        d.out_hi = out_split.data_ptr() + 2 * out_elem_offset
        d.out_plane = _plane16(out_split)
        d.out_half = 1 if out_split.dtype == torch.float16 else 0
    d.os_z, d.os_y, d.os_c = os_z, os_y, os_c
    d.os_x = N if os_x is None else os_x
    d.rowmap = rowmap.data_ptr() if rowmap is not None else None
    d.lin_batch = lin_batch
    d.terms = 1 if f16 else 3
    # algorithmic work: every valid output position x N x (taps * real input channels), padding excluded
    # (alg_k: the layer's true reduction length per output when the packed weight carries structural zeros, e.g. a
    #  grouped convolution run as block-diagonal super-groups — zeros are not algorithmic work)
    m = out_w * out_h * out_z
    kk = kx * ky * kz * k_real if alg_k is None else alg_k
    flops = 2.0 * m * N * kk
    nbytes = 4.0 * (m * k_real * stride * stride + N * kk + m * N)
    with _Prof("gemm_tc", tag, flops, nbytes):
        check(lib.fgt_gemm_tc(ctypes.byref(d), stream_ptr()), "fgt_gemm_tc")


def attention(q, k, v, out, *, batches, heads, Lq, Lk, Lk_rows=None, q_ld, k_ld, v_ld, out_ld,
              q_batch_stride, k_batch_stride, v_batch_stride, out_batch_stride, scale, mode=0,
              glob_start=0, glob_count=0, q_off=0, k_off=0, v_off=0, out_rowmap=None, tag=""):
    """fgt_attention launcher. q/k/v/out are split-bf16 row-major tensors, or all four plain fp16 tensors (the
    single-plane fp16 mode); strides in elements; q_off/k_off/v_off are element offsets into the plane (e.g. when Q,
    K and V share one [rows, 3*C] projection buffer)."""
    lib = load()
    d = FgtAttnDesc()
    d.f16 = 1 if q.dtype == torch.float16 else 0
    d.q_hi, d.q_plane, d.q_batch_stride, d.q_ld = q.data_ptr() + 2 * q_off, _plane16(q), q_batch_stride, q_ld
    d.k_hi, d.k_plane, d.k_batch_stride, d.k_ld = k.data_ptr() + 2 * k_off, _plane16(k), k_batch_stride, k_ld
    d.v_hi, d.v_plane, d.v_batch_stride, d.v_ld = v.data_ptr() + 2 * v_off, _plane16(v), v_batch_stride, v_ld
    d.out_hi, d.out_plane, d.out_batch_stride, d.out_ld = out.data_ptr(), _plane16(out), out_batch_stride, out_ld
    d.batches, d.heads, d.head_dim = batches, heads, 128
    d.Lq, d.Lk = Lq, Lk
    d.Lk_rows = Lk if Lk_rows is None else Lk_rows
    d.scale, d.mode, d.glob_start, d.glob_count = scale, mode, glob_start, glob_count
    d.out_rowmap = out_rowmap.data_ptr() if out_rowmap is not None else None
    keys = Lk if mode == 0 else 64 + glob_count
    flops = 4.0 * batches * heads * Lq * keys * 128
    nbytes = 4.0 * batches * heads * 128 * (2 * Lq + 2 * (Lk if mode == 0 else d.Lk_rows))
    with _Prof("flash", tag, flops, nbytes):
        check(lib.fgt_attention(ctypes.byref(d), stream_ptr()), "fgt_attention")


def _dp(t):
    return t.data_ptr() if t is not None else None


def pack_nchw(src0, src1, out_split, pad=0, tag=""):
    """[n,c0,H,W] (+ [n,c1,H,W]) fp32 -> NHWC split [2, n, H+2p, W+2p, cpad] with replication pad."""
    n, c0, H, W = src0.shape
    c1 = src1.shape[1] if src1 is not None else 0
    cpad = out_split.shape[-1]
    with _Prof("pack_nchw", tag, 0, 4.0 * n * (c0 + c1) * H * W + 4.0 * out_split[0].numel()):
        check(load().fgt_pack_nchw(_dp(src0), c0, _dp(src1), c1, n, H, W, pad, cpad, _dp(out_split),
                                   plane_elems(out_split), stream_ptr()), "fgt_pack_nchw")


def im2col_nchw(src0, src1, out_split, *, k, stride, pad, replicate, OH, OW, scale=1.0, shift=0.0, tag=""):
    """[n,c0,H,W] (+[n,c1,H,W]) fp32 -> [2, n, OH, OW, cpad] split rows of k*k*cin gathered inputs."""
    n, c0, H, W = src0.shape
    c1 = src1.shape[1] if src1 is not None else 0
    cpad = out_split.shape[-1]
    half = out_split.dtype == torch.float16  # plain fp16 rows [n, OH, OW, cpad] for a 1-term layer
    nbytes = 4.0 * n * (c0 + c1) * H * W + (2.0 * out_split.numel() if half else 4.0 * out_split[0].numel())
    with _Prof("im2col_nchw", tag, 0, nbytes):
        check(load().fgt_im2col_nchw(_dp(src0), c0, _dp(src1), c1, n, H, W, k, stride, pad, 1 if replicate else 0,
                                     OH, OW, cpad, scale, shift, _dp(out_split), 0 if half else plane_elems(out_split),
                                     stream_ptr()),
              "fgt_im2col_nchw")


def rownorm(a, b, out_split, *, gather=None, rows_per_batch, total_rows, dst_batch_rows, dst_row0=0, eps=1e-5,
            gamma=None, beta=None, tag=""):
    """out_split: split-bf16 [2, ...] or a plain fp16 tensor (single-plane rows of a 1-term layer)."""
    ca, lda = a.shape[-1], a.shape[-1]
    cb, ldb = (b.shape[-1], b.shape[-1]) if b is not None else (0, 0)
    with _Prof("rownorm", tag, 0, 8.0 * total_rows * (ca + cb)):
        check(load().fgt_rownorm(_dp(a), ca, lda, _dp(b), cb, ldb, _dp(gather), rows_per_batch, total_rows,
                                 dst_batch_rows, dst_row0, _dp(gamma), _dp(beta), _dp(out_split),
                                 _plane16(out_split), eps, stream_ptr()), "fgt_rownorm")


def rownorm_bcast(a, dst_ptrs, plane, *, gather=None, rows_per_batch, total_rows, dst_batch_rows, dst_row0=0, eps=1e-5,
                  gamma=None, beta=None, tag=""):
    """LayerNorm rows of `a` stored to every buffer in dst_ptrs (raw device addresses of split-bf16 buffers with
    the lo plane `plane` elements after the hi plane; local or peer-mapped)."""
    ca = a.shape[-1]
    arr = (_c_p * len(dst_ptrs))(*dst_ptrs)
    with _Prof("rownorm", tag, 0, 4.0 * total_rows * ca * (1 + len(dst_ptrs))):
        check(load().fgt_rownorm_bcast(_dp(a), ca, ca, None, 0, 0, _dp(gather), rows_per_batch, total_rows,
                                       dst_batch_rows, dst_row0, _dp(gamma), _dp(beta), arr, len(dst_ptrs), plane, eps,
                                       stream_ptr()), "fgt_rownorm_bcast")


def tapsum(y, n, H, W, cout, k, bias, act, out, *, nchw, tag=""):
    """out = act(bias + sum over the k*k taps of the shifted columns of the column-planar y [cols, n*H*W]);
    out is [n,cout,H,W] (nchw) or [n,H,W,cout] fp32. The producing GEMM stores with os_x=1, os_c=n*H*W."""
    ycol = y.shape[-1]
    st = (cout * H * W, W, 1, H * W) if nchw else (H * W * cout, W * cout, cout, 1)
    with _Prof("tapsum", tag, 0, 4.0 * n * H * W * (k * k * cout + cout)):
        check(load().fgt_tapsum(_dp(y), n, H, W, cout, k, k, k // 2, k // 2, ycol, _dp(bias), act, _dp(out), *st,
                                stream_ptr()), "fgt_tapsum")


def pack_taps_as_n(w, n_pad=32):
    """[cout, cin, k, k] conv weight -> [n_pad, cin, 1, 1] weight of the equivalent 1x1 'taps as N' GEMM
    (row tap*cout + c = W[c, :, ty, tx]; zero rows up to n_pad so that the epilogue takes the vector path)."""
    cout, cin, ky, kx = w.shape
    assert ky * kx * cout <= n_pad
    t = torch.zeros(n_pad, cin, 1, 1, dtype=w.dtype, device=w.device)
    t[:ky * kx * cout, :, 0, 0] = w.permute(2, 3, 0, 1).reshape(ky * kx * cout, cin)
    return t


def dwpool(a, b, bt, h, w, k, gh, gw, weight, bias, out, tag=""):
    ca = a.shape[-1]
    cb = b.shape[-1] if b is not None else 0
    with _Prof("dwpool", tag, 0, 4.0 * bt * (h * w + gh * gw) * (ca + cb)):
        check(load().fgt_dwpool(_dp(a), ca, _dp(b), cb, bt, h, w, k, gh, gw, _dp(weight), _dp(bias), _dp(out),
                                stream_ptr()), "fgt_dwpool")


def conv_tail(x_split, n, H, W, cin, w_split, cout, bias, act, out, *, nchw, tag=""):
    """3x3 conv (pad 1) with cout <= 3 + bias + activation: x_split [2,n,H,W,cin] -> out [n,cout,H,W] (nchw) or
    [n,H,W,cout] fp32, one kernel (taps-as-N GEMM + in-SM tap sum). w_split = pack_weight(pack_taps_as_n(w)).
    x_split and w_split may instead both be plain fp16 tensors (1-term fp16 MMAs)."""
    st = (cout * H * W, H * W, W, 1) if nchw else (H * W * cout, 1, W * cout, cout)
    # 2*9*cout*cin FLOP per 4*(cin+cout) bytes = ~13 FLOP/B at 64 -> 3: HBM-bound, reported against the copy roofline
    nbytes = 4.0 * n * H * W * (cin + cout)
    with _Prof("conv_tail", tag, 0.0, nbytes):
        check(load().fgt_conv_tail(_dp(x_split), _plane16(x_split), n, H, W, cin, _dp(w_split), _plane16(w_split),
                                   w_split.shape[-1], cout, _dp(bias), act, _dp(out), *st, stream_ptr()), "fgt_conv_tail")


def swin_prep(x, fp, bt, h, w, win_map, nl, R, gd, gh, gw, gk_w, gk_b, gv_w, gv_b, qkn, vn, eps=1e-5, tag=""):
    """SWMHSA operand preparation in one launch: LayerNorm'd window rows and pooled global rows of [x ; f'] -> qkn
    and of x -> vn (split-bf16 [bt*R, .], or both plain fp16); see include/fgt_b200.h."""
    d, df = x.shape[-1], fp.shape[-1]
    G = gh * gw
    nbytes = 4.0 * bt * ((nl + 2 * h * w) * (d + df) + (nl + G) * (2 * d + df))  # reads (rows + pooling) + split writes
    with _Prof("swin_prep", tag, 0, nbytes):
        check(load().fgt_swin_prep(_dp(x), _dp(fp), d, df, bt, h, w, _dp(win_map), nl, R, gd, gh, gw, _dp(gk_w),
                                   _dp(gk_b), _dp(gv_w), _dp(gv_b), _dp(qkn), _plane16(qkn), _dp(vn),
                                   _plane16(vn), eps, stream_ptr()), "fgt_swin_prep")


def dwconv3x3_res(x, bt, h, w, C, weight, bias, out, out_split=None, tag=""):
    """out_split (optional 16-bit copy): split-bf16 or plain fp16."""
    with _Prof("dwconv3x3_res", tag, 0, 12.0 * bt * h * w * C):
        check(load().fgt_dwconv3x3_res(_dp(x), bt, h, w, C, _dp(weight), _dp(bias), _dp(out), _dp(out_split),
                                       _plane16(out_split), stream_ptr()),
              "fgt_dwconv3x3_res")


def fold(hid, bt, th, tw, C, kh, kw, stride, pad, OH, OW, *, normalize, add=None, out=None, out_split=None, tag=""):
    """out_split (optional 16-bit output): split-bf16 or plain fp16."""
    with _Prof("fold", tag, 0, 4.0 * bt * (th * tw * kh * kw * C + OH * OW * C * (2 if add is not None else 1))):
        check(load().fgt_fold(_dp(hid), bt, th, tw, C, kh, kw, stride, pad, OH, OW, 1 if normalize else 0, _dp(add),
                              _dp(out), _dp(out_split), _plane16(out_split), stream_ptr()), "fgt_fold")


def unfold(img, bt, th, tw, C, kh, kw, stride, pad, OH, OW, out_split, relu=True, tag=""):
    with _Prof("unfold", tag, 0, 4.0 * bt * (th * tw * kh * kw * C + OH * OW * C)):
        check(load().fgt_unfold(_dp(img), bt, th, tw, C, kh, kw, stride, pad, OH, OW, 1 if relu else 0,
                                _dp(out_split), plane_elems(out_split), stream_ptr()), "fgt_unfold")


def fold_unfold(hid, bt, th, tw, C, kh, kw, stride, pad, OH, OW, out_split, relu=True, tag=""):
    """fold (normalised) + unfold (+ReLU) of the fusion FFN in one launch: hid fp32 [bt*th*tw, kh*kw*C] -> split-bf16
    (or plain fp16)."""
    with _Prof("fold_unfold", tag, 0, 8.0 * bt * th * tw * kh * kw * C):
        check(load().fgt_fold_unfold(_dp(hid), bt, th, tw, C, kh, kw, stride, pad, OH, OW, 1 if relu else 0,
                                     _dp(out_split), _plane16(out_split), stream_ptr()), "fgt_fold_unfold")


def upsample2x(in_split, n, H, W, C, out_split, tag=""):
    with _Prof("upsample2x", tag, 0, 4.0 * n * H * W * C * 5):
        check(load().fgt_upsample2x(_dp(in_split), plane_elems(in_split), n, H, W, C, _dp(out_split),
                                    plane_elems(out_split), stream_ptr()), "fgt_upsample2x")


# ------------------------------------------------------------------------------------------ RAFT helpers
def chan_stats(x, n, HW, C, stats, tag=""):
    with _Prof("chan_stats", tag, 0, 4.0 * n * HW * C):
        check(load().fgt_chan_stats(_dp(x), n, HW, C, _dp(stats), stream_ptr()), "fgt_chan_stats")


def _plane16(t):
    """Plane offset of a 16-bit kernel output: 0 selects single-plane fp16 (a torch.float16 tensor), otherwise the
    split-bf16 lo-plane offset."""
    return 0 if t is None or t.dtype == torch.float16 else plane_elems(t)


def instnorm_act(x, stats, n, HW, C, *, relu=True, res=None, out=None, out_split=None, eps=1e-5, tag=""):
    """out_split: split-bf16 [2, ...] or a plain fp16 tensor (single-plane rows of a 1-term layer)."""
    with _Prof("instnorm_act", tag, 0, 4.0 * n * HW * C * (3 if res is not None else 2)):
        check(load().fgt_instnorm_act(_dp(x), _dp(stats), n, HW, C, eps, 1 if relu else 0, _dp(res), _dp(out),
                                      _dp(out_split), _plane16(out_split), stream_ptr()), "fgt_instnorm_act")


def avgpool2(src, rows, h, w, dst, tag=""):
    with _Prof("avgpool2", tag, 0, 5.0 * rows * h * w):
        check(load().fgt_avgpool2(_dp(src), rows, h, w, _dp(dst), stream_ptr()), "fgt_avgpool2")


def corr_lookup(levels, coords, n_pix, radius, out_split, tag=""):
    """levels: list of fp32 tensors [n_pix, h_l, w_l]; out_split: split-bf16 [2, n_pix, pitch] or fp16 [n_pix, pitch]."""
    nl = len(levels)
    ptrs = (_c_p * nl)(*[t.data_ptr() for t in levels])
    hs = (ctypes.c_int * nl)(*[t.shape[1] for t in levels])
    ws = (ctypes.c_int * nl)(*[t.shape[2] for t in levels])
    win = 2 * radius + 1
    with _Prof("corr_lookup", tag, 0, 4.0 * n_pix * nl * ((win + 1) ** 2 + win * win)):
        check(load().fgt_corr_lookup(ptrs, hs, ws, nl, radius, _dp(coords), n_pix, out_split.shape[-1],
                                     _dp(out_split), _plane16(out_split), stream_ptr()), "fgt_corr_lookup")


def raft_flow_update(coords, delta, h, w, flow_nchw, x_split=None, x_chan=0, n=1, delta_f16=False, tag=""):
    """x_split: split-bf16 GRU input, or fp16 for the mixed-precision path; delta_f16: round delta to fp16 first."""
    with _Prof("raft_flow_update", tag, 0, 32.0 * n * h * w):
        check(load().fgt_raft_flow_update(_dp(coords), _dp(delta), 1 if delta_f16 else 0, n, h, w, _dp(flow_nchw),
                                          _dp(x_split),
                                          _plane16(x_split),
                                          x_split.shape[-1] if x_split is not None else 0, x_chan, stream_ptr()),
              "fgt_raft_flow_update")


def convex_upsample(mask, flow_nchw, h, w, out, n=1, tag=""):
    with _Prof("convex_upsample", tag, 0, 4.0 * n * h * w * (576 + 128)):
        check(load().fgt_convex_upsample(_dp(mask), _dp(flow_nchw), n, h, w, _dp(out), stream_ptr()),
              "fgt_convex_upsample")


def f16_to_split(src, out_split, tag=""):
    """fp16 tensor -> split-bf16 [2, ...] of the same element count (exact)."""
    with _Prof("f16_to_split", tag, 0, 6.0 * src.numel()):
        check(load().fgt_f16_to_split(_dp(src), src.numel(), _dp(out_split), plane_elems(out_split), stream_ptr()),
              "fgt_f16_to_split")
