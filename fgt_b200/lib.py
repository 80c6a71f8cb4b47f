"""ctypes binding of libfgt_sm90a.so (the C-ABI in include/fgt_b200.h).

PyTorch is used here only to own device memory and the CUDA stream; all arithmetic on the path
is done by the kernels in the shared library. There is no CPU fallback: if the library is missing
or a call fails, a RuntimeError is raised.
"""
import collections
import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfgt_sm90a.so")
HEADER = os.path.join(os.path.dirname(_HERE), "include", "fgt_b200.h")

_SCALARS = {"int": ctypes.c_int, "unsigned": ctypes.c_uint, "long long": ctypes.c_longlong, "float": ctypes.c_float,
            "double": ctypes.c_double, "size_t": ctypes.c_size_t, "fgt_stream_t": ctypes.c_void_p}
_RESTYPES = {"int": ctypes.c_int, "long long": ctypes.c_longlong, "const char*": ctypes.c_char_p}

Proto = collections.namedtuple("Proto", "restype argtypes names stream")


def _declarator(decl):
    """'const float* x' / 'unsigned char h[64]' -> (C type, name, array length or None)."""
    m = re.fullmatch(r"(.+?)\s*\b(\w+)\s*(?:\[(\d*)\])?", decl.strip())
    if m is None:
        raise ValueError(f"cannot parse the declaration '{decl.strip()}'")
    return " ".join(re.sub(r"\s*\*", "*", m.group(1)).split()), m.group(2), m.group(3)


def _ctype(ctype, types, decl):
    """ctypes type of a non-array C type: any pointer is c_void_p, other types must be in `types`."""
    if "*" in ctype:
        return ctypes.c_void_p
    t = types.get(" ".join(re.sub(r"\bconst\b", " ", ctype).split()))
    if t is None:
        raise ValueError(f"no ctypes mapping for the type '{ctype}' in '{' '.join(decl.split())}'")
    return t


def parse_header(text):
    """The C ABI declared by `text`: ({struct: ctypes.Structure}, {enum constant: value}, {entry: Proto}).
    Pointers and array parameters become c_void_p; any other type without a ctypes mapping raises ValueError."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)
    structs = {}
    for body, sname in re.findall(r"typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;", text, flags=re.S):
        fields = []
        for stmt in filter(str.strip, body.split(";")):
            first, *more = stmt.split(",")
            ctype = _declarator(first)[0]
            t = _ctype(ctype, {**_SCALARS, **structs}, stmt)
            for d in [first] + [f"{ctype} {m}" for m in more]:   # `int C, DX, DY, DZ;`
                _, name, n = _declarator(d)
                fields.append((name, t * int(n) if n else t))
        structs[sname] = type(sname, (ctypes.Structure,), {"_fields_": fields})
    enums = {}
    for body in re.findall(r"\benum\s*\{(.*?)\}", text, flags=re.S):
        v = -1
        for item in filter(str.strip, body.split(",")):
            k, _, val = item.partition("=")
            v = int(val, 0) if val.strip() else v + 1
            enums[k.strip()] = v
    protos = {}
    for ret, name, params in re.findall(r"([^;{}()]*?)\b(fgt_\w+)\s*\(([^()]*)\)\s*;", text):
        decl = f"{ret.strip()} {name}({params})"
        ret = _declarator(f"{ret} {name}")[0]
        if ret not in _RESTYPES:
            raise ValueError(f"no ctypes mapping for the return type '{ret}' in '{' '.join(decl.split())}'")
        ps = [_declarator(p) for p in params.split(",")] if params.strip() not in ("", "void") else []
        argtypes = [ctypes.c_void_p if n is not None else _ctype(t, _SCALARS, decl) for t, _, n in ps]
        protos[name] = Proto(_RESTYPES[ret], argtypes, [p for _, p, _ in ps], bool(ps) and ps[-1][0] == "fgt_stream_t")
    return structs, enums, protos


with open(HEADER) as _f:
    _STRUCTS, _ENUMS, PROTOS = parse_header(_f.read())
FgtASeg, FgtGemmDesc, FgtAttnDesc = _STRUCTS["FgtASeg"], _STRUCTS["FgtGemmDesc"], _STRUCTS["FgtAttnDesc"]
globals().update({k[len("FGT_"):]: v for k, v in _ENUMS.items()})   # ACT_*, AUX_*, OK, ERR_*

_lib = None


def load():
    """Loads the shared library (fails loudly if it has not been built) and declares every entry of the header."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: run `python -m fgt_b200.build` (or __graft_entry__.build()). "
            "fgt_b200 has no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, p in PROTOS.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = p.argtypes, p.restype
    _lib = lib
    return lib


def call(name, *args, kernels=None):
    """Calls the C entry `name`: tensors are passed as their data_ptr(), None as NULL, anything else as given, and the
    current stream is appended when the entry takes one. A nonzero status of an `int` entry, or a negative value of a
    `long long` one, raises RuntimeError with fgt_last_error(); the value is returned otherwise. `kernels`: the number
    of kernels the call enqueues, added to COUNTERS["launches"] (default 1 for an entry that takes a stream, else 0)."""
    p = PROTOS[name]
    args = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    if p.stream:
        args.append(stream_ptr())
    r = getattr(load(), name)(*args)
    if r < 0 or (r != 0 and p.restype is ctypes.c_int):
        msg = load().fgt_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{name} failed (code {r}): {msg}")
    COUNTERS["launches"] += (1 if p.stream else 0) if kernels is None else kernels
    return r


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


def act16_dtype(mixed):
    """dtype of the 16-bit activations: fp16 in mixed precision, split-bf16 otherwise."""
    return torch.float16 if mixed else torch.bfloat16


def view16(t, *shape):
    """A 16-bit activation tensor viewed as `shape`: [2, *shape] when split-bf16, [*shape] when fp16."""
    return t.view(*shape) if t.dtype == torch.float16 else t.view(2, *shape)


def plane16(t, split_only=False):
    """The C ABI's plane offset of a 16-bit activation: hi-to-lo element offset of a split-bf16 tensor (row-sliced views
    too), 0 for an fp16 tensor or None. split_only: the entry takes split-bf16 only, and fp16 raises TypeError."""
    if t is None or (t.dtype == torch.float16 and not split_only):
        return 0
    if t.dtype != torch.bfloat16:
        raise TypeError(f"a {'split-bf16' if split_only else 'split-bf16 or fp16'} tensor is required, got {t.dtype}")
    if t.dim() == 0 or t.shape[0] != 2:
        raise ValueError(f"a split-bf16 tensor has a leading plane dimension of 2, got shape {tuple(t.shape)}")
    return t.stride(0)


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
            alg_k=None, autocast=False, tag=""):
    """Generic launcher for fgt_gemm_tc. Output strides are in elements; see include/fgt_b200.h.
    The weight's dtype selects the MMA form: a split-bf16 weight takes split-bf16 A segments (3 terms), an fp16 weight
    plain fp16 ones (1 term). out_split, the optional 16-bit output, is split-bf16 or plain fp16. Optional checks of
    the caller's expectation: terms, the MMA form; out_f16, a 16-bit output that must be fp16. autocast (fp16 weights
    only): round at every point where the layer under torch.autocast makes an fp16 tensor (FGT_OUT_HALF_AUTOCAST), so
    that every output, out_f32 included, holds fp16 values."""
    f16 = w_split.dtype == torch.float16
    assert terms is None or terms == (1 if f16 else 3), "terms=1 takes fp16 weights, terms=3 split-bf16 ones"
    assert not autocast or f16, "autocast rounding takes fp16 weights"
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
        a.plane = plane16(s.split)
        a.C, a.DX, a.DY, a.DZ = s.C, s.DX, s.DY, s.DZ
        a.sx, a.sy, a.sz = s.sx, s.sy, s.sz
        a.c_base, a.c_per_group, a.c_count = s.c_base, s.c_per_group, s.c_count
        k_real += s.c_count
    d.kx, d.ky, d.kz, d.stride, d.dil = kx, ky, kz, stride, dil
    d.pad_x, d.pad_y, d.pad_z = pad_x, pad_y, pad_z
    d.w_hi = w_split.data_ptr()
    d.w_plane = plane16(w_split)
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
        d.out_plane = plane16(out_split)
        d.out_half = 1 if out_split.dtype == torch.float16 else 0
        assert not autocast or d.out_half, "autocast rounding: the 16-bit output is fp16"
    if autocast:
        d.out_half = OUT_HALF_AUTOCAST
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
        call("fgt_gemm_tc", ctypes.byref(d))


def attention(q, k, v, out, *, batches, heads, Lq, Lk, Lk_rows=None, q_ld, k_ld, v_ld, out_ld,
              q_batch_stride, k_batch_stride, v_batch_stride, out_batch_stride, scale, mode=0,
              glob_start=0, glob_count=0, q_off=0, k_off=0, v_off=0, out_rowmap=None, tag=""):
    """fgt_attention launcher. q/k/v/out are split-bf16 row-major tensors, or all four plain fp16 tensors (the
    single-plane fp16 mode); strides in elements; q_off/k_off/v_off are element offsets into the plane (e.g. when Q,
    K and V share one [rows, 3*C] projection buffer)."""
    d = FgtAttnDesc()
    d.f16 = 1 if q.dtype == torch.float16 else 0
    d.q_hi, d.q_plane, d.q_batch_stride, d.q_ld = q.data_ptr() + 2 * q_off, plane16(q), q_batch_stride, q_ld
    d.k_hi, d.k_plane, d.k_batch_stride, d.k_ld = k.data_ptr() + 2 * k_off, plane16(k), k_batch_stride, k_ld
    d.v_hi, d.v_plane, d.v_batch_stride, d.v_ld = v.data_ptr() + 2 * v_off, plane16(v), v_batch_stride, v_ld
    d.out_hi, d.out_plane, d.out_batch_stride, d.out_ld = out.data_ptr(), plane16(out), out_batch_stride, out_ld
    d.batches, d.heads, d.head_dim = batches, heads, 128
    d.Lq, d.Lk = Lq, Lk
    d.Lk_rows = Lk if Lk_rows is None else Lk_rows
    d.scale, d.mode, d.glob_start, d.glob_count = scale, mode, glob_start, glob_count
    d.out_rowmap = out_rowmap.data_ptr() if out_rowmap is not None else None
    keys = Lk if mode == 0 else 64 + glob_count
    flops = 4.0 * batches * heads * Lq * keys * 128
    nbytes = 4.0 * batches * heads * 128 * (2 * Lq + 2 * (Lk if mode == 0 else d.Lk_rows))
    with _Prof("flash", tag, flops, nbytes):
        call("fgt_attention", ctypes.byref(d))


def pack_nchw(src0, src1, out_split, pad=0, tag=""):
    """[n,c0,H,W] (+ [n,c1,H,W]) fp32 -> NHWC split [2, n, H+2p, W+2p, cpad] with replication pad."""
    n, c0, H, W = src0.shape
    c1 = src1.shape[1] if src1 is not None else 0
    cpad = out_split.shape[-1]
    with _Prof("pack_nchw", tag, 0, 4.0 * n * (c0 + c1) * H * W + 4.0 * out_split[0].numel()):
        call("fgt_pack_nchw", src0, c0, src1, c1, n, H, W, pad, cpad, out_split, plane16(out_split, split_only=True))


def im2col_nchw(src0, src1, out_split, *, k, stride, pad, replicate, OH, OW, scale=1.0, shift=0.0, tag=""):
    """[n,c0,H,W] (+[n,c1,H,W]) fp32 -> [2, n, OH, OW, cpad] split rows of k*k*cin gathered inputs."""
    n, c0, H, W = src0.shape
    c1 = src1.shape[1] if src1 is not None else 0
    cpad = out_split.shape[-1]
    nbytes = 4.0 * n * (c0 + c1) * H * W + 2.0 * out_split.numel()
    with _Prof("im2col_nchw", tag, 0, nbytes):
        call("fgt_im2col_nchw", src0, c0, src1, c1, n, H, W, k, stride, pad, 1 if replicate else 0, OH, OW, cpad, scale,
             shift, out_split, plane16(out_split))


def rownorm(a, b, out_split, *, gather=None, rows_per_batch, total_rows, dst_batch_rows, dst_row0=0, eps=1e-5,
            gamma=None, beta=None, tag=""):
    """out_split: split-bf16 [2, ...] or a plain fp16 tensor (single-plane rows of a 1-term layer)."""
    ca, lda = a.shape[-1], a.shape[-1]
    cb, ldb = (b.shape[-1], b.shape[-1]) if b is not None else (0, 0)
    with _Prof("rownorm", tag, 0, 8.0 * total_rows * (ca + cb)):
        call("fgt_rownorm", a, ca, lda, b, cb, ldb, gather, rows_per_batch, total_rows, dst_batch_rows, dst_row0, gamma, beta,
             out_split, plane16(out_split), eps)


def rownorm_bcast(a, dst_ptrs, plane, *, gather=None, rows_per_batch, total_rows, dst_batch_rows, dst_row0=0, eps=1e-5,
                  gamma=None, beta=None, tag=""):
    """LayerNorm rows of `a` stored to every buffer in dst_ptrs (raw device addresses of split-bf16 buffers with
    the lo plane `plane` elements after the hi plane; local or peer-mapped)."""
    ca = a.shape[-1]
    arr = (ctypes.c_void_p * len(dst_ptrs))(*dst_ptrs)
    with _Prof("rownorm", tag, 0, 4.0 * total_rows * ca * (1 + len(dst_ptrs))):
        call("fgt_rownorm_bcast", a, ca, ca, None, 0, 0, gather, rows_per_batch, total_rows, dst_batch_rows, dst_row0, gamma,
             beta, arr, len(dst_ptrs), plane, eps)


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
        call("fgt_dwpool", a, ca, b, cb, bt, h, w, k, gh, gw, weight, bias, out)


def conv_tail(x_split, n, H, W, cin, w_split, cout, bias, act, out, *, nchw, tag=""):
    """3x3 conv (pad 1) with cout <= 3 + bias + activation: x_split [2,n,H,W,cin] -> out [n,cout,H,W] (nchw) or
    [n,H,W,cout] fp32, one kernel (taps-as-N GEMM + in-SM tap sum). w_split = pack_weight(pack_taps_as_n(w)).
    x_split and w_split may instead both be plain fp16 tensors (1-term fp16 MMAs)."""
    os_n, os_c, os_y, os_x = (cout * H * W, H * W, W, 1) if nchw else (H * W * cout, 1, W * cout, cout)
    # 2*9*cout*cin FLOP per 4*(cin+cout) bytes = ~13 FLOP/B at 64 -> 3: HBM-bound, reported against the copy roofline
    nbytes = 4.0 * n * H * W * (cin + cout)
    with _Prof("conv_tail", tag, 0.0, nbytes):
        call("fgt_conv_tail", x_split, plane16(x_split), n, H, W, cin, w_split, plane16(w_split), w_split.shape[-1], cout,
             bias, act, out, os_n, os_c, os_y, os_x)


def swin_prep(x, fp, bt, h, w, win_map, nl, R, gd, gh, gw, gk_w, gk_b, gv_w, gv_b, qkn, vn, eps=1e-5, tag=""):
    """SWMHSA operand preparation in one launch: LayerNorm'd window rows and pooled global rows of [x ; f'] -> qkn
    and of x -> vn (split-bf16 [bt*R, .], or both plain fp16); see include/fgt_b200.h."""
    d, df = x.shape[-1], fp.shape[-1]
    G = gh * gw
    nbytes = 4.0 * bt * ((nl + 2 * h * w) * (d + df) + (nl + G) * (2 * d + df))  # reads (rows + pooling) + split writes
    with _Prof("swin_prep", tag, 0, nbytes):
        call("fgt_swin_prep", x, fp, d, df, bt, h, w, win_map, nl, R, gd, gh, gw, gk_w, gk_b, gv_w, gv_b, qkn, plane16(qkn),
             vn, plane16(vn), eps)


def dwconv3x3_res(x, bt, h, w, C, weight, bias, out, out_split=None, tag=""):
    """out_split (optional 16-bit copy): split-bf16 or plain fp16."""
    with _Prof("dwconv3x3_res", tag, 0, 12.0 * bt * h * w * C):
        call("fgt_dwconv3x3_res", x, bt, h, w, C, weight, bias, out, out_split, plane16(out_split))


def fold(hid, bt, th, tw, C, kh, kw, stride, pad, OH, OW, *, normalize, add=None, out=None, out_split=None, tag=""):
    """out_split (optional 16-bit output): split-bf16 or plain fp16."""
    with _Prof("fold", tag, 0, 4.0 * bt * (th * tw * kh * kw * C + OH * OW * C * (2 if add is not None else 1))):
        call("fgt_fold", hid, bt, th, tw, C, kh, kw, stride, pad, OH, OW, 1 if normalize else 0, add, out, out_split,
             plane16(out_split))


def unfold(img, bt, th, tw, C, kh, kw, stride, pad, OH, OW, out_split, relu=True, tag=""):
    with _Prof("unfold", tag, 0, 4.0 * bt * (th * tw * kh * kw * C + OH * OW * C)):
        call("fgt_unfold", img, bt, th, tw, C, kh, kw, stride, pad, OH, OW, 1 if relu else 0, out_split,
             plane16(out_split, split_only=True))


def fold_unfold(hid, bt, th, tw, C, kh, kw, stride, pad, OH, OW, out_split, relu=True, tag=""):
    """fold (normalised) + unfold (+ReLU) of the fusion FFN in one launch: hid fp32 [bt*th*tw, kh*kw*C] -> split-bf16
    (or plain fp16)."""
    with _Prof("fold_unfold", tag, 0, 8.0 * bt * th * tw * kh * kw * C):
        call("fgt_fold_unfold", hid, bt, th, tw, C, kh, kw, stride, pad, OH, OW, 1 if relu else 0, out_split,
             plane16(out_split))


def upsample2x(in_split, n, H, W, C, out_split, tag=""):
    """Nearest x2 of NHWC [n, H, W, C]: split-bf16 in and out, or plain fp16 in and out."""
    with _Prof("upsample2x", tag, 0, (2.5 if in_split.dtype == torch.float16 else 5.0) * n * H * W * C * 4):
        call("fgt_upsample2x", in_split, plane16(in_split), n, H, W, C, out_split, plane16(out_split))


# ------------------------------------------------------------------------------------------ RAFT helpers
def chan_stats(x, n, HW, C, stats, tag=""):
    with _Prof("chan_stats", tag, 0, 4.0 * n * HW * C):
        call("fgt_chan_stats", x, n, HW, C, stats)


def instnorm_act(x, stats, n, HW, C, *, relu=True, res=None, out=None, out_split=None, eps=1e-5, tag=""):
    """out_split: split-bf16 [2, ...] or a plain fp16 tensor (single-plane rows of a 1-term layer)."""
    with _Prof("instnorm_act", tag, 0, 4.0 * n * HW * C * (3 if res is not None else 2)):
        call("fgt_instnorm_act", x, stats, n, HW, C, eps, 1 if relu else 0, res, out, out_split, plane16(out_split))


def avgpool2(src, rows, h, w, dst, tag=""):
    with _Prof("avgpool2", tag, 0, 5.0 * rows * h * w):
        call("fgt_avgpool2", src, rows, h, w, dst)


def corr_lookup(levels, coords, n_pix, radius, out_split, tag=""):
    """levels: list of fp32 tensors [n_pix, h_l, w_l]; out_split: split-bf16 [2, n_pix, pitch] or fp16 [n_pix, pitch]."""
    nl = len(levels)
    ptrs = (ctypes.c_void_p * nl)(*[t.data_ptr() for t in levels])
    hs = (ctypes.c_int * nl)(*[t.shape[1] for t in levels])
    ws = (ctypes.c_int * nl)(*[t.shape[2] for t in levels])
    win = 2 * radius + 1
    with _Prof("corr_lookup", tag, 0, 4.0 * n_pix * nl * ((win + 1) ** 2 + win * win)):
        call("fgt_corr_lookup", ptrs, hs, ws, nl, radius, coords, n_pix, out_split.shape[-1], out_split,
             plane16(out_split))


def raft_flow_update(coords, delta, h, w, flow_nchw, x_split=None, x_chan=0, n=1, delta_f16=False, tag=""):
    """x_split: split-bf16 GRU input, or fp16 for the mixed-precision path; delta_f16: round delta to fp16 first."""
    with _Prof("raft_flow_update", tag, 0, 32.0 * n * h * w):
        call("fgt_raft_flow_update", coords, delta, 1 if delta_f16 else 0, n, h, w, flow_nchw, x_split, plane16(x_split),
             x_split.shape[-1] if x_split is not None else 0, x_chan)


def convex_upsample(mask, flow_nchw, h, w, out, n=1, tag=""):
    with _Prof("convex_upsample", tag, 0, 4.0 * n * h * w * (576 + 128)):
        call("fgt_convex_upsample", mask, flow_nchw, n, h, w, out)


def upflow8(flow_nchw, h, w, out, n=1, tag=""):
    """8 * bilinear x8 upsampling (align_corners=True) of [n,2,h,w] fp32 flow into out [n,2,8h,8w] fp32."""
    with _Prof("upflow8", tag, 0, 4.0 * n * 2 * h * w * 65):
        call("fgt_upflow8", flow_nchw, n, h, w, out)


def f16_to_split(src, out_split, tag=""):
    """fp16 tensor -> split-bf16 [2, ...] of the same element count (exact)."""
    with _Prof("f16_to_split", tag, 0, 6.0 * src.numel()):
        call("fgt_f16_to_split", src, src.numel(), out_split, plane16(out_split, split_only=True))
