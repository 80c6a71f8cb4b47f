"""A float64 interpreter of one `fgt_gemm_tc` descriptor (include/fgt_b200.h), for CPU tensors.

`emulating()` swaps the library `lib.load()` returns for this interpreter, the way tests/test_launch_trace.py swaps it
for its recorder, so the production launchers (`ops.conv`, `ops.linear`, `lib.gemm_tc`) fill their descriptors as they
do on the GPU and the interpreter executes them on CPU tensors. Every pointer is resolved to a live CPU tensor's storage
plus an offset. `fgt_gemm_tc` is the only entry served: calling any other entry while the interpreter is installed is
an error.

Semantics, restated from the header and the engine rather than from its code paths:
- A operands: segment `s`, group `g` reads channels [c_base + g * c_per_group, + 64 * ceil(c_count / 64)); channels
  at or beyond C read 0 (the TMA box), channels past c_count but below C are read from the tensor (their weights are
  the packing's zeros). Input positions are `out * stride + tap * dil - pad` in x and y and `out + tap - pad_z` in z,
  computed directly (no stride-phase views); positions outside [0, DX) x [0, DY) x [0, DZ) read 0.
- K order: taps z-major, then y, then x; inside a tap the segments in order (packing.py).
- Products in float64 of the operands as stored: hi + lo for split-bf16, the fp16 value for 1-term layers.
- Epilogue: v = acc * alpha + bias, then the activation / aux modes in the order of the engine's per-pair epilogue,
  with the fp16 roundings of the extended (kExt = 1) instantiation where it applies. Stores: fp32 values rounded once,
  split-bf16 as `lib.to_split`, fp16 rounded to nearest.
- Only the elements the descriptor addresses are written (rowmap < 0 rows, rows past out_w and N tails are not).
Each launch appends {"v": float64 [out_z, out_h, out_w, N] values before the store rounding, "desc": the descriptor}
to `emulator.launches`, so tests can compare the arithmetic itself with a float64 reference; `written_mask(t)` gives
the elements of a buffer the stores addressed.
"""
import contextlib

import torch

from fgt_b200 import lib
from tests.test_launch_trace import _Recorder, recording


class _Refused:
    def __init__(self, name):
        self.name, self.argtypes, self.restype = name, None, None

    def __call__(self, *args):
        raise AssertionError(f"{self.name} called while the fgt_gemm_tc emulator is installed")


class _GemmEntry:
    def __init__(self, emu):
        self.emu, self.argtypes, self.restype = emu, None, None

    def __call__(self, desc_ref, stream):
        self.emu.run(desc_ref._obj)
        return 0


def _r16(x):
    return x.half().double()


def _act(v, act):
    if act == lib.ACT_LEAKY02:
        return torch.where(v > 0, v, 0.2 * v)
    if act == lib.ACT_LEAKY001:
        return torch.where(v > 0, v, 0.01 * v)
    if act == lib.ACT_RELU:
        return v.clamp_min(0.0)
    if act == lib.ACT_SIGMOID:
        return 1.0 / (1.0 + torch.exp(-v))
    if act == lib.ACT_TANH:
        return torch.tanh(v)
    assert act == lib.ACT_NONE, act
    return v


class GemmEmulator(_Recorder):
    """Stands in for the ctypes library: `fgt_gemm_tc` runs in float64 on the CPU, every other entry is refused."""

    def __init__(self):
        super().__init__()
        self.launches = []
        self.written = []   # (flat view, element indices) of every store

    def __getattr__(self, name):
        if not name.startswith("fgt_"):
            raise AttributeError(name)
        e = _GemmEntry(self) if name == "fgt_gemm_tc" else _Refused(name)
        setattr(self, name, e)
        return e

    def flat(self, p, dtype):
        """1-D `dtype` view of the storage behind address p, starting at p."""
        _, i, off = self._ptr(p)
        st = self._storages[i][2].untyped_storage()
        es = torch.empty((), dtype=dtype).element_size()
        assert off % es == 0, "misaligned pointer"
        return torch.empty(0, dtype=dtype).set_(st, off // es, ((st.nbytes() - off) // es,), (1,))

    def _plane_pair(self, p, plane, shape, strides, f16):
        """float64 values of a 16-bit operand: the fp16 plane, or hi + lo of a split-bf16 pair."""
        fl = self.flat(p, torch.float16 if f16 else torch.bfloat16)
        hi = fl.as_strided(shape, strides, fl.storage_offset()).double()
        if f16:
            return hi
        return hi + fl.as_strided(shape, strides, fl.storage_offset() + plane).double()

    def run(self, d):
        f16 = d.terms == 1
        assert d.terms in (0, 1, 3), d.terms
        s, dil = d.stride, d.dil
        oz = torch.arange(d.out_z)
        oy = torch.arange(d.out_h)
        ox = torch.arange(d.out_w)
        M = d.out_z * d.out_h * d.out_w
        W = self._plane_pair(d.w_hi, d.w_plane, (d.N, d.k_pad), (d.k_pad, 1), f16)
        segs = []
        for i in range(d.num_segs):
            sg = d.seg[i]
            A = self._plane_pair(sg.hi, sg.plane, (sg.DZ, sg.DY, sg.DX, sg.C), (sg.sz, sg.sy, sg.sx, 1), f16)
            segs.append((sg, A, -(-sg.c_count // 64) * 64))
        k_blk = sum(w for _, _, w in segs)
        assert d.kx * d.ky * d.kz * k_blk == d.k_pad, "k_pad does not match the taps and segments"
        cpg = d.N // d.groups
        acc = torch.zeros(M, d.N, dtype=torch.float64)
        k0 = 0
        for tz in range(d.kz):
            for ty in range(d.ky):
                for tx in range(d.kx):
                    for sg, A, width in segs:
                        iz = oz + tz - d.pad_z
                        iy = oy * s + ty * dil - d.pad_y
                        ix = ox * s + tx * dil - d.pad_x
                        ok = (((iz >= 0) & (iz < sg.DZ))[:, None, None] & ((iy >= 0) & (iy < sg.DY))[None, :, None]
                              & ((ix >= 0) & (ix < sg.DX))[None, None, :]).reshape(M, 1)
                        X = A[iz.clamp(0, sg.DZ - 1)[:, None, None], iy.clamp(0, sg.DY - 1)[None, :, None],
                              ix.clamp(0, sg.DX - 1)[None, None, :]].reshape(M, sg.C)
                        for g in range(d.groups):
                            ch = sg.c_base + g * sg.c_per_group + torch.arange(width)
                            assert int(ch[0]) >= 0
                            x = torch.where(ok & (ch < sg.C)[None, :], X[:, ch.clamp(max=sg.C - 1)], 0.0)
                            cols = slice(g * cpg, (g + 1) * cpg)
                            acc[:, cols] += x @ W[cols, k0:k0 + width].t()
                        k0 += width
        v = acc * float(d.alpha)
        if d.bias:
            v = v + self.flat(d.bias, torch.float32)[:d.N].double()
        self._epilogue(d, v, oz, oy, ox)

    def _epilogue(self, d, v, oz, oy, ox):
        M, N = v.shape
        mode, out_half = d.aux_mode, bool(d.out_half)
        ext = (mode in (lib.AUX_ADD_PRE, lib.AUX_ADD_RELU, lib.AUX_GRU, lib.AUX_GRU_ZR) or d.act == lib.ACT_LEAKY001
               or (out_half and bool(d.out_f32)))
        # output element offset of each row; rows a rowmap drops or past the map are not stored
        if d.rowmap or d.lin_batch:
            assert d.out_h == 1 and d.out_z == 1 and d.box_h == 1, "rowmap / lin_batch need linear mode"
            rows = torch.arange(d.out_w, dtype=torch.int64)
            if d.rowmap:
                rows = self.flat(d.rowmap, torch.int32)[:d.out_w].long()
            keep = rows >= 0
            if d.lin_batch > 0:
                off = (rows // d.lin_batch) * d.os_z + (rows % d.lin_batch) * d.os_x
            else:
                off = rows * d.os_x
        else:
            off = (oz[:, None, None] * d.os_z + oy[None, :, None] * d.os_y + ox[None, None, :] * d.os_x).reshape(M)
            keep = torch.ones(M, dtype=torch.bool)
        col = torch.arange(N, dtype=torch.int64)
        O = off[:, None] + col[None, :] * d.os_c

        def aux(p, at):
            return self.flat(p, torch.float32)[at].double()

        if mode == lib.AUX_GRU_ZR:
            half = N // 2
            assert ext and d.os_c == 1 and d.out_f32 and d.out_hi and d.groups == 1
            if out_half:
                v = _r16(v)
            v = _act(v, d.act)
            if out_half:
                v = _r16(v)
            Orh = off[:, None] + col[None, half:] - half
            v = torch.cat([v[:, :half], v[:, half:] * aux(d.aux, Orh)], 1)
            self._store(d, v[keep][:, :half], O[keep][:, :half], None, None)
            self._store(d, None, None, v[keep][:, half:], Orh[keep])
            self.launches.append(dict(v=v.reshape(d.out_z, d.out_h, d.out_w, N), desc=d))
            return
        if ext and mode == lib.AUX_ADD_PRE:
            v = v + aux(d.aux, O)
        if ext and out_half:
            v = _r16(v)
        v = _act(v, d.act)
        if ext and out_half and mode == lib.AUX_GRU:
            v = _r16(v)
        if mode == lib.AUX_ADD:
            v = v + aux(d.aux, O)
        elif mode == lib.AUX_MUL:
            v = v * aux(d.aux, O)
        elif mode == lib.AUX_ADD_RELU:
            if out_half:
                v = _r16(v)
            v = (v + aux(d.aux, O)).clamp_min(0.0)
        elif mode == lib.AUX_GRU:   # h' = (1 - z) h + z q
            h, z = aux(d.aux, O), aux(d.aux2, O)
            if out_half:
                v = _r16(_r16(_r16(1.0 - z) * h) + _r16(z * v))
            else:
                v = (1.0 - z) * h + z * v
        else:
            assert mode in (lib.AUX_NONE, lib.AUX_ADD_PRE), mode
        if ext and out_half:
            v = _r16(v)
        self._store(d, v[keep], O[keep], v[keep], O[keep])
        self.launches.append(dict(v=v.reshape(d.out_z, d.out_h, d.out_w, N), desc=d))

    def written_mask(self, t):
        """Boolean mask of the elements of contiguous tensor `t` that a store of the emulated launches addressed."""
        mask = torch.zeros(t.numel(), dtype=torch.bool)
        base = t.untyped_storage().data_ptr()
        for fl, idx in self.written:
            if fl.untyped_storage().data_ptr() != base or fl.dtype != t.dtype:
                continue
            pos = fl.storage_offset() + idx - t.storage_offset()
            mask[pos[(pos >= 0) & (pos < t.numel())]] = True
        return mask.view(t.shape)

    def _store(self, d, v32, o32, v16, o16):
        """fp32 values v32 at offsets o32 of out_f32, 16-bit values v16 at o16 of out_hi (fp16 or split-bf16)."""
        if d.out_f32 and v32 is not None:
            fl = self.flat(d.out_f32, torch.float32)
            fl[o32.reshape(-1)] = v32.reshape(-1).float()
            self.written.append((fl, o32.reshape(-1)))
        if d.out_hi and v16 is not None:
            if d.out_half:
                fl = self.flat(d.out_hi, torch.float16)
                fl[o16.reshape(-1)] = v16.reshape(-1).half()
                self.written.append((fl, o16.reshape(-1)))
            else:
                sp = lib.to_split(v16.reshape(-1).float())
                fl = self.flat(d.out_hi, torch.bfloat16)
                fl[o16.reshape(-1)] = sp[0]
                fl[o16.reshape(-1) + d.out_plane] = sp[1]
                self.written.append((fl, o16.reshape(-1)))
                self.written.append((fl, o16.reshape(-1) + d.out_plane))


@contextlib.contextmanager
def emulating():
    """`with emulating() as emu:` runs every fgt_gemm_tc launch of the block through the float64 interpreter."""
    emu = GemmEmulator()
    with recording(emu):
        yield emu
