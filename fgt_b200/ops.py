"""Launch helpers shared by the FGT / LAFC / RAFT host modules: NHWC convolutions and row-major linears on the
tensor-core engine (fgt_gemm_tc), with the tile heuristics in one place."""
import functools

from . import lib
from .packing import pack_weight, pack_weight_im2col

# Output boxes the GEMM engine takes: box_w x box_h <= 128 positions, a multiple of 8 (the 8-row swizzle atom of the
# A tile). Five 128-position boxes come first and the rest by size, so a tie in tile count keeps the larger box.
_FIRST = ((16, 8), (32, 4), (8, 16), (64, 2), (128, 1))
_BOXES = _FIRST + tuple(sorted(((bw, bh) for bh in range(1, 129) for bw in range(1, 128 // bh + 1)
                                if bw * bh % 8 == 0 and (bw, bh) not in _FIRST),
                               key=lambda b: (-b[0] * b[1], -b[0])))


@functools.lru_cache(maxsize=None)
def pick_box(ow, oh):
    """Output box (box_w, box_h) for an ow x oh map: the fewest tiles, since every tile runs 128 MMA rows whatever its
    box holds (the 20 x 36 token grid: 12 x 10, 6 tiles instead of 9 with 16 x 8). The box may be wider or taller than
    the map."""
    return min(_BOXES, key=lambda b: -(-ow // b[0]) * -(-oh // b[1]))


# Channel-tile (bn) policy of the conv networks (LAFC, RAFT): halve a 128-wide tile while the launch has fewer tiles
# than SMs. FGT passes its own policy (fgt_model._tile: halve while the launch covers at most half a wave, down to 64);
# the two differ on purpose, each tuned on its own networks' shapes.
def pick_bn(n_per_group, groups=1):
    if n_per_group % 128 == 0:
        return 128
    if n_per_group % 96 == 0 and n_per_group <= 384:
        return 96
    if n_per_group <= 128:
        return (n_per_group + 15) // 16 * 16 if groups == 1 else n_per_group
    if groups > 1:
        for bn in (96, 80, 64, 48, 32, 16):
            if n_per_group % bn == 0:
                return bn
    return 128


def fill_sms(bn, n_total, m_positions, groups=1, n_sms=132):
    """Small-M problems (RAFT's 1/8-resolution update block: 51 tiles of 128 positions) leave most SMs idle
    with 128-wide channel tiles; halve the tile while that raises the number of busy SMs."""
    m_tiles = -(-m_positions // 128)
    while bn >= 128 and bn % 32 == 0 and m_tiles * -(-n_total // bn) < n_sms and (groups == 1 or (n_total // groups) % (bn // 2) == 0):
        bn //= 2
    return bn


def conv_tile(n_total, groups, m_positions):
    return fill_sms(pick_bn(n_total // groups, groups), n_total, m_positions, groups)


def packed(name, weight, bias, dev, seg_counts=None, im2col_pad=None, half=False):
    """Weight record consumed by conv()/linear(): split-bf16 packed weight + fp32 bias. half=True: fp16 packed weight,
    which makes the layer a 1-term one (its A operands are single-plane fp16 tensors)."""
    if im2col_pad is not None:
        w = pack_weight_im2col(weight, im2col_pad, half=half)
    else:
        w = pack_weight(weight, seg_counts, half=half)
    return dict(w=w.to(dev), b=bias.detach().float().contiguous().to(dev), N=weight.shape[0], name=name)


def conv(xs, wp, *, kx=1, ky=1, kz=1, stride=1, dil=1, pad_x=0, pad_y=0, pad_z=0, out_z=None, act=lib.ACT_LEAKY02,
         out_split=None, out_f32=None, aux=None, aux_mode=lib.AUX_NONE, groups=1, seg_counts=None, nchw_out=False,
         alpha=1.0, aux2=None, out_c_total=None, out_c_offset=0, out_phase=None, tile=conv_tile, bn=None, alg_k=None):
    """xs: list of (split tensor [2, Z, Y, X, C], C) sharing Z/Y/X, or of fp16 tensors [Z, Y, X, C] for a layer with
    fp16 weights. Output NHWC [Z', Y', X', N] (or NCHW fp32 when nchw_out). out_phase=(py, px): the output is one
    phase of a 2x upsampled map, pixel (y, x) stored at (2y+py, 2x+px) of [Z, 2Y, 2X, N]. The channel tile is `bn`,
    or the caller's policy `tile`. Returns (oz, oy, ox)."""
    x0, c0 = xs[0]
    Z, Y, X = x0.shape[-4], x0.shape[-3], x0.shape[-2]
    if out_phase is None:
        oy = (Y + 2 * pad_y - dil * (ky - 1) - 1) // stride + 1
        ox = (X + 2 * pad_x - dil * (kx - 1) - 1) // stride + 1
    else:
        oy, ox = Y, X
    oz = (Z + 2 * pad_z - (kz - 1)) if out_z is None else out_z
    N = wp["N"]
    segs = []
    for i, (t, c) in enumerate(xs):
        cnt = c if seg_counts is None else seg_counts[i]
        segs.append(lib.ASeg(t, c, X, Y, Z, c_per_group=(cnt if groups > 1 else 0), c_count=cnt))
    bw, bh = pick_box(ox, oy)
    if nchw_out:
        strides = dict(os_z=N * oy * ox, os_y=ox, os_x=1, os_c=oy * ox)
    elif out_phase is not None:
        py, px = out_phase
        strides = dict(os_z=4 * oy * ox * N, os_y=4 * ox * N, os_x=2 * N, os_c=1, out_elem_offset=(py * 2 * ox + px) * N)
    else:
        ct = N if out_c_total is None else out_c_total  # write into a channel slice of a wider NHWC buffer
        strides = dict(os_z=oy * ox * ct, os_y=ox * ct, os_x=ct, os_c=1, out_elem_offset=out_c_offset)
    lib.gemm_tc(segs, wp["w"], N, kx=kx, ky=ky, kz=kz, stride=stride, dil=dil, pad_x=pad_x, pad_y=pad_y, pad_z=pad_z,
                groups=groups, out_w=ox, out_h=oy, out_z=oz, box_w=bw, box_h=bh,
                bn=tile(N, groups, ox * oy * oz) if bn is None else bn,
                bias=wp["b"], alpha=alpha, act=act, aux=aux, aux_mode=aux_mode, aux2=aux2, out_f32=out_f32, out_split=out_split,
                tag=wp["name"], alg_k=alg_k, **strides)
    return oz, oy, ox


def linear(segs, wp, rows, *, tile=conv_tile, bn=None, **kw):
    """segs: list of (split tensor [2, rows, C], C), or of fp16 [rows, C] for a layer with fp16 weights. Row-major
    [rows, N] outputs. The channel tile is `bn`, or the caller's policy `tile`."""
    asegs = [lib.ASeg(t, c, rows) for t, c in segs]
    lib.gemm_tc(asegs, wp["w"], wp["N"], out_w=rows, bn=tile(wp["N"], 1, rows) if bn is None else bn,
                bias=wp["b"], tag=wp["name"], **kw)
