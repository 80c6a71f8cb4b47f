"""One-time weight preparation for the tensor-core engine (runs at load_state_dict time, not on the
hot path): re-orders conv / linear weights into the engine's K-iteration order and splits them into
bf16 hi/lo planes.

K-iteration order (must match gemm_tc.cu): taps z-major, then y, then x; inside a tap the channel
segments in order; each (tap, segment) block zero-padded to a multiple of 64 channels.
"""
import torch

from .lib import to_split

KB = 64


def pad64(c):
    return (c + KB - 1) // KB * KB


def pack_weight(w, seg_counts=None, half=False):
    """w: [N, Cin_per_group, *taps] (torch conv layout; taps = (), (kh,kw) or (kt,kh,kw)).

    seg_counts: channels per group taken from each A segment (sum == Cin_per_group).
    Returns split-bf16 tensor [2, N, k_pad], or a plain fp16 [N, k_pad] for a 1-term layer (half=True).
    """
    w = w.detach().float()
    n, cin = w.shape[0], w.shape[1]
    taps = 1
    for s in w.shape[2:]:
        taps *= s
    if seg_counts is None:
        seg_counts = [cin]
    assert sum(seg_counts) == cin, (seg_counts, cin)
    w = w.reshape(n, cin, taps).permute(0, 2, 1)  # [N, taps, Cin]
    blocks = []
    c0 = 0
    for c in seg_counts:
        blk = w[:, :, c0:c0 + c]
        if pad64(c) != c:
            blk = torch.nn.functional.pad(blk, (0, pad64(c) - c))
        blocks.append(blk)
        c0 += c
    packed = torch.cat(blocks, dim=2).reshape(n, -1).contiguous()
    return packed.to(torch.float16) if half else to_split(packed)


def fold_layernorm(weight, bias, gamma, beta, half=False):
    """Folds a LayerNorm affine (gamma, beta) that precedes Linear(weight, bias) into the Linear:
    W (gamma * n + beta) + b == (W * gamma) n + (W beta + b). Computed in fp64, rounded once to fp32 (or, half=True,
    to fp16 values, returned as fp32 tensors)."""
    w = weight.detach().double()
    g = gamma.detach().double()
    b = beta.detach().double()
    w2 = w * g[None, :]
    b2 = w @ b + (bias.detach().double() if bias is not None else 0.0)
    if half:
        return w2.half().float(), b2.half().float()
    return w2.float(), b2.float()


def pack_weight_im2col(w, cpad=KB, half=False):
    """Conv weight [N, cin, k, k] for a layer whose input was gathered by fgt_im2col_nchw:
    K index = (ky*k + kx)*cin + c, zero-padded to cpad."""
    w = w.detach().float()
    n = w.shape[0]
    flat = w.permute(0, 2, 3, 1).reshape(n, -1)
    assert flat.shape[1] <= cpad
    flat = torch.nn.functional.pad(flat, (0, cpad - flat.shape[1])).contiguous()
    return flat.to(torch.float16) if half else to_split(flat)
