"""GPU bring-up diagnostic for the wgmma GEMM engine: runs cases from trivial to complex and
prints error statistics (and error structure for the first failure). Run under gpurun."""
import sys
import os
import traceback

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import lib, packing  # noqa: E402

dev = torch.device("cuda:0")
torch.manual_seed(0)


def report(name, got, ref, tol=2e-4):
    got = got.double().cpu()
    ref = ref.double().cpu()
    err = (got - ref).abs()
    rel = (got - ref).norm() / (ref.norm() + 1e-30)
    mx = err.max().item() / (ref.abs().max().item() + 1e-30)
    ok = rel < tol and mx < tol and torch.isfinite(got).all()
    print(f"[{'OK' if ok else 'FAIL'}] {name}: rel_l2={rel:.3e} max/max={mx:.3e} shape={tuple(got.shape)}", flush=True)
    if not ok:
        g2 = got.reshape(-1, got.shape[-1])
        r2 = ref.reshape(-1, ref.shape[-1])
        e2 = (g2 - r2).abs()
        print("  row err (first 16 rows):", [f"{v:.2e}" for v in e2.max(1).values[:16].tolist()])
        print("  col err (first 16 cols):", [f"{v:.2e}" for v in e2.max(0).values[:16].tolist()])
        print("  got[0,:8]", g2[0, :8].tolist())
        print("  ref[0,:8]", r2[0, :8].tolist())
        print("  nan count", torch.isnan(g2).sum().item(), "zeros", (g2 == 0).sum().item(), "/", g2.numel())
    return ok


def linear_case(M, N, K, bn=128, bias=True, act=lib.ACT_NONE, split_out=False, aux_mode=lib.AUX_NONE, scale=1.0,
                split_only=False, terms=3):
    """split_only: the 16-bit output alone (the launch then stores through shared memory + TMA, like an fp32-only
    launch); terms=1: single-plane fp16 operands (and, with split_only, a single-plane fp16 output), checked against
    the product of the fp16-rounded operands."""
    a = torch.randn(M, K, device=dev) * scale
    w = torch.randn(N, K, device=dev) / K ** 0.5
    b = torch.randn(N, device=dev) if bias else None
    one = terms == 1
    a_s = a.half().contiguous() if one else lib.to_split(a)
    w_s = packing.pack_weight(w, half=one).to(dev)
    out = None if split_only else torch.full((M, N), float("nan"), device=dev)
    out_s = out_h = None
    if one and split_only:
        out_h = torch.full((M, N), float("nan"), dtype=torch.float16, device=dev)
    elif split_out or split_only:
        out_s = lib.empty_split((M, N), dev)
        out_s.fill_(float("nan"))
    aux = torch.randn(M, N, device=dev) if aux_mode else None
    lib.gemm_tc([lib.ASeg(a_s, K, M)], w_s, N, out_w=M, bn=bn, bias=b, act=act, out_f32=out, out_split=out_s,
                out_f16=out_h, aux=aux, aux_mode=aux_mode, terms=terms)
    torch.cuda.synchronize()
    if one:
        ref = a.half().double() @ w.half().double().t()
    else:
        ref = a.double() @ w.double().t()
    if bias:
        ref = ref + b.double()
    if act == lib.ACT_LEAKY02:
        ref = F.leaky_relu(ref, 0.2)
    elif act == lib.ACT_RELU:
        ref = F.relu(ref)
    elif act == lib.ACT_SIGMOID:
        ref = torch.sigmoid(ref)
    elif act == lib.ACT_TANH:
        ref = torch.tanh(ref)
    if aux_mode == lib.AUX_ADD:
        ref = ref + aux.double()
    elif aux_mode == lib.AUX_MUL:
        ref = ref * aux.double()
    name = f"linear M={M} N={N} K={K} bn={bn} act={act} aux={aux_mode} terms={terms}"
    if split_only and one:
        return report(name + " fp16-only", out_h, ref, tol=1e-3)  # the fp16 store itself rounds to 2^-12
    if split_only:
        return report(name + " split-only", lib.from_split(out_s), ref)
    ok = report(name, out, ref)
    if split_out:
        ok &= report("  split output", lib.from_split(out_s), ref, tol=2e-4)
    return ok


def conv_case(n, h, w, cin, cout, k, stride=1, pad=None, dil=1, groups=1, bn=64, box=(16, 8), act=lib.ACT_LEAKY02,
              split_only=False, terms=3):
    pad = (k // 2) * dil if pad is None else pad
    x = torch.randn(n, cin, h, w, device=dev)
    wt = torch.randn(cout, cin // groups, k, k, device=dev) / (cin // groups * k * k) ** 0.5
    b = torch.randn(cout, device=dev)
    xr, wr = (x.half(), wt.half()) if terms == 1 else (x, wt)
    ref = F.conv2d(xr.double(), wr.double(), b.double(), stride=stride, padding=pad, dilation=dil, groups=groups)
    if act == lib.ACT_LEAKY02:
        ref = F.leaky_relu(ref, 0.2)
    oh, ow = ref.shape[2], ref.shape[3]
    one = terms == 1
    xn = x.permute(0, 2, 3, 1).contiguous()
    x_s = xn.half() if one else lib.to_split(xn)  # [2, n, h, w, c] split-bf16, or [n, h, w, c] fp16
    w_s = packing.pack_weight(wt, half=one).to(dev)
    out = torch.full((n, oh, ow, cout), float("nan"), device=dev)
    out_s = out_h = None
    if split_only and one:
        out_h = torch.full((n, oh, ow, cout), float("nan"), dtype=torch.float16, device=dev)
    elif split_only:
        out_s = lib.empty_split((n, oh, ow, cout), dev)
        out_s.fill_(float("nan"))
    seg = lib.ASeg(x_s, cin, w, h, n, c_per_group=(cin // groups if groups > 1 else 0), c_count=cin // groups)
    lib.gemm_tc([seg], w_s, cout, kx=k, ky=k, stride=stride, dil=dil, pad_x=pad, pad_y=pad, groups=groups,
                out_w=ow, out_h=oh, out_z=n, box_w=box[0], box_h=box[1], bn=bn, bias=b, act=act,
                out_f32=None if split_only else out, out_split=out_s, out_f16=out_h,
                os_z=oh * ow * cout, os_y=ow * cout, os_x=cout, os_c=1, terms=terms)
    torch.cuda.synchronize()
    if split_only:
        out = out_h.float() if one else lib.from_split(out_s)
    return report(f"conv n={n} {h}x{w} cin={cin} cout={cout} k={k} s={stride} p={pad} d={dil} g={groups} bn={bn} "
                  f"terms={terms}", out.permute(0, 3, 1, 2), ref, tol=1e-3 if (one and split_only) else 2e-4)


def main():
    print(torch.cuda.get_device_name(0), "lib version", lib.load().fgt_version(), flush=True)
    cases = [
        lambda: linear_case(128, 128, 64, bias=False),
        lambda: linear_case(128, 128, 128, bias=False),
        lambda: linear_case(128, 64, 512, bn=64),
        lambda: linear_case(256, 256, 512, bn=128),
        lambda: linear_case(1000, 520, 1960, bn=128, act=lib.ACT_RELU, split_out=True),
        lambda: linear_case(7200, 1536, 512, bn=256, aux_mode=lib.AUX_ADD),
        lambda: linear_case(300, 48, 200, bn=48, act=lib.ACT_SIGMOID, aux_mode=lib.AUX_MUL),
        lambda: linear_case(40000, 512, 512, bn=128, scale=3.0),
        lambda: linear_case(7200, 1960, 512, bn=128),                                  # N tail (partial tile)
        lambda: linear_case(1000, 520, 1960, bn=128, act=lib.ACT_RELU, split_only=True, aux_mode=lib.AUX_ADD),
        lambda: linear_case(7200, 1536, 512, bn=128, split_only=True),
        lambda: linear_case(333, 256, 320, bn=256, split_only=True, act=lib.ACT_SIGMOID, aux_mode=lib.AUX_MUL),
        lambda: linear_case(7200, 256, 768, bn=128, terms=1, split_only=True),
        lambda: linear_case(1000, 192, 576, bn=64, terms=1, act=lib.ACT_LEAKY02),       # fp16 operands, fp32 output
        lambda: linear_case(2000, 256, 6272, bn=128, terms=1, split_out=True),          # f_patch2vec shape: two outputs
        lambda: conv_case(2, 61, 107, 64, 128, 3, stride=2, bn=128, split_only=True),
        lambda: conv_case(2, 60, 108, 128, 128, 3, bn=128, terms=1, split_only=True),
        lambda: conv_case(1, 16, 32, 64, 64, 3),
        lambda: conv_case(2, 60, 108, 128, 256, 3, bn=128),
        lambda: conv_case(2, 61, 107, 64, 128, 3, stride=2, bn=128),
        lambda: conv_case(1, 60, 108, 128, 512, 7, stride=3, pad=3, bn=128, act=lib.ACT_NONE),
        lambda: conv_case(1, 30, 54, 192, 192, 3, dil=4, bn=64),
        lambda: conv_case(2, 24, 40, 128, 256, 3, groups=2, bn=128),
        lambda: conv_case(1, 24, 40, 8, 64, 3, bn=64),
        lambda: conv_case(1, 20, 36, 64, 3, 3, bn=16, act=lib.ACT_NONE),
    ]
    nfail = 0
    for c in cases:
        try:
            if not c():
                nfail += 1
        except Exception:
            traceback.print_exc()
            nfail += 1
            break
    print("FAILURES:", nfail, flush=True)
    return 1 if nfail else 0


if __name__ == "__main__":
    sys.exit(main())
