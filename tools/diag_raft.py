"""GPU bring-up diagnostic for RAFT: compares the sm_90a path with the CPU oracle per iteration count."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fgt_b200 import synth  # noqa: E402
from fgt_b200.raft_model import RAFT  # noqa: E402
from oracle import raft_oracle as RO  # noqa: E402


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item(), ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


def run(H, W, iters, seed=3):
    sd = synth.raft_state_dict(seed=seed)
    m = RAFT(argparse.Namespace(small=False, mixed_precision=False, alternate_corr=False))
    m.load_state_dict(sd)
    m = m.cuda().eval()
    im1, im2 = synth.raft_inputs(seed=1, H=H, W=W)
    with torch.no_grad():
        lo, up = m(im1.cuda(), im2.cuda(), iters=iters, test_mode=True)
        torch.cuda.synchronize()
        olo, oup = RO.raft_forward(sd, im1, im2, iters=iters)
    e1, e2 = rel(lo, olo), rel(up, oup)
    ok = max(e1 + e2) < 1e-3
    print(f"{H}x{W} iters={iters}: low rel={e1[0]:.2e} max={e1[1]:.2e} | up rel={e2[0]:.2e} max={e2[1]:.2e} "
          f"| |flow|max={olo.abs().max().item():.2f} -> {'OK' if ok else 'FAIL'}", flush=True)
    return ok


if __name__ == "__main__":
    ok = True
    for it in (1, 2, 6, 20):
        ok &= run(128, 192, it)
    if len(sys.argv) > 1 and sys.argv[1] == "full":
        ok &= run(480, 864, 20)
    print("ALL OK" if ok else "SOME FAILED")
