"""Builds libfgt_sm90a.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libfgt_sm90a.so")
STAMP = os.path.join(HERE, "csrc", ".build_stamp")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xptxas=-v",
    "-Xcompiler", "-fPIC,-O2,-Wall,-Wno-unused-function", "--shared", "-cudart", "static",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    root = os.path.dirname(HERE)
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".h"))]
    files.append(os.path.join(root, "include", "fgt_b200.h"))
    for f in files:
        with open(f, "rb") as fh:
            h.update(os.path.relpath(f, root).encode())
            h.update(fh.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as fh:
            if fh.read().strip() == dig:
                return LIB
    cmd = [NVCC] + FLAGS + ["-o", LIB] + sources()
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building libfgt_sm90a.so")
    with open(STAMP, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
    print(LIB)
