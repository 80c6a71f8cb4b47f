"""Writes lafc_mixed_trace.json.gz: the C-ABI call sequence of one mixed-precision LAFC forward at 64x96, T=3
(tests/test_lafc_mixed.py), recorded as tests/test_launch_trace.py records the other networks.

    python tests/golden/make_lafc_mixed_trace.py

Runs on the CPU without the shared library. Regenerate only for a change meant to alter the launches.
"""
import gzip
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.test_lafc_mixed import GOLDEN, _trace  # noqa: E402

if __name__ == "__main__":
    _, calls = _trace(True)
    with gzip.GzipFile(GOLDEN, "wb", mtime=0) as f:
        f.write(json.dumps(calls, sort_keys=True).encode())
    print(f"lafc mixed: {len(calls)} launches")
