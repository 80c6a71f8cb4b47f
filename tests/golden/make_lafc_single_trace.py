"""Writes lafc_single_trace.json.gz: the C-ABI call sequence of one 2D-LAFC forward at 64x96, n = 2
(tests/test_lafc_single.py), recorded as tests/test_launch_trace.py records the other networks.

    python tests/golden/make_lafc_single_trace.py

Runs on the CPU without the shared library. Regenerate only for a change meant to alter the launches.
"""
import gzip
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.test_lafc_single import TRACE, trace  # noqa: E402

if __name__ == "__main__":
    calls = trace()
    with gzip.GzipFile(TRACE, "wb", mtime=0) as f:
        f.write(json.dumps(calls, sort_keys=True).encode())
    print(f"2D LAFC: {len(calls)} launches")
