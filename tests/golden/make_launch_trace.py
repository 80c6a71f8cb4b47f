"""Writes launch_trace.json.gz: the C-ABI call sequence of each network's forward (tests/test_launch_trace.py).

    python tests/golden/make_launch_trace.py

Runs on the CPU without the shared library. Regenerate only for a change meant to alter the launches.
"""
import gzip
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.test_launch_trace import CASES, GOLDEN, trace  # noqa: E402

if __name__ == "__main__":
    out = {case: trace(case) for case in sorted(CASES)}
    with gzip.GzipFile(GOLDEN, "wb", mtime=0) as f:
        f.write(json.dumps(out, sort_keys=True).encode())
    for case, calls in out.items():
        print(f"{case}: {len(calls)} launches")
