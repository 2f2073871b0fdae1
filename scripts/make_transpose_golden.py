"""Write tests/golden/reference/transpose.json: the sha256 of what the stock reference's transpose tool
(tools/transpose.cpp, built unmodified, e.g. `g++ -O3 -w tools/transpose.cpp -o transpose` in the reference's
src/libfm) writes for each input of tests/test_stream_mcmc_cpu.py's transpose_inputs(), beside the sha256 of that
input, so that bin/transpose and write_transposed are checked against the stock tool without it.

  python scripts/make_transpose_golden.py --transpose PATH_TO_STOCK_TRANSPOSE
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_stream_mcmc_cpu import TRANSPOSE_GOLDEN, _sha, transpose_inputs  # noqa: E402

if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--transpose", required=True, help="the stock reference's transpose binary")
    a = ap.parse_args()
    out = {"x": {}, "xt": {}}
    with tempfile.TemporaryDirectory() as d:
        for name, stem in sorted(transpose_inputs(d).items()):
            subprocess.run([a.transpose, "-ifile", stem + ".x", "-ofile", stem + ".xt"], check=True,
                           capture_output=True)
            out["x"][name] = _sha(stem + ".x")
            out["xt"][name] = _sha(stem + ".xt")
    with open(TRANSPOSE_GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(TRANSPOSE_GOLDEN)
