"""Record what the ORDERED epoch computes as SHA-256 digests.

    python scripts/make_ordered_digests.py OUT.json

For every entry of tests/test_ordered_digests_gpu.py's matrix (every kernel instantiation the launcher can pick,
in every configuration it can run in, both tasks, C2 at full size): the digests of w0, w and V (float64, as
fmb200_get_params returns them) after two epochs from a seeded model, and the launch configuration the epoch
reports.  The ORDERED epoch is deterministic, so these are exact pins: tests/test_ordered_digests_gpu.py compares
against tests/golden/ordered_digests.json, recorded on an H100 with this script.  FMB200_LIB selects the library
build that computes them.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_ordered_digests_gpu import EPOCHS, MATRIX, run  # noqa: E402


def main():
    import torch
    rec = {"gpu": torch.cuda.get_device_name(0), "epochs": EPOCHS, "digests": {c: run(c) for c in MATRIX}}
    with open(sys.argv[1], "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print("%d cases recorded" % len(rec["digests"]))


if __name__ == "__main__":
    main()
