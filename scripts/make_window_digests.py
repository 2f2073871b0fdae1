"""Record what the windowed HOGWILD epochs compute as SHA-256 digests.

    python scripts/make_window_digests.py OUT.json

Runs every case of tests/test_window_digests_gpu.py (the reproducible SGD epoch, fm_sgd_window.cu, and the HOGWILD
SGDA epoch, fm_sgda_hogwild.cu) and writes a digest of w0, w and V (float64, as fmb200_get_params returns them)
after each epoch, for SGDA also of reg_w, reg_v and the moments.  Both epochs compute the same bits at every grid
size, so the digests hold on any H100; the test compares against tests/golden/window_digests.json, recorded with
this script.  FMB200_LIB selects the library build that computes them.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_window_digests_gpu import EPOCHS, cases  # noqa: E402


def main():
    import torch
    rec = {"gpu": torch.cuda.get_device_name(0), "epochs": EPOCHS,
           "digests": {name: run() for name, run in sorted(cases().items())}}
    with open(sys.argv[1], "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
