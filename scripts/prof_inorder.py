"""Time the in-order SGD epoch on the full C2 shape (1 000 209 rows, k = 8): the wavefront kernel, the
default for this shape.

  python scripts/prof_inorder.py [--rows N] [--epochs 7] [--warmup 2]

Prints the card's name and power limit, the library's CUDA-event time of each timed epoch, and their
median.  FMB200_LIB selects another build of the library (A/B timing in one session).
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from libfm_b200 import MODE_INORDER, FmLearnSgdElement, FmModel, synth  # noqa: E402


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rows", type=int, default=1_000_209)
    ap.add_argument("--epochs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    d = synth.movielens_1m_shaped(seed=7, n_rows=a.rows)
    fm = FmModel(d.num_feature, 8)
    fm.init_stdev = 0.1
    fm.init_numpy(42)
    l = FmLearnSgdElement(fm, mode=MODE_INORDER)
    l.task, l.learn_rate = 0, 0.01
    l.min_target, l.max_target = d.min_target, d.max_target
    l.push_hparams()
    l.push_params()
    for _ in range(a.warmup):
        l.sgd_epoch(d)
    times = [l.sgd_epoch(d) for _ in range(a.epochs)]
    slots = l.epoch_config()["slots"]
    l.close()
    print("card (name, power limit): %s" % gpu_info())
    print("in-order SGD epoch, %d rows, k = 8, %s kernel: median %.4f s  (epochs: %s)"
          % (a.rows, "wavefront" if slots == 4 else "row-at-a-time", sorted(times)[len(times) // 2],
             ", ".join("%.4f" % t for t in times)))


if __name__ == "__main__":
    main()
