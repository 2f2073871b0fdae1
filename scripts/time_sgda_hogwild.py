"""Time the C2-shaped SGDA epoch with lambda-steps in HOGWILD mode (the windowed fp32 epoch, fm_sgda_hogwild.cu)
beside the fp64 wavefront epoch, on the data of scripts/time_sgda.py.

  python scripts/time_sgda_hogwild.py [--reps 3] [--out FILE]

  hogwild     fmb200_sgda_epoch in HOGWILD mode at the default window, the library's CUDA-event time
  wavefront   fm_sgda_wavefront_kernel (INORDER mode), likewise
The epochs timed are the second and third of a learner (the first has no lambda-steps); the median over --reps
learners of the second is reported.  Prints the card's name and power limit with the times.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from libfm_b200 import MODE_HOGWILD, FmLearnSgdElement, FmModel  # noqa: E402
from time_sgda import K, LR, N_TRAIN, N_VAL, data, gpu_epoch_ms, gpu_info  # noqa: E402


def hogwild_ms(tr, va, reps: int):
    first, lam, cfg = [], [], None
    n = tr.num_feature
    group = (np.arange(n) >= 6040).astype(np.uint32)
    for r in range(reps):
        fm = FmModel(n, K)
        fm.init_stdev = 0.1
        fm.init_numpy(42 + r)
        l = FmLearnSgdElement(fm, mode=MODE_HOGWILD)
        l.task, l.learn_rate = 0, LR
        l.min_target, l.max_target = tr.min_target, tr.max_target
        l.push_hparams()
        l.push_params()
        l.sgda_begin(group)
        first.append(l.sgda_epoch(tr, va, False) * 1e3)
        lam.append(l.sgda_epoch(tr, va, True) * 1e3)
        l.sgda_epoch(tr, va, True)
        cfg = l.epoch_config()
        l.close()
    return first, lam, cfg


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", help="also write the report to this file")
    a = ap.parse_args()
    tr, va = data()
    first, lam, cfg = hogwild_ms(tr, va, a.reps)
    wf = gpu_epoch_ms(tr, va, 0, a.reps)
    med = lambda xs: sorted(xs)[len(xs) // 2]  # noqa: E731
    lines = ["SGDA epoch, C2 shape: %d train rows, %d validation rows, k = %d, 2 groups" % (N_TRAIN, N_VAL, K),
             "card (name, power limit): %s" % gpu_info(),
             "hogwild, lambda-steps    %8.1f ms  (runs: %s; window %d rows, grid %d x %d threads)"
             % (med(lam), ", ".join("%.1f" % x for x in lam), cfg["rows_per_tile"], cfg["grid"], cfg["block"]),
             "hogwild, first epoch     %8.1f ms  (runs: %s; no lambda-steps)"
             % (med(first), ", ".join("%.1f" % x for x in first)),
             "wavefront (fp64)         %8.1f ms  (runs: %s)" % (med(wf), ", ".join("%.1f" % x for x in wf)),
             "wavefront / hogwild = %.1f" % (med(wf) / med(lam))]
    text = "\n".join(lines) + "\n"
    sys.stdout.write(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
