"""Time one C2-shaped SGDA epoch with lambda-steps three ways.

  python scripts/time_sgda.py [--reps 3] [--out FILE]

  one_warp    fm_sgda_epoch_kernel (fmb200_set_tuning variant 1), the library's CUDA-event time
  wavefront   fm_sgda_wavefront_kernel (the default for this shape), likewise
  reference   the stock reference's time_learn (user time of its epoch loop on one host core) for the
              second iteration of oracle/_ref/libFM -method sgda on the same rows, from its -rlog

Data: 1 000 209 training rows of the C2 shape (6040 users x 3706 items, 2 entries per row) and 100 000
validation rows of the same planted model, k = 8, two attribute groups (users, items), learn rate 0.01.
The GPU epochs are the second of a learner (the first has no lambda-steps); the median of --reps learners
is reported.  Prints the card's name and power limit with the times.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from libfm_b200 import MODE_INORDER, FmLearnSgdElement, FmModel, synth  # noqa: E402

K, LR, N_TRAIN, N_VAL = 8, 0.01, 1_000_209, 100_000


def data():
    full = synth.movielens_1m_shaped(seed=7, planted_k=4, n_rows=N_TRAIN + N_VAL)
    return synth.split_rows(full, N_TRAIN)


def gpu_epoch_ms(tr, va, variant: int, reps: int) -> list[float]:
    out = []
    n = tr.num_feature
    group = (np.arange(n) >= 6040).astype(np.uint32)
    for r in range(reps):
        fm = FmModel(n, K)
        fm.init_stdev = 0.1
        fm.init_numpy(42 + r)
        l = FmLearnSgdElement(fm, mode=MODE_INORDER)
        l.task, l.learn_rate = 0, LR
        l.min_target, l.max_target = tr.min_target, tr.max_target
        l.push_hparams()
        l.push_params()
        l.set_tuning(variant=variant)
        l.sgda_begin(group)
        l.sgda_epoch(tr, va, False)
        out.append(l.sgda_epoch(tr, va, True) * 1e3)
        slots = l.epoch_config()["slots"]
        l.close()
        assert slots == (1 if variant == 1 else 4), "unexpected schedule: %d slots" % slots
    return out


def reference_ms(tr, va) -> float | None:
    exe = os.path.join(ROOT, "oracle", "_ref", "libFM")
    if not os.path.exists(exe):
        return None
    with tempfile.TemporaryDirectory() as d:
        paths = {}
        for name, ds in (("train", tr), ("val", va)):
            paths[name] = os.path.join(d, name + ".libfm")
            synth.to_libfm_text(ds, paths[name])
        meta = os.path.join(d, "groups.meta")
        with open(meta, "w") as f:
            f.write("".join("%d\n" % (0 if i < 6040 else 1) for i in range(tr.num_feature)))
        rlog = os.path.join(d, "rlog")
        cmd = [exe, "-task", "r", "-method", "sgda", "-dim", "1,1,%d" % K, "-learn_rate", str(LR), "-iter", "2",
               "-train", paths["train"], "-test", paths["val"], "-validation", paths["val"], "-meta", meta,
               "-init_stdev", "0.1", "-seed", "42", "-rlog", rlog]
        subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        with open(rlog) as f:
            lines = f.read().splitlines()
        head = lines[0].split("\t")
        return float(lines[2].split("\t")[head.index("time_learn")]) * 1e3


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", help="also write the report to this file")
    a = ap.parse_args()
    tr, va = data()
    one = gpu_epoch_ms(tr, va, 1, a.reps)
    wf = gpu_epoch_ms(tr, va, 0, a.reps)
    ref = reference_ms(tr, va)
    med = lambda xs: sorted(xs)[len(xs) // 2]  # noqa: E731
    lines = ["SGDA epoch with lambda-steps, C2 shape: %d train rows, %d validation rows, k = %d, 2 groups"
             % (N_TRAIN, N_VAL, K),
             "card (name, power limit): %s" % gpu_info(),
             "one_warp   %10.1f ms  (runs: %s)" % (med(one), ", ".join("%.1f" % x for x in one)),
             "wavefront  %10.1f ms  (runs: %s)" % (med(wf), ", ".join("%.1f" % x for x in wf)),
             "reference  %10s ms  (stock libFM -method sgda, time_learn of iteration 1, one host core)"
             % ("%.1f" % ref if ref is not None else "n/a"),
             "one_warp / wavefront = %.2f" % (med(one) / med(wf))]
    text = "\n".join(lines) + "\n"
    sys.stdout.write(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
