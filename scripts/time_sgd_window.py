"""Time the reproducible HOGWILD SGD epoch (fmb200_set_reproducible, fm_sgd_window.cu) beside the default dispatch
on C2, C2 with Zipf(1) ids and C3 at full size.

  python scripts/time_sgd_window.py [--reps 3] [--c3-rows 10000000] [--out FILE]

For each shape one learner per dispatch is uploaded and warmed by one epoch (the bias ramp), then the two are
alternated --reps times; every timed epoch follows an L2 flush (a 256 MB device write) and is the library's
CUDA-event time.  C3 also runs one windowed epoch with the kernel's phase timers.  The C3 line adds the windowed epoch's HBM share: the bytes it must move (the CSR once; per
window, for every feature it touches, its k + 1 state floats read and written and their u64 accumulator words
read and cleared) over the epoch time, against 3.35 TB/s.  Prints the card's name and power limit with the times.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from libfm_b200 import MODE_HOGWILD, FmLearnSgdElement, FmModel, synth  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def learner(d, k, task, lr, windowed):
    fm = FmModel(d.num_feature, k)
    fm.init_stdev = 0.01
    fm.init_numpy(1)
    l = FmLearnSgdElement(fm, mode=MODE_HOGWILD)
    l.task, l.learn_rate = task, lr
    l.min_target, l.max_target = d.min_target, d.max_target
    l.push_hparams()
    l.push_params()
    l.set_reproducible(windowed)
    l.upload(d, 0)
    l.sgd_epoch(d)  # warm-up: module load, the bias ramp
    return l


def min_bytes(d, k, W=16384):
    """The windowed epoch's compulsory traffic: CSR (8 bytes an entry, 12 a row) once, and per window each touched
    feature's k + 1 floats read and written (8 bytes) and accumulator words read and cleared (16 bytes)."""
    rp = d.row_ptr.astype(np.int64)
    touched = 0
    for r0 in range(0, d.num_cases, W):
        touched += np.unique(d.col[rp[r0]:rp[min(d.num_cases, r0 + W)]]).size
    return 8 * int(rp[-1]) + 12 * d.num_cases + touched * (k + 1) * 24, touched


def phases(d, k, task, lr) -> str:
    """One more windowed epoch with the kernel's phase timers (tuning variant 132), whose line the library writes
    to stderr: captured through the file descriptor."""
    import tempfile
    l = learner(d, k, task, lr, True)
    l.set_tuning(variant=132)
    sys.stderr.flush()
    with tempfile.TemporaryFile(mode="w+") as cap:
        saved = os.dup(2)
        os.dup2(cap.fileno(), 2)
        try:
            l.sgd_epoch(d)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        cap.seek(0)
        got = [x for x in cap.read().splitlines() if x.startswith("[window phases")]
    l.close()
    return got[-1] if got else "[window phases: no line]"


def main() -> None:
    import torch
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--c3-rows", type=int, default=10_000_000)
    ap.add_argument("--out", help="also write the report to this file")
    a = ap.parse_args()
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    shapes = [("C2", lambda: synth.movielens_1m_shaped(seed=7), 8, 0, 0.01),
              ("C2-Zipf", lambda: synth.movielens_1m_shaped(seed=7, zipf=1.0), 8, 0, 0.01),
              ("C3", lambda: synth.multi_field(a.c3_rows, 39, 1_000_000, 11), 64, 1, 0.01)]
    lines = ["Reproducible HOGWILD SGD epoch (windows of 256 x 64 rows) against the default dispatch; ms per epoch,",
             "L2 flushed before each, %d alternations" % a.reps,
             "card (name, power limit): %s" % gpu_info()]
    for name, make, k, task, lr in shapes:
        d = make()
        if task == 1:
            d.binarize_targets()
        ls = {w: learner(d, k, task, lr, w) for w in (False, True)}
        cfg = {w: ls[w].epoch_config() for w in ls}
        t = {False: [], True: []}
        for _ in range(a.reps):
            for w in (False, True):
                flush.zero_()
                torch.cuda.synchronize()
                t[w].append(ls[w].sgd_epoch(d) * 1e3)
        for l in ls.values():
            l.close()
        med = {w: sorted(x)[len(x) // 2] for w, x in t.items()}
        lines.append("%-8s %9d rows, k = %3d: default %8.2f ms (%s; grid %d x %d)   windowed %8.2f ms (%s; grid %d x "
                     "%d)   windowed / default %.2f"
                     % (name, d.num_cases, k, med[False], ", ".join("%.2f" % x for x in t[False]), cfg[False]["grid"],
                        cfg[False]["block"], med[True], ", ".join("%.2f" % x for x in t[True]), cfg[True]["grid"],
                        cfg[True]["block"], med[True] / med[False]))
        if name == "C3":
            lines.append(phases(d, k, task, lr))
            b, touched = min_bytes(d, k)
            lines.append("C3 windowed: %.2f GB compulsory (%d feature-windows touched), %.0f GB/s = %.1f%% of 3.35 TB/s"
                         % (b / 1e9, touched, b / (med[True] * 1e-3) / 1e9,
                            100 * b / (med[True] * 1e-3) / HBM_BYTES_PER_S))
        del d
    text = "\n".join(lines) + "\n"
    sys.stdout.write(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
