"""Streamed SGDA epochs (-method sgda -cache_size) against resident ones, on one GPU.

Generates, from a seed in a temporary directory, a C2-shaped binary data set (ML-1M: 1 000 209 rows of (user,
item), k = 8, two attribute groups), a validation set of 100 000 rows and a test set of 100 000 rows, and times
the second epoch of bin/libFM -method sgda -mode inorder (the first with lambda-steps; the rlog's time_learn: the
wall time of the epoch, the reading and the uploads of the streamed blocks included) with everything resident and
streamed at three -cache_size budgets.  Every run's Final line is printed beside its time: the streamed runs train
the same model.

  python scripts/stream_sgda.py [--out FILE]
"""
from __future__ import annotations

import argparse
import csv
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CLI = os.path.join(ROOT, "bin", "libFM")


def epoch_seconds(d: str, args: list[str], cache_size: int) -> tuple[float, str]:
    extra = ["-cache_size", str(cache_size)] if cache_size else []
    log = os.path.join(d, "rlog.tsv")
    r = subprocess.run([CLI] + args + extra + ["-iter", "2", "-rlog", log], capture_output=True, text=True, cwd=d)
    if r.returncode != 0:
        raise RuntimeError(r.stderr)
    rows = list(csv.DictReader(open(log), delimiter="\t"))
    plan = [l.split(": ", 1)[1] for l in r.stdout.splitlines() if l.startswith("streaming ")]
    final = [l for l in r.stdout.splitlines() if l.startswith("Final")]
    return float(rows[-1]["time_learn"]), ("; ".join(plan) if plan else "resident") + " | " + final[0]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = []

    def out(s):
        print(s, flush=True)
        lines.append(s)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    out("GPU: " + q.stdout.strip().splitlines()[0])
    from libfm_b200 import synth
    from libfm_b200.model import write_binary
    with tempfile.TemporaryDirectory() as d:
        full = synth.movielens_1m_shaped(seed=7)
        va = synth.movielens_1m_shaped(seed=8).rows(0, 100_000)
        write_binary(full, os.path.join(d, "c2.x"), os.path.join(d, "c2.y"))
        write_binary(va, os.path.join(d, "c2v.x"), os.path.join(d, "c2v.y"))
        write_binary(full.rows(0, 100_000), os.path.join(d, "c2t.x"), os.path.join(d, "c2t.y"))
        with open(os.path.join(d, "c2.meta"), "w") as f:  # the lower half of the ids one group, the rest the other
            n = full.num_feature
            f.write("\n".join("0" if i < n // 2 else "1" for i in range(n)) + "\n")
        args = ["-task", "r", "-train", "c2", "-test", "c2t", "-validation", "c2v", "-meta", "c2.meta",
                "-method", "sgda", "-mode", "inorder", "-dim", "1,1,8", "-init_stdev", "0.1", "-learn_rate", "0.01",
                "-seed", "42"]
        x = os.path.getsize(os.path.join(d, "c2v.x")) - 24  # the smallest streamed file
        out(f"SGDA epoch with lambda-steps, C2 shape: {full.num_cases} train, {va.num_cases} validation and "
            f"100000 test rows, k = 8, 2 groups, -mode inorder")
        res, info = epoch_seconds(d, args, 0)
        out(f"  resident          epoch {res:.3f} s   ({info})")
        for c in (x, x // 4, x // 16):
            t, info = epoch_seconds(d, args, c)
            out(f"  cache {c / 1e6:7.3f} MB   epoch {t:.3f} s   streamed / resident = {t / res:.3f}   ({info})")
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
