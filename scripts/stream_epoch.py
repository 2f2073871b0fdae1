"""Streamed SGD epochs (-cache_size) against resident ones, on one GPU.

Generates, from a seed in a temporary directory, a C3-shaped binary data set (10 M rows, 39 one-hot fields over
1 M features, about 3.2 GB of .x, -task c, k = 64) and a C2-shaped one (ML-1M: 1 000 209 rows of (user, item),
k = 8), and times in one run:
  * the pinned host-to-device copy rate (torch, CUDA events, 1 GiB);
  * the epoch of bin/libFM with everything resident, and streamed at a few -cache_size budgets (the rlog's
    time_learn of the second epoch: the wall time of the epoch pass, reading and uploading included).
For each streamed run it prints  streamed / max(resident epoch, .x bytes / copy rate): near 1 when the copy of
block b + 1 hides behind the epoch on block b (or the epoch behind the copy), near 2 when they serialise.  It also
prints the time of one sequential host read of the .x: a streamed pass reads the file again, so that time bounds
the streamed epoch from below as well.

  python scripts/stream_epoch.py [--out FILE]
"""
from __future__ import annotations

import argparse
import csv
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CLI = os.path.join(ROOT, "bin", "libFM")


def write_c3(stem: str, n_rows: int, seed: int, n_fields: int = 39, n_features: int = 1_000_000) -> None:
    """One-hot rows of n_fields fields (field f owns ids [f * n / F, (f + 1) * n / F)), targets +-1."""
    r = np.random.default_rng(seed)
    per = n_features // n_fields
    with open(stem + ".x", "wb") as f:
        f.write(np.array([2, 4], np.uint32).tobytes() + np.array([n_rows * n_fields], np.uint64).tobytes()
                + np.array([n_rows, per * n_fields], np.uint32).tobytes())
        one = np.float32(1.0).view(np.uint32)
        for lo in range(0, n_rows, 500_000):
            m = min(500_000, n_rows - lo)
            rec = np.empty((m, 1 + 2 * n_fields), np.uint32)
            rec[:, 0] = n_fields
            rec[:, 1::2] = r.integers(0, per, (m, n_fields), dtype=np.uint32) + np.arange(n_fields, dtype=np.uint32) * per
            rec[:, 2::2] = one
            f.write(rec.tobytes())
    y = np.where(r.random(n_rows) < 0.25, 1.0, -1.0).astype(np.float32)
    with open(stem + ".y", "wb") as f:
        f.write(np.array([1, 4, n_rows], np.uint32).tobytes() + y.tobytes())


def copy_rate() -> float:
    import torch
    n = 1 << 30
    h = torch.empty(n, dtype=torch.uint8).pin_memory()
    d = torch.empty(n, dtype=torch.uint8, device="cuda")
    d.copy_(h, non_blocking=True)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(5):
        d.copy_(h, non_blocking=True)
    b.record()
    torch.cuda.synchronize()
    return 5 * n / (a.elapsed_time(b) * 1e-3)


def epoch_seconds(d: str, args: list[str], cache_size: int) -> tuple[float, str]:
    extra = ["-cache_size", str(cache_size)] if cache_size else []
    log = os.path.join(d, "rlog.tsv")
    r = subprocess.run([CLI] + args + extra + ["-iter", "2", "-rlog", log], capture_output=True, text=True, cwd=d)
    if r.returncode != 0:
        raise RuntimeError(r.stderr)
    rows = list(csv.DictReader(open(log), delimiter="\t"))
    plan = [l for l in r.stdout.splitlines() if l.startswith("streaming ")]
    final = [l for l in r.stdout.splitlines() if l.startswith("Final")]
    return float(rows[-1]["time_learn"]), (plan[0] if plan else "resident") + " | " + final[0]


def read_rate(path: str) -> float:
    """Bytes per second of one sequential read of `path` in 256 MiB pieces (what the block reader does)."""
    buf = bytearray(256 << 20)
    t0 = time.perf_counter()
    n = 0
    with open(path, "rb", buffering=0) as f:
        while True:
            k = f.readinto(buf)
            if not k:
                break
            n += k
    return n / (time.perf_counter() - t0)


def run_case(name: str, d: str, args: list[str], x_bytes: int, budgets: list[int], rate: float, out) -> None:
    res, info = epoch_seconds(d, args, 0)
    rd = read_rate(os.path.join(d, args[args.index("-train") + 1] + ".x"))
    out(f"{name}: .x {x_bytes / 1e9:.3f} GB, copy of the .x at the pinned rate {x_bytes / rate:.3f} s, "
        f"one host read of the .x {x_bytes / rd:.3f} s ({rd / 1e9:.2f} GB/s)")
    out(f"  resident        epoch {res:.3f} s   ({info})")
    for c in budgets:
        t, info = epoch_seconds(d, args, c)
        bound = max(res, x_bytes / rate)
        out(f"  cache {c / 1e6:9.1f} MB  epoch {t:.3f} s   streamed / max(resident, copy) = {t / bound:.2f}   ({info})")


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
    rate = copy_rate()
    out(f"pinned host-to-device copy: {rate / 1e9:.2f} GB/s (1 GiB, torch, CUDA events)")
    from libfm_b200 import synth
    from libfm_b200.model import write_binary
    with tempfile.TemporaryDirectory() as d:
        write_c3(os.path.join(d, "c3"), 10_000_000, seed=3)
        write_c3(os.path.join(d, "c3t"), 100_000, seed=4)
        c3 = ["-task", "c", "-train", "c3", "-test", "c3t", "-method", "sgd", "-dim", "1,1,64", "-init_stdev", "0.01",
              "-learn_rate", "0.01", "-seed", "42"]
        x = os.path.getsize(os.path.join(d, "c3.x")) - 24
        run_case("C3 (10 M rows x 39, k = 64, hogwild)", d, c3, x, [x // 2, x // 4, x // 16], rate, out)
        for f in ("c3.x", "c3.y"):
            os.remove(os.path.join(d, f))
        tr = synth.movielens_1m_shaped(seed=7)
        write_binary(tr, os.path.join(d, "c2.x"), os.path.join(d, "c2.y"))
        write_binary(tr.rows(0, 100_000), os.path.join(d, "c2t.x"), os.path.join(d, "c2t.y"))
        c2 = ["-task", "r", "-train", "c2", "-test", "c2t", "-method", "sgd", "-dim", "1,1,8", "-init_stdev", "0.1",
              "-learn_rate", "0.01", "-seed", "42"]
        x = os.path.getsize(os.path.join(d, "c2.x")) - 24
        for mode in ("hogwild", "ordered"):
            run_case(f"C2 (1 M rows x 2, k = 8, {mode})", d, c2 + ["-mode", mode], x, [x // 2, x // 8], rate, out)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
