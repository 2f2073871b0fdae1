"""One MCMC iteration resident against streamed from .xt blocks (fmb200_mcmc_begin_xt), on one GPU.

The C4 shape of BASELINE (synth.two_field(10 000 054, 71 567, 10 681), test 200 000 cases, k = 16, -method mcmc)
is written as .xt files in a temporary directory (write_transposed) and run through the library: resident, and
streamed at -cache_size budgets that cut the training .xt into about 2, 8 and 32 blocks.  The blocks come from
page-locked host memory, so the times cover the device passes and the copies, not reading the file (the command
line's reader thread reads it as it goes).  Each time is the wall clock of fmb200_mcmc_iteration, which ends in a
synchronise, averaged over the timed iterations after one warm-up iteration; the streamed runs must leave the
same test predictions, bit for bit, as the resident one.  Prints the card name and power limit first.

  python scripts/stream_mcmc.py [--iters 2] [--out FILE]
"""
from __future__ import annotations

import argparse
import hashlib
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from libfm_b200 import MODE_INORDER, FmLearnSgdElement, FmModel, synth  # noqa: E402
from libfm_b200.model import XtBlocks, _LibcRand, pinned_copy, write_transposed  # noqa: E402

K = 16


def card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def learner(n):
    l = FmLearnSgdElement(FmModel(n, K), mode=MODE_INORDER)
    l.fm.init_numpy(7)
    l.push_params()
    _LibcRand().srand(7)  # every run draws the same libc rand() stream
    l.task = 0
    return l


def run(l, begin, iters):
    t0 = time.perf_counter()
    begin()
    t_begin = time.perf_counter() - t0
    l.mcmc_iteration()  # warm-up
    t0 = time.perf_counter()
    for _ in range(iters):
        l.mcmc_iteration()
    dt = (time.perf_counter() - t0) / iters
    pred = l.mcmc_pred(te)[0]
    return t_begin, dt, hashlib.sha256(pred.tobytes()).hexdigest()[:16]


def pinned(x: XtBlocks) -> XtBlocks:
    x.blocks = [(lo, hi, pinned_copy(w), pinned_copy(s)) for lo, hi, w, s in x.blocks]
    return x


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = [f"GPU: {card()}"]
    print(out[0], flush=True)
    tr = synth.two_field(10_000_054, 71_567, 10_681, seed=5)
    te = synth.two_field(200_000, 71_567, 10_681, seed=6)
    n = max(tr.num_feature, te.num_feature)
    reg = dict(do_sample=True, do_multilevel=True, reg0=0.0, w_lambda=np.zeros(1), v_lambda=np.zeros((1, K)))
    with tempfile.TemporaryDirectory() as d:
        ptr, pte = os.path.join(d, "train.xt"), os.path.join(d, "test.xt")
        write_transposed(tr, ptr)
        write_transposed(te, pte)
        xt_bytes = os.path.getsize(ptr) - 24
        line = (f"C4 (10 000 054 cases x 2, 82 248 features, k = {K}, mcmc): train .xt {xt_bytes / 1e9:.3f} GB, "
                f"test .xt {(os.path.getsize(pte) - 24) / 1e9:.3f} GB; {a.iters} timed iterations after 1 warm-up")
        print(line, flush=True)
        out.append(line)
        l = learner(n)
        l.min_target, l.max_target = tr.min_target, tr.max_target
        tb, dt, dig = run(l, lambda: l.mcmc_begin(tr, te, **reg), a.iters)
        line = f"  resident                     begin {tb:7.3f} s  iteration {dt:7.3f} s   runs {l.mcmc_runs()}  pred {dig}"
        print(line, flush=True)
        out.append(line)
        l.close()
        want = dig
        for nb in (2, 8, 32):
            cache = 2 * (xt_bytes // nb + 1)
            xtr = pinned(XtBlocks(ptr, tr.target, cache, (2, 4)))
            xte = pinned(XtBlocks(pte, te.target, cache, (3, 5)))
            l = learner(n)
            l.min_target, l.max_target = tr.min_target, tr.max_target
            tb, dt, dig = run(l, lambda: l.mcmc_begin_xt(xtr, xte, **reg), a.iters)
            passes = xtr.fetches // xtr.n_blocks, xte.fetches // xte.n_blocks
            line = (f"  cache {cache / 1e6:8.1f} MB  train {xtr.n_blocks:3d} blocks, test {xte.n_blocks:2d}  "
                    f"begin {tb:7.3f} s  iteration {dt:7.3f} s   runs {l.mcmc_runs()}  pred {dig}"
                    f"{'' if dig == want else '  DIFFERS FROM RESIDENT'}  (passes so far: train {passes[0]}, "
                    f"test {passes[1]})")
            print(line, flush=True)
            out.append(line)
            l.close()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(out) + "\n")
