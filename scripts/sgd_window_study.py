"""Choice of the reproducible HOGWILD SGD epoch's window W (fmb200_set_reproducible): held-out RMSE after each epoch
at several W against the sequential SGD epoch (oracle.Port, fp64) and the free-running HOGWILD kernel, on planted
C2- and C3-shaped data.

The windowed epoch is the fp64 model of its windows to within fp32 rounding (tests/test_sgd_window_gpu.py), so the
kernel stands in for the model here: the same numbers, in seconds instead of hours at C3 size.  Tiles stay 256
rows; W = 256 x --tiles.  Every learner starts from one init.  Needs a GPU.

    python scripts/sgd_window_study.py [--epochs 3] [--tiles 16 64 256] [--out FILE]
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from libfm_b200 import MODE_HOGWILD, Data, FmLearnSgdElement, FmModel, synth  # noqa: E402
from oracle import Port  # noqa: E402


def planted_c3(n_train, n_test, seed=5):
    """39 one-hot fields over 1 M features, y = sum of per-feature effects N(0, 0.15) + N(0, 0.5) noise."""
    d = synth.multi_field(n_train + n_test, 39, 1_000_000, seed=seed)
    r = np.random.default_rng(seed)
    b = r.normal(0.0, 0.15, d.num_feature)
    y = np.add.reduceat(b[d.col.astype(np.int64)], d.row_ptr[:-1].astype(np.int64)) + r.normal(0, 0.5, d.num_cases)
    return synth.split_rows(Data(d.row_ptr, d.col, d.val, y.astype(np.float32), d.num_feature), n_train)


def init(n, k):
    fm = FmModel(n, k)
    fm.init_stdev = 0.01
    fm.init_numpy(3)
    return fm


def rmse_of(fm, test, k, mn, mx):
    p = Port(test.num_feature, k)
    p.set_params(fm.w0, fm.w, fm.v)
    return p.metric(test, 0, mn, mx)


def gpu_run(train, test, k, lr, epochs, tiles):
    """tiles None: the default (free-running) dispatch.  Returns (held-out RMSE per epoch, ms per epoch)."""
    mn, mx = float(train.target.min()), float(train.target.max())
    l = FmLearnSgdElement(init(train.num_feature, k), device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate, l.min_target, l.max_target = 0, lr, mn, mx
    l.push_hparams()
    if tiles is not None:
        l.set_reproducible(True, 256, tiles)
    l.upload(train, 0)
    out, ms = [], []
    for _ in range(epochs):
        ms.append(l.sgd_epoch(train) * 1e3)
        l.pull_params()
        out.append(rmse_of(l.fm, test, k, mn, mx))
    l.close()
    return out, ms


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--tiles", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--out", help="also write the report to this file")
    a = ap.parse_args()
    shapes = [("C2 planted (1 M rows, 2 entries, k = 8)", lambda: synth.movielens_1m_planted(), 8),
              ("C3 planted (1 M rows, 39 entries, k = 64)", lambda: planted_c3(1_000_000, 100_000), 64)]
    lines = []
    lr = 0.01
    for name, make, k in shapes:
        train, test = make()
        mn, mx = float(train.target.min()), float(train.target.max())
        fm = init(train.num_feature, k)
        port = Port(train.num_feature, k)
        port.set_params(fm.w0, fm.w, fm.v)
        seq = []
        for _ in range(a.epochs):
            port.sgd_epoch(train, 0, lr, mn, mx)
            seq.append(port.metric(test, 0, mn, mx))
        lines.append("%s, lr %g: held-out RMSE after each epoch (gap to sequential), ms per epoch" % (name, lr))
        lines.append("  %-22s %s" % ("sequential (oracle)", "  ".join("%.5f" % x for x in seq)))
        for tiles in [None] + a.tiles:
            got, ms = gpu_run(train, test, k, lr, a.epochs, tiles)
            label = "free-running" if tiles is None else "W = %d" % (256 * tiles)
            lines.append("  %-22s %s   %s ms" % (label, "  ".join("%.5f (%+.4f)" % (g, g - s) for g, s in zip(got, seq)),
                                                 " ".join("%.2f" % x for x in ms)))
        sys.stdout.write("\n".join(lines[-(len(a.tiles) + 3):]) + "\n")
        sys.stdout.flush()
    text = "\n".join(lines) + "\n"
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
