"""Choice of the HOGWILD SGDA window W: the windowed model (oracle/sgda_window_model.py) at several W against the
reference's SGDA (oracle/fm_oracle_sgda.c) on planted C2-shaped data.

The held-out rows of synth.movielens_1m_planted are split into validation (first half) and test (second half).
Both learners start from the same model (k = 8, init_stdev 0.1, two groups: users and items) and run `--epochs`
epochs with lambda-steps from the second on.  Per epoch and W it prints the test RMSE of each and the gap, and
the learned reg_w and reg_v.  CPU only.

    python scripts/sgda_window_study.py --epochs 10 --windows 1024 4096 16384
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from libfm_b200 import synth  # noqa: E402
from oracle import HParams, Port, State  # noqa: E402
from oracle import sgda_window_model as sm  # noqa: E402


def rmse(st, d):
    rp = d.row_ptr.astype(np.int64)
    er = np.repeat(np.arange(d.num_cases), np.diff(rp))
    ids, x = d.col.astype(np.int64), d.val.astype(np.float64)
    vx = st.v[:, ids] * x
    s = np.stack([np.bincount(er, weights=vx[f], minlength=d.num_cases) for f in range(st.v.shape[0])])
    sq = np.bincount(er, weights=(vx * vx).sum(0), minlength=d.num_cases)
    p = st.w0 + np.bincount(er, weights=st.w[ids] * x, minlength=d.num_cases) + 0.5 * ((s * s).sum(0) - sq)
    p = np.clip(p, 1.0, 5.0)
    return float(np.sqrt(np.mean((p - d.target) ** 2)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--windows", type=int, nargs="+", default=[1024, 4096, 16384])
    ap.add_argument("--lr", type=float, default=0.01)
    args = ap.parse_args()
    train, held = synth.movielens_1m_planted()
    val, test = synth.split_rows(held, held.num_cases // 2)
    n, k = train.num_feature, 8
    group = (np.arange(n) >= 6040).astype(np.uint32)
    r = np.random.default_rng(1)
    v0 = np.asarray(0.1 * r.standard_normal((k, n)), dtype=np.float32).astype(np.float64)
    hp = HParams(0, args.lr, min_target=1.0, max_target=5.0)

    o = Port(n, k)
    o.set_params(0.0, np.zeros(n), v0)
    o.sgda_begin(group)
    ref = []
    for e in range(args.epochs):
        o.sgda_epoch(train, val, 0, args.lr, 1.0, 5.0, e > 0)
        ref.append((rmse(State(o.w0.value, o.w, o.v), test), o.reg_w.copy(), o.reg_v.copy()))
    print("reference: test RMSE per epoch " + " ".join("%.4f" % t for t, _, _ in ref))
    print("reference: reg_w %s  reg_v[0] %s" % (np.array2string(ref[-1][1], precision=4),
                                              np.array2string(ref[-1][2][0], precision=4)))
    for W in args.windows:
        st, sg = State(0.0, np.zeros(n), v0.copy()), sm.Sgda.begin(n, k, group)
        gaps = []
        for e in range(args.epochs):
            st, sg, _, _, _ = sm.sgda_window_epoch(st, sg, train, val, hp, W, e > 0)
            t = rmse(st, test)
            gaps.append(t - ref[e][0])
            print("W %6d epoch %2d  test RMSE %.4f  reference %.4f  gap %+.4f" % (W, e, t, ref[e][0], gaps[-1]),
                  flush=True)
        print("W %6d: worst |gap| after the first epoch %.4f; reg_w %s  reg_v[0] %s" % (
            W, max(abs(g) for g in gaps[1:]), np.array2string(sg.reg_w, precision=4),
            np.array2string(sg.reg_v[0], precision=4)), flush=True)


if __name__ == "__main__":
    main()
