"""fp64 model of the windowed HOGWILD SGD epoch (fmb200_set_reproducible, fm_sgd_window.cu).  TEST INFRASTRUCTURE.

The epoch's semantics are oracle/rowlane_model.py's: windows of file-order rows, every row scored from the state the
window found, damped steps rounded to 2^-32 and summed exactly, one bias step per tile, all folded after the window.
window_epoch_model computes exactly what rowlane_epoch_model computes (TR = the tile rows, grid = the window tiles),
state and budget alike, and adds to the budget a term for what the row-lane model's calibration did not cover: rows
of tens of entries and k up to 128.  A warp scores a row with its lanes over factors, each lane summing
n * ceil(k / 32) terms in sequence before a 5-level shuffle tree, so with L = eps_seq (n ceil(k / 32) + SEQ_EXTRA)

    the score carries      L (|w0| + sum_i |w_i x_i| + sum_f (sum_i |v_if x_i|)^2 + sum_i,f (v_if x_i)^2) more,
    each per-factor sum    L sum_i |v_if x_i|,
    h_row (damped steps)   L (xx + 3 |xx - 2| sum_f (sum_i |v_if x_i|)^2 + sq) relative to h_row,

as oracle/rowgroup_model.py bounds its sub-warp rows with EPS_S = 2^-22.  eps_seq = 0 adds nothing, and
tests/test_window_model.py checks that the two models then agree bit for bit.
"""
from __future__ import annotations

import numpy as np

from oracle.rowlane_model import (ACC_SCALE, EPS_GAMMA, EPS_M, EPS_P, EPS_SEQ, KAPPA, SEQ_EXTRA, Budget, HParams,
                                  State, _exact_sums, fold, gamma, gamma_cut_edge, loss_step, quantise, row_curvature,
                                  windows)

__all__ = ["EPS_SEQ", "SEQ_EXTRA", "window_epoch_model", "Budget", "HParams", "State"]


def window_epoch_model(state: State, data, hp: HParams, T: int, B: int, damp: bool, ramp_tiles: int,
                       budget: Budget | None = None, eps_seq: float = EPS_SEQ):
    """One epoch over `data` (row_ptr, col, val, target) in tiles of T rows and windows of B tiles.
    Returns (state, budget); pass the budget of the previous epoch to carry it on."""
    n = state.w.shape[0]
    k = state.v.shape[0]
    N = int(data.row_ptr.shape[0] - 1)
    rp = data.row_ptr.astype(np.int64)
    col = data.col.astype(np.int64)
    val = data.val.astype(np.float64)
    tgt = data.target.astype(np.float64)
    erow = np.repeat(np.arange(N, dtype=np.int64), np.diff(rp))
    count = np.bincount(col, minlength=n).astype(np.float32)
    n_tiles = (N + T - 1) // T
    lr = hp.lr
    lanes_seq = -(-k // 32)  # factors per lane

    st = state.copy()
    bud = Budget.zero(st) if budget is None else Budget(budget.w0, budget.w.copy(), budget.v.copy(), budget.windows)

    for j, (t0, nt) in enumerate(windows(n_tiles, ramp_tiles, B)):
        in_ramp = j < ramp_tiles
        flight = T if in_ramp else min(N, B * T)
        conc_scale = np.float32(flight / N)
        w0_conc = float(flight)
        r0, r1 = t0 * T, min(N, (t0 + nt) * T)
        R = r1 - r0
        e0, e1 = rp[r0], rp[r1]
        ids, x, er = col[e0:e1], val[e0:e1], erow[e0:e1] - r0
        y = tgt[r0:r1]
        grow = 1.0 + KAPPA * bud.windows

        # ---- the rows' scores, from the state as the window found it ----
        vv = st.v[:, ids]
        vx = vv * x
        sums = np.stack([np.bincount(er, weights=vx[f], minlength=R) for f in range(k)]) if k else np.zeros((0, R))
        sq = np.bincount(er, weights=(vx * vx).sum(0), minlength=R)
        s2 = (sums * sums).sum(0)
        wv = st.w[ids] if hp.k1 else np.zeros(ids.shape)
        lin = np.bincount(er, weights=wv * x, minlength=R)
        p = (st.w0 if hp.k0 else 0.0) + lin + 0.5 * (s2 - sq)
        mult, curv, edge = loss_step(hp, p, y)
        xx = np.bincount(er, weights=x * x, minlength=R)
        hrow, hjoint = row_curvature(hp, curv, xx, s2, sq, damp)
        row_err = EPS_P * (1.0 + np.abs(p)) + EPS_M * np.abs(mult)
        # ---- the lanes' sequences (the term rowlane_epoch_model does not have) ----
        L = eps_seq * (np.diff(rp[r0:r1 + 1]).astype(np.float64) * lanes_seq + SEQ_EXTRA)
        abs_s = np.stack([np.bincount(er, weights=np.abs(vx[f]), minlength=R) for f in range(k)]) if k \
            else np.zeros((0, R))
        abs_s2 = (abs_s * abs_s).sum(0)
        if eps_seq:
            row_err = row_err + L * ((abs(st.w0) if hp.k0 else 0.0) +
                                     np.bincount(er, weights=np.abs(wv * x), minlength=R) + abs_s2 + sq)
        rel_h = np.minimum(1.0, L * (xx + 3.0 * np.abs(xx - 2.0) * abs_s2 + sq) / np.maximum(hrow, 1e-300)) \
            * (hrow > 0)

        # ---- per entry: concurrency, damping, steps ----
        c = (count[ids] * conc_scale).astype(np.float64)
        damped = (c > 1.0) if damp else np.zeros(ids.shape, dtype=bool)
        sv = np.where(damped, gamma(c, lr * (hjoint[er] + hp.regv)), 1.0)
        sw = np.where(damped, gamma(c, lr * (hjoint[er] + hp.regw)), 1.0)
        x2 = x * x
        grad = sums[:, er] * x - vv * x2
        dv = sv * (-lr * mult[er] * grad - lr * hp.regv * vv)
        cut_v = damped * gamma_cut_edge(c, lr * (hjoint[er] + hp.regv))
        cut_w = damped * gamma_cut_edge(c, lr * (hjoint[er] + hp.regw))
        bv = sv * (lr * np.abs(grad) * row_err[er] + EPS_M * lr * hp.regv * np.abs(vv)) + 1.0 / ACC_SCALE \
            + np.abs(dv) * (EPS_GAMMA * damped + cut_v + edge[er])
        if eps_seq:
            bv = bv + sv * lr * np.abs(mult[er] * x) * (L * abs_s)[:, er] + np.abs(dv) * damped * rel_h[er]
        for f in range(k):
            st.v[f] = fold(st.v[f], _exact_sums(ids, quantise(dv[f]), n))
            bud.v[f] += grow * np.bincount(ids, weights=bv[f], minlength=n)
        if hp.k1:
            dw = sw * (-lr * mult[er] * x - lr * hp.regw * wv)
            bw = sw * (lr * np.abs(x) * row_err[er] + EPS_M * lr * hp.regw * np.abs(wv)) + 1.0 / ACC_SCALE \
                + np.abs(dw) * (EPS_GAMMA * damped + cut_w + edge[er])
            if eps_seq:
                bw = bw + np.abs(dw) * damped * rel_h[er]
            st.w = fold(st.w, _exact_sums(ids, quantise(dw), n))
            bud.w += grow * np.bincount(ids, weights=bw, minlength=n)

        # ---- per tile: the bias step ----
        if hp.k0:
            starts = np.arange(0, R, T)
            Tn = np.minimum(T, R - starts).astype(np.float64)
            M = np.add.reduceat(mult, starts) + Tn * hp.reg0 * st.w0
            H = np.add.reduceat(hjoint, starts)
            cb = max(w0_conc, 1.0)
            gb = gamma(cb, lr * (H / Tn + hp.reg0))
            step = -lr * gb * M
            h_edge = np.add.reduceat(edge * ((1.0 if damp else 0.0) * hrow + 1.0), starts)
            rel_edge = np.minimum(1.0, h_edge / np.maximum(H, 1e-300)) * (h_edge > 0)
            b0 = gb * lr * (np.add.reduceat(row_err, starts) + EPS_M * Tn * hp.reg0 * abs(st.w0)) + 1.0 / ACC_SCALE \
                + np.abs(step) * (EPS_GAMMA * (cb > 1.0) + gamma_cut_edge(cb, lr * (H / Tn + hp.reg0)) + rel_edge)
            st.w0 = float(fold(st.w0, quantise(step).sum()))
            bud.w0 += grow * float(b0.sum())
        bud.windows += 1
    return st, bud
