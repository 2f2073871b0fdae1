"""fp64 model of the windowed SGDA epoch of HOGWILD mode (DESIGN.md section 3.5).  TEST INFRASTRUCTURE ONLY.

SGDA (fm_learn_sgd_element_adapt_reg.h) interleaves a theta-step on each training row with a lambda-step on the
next validation row.  The windowed epoch cuts the training rows into windows of W consecutive rows, the first
at row 0 of every epoch, and runs each window as two phases:

  theta   every row of the window is scored from the state as the window found it and takes the reference's
          theta-step (:136-169) from that state, with reg as the previous window left it.  A row that names a
          feature twice steps it twice in a row, as the reference does.  Each step is damped by the row-lane
          epoch's gamma(c, u) -- c the feature's count * W / N, W for the bias, u = lr (row curvature + 2 reg) --
          rounded to 2^-32, summed exactly and folded into the fp32 state.  The stored gradient of every feature
          the window names (a per-feature stamp, not a nonzero test: a zero gradient is stored too) becomes the
          sum of its rows' gradients, each row's the one its last entry of the feature left, quantised alike.
  lambda  (not in an epoch's first pass, :301) one lambda-step per theta-step, on the validation rows the
          cursor names (restarting at 0 every epoch, wrapping at V).  Each reads the folded state and stored
          gradients and the reg the theta-phase read, and computes sgd_lambda_step's per-group terms
          (:201-248); the window's terms are summed and reg <- max(0, reg + sum), once per window.

The moments (rlog wvar / vvar) are taken from the state the lambda-steps read in the window that holds the
epoch's last cursor restart, or from the epoch's start when the cursor does not restart.

With W = 1, no damping, no quantisation and fp64 state this is the reference's SGDA step for step
(tests/test_sgda_window_model.py holds it to oracle/fm_oracle_sgda.c).  Beside the state the model carries the
row-lane model's per-element budget (rowlane_model.Budget; the same constants) with two more terms: the steps a
difference in reg moves (2 lr |reg - reg'| |theta|) and, for reg itself, REG_REL of every lambda contribution.

eps_seq > 0 (EPS_SEQ) adds the term rowlane_epoch_model's eps_seq states for the windowed SGD epoch's warp-per-row
score, which the row-lane calibration never saw: a lane adds n ceil(k / 32) terms in sequence before a 5-level shuffle
tree, so with L = eps_seq (n ceil(k / 32) + SEQ_EXTRA) the score carries scale L (|w0| + sum_i |w_i x_i| +
sum_f (sum_i |v_if x_i|)^2 + sum_i,f (v_if x_i)^2) more, each per-factor sum s_f (and so each V gradient) L sum_i
|v_if x_i|, and h_row, which damped steps read, L (xx + 3 |xx - 2| sum_f (sum_i |v_if x_i|)^2 + sq) relative.  Only
the theta-phase is fp32; the lambda-phase is fp64.  eps_seq = 0 (the default) leaves the budget as it was.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from .rowlane_model import (ACC_SCALE, EPS_GAMMA, EPS_M, EPS_P, EPS_SEQ, KAPPA, SEQ_EXTRA, Budget, HParams,
                            State, gamma, gamma_cut_edge, loss_step, quantise, row_curvature, ulp32)

REG_REL = 2e-3  # relative difference of a lambda contribution: it is read from fp32 state within the budget

DEFAULT_W = 4096  # libfm_b200/csrc/fm_sgda_hogwild.cu: kSgdaWindowRows


@dataclass
class Sgda:
    """The SGDA learner state beside the parameters: stored gradients and per-group regularisation."""
    grad_w: np.ndarray  # [n]
    grad_v: np.ndarray  # [k][n]
    reg_w: np.ndarray   # [G]
    reg_v: np.ndarray   # [G][k]
    group: np.ndarray   # [n] attribute group

    @staticmethod
    def begin(n: int, k: int, group=None) -> "Sgda":
        g = np.zeros(n, dtype=np.int64) if group is None else np.asarray(group, dtype=np.int64)
        G = int(g.max()) + 1 if n else 1
        return Sgda(np.zeros(n), np.zeros((k, n)), np.zeros(G), np.zeros((G, k)), g)

    def copy(self) -> "Sgda":
        return Sgda(self.grad_w.copy(), self.grad_v.copy(), self.reg_w.copy(), self.reg_v.copy(), self.group)


@dataclass
class RegBudget:
    """Bound on |kernel - model| of reg_w, reg_v and of the moments of the last epoch."""
    reg_w: np.ndarray
    reg_v: np.ndarray
    var_w: float = 0.0
    var_v: np.ndarray | None = None


def last_moments_step(N: int, V: int, lam: bool) -> int:
    """fm_sgda_plan.h: the step whose lambda-step follows the epoch's last update_means, 0 for the epoch start."""
    if not lam or V == 0 or N <= V:
        return 0
    return (N - 1) // V * V


def moments(st: State):
    """update_means (:250-274) of the state: (var_w, var_v[k]) = sum x^2 / n - mean^2 per column."""
    n = st.w.shape[0]
    col = lambda x: float(np.sum(x * x) / n - (np.sum(x) / n) ** 2)
    return col(st.w), np.array([col(st.v[f]) for f in range(st.v.shape[0])])


def _moment_bound(st: State, bw, bv):
    """What the moments of two states whose elements differ by at most (bw, bv) may differ by, plus rounding."""
    n = st.w.shape[0]
    col = lambda x, b: float(np.sum((2.0 * np.abs(x) + 2.0 * abs(np.mean(x)) + b) * b) / n + 1e-12 * (np.mean(x * x) + 1e-30))
    return col(st.w, bw), np.array([col(st.v[f], bv[f]) for f in range(st.v.shape[0])])


def _rows(d, lo: np.ndarray):
    """(entry index, row-in-list) of the rows lo of CSR data d."""
    rp = d.row_ptr.astype(np.int64)
    lens = rp[lo + 1] - rp[lo]
    first = np.repeat(rp[lo] - np.concatenate(([0], np.cumsum(lens)[:-1])), lens)
    return first + np.arange(int(lens.sum()), dtype=np.int64), np.repeat(np.arange(lo.shape[0]), lens)


def _occurrences(er, ids):
    """(prev, last): the entry of the same row naming the same feature just before each entry (-1 for none), and
    whether no later entry of the row names it."""
    E = ids.shape[0]
    o = np.lexsort((np.arange(E), ids, er))
    same = np.zeros(E, dtype=bool)
    same[1:] = (er[o][1:] == er[o][:-1]) & (ids[o][1:] == ids[o][:-1])
    prev = np.full(E, -1, dtype=np.int64)
    prev[o[1:][same[1:]]] = o[:-1][same[1:]]
    last = np.ones(E, dtype=bool)
    last[o[:-1][same[1:]]] = False
    return prev, last


def _fold_sum(x, idx, d, n, quant, fp32):
    """x plus the per-index sums of the steps d: quantised and folded as the accumulator does, or in fp64."""
    if quant:
        q = np.bincount(idx, weights=quantise(d), minlength=n)
        assert np.abs(q).max(initial=0.0) < 2.0 ** 53
        step = q / ACC_SCALE
    else:
        step = np.bincount(idx, weights=d, minlength=n)
    if fp32:
        return np.where(step != 0.0, (x.astype(np.float32) + step.astype(np.float32)).astype(np.float64), x)
    return x + step


def _window_sum(idx, d, n, quant, fp32):
    """The per-index sums of the gradients d as the stored gradient takes them."""
    if quant:
        s = np.bincount(idx, weights=quantise(d), minlength=n) / ACC_SCALE
    else:
        s = np.bincount(idx, weights=d, minlength=n)
    return s.astype(np.float32).astype(np.float64) if fp32 else s


def sgda_window_epoch(state: State, sg: Sgda, train, val, hp: HParams, W: int, lambda_steps: bool,
                      damp: bool = True, quant: bool = True, fp32: bool = True, budget: Budget | None = None,
                      reg_budget: RegBudget | None = None, trace: list | None = None, eps_seq: float = 0.0):
    """One windowed SGDA epoch over train (row_ptr, col, val, target) with validation set val.
    Returns (state, sgda, (var_w, var_v), budget, reg_budget); pass the budgets back to carry them on.
    trace: a list that receives the state after each window's fold.
    eps_seq: the budget's term for the lanes' serial sums (EPS_SEQ; 0 leaves it out, see the module's notes)."""
    n, k = state.w.shape[0], state.v.shape[0]
    N, V = int(train.row_ptr.shape[0] - 1), int(val.row_ptr.shape[0] - 1)
    G = sg.reg_w.shape[0]
    lr = hp.lr
    lam = bool(lambda_steps) and V > 0
    st, sg = state.copy(), sg.copy()
    bud = Budget.zero(st) if budget is None else Budget(budget.w0, budget.w.copy(), budget.v.copy(), budget.windows)
    rb = RegBudget(np.zeros(G), np.zeros((G, k))) if reg_budget is None else \
        RegBudget(reg_budget.reg_w.copy(), reg_budget.reg_v.copy())
    tcol, tval, tgt = train.col.astype(np.int64), train.val.astype(np.float64), train.target.astype(np.float64)
    count = np.bincount(tcol, minlength=n).astype(np.float32)
    conc_scale = np.float32(min(W, N) / N) if N else np.float32(1.0)
    cb = float(np.float32(min(W, N)))
    scale = 2.0 if hp.task == 0 else 1.0  # SGDA's regression loss is (p - y)^2: twice SGD's multiplier
    lanes_seq = -(-k // 32)  # factors per lane
    row_len = np.diff(train.row_ptr.astype(np.int64)).astype(np.float64)
    t_star = last_moments_step(N, V, lam)
    j_star = t_star // W if t_star > 0 else -1
    mom = mom_b = None
    if j_star < 0:
        mom = moments(st)
        b = bud.bound(st)
        mom_b = _moment_bound(st, b[1], b[2])

    for j, r0 in enumerate(range(0, N, W)):
        r1 = min(N, r0 + W)
        R = r1 - r0
        grow = 1.0 + KAPPA * bud.windows
        e, er = _rows(train, np.arange(r0, r1))
        ids, x = tcol[e], tval[e]
        g = sg.group[ids]
        y = tgt[r0:r1]
        reg_w, reg_v = sg.reg_w.copy(), sg.reg_v.copy()  # as the previous window left them

        # ---- theta: scores from the state as the window found it ----
        vv = st.v[:, ids]
        vx = vv * x
        sums = np.stack([np.bincount(er, weights=vx[f], minlength=R) for f in range(k)]) if k else np.zeros((0, R))
        sq = np.bincount(er, weights=(vx * vx).sum(0), minlength=R)
        s2 = (sums * sums).sum(0)
        wv = st.w[ids] if hp.k1 else np.zeros(ids.shape)
        p = (st.w0 if hp.k0 else 0.0) + np.bincount(er, weights=wv * x, minlength=R) + 0.5 * (s2 - sq)
        m1, curv, edge = loss_step(hp, p, y)
        mult, hc = scale * m1, scale * curv
        xx = np.bincount(er, weights=x * x, minlength=R)
        hrow, hjoint = row_curvature(hp, hc, xx, s2, sq, damp)
        # fp32 score: relative to the magnitude of its terms, which bounds |p| and grows with the row's length
        abs_s = np.stack([np.bincount(er, weights=np.abs(vx[f]), minlength=R) for f in range(k)]) if k else \
            np.zeros((0, R))
        p_abs = (abs(st.w0) if hp.k0 else 0.0) + np.bincount(er, weights=np.abs(wv * x), minlength=R) \
            + 0.5 * (abs_s ** 2).sum(0) + 0.5 * sq
        row_err = scale * EPS_P * (1.0 + p_abs) + EPS_M * np.abs(mult)
        if eps_seq:  # the lanes' serial sums: the score, each per-factor sum s_f and h_row
            seq = eps_seq * (row_len[r0:r1] * lanes_seq + SEQ_EXTRA)  # L of the module's notes, per row
            abs_s2 = (abs_s * abs_s).sum(0)
            row_err = row_err + scale * seq * ((abs(st.w0) if hp.k0 else 0.0) +
                                             np.bincount(er, weights=np.abs(wv * x), minlength=R) + abs_s2 + sq)
            rel_h = np.minimum(1.0, seq * (xx + 3.0 * np.abs(xx - 2.0) * abs_s2 + sq) / np.maximum(hrow, 1e-300)) \
                * (hrow > 0)

        # a row steps a feature it names twice twice: the second step starts where the first one ended
        prev, last = _occurrences(er, ids)
        lvl = np.zeros(ids.shape[0], dtype=np.int64)
        for i in np.nonzero(prev >= 0)[0]:  # ascending: an entry's previous occurrence comes first
            lvl[i] = lvl[prev[i]] + 1
        cur_w, cur_v = wv.copy(), vv.copy()
        me = mult[er]
        step_w, step_v = np.zeros(ids.shape), np.zeros(vv.shape)
        grad_v = np.zeros(vv.shape)
        rw, rv = reg_w[g], reg_v[g].T  # [E], [k][E]
        for L in range(int(lvl.max(initial=0)) + 1):
            s = lvl == L
            if L:
                pi = prev[s]
                cur_w[s] = cur_w[pi] + step_w[pi]
                cur_v[:, s] = cur_v[:, pi] + step_v[:, pi]
            step_w[s] = -lr * (me[s] * x[s] + 2 * rw[s] * cur_w[s])
            grad_v[:, s] = me[s] * (x[s] * (sums[:, er[s]] - cur_v[:, s] * x[s]))
            step_v[:, s] = -lr * (grad_v[:, s] + 2 * rv[:, s] * cur_v[:, s])

        c = (count[ids] * conc_scale).astype(np.float64)
        damped = (c > 1.0) if damp else np.zeros(ids.shape, dtype=bool)
        uv = lr * (hjoint[er][None, :] + 2 * rv)
        uw = lr * (hjoint[er] + 2 * rw)
        sv = np.where(damped[None, :], gamma(c[None, :], uv), 1.0)
        sw = np.where(damped, gamma(c, uw), 1.0)
        dv, dw = sv * step_v, sw * step_w

        # budget: fp32 row arithmetic, gamma, quantisation, and the steps a difference in reg moves
        gv_abs = np.abs(sums[:, er] * x - vv * x * x)
        bv = sv * (lr * gv_abs * row_err[er] + EPS_M * lr * np.abs(me * x) * abs_s[:, er] + EPS_M * 2 * lr * rv * np.abs(vv)
                   + 2 * lr * rb.reg_v[g].T * np.abs(vv)) + 1.0 / ACC_SCALE \
            + np.abs(dv) * (EPS_GAMMA * damped + damped * gamma_cut_edge(c[None, :], uv) + edge[er])
        if eps_seq:
            bv = bv + sv * lr * np.abs(me * x) * (seq * abs_s)[:, er] + np.abs(dv) * damped * rel_h[er]
        for f in range(k):
            st.v[f] = _fold_sum(st.v[f], ids, dv[f], n, quant, fp32)
            bud.v[f] += grow * np.bincount(ids, weights=bv[f], minlength=n)
        touched = np.bincount(ids, minlength=n) > 0
        keep = last
        for f in range(k):
            sg.grad_v[f] = np.where(touched, _window_sum(ids[keep], grad_v[f][keep], n, quant, fp32), sg.grad_v[f])
        if hp.k1:
            bw = sw * (lr * np.abs(x) * row_err[er] + EPS_M * 2 * lr * rw * np.abs(wv)
                       + 2 * lr * rb.reg_w[g] * np.abs(wv)) + 1.0 / ACC_SCALE \
                + np.abs(dw) * (EPS_GAMMA * damped + damped * gamma_cut_edge(c, uw) + edge[er])
            if eps_seq:
                bw = bw + np.abs(dw) * damped * rel_h[er]
            st.w = _fold_sum(st.w, ids, dw, n, quant, fp32)
            bud.w += grow * np.bincount(ids, weights=bw, minlength=n)
            sg.grad_w = np.where(touched, _window_sum(ids[keep], (me * x)[keep], n, quant, fp32), sg.grad_w)
        if hp.k0:
            on = damp and cb > 1.0
            gb = gamma(cb, lr * hjoint) if on else np.ones(R)
            db = -lr * gb * mult
            h_edge = edge * ((1.0 if damp else 0.0) * hrow + 1.0)
            b0 = gb * lr * row_err + 1.0 / ACC_SCALE + np.abs(db) * (
                EPS_GAMMA * on + (gamma_cut_edge(cb, lr * hjoint) if on else 0.0) + np.minimum(1.0, h_edge))
            if eps_seq and on:
                b0 = b0 + np.abs(db) * rel_h
            st.w0 = float(_fold_sum(np.array([st.w0]), np.zeros(R, dtype=np.int64), db, 1, quant, fp32)[0])
            bud.w0 += grow * float(b0.sum())
        bud.windows += 1
        if trace is not None:
            trace.append(st.copy())

        if j == j_star:
            mom = moments(st)
            b = bud.bound(st)
            mom_b = _moment_bound(st, b[1], b[2])
        if not lam:
            continue

        # ---- lambda: one step per theta-step, on the rows the cursor names ----
        ve, vr = _rows(val, np.arange(r0, r1) % V)
        ids, x = val.col[ve].astype(np.int64), val.val[ve].astype(np.float64)
        y = val.target[np.arange(r0, r1) % V].astype(np.float64)
        g = sg.group[ids]
        w_, v_ = st.w[ids], st.v[:, ids]
        rw, rv = reg_w[g], reg_v[g].T
        wd = w_ - lr * (sg.grad_w[ids] + 2 * rw * w_)
        vd = v_ - lr * (sg.grad_v[:, ids] + 2 * rv * v_)
        p = np.full(R, st.w0 if hp.k0 else 0.0)
        if hp.k1:
            p += np.bincount(vr, weights=wd * x, minlength=R)
        sfd = np.stack([np.bincount(vr, weights=vd[f] * x, minlength=R) for f in range(k)]) if k else np.zeros((0, R))
        for f in range(k):
            p += 0.5 * (sfd[f] * sfd[f] - np.bincount(vr, weights=(vd[f] * x) ** 2, minlength=R))
        if hp.task == 0:
            gl = 2 * (np.clip(p, hp.min_target, hp.max_target) - y)
        else:
            gl = y * ((1.0 / (1.0 + np.exp(-y * p))) - 1.0)
        key = vr * G + g
        if hp.k1:
            lwg = -2 * lr * np.bincount(key, weights=x * w_, minlength=R * G).reshape(R, G)
            cw = -(lr * gl[:, None] * lwg)
            sg.reg_w = np.maximum(0.0, reg_w + cw.sum(0))
            rb.reg_w += grow * (REG_REL * np.abs(cw).sum(0) + 1e-300)
        if k:
            sum_f = np.stack([np.bincount(key, weights=v_[f] * x, minlength=R * G) for f in range(k)], -1)
            sdf = np.stack([np.bincount(key, weights=vd[f] * x * v_[f] * x, minlength=R * G) for f in range(k)], -1)
            lvg = -2 * lr * (np.repeat(sfd.T, G, axis=0) * sum_f - sdf)  # [R*G][k]
            cv = -(lr * np.repeat(gl, G)[:, None] * lvg)
            sg.reg_v = np.maximum(0.0, reg_v + cv.reshape(R, G, k).sum(0))
            rb.reg_v += grow * (REG_REL * np.abs(cv).reshape(R, G, k).sum(0) + 1e-300)
    rb.var_w, rb.var_v = mom_b
    return st, sg, mom, bud, rb
