"""fp64 model of the reproducible row-lane HOGWILD epoch (DESIGN.md section 3.3).  TEST INFRASTRUCTURE ONLY.

The epoch is a sequence of windows of file-order rows.  Every row of a window is scored from the state as
the window found it; its steps are damped by the mean-field scale gamma(c, u), rounded to multiples of
2^-32, summed exactly and folded into the fp32 state behind the window.  Nothing here knows about CTAs,
warps, the dealt order or the in-warp merge: the design's claim is that none of them changes the result
beyond fp32 rounding, and tests/test_rowlane_model_gpu.py holds the kernel to that.

Plain vectorised numpy; it never calls into the library.  The state is fp64 values that are exactly
representable in fp32, v factor-major [k][n] as oracle.Port holds it.

Beside the state the model accumulates, per element, a bound on what fp32 row arithmetic may differ by
(`Budget`):

    sum over the rows that step it of  gamma lr |dp/dtheta| (EPS_P (1 + |p|) + EPS_M |mult|)
  + EPS_GAMMA * sum |step|  over damped steps          (__expf(c * __logf(1 - u)))
  + 5e-4 |step| where c u is within 1e-5 of gamma's q < 1e-3 cut
  + 2^-32 per step                                     (quantisation)
  + the whole step of a row within 1e-5 of a clamp bound its target sits on (the secant curvature jumps)

each window's share scaled by (1 + KAPPA * windows so far) for what earlier differences feed forward, plus
one fp32 ulp of the element when compared.  The four constants were calibrated on an H100 from one-window
epochs (DESIGN.md section 3.3 has the measured ratios).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

EPS_P = 2e-6      # relative error of an fp32 score (about 30 fp32 half-ulps: a dozen fused operations)
EPS_M = 2e-6      # relative error of a step's fp32 products and of a tile's fp32 sums
EPS_GAMMA = 2e-4  # relative error of gamma: the exponent c log(1 - u) carries c times the error of __logf
KAPPA = 0.1       # feed-forward of earlier windows' differences, per window
GAMMA_CUT_JUMP = 5e-4  # gamma drops from 1 to 1 - q/2 at its q < 1e-3 cut; fp32 may put c u on the other side
# The windowed epochs' warp-per-row score (rowlane_epoch_model's eps_seq, oracle/sgda_window_model.py): each lane
# adds n ceil(k / 32) terms in sequence, then a shuffle tree; the row-lane calibration above never saw such rows.
EPS_SEQ = 2.0 ** -22  # error of an fp32 sum per term it adds in sequence, relative to the terms' magnitudes
SEQ_EXTRA = 6         # the shuffle tree over 32 lanes (5 levels) and the bias add

ACC_SCALE = 2.0 ** 32
CLAMP_EDGE = 1e-5


@dataclass
class HParams:
    task: int  # 0 regression, 1 classification (targets -1 / +1)
    lr: float
    reg0: float = 0.0
    regw: float = 0.0
    regv: float = 0.0
    min_target: float = 0.0
    max_target: float = 0.0
    k0: bool = True
    k1: bool = True


@dataclass
class State:
    w0: float
    w: np.ndarray  # [n]
    v: np.ndarray  # [k][n]

    def copy(self) -> "State":
        return State(float(self.w0), self.w.copy(), self.v.copy())


@dataclass
class Budget:
    """Per-element bound on |kernel - model|, and the windows it was accumulated over."""
    w0: float
    w: np.ndarray
    v: np.ndarray
    windows: int = 0

    @staticmethod
    def zero(state: State) -> "Budget":
        return Budget(0.0, np.zeros_like(state.w), np.zeros_like(state.v))

    def bound(self, state: State):
        """(w0, w, v) bounds: what was accumulated plus one fp32 ulp of the element."""
        return (self.w0 + ulp32(state.w0), self.w + ulp32(state.w), self.v + ulp32(state.v))


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def gamma(c, u):
    """gamma(c, u) = (1 - (1-u)^c) / (c u): the scale at which c concurrent steps move a parameter as far as
    c sequential steps that each contract the residual by (1 - u).  1 for c <= 1, u <= 0 and c u < 1e-3."""
    c, u = np.broadcast_arrays(np.asarray(c, dtype=np.float64), np.asarray(u, dtype=np.float64))
    q = c * u
    on = (c > 1.0) & (u > 0.0) & (q >= 1e-3)
    qs = np.where(on, q, 1.0)
    log_a = np.where(u < 1.0, np.log1p(-np.where(u < 1.0, u, 0.0)), -np.inf)  # u >= 1: (1-u)^c is taken as 0
    g = -np.expm1(np.where(on, c * log_a, 0.0)) / qs
    return np.where(on, np.minimum(1.0, g), 1.0)


def gamma_cut_edge(c, u):
    """GAMMA_CUT_JUMP where fp32 may see c u on the other side of gamma's cut, else 0."""
    q = np.asarray(c, dtype=np.float64) * u
    return GAMMA_CUT_JUMP * ((np.asarray(c) > 1.0) & (np.abs(q - 1e-3) < 1e-8))


def quantise(d):
    """A step as the accumulator takes it: the nearest multiple of 2^-32, ties to even (__float2ll_rn)."""
    return np.rint(np.asarray(d, dtype=np.float64) * ACC_SCALE)


def fold(x, q):
    """state <- fp32(state + fp32(sum 2^-32)) where the integer sum q is not zero (acc_fold)."""
    x = np.asarray(x, dtype=np.float64)
    q = np.asarray(q, dtype=np.float64)
    step = (q / ACC_SCALE).astype(np.float32)
    return np.where(q != 0.0, (x.astype(np.float32) + step).astype(np.float64), x)


def windows(n_tiles: int, ramp_tiles: int, grid: int):
    """[(first tile, tiles)]: ramp_tiles windows of one tile, then windows of grid tiles, the last what is left."""
    out = [(t, 1) for t in range(min(ramp_tiles, n_tiles))]
    t = len(out)
    while t < n_tiles:
        out.append((t, min(grid, n_tiles - t)))
        t += grid
    return out


def loss_step(hp: HParams, p, y):
    """(mult, curv, edge): the loss multiplier, the secant curvature of the loss in the raw score, and the rows
    whose curvature fp32 may see on the other side of its jump (score at a clamp bound the target sits on)."""
    if hp.task == 0:
        pc = np.clip(p, hp.min_target, hp.max_target)
        mult = pc - y
        den = p - y
        with np.errstate(divide="ignore", invalid="ignore"):
            sec = np.where(np.abs(den) > 1e-12, np.clip(mult / np.where(den == 0.0, 1.0, den), 0.0, 1.0), 0.0)
        curv = np.where(pc == p, 1.0, sec)
        tol = CLAMP_EDGE * (1.0 + np.abs(p))
        edge = ((np.abs(p - hp.min_target) < tol) & (np.abs(y - hp.min_target) < tol)) | \
               ((np.abs(p - hp.max_target) < tol) & (np.abs(y - hp.max_target) < tol))
        return mult, curv, edge
    sg = 1.0 / (1.0 + np.exp(-y * p))
    return -y * (1.0 - sg), sg * (1.0 - sg), np.zeros(p.shape, dtype=bool)


def row_curvature(hp: HParams, curv, xx, s2, sq, damp: bool):
    """(hrow, hjoint) of rows whose score has per-factor sums s_f (s2 = sum_f s_f^2), sq = sum_i,f (v_if x_i)^2
    and xx = sum_i x_i^2: hrow = |d p / d(w, V)|^2 by the one-hot identity (RowGroup::reduce), and the joint
    curvature every block of the row contracts with (the loss curvature alone without damping)."""
    hrow = (xx if hp.k1 else 0.0) + np.maximum((xx - 2.0) * s2 + sq, 0.0)
    hjoint = curv * ((1.0 if hp.k0 else 0.0) + hrow) if damp else curv
    return hrow, hjoint


def _exact_sums(idx, q, n):
    """Per-index sums of the integers q, exact: integers add exactly in fp64 while every partial sum stays
    below 2^53, which is checked."""
    assert np.abs(q).sum() < 2.0 ** 53, "integer step sums leave the exact range of fp64"
    return np.bincount(idx, weights=q, minlength=n)


def rowlane_epoch_model(state: State, data, hp: HParams, TR: int, grid: int, damp: bool, ramp_tiles: int,
                        budget: Budget | None = None, eps_seq: float = 0.0):
    """One epoch over `data` (row_ptr, col, val, target) in tiles of TR rows and windows of `grid` tiles.
    Returns (state, budget); pass the budget of the previous epoch to carry it on.

    It is also the windowed HOGWILD SGD epoch (fmb200_set_reproducible, fm_sgd_window.cu) with TR = its tile rows
    and grid = its window tiles.  eps_seq > 0 (EPS_SEQ) adds to the budget a term for what the row-lane calibration
    did not cover there: rows of tens of entries and k up to 128.  A warp scores a row with its lanes over factors,
    each lane summing n * ceil(k / 32) terms in sequence before a 5-level shuffle tree, so with
    L = eps_seq (n ceil(k / 32) + SEQ_EXTRA)

        the score carries      L (|w0| + sum_i |w_i x_i| + sum_f (sum_i |v_if x_i|)^2 + sum_i,f (v_if x_i)^2) more,
        each per-factor sum    L sum_i |v_if x_i|,
        h_row (damped steps)   L (xx + 3 |xx - 2| sum_f (sum_i |v_if x_i|)^2 + sq) relative to h_row,

    as oracle/rowgroup_model.py bounds its sub-warp rows with EPS_S = 2^-22.  The term widens the budget and never
    changes the state; eps_seq = 0 leaves it out."""
    n = state.w.shape[0]
    k = state.v.shape[0]
    N = int(data.row_ptr.shape[0] - 1)
    rp = data.row_ptr.astype(np.int64)
    col = data.col.astype(np.int64)
    val = data.val.astype(np.float64)
    tgt = data.target.astype(np.float64)
    erow = np.repeat(np.arange(N, dtype=np.int64), np.diff(rp))
    count = np.bincount(col, minlength=n).astype(np.float32)
    n_tiles = (N + TR - 1) // TR
    lr = hp.lr
    lanes_seq = -(-k // 32)  # factors per lane of the windowed epoch's warp

    st = state.copy()
    bud = Budget.zero(st) if budget is None else Budget(budget.w0, budget.w.copy(), budget.v.copy(), budget.windows)

    for j, (t0, nt) in enumerate(windows(n_tiles, ramp_tiles, grid)):
        in_ramp = j < ramp_tiles
        flight = TR if in_ramp else min(N, grid * TR)
        conc_scale = np.float32(flight / N)  # the launcher's fp32 value, so c > 1 decides as on the device
        w0_conc = float(flight)
        r0, r1 = t0 * TR, min(N, (t0 + nt) * TR)
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
        if eps_seq:  # the lanes' sequences (L of the notes above, per row)
            L = eps_seq * (np.diff(rp[r0:r1 + 1]).astype(np.float64) * lanes_seq + SEQ_EXTRA)
            abs_s = np.stack([np.bincount(er, weights=np.abs(vx[f]), minlength=R) for f in range(k)]) if k \
                else np.zeros((0, R))
            abs_s2 = (abs_s * abs_s).sum(0)
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
            starts = np.arange(0, R, TR)
            T = np.minimum(TR, R - starts).astype(np.float64)
            M = np.add.reduceat(mult, starts) + T * hp.reg0 * st.w0
            H = np.add.reduceat(hjoint, starts)
            cb = max(w0_conc, 1.0)
            gb = gamma(cb, lr * (H / T + hp.reg0))
            step = -lr * gb * M
            # a row at a clamp edge may enter H with curvature 1 or 0: |d gamma / gamma| <= |dH / H|
            h_edge = np.add.reduceat(edge * ((1.0 if damp else 0.0) * hrow + 1.0), starts)
            rel_edge = np.minimum(1.0, h_edge / np.maximum(H, 1e-300)) * (h_edge > 0)
            b0 = gb * lr * (np.add.reduceat(row_err, starts) + EPS_M * T * hp.reg0 * abs(st.w0)) + 1.0 / ACC_SCALE \
                + np.abs(step) * (EPS_GAMMA * (cb > 1.0) + gamma_cut_edge(cb, lr * (H / T + hp.reg0)) + rel_edge)
            st.w0 = float(fold(st.w0, quantise(step).sum()))
            bud.w0 += grow * float(b0.sum())
        bud.windows += 1
    return st, bud
