"""fp64 model of the free-running row-group HOGWILD epoch (fm_sgd_hogwild_kernel, DESIGN.md section 3.3) on
data whose result no schedule can change.  TEST INFRASTRUCTURE ONLY.

The kernel claims tiles from a counter and its fp32 reductions land in any order, so in general its result is
not a function of its input.  It is one on data built like this, and the model refuses any other:

  * every non-zero entry names a feature that no other non-zero entry names.  Each row then reads its own
    features at the value the epoch started with, and each element takes exactly one non-zero step;
  * zero-valued entries name those features again, in any row (their live entry's row included).  They raise
    the occurrence table that c_i = count_i * conc_scale is read from, so gamma drops far below 1, but with
    regw = regv = 0 each adds exactly 0 to every sum of the score and of hrow, and its step is exactly +-0;
  * the bias is off, or the epoch is one tile: warp 0 reads w0 once and one damped reduction writes it.

On such data the epoch is: every row scored from the state the epoch found; its steps damped by
gamma(c_i, lr (h_joint + reg)) where DAMP is compiled in and c_i > 1; each element's step added to it in fp32;
one bias step -lr gamma(max(w0_conc, 1), lr (H/T + reg0)) M for the tile.  Plain vectorised numpy over the
entries; it never calls into the library.  The state is fp64 values exactly representable in fp32, v
factor-major [k][n] as oracle.Port holds it.

Beside the state the model returns, per element, a bound on what the kernel's fp32 arithmetic may differ by
(`Budget`).  A row of n entries is summed by its lanes in sequences of at most n terms and then by a shuffle
tree, so its score is off by at most

    dp = EPS_S (n + SEQ_EXTRA) (|w0| + sum_i |w_i x_i| + sum_f (sum_i |v_if x_i|)^2 + sum_i,f (v_if x_i)^2)

and each per-factor sum s_f by EPS_S (n + SEQ_EXTRA) sum_i |v_if x_i|; hrow, whose (xx - 2) s2 + sq may cancel,
by EPS_S (n + SEQ_EXTRA) (xx + 3 |xx - 2| sum_f (sum_i |v_if x_i|)^2 + sq).  A step
gamma lr (-mult g - reg theta) then carries

    gamma lr (|g| dmult + |mult| (|x| ds_f + EPS_M (|s_f x| + |v x^2|)) + EPS_M reg |theta|)
  + |step| (EPS_GAMMA + du/u + the q < 1e-3 cut)   where damped   (__expf(c __logf(1 - u)), and u's own error)
  + |step|                                          at a clamp edge (the secant curvature jumps)

with dmult <= dp (the loss multiplier is 1-Lipschitz in the score) and u = lr (h_joint + reg), whose relative
error follows from dp (through the curvature) and from hrow's.  The bias step's bound is the same sum over the
tile's rows, with EPS_M (T + SEQ_EXTRA) for the fp32 sums of the T rows' multipliers and curvatures.  One fp32
ulp of the element is added when compared (Budget.bound).  EPS_S was calibrated on an H100 (DESIGN.md
section 3.3 has the measured ratios); EPS_M and EPS_GAMMA are the row-lane model's.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from .rowlane_model import (EPS_GAMMA, EPS_M, Budget, HParams, State, gamma, gamma_cut_edge, loss_step,
                            row_curvature, ulp32)

__all__ = ["EPS_S", "SEQ_EXTRA", "Geometry", "geometry", "concurrency", "row_scores", "rowgroup_epoch_model",
           "Budget", "HParams", "State", "ulp32"]

EPS_S = 2.0 ** -22  # error of an fp32 sum per term it adds in sequence, relative to the terms' magnitudes
SEQ_EXTRA = 6       # the shuffle tree over a group's <= 32 lanes (5 levels) and the bias add

# row_class (fmb200_internal.h): register-cache class -> (R factor chunks, RW weights cached per lane, U row sets)
CLASSES = {-1: (1, 1, 4), 0: (2, 1, 2), 1: (8, 2, 1), 2: (20, 2, 1), 3: (40, 2, 1)}


@dataclass(frozen=True)
class Geometry:
    G: int    # lanes spanning a factor row (float4 chunks)
    S: int    # slots walking a row's entries
    cls: int  # register-cache class
    R: int
    RW: int
    U: int
    rows_per_cta_step: float  # rows a CTA has in flight: warps x rows per warp x U

    @property
    def E(self) -> int:
        return self.G * self.S


def geometry(k: int, n_rows: int, nnz: int, threads: int = 0) -> Geometry:
    """pick_geometry, pick_r and the launcher's rows_per_cta_step (fm_hogwild.cu) for k factors, a data set of
    n_rows rows and nnz entries, and the tuning's thread count (0: the default 256)."""
    gp = ((k + 3) & ~3) // 4
    g = 1
    while g < gp:
        g <<= 1
    g = min(g, 32)
    avg = nnz / n_rows if n_rows else 1.0
    s = 1
    while s < avg and s < 8:
        s <<= 1
    while g * s > 32:
        s >>= 1
    s = max(s, 1)
    iters = int((avg + s - 1) / s)
    cls = -1 if iters <= 1 else (0 if iters <= 2 else (1 if iters <= 8 else (2 if (iters <= 20 or g < 32) else 3)))
    R, RW, U = CLASSES[cls]
    threads = min(threads, 256) if threads > 0 else 256
    return Geometry(g, s, cls, R, RW, U, (threads // 32) * (32.0 / (g * s)) * U)


def concurrency(geo: Geometry, n_rows: int, grid: int, tile_rows: int):
    """(conc_scale, w0_conc) as the launcher computes them for a grid of `grid` CTAs, in fp32."""
    conc_scale = float(np.float32(min(float(n_rows), grid * geo.rows_per_cta_step) / n_rows))
    w0_conc = float(np.float32(min(float(n_rows), float(grid * tile_rows))))
    return conc_scale, w0_conc


def _entries(data):
    rp = data.row_ptr.astype(np.int64)
    N = int(rp.shape[0] - 1)
    n_row = np.diff(rp)
    return N, n_row, np.repeat(np.arange(N, dtype=np.int64), n_row), data.col.astype(np.int64), \
        data.val.astype(np.float64)


def _rows(st: State, data, hp: HParams):
    """Scores and the sums behind them, per row, from the fp32 state `st`, with their fp32 error bounds."""
    N, n_row, er, ids, x = _entries(data)
    k = st.v.shape[0]
    vv = st.v[:, ids]
    vx = vv * x
    sums = np.stack([np.bincount(er, weights=vx[f], minlength=N) for f in range(k)]) if k else np.zeros((0, N))
    a_f = np.stack([np.bincount(er, weights=np.abs(vx[f]), minlength=N) for f in range(k)]) if k \
        else np.zeros((0, N))
    sq = np.bincount(er, weights=(vx * vx).sum(0), minlength=N)
    s2 = (sums * sums).sum(0)
    s2abs = (a_f * a_f).sum(0)
    wv = st.w[ids] if hp.k1 else np.zeros(ids.shape)
    lin = np.bincount(er, weights=wv * x, minlength=N)
    labs = np.bincount(er, weights=np.abs(wv * x), minlength=N)
    w0 = st.w0 if hp.k0 else 0.0
    p = w0 + lin + 0.5 * (s2 - sq)
    xx = np.bincount(er, weights=x * x, minlength=N)
    seq = EPS_S * (n_row + SEQ_EXTRA)
    dp = seq * (abs(w0) + labs + s2abs + sq)
    ds = seq * a_f
    dhrow = seq * (xx + 3.0 * np.abs(xx - 2.0) * s2abs + sq)
    return dict(N=N, er=er, ids=ids, x=x, vv=vv, wv=wv, sums=sums, sq=sq, s2=s2, xx=xx, p=p, dp=dp, ds=ds,
                dhrow=dhrow)


def row_scores(state: State, data, hp: HParams):
    """(p, dp): every row's score from `state` in fp64 and the bound on the fp32 kernels' error in it."""
    r = _rows(state, data, hp)
    return r["p"], r["dp"]


def _curv_error(hp: HParams, p, y, mult, curv, dp):
    """Bound on the fp32 curvature's error from the score's: s(1-s) moves by at most s(1-s) dp; the secant
    (pc - y)/(p - y) of a clamped row by |mult| dp / (p - y)^2, and never by more than 1."""
    if hp.task == 1:
        return curv * dp
    den = p - y
    clamped = np.clip(p, hp.min_target, hp.max_target) != p
    with np.errstate(divide="ignore", invalid="ignore"):
        sec = np.where(np.abs(den) > 0.0, np.abs(mult) * dp / np.where(den == 0.0, 1.0, den) ** 2, 1.0)
    return np.where(clamped, np.minimum(sec, 1.0), 0.0)


def check_preconditions(data, hp: HParams, tile_rows: int) -> None:
    """Refuses data on which the kernel's result depends on its schedule (ValueError)."""
    live = data.val != 0
    ids = data.col[live]
    if np.unique(ids).size != ids.size:
        raise ValueError("a non-zero entry shares its feature with another non-zero entry: which row reads "
                         "the feature first would decide the result")
    if (~live).any() and (hp.regw != 0.0 or hp.regv != 0.0):
        raise ValueError("zero-valued entries with regw or regv != 0: each would take a regulariser step, "
                         "read whenever its row runs")
    N = int(data.row_ptr.shape[0] - 1)
    if hp.k0 and N > tile_rows:
        raise ValueError("k0 over more than one tile: each tile reads the bias whenever it starts")


def rowgroup_epoch_model(state: State, data, hp: HParams, conc_scale: float, w0_conc: float, damp: bool,
                         tile_rows: int):
    """One epoch of fm_sgd_hogwild_kernel over `data` (row_ptr, col, val, target), on tiles of `tile_rows` rows,
    with the launcher's conc_scale and w0_conc and DAMP = damp.  Returns (state, budget)."""
    check_preconditions(data, hp, tile_rows)
    n = state.w.shape[0]
    st = state.copy()
    bud = Budget.zero(st)
    r = _rows(st, data, hp)
    N, er, ids, x = r["N"], r["er"], r["ids"], r["x"]
    if N == 0:
        return st, bud
    lr = hp.lr
    y = data.target.astype(np.float64)
    p, dp = r["p"], r["dp"]
    mult, curv, edge = loss_step(hp, p, y)
    hrow, hjoint = row_curvature(hp, curv, r["xx"], r["s2"], r["sq"], damp)
    dcurv = _curv_error(hp, p, y, mult, curv, dp)
    k0 = 1.0 if hp.k0 else 0.0
    dhjoint = dcurv * (k0 + hrow) + curv * r["dhrow"] if damp else dcurv

    # ---- per entry: concurrency, damping, steps ----
    count = np.bincount(ids, minlength=n).astype(np.float32)
    c = (count[ids] * np.float32(conc_scale)).astype(np.float64)  # fp32, as the kernel decides c > 1
    damped = (c > 1.0) if damp else np.zeros(ids.shape, dtype=bool)
    dm = dp[er]
    ed = edge[er].astype(np.float64)

    def scale(reg):
        u = lr * (hjoint[er] + reg)
        g = np.where(damped, gamma(c, u), 1.0)
        with np.errstate(divide="ignore", invalid="ignore"):
            rho = np.where(u > 0.0, lr * dhjoint[er] / np.where(u > 0.0, u, 1.0), 0.0)
        rel = damped * (EPS_GAMMA + rho + gamma_cut_edge(c, u))
        return g, rel

    sv, rel_v = scale(hp.regv)
    vv, sums = r["vv"], r["sums"]
    x2 = x * x
    grad = sums[:, er] * x - vv * x2
    dv = sv * (-lr * mult[er] * grad - lr * hp.regv * vv)
    bv = sv * lr * (np.abs(grad) * dm + np.abs(mult[er]) * (np.abs(x) * r["ds"][:, er] + EPS_M * (
        np.abs(sums[:, er] * x) + np.abs(vv * x2))) + EPS_M * hp.regv * np.abs(vv)) + np.abs(dv) * (rel_v + ed)
    for f in range(st.v.shape[0]):
        step = np.bincount(ids, weights=dv[f], minlength=n)  # one non-zero step per element: exact
        st.v[f] = (st.v[f].astype(np.float32) + step.astype(np.float32)).astype(np.float64)
        bud.v[f] = np.bincount(ids, weights=bv[f], minlength=n)
    if hp.k1:
        sw, rel_w = scale(hp.regw)
        wv = r["wv"]
        dw = sw * (-lr * mult[er] * x - lr * hp.regw * wv)
        bw = sw * lr * (np.abs(x) * dm + EPS_M * (np.abs(mult[er] * x) + hp.regw * np.abs(wv))) \
            + np.abs(dw) * (rel_w + ed)
        step = np.bincount(ids, weights=dw, minlength=n)
        st.w = (st.w.astype(np.float32) + step.astype(np.float32)).astype(np.float64)
        bud.w = np.bincount(ids, weights=bw, minlength=n)

    # ---- the tile's bias step (one tile: every row read the w0 the epoch found) ----
    if hp.k0:
        T = float(N)
        M = mult.sum() + T * hp.reg0 * st.w0
        H = hjoint.sum()
        cb = max(w0_conc, 1.0)
        u = lr * (H / T + hp.reg0)
        gb = float(gamma(cb, u))
        step0 = -lr * gb * M
        sums_err = EPS_M * (T + SEQ_EXTRA)
        dM = dp.sum() + sums_err * (np.abs(mult).sum() + T * hp.reg0 * abs(st.w0))
        # a row at a clamp edge may enter H with curvature 1 or 0
        dH = dhjoint.sum() + sums_err * H + (edge * ((1.0 if damp else 0.0) * hrow + 1.0)).sum()
        rho = min(1.0, dH / (H + T * hp.reg0)) if H + T * hp.reg0 > 0.0 else 0.0
        b0 = gb * lr * dM + abs(step0) * ((EPS_GAMMA + rho) * (cb > 1.0 and u > 0.0) + float(gamma_cut_edge(cb, u)))
        st.w0 = float(np.float32(np.float32(st.w0) + np.float32(step0)))
        bud.w0 = float(b0)
    bud.windows = 1
    return st, bud
