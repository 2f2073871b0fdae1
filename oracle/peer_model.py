"""fp64 model of the per-epoch peer exchange (libfm_b200/csrc/fm_peer.cu).  TEST INFRASTRUCTURE ONLY.

The row-sharded path combines its G replicas once per epoch, in one of two ways:

  mean_combine        fm_peer_mean_kernel: s = 0; s += theta_q in rank order; s *= 1/G, all in fp32.  numpy's
                      fp32 arithmetic is the same IEEE arithmetic, so this model is exact and the kernel must
                      match it bit for bit.
  meanfield_combine   fm_peer_counts_mean_kernel + fm_peer_meanfield_kernel (one-shot) or
                      fm_peer_meanfield_sliced_kernel (sliced):  theta = b + gamma_i d_i  per element, with
                      b = theta0 (the state the epoch started from), d = the rank-order fp32 sum of (theta_q - b),
                      gamma = (1 - e^{-G u}) / (G (1 - e^{-u}))  (1 where u <= 1e-6) and
                          u = lr (1 + reg0) rows    for the bias       (rows = mean rows per shard)
                          u = lr (1 + regw) cnt_i   for w_i            (cnt_i = mean count of feature i per shard)
                          u = lr (hv + regv) cnt_i  for every element of V's row i,
                      hv = the mean squared V-row norm of theta0.  Padding and the words between the bias and w
                      get gamma 0: they keep exactly what theta0 holds.

States are the packed fp32 buffers as the device holds them ([w0, 0 .. | w (stride ws) .. | V[n][kp]]); the
layout is FmLearnSgdElement.params_layout()'s dict plus the factor count k.  d is formed in fp32 exactly as the
kernel forms it; gamma and the combine are fp64.  What the kernel may differ by, per element (`budget`):

  * gamma's own fp32 evaluation: G u, two expm1f (<= 1 ulp each, CUDA Programming Guide), the product G b and
    the quotient -- EPS_GAMMA = 8 half-ulps of gamma, relative, times |d|;
  * u's fp32 inputs and products: lr, (1 + reg) and the products each round once -- EPS_U = 6 half-ulps of u,
    relative; for V also hv's own error (below), weighted by hv / (hv + regv).  An error e in u moves gamma by
    |gamma'(u)| u e, and gamma' is taken in closed form;
  * hv: the kernel sums the squares in fp32 -- per thread over its float4s (4 terms each), a 256-way block tree,
    then in the next exchange's prologue over the n_part block partials (a per-thread loop and another 256-way
    tree), and divides by n.  A sum of non-negative terms whose every term passes through at most L roundings is
    within L half-ulps of the exact sum, relative: L = 4 m + 8 + ceil(n_part / 256) + 8 + 2, m = float4s per
    thread.  hv_rel_bound() states it for the launch shapes of fm_peer.cu;
  * where fp32 u may fall on the other side of the 1e-6 cut than the fp64 one: the jump |1 - gamma(u)| |d|;
  * the combine b + g d: a rounding of the product and one of the sum -- half an ulp of |gamma d| and one ulp
    of the result (a full one: the kernel's result may sit on the other side of a binade edge than the model's).
"""
from __future__ import annotations

import numpy as np

EPS32 = 2.0 ** -24  # half an fp32 ulp, relative
EPS_GAMMA = 8 * EPS32
EPS_U = 6 * EPS32
U_CUT = 1e-6
U_CUT_EDGE = 1e-5  # relative distance to the cut within which fp32 and fp64 may disagree about it


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def mean_combine(states):
    """fm_peer_mean_kernel: the rank-order fp32 sum times fp32(1 / G)."""
    s = np.zeros_like(np.asarray(states[0], dtype=np.float32))
    for q in states:
        s = s + np.asarray(q, dtype=np.float32)
    return s * np.float32(np.float32(1.0) / np.float32(len(states)))


def gamma(u, world):
    """(1 - e^{-G u}) / (G (1 - e^{-u})) in fp64; 1 where u <= 1e-6 (fm_peer.cu: mf_gamma)."""
    u = np.asarray(u, dtype=np.float64)
    on = u > U_CUT
    us = np.where(on, u, 1.0)
    g = -np.expm1(-world * us) / (world * -np.expm1(-us))
    return np.where(on, g, 1.0)


def gamma_prime(u, world):
    """d gamma / d u in closed form (0 on the u <= 1e-6 branch)."""
    u = np.asarray(u, dtype=np.float64)
    on = u > U_CUT
    us = np.where(on, u, 1.0)
    a, b = -np.expm1(-world * us), -np.expm1(-us)
    gp = (world * np.exp(-world * us) * b - a * np.exp(-us)) / (world * b * b)
    return np.where(on, gp, 0.0)


def layout_masks(layout, k, n_floats):
    """Per element of the packed state: kind (0 = gamma 0, 1 = bias, 2 = w, 3 = V) and feature index (-1: none)."""
    off_w, ws, off_v, kp, n = (int(layout[x]) for x in ("off_w", "ws", "off_v", "kp", "n"))
    kind = np.zeros(n_floats, dtype=np.int8)
    feat = np.full(n_floats, -1, dtype=np.int64)
    kind[0] = 1
    wi = off_w + np.arange(n, dtype=np.int64) * ws
    kind[wi] = 2
    feat[wi] = np.arange(n)
    vi = (off_v + np.arange(n, dtype=np.int64)[:, None] * kp + np.arange(k)[None, :]).ravel()
    kind[vi] = 3
    feat[vi] = np.repeat(np.arange(n), k)
    return kind, feat


def pack(w0, w, v, layout, k):
    """The packed fp32 state of (w0, w[n], v[k][n]), zero padding (fmb200_set_params)."""
    off_w, ws, off_v, kp, n = (int(layout[x]) for x in ("off_w", "ws", "off_v", "kp", "n"))
    out = np.zeros(off_v + n * kp, dtype=np.float32)
    out[0] = w0
    out[off_w:off_w + n * ws:ws] = w
    out[off_v:].reshape(n, kp)[:, :k] = np.asarray(v).T
    return out


def unpack(state, layout, k):
    """(w0, w[n], v[k][n]) as fp64 from a packed fp32 state."""
    off_w, ws, off_v, kp, n = (int(layout[x]) for x in ("off_w", "ws", "off_v", "kp", "n"))
    s = np.asarray(state, dtype=np.float32).astype(np.float64)
    return float(s[0]), s[off_w:off_w + n * ws:ws].copy(), s[off_v:off_v + n * kp].reshape(n, kp)[:, :k].T.copy()


def hv(theta, layout):
    """Mean squared V-row norm of a packed state, fp64: the h of V's gamma (padding columns are zero)."""
    off_v, n = int(layout["off_v"]), int(layout["n"])
    v = np.asarray(theta, dtype=np.float32)[off_v:].astype(np.float64)
    return float(np.dot(v, v)) / n if n else 0.0


def hv_rel_bound(n_vec, world, sm_count):
    """Relative error bound of the kernel's fp32 hv (module docstring), over the launch shapes that may have
    written the partials: the capture and the one-shot kernel (peer_grid over the state) and the sliced one
    (peer_grid over a slice, at most 4096 / G blocks)."""
    cdiv = lambda a, b: -(-a // b)  # noqa: E731
    grid = max(1, min(cdiv(n_vec, 256), 2 * sm_count))
    per = cdiv(n_vec, world)
    gs = max(1, min(cdiv(per, 256), 2 * sm_count, 4096 // world))
    m = max(cdiv(n_vec, 256 * grid), cdiv(per, 256 * gs))
    n_part = max(grid, gs * world)
    return (4 * m + 8 + cdiv(n_part, 256) + 8 + 2) * EPS32


def _gamma_err(u, world, rel_u):
    """|gamma_kernel - gamma| bound for fp64 u whose fp32 image has relative error rel_u."""
    g = gamma(u, world)
    err = EPS_GAMMA * g + np.abs(gamma_prime(u, world)) * u * rel_u
    near = np.abs(u - U_CUT) <= U_CUT_EDGE * U_CUT
    jump = (world - 1) / 2.0 * U_CUT * (1.0 + U_CUT_EDGE)  # 1 - gamma(u) = (G - 1) u / 2 + O(u^2) at the cut
    return np.where(near, err + jump, err)


def meanfield_combine(theta0, states, counts, rows, hv_value, hp, layout, k, hv_rel=0.0):
    """theta0 + gamma * sum_q (theta_q - theta0) over packed fp32 states.

    counts: per rank, the shard's per-feature occurrence counts [n]; rows: per rank, the shard's row count;
    hv_value: hv(theta0) (fp64); hp: lr, reg0, regw, regv; hv_rel: relative error of the kernel's hv.
    Returns (fp64 result, per-element budget, gamma per element); budget 0 where gamma is 0."""
    G = len(states)
    b = np.asarray(theta0, dtype=np.float32)
    d = np.zeros_like(b)
    for q in states:  # fp32, rank order: the kernel's sum exactly
        d = d + (np.asarray(q, dtype=np.float32) - b)
    kind, feat = layout_masks(layout, k, b.size)
    cnt = np.zeros(int(layout["n"]), dtype=np.float32)
    for c in counts:
        cnt = cnt + np.asarray(c, dtype=np.float32)
    cnt = (cnt / np.float32(G)).astype(np.float64)
    mrows = float(np.float32(sum(np.float32(r) for r in rows)) / np.float32(G))

    u = np.zeros(b.size)
    rel = np.zeros(b.size)
    u[kind == 1] = hp.lr * (1.0 + hp.reg0) * mrows
    rel[kind == 1] = EPS_U
    fw = feat[kind == 2]
    u[kind == 2] = hp.lr * (1.0 + hp.regw) * cnt[fw]
    rel[kind == 2] = EPS_U
    fv = feat[kind == 3]
    h = hv_value + hp.regv
    u[kind == 3] = hp.lr * h * cnt[fv]
    rel[kind == 3] = EPS_U + (hv_rel * hv_value / h if h > 0 else 0.0)

    g = np.where(kind > 0, gamma(u, G), 0.0)
    gerr = np.where(kind > 0, _gamma_err(u, G, rel), 0.0)
    d64 = d.astype(np.float64)
    gd = g * d64
    out = b.astype(np.float64) + gd
    budget = np.where(kind > 0, gerr * np.abs(d64) + 0.5 * ulp32(gd) + ulp32(out), 0.0)
    return out, budget, g


def combine_ratio(got, want, budget):
    """Worst |got - want| / budget over the elements with a budget (0 if none differ)."""
    got = np.asarray(got, dtype=np.float32).astype(np.float64)
    on = budget > 0
    if not np.any(on):
        return 0.0
    return float(np.max(np.abs(got[on] - want[on]) / budget[on]))


def counts_of(data, n):
    """The per-feature occurrence counts an upload publishes: every stored entry, zero-valued ones included."""
    return np.bincount(np.asarray(data.col, dtype=np.int64), minlength=n)[:n].astype(np.float64)


__all__ = ["mean_combine", "meanfield_combine", "gamma", "gamma_prime", "hv", "hv_rel_bound", "pack", "unpack",
           "layout_masks", "combine_ratio", "counts_of", "ulp32"]
