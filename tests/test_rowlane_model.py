"""CPU: the fp64 window model of the reproducible row-lane epoch (oracle/rowlane_model.py) is itself right.

tests/test_rowlane_model_gpu.py holds the kernel to this model, so the model is tied down first, where no GPU
is needed: to the sequential oracle where the two must agree (windows of one row; rows that share nothing),
to the closed form and the recurrence gamma stands for, and to a window schedule worked out by hand.
"""
import math

import numpy as np
import pytest

from libfm_b200 import Data, synth
from oracle import HParams, Port, State, rowlane_epoch_model
from oracle import rowlane_model as rm


def _state(n, k, seed, w0=0.0):
    r = np.random.default_rng(seed)
    f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
    return State(float(np.float32(w0)), f32(0.05 * r.standard_normal(n)), f32(0.1 * r.standard_normal((k, n))))


def _port_epoch(st, d, hp):
    o = Port(st.w.shape[0], st.v.shape[0], hp.k0, hp.k1)
    o.set_params(st.w0, st.w, st.v)
    o.reg0, o.regw, o.regv = hp.reg0, hp.regw, hp.regv
    o.sgd_epoch(d, hp.task, hp.lr, hp.min_target, hp.max_target)
    return State(o.w0.value, o.w, o.v)


def _rounding_tolerance(init, end, d, hp):
    """What a model epoch of one-row windows may differ from the fp64 oracle by.  The model rounds every step
    to 2^-32, the window's step to fp32 and every stepped element to fp32; the oracle does none of it.  A step
    is smaller than the element's range here, so that is two roundings of at most half an ulp of the element
    each.  m independent pairs, each rounding uniform within half an ulp, sum to sqrt(m / 6) ulp (one sigma);
    six sigma is 2.45 sqrt(m) ulp.  Those differences also shift every later score by at most E_p (bias + two
    weights + two factor rows, each |dp/dtheta| <= 1 here), and so each later step by lr E_p."""
    m = np.bincount(d.col, minlength=init.w.shape[0]).astype(np.float64)
    direct = lambda a, b, cnt: 2.45 * np.sqrt(cnt) * (rm.ulp32(np.maximum(np.abs(a), np.abs(b))) + 2.0 ** -32)
    t0 = direct(init.w0, end.w0, d.num_cases) if hp.k0 else 0.0
    tw = direct(init.w, end.w, m) if hp.k1 else np.zeros_like(m)
    tv = direct(init.v, end.v, m[None, :])
    e_p = float(t0) + 2.0 * tw.max() + 2.0 * tv.max()
    return t0 + hp.lr * d.num_cases * e_p, tw + hp.lr * m * e_p, tv + hp.lr * m[None, :] * e_p


def _assert_close(got, want, tol):
    t0, tw, tv = tol
    assert abs(got.w0 - want.w0) <= t0
    assert np.all(np.abs(got.w - want.w) <= tw)
    assert np.all(np.abs(got.v - want.v) <= tv)


@pytest.mark.parametrize("k0,k1", [(True, True), (False, True), (True, False), (False, False)])
@pytest.mark.parametrize("task", [0, 1])
def test_windows_of_one_row_are_the_sequential_oracle(task, k0, k1):
    d = synth.two_field(300, 40, 30, seed=11)
    if task == 1:
        d.target = np.where(d.target > 3, 1.0, -1.0).astype(np.float32)
    # the clamp is active on some rows: the initial scores lie around 0 and the bounds are 1 and 5
    hp = HParams(task, 0.01, 0.01, 0.02, 0.03, 1.0, 5.0, k0, k1)
    init = _state(d.num_feature, 4, seed=3)
    got, _ = rowlane_epoch_model(init, d, hp, TR=1, grid=1, damp=False, ramp_tiles=0)
    want = _port_epoch(init, d, hp)
    assert abs(got.w0 - init.w0) > 0.1 or not k0  # the epoch moved the state
    _assert_close(got, want, _rounding_tolerance(init, want, d, hp))
    # the fold left the state on the fp32 lattice
    assert np.array_equal(got.v, got.v.astype(np.float32).astype(np.float64))


@pytest.mark.parametrize("TR,grid,ramp", [(1, 1, 0), (4, 3, 0), (32, 2, 4), (64, 100, 0)])
def test_rows_that_share_nothing_make_the_windows_irrelevant(TR, grid, ramp):
    n_rows = 200
    r = np.random.default_rng(5)
    cols = r.permutation(2 * n_rows).reshape(n_rows, 2)  # every feature in exactly one row
    d = Data(np.arange(0, 2 * n_rows + 1, 2), cols.reshape(-1), r.uniform(0.5, 1.5, 2 * n_rows),
             r.integers(1, 6, n_rows), 2 * n_rows)
    hp = HParams(0, 0.02, 0.0, 0.02, 0.03, 1.0, 5.0, k0=False, k1=True)
    init = _state(d.num_feature, 8, seed=4)
    want = _port_epoch(init, d, hp)
    for damp in (False, True):  # every count is 1, so damping changes nothing either
        got, _ = rowlane_epoch_model(init, d, hp, TR, grid, damp, ramp)
        # one step per element: quantised (2^-33), rounded to fp32, and the element rounded to fp32 once more
        one = lambda a, b: 0.5 * (rm.ulp32(b - a) + rm.ulp32(np.maximum(np.abs(a), np.abs(b)))) + 2.0 ** -33
        assert np.all(np.abs(got.w - want.w) <= one(init.w, want.w))
        assert np.all(np.abs(got.v - want.v) <= one(init.v, want.v))
        assert got.w0 == init.w0


def test_gamma_is_the_closed_form():
    for c in [1.5, 2.0, 7.0, 33.0, 400.0, 4224.0, 1e6]:
        for u in [1e-4, 1e-3, 0.01, 0.03, 0.25, 0.9, 0.999]:
            want = 1.0 if c * u < 1e-3 else min(1.0, -math.expm1(c * math.log1p(-u)) / (c * u))
            assert rm.gamma(c, u) == pytest.approx(want, rel=1e-14), (c, u)
    assert rm.gamma(400.0, 1.0) == pytest.approx(1.0 / 400.0)  # (1-u)^c = 0 from u = 1 on
    assert rm.gamma(400.0, 1.5) == pytest.approx(1.0 / 600.0)
    for c in [0.0, 0.5, 1.0]:
        assert rm.gamma(c, 0.3) == 1.0
    assert rm.gamma(5.0, 0.0) == 1.0 and rm.gamma(5.0, -0.1) == 1.0
    assert rm.gamma(9.0, 1e-4) == 1.0 and rm.gamma(11.0, 1e-4) < 1.0  # the cut at c u = 1e-3
    g = rm.gamma(np.array([1.0, 4.0]), np.array([0.25, 0.25]))
    assert g.tolist() == [1.0, 1.0 - 0.75 ** 4]


@pytest.mark.parametrize("c,u", [(2, 0.5), (4, 0.25), (37, 0.03), (400, 0.012)])
def test_gamma_scaled_concurrent_steps_move_as_far_as_sequential_ones(c, u):
    """DESIGN.md section 3.3: c sequential steps each contract the residual by (1 - u); c concurrent steps, all
    taken from the starting residual and scaled by gamma(c, u), end at the same place."""
    theta, target = 0.3, 2.0
    seq = theta
    for _ in range(c):
        seq -= u * (seq - target)
    conc = theta + c * float(rm.gamma(float(c), u)) * (-u * (theta - target))
    assert conc == pytest.approx(seq, rel=1e-12)


def test_window_arithmetic_by_hand():
    """Three tiles of two rows, windows of two tiles, every row naming feature 0 with x = 1; no factors (v = 0).
    lr = 1/4, no clamp, no feature damping.  The bias step of a tile of T = 2 rows is
    -lr gamma(4, lr H/T) M with H = 2 (curvature 1 per row), so gamma(4, 1/4) = 1 - (3/4)^4 = 175/256.

    Window 1 (rows 0-3, y = 1) reads w0 = w = 0: p = 0, mult = -1 for all four rows, though rows 2-3 are the
    second tile.  w <- 4/4 = 1; each tile's M = -2 steps the bias by (1/4)(175/256) 2: w0 <- 175/256.
    Window 2 (rows 4-5, y = 3) reads the fold: p = 1 + 175/256, mult = -337/256.
    w <- 1 + 2 (337/1024); w0 <- 175/256 + (1/4)(175/256)(337/128)."""
    d = Data(np.arange(7), np.zeros(6), np.ones(6), [1, 1, 1, 1, 3, 3], 1)
    hp = HParams(0, 0.25, 0.0, 0.0, 0.0, -100.0, 100.0)
    init = State(0.0, np.zeros(1), np.zeros((1, 1)))
    got, bud = rowlane_epoch_model(init, d, hp, TR=2, grid=2, damp=False, ramp_tiles=0)
    assert bud.windows == 2
    assert got.w[0] == 1.0 + 674.0 / 1024.0
    assert got.w0 == 175.0 / 256.0 + 175.0 * 337.0 / (4.0 * 256.0 * 128.0)
    assert got.v[0, 0] == 0.0
    # a ramp window has its own concurrency: tile 0 alone, c = TR = 2, gamma(2, 1/4) = 7/8
    got, bud = rowlane_epoch_model(init, d, hp, TR=2, grid=2, damp=False, ramp_tiles=1)
    assert bud.windows == 2  # tile 0 | tiles 1, 2
    # tile 0: w = 1/2, w0 = (1/4)(7/8) 2 = 7/16; tiles 1 and 2 read p = 15/16: rows 2-3 mult = -1/16,
    # rows 4-5 mult = -33/16; w <- 1/2 + (2/16 + 66/16)/4; w0 <- 7/16 + (1/4)(175/256)(2/16 + 66/16)
    assert got.w[0] == 0.5 + 68.0 / 64.0
    assert got.w0 == 7.0 / 16.0 + 175.0 * 68.0 / (4.0 * 256.0 * 16.0)


def test_feature_damping_and_regularisation_by_hand():
    """Two rows of one tile share feature 0 (count 2, whole data set in flight: c = 2), k0 off, damping on.
    hjoint = curv (0 + xx) = 1, u = lr (1 + regw) = 1/4 (1 + 1) = 1/2, gamma(2, 1/2) = 3/4.
    w = 1/2, y = 2: p = 1/2, mult = -3/2; step = (3/4)(-lr mult - lr regw w) = (3/4)(3/8 - 1/8) = 3/16 per
    row; w <- 1/2 + 3/8.  Undamped: 1/2 + 2 (1/4)."""
    d = Data(np.arange(3), np.zeros(2), np.ones(2), [2, 2], 1)
    hp = HParams(0, 0.25, 0.0, 1.0, 0.0, -100.0, 100.0, k0=False)
    init = State(0.0, np.array([0.5]), np.zeros((1, 1)))
    got, _ = rowlane_epoch_model(init, d, hp, TR=2, grid=1, damp=True, ramp_tiles=0)
    assert got.w[0] == 0.5 + 3.0 / 8.0
    undamped, _ = rowlane_epoch_model(init, d, hp, TR=2, grid=1, damp=False, ramp_tiles=0)
    assert undamped.w[0] == 0.5 + 2.0 / 4.0


def test_quantisation_rounds_to_even_and_cancels():
    q = rm.quantise(np.array([2.0 ** -33, 3 * 2.0 ** -33, -(2.0 ** -33), 0.3, -0.3]))
    assert q[:3].tolist() == [0.0, 2.0, -0.0]  # ties go to the even multiple
    assert q[3] == -q[4] and q[3] == np.rint(0.3 * 2.0 ** 32)
    assert rm._exact_sums(np.zeros(5, dtype=np.int64), q, 1)[0] == 2.0
    # +q and -q in one window leave the element untouched, bit for bit
    # (p = 0 and mult = -0.7 in both rows, x = +1 and -1: the steps are +0.21 and -0.21)
    d = Data(np.arange(3), np.zeros(2), [1.0, -1.0], [0.7, 0.7], 1)
    hp = HParams(0, 0.3, k0=False, min_target=-100.0, max_target=100.0)
    got, _ = rowlane_epoch_model(State(0.0, np.zeros(1), np.zeros((2, 1))), d, hp, TR=2, grid=1, damp=False,
                                 ramp_tiles=0)
    assert got.w[0] == 0.0 and not np.signbit(got.w[0])
    # the fold rounds the integer sum to fp32, then adds in fp32
    assert rm.fold(1.0, 2.0 ** 32 * 2.0 ** -24) == 1.0  # 1 + 2^-24 ties to even
    assert rm.fold(1.0, 2.0 ** 32 * 2.0 ** -23) == 1.0 + 2.0 ** -23
    assert rm.fold(0.123, 0.0) == 0.123  # no step: the element is not rewritten


@pytest.mark.parametrize("n_tiles,grid,ramp", [(t, g, r) for t in [1, 4, 32, 33, 40] for g in [1, 3, 32, 132]
                                               for r in [0, 4] if r <= t])
def test_window_list_matches_the_kernels_count(n_tiles, grid, ramp):
    wins = rm.windows(n_tiles, ramp, grid)
    assert len(wins) == ramp + (n_tiles - ramp + grid - 1) // grid  # rowlane_windows, fm_hogwild_common.cuh
    assert [w for w in wins[:ramp]] == [(t, 1) for t in range(ramp)]
    assert all(nt == grid for _, nt in wins[ramp:-1])
    tiles = [t for t0, nt in wins for t in range(t0, t0 + nt)]
    assert tiles == list(range(n_tiles))  # every tile once, in file order
    assert 1 <= wins[-1][1] <= max(grid, 1)


def test_c2_sized_epochs_run_in_seconds():
    import time
    d = synth.movielens_1m_shaped(seed=7)
    st = _state(d.num_feature, 8, seed=2)
    hp = HParams(0, 0.01, min_target=1.0, max_target=5.0)
    t = time.process_time()
    bud = None
    for e in range(3):
        st, bud = rowlane_epoch_model(st, d, hp, TR=256, grid=396, damp=True, ramp_tiles=4 if e == 0 else 0, budget=bud)
    assert time.process_time() - t < 60.0
    assert bud.windows == 3 * 10 + 4 and np.isfinite(st.v).all()
