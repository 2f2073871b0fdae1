"""CPU: the model of the windowed HOGWILD SGD epoch, oracle/rowlane_model.py's rowlane_epoch_model with the budget's
sequence term (eps_seq).  The term widens the budget and never changes the state; a one-row window checked by hand
shows what the term adds."""
import numpy as np
import pytest

from libfm_b200 import Data, synth
from oracle import HParams, State, rowlane_epoch_model
from oracle.rowlane_model import EPS_SEQ, SEQ_EXTRA


def _state(n, k, seed):
    r = np.random.default_rng(seed)
    v = r.standard_normal((k, n)).astype(np.float32).astype(np.float64) * 0.1
    w = r.standard_normal(n).astype(np.float32).astype(np.float64) * 0.1
    return State(0.5, w, v)


def _same(a, b):
    return a.w0 == b.w0 and np.array_equal(a.w, b.w) and np.array_equal(a.v, b.v)


@pytest.mark.parametrize("k,task,damp,ramp,k0,k1", [(5, 0, True, 4, True, True), (40, 0, False, 0, True, False),
                                                     (3, 1, True, 0, False, True)])
def test_the_term_widens_the_budget_only(k, task, damp, ramp, k0, k1):
    d = synth.ragged(3000, 200, 12, seed=4)
    if task == 1:
        d = Data(d.row_ptr, d.col, d.val, np.where(d.target > 3, 1.0, -1.0), d.num_feature)
    hp = HParams(task, 0.01, 0.01, 0.02, 0.03, float(d.target.min()), float(d.target.max()), k0, k1)
    st = _state(200, k, 1)
    a, ba = rowlane_epoch_model(st, d, hp, TR=32, grid=4, damp=damp, ramp_tiles=ramp)
    c, bc = rowlane_epoch_model(st, d, hp, TR=32, grid=4, damp=damp, ramp_tiles=ramp, eps_seq=EPS_SEQ)
    assert _same(a, c) and ba.windows == bc.windows
    assert bc.w0 >= ba.w0 and np.all(bc.w >= ba.w) and np.all(bc.v >= ba.v) and np.any(bc.v > ba.v)
    # a second epoch carries the budget on alike
    a2, ba2 = rowlane_epoch_model(a, d, hp, TR=32, grid=4, damp=damp, ramp_tiles=0, budget=ba)
    c2, bc2 = rowlane_epoch_model(c, d, hp, TR=32, grid=4, damp=damp, ramp_tiles=0, budget=bc, eps_seq=EPS_SEQ)
    assert _same(a2, c2)
    assert bc2.w0 >= ba2.w0 and np.all(bc2.w >= ba2.w) and np.all(bc2.v >= ba2.v)


def test_one_row_by_hand():
    """One row naming features 0 (x = 1) and 1 (x = 2), k = 1, v = (0.5, 0.25), no bias or linear terms, no
    damping.  s = 0.5 + 0.5 = 1, sq = 0.25 + 0.25 = 0.5, p = 0.5 (s^2 - sq) = 0.25, mult = p - y = -0.75.
    L = eps (2 entries * 1 factor per lane + SEQ_EXTRA); the score's extra error L (s_abs^2 + sq) = 1.5 L
    enters each step through lr |grad|, and s_f's, L s_abs = L, through lr |mult x|."""
    d = Data(np.array([0, 2], np.uint64), np.array([0, 1], np.uint32), np.array([1.0, 2.0], np.float32),
             np.array([1.0], np.float32), 2)
    hp = HParams(0, 0.1, min_target=0.0, max_target=5.0, k0=False, k1=False)
    st = State(0.0, np.zeros(2), np.array([[0.5, 0.25]]))
    _, b0 = rowlane_epoch_model(st, d, hp, TR=1, grid=1, damp=False, ramp_tiles=0)
    _, b1 = rowlane_epoch_model(st, d, hp, TR=1, grid=1, damp=False, ramp_tiles=0, eps_seq=EPS_SEQ)
    L = EPS_SEQ * (2 + SEQ_EXTRA)
    lr, mult = 0.1, 0.75
    grad = np.array([1.0 * 1 - 0.5 * 1, 1.0 * 2 - 0.25 * 4])  # s x - v x^2
    x = np.array([1.0, 2.0])
    want = lr * grad * 1.5 * L + lr * mult * x * L
    assert np.allclose(b1.v[0] - b0.v[0], want, rtol=1e-9, atol=0)
    assert b1.w0 == b0.w0 and np.array_equal(b1.w, b0.w)


def test_wide_rows_count_each_lanes_factors():
    """k = 64: each lane sums two factors per entry, so L doubles its per-entry part."""
    d = Data(np.array([0, 3], np.uint64), np.array([0, 1, 2], np.uint32), np.ones(3, np.float32),
             np.array([1.0], np.float32), 3)
    hp = HParams(0, 0.1, min_target=0.0, max_target=5.0, k0=False, k1=False)
    r = np.random.default_rng(2)
    extra = {}
    for k in (32, 64):
        st = State(0.0, np.zeros(3), r.uniform(0.1, 0.2, (k, 3)).round(6))
        _, b0 = rowlane_epoch_model(st, d, hp, TR=1, grid=1, damp=False, ramp_tiles=0)
        _, b1 = rowlane_epoch_model(st, d, hp, TR=1, grid=1, damp=False, ramp_tiles=0, eps_seq=1.0)
        # the per-factor-sum term of factor 0, entry 0: lr |mult x| L s_abs_0, with L = 3 * lanes + SEQ_EXTRA
        extra[k] = (b1.v[0, 0] - b0.v[0, 0])
    assert extra[32] > 0 and extra[64] > extra[32]
