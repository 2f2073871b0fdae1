"""CPU: the fp64 model of the windowed SGDA epoch (oracle/sgda_window_model.py) is itself right.

tests/test_sgda_hogwild_gpu.py holds the HOGWILD SGDA kernel to this model, so the model is tied down first: to
the reference's SGDA (oracle/fm_oracle_sgda.c) where the two must agree -- windows of one row, no damping, no
quantisation, fp64 state --, to update_means at the window the moments rule names, to a two-window case worked
out by hand, and, at the default window, to the reference's test RMSE on planted C2-shaped data.  The budget's
term for the kernel's serial sums (eps_seq) is checked too: left out, the model computes what it computed before
the term existed, bit for bit; put in, it widens the budget and nothing else, by what a case worked out by hand
gives.
"""
import json
import os
from importlib import util

import numpy as np
import pytest

from libfm_b200 import Data, synth
from oracle import HParams, Port, State
from oracle import sgda_window_model as sm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _script(name):
    spec = util.spec_from_file_location(name, os.path.join(ROOT, "scripts", name + ".py"))
    mod = util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _init(n, k, seed, stdev=0.1):
    r = np.random.default_rng(seed)
    v = np.asarray(stdev * r.standard_normal((k, n)), dtype=np.float32).astype(np.float64)
    return State(0.0, np.zeros(n), v)


def _cls(d):
    return Data(d.row_ptr, d.col, d.val, np.where(d.target > 3, 1.0, -1.0).astype(np.float32), d.num_feature)


def _compare_w1(train, val, k, G, task, epochs=3, k0=True, k1=True, lr=0.01, stdev=0.1):
    n = train.num_feature
    group = np.arange(n) % G
    st = _init(n, k, 3, stdev)
    hp = HParams(task, lr, min_target=1.0, max_target=5.0, k0=k0, k1=k1)
    o = Port(n, k, k0, k1)
    o.set_params(st.w0, st.w, st.v)
    o.sgda_begin(group)
    sg = sm.Sgda.begin(n, k, group)
    for e in range(epochs):
        o.sgda_epoch(train, val, task, lr, 1.0, 5.0, e > 0)
        st, sg, _, _, _ = sm.sgda_window_epoch(st, sg, train, val, hp, 1, e > 0, damp=False, quant=False,
                                               fp32=False)
        for got, want in [(st.w0, o.w0.value), (st.w, o.w), (st.v, o.v), (sg.grad_w, o.grad_w),
                          (sg.grad_v, o.grad_v), (sg.reg_w, o.reg_w), (sg.reg_v, o.reg_v)]:
            np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    assert np.isfinite(st.v).all() and np.isfinite(sg.reg_v).all()
    assert e == 0 or np.any(sg.reg_v > 0)  # the lambda-steps moved reg


@pytest.mark.parametrize("task", [0, 1])
@pytest.mark.parametrize("G", [1, 3])
@pytest.mark.parametrize("n_val", [70, 400])  # V < N: the cursor wraps; V > N: it never does
def test_windows_of_one_row_are_the_reference(task, G, n_val):
    d = synth.two_field(200 + n_val, 40, 30, seed=11)
    train, val = synth.split_rows(d, 200)
    if task:
        train, val = _cls(train), _cls(val)
    _compare_w1(train, val, 4, G, task)


@pytest.mark.parametrize("k0,k1", [(True, False), (False, True)])
def test_windows_of_one_row_model_switches(k0, k1):
    train, val = synth.split_rows(synth.two_field(300, 30, 20, seed=4), 250)
    _compare_w1(train, val, 3, 2, 0, k0=k0, k1=k1)


def test_windows_of_one_row_ragged_rows():
    """Repeated ids in a row, x != 1, empty rows, and zero gradients (x = 0 entries): the stamp stores them."""
    d = synth.ragged(400, 50, 6, seed=8)
    d.val[::7] = 0.0
    train, val = synth.split_rows(d, 300)
    _compare_w1(train, val, 5, 3, 0)
    _compare_w1(_cls(train), _cls(val), 5, 3, 1)


@pytest.mark.parametrize("k", [33, 100])
def test_windows_of_one_row_long_rows_wide_k(k):
    """Rows of 0-60 entries that name a feature two and three times, x in [0.5, 1.5], at k = 33 (a lane's second
    factor) and k = 100, three groups, both tasks."""
    d = synth.long_rows(300, 120, 60, seed=k)
    train, val = synth.split_rows(d, 220)
    _compare_w1(train, val, k, 3, 0, lr=0.002, stdev=0.02)
    _compare_w1(_cls(train), _cls(val), k, 3, 1, epochs=2, lr=0.002, stdev=0.02)


# ---- the budget's term for the lanes' serial sums (eps_seq) ----

def test_default_eps_seq_is_the_recorded_model():
    """eps_seq = 0, and leaving it out, compute what the model computed before the term existed, bit for bit:
    state, stored gradients, reg, moments and both budgets (scripts/make_sgda_model_digests.py)."""
    mk = _script("make_sgda_model_digests")
    with open(os.path.join(ROOT, "tests", "golden", "sgda_window_model_digests.json")) as f:
        want = json.load(f)
    assert sorted(want) == sorted(mk.CASES)
    for name in mk.CASES:
        for kw in ({}, dict(eps_seq=0.0)):
            got = mk.model_digests(name, **kw)
            for e, (g, w) in enumerate(zip(got, want[name])):
                bad = sorted(q for q in w if g[q] != w[q])
                assert not bad, "%s %s epoch %d: %s differ" % (name, kw, e, bad)


def test_eps_seq_widens_the_budget_only():
    """eps_seq > 0 leaves the state, the SGDA state and the moments as they were, and makes no budget element
    smaller; the V budget of every feature a row stepped grows, and grows more at larger k."""
    mk = _script("make_sgda_model_digests")
    for name in mk.CASES:
        train, val, st0, sg0, hp, W, damp = mk.long_case(name)
        runs = {}
        for eps in (0.0, sm.EPS_SEQ):
            st, sg, bud, rb = st0, sg0, None, None
            for e in range(2):
                st, sg, mom, bud, rb = sm.sgda_window_epoch(st, sg, train, val, hp, W, e > 0, damp=damp,
                                                            budget=bud, reg_budget=rb, eps_seq=eps)
            runs[eps] = (st, sg, mom, bud, rb)
        (st, sg, mom, bud, rb), (st1, sg1, mom1, bud1, rb1) = runs[0.0], runs[sm.EPS_SEQ]
        same = [(st.w0, st1.w0), (st.w, st1.w), (st.v, st1.v), (sg.grad_w, sg1.grad_w), (sg.grad_v, sg1.grad_v),
                (sg.reg_w, sg1.reg_w), (sg.reg_v, sg1.reg_v), (mom[0], mom1[0]), (mom[1], mom1[1])]
        for a, b in same:
            assert np.array_equal(np.float64(a).view(np.uint64), np.float64(b).view(np.uint64)), name
        for a, b in [(bud.w0, bud1.w0), (bud.w, bud1.w), (bud.v, bud1.v), (rb.reg_w, rb1.reg_w),
                     (rb.reg_v, rb1.reg_v), (rb.var_w, rb1.var_w), (rb.var_v, rb1.var_v)]:
            assert np.all(np.asarray(b) >= np.asarray(a)), name
        stepped = np.bincount(train.col.astype(np.int64), minlength=train.num_feature) > 0
        assert np.all(bud1.v[:, stepped] > bud.v[:, stepped]) and np.all(rb1.var_v > rb.var_v), name
        assert bud1.w0 > bud.w0 and np.all(bud1.w[stepped] >= bud.w[stepped]), name


def test_eps_seq_term_by_hand():
    """One row of three entries (the first feature named twice), k = 40, one window, no damping: the V budget of
    each entry grows by lr |mult x| L sum_i |v_f,i x_i| plus what the wider score error moves, with
    L = eps_seq (3 ceil(40 / 32) + SEQ_EXTRA) = eps_seq 12."""
    n, k, lr = 3, 40, 0.01
    train = Data(np.array([0, 3]), np.array([0, 1, 0]), np.array([1.0, 0.5, 1.5]), np.array([4.0]), n)
    val = Data(np.array([0, 1]), np.array([2]), np.array([1.0]), np.array([3.0]), n)
    st = _init(n, k, 9)
    hp = HParams(0, lr, min_target=1.0, max_target=5.0, k0=False)
    eps = 1e-3
    runs = [sm.sgda_window_epoch(st, sm.Sgda.begin(n, k), train, val, hp, 1, False, damp=False, eps_seq=e)
            for e in (0.0, eps)]
    (_, _, _, b0, _), (_, _, _, b1, _) = runs
    x = train.val.astype(np.float64)
    ids = train.col.astype(np.int64)
    vx = st.v[:, ids] * x
    abs_s = np.abs(vx).sum(1)
    s = vx.sum(1)
    L = eps * 12
    term_score = 2 * L * (np.abs(st.w[ids] * x).sum() + (abs_s ** 2).sum() + (vx ** 2).sum())
    p = st.w[ids] @ x + 0.5 * ((s ** 2).sum() - (vx ** 2).sum())
    mult = 2 * (np.clip(p, 1.0, 5.0) - 4.0)
    want = np.zeros((k, n))
    for i, (f, xi) in enumerate(zip(ids, x)):
        want[:, f] += lr * np.abs(s - st.v[:, f] * xi) * abs(xi) * term_score + lr * abs(mult * xi) * L * abs_s
    # the second step of feature 0 starts where the first ended: its gradient reads v + step, not v, which moves
    # the by-hand |s - v x| by far less than the 1e-6 relative tolerance
    np.testing.assert_allclose(b1.v - b0.v, want, rtol=1e-6, atol=0)


def test_zero_gradient_is_stored():
    """A feature whose only entry of the window has x = 0 gets its stored gradient replaced by 0."""
    n, k = 4, 2
    train = Data(np.array([0, 1, 2]), np.array([0, 1]), np.array([1.0, 0.0]), np.array([3.0, 3.0]), n)
    val = Data(np.array([0, 1]), np.array([2]), np.array([1.0]), np.array([3.0]), n)
    st = _init(n, k, 1)
    sg = sm.Sgda.begin(n, k)
    sg.grad_w[:] = 5.0
    sg.grad_v[:] = 5.0
    hp = HParams(0, 0.01, min_target=1.0, max_target=5.0)
    _, out, _, _, _ = sm.sgda_window_epoch(st, sg, train, val, hp, 2, False)
    assert out.grad_w[1] == 0.0 and np.all(out.grad_v[:, 1] == 0.0)
    assert out.grad_w[0] != 5.0 and out.grad_w[2] == 5.0 and out.grad_w[3] == 5.0


@pytest.mark.parametrize("N,V,W", [(50, 20, 1), (50, 20, 7), (50, 80, 8), (40, 20, 16), (30, 10, 30)])
def test_moments_at_the_named_window(N, V, W):
    """The moments are update_means of the state after the fold of the window holding step t*, the epoch's last
    cursor restart, or of the epoch's start state when the cursor does not restart."""
    train, val = synth.split_rows(synth.two_field(N + V, 20, 10, seed=2), N)
    n = train.num_feature
    hp = HParams(0, 0.02, min_target=1.0, max_target=5.0)
    st0 = _init(n, 3, 5)
    st0.w[:] = np.float32(0.01) * np.arange(n)
    trace = []
    _, _, mom, _, _ = sm.sgda_window_epoch(st0, sm.Sgda.begin(n, 3), train, val, hp, W, True, trace=trace)
    assert len(trace) == (N + W - 1) // W
    t_star = (N - 1) // V * V if N > V else 0
    ref = trace[t_star // W] if t_star else st0

    def update_means(x):
        mean, var = 0.0, 0.0
        for xi in x:
            mean += xi
            var += xi * xi
        mean /= len(x)
        return var / len(x) - mean * mean
    np.testing.assert_allclose(mom[0], update_means(ref.w), rtol=1e-12, atol=1e-18)
    for f in range(3):
        np.testing.assert_allclose(mom[1][f], update_means(ref.v[f]), rtol=1e-12, atol=1e-18)


def test_two_windows_by_hand():
    """One feature, one factor-free model (k = 0, w only), W = 2, two windows, two lambda-rows each: the four
    lambda contributions of a window are summed and clamped once, from the reg the window's theta-steps read."""
    n, lr = 1, 0.1
    train = Data(np.arange(5), np.zeros(4), np.ones(4), np.array([1.0, 1.0, 1.0, 1.0]), n)
    val = Data(np.arange(3), np.zeros(2), np.array([1.0, 2.0]), np.array([3.0, 0.5]), n)
    hp = HParams(0, lr, min_target=-10.0, max_target=10.0, k0=False, k1=True)
    st = State(0.0, np.array([0.5]), np.zeros((0, n)))
    sg = sm.Sgda.begin(n, 0)
    sg.reg_w[:] = 0.25
    out, sgo, _, _, _ = sm.sgda_window_epoch(st, sg, train, val, hp, 2, True, damp=False, quant=False, fp32=False)
    w, reg = 0.5, 0.25
    for _ in range(2):  # windows
        # theta: both rows read w; grad = 2 (w - 1) x, step = -lr (grad + 2 reg w); the window adds both
        grad = 2 * (w - 1.0)
        w1 = w + 2 * (-lr * (grad + 2 * reg * w))
        # lambda: rows 0 and 1 of val (x = 1, 2), each from w1, the stored gradient (both rows' sum) and reg
        total = 0.0
        for x, y in [(1.0, 3.0), (2.0, 0.5)]:
            wd = w1 - lr * (2 * grad + 2 * reg * w1)
            gl = 2 * (wd * x - y)
            total += -lr * gl * (-2 * lr * x * w1)
        reg = max(0.0, reg + total)
        wprev, w = w, w1
    assert out.w[0] == pytest.approx(w, abs=1e-15)
    assert sgo.grad_w[0] == pytest.approx(2 * 2 * (wprev - 1.0), abs=1e-15)  # both rows' gradients, summed
    assert sgo.reg_w[0] == pytest.approx(reg, abs=1e-15)


def test_the_window_clamp_is_once_per_window():
    """Two lambda contributions of opposite sign, the negative one first: clamped once per window their sum
    counts; clamped per step the first would stop at 0 and the second alone would remain."""
    n, lr = 1, 0.1
    train = Data(np.arange(3), np.zeros(2), np.ones(2), np.array([0.0, 0.0]), n)
    val = Data(np.arange(3), np.zeros(2), np.array([-1.0, 1.0]), np.array([-5.0, -5.0]), n)
    hp = HParams(0, lr, min_target=-10.0, max_target=10.0, k0=False, k1=True)
    st = State(0.0, np.array([1.0]), np.zeros((0, n)))
    out, sgo, _, _, _ = sm.sgda_window_epoch(st, sm.Sgda.begin(n, 0), train, val, hp, 2, True, damp=False,
                                             quant=False, fp32=False)
    w1 = out.w[0]
    grad = 2 * 2 * (1.0 - 0.0)  # both theta rows read w = 1 against y = 0
    c = []
    for x, y in [(-1.0, -5.0), (1.0, -5.0)]:
        wd = w1 - lr * grad
        gl = 2 * (wd * x - y)
        c.append(-lr * gl * (-2 * lr * x * w1))
    assert c[0] < 0 < c[0] + c[1] < c[1]
    assert sgo.reg_w[0] == pytest.approx(c[0] + c[1], abs=1e-15)


def test_default_window_tracks_the_reference_on_c2():
    """Planted C2-shaped data (held-out rows split into validation and test), the default W with damping and
    quantisation, against the reference's SGDA from the same model: the test RMSE stays within 0.01 of the
    reference's at every epoch after the first.  scripts/sgda_window_study.py measured gaps of at most 0.0004
    at W = 1024 and 4096 over ten epochs, and 0.011 at W = 16384 (DESIGN.md section 3.5)."""
    from importlib import util
    import os
    spec = util.spec_from_file_location("study", os.path.join(os.path.dirname(__file__), "..", "scripts",
                                                              "sgda_window_study.py"))
    study = util.module_from_spec(spec)
    spec.loader.exec_module(study)
    train, held = synth.movielens_1m_planted()
    val, test = synth.split_rows(held, held.num_cases // 2)
    n, k = train.num_feature, 8
    group = (np.arange(n) >= 6040).astype(np.uint32)
    v0 = _init(n, k, 1).v
    hp = HParams(0, 0.01, min_target=1.0, max_target=5.0)
    o = Port(n, k)
    o.set_params(0.0, np.zeros(n), v0)
    o.sgda_begin(group)
    st, sg = State(0.0, np.zeros(n), v0.copy()), sm.Sgda.begin(n, k, group)
    for e in range(3):
        o.sgda_epoch(train, val, 0, 0.01, 1.0, 5.0, e > 0)
        st, sg, _, _, _ = sm.sgda_window_epoch(st, sg, train, val, hp, sm.DEFAULT_W, e > 0)
        gap = study.rmse(st, test) - study.rmse(State(o.w0.value, o.w, o.v), test)
        if e > 0:
            assert abs(gap) < 0.01, "epoch %d: test RMSE gap %.4f" % (e, gap)
