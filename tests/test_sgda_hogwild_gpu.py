"""GPU: SGDA in HOGWILD mode (fm_sgda_hogwild.cu) computes what the fp64 window model computes.

oracle/sgda_window_model.py states the windowed epoch without warps or grid: every row of a window reads one
state and one reg, its steps are damped, rounded to 2^-32, summed and folded, then the window's lambda-steps move
reg once.  After every epoch each of w0, w and V must lie within the model's per-element budget, and reg_w, reg_v
and the moments within the model's bound for them.  The epoch must also compute the same bits on every run and
at every grid size, turn a diverging run into NaN, and refuse what it does not support by naming the limit.
"""

import numpy as np
import pytest

from libfm_b200 import Data, FmError, FmLearnSgdElement, FmModel, MODE_HOGWILD, synth
from oracle import HParams, State
from oracle import sgda_window_model as sm

pytestmark = pytest.mark.gpu

def _cls(d):
    return Data(d.row_ptr, d.col, d.val, np.where(d.target > 3, 1.0, -1.0).astype(np.float32), d.num_feature)

def _learner(n, k, task, lr, tuning, k0=True, k1=True, stdev=0.1):
    fm = FmModel(n, k, k0, k1)
    fm.init_stdev = stdev
    fm.init_numpy(42)
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate = task, lr
    l.min_target, l.max_target = 1.0, 5.0
    l.push_hparams()
    l.set_tuning(**tuning)
    return l

def _pull(l):
    l.pull_params()
    return State(float(l.fm.w0), l.fm.w.copy(), l.fm.v.copy())

def run_case(name, train, val, k=8, task=0, G=1, W=None, damp=1, epochs=3, lr=0.01, k0=True, k1=True, stdev=0.1,
             eps_seq=0.0, ctas_per_sm=0):
    """Hold `epochs` epochs to the model; eps_seq goes to its budget (sm.EPS_SEQ for long rows and wide k).
    Returns the worst (theta / budget, reg / bound, moments / bound) over the epochs."""
    n = train.num_feature
    group = np.arange(n) % G
    tuning = dict(rows_per_tile=W or 0, damp=damp, ctas_per_sm=ctas_per_sm)
    l = _learner(n, k, task, lr, tuning, k0, k1, stdev)
    hp = HParams(task, lr, min_target=1.0, max_target=5.0, k0=k0, k1=k1)
    worst = np.zeros(3)
    try:
        l.upload(train, 0)
        l.upload(val, 1)
        l.sgda_begin(group if G > 1 else None)
        want = _pull(l)
        assert np.all(want.w == 0)
        sg, bud, rb = sm.Sgda.begin(n, k, group), None, None
        for e in range(epochs):
            l.sgda_epoch(train, val, e > 0)
            want, sg, mom, bud, rb = sm.sgda_window_epoch(want, sg, train, val, hp, W or sm.DEFAULT_W, e > 0,
                                                          damp=damp >= 0, budget=bud, reg_budget=rb,
                                                          eps_seq=eps_seq)
            got = _pull(l)
            b0, bw, bv = bud.bound(want)
            ratio = max(abs(got.w0 - want.w0) / b0, np.max(np.abs(got.w - want.w) / bw),
                        np.max(np.abs(got.v - want.v) / bv, initial=0.0))
            reg_w, reg_v = l.sgda_reg()
            tiny = 1e-300
            rr = max(np.max(np.abs(reg_w - sg.reg_w) / (rb.reg_w + tiny)),
                     np.max(np.abs(reg_v - sg.reg_v) / (rb.reg_v + tiny)) if k else 0.0)
            var_w, var_v = l.sgda_moments()
            mr = max(abs(var_w - mom[0]) / rb.var_w, np.max(np.abs(var_v - mom[1]) / rb.var_v) if k else 0.0)
            print("sgda-hogwild %-18s epoch %d  theta/budget %.3f  reg/bound %.3f  moments/bound %.3f  reg_v[0,0] "
                  "%.4g" % (name, e, ratio, rr, mr, reg_v[0, 0] if k else reg_w[0]))
            assert ratio < 1.0, "epoch %d: a parameter is %.2f budgets away from the model" % (e, ratio)
            assert rr < 1.0, "epoch %d: reg is %.2f bounds away from the model" % (e, rr)
            assert mr < 1.0, "epoch %d: the moments are %.2f bounds away from the model" % (e, mr)
            if e > 0 and lr > 0:
                assert np.any(reg_v > 0) or np.any(reg_w > 0), "the lambda-steps did not move reg"
            worst = np.maximum(worst, [ratio, rr, mr])
    finally:
        l.close()
    return worst

def _two_field(n_train, n_val, seed=3):
    return synth.split_rows(synth.two_field(n_train + n_val, 300, 200, seed=seed), n_train)

@pytest.mark.parametrize("k", [1, 5, 8, 32, 128])
def test_factor_widths(k, built_lib):
    train, val = _two_field(6000, 1500)
    run_case("k%d" % k, train, val, k=k, W=512)

@pytest.mark.parametrize("task", [0, 1])
@pytest.mark.parametrize("G", [1, 3])
def test_tasks_and_groups(task, G, built_lib):
    train, val = _two_field(6000, 1500)
    if task:
        train, val = _cls(train), _cls(val)
    run_case("task%d_G%d" % (task, G), train, val, task=task, G=G, W=512, lr=0.05 if task else 0.01)

def test_damping_hot_features(built_lib):
    d = synth.two_field(8000, 50, 40, seed=5, zipf=1.2)  # concurrencies in the hundreds: gamma far below 1
    train, val = synth.split_rows(d, 6000)
    run_case("damp_hot", train, val, W=1000, damp=1)

def test_damping_off(built_lib):
    """Plain summed steps (fmb200_set_tuning damp = -1), on features no window steps often enough to diverge."""
    train, val = _two_field(6000, 1500)
    run_case("damp_off", train, val, W=1000, damp=-1)

@pytest.mark.parametrize("W", [1, 37, 6000])  # one row; a window that does not divide N; one window
def test_window_sizes(W, built_lib):
    train, val = _two_field(3000, 400)  # V < N: the cursor wraps, and inside a window when W > V
    run_case("W%d" % W, train, val, W=W, G=2)

def test_multi_field_rows(built_lib):
    d = synth.multi_field(5000, 39, 20_000, seed=4)
    d.target = (1.0 + 4.0 * d.target).astype(np.float32)  # ratings 1 and 5
    train, val = synth.split_rows(d, 4000)
    run_case("multi_field39", train, val, k=8, G=3, W=256)

def test_ragged_rows_with_repeats(built_lib):
    """Empty rows, x != 1, a feature named twice in a row."""
    d = synth.ragged(5000, 300, 6, seed=8)
    train, val = synth.split_rows(d, 4000)
    run_case("ragged", train, val, k=5, G=3, W=300)

def test_model_switches(built_lib):
    train, val = _two_field(4000, 900)
    run_case("no_bias", train, val, W=256, k0=False)
    run_case("no_linear", train, val, W=256, k1=False)

def test_c2_full_size_default_window(built_lib):
    train, held = synth.movielens_1m_planted()
    val = held.rows(0, held.num_cases)
    run_case("c2", train, val, G=2, epochs=3)

# ---- reproducibility ----

def _bits(train, val, tuning, epochs=2):
    n = train.num_feature
    l = _learner(n, 8, 0, 0.01, tuning)
    try:
        l.upload(train, 0)
        l.upload(val, 1)
        l.sgda_begin(np.arange(n) % 2)
        for e in range(epochs):
            l.sgda_epoch(train, val, e > 0)
        st = _pull(l)
        reg = l.sgda_reg()
        mom = l.sgda_moments()
        cfg = l.epoch_config()
    finally:
        l.close()
    return [np.float64(st.w0), st.w, st.v, reg[0], reg[1], np.float64(mom[0]), mom[1]], cfg["grid"]

def test_same_bits_every_run_and_grid(built_lib):
    train, val = _two_field(30_000, 5000)
    a, ga = _bits(train, val, dict(rows_per_tile=2048))
    b, _ = _bits(train, val, dict(rows_per_tile=2048))
    c, gc = _bits(train, val, dict(rows_per_tile=2048, ctas_per_sm=1))
    assert gc < ga, "the two grids must differ"
    for x, y, z in zip(a, b, c):
        assert np.array_equal(x.view(np.uint64), y.view(np.uint64))
        assert np.array_equal(x.view(np.uint64), z.view(np.uint64))

def test_divergence_turns_the_state_nan(built_lib):
    train, val = _two_field(3000, 500)
    l = _learner(train.num_feature, 8, 0, 50.0, dict(rows_per_tile=256))
    try:
        l.upload(train, 0)
        l.upload(val, 1)
        l.sgda_begin()
        for e in range(3):
            l.sgda_epoch(train, val, e > 0)
        st = _pull(l)
        assert np.all(np.isnan(st.v)) and np.all(np.isnan(st.w)) and np.isnan(st.w0)
    finally:
        l.close()

# ---- refusals ----

def test_refuses_wide_factors(built_lib):
    train, val = _two_field(500, 100)
    l = _learner(train.num_feature, 129, 0, 0.01, {})
    try:
        with pytest.raises(FmError, match="num_factor <= 128"):
            l.sgda_begin()
    finally:
        l.close()

def test_refuses_too_many_groups(built_lib):
    train, _ = _two_field(500, 100)
    l = _learner(train.num_feature, 128, 0, 0.01, {})
    try:
        with pytest.raises(FmError, match="at most 8192"):
            l.sgda_begin(np.arange(train.num_feature) % 64)
    finally:
        l.close()

def test_refuses_streamed_sets(built_lib, tmp_path):
    from libfm_b200.model import XtBlocks, write_binary
    train, val = _two_field(500, 100)
    write_binary(train, str(tmp_path / "t.x"), str(tmp_path / "t.y"))
    l = _learner(train.num_feature, 8, 0, 0.01, {})
    try:
        l.upload(val, 1)
        l.sgda_begin()
        blocks = XtBlocks(str(tmp_path / "t.x"), train.target, 4096, slots=(2, 4), transposed=False)
        with pytest.raises(FmError, match="resident data sets"):
            l.sgda_epoch_x(blocks, val, False)
    finally:
        l.close()
