"""GPU: the wavefront SGDA epoch (fm_sgda_wavefront_kernel) against the one-warp kernel
(fm_sgda_epoch_kernel, fmb200_set_tuning variant 1), bit for bit: w0, w, V, reg_w, reg_v and the epoch's
update_means variances.  The one-warp kernel is pinned to the reference through the oracle restatement
(tests/test_sgda_gpu.py, tests/test_wide_k_gpu.py); the variances are also checked against a Python statement
of update_means on the oracle's state at the step where the reference takes them."""
import numpy as np
import pytest

from conftest import make_learner
from libfm_b200 import MODE_INORDER, Data, synth
from oracle import Port

pytestmark = pytest.mark.gpu

WAVEFRONT_SLOTS, ONE_WARP_SLOTS = 4, 1  # epoch_config()["slots"] of the two schedules


def _binarise(d):
    d.target[:] = np.where(d.target > 3, 1.0, -1.0)


def _groups(n, groups):
    return (np.arange(n) * groups // n).astype(np.uint32)


def _run(tr, va, k, groups, task, variant, epochs=3, k0=1, k1=1, lr=0.02, seed=2):
    n = max(tr.num_feature, va.num_feature)
    mn, mx = float(tr.target.min()), float(tr.target.max())
    init = (0.0, np.zeros(n), np.random.default_rng(seed).standard_normal((k, n)) * 0.1)
    cfg = dict(n=n, k=k, k0=k0, k1=k1, task=task, lr=lr, regs=np.zeros(3), min_target=mn, max_target=mx)
    l = make_learner(cfg, init, mode=MODE_INORDER)
    l.set_tuning(variant=variant)
    l.sgda_begin(_groups(n, groups) if groups > 1 else None)
    moments = []
    for e in range(epochs):
        l.sgda_epoch(tr, va, e > 0)
        moments.append(l.sgda_moments())
    cfg_run = l.epoch_config()
    l.pull_params()
    reg_w, reg_v = l.sgda_reg()
    out = dict(w0=l.fm.w0, w=l.fm.w.copy(), v=l.fm.v.copy(), reg_w=reg_w, reg_v=reg_v, moments=moments,
               slots=cfg_run["slots"], init=init, cfg=cfg)
    l.close()
    return out


def _assert_same(a, b):
    assert a["slots"] == WAVEFRONT_SLOTS and b["slots"] == ONE_WARP_SLOTS
    assert np.float64(a["w0"]).tobytes() == np.float64(b["w0"]).tobytes()
    assert a["w"].tobytes() == b["w"].tobytes()
    assert a["v"].tobytes() == b["v"].tobytes()
    assert a["reg_w"].tobytes() == b["reg_w"].tobytes()
    assert a["reg_v"].tobytes() == b["reg_v"].tobytes()
    for (aw, av), (bw, bv) in zip(a["moments"], b["moments"]):
        assert np.float64(aw).tobytes() == np.float64(bw).tobytes() and av.tobytes() == bv.tobytes()


def _compare(tr, va, k, groups, task, **kw):
    a = _run(tr, va, k, groups, task, 0, **kw)
    b = _run(tr, va, k, groups, task, 1, **kw)
    _assert_same(a, b)
    assert a["reg_v"].max() > 0
    return a


def _case(name):
    if name == "dense_conflicts":  # few features: most windows are short
        full = synth.two_field(3000, 12, 9, seed=21, planted_k=2)
        return synth.split_rows(full, 2000)
    if name == "val_is_train":  # s_t = r_t: every pair meets its own train row (split windows)
        tr = synth.two_field(1500, 300, 200, seed=22, planted_k=2)
        return tr, tr.rows(0, tr.num_cases)
    if name == "val_is_next_train":  # s_t = r_{t+1}: lambda rows share features with later train rows
        full = synth.two_field(1501, 300, 200, seed=23, planted_k=2)
        return full.rows(0, 1500), full.rows(1, 1501)
    if name == "wrap_in_window":  # 7 validation rows: the cursor restarts several times per window
        full = synth.two_field(2007, 400, 300, seed=24, planted_k=2)
        return full.rows(0, 2000), full.rows(2000, 2007)
    if name == "ragged":  # repeated ids in a row, empty rows, x != 1
        tr = synth.ragged(2000, 500, 4, seed=25)
        va = synth.ragged(700, 500, 4, seed=26)
        return tr, va
    if name == "val_longer":  # V > N: no restart, the moments at the epoch's start
        full = synth.two_field(3000, 300, 200, seed=27, planted_k=2)
        return synth.split_rows(full, 1000)
    raise KeyError(name)


CASES = ["dense_conflicts", "val_is_train", "val_is_next_train", "wrap_in_window", "ragged", "val_longer"]


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("k", [1, 5, 8])
def test_wavefront_matches_one_warp(name, k, built_lib):
    tr, va = _case(name)
    _compare(tr, va, k, 3, 0)


@pytest.mark.parametrize("name", ["dense_conflicts", "val_is_train", "wrap_in_window", "ragged"])
@pytest.mark.parametrize("groups", [1, 3])
def test_wavefront_matches_one_warp_classification(name, groups, built_lib):
    tr, va = _case(name)
    for d in (tr, va):
        _binarise(d)
    _compare(tr, va, 5, groups, 1)


@pytest.mark.parametrize("k0,k1", [(0, 0), (1, 0), (0, 1)])
def test_wavefront_without_bias_or_linear(k0, k1, built_lib):
    tr, va = _case("wrap_in_window")
    _compare(tr, va, 5, 3, 0, k0=k0, k1=k1)


def _update_means(w, v):
    """fm_learn_sgd_element_adapt_reg.h:250-274 in Python floats (IEEE binary64, the same serial sums)."""
    n = len(w)

    def var(xs):
        m = s = 0.0
        for x in xs.tolist():
            m += x
            s += x * x
        m /= n
        return s / n - m * m

    return var(w), np.array([var(v[f]) for f in range(v.shape[0])])


def _last_moments_step(n_train, n_val, lambda_steps):
    """:298-310: update_means at the epoch's start and before every lambda-step that finds the cursor at
    the end of the validation rows; the last such step, or 0 for the call at the start."""
    last = 0
    if lambda_steps:
        cursor = 0
        for t in range(n_train):
            if cursor == n_val:
                last, cursor = t, 0
            cursor += 1
    return last


@pytest.mark.parametrize("name", ["wrap_in_window", "val_longer", "ragged"])
def test_moments_match_update_means_on_the_oracle_state(name, built_lib):
    tr, va = _case(name)
    k, groups, epochs = 5, 3, 3
    a = _run(tr, va, k, groups, 0, 0, epochs=epochs)
    n = a["cfg"]["n"]
    mn, mx = a["cfg"]["min_target"], a["cfg"]["max_target"]
    for e in range(epochs):
        t_star = _last_moments_step(tr.num_cases, va.num_cases, e > 0)
        p = Port(n, k, 1, 1)
        p.set_params(*a["init"])
        p.sgda_begin(_groups(n, groups))
        for e2 in range(e):
            p.sgda_epoch(tr, va, 0, 0.02, mn, mx, e2 > 0)
        if t_star:  # theta-steps 0..t*: the lambda-step t* that follows moves only reg_w / reg_v
            p.sgda_epoch(tr.rows(0, t_star + 1), va, 0, 0.02, mn, mx, e > 0)
        var_w, var_v = _update_means(np.array(p.w), np.array(p.v))
        gw, gv = a["moments"][e]
        assert np.float64(gw).tobytes() == np.float64(var_w).tobytes(), (e, gw, var_w)
        assert gv.tobytes() == var_v.tobytes(), (e, gv, var_v)


def test_dispatch(built_lib):
    tr, va = _case("wrap_in_window")
    assert _run(tr, va, 8, 1, 0, 0, epochs=2)["slots"] == WAVEFRONT_SLOTS
    assert _run(tr, va, 9, 1, 0, 0, epochs=2)["slots"] == ONE_WARP_SLOTS  # k > 8
    r = np.random.default_rng(28)  # 50 validation rows of 5 entries
    long_va = Data(np.arange(51, dtype=np.uint64) * 5, r.integers(0, 500, 250).astype(np.uint32),
                   np.ones(250, dtype=np.float32), r.integers(1, 6, 50).astype(np.float32), 500)
    tr5 = synth.ragged(2000, 500, 4, seed=25)
    assert _run(tr5, long_va, 5, 1, 0, 0, epochs=2)["slots"] == ONE_WARP_SLOTS  # validation rows of 5 entries
    # without lambda-steps the validation rows are not read: their length does not matter
    one = _run(tr5, long_va, 5, 1, 0, 0, epochs=1)
    assert one["slots"] == WAVEFRONT_SLOTS


def test_c2_two_epochs(built_lib):
    full = synth.movielens_1m_shaped(seed=7, planted_k=4, n_rows=1_100_209)
    tr, va = synth.split_rows(full, 1_000_209)
    _compare(tr, va, 8, 2, 0, epochs=2, lr=0.01)
