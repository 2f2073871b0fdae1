"""GPU: HOGWILD SGDA (fm_sgda_hogwild.cu) at every shape fmb200_sgda_begin accepts.

tests/test_sgda_hogwild_gpu.py holds the kernel to oracle/sgda_window_model.py on short rows.  Here the same check
-- after each epoch w0, w and V within the model's budget, reg and the moments within their bounds -- runs on rows
of 0-60 entries that name features two and three times, where a lane scores the row serially and a repeated
feature steps from where its previous entry left it, with the budget's term for those serial sums
(sm.EPS_SEQ).  The cases cover every factor class the launch dispatches (k <= 32, <= 64, <= 128: one, two and four
factors per lane, partly idle lanes included), the model switches, damping, the group ceiling
G (k + 1) <= 8192 and G <= 1024, the windows the moments are taken in, several rows per warp, the same bits at
two grids, a context that starts SGDA again after SGDA or after reproducible SGD epochs, and divergence.
"""
import numpy as np
import pytest

from libfm_b200 import FmError, FmLearnSgdElement, FmModel, MODE_HOGWILD, synth
from oracle import sgda_window_model as sm
from test_sgda_hogwild_gpu import _cls, _learner, _pull, run_case

pytestmark = pytest.mark.gpu

LR, STDEV = 0.002, 0.02  # rows of 30 entries at k = 128: lr * h_row stays well below 1


def _long(n_train, n_val, n_feat=900, seed=1, max_nnz=60, val_nnz=None, zipf=0.0):
    """Training and validation rows of 0 .. max_nnz (validation: val_nnz) entries over the same features."""
    train = synth.long_rows(n_train, n_feat, max_nnz, seed=seed, zipf=zipf)
    val = synth.long_rows(n_val, n_feat, val_nnz or max_nnz, seed=seed + 1000, zipf=zipf)
    return train, val


def _case(name, train, val, k, **kw):
    kw.setdefault("lr", LR)
    kw.setdefault("stdev", STDEV)
    worst = run_case(name, train, val, k=k, eps_seq=sm.EPS_SEQ, **kw)
    print("sgda-hogwild %-18s k %3d  worst theta/budget %.3f  reg/bound %.3g  moments/bound %.3g"
          % (name, k, *worst))
    return worst


# ---- the factor classes: KF = 1 (k <= 32), 2 (k <= 64), 4 (k <= 128) ----

@pytest.mark.parametrize("k", [0, 31, 32, 33, 48, 64, 65, 100, 127, 128])
def test_factor_classes_long_rows(k, built_lib):
    """3001 rows in windows of 256: eleven full windows and a short one; three groups; V < N."""
    train, val = _long(3001, 700, seed=k + 1)
    _case("classes", train, val, k, G=3, W=256)


@pytest.mark.parametrize("k", [64, 100])
def test_switches_at_wide_k(k, built_lib):
    train, val = _long(2500, 600, seed=7)
    _case("no_bias", train, val, k, G=3, W=256, k0=False)
    _case("no_linear", train, val, k, G=3, W=256, k1=False)


@pytest.mark.parametrize("k", [48, 100])
def test_classification_at_wide_k(k, built_lib):
    train, val = _long(2500, 600, seed=8)
    _case("classification", _cls(train), _cls(val), k, task=1, G=3, W=256, lr=0.01)


def test_damping_hot_features_wide_k(built_lib):
    """Zipf(1.1) ids: the hottest features are named in most rows, concurrencies in the hundreds."""
    train, val = _long(3000, 600, n_feat=2000, seed=9, zipf=1.1)
    _case("damp_hot", train, val, 100, G=3, W=256, damp=1)


def test_damping_off_wide_k(built_lib):
    """Plain summed steps (damp = -1) on uniform ids over many features: no window steps a feature often."""
    train, val = _long(3000, 600, n_feat=3000, seed=10, max_nnz=20)
    _case("damp_off", train, val, 64, G=3, W=256, damp=-1)


# ---- the group ceiling: G (k + 1) <= 8192 and G <= 1024 ----

@pytest.mark.parametrize("k,G", [(127, 64), (128, 63), (7, 1024)])
def test_group_ceiling(k, G, built_lib):
    """The largest accepted group count runs two epochs against the model (lambda rows of 8192, 8127 and 8192
    terms); one group more is refused by a message that names 8192 and the largest count."""
    n = max(1200, G + 1)  # sgda_begin counts max(group) + 1 groups: G + 1 of them needs G + 1 features
    train, val = _long(1500, 400, n_feat=n, seed=k, max_nnz=40)
    _case("G%d" % G, train, val, k, G=G, W=256, epochs=2)
    l = _learner(n, k, 0, LR, {})
    try:
        with pytest.raises(FmError, match="at most 8192") as e:
            l.sgda_begin(np.arange(n) % (G + 1))
        assert "use at most %d groups" % G in str(e.value)
    finally:
        l.close()


# ---- the windows the moments are taken in ----

@pytest.mark.parametrize("N,V,W,val_nnz", [
    (3000, 3000, 256, None),  # N <= V: the moments of the epoch's start, with lambda-steps on
    (3000, 500, 250, None),   # t* = 2500 is the first row of window 10
    (3000, 1, 512, None),     # one validation row
    (2000, 5000, 4096, None),  # one window, V > N
    (3000, 600, 256, 60),     # validation rows longer than training rows
])
def test_moments_and_cursor_edges(N, V, W, val_nnz, built_lib):
    max_nnz = 20 if val_nnz else 60
    train, val = _long(N, max(V, 50), seed=N + V + W, max_nnz=max_nnz, val_nnz=val_nnz)
    if V == 1:
        lens = np.diff(val.row_ptr.astype(np.int64))
        i = int(np.flatnonzero(lens > 10)[0])
        val = val.rows(i, i + 1)
    else:
        val = val.rows(0, V)
    assert val.num_cases == V and train.num_cases == N
    _case("N%d_V%d_W%d" % (N, V, W), train, val, 40, G=3, W=W)


# ---- several rows per warp ----

@pytest.mark.parametrize("k", [48, 100])
def test_several_rows_per_warp(k, built_lib):
    """One CTA per SM and one window of all 3000 rows (W = 8192 > N): each warp takes several rows of it."""
    train, val = _long(3000, 600, seed=11)
    _case("rows_per_warp", train, val, k, G=3, W=8192, ctas_per_sm=1)


# ---- the same bits ----

def _bits(train, val, k, tuning, G=3, epochs=2):
    n = train.num_feature
    l = _learner(n, k, 0, LR, tuning, stdev=STDEV)
    try:
        l.upload(train, 0)
        l.upload(val, 1)
        l.sgda_begin(np.arange(n) % G)
        for e in range(epochs):
            l.sgda_epoch(train, val, e > 0)
        return _state(l), l.epoch_config()["grid"]
    finally:
        l.close()


def _state(l):
    st = _pull(l)
    reg_w, reg_v = l.sgda_reg()
    var_w, var_v = l.sgda_moments()
    return [np.float64(st.w0), st.w, st.v, reg_w, reg_v, np.float64(var_w), var_v]


def _assert_same_bits(a, b, what):
    names = ["w0", "w", "v", "reg_w", "reg_v", "var_w", "var_v"]
    for name, x, y in zip(names, a, b):
        assert np.array_equal(np.asarray(x).view(np.uint64), np.asarray(y).view(np.uint64)), (what, name)
    assert np.isfinite(a[2]).all() and np.any(a[4] > 0), what


@pytest.mark.parametrize("k", [48, 100])
def test_same_bits_at_two_grids(k, built_lib):
    train, val = _long(3000, 600, seed=12)
    a, ga = _bits(train, val, k, dict(rows_per_tile=256))
    b, gb = _bits(train, val, k, dict(rows_per_tile=256, ctas_per_sm=1))
    assert gb < ga, "the two grids must differ"
    _assert_same_bits(a, b, "grid %d against %d" % (ga, gb))


# ---- a context starts clean ----

def _fresh(st, k, tuning):
    """A new context holding the parameters st."""
    fm = FmModel(st.w.shape[0], k)
    fm.w0, fm.w, fm.v = st.w0, st.w.copy(), st.v.copy()
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate, l.min_target, l.max_target = 0, LR, 1.0, 5.0
    l.push_hparams()
    l.set_tuning(**tuning)
    return l


def _sgda(l, train, val, group, epochs=2):
    l.upload(train, 0)
    l.upload(val, 1)
    l.sgda_begin(group)
    for e in range(epochs):
        l.sgda_epoch(train, val, e > 0)
    return _state(l)


@pytest.mark.parametrize("k", [48, 100])
def test_sgda_begin_again_starts_clean(k, built_lib):
    """Two SGDA epochs, then sgda_begin with the same groups and with other groups: the next two epochs are what
    a new context given the same parameters computes, bit for bit (stored gradients, accumulators, stamps, reg
    and the divergence flag all start over)."""
    train, val = _long(3000, 600, seed=13)
    n = train.num_feature
    tuning = dict(rows_per_tile=256)
    for name, group in (("same groups", np.arange(n) % 3), ("other groups", np.arange(n) % 5)):
        l = _learner(n, k, 0, LR, tuning, stdev=STDEV)
        try:
            _sgda(l, train, val, np.arange(n) % 3)
            st = _pull(l)
            got = _sgda(l, train, val, group)
        finally:
            l.close()
        f = _fresh(st, k, tuning)
        try:
            want = _sgda(f, train, val, group)
        finally:
            f.close()
        _assert_same_bits(got, want, name)


@pytest.mark.parametrize("k", [48, 100])
def test_sgda_after_reproducible_sgd_starts_clean(k, built_lib):
    """Two reproducible SGD epochs (which share the u64 accumulator), then sgda_begin and two SGDA epochs: what a
    new context given the parameters the SGD epochs left computes, bit for bit."""
    train, val = _long(3000, 600, seed=14)
    n = train.num_feature
    tuning = dict(rows_per_tile=256)
    group = np.arange(n) % 3
    l = _learner(n, k, 0, LR, tuning, stdev=STDEV)
    try:
        l.set_reproducible(True, 32, 4)
        l.upload(train, 0)
        init = _pull(l)
        for _ in range(2):
            l.sgd_epoch(train)
        st = _pull(l)
        got = _sgda(l, train, val, group)
    finally:
        l.close()
    assert not np.array_equal(st.v, init.v), "the SGD epochs did not move V"
    f = _fresh(st, k, tuning)
    try:
        want = _sgda(f, train, val, group)
    finally:
        f.close()
    _assert_same_bits(got, want, "after reproducible SGD")


# ---- divergence ----

@pytest.mark.parametrize("k", [48, 100])
def test_divergence_turns_the_state_nan(k, built_lib):
    train, val = _long(3000, 500, seed=15)
    l = _learner(train.num_feature, k, 0, 50.0, dict(rows_per_tile=256))
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
