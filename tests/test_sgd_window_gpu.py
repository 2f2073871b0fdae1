"""GPU: the reproducible HOGWILD SGD epoch (fmb200_set_reproducible, fm_sgd_window.cu).

The windowed epoch is oracle/rowlane_model.py's rowlane_epoch_model with TR = the tile rows and grid = the window
tiles, at any k <= 128 and any row length, with its budget widened for long rows and wide k (eps_seq = EPS_SEQ).
After every epoch each parameter must lie within that budget plus one fp32 ulp, and each of w0, w and v within a
small relative distance of what the run moved it.  The same bits on every run, grid, CTAs per SM and
threads per CTA; a held-out RMSE at C3 shape as close to the sequential oracle's as the free-running kernel's.
"""
import numpy as np
import pytest

from libfm_b200 import Data, FmError, FmLearnSgdElement, FmModel, MODE_HOGWILD, synth
from oracle import HParams, Port, State, rowlane_epoch_model
from oracle.rowlane_model import EPS_SEQ

pytestmark = pytest.mark.gpu

RAMP_TILES = 4


def _pull(l):
    l.pull_params()
    return State(float(l.fm.w0), l.fm.w.copy(), l.fm.v.copy())


def _rel(got, want, init):
    moved = np.linalg.norm(np.ravel(got - init))
    diff = np.linalg.norm(np.ravel(got - want))
    return diff / moved if moved > 0 else (0.0 if diff == 0 else np.inf)


def _learner(d, k, task=0, regs=(0.0, 0.0, 0.0), k0=True, k1=True, lr=0.01, stdev=0.05, T=0, B=0, tuning=None,
             seed=42):
    fm = FmModel(d.num_feature, k, k0, k1)
    fm.init_stdev = stdev
    fm.init_numpy(seed)
    fm.reg0, fm.regw, fm.regv = regs
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate = task, lr
    l.min_target, l.max_target = d.min_target, d.max_target
    l.push_hparams()
    l.set_tuning(**(tuning or {}))
    l.set_reproducible(True, T, B)
    l.upload(d, 0)
    return l


def run_case(name, d, k, T, B, task=0, regs=(0.0, 0.0, 0.0), k0=True, k1=True, damp=1, lr=0.01, stdev=0.05,
             epochs=3, aggregate=1e-4):
    l = _learner(d, k, task, regs, k0, k1, lr, stdev, T, B, dict(damp=damp))
    hp = HParams(task, lr, regs[0], regs[1], regs[2], d.min_target, d.max_target, k0, k1)
    n_tiles = (d.num_cases + T - 1) // T
    try:
        init = _pull(l)
        want, bud = init, None
        for e in range(epochs):
            l.sgd_epoch(d)
            cfg = l.epoch_config()
            assert cfg["rows_per_tile"] == T and cfg["lanes_per_row"] == 32, "the windowed epoch did not run"
            ramp = RAMP_TILES if e == 0 and k0 and damp >= 0 and n_tiles > 8 * RAMP_TILES else 0
            want, bud = rowlane_epoch_model(want, d, hp, TR=T, grid=B, damp=bool(cfg["damp"]), ramp_tiles=ramp,
                                            budget=bud, eps_seq=EPS_SEQ)
            got = _pull(l)
            b0, bw, bv = bud.bound(want)
            ratio = max(abs(got.w0 - want.w0) / b0, np.max(np.abs(got.w - want.w) / bw),
                        np.max(np.abs(got.v - want.v) / bv))
            agg = max(_rel(got.w0, want.w0, init.w0), _rel(got.w, want.w, init.w), _rel(got.v, want.v, init.v))
            print("window-model %-24s epoch %d  T %4d B %3d damp %d windows %4d  worst/budget %.3f  aggregate %.2e"
                  % (name, e, T, B, cfg["damp"], bud.windows, ratio, agg))
            assert ratio < 1.0, "epoch %d: a parameter is %.2f budgets away from the model" % (e, ratio)
            assert agg < aggregate, "epoch %d: relative distance to the model %.2e" % (e, agg)
            if not k0:
                assert got.w0 == init.w0
            if not k1:
                assert np.array_equal(got.w, init.w)
    finally:
        l.close()


def _long_rows(n_rows, n_feat, max_nnz, seed, zipf=0.0, twice=0.05):
    """Rows of 0 .. max_nnz entries, values in [0.5, 1.5], some naming a feature twice; ids uniform or Zipf."""
    r = np.random.default_rng(seed)
    lens = r.integers(0, max_nnz + 1, size=n_rows)
    lens[r.random(n_rows) < 0.05] = 0
    row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
    row_ptr[1:] = np.cumsum(lens)
    nnz = int(row_ptr[-1])
    if zipf > 0:
        p = 1.0 / np.arange(1, n_feat + 1) ** zipf
        col = r.choice(n_feat, size=nnz, p=p / p.sum()).astype(np.uint32)
    else:
        col = r.integers(0, n_feat, size=nnz).astype(np.uint32)
    for row in np.flatnonzero((lens >= 2) & (r.random(n_rows) < twice)):
        a = int(row_ptr[row])
        col[a + 1] = col[a]
    val = r.uniform(0.5, 1.5, size=nnz).astype(np.float32)
    y = r.integers(1, 6, size=n_rows).astype(np.float32)
    return Data(row_ptr, col, val, y, n_feat)


# ---- against the model ----

@pytest.mark.parametrize("k", [1, 5, 8, 16, 33, 64, 100, 128])
def test_factor_widths_long_rows(k, built_lib):
    """Rows of 0-60 entries, a feature named twice, non-unit values; small tiles and windows: many windows and a
    short last tile and window (4003 rows = 250 tiles of 16 and 3 rows; windows of 8 tiles)."""
    d = _long_rows(4003, 900, 60, seed=k)
    run_case("k%d" % k, d, k, T=16, B=8, lr=0.002, stdev=0.02)


@pytest.mark.parametrize("n_rows", [32 * 40, 32 * 40 + 1])
def test_exact_and_short_last_tile(n_rows, built_lib):
    """40 tiles of 32 rows in windows of 4 tiles: the ramp, then windows that end exactly or leave one row."""
    run_case("edge%d" % n_rows, _long_rows(n_rows, 300, 10, seed=3), 8, T=32, B=4)


def test_classification(built_lib):
    d = _long_rows(6000, 500, 20, seed=8)
    d = Data(d.row_ptr, d.col, d.val, np.where(d.target > 3, 1.0, -1.0), d.num_feature)
    run_case("classification", d, 16, T=64, B=8, task=1, lr=0.02)


def test_clamped_regression(built_lib):
    """Targets at the bounds and scores pushed past them: the clamp and its secant curvature."""
    d = _long_rows(6000, 400, 12, seed=9)
    d = Data(d.row_ptr, d.col, d.val, np.where(d.target > 3, 5.0, 1.0).astype(np.float32), d.num_feature)
    run_case("clamped", d, 8, T=64, B=8, lr=0.02, stdev=0.3)


@pytest.mark.parametrize("name,regs,k0,k1", [("regularised", (0.01, 0.02, 0.03), True, True),
                                             ("no_linear", (0.01, 0.02, 0.03), True, False),
                                             ("no_bias", (0.0, 0.02, 0.03), False, True)])
def test_model_switches(name, regs, k0, k1, built_lib):
    run_case(name, _long_rows(6000, 400, 16, seed=5), 16, T=64, B=8, regs=regs, k0=k0, k1=k1)


@pytest.mark.parametrize("damp", [1, -1])
def test_damping_forced(damp, built_lib):
    """On: hot Zipf ids, concurrencies far above 1, gamma well below 1.  Off: plain summed steps and no ramp, on
    uniform ids (undamped hot features amplify earlier windows' rounding beyond the model's feed-forward term)."""
    d = _long_rows(8000, 300, 8, seed=6, zipf=1.1) if damp > 0 else _long_rows(8000, 3000, 8, seed=6)
    run_case("damp%d" % damp, d, 8, T=64, B=16, damp=damp, aggregate=1e-3)


def test_c2_zipf_default_geometry(built_lib):
    """Full-size C2 with Zipf(1) ids, the default T = 256, B = 64 (62 windows after the ramp) and automatic damping."""
    d = synth.movielens_1m_shaped(seed=7, zipf=1.0)
    run_case("c2_zipf", d, 8, T=256, B=64, damp=0, aggregate=1e-3)


# ---- the same bits ----

def _c3(n_rows, seed=11):
    d = synth.multi_field(n_rows, 39, 1_000_000, seed=seed)
    d.binarize_targets()
    return d


def _bits(d, k, task, lr, tuning, epochs=2):
    l = _learner(d, k, task=task, lr=lr, stdev=0.01, tuning=tuning)
    try:
        out = []
        for _ in range(epochs):
            l.sgd_epoch(d)
            s = _pull(l)
            out.append((s.w0, s.w, s.v))
        return out, l.epoch_config()
    finally:
        l.close()


@pytest.mark.parametrize("shape", ["c3", "c2_zipf"])
def test_same_bits_every_run_and_launch(shape, built_lib):
    if shape == "c3":
        d, k, task, lr = _c3(1_000_000), 64, 1, 0.01
    else:
        d, k, task, lr = synth.movielens_1m_shaped(seed=7, zipf=1.0), 8, 0, 0.01
    ref, cfg0 = _bits(d, k, task, lr, {})
    grids = {cfg0["grid"]}
    for tuning in ({}, dict(ctas_per_sm=1), dict(threads=128), dict(threads=128, ctas_per_sm=1)):
        got, cfg = _bits(d, k, task, lr, tuning)
        grids.add(cfg["grid"])
        for e, (a, b) in enumerate(zip(ref, got)):
            assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), (tuning, e)
    assert len(grids) >= 2
    assert all(np.isfinite(x).all() for x in ref[-1][1:])


# ---- statistical parity at C3 shape ----

def _planted_c3(n_train, n_test, seed=5):
    d = synth.multi_field(n_train + n_test, 39, 1_000_000, seed=seed)
    r = np.random.default_rng(seed)
    b = r.normal(0.0, 0.15, d.num_feature)
    y = np.add.reduceat(b[d.col.astype(np.int64)], d.row_ptr[:-1].astype(np.int64)) + r.normal(0, 0.5, d.num_cases)
    d = Data(d.row_ptr, d.col, d.val, y.astype(np.float32), d.num_feature)
    return synth.split_rows(d, n_train)


def test_c3_statistical_parity(built_lib):
    """Three epochs at C3 shape (1 M planted rows, 39 entries, k = 64): after each the windowed epoch's held-out RMSE
    is as close to the sequential epoch's as twice the free-running kernel's gap, or 1e-3, at the default window
    (windows of 65 536 rows fall behind here by the third epoch; scripts/sgd_window_study.py, DESIGN.md section 3.3)."""
    train, test = _planted_c3(1_000_000, 100_000)
    k, lr = 64, 0.01
    mn, mx = float(train.target.min()), float(train.target.max())
    fm = FmModel(train.num_feature, k)
    fm.init_stdev = 0.01
    fm.init_numpy(3)
    port = Port(train.num_feature, k)
    port.set_params(fm.w0, fm.w, fm.v)
    runs = {}
    for on in (False, True):
        m = FmModel(train.num_feature, k)
        m.init_stdev = 0.01
        m.init_numpy(3)
        l = FmLearnSgdElement(m, device=0, mode=MODE_HOGWILD)
        l.task, l.learn_rate, l.min_target, l.max_target = 0, lr, mn, mx
        l.push_hparams()
        l.set_reproducible(on)
        l.upload(train, 0)
        rm = []
        for _ in range(3):
            l.sgd_epoch(train)
            l.pull_params()
            p = Port(train.num_feature, k)
            p.set_params(l.fm.w0, l.fm.w, l.fm.v)
            rm.append(p.metric(test, 0, mn, mx))
        runs[on] = rm
        l.close()
    for e in range(3):
        port.sgd_epoch(train, 0, lr, mn, mx)
        seq = port.metric(test, 0, mn, mx)
        gap_win, gap_free = abs(runs[True][e] - seq), abs(runs[False][e] - seq)
        print("C3 parity epoch %d: sequential %.5f  windowed %.5f  free-running %.5f" % (e, seq, runs[True][e],
                                                                                        runs[False][e]))
        assert gap_win <= max(2 * gap_free, 1e-3), e


# ---- divergence and the switch ----

def test_divergence_turns_the_state_nan(built_lib):
    d = _long_rows(5000, 200, 30, seed=2)
    l = _learner(d, 16, lr=50.0, stdev=0.5, T=32, B=4, tuning=dict(damp=-1))
    try:
        l.sgd_epoch(d)
        s = _pull(l)
        assert np.isnan(s.w0) and np.isnan(s.w).all() and np.isnan(s.v).all()
    finally:
        l.close()


def test_geometry_limits_are_refused(built_lib):
    d = synth.two_field(1000, 50, 40, seed=1)
    l = _learner(d, 8)
    try:
        for args, limit in (((1025, 0), "[1,1024]"), ((-1, 0), "[1,1024]"), ((0, 65537), "[1,65536]"),
                            ((0, -2), "[1,65536]")):
            with pytest.raises(FmError, match=r"\[") as e:
                l.set_reproducible(True, *args)
            assert limit in str(e.value)
        l.set_reproducible(True, 1024, 65536)
    finally:
        l.close()


@pytest.mark.parametrize("shape", ["c2", "long"])
def test_switch_off_restores_the_default_dispatch(shape, built_lib):
    d = synth.movielens_1m_shaped(seed=7, n_rows=200_000) if shape == "c2" else _long_rows(50_000, 3000, 20, seed=4)
    cfgs, launches = {}, {}
    for on in (None, True, False):
        fm = FmModel(d.num_feature, 8)
        fm.init_stdev = 0.05
        fm.init_numpy(1)
        l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
        l.task, l.learn_rate, l.min_target, l.max_target = 0, 0.01, d.min_target, d.max_target
        l.push_hparams()
        if on is not None:
            l.set_reproducible(True)
            if not on:
                l.set_reproducible(False)
        l.upload(d, 0)
        n0 = l.kernel_launches()
        for _ in range(2):
            l.sgd_epoch(d)
        launches[on] = l.kernel_launches() - n0
        cfgs[on] = (l.epoch_config(), l.epoch_dealt())
        l.close()
    assert cfgs[False] == cfgs[None] and launches[False] == launches[None]
    assert cfgs[True][0]["rows_per_tile"] == 256 and cfgs[True][0]["lanes_per_row"] == 32
    assert launches[True] == 2
