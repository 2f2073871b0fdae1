"""GPU: the free-running row-group HOGWILD epoch (fm_sgd_hogwild_kernel, fm_hogwild.cu) computes what the fp64
model of oracle/rowgroup_model.py computes, at every geometry the launcher can pick, with damping on and off.

The kernel's result is a function of its input only on data where every non-zero entry names a feature no other
non-zero entry names; zero-valued entries name the live features again (Zipf counts), so the occurrence table
and with it the concurrency c_i and gamma span their range while no sum and no step can depend on when a row
runs.  Each case reads the geometry and grid the device chose (epoch_config), restates conc_scale and w0_conc
from them, and compares every epoch as one model step from the device state before it: every parameter within
the model's per-element budget, each of w0, w, v within 1e-4 of the distance moved in 2-norm, and a second run
from the same state equal bit for bit (this data admits no race).  predict and evaluate are checked against
fp64 scores of the pulled state.  No case depends on the SM count and none skips.

tests/test_rowgroup_model.py checks the model itself and that MATRIX covers every (G, S, class) x DAMP
instantiation, on the CPU.
"""
import numpy as np
import pytest

from libfm_b200 import Data, FmLearnSgdElement, FmModel, MODE_HOGWILD
from oracle import HParams, State, geometry, concurrency, row_scores, rowgroup_epoch_model, ulp32

pytestmark = pytest.mark.gpu

# (k, average row length): each lands on one (G, S, class) of pick_geometry; the comment names it.  k cycles
# through factor widths that are not a multiple of 4 and chunk counts that are not a power of two.
MATRIX = [
    (3, 0.8),  (4, 1.6),  (1, 3.2),                          # G=1  S=1,2,4 class -1
    (4, 6.5),  (3, 13.0), (2, 35.0), (4, 75.0),              # G=1  S=8 class -1,0,1,2
    (5, 0.8),  (8, 1.6),  (7, 3.2),                          # G=2  S=1,2,4 class -1
    (8, 6.5),  (6, 13.0), (8, 35.0), (5, 75.0),              # G=2  S=8 class -1,0,1,2
    (12, 0.8), (16, 1.6), (13, 3.2),                         # G=4  S=1,2,4 class -1   (k=12, 13: gp=3)
    (16, 6.5), (12, 13.0), (9, 35.0), (16, 75.0),            # G=4  S=8 class -1,0,1,2
    (20, 0.8), (32, 1.6),                                    # G=8  S=1,2 class -1     (k=20: gp=5)
    (32, 3.8), (24, 7.0), (20, 20.0), (32, 45.0),            # G=8  S=4 class -1,0,1,2
    (40, 0.8),                                               # G=16 S=1 class -1       (k=40: 6 idle chunk lanes)
    (64, 2.0), (40, 4.0), (64, 10.0), (40, 25.0),            # G=16 S=2 class -1,0,1,2
    (100, 1.5), (128, 2.5), (100, 6.0), (128, 14.0), (100, 26.0),  # G=32 S=1 class -1,0,1,2,3 (k=100: gp=25)
]
NNZ = 30_000  # entries per matrix case


def make_data(n_rows, avg, geo=None, seed=0, live=0.5, zipf=1.0, task=0, long_rows=8, spare=3):
    """Rows of Poisson(avg) entries and `long_rows` rows longer than the register caches (q >= R, t >= RW).
    A fraction `live` of the entries are non-zero, each naming its own feature; the rest are zero-valued and
    name live features again with Zipf(zipf) counts.  `spare` features are never named."""
    r = np.random.default_rng(seed)
    long_len = 0
    if geo is not None and long_rows:
        long_len = int(max(3 * avg, geo.R * geo.S, geo.RW * geo.E)) + 2
    mb = max(0.0, (avg * n_rows - long_rows * long_len) / (n_rows - long_rows))
    lengths = r.poisson(mb, n_rows)
    if long_len:
        lengths[r.choice(n_rows, long_rows, replace=False)] = long_len + r.integers(0, 3, long_rows)
    nnz = int(lengths.sum())
    n_live = max(1, int(round(live * nnz)))
    n_zero = nnz - n_live
    feat = r.permutation(n_live)  # rank -> live feature
    rank_p = 1.0 / np.arange(1, n_live + 1) ** zipf
    zero_ids = feat[r.choice(n_live, n_zero, p=rank_p / rank_p.sum())]
    ids = np.concatenate([np.arange(n_live), zero_ids])
    x = r.uniform(0.5, 1.5, n_live) * r.choice([-1.0, 1.0], n_live)
    x[r.random(n_live) < 0.2] = 1.0
    vals = np.concatenate([x, np.where(r.random(n_zero) < 0.1, -0.0, 0.0)])
    order = r.permutation(nnz)  # live and zero-valued entries anywhere, their live entry's row included
    row_ptr = np.concatenate([[0], np.cumsum(lengths)])
    y = np.where(r.random(n_rows) < 0.5, 1.0, -1.0) if task == 1 else r.standard_normal(n_rows)
    return Data(row_ptr, ids[order], vals[order], y, n_live + spare)


def matrix_case(i):
    """Data of MATRIX[i] and its geometry (computed from the data: the realised average decides)."""
    k, avg = MATRIX[i]
    n_rows = int(np.clip(NNZ / avg, 400, 40_000))
    geo0 = geometry(k, n_rows, int(avg * n_rows))
    d = make_data(n_rows, avg, geo0, seed=100 + i)
    return k, d, geometry(k, d.num_cases, d.num_values)


def tuning_for(k, d, **t):
    """variant 1 keeps the row-lane kernel (k <= 8, rows of <= 4 entries) off every shape it could take."""
    if ((k + 3) // 4) <= 2:
        t["variant"] = 1
    return t


def _pull(l):
    l.pull_params()
    return State(float(l.fm.w0), l.fm.w.copy(), l.fm.v.copy())


def _push(l, st):
    l.fm.w0, l.fm.w, l.fm.v = st.w0, st.w.copy(), st.v.copy()
    l.push_params()


def _rel(got, want, init):
    moved = np.linalg.norm(np.ravel(got - init))
    diff = np.linalg.norm(np.ravel(got - want))
    return diff / moved if moved > 0 else (0.0 if diff == 0 else np.inf)


def check_scores(l, d, hp, st):
    """predict (raw and transformed) and evaluate against fp64 scores of the state `st` the device holds."""
    p, dp = row_scores(st, d, hp)
    tol = dp + ulp32(p)
    raw = l.predict(d, transform=False)
    assert np.all(np.abs(raw - p) <= tol), "raw scores: worst %.3g" % np.max(np.abs(raw - p) / tol)
    y = d.target.astype(np.float64)
    out = l.predict(d, transform=True)
    metric = l.evaluate(d)
    if hp.task == 0:
        pc = np.clip(p, np.float32(hp.min_target), np.float32(hp.max_target))
        assert np.all(np.abs(out - pc) <= tol)
        err = pc - y
        t = float(np.max(tol)) + 1e-12
        assert abs(metric - np.sqrt(np.mean(err * err))) <= t
        assert abs(l.last_mae - np.mean(np.abs(err))) <= t
    else:
        s = 1.0 / (1.0 + np.exp(-p))
        assert np.all(np.abs(out - s) <= tol * s * (1.0 - s) + 4.0 * ulp32(s))
        ok = ((p >= 0) & (y >= 0)) | ((p < 0) & (y < 0))
        unsure = np.abs(p) <= tol
        assert abs(metric - ok.mean()) <= unsure.sum() / d.num_cases + 1e-15
        assert l.last_mae == 0.0


def run_case(name, d, k, damp, tuning, task=0, regs=(0.0, 0.0, 0.0), k0=False, k1=True, epochs=2, lr=0.01,
             w0=0.0, targets=None, expect=None, one_tile=False):
    """Runs `epochs` epochs and compares each with one model step from the device state before it.  expect:
    the (G, S, class) the data must select.  Returns the worst |got - want| / budget and the last epoch_config."""
    geo = geometry(k, d.num_cases, d.num_values, tuning.get("threads", 0))
    if expect is not None:
        assert (geo.G, geo.S, geo.cls) == expect
    lo, hi = targets if targets is not None else (d.min_target, d.max_target)
    r = np.random.default_rng(7)
    fm = FmModel(d.num_feature, k, k0, k1)
    fm.init_stdev = 0.1
    fm.init_numpy(42)
    fm.w0 = w0
    fm.w = np.asarray(0.05 * r.standard_normal(d.num_feature), dtype=np.float32).astype(np.float64)
    fm.reg0, fm.regw, fm.regv = regs
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate = task, lr
    l.min_target, l.max_target = lo, hi
    l.push_hparams()
    l.set_tuning(damp=damp, **tuning)
    l.upload(d, 0)
    hp = HParams(task, lr, regs[0], regs[1], regs[2], lo, hi, k0, k1)
    worst, cfg = 0.0, None
    try:
        init = _pull(l)
        for e in range(epochs):
            before = _pull(l)
            l.sgd_epoch(d)
            cfg = l.epoch_config()
            got = _pull(l)
            _push(l, before)  # the same epoch once more from the same state
            l.sgd_epoch(d)
            again = _pull(l)
            assert again.w0 == got.w0 and np.array_equal(again.w, got.w) and np.array_equal(again.v, got.v), \
                "two runs from one state differ"
            assert (cfg["lanes_per_row"], cfg["slots"]) == (geo.G, geo.S), "the row-group kernel did not run"
            assert cfg["damp"] == (1 if damp == 1 else 0)
            TR, grid = cfg["rows_per_tile"], cfg["grid"]
            if one_tile:
                assert d.num_cases <= TR and grid == 1
            conc_scale, w0_conc = concurrency(geo, d.num_cases, grid, TR)
            want, bud = rowgroup_epoch_model(before, d, hp, conc_scale, w0_conc, damp == 1, TR)
            # the budget plus one fp32 ulp of the element (on whichever side of a binade edge it ends): model and
            # kernel each round their sum once, so a step that differs by far less than an ulp may still land
            # one ulp apart.  `arith` is what exceeds that ulp, against the budget: the constants' margin.
            ratio, arith = 0.0, 0.0
            for g_, w_, b_ in ((got.w0, want.w0, bud.w0), (got.w, want.w, bud.w), (got.v, want.v, bud.v)):
                diff = np.abs(np.asarray(g_ - w_, dtype=np.float64))
                ulp = ulp32(np.maximum(np.abs(g_), np.abs(w_)))
                b_ = np.asarray(b_, dtype=np.float64)
                ratio = max(ratio, float(np.max(diff / (b_ + ulp))))
                over = np.maximum(diff - ulp, 0.0)
                arith = max(arith, float(np.max(np.where(b_ > 0, over / np.where(b_ > 0, b_, 1.0),
                                                        np.where(over > 0, np.inf, 0.0)))))
            agg = max(_rel(got.w0, want.w0, before.w0), _rel(got.w, want.w, before.w),
                      _rel(got.v, want.v, before.v))
            c_max = float(np.bincount(d.col.astype(np.int64), minlength=d.num_feature).max()) * conc_scale
            print("rowgroup-model %-16s epoch %d  G %2d S %d class %2d  k %3d TR %3d block %3d grid %3d damp %d "
                  "c_max %7.1f  worst/budget %.3f  beyond one ulp %.3f  aggregate %.2e" % (
                      name, e, geo.G, geo.S, geo.cls, k, TR, cfg["block"], grid, cfg["damp"], c_max, ratio, arith,
                      agg))
            assert ratio < 1.0, "epoch %d: a parameter is %.2f budgets away from the model" % (e, ratio)
            assert agg < 1e-4, "epoch %d: relative distance to the model %.2e" % (e, agg)
            if not k0:
                assert got.w0 == init.w0
            if not k1:
                assert np.array_equal(got.w, init.w)
            worst = max(worst, ratio)
        check_scores(l, d, hp, _pull(l))
    finally:
        l.close()
    return worst, cfg


# ---- the matrix: every (G, S, class) with DAMP on and off ----

@pytest.mark.parametrize("damp", [1, -1])
@pytest.mark.parametrize("i", range(len(MATRIX)))
def test_geometry_matrix(i, damp, built_lib):
    k, d, geo = matrix_case(i)
    run_case("matrix%02d" % i, d, k, damp, tuning_for(k, d), expect=(geo.G, geo.S, geo.cls))


# ---- the bias: one tile, so every row reads the w0 the epoch found ----

ONE_TILE = dict(rows_per_tile=512)


@pytest.mark.parametrize("k,avg", [(8, 13.0), (24, 7.0), (128, 26.0), (40, 0.8)])
def test_bias_with_hot_features(k, avg, built_lib):
    """Zero-valued entries and DAMP: the tile's H carries every row's hrow, and gamma of the bias is far below 1."""
    d = make_data(32, avg, geometry(k, 32, int(32 * avg)), seed=k)
    run_case("bias_hot_k%d" % k, d, k, 1, tuning_for(k, d, **ONE_TILE), k0=True, w0=0.2, lr=0.02, one_tile=True)


@pytest.mark.parametrize("damp", [1, -1])
@pytest.mark.parametrize("name,k,avg,task,k1,targets", [
    ("clamped", 16, 6.5, 0, True, (-0.3, 0.3)),     # most scores outside [-0.3, 0.3]: secant curvature
    ("classification", 40, 4.0, 1, True, None),
    ("no_linear", 7, 35.0, 0, False, (-2.0, 2.0)),  # k1 = 0: hrow without xx, w untouched
    ("long_rows", 100, 26.0, 0, True, None),
])
def test_bias_regularised(name, k, avg, task, k1, targets, damp, built_lib):
    """No zero-valued entries, reg0, regw, regv != 0 (every c_i <= 1): reg0 enters M and the bias's gamma."""
    geo = geometry(k, 200, int(200 * avg))
    d = make_data(200, avg, geo, seed=len(name), live=1.0, task=task)
    d = d.rows(0, 32 if avg > 10 else 200)
    run_case("bias_" + name, d, k, damp, tuning_for(k, d, **ONE_TILE), task=task, regs=(0.05, 0.02, 0.03),
             k0=True, k1=k1, w0=0.3, lr=0.03, targets=targets, one_tile=True)


# ---- launch shapes ----

SHAPES = [(t, c, rpt) for t in (32, 96, 256) for c in (1, 2, 3) for rpt in (32, 512)]


@pytest.mark.parametrize("threads,ctas,rpt", SHAPES)
@pytest.mark.parametrize("k,avg", [(64, 10.0), (8, 13.0)])
def test_launch_shapes(k, avg, threads, ctas, rpt, built_lib):
    d = make_data(20_000, avg, geometry(k, 20_000, int(20_000 * avg)), seed=threads + ctas + rpt)
    run_case("shape_t%d_c%d_r%d" % (threads, ctas, rpt), d, k, 1,
             tuning_for(k, d, threads=threads, ctas_per_sm=ctas, rows_per_tile=rpt), epochs=1)


def _stage_bytes(TR, cap):
    return ((TR + 2) * 8 + TR * 4 + 2 * cap * 4 + 15) & ~15  # hw_stage_bytes, fm_hogwild_common.cuh


@pytest.mark.parametrize("k", [4, 128])
def test_global_entries(k, built_lib):
    """Rows of ~500 entries, mostly zero-valued: no 32-row tile fits the staging ring, so the lanes read ids and
    values from global memory (tiles of 64 rows, only offsets and targets staged)."""
    d = make_data(300, 500.0, geometry(k, 300, 150_000), seed=k, live=0.1, long_rows=0)
    _, cfg = run_case("global_k%d" % k, d, k, 1, tuning_for(k, d), epochs=1)
    assert cfg["rows_per_tile"] == 64 and cfg["smem_bytes"] == 256 + 3 * _stage_bytes(64, 0)
