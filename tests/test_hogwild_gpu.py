"""GPU: the throughput path (HOGWILD mode, fp32 state, L2 reductions).

Hogwild cannot reproduce the sequential trajectory parameter-for-parameter (the
reference is strictly in-order, fm_learn_sgd_element.h:56-67).  What is pinned:
  * the fp32 score equals the oracle's fm_model::predict to fp32 accuracy;
  * a 1-row epoch equals one reference step (no concurrency => same arithmetic);
  * with rows that share no feature the epoch equals the oracle up to the bias carry;
  * on learnable data the per-epoch RMSE trajectory tracks the oracle's;
  * size-independent properties at BASELINE C2 size (finite state, loss decreases,
    linearity of the zero-learning-rate epoch, padding stays zero).
"""
import numpy as np
import pytest

from conftest import GOLDEN_CASES, load_golden, make_learner
from libfm_b200 import MODE_HOGWILD, MODE_INORDER, Data, FmLearnSgdElement, FmModel, synth
from oracle import Port

pytestmark = pytest.mark.gpu


def _cfg(n, k, task=0, lr=0.01, regs=(0, 0, 0), k0=1, k1=1, mn=1.0, mx=5.0):
    return dict(n=n, k=k, k0=k0, k1=k1, task=task, lr=lr, regs=np.array(regs, dtype=float),
                min_target=mn, max_target=mx)


def _port(cfg, init):
    p = Port(cfg["n"], cfg["k"], cfg["k0"], cfg["k1"])
    p.set_params(*init)
    p.reg0, p.regw, p.regv = [float(x) for x in cfg["regs"]]
    return p


def _rand_init(n, k, seed, stdev=0.1):
    r = np.random.default_rng(seed)
    return (float(r.standard_normal() * 0.1), r.standard_normal(n) * 0.1,
            r.standard_normal((k, n)) * stdev)


@pytest.mark.parametrize("k,maxnnz", [(1, 3), (4, 1), (8, 2), (8, 9), (12, 5), (16, 4), (32, 17),
                                      (64, 39), (128, 6), (128, 40)])
def test_fp32_score_matches_oracle(k, maxnnz, built_lib):
    d = synth.ragged(1500, 300, maxnnz, seed=k * 100 + maxnnz)
    cfg = _cfg(300, k, mn=-1e30, mx=1e30)
    init = _rand_init(300, k, k + 1, stdev=0.3)
    l = make_learner(cfg, init, mode=MODE_HOGWILD)
    got = l.predict(d, transform=False)
    want = _port(cfg, init).predict(d, 0, 0, 0, transform=False)
    scale = 1.0 + np.abs(want)
    assert np.max(np.abs(got - want) / scale) < 5e-5
    l.close()


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_fp32_metrics_on_reference_final_state(name, built_lib):
    """evaluate()/predict() of the reference's FINAL parameters, fp32 path."""
    z, tr, te = load_golden(name)
    l = make_learner(z, (float(z["w0"]), z["w"], z["v"]), mode=MODE_HOGWILD)
    e = int(z["epochs"]) - 1
    tol = 2e-5 if int(z["task"]) == 0 else 0.011  # accuracy: a borderline score may flip sign
    assert abs(l.evaluate(tr) - z["metric_train"][e]) < tol
    assert abs(l.evaluate(te) - z["metric_test"][e]) < tol
    np.testing.assert_allclose(l.predict(te), z["pred_test"], atol=2e-5)
    l.close()


@pytest.mark.parametrize("task", [0, 1])
def test_single_row_epoch_equals_reference_step(task, built_lib):
    d = Data(np.array([0, 4], dtype=np.uint64), np.array([3, 17, 5, 3], dtype=np.uint32),
             np.array([1.0, -0.5, 2.0, 0.25], dtype=np.float32),
             np.array([1.0 if task else 4.0], dtype=np.float32), 20)
    cfg = _cfg(20, 8, task=task, lr=0.05, regs=(0.01, 0.02, 0.03), mn=1.0, mx=5.0)
    init = _rand_init(20, 8, 4, stdev=0.2)
    l = make_learner(cfg, init, mode=MODE_HOGWILD)
    p = _port(cfg, tuple(np.float32(x).astype(np.float64) for x in init))
    l.sgd_epoch(d)
    p.sgd_epoch(d, task, 0.05, 1.0, 5.0)
    l.pull_params()
    # id 3 repeats inside the row: the reference re-reads v after the first update
    # (fm_sgd.h:44-50); Hogwild applies both deltas from the pre-update value.  The
    # difference is O(lr^2); everything else agrees to fp32 rounding.
    assert abs(l.fm.w0 - p.w0.value) < 1e-6
    np.testing.assert_allclose(l.fm.w, p.w, atol=5e-3)
    np.testing.assert_allclose(l.fm.v, p.v, atol=5e-3)
    mask = np.ones(20, bool)
    mask[3] = False
    np.testing.assert_allclose(l.fm.w[mask], p.w[mask], atol=1e-6)
    np.testing.assert_allclose(l.fm.v[:, mask], p.v[:, mask], atol=1e-6)
    l.close()


def test_disjoint_rows_match_oracle_without_bias(built_lib):
    """Rows that share no feature and no bias are independent: any schedule is
    sequentially equivalent, so Hogwild must equal the oracle (fp32 rounding)."""
    n_rows, z = 3000, 3
    n = n_rows * z
    r = np.random.default_rng(3)
    col = r.permutation(n).astype(np.uint32)
    d = Data(np.arange(0, n + 1, z, dtype=np.uint64), col, r.standard_normal(n).astype(np.float32),
             r.integers(1, 6, n_rows).astype(np.float32), n)
    cfg = _cfg(n, 8, k0=0, lr=0.05, regs=(0, 0.01, 0.02))
    init = _rand_init(n, 8, 5, stdev=0.3)
    init32 = tuple(np.float32(x).astype(np.float64) for x in init)
    l = make_learner(cfg, init, mode=MODE_HOGWILD)
    p = _port(cfg, init32)
    l.sgd_epoch(d)
    p.sgd_epoch(d, 0, 0.05, 1.0, 5.0)
    l.pull_params()
    np.testing.assert_allclose(l.fm.w, p.w, atol=2e-6)
    np.testing.assert_allclose(l.fm.v, p.v, atol=2e-6)
    l.close()


@pytest.mark.parametrize("k,maxnnz", [(8, 2), (8, 4), (4, 3), (3, 1), (7, 4)])
def test_rowlane_and_rowgroup_kernels_agree(k, maxnnz, built_lib):
    """The two HOGWILD epoch kernels implement the same step: on rows that share no
    feature (any schedule is sequentially equivalent) both must equal the oracle."""
    n_rows = 4000
    r = np.random.default_rng(k * 10 + maxnnz)
    lens = r.integers(0, maxnnz + 1, n_rows)
    rp = np.zeros(n_rows + 1, dtype=np.uint64)
    rp[1:] = np.cumsum(lens)
    n = int(rp[-1]) + 5
    d = Data(rp, r.permutation(n)[: int(rp[-1])].astype(np.uint32),
             r.standard_normal(int(rp[-1])).astype(np.float32),
             r.integers(1, 6, n_rows).astype(np.float32), n)
    cfg = _cfg(n, k, k0=0, lr=0.05, regs=(0, 0.01, 0.02))
    init = _rand_init(n, k, 5, stdev=0.3)
    init32 = tuple(np.float32(x).astype(np.float64) for x in init)
    p = _port(cfg, init32)
    p.sgd_epoch(d, 0, 0.05, 1.0, 5.0)
    for variant, lanes in ((1, None), (2, 1), (3, 1)):  # row-group, row-lane, warp-specialised row-lane
        l = make_learner(cfg, init, mode=MODE_HOGWILD)
        l.set_tuning(variant=variant)
        l.sgd_epoch(d)
        if lanes is not None:
            assert l.epoch_config()["lanes_per_row"] == lanes
        else:
            assert l.epoch_config()["lanes_per_row"] >= 1 and l.epoch_config()["rows_per_tile"] >= 32
        l.pull_params()
        np.testing.assert_allclose(l.fm.w, p.w, atol=2e-6)
        np.testing.assert_allclose(l.fm.v, p.v, atol=2e-6)
        l.close()


def test_zero_learning_rate_epoch_is_identity(built_lib):
    d = synth.two_field(20000, 300, 200, seed=8)
    cfg = _cfg(500, 8, lr=0.0)
    init = _rand_init(500, 8, 6)
    l = make_learner(cfg, init, mode=MODE_HOGWILD)
    l.pull_params()
    before = (l.fm.w0, l.fm.w.copy(), l.fm.v.copy())
    l.sgd_epoch(d)
    l.pull_params()
    assert abs(l.fm.w0 - before[0]) < 1e-6
    assert np.array_equal(l.fm.w, before[1]) and np.array_equal(l.fm.v, before[2])
    l.close()


def test_rmse_trajectory_tracks_oracle_on_learnable_data(built_lib):
    """Statistical parity of the throughput mode: planted-FM ratings, 6 epochs."""
    tr = synth.two_field(200_000, 3000, 2000, seed=31, planted_k=4)
    te = synth.two_field(20_000, 3000, 2000, seed=32, planted_k=4)
    # the same hidden model must generate train and test: regenerate jointly
    both = synth.two_field(220_000, 3000, 2000, seed=31, planted_k=4)
    tr, te = both.rows(0, 200_000), both.rows(200_000, 220_000)
    n, k = 5000, 8
    cfg = _cfg(n, k, lr=0.01, regs=(0, 0, 0.0), mn=1.0, mx=5.0)
    r = np.random.default_rng(0)
    init = (0.0, np.zeros(n), r.standard_normal((k, n)) * 0.1)
    l = make_learner(cfg, init, mode=MODE_HOGWILD)
    p = _port(cfg, init)
    worst, gaps = 0.0, []
    for e in range(6):
        l.sgd_epoch(tr)
        p.sgd_epoch(tr, 0, 0.01, 1.0, 5.0)
        g_tr, g_te = l.evaluate(tr), l.evaluate(te)
        o_tr, o_te = p.metric(tr, 0, 1.0, 5.0), p.metric(te, 0, 1.0, 5.0)
        worst = max(worst, abs(g_tr - o_tr), abs(g_te - o_te))
        gaps.append(max(abs(g_tr - o_tr), abs(g_te - o_te)))
        print("[hogwild 200k] epoch %d  gpu train %.5f test %.5f | oracle train %.5f test %.5f" % (e, g_tr, g_te, o_tr, o_te))
    # the concurrent schedule lags the sequential one in the first epochs (one damped
    # Jacobi-like sweep vs 200k Gauss-Seidel steps) and converges to the same optimum
    # (r02 runs: 0.057 in epoch 0 -- this 200k-row set is smaller than the 113k-row window is comfortable with --
    # and 0.003 after 6 epochs; the C2-size trajectory test below holds the tighter bars)
    assert worst < 0.07, worst
    assert gaps[-1] < 0.006 and gaps[-1] < gaps[0], gaps
    assert g_te < 1.0  # it learned: the no-signal RMSE of these ratings is ~1.17
    l.close()


@pytest.mark.parametrize("zipf", [0.0, 1.0])
def test_small_and_skewed_data_stay_stable(zipf, built_lib):
    """All rows in flight at once (tiny data set) and Zipf-popular features: plain summed
    Hogwild diverges here; the mean-field step scale keeps the trajectory near the oracle's."""
    both = synth.two_field(44_000, 600, 400, seed=41, zipf=zipf, planted_k=4)
    tr, te = both.rows(0, 40_000), both.rows(40_000, 44_000)
    n, k = 1000, 8
    cfg = _cfg(n, k, lr=0.01, mn=1.0, mx=5.0)
    r = np.random.default_rng(2)
    init = (0.0, np.zeros(n), r.standard_normal((k, n)) * 0.1)
    l = make_learner(cfg, init, mode=MODE_HOGWILD)
    p = _port(cfg, init)
    for e in range(5):
        l.sgd_epoch(tr)
        p.sgd_epoch(tr, 0, 0.01, 1.0, 5.0)
        g_te, o_te = l.evaluate(te), p.metric(te, 0, 1.0, 5.0)
        print("zipf %.1f epoch %d gpu test %.4f oracle test %.4f damp=%d" % (zipf, e, g_te, o_te, l.epoch_config()["damp"]))
    assert g_te < o_te + 0.08, (g_te, o_te)
    l.close()


def test_hogwild_c2_trajectory_vs_oracle(built_lib):
    """BASELINE config C2 at full size (the configuration the headline is timed on), planted signal, train +
    held-out rows of the same planted model, 5 epochs from the same initial model as the oracle.  HOGWILD is
    outside the 1e-5 gate by construction (rows in flight share stale parameters); what it does deliver, with the
    first-epoch bias ramp (fm_hogwild.cu), is asserted here."""
    tr, te = synth.movielens_1m_planted(100_000, seed=7)
    n, k = tr.num_feature, 8
    cfg = _cfg(n, k, lr=0.01, mn=tr.min_target, mx=tr.max_target)
    init = (0.0, np.zeros(n), np.random.default_rng(42).standard_normal((k, n)) * 0.1)
    l = make_learner(cfg, init, mode=MODE_HOGWILD)
    p = _port(cfg, init)
    gaps = []
    for e in range(5):
        l.sgd_epoch(tr)
        p.sgd_epoch(tr, 0, 0.01, cfg["min_target"], cfg["max_target"])
        g = (l.evaluate(tr), l.evaluate(te))
        o = (p.metric(tr, 0, cfg["min_target"], cfg["max_target"]), p.metric(te, 0, cfg["min_target"], cfg["max_target"]))
        gaps.append(max(abs(g[0] - o[0]), abs(g[1] - o[1])))
    print("\n[hogwild C2 full] RMSE gap to the oracle per epoch: " + " ".join("%.5f" % x for x in gaps))
    assert gaps[0] < 0.02 and max(gaps[1:]) < 0.003, gaps
    l.close()


def test_c2_size_properties(built_lib):
    """BASELINE config C2 at full size: size-independent checks."""
    d = synth.movielens_1m_shaped(seed=7, planted_k=4)
    n, k = d.num_feature, 8
    cfg = _cfg(n, k, lr=0.01, mn=d.min_target, mx=d.max_target)
    r = np.random.default_rng(1)
    init = (0.0, np.zeros(n), r.standard_normal((k, n)) * 0.1)
    l = make_learner(cfg, init, mode=MODE_HOGWILD)
    base = l.evaluate(d)
    hist = []
    for _ in range(4):
        l.sgd_epoch(d)
        hist.append(l.evaluate(d))
    l.pull_params()
    assert np.isfinite(l.fm.v).all() and np.isfinite(l.fm.w).all() and np.isfinite(l.fm.w0)
    assert hist[0] < base and hist[-1] < hist[0]
    cfgd = l.epoch_config()
    assert cfgd["lanes_per_row"] == 1 and cfgd["slots"] == 2  # one-lane-per-row kernel, 2 nnz/row
    # INORDER evaluate of the same state agrees with the fp32 evaluate
    l.set_mode(MODE_INORDER)
    assert abs(l.evaluate(d) - hist[-1]) < 1e-5
    l.close()


def test_peer_allreduce_mean_two_contexts(built_lib):
    """fm_peer.cu: two replicas (two contexts of one process, same device) average
    their packed state through mapped peer buffers; both end bit-identical."""
    import ctypes as C
    n, k = 300, 8
    cfg = _cfg(n, k)
    a = make_learner(cfg, _rand_init(n, k, 1), mode=MODE_HOGWILD)
    b = make_learner(cfg, _rand_init(n, k, 2), mode=MODE_HOGWILD)
    arr = (C.c_void_p * 2)(a._ctx, b._ctx)
    for rank, l in enumerate((a, b)):
        assert l.lib.fmb200_peer_attach_local(l._ctx, 2, rank, arr) == 0, l.lib.fmb200_last_error()
    a.pull_params(); b.pull_params()
    want_w0 = np.float32(0.5) * (np.float32(a.fm.w0) + np.float32(b.fm.w0))
    want_v = (np.float32(0.5) * (a.fm.v.astype(np.float32) + b.fm.v.astype(np.float32))).astype(np.float64)
    want_w = (np.float32(0.5) * (a.fm.w.astype(np.float32) + b.fm.w.astype(np.float32))).astype(np.float64)
    for rounds in range(3):  # exercises the double buffering
        for l in (a, b):
            assert l.lib.fmb200_allreduce_mean(l._ctx) == 0, l.lib.fmb200_last_error()
        for l in (a, b):
            assert l.lib.fmb200_sync(l._ctx) == 0
        a.pull_params(); b.pull_params()
        assert a.fm.w0 == b.fm.w0 and np.array_equal(a.fm.v, b.fm.v) and np.array_equal(a.fm.w, b.fm.w)
        assert abs(a.fm.w0 - float(want_w0)) < 1e-7
        np.testing.assert_allclose(a.fm.v, want_v, atol=1e-7)
        np.testing.assert_allclose(a.fm.w, want_w, atol=1e-7)
    # training continues on the swapped buffer
    d = synth.two_field(5000, 200, 100, seed=3)
    a.sgd_epoch(d)
    assert np.isfinite(a.evaluate(d))
    a.close(); b.close()


def test_c3_shape_properties(built_lib):
    """BASELINE config C3 shape (Criteo-like: 39 one-hot fields over 1M features, k=64,
    classification), 300k rows: score parity on a sample, loss decreases, state finite."""
    d = synth.multi_field(300_000, 39, 1_000_000, seed=11)
    d.binarize_targets()
    n, k = d.num_feature, 64
    cfg = _cfg(n, k, task=1, lr=0.01, regs=(0, 0, 0.0), mn=-1.0, mx=1.0)
    r = np.random.default_rng(4)
    init = (0.0, np.zeros(n), (r.standard_normal((k, n)) * 0.01))
    l = make_learner(cfg, init, mode=MODE_HOGWILD)
    sample = d.rows(1000, 3000)
    got = l.predict(sample, transform=False)
    want = _port(cfg, init).predict(sample, 1, 0, 0, transform=False)
    assert np.max(np.abs(got - want)) < 5e-5
    acc0 = l.evaluate(d)
    for _ in range(3):
        l.sgd_epoch(d)
    acc1 = l.evaluate(d)
    cfgd = l.epoch_config()
    assert cfgd["lanes_per_row"] == 16  # k=64 -> 16 float4 lanes per factor row
    assert acc1 > acc0 + 0.02  # random labels: it can only memorise, and it does
    l.pull_params()
    assert np.isfinite(l.fm.v).all() and np.isfinite(l.fm.w).all()
    l.close()


def test_in_warp_combining_sums_every_step(built_lib):
    """Skewed ids switch the row-lane kernel to in-warp merging of same-feature steps.
    With a tiny learning rate an epoch is linear in the per-row steps (every row sees
    ~the initial state), so the write-back of BOTH epoch kernels must equal the sum of
    the reference's per-row fm_SGD steps evaluated at the initial state (numpy, fp64):
    nothing may be dropped or double-counted by the merge."""
    d = synth.two_field(30_000, 50, 40, seed=9, zipf=1.2)
    n, k, lr = 90, 8, 1e-6
    cfg = _cfg(n, k, lr=lr, regs=(0, 0.5, 0.25), mn=1.0, mx=5.0)
    init = _rand_init(n, k, 11, stdev=0.3)
    w0, w, v = [np.float32(x).astype(np.float64) for x in init]
    v = v.reshape(k, n)
    # ---- fp64 ground truth of the linearised epoch (fm_model.h:105-127, fm_sgd.h:33-51) ----
    ids = d.col.reshape(-1, 2).astype(np.int64)
    vu, vi = v[:, ids[:, 0]], v[:, ids[:, 1]]          # [k, rows]
    p = w0 + w[ids[:, 0]] + w[ids[:, 1]] + (vu * vi).sum(0)
    mult = np.clip(p, 1.0, 5.0) - d.target
    dw, aw = np.zeros(n), np.zeros(n)            # sum of steps, sum of |steps|
    dv, av = np.zeros((k, n)), np.zeros((k, n))
    for side, other in ((0, vi), (1, vu)):
        sw_ = -lr * (mult + 0.5 * w[ids[:, side]])
        np.add.at(dw, ids[:, side], sw_)
        np.add.at(aw, ids[:, side], np.abs(sw_))
        step = -lr * (mult[None, :] * other + 0.25 * v[:, ids[:, side]])   # grad = s_f - v_f = other side
        for f in range(k):
            np.add.at(dv[f], ids[:, side], step[f])
            np.add.at(av[f], ids[:, side], np.abs(step[f]))
    for variant in (1, 2):
        l = make_learner(cfg, init, mode=MODE_HOGWILD)
        l.set_tuning(damp=-1, variant=variant)
        l.sgd_epoch(d)
        l.pull_params()
        assert (l.epoch_config()["lanes_per_row"] == 1) == (variant == 2)
        got_w, got_v = l.fm.w - w, l.fm.v - v
        l.close()
        # rows see a state that has drifted by up to ~1% (order-dependent) and fp32 adds
        # round: allow 2% of the summed |steps| per element; a dropped or doubled merged
        # step would be a 10-50% error on the hot features
        assert np.all(np.abs(got_w - dw) <= 0.02 * aw + 2e-6), "variant %d w" % variant
        assert np.all(np.abs(got_v - dv) <= 0.02 * av + 2e-6), "variant %d v" % variant
        hot = np.argmax(aw)
        assert abs(got_w[hot] - dw[hot]) < 0.05 * abs(dw[hot])  # the hottest feature, relative


def test_c3_full_size_properties(built_lib):
    """BASELINE config C3 at its full size: 10M rows x 39 one-hot fields over 1M features,
    k=64, classification (390M entries, 3.2 GB of CSR).  Size-independent checks: a
    zero-learning-rate epoch is the identity, training accuracy rises, state stays finite."""
    n_rows, fields, n = 10_000_000, 39, 1_000_000
    r = np.random.default_rng(11)
    per = n // fields
    col = r.integers(0, per, size=(n_rows, fields), dtype=np.uint32)
    col += (np.arange(fields, dtype=np.uint32) * np.uint32(per))[None, :]
    d = Data(np.arange(0, (n_rows + 1) * fields, fields, dtype=np.uint64), col.reshape(-1),
             np.ones(n_rows * fields, dtype=np.float32),
             np.where(r.random(n_rows) < 0.5, -1.0, 1.0).astype(np.float32), n)
    del col
    k = 64
    cfg = _cfg(n, k, task=1, lr=0.0, mn=-1.0, mx=1.0)
    init = (0.0, np.zeros(n), (r.standard_normal((k, n)) * 0.01))
    l = make_learner(cfg, init, mode=MODE_HOGWILD)
    l.pull_params()
    v_before = l.fm.v.copy()
    t0 = l.sgd_epoch(d)
    l.pull_params()
    assert np.array_equal(l.fm.v, v_before) and not l.fm.w.any()  # lr = 0: identity
    acc0 = l.evaluate(d)
    l.learn_rate = 0.01
    l.push_hparams()
    secs = [l.sgd_epoch(d) for _ in range(2)]
    acc1 = l.evaluate(d)
    print("C3 full size: %.1f ms/epoch (%.2f G ex/s), accuracy %.4f -> %.4f" % (
        1e3 * min(secs), n_rows / min(secs) / 1e9, acc0, acc1))
    assert acc1 > acc0 + 0.005
    l.pull_params()
    assert np.isfinite(l.fm.v).all() and np.isfinite(l.fm.w).all() and np.isfinite(l.fm.w0)
    assert min(secs) < 0.2  # 10M rows: tens of milliseconds, not seconds
    l.close()


@pytest.mark.parametrize("k,maxnnz", [(8, 2), (16, 3), (0, 3), (64, 12)])
def test_launch_geometry_matrix(k, maxnnz, built_lib):
    """Every tuning knob (CTAs/SM, rows per tile, threads, kernel variant) must leave the
    result unchanged on rows that share no feature: oracle equality for all of them."""
    n_rows = 1500
    r = np.random.default_rng(k + maxnnz)
    lens = r.integers(0, maxnnz + 1, n_rows)
    rp = np.zeros(n_rows + 1, dtype=np.uint64)
    rp[1:] = np.cumsum(lens)
    n = int(rp[-1]) + 3
    d = Data(rp, r.permutation(n)[: int(rp[-1])].astype(np.uint32),
             r.standard_normal(int(rp[-1])).astype(np.float32),
             r.integers(1, 6, n_rows).astype(np.float32), n)
    cfg = _cfg(n, k, k0=0, lr=0.05, regs=(0, 0.01, 0.02))
    init = _rand_init(n, k, 5, stdev=0.3)
    p = _port(cfg, tuple(np.float32(x).astype(np.float64) for x in init))
    p.sgd_epoch(d, 0, 0.05, 1.0, 5.0)
    for ctas, rows, threads, variant in [(0, 0, 0, 0), (1, 32, 32, 0), (2, 64, 64, 1), (0, 128, 128, 2),
                                         (1, 0, 256, 3), (0, 512, 256, 1), (3, 32, 96, 0)]:
        l = make_learner(cfg, init, mode=MODE_HOGWILD)
        l.set_tuning(ctas_per_sm=ctas, rows_per_tile=rows, threads=threads, variant=variant)
        l.sgd_epoch(d)
        l.sgd_epoch(Data(np.zeros(1, dtype=np.uint64), np.zeros(0, np.uint32), np.zeros(0, np.float32),
                         np.zeros(0, np.float32), n))  # an empty data set between real ones
        l.pull_params()
        tol = 2e-6 * max(1, k // 8)  # fp32 sums over k*nnz terms vs the fp64 oracle
        np.testing.assert_allclose(l.fm.w, p.w, atol=tol, err_msg=str((ctas, rows, threads, variant)))
        np.testing.assert_allclose(l.fm.v, p.v, atol=tol, err_msg=str((ctas, rows, threads, variant)))
        l.close()


def _mf_gamma(u, G):
    u = np.asarray(u, dtype=np.float64)
    out = np.ones_like(u)
    m = u > 1e-6
    out[m] = -np.expm1(-G * u[m]) / (G * -np.expm1(-u[m]))
    return out


def test_peer_meanfield_two_contexts(built_lib):
    """fm_peer.cu mean-field combine: theta = theta0 + gamma_i * sum_g (theta_g - theta0).  Two replicas
    (two contexts, one device) train one epoch on their own shard from a common theta0, then combine:
    both end bit-identical, equal to a numpy restatement of the rule, and -- over a few epochs -- closer
    to the single-stream oracle than plain averaging is."""
    import ctypes as C
    full, te = synth.split_rows(synth.two_field(140_000, 1500, 1000, seed=5, planted_k=4), 120_000)
    n, k, lr, G = full.num_feature, 8, 0.01, 2
    half = full.num_cases // 2
    shards = [full.rows(0, half), full.rows(half, full.num_cases)]
    cfg = _cfg(n, k, lr=lr, mn=full.min_target, mx=full.max_target)
    init = (0.0, np.zeros(n), _rand_init(n, k, 7)[2])

    def pair():
        ls = [make_learner(cfg, init, mode=MODE_HOGWILD) for _ in range(G)]
        arr = (C.c_void_p * G)(*[l._ctx for l in ls])
        for rank, l in enumerate(ls):
            assert l.lib.fmb200_peer_attach_local(l._ctx, G, rank, arr) == 0, l.lib.fmb200_last_error()
        return ls

    def exchange(ls, fn):
        for l in ls:
            assert getattr(l.lib, fn)(l._ctx) == 0, l.lib.fmb200_last_error()
        for l in ls:
            assert l.lib.fmb200_sync(l._ctx) == 0

    # --- one exchange against the numpy restatement ---
    ls = pair()
    for l, d in zip(ls, shards):
        l.sgd_epoch(d)
        l.pull_params()
    th = [(np.float32(l.fm.w0), l.fm.w.astype(np.float32), l.fm.v.astype(np.float32)) for l in ls]
    w0_0, w_0, v_0 = np.float32(init[0]), init[1].astype(np.float32), init[2].astype(np.float32)
    cnt = np.mean([np.bincount(d.col, minlength=n) for d in shards], axis=0)
    rows = np.mean([d.num_cases for d in shards])
    hv = float(np.sum(v_0.astype(np.float64) ** 2) / n)
    g0 = _mf_gamma(np.array([lr * rows]), G)[0]
    gw, gv = _mf_gamma(lr * cnt, G), _mf_gamma(lr * hv * cnt, G)
    want_w0 = w0_0 + g0 * sum(t[0] - w0_0 for t in th)
    want_w = w_0 + gw * sum(t[1] - w_0 for t in th)
    want_v = v_0 + gv[None, :] * sum(t[2] - v_0 for t in th)
    exchange(ls, "fmb200_allreduce_meanfield")
    for l in ls:
        l.pull_params()
    a, b = ls
    assert a.fm.w0 == b.fm.w0 and np.array_equal(a.fm.w, b.fm.w) and np.array_equal(a.fm.v, b.fm.v)
    assert abs(a.fm.w0 - want_w0) < 1e-5
    np.testing.assert_allclose(a.fm.w, want_w, atol=2e-6)
    np.testing.assert_allclose(a.fm.v, want_v, atol=2e-6)
    for l in ls:
        l.close()

    # --- the sliced exchange (reduce-scatter + all-gather in one kernel, the path of C5-sized state) gives
    # the one-shot kernel's result: same per-element arithmetic; only h_V's partial sums are cut differently ---
    finals = {}
    for variant in (9, 8):  # 9 = one-shot, 8 = sliced
        ls = pair()
        for l in ls:
            l.set_tuning(variant=variant)
        for _ in range(3):
            for l, d in zip(ls, shards):
                l.sgd_epoch(d)
            exchange(ls, "fmb200_allreduce_meanfield")
        for l in ls:
            l.pull_params()
        assert ls[0].fm.w0 == ls[1].fm.w0 and np.array_equal(ls[0].fm.w, ls[1].fm.w) and \
            np.array_equal(ls[0].fm.v, ls[1].fm.v), "sliced replicas diverged" if variant == 8 else "one-shot"
        finals[variant] = (ls[0].fm.w0, ls[0].fm.w.copy(), ls[0].fm.v.copy())
        for l in ls:
            l.close()
    # the two exchanges cut h_V's partial sums differently: equal to rounding, carried through 3 epochs
    assert abs(finals[8][0] - finals[9][0]) < 2e-3
    assert np.sqrt(np.mean((finals[8][2] - finals[9][2]) ** 2)) < 2e-3

    # --- trajectories: single stream (oracle) vs mean-field vs plain averaging, 3 epochs ---
    p = _port(cfg, init)
    rmse = {}
    for name, fn in (("meanfield", "fmb200_allreduce_meanfield"), ("average", "fmb200_allreduce_mean")):
        ls = pair()
        for _ in range(3):
            for l, d in zip(ls, shards):
                l.sgd_epoch(d)
            exchange(ls, fn)
        rmse[name] = ls[0].evaluate(te)
        for l in ls:
            l.close()
    for _ in range(3):
        p.sgd_epoch(full, 0, lr, cfg["min_target"], cfg["max_target"])
    seq = p.metric(te, 0, cfg["min_target"], cfg["max_target"])
    print("\n[peer combine, 2 shards, 3 epochs] held-out RMSE: sequential %.4f  meanfield %.4f  average %.4f" %
          (seq, rmse["meanfield"], rmse["average"]))
    assert abs(rmse["meanfield"] - seq) < abs(rmse["average"] - seq)
    assert abs(rmse["meanfield"] - seq) < 0.03


def test_hogwild_rows_longer_than_the_staging_ring(built_lib):
    """ADVICE r01: any 32-row window with more than ~9.6k non-zeros used to fail the launch
    ('invalid configuration').  Such rows (dense libsvm / text data) now train with their ids and
    values read from global memory; a one-row epoch still equals one reference step."""
    r = np.random.default_rng(3)
    n, k, per_row = 4000, 8, 1200           # 32 rows x 1200 entries = 38k entries >> the ring
    rows = 96
    col = np.concatenate([np.sort(r.choice(n, size=per_row, replace=False)) for _ in range(rows)]).astype(np.uint32)
    d = Data(np.arange(rows + 1, dtype=np.uint64) * np.uint64(per_row), col,
             (r.standard_normal(rows * per_row) * 0.05).astype(np.float32),
             r.integers(1, 6, size=rows).astype(np.float32), n)
    cfg = _cfg(n, k, lr=0.001, mn=-10.0, mx=10.0)   # wide bounds: the clamp must not hide the learning
    init = _rand_init(n, k, 4)
    l = make_learner(cfg, init, mode=MODE_HOGWILD)
    got = l.predict(d, transform=False)
    want = _port(cfg, init).predict(d, 0, 0, 0, transform=False)
    assert np.max(np.abs(got - want)) < 5e-4
    before = l.evaluate(d)
    for _ in range(3):
        l.sgd_epoch(d)
    assert l.evaluate(d) < before
    # one row, one epoch == one fm_SGD step of the reference (fp32 rounding)
    one = d.rows(5, 6)
    m = make_learner(cfg, init, mode=MODE_HOGWILD)
    p = _port(cfg, init)
    m.sgd_epoch(one)
    p.sgd_epoch(one, 0, cfg["lr"], -10.0, 10.0)
    m.pull_params()
    np.testing.assert_allclose(m.fm.v, p.v, atol=2e-6)
    np.testing.assert_allclose(m.fm.w, p.w, atol=2e-6)
    l.close()
    m.close()


def _c2_learner(d, lr=0.01):
    fm = FmModel(d.num_feature, 8)
    fm.init_stdev = 0.1
    fm.init_numpy(42)
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate = 0, lr
    l.min_target, l.max_target = d.min_target, d.max_target
    l.push_hparams()
    return l


@pytest.mark.parametrize("zipf", [0.0, 1.0])
def test_rowlane_epochs_are_reproducible(zipf, built_lib):
    """The row-lane epoch (C2 shape, and C2 with Zipf ids through the in-warp merge) adds each window's
    steps to a fixed-point accumulator and folds them in after the window: two runs from the same state
    leave the same parameters, bit for bit, after the ramp epoch and two more."""
    d = synth.movielens_1m_shaped(seed=7, zipf=zipf)
    finals = []
    for _ in range(2):
        l = _c2_learner(d)
        for _ in range(3):
            l.sgd_epoch(d)
        assert l.epoch_config()["lanes_per_row"] == 1  # the row-lane kernel ran
        l.pull_params()
        finals.append((l.fm.w0, l.fm.w.copy(), l.fm.v.copy()))
        l.close()
    (a0, aw, av), (b0, bw, bv) = finals
    assert np.isfinite(av).all()
    assert a0 == b0 and np.array_equal(aw, bw) and np.array_equal(av, bv)


def test_rowlane_divergence_turns_the_state_into_nan(built_lib):
    """A step the fixed point cannot hold (here: learning rate 1e6) is not wrapped into a finite value:
    the fold turns the whole state into NaN, and a fresh set_params clears the condition."""
    d = synth.movielens_1m_shaped(seed=7, n_rows=200_000)
    l = _c2_learner(d, lr=1e6)
    l.sgd_epoch(d)
    l.pull_params()
    assert np.isnan(l.fm.w0) and np.isnan(l.fm.v).all()
    l.fm.init_numpy(42)
    l.push_params()
    l.learn_rate = 0.01
    l.push_hparams()
    l.sgd_epoch(d)
    l.pull_params()
    assert np.isfinite(l.fm.w0) and np.isfinite(l.fm.w).all() and np.isfinite(l.fm.v).all()
    l.close()
