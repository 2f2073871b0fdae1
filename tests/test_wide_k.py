"""CPU: the fp64 learners at the factor widths the one-warp and ORDERED kernels are compiled for beyond k = 128.

tests/golden/reference/wide_k.npz (scripts/make_wide_golden.py) holds what the reference itself computes at
k in WIDE_K_REF on the seeded data sets below: 2 SGD epochs (regression, classification), predict, 3 SGDA epochs
over 3 attribute groups, the MCMC e-terms, and 4 iterations of MCMC and of ALS.  Here the oracle (oracle/fm_oracle.c,
fm_oracle_sgda.c) must reproduce every SGD, SGDA and e-term record bit for bit; that makes it a valid yardstick for
tests/test_wide_k_gpu.py at those widths, which also replays the MCMC / ALS records on the GPU.

The second half restates the kernels' width classes -- `with_kf` (fmb200_internal.h: KF factors per lane of
fm_inorder.cu's one-warp kernels) and `ordered_shape` (fm_ordered.cu: GL lanes x KF consecutive factors per
example) -- and checks that GPU_WIDTHS reaches every class with odd and even k, a partially filled and an empty
factor slot.
"""
import hashlib
import os

import numpy as np
import pytest

from conftest import digest
from libfm_b200 import synth
from oracle import Port

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "wide_k.npz")

WIDE_K_REF = (33, 97, 129, 200, 256)
SGD_EPOCHS, SGDA_EPOCHS, MCMC_ITERS = 2, 3, 4
SGD_LR, SGDA_LR = 0.01, 0.01
SGD_REGS = (0.01, 0.02, 0.03)   # regression; classification runs unregularised
SGDA_GROUPS = 3
ETERM_W0 = 0.25

# the widths tests/test_wide_k_gpu.py runs
GPU_WIDTHS = (5, 7, 8, 9, 16, 17, 31, 32, 33, 63, 64, 65, 96, 97, 127, 129, 130, 160, 200, 255, 256)


# ---- seeded inputs (shared with scripts/make_wide_golden.py and tests/test_wide_k_gpu.py) ---------------------

def sgd_sets(task=0):
    """train / validation / test: ragged rows of 0-12 entries (rows of exactly 8 and 9 among them), unsorted and
    repeated ids, real values, empty rows.  Classification maps ratings 4 and 5 to +1, the rest to -1."""
    d = synth.ragged(1600, 240, 12, seed=61)
    tr, rest = synth.split_rows(d, 1000)
    va, te = synth.split_rows(rest, 300)
    if task == 1:
        for s in (tr, va, te):
            s.target = np.where(s.target >= 4, 1.0, -1.0).astype(np.float32)
    return tr, va, te


def sgda_groups(n):
    return (np.arange(n) % SGDA_GROUPS).astype(np.uint32)


def eterm_w(n):
    return np.random.default_rng(62).standard_normal(n) * 0.1


def mcmc_sets():
    """train / test of the MCMC and ALS cases: ragged as above on 150 features, values scaled down (at unit
    scale ALS with 38 400 factors on 800 cases overflows within two iterations)"""
    d = synth.ragged(1000, 150, 12, seed=63)
    d.val = (d.val * 0.3).astype(np.float32)
    tr, te = synth.split_rows(d, 800)
    return tr, te


def mcmc_cases():
    """name -> dict(k, sample, group, per_group, reg0, wl, vl, seed) -- MCMC with one group and no
    regularisation prior (libfm.cpp:331), ALS with two interleaved groups and per-group values (:349-364)"""
    tr, _ = mcmc_sets()
    n = tr.num_feature
    out = {}
    for k in WIDE_K_REF:
        out["k%d_mcmc" % k] = dict(k=k, sample=1, group=np.zeros(n, np.uint32), per_group=np.array([n], np.uint32),
                                  reg0=0.0, wl=np.zeros(1), vl=np.zeros((1, k)), seed=7)
        grp = (np.arange(n) % 2).astype(np.uint32)
        out["k%d_als" % k] = dict(k=k, sample=0, group=grp, per_group=np.bincount(grp, minlength=2).astype(np.uint32),
                                 reg0=0.1, wl=np.array([0.2, 0.3]),
                                 vl=np.repeat(np.array([[0.4], [0.5]]), k, axis=1), seed=7)
    return out


def mcmc_record(z, name):
    """One MCMC / ALS record of wide_k.npz with its inputs regenerated, keyed as tests/golden/reference/mcmc.npz is
    (the form tests/test_mcmc_sweep_gpu.py replays)."""
    tr, te = mcmc_sets()
    c = mcmc_cases()[name]
    rec = {key[len(name) + 1:]: z[key] for key in z.files if key.startswith(name + "/")}
    rec.update(tr_row_ptr=tr.row_ptr, tr_col=tr.col, tr_val=tr.val, tr_target=tr.target, te_row_ptr=te.row_ptr,
               te_col=te.col, te_val=te.val, te_target=te.target, group=c["group"], per_group=c["per_group"],
               wl=c["wl"], vl=c["vl"])
    return {"%s/%s" % (name, key): v for key, v in rec.items()}


def input_digests():
    """digests of every generated input: a failing test then tells a changed generator from a changed result"""
    out = {}
    for tag, sets in (("sgd0", sgd_sets(0)), ("sgd1", sgd_sets(1)), ("mcmc", mcmc_sets())):
        for i, d in enumerate(sets):
            out["%s_%d" % (tag, i)] = "".join(digest(a) for a in (d.row_ptr, d.col, d.val, d.target))
    return out


def fp64_digest(a) -> str:
    """the digest of mcmc.npz (scripts/make_mcmc_golden.py): SHA-256 of the float64 bytes"""
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()


# ---- the oracle against the reference's records -------------------------------------------------------------

@pytest.fixture(scope="module")
def wide():
    return np.load(GOLDEN)


def test_inputs_are_the_recorded_ones(wide):
    for key, want in input_digests().items():
        assert str(wide["inputs/" + key]) == want, key
    tr, _, _ = sgd_sets()
    sizes = np.diff(tr.row_ptr.astype(np.int64))
    assert {0, 8, 9, 12} <= set(sizes.tolist())


@pytest.mark.parametrize("task", [0, 1])
@pytest.mark.parametrize("k", WIDE_K_REF)
def test_port_sgd_and_predict_bit_identical_to_reference(k, task, wide):
    tr, _, te = sgd_sets(task)
    n, mn, mx = tr.num_feature, float(tr.target.min()), float(tr.target.max())
    p = Port(n, k)
    p.init(42, 0.0, 0.1)
    if task == 0:
        p.reg0, p.regw, p.regv = SGD_REGS
    key = "sgd/%d/%d/" % (k, task)
    for e in range(SGD_EPOCHS):
        p.sgd_epoch(tr, task, SGD_LR, mn, mx)
        # the learner reports its metrics as it prints them, to 6 significant digits
        assert float("%g" % p.metric(tr, task, mn, mx)) == wide[key + "metric_train"][e]
        assert float("%g" % p.metric(te, task, mn, mx)) == wide[key + "metric_test"][e]
    assert p.w0.value == wide[key + "w0"]
    assert digest(p.w) + digest(p.v) == wide[key + "wv"]
    assert digest(p.predict(te, task, mn, mx, True)) == wide[key + "pred"]


@pytest.mark.parametrize("k", WIDE_K_REF)
def test_port_sgda_bit_identical_to_reference(k, wide):
    tr, va, _ = sgd_sets(0)
    n, mn, mx = tr.num_feature, float(tr.target.min()), float(tr.target.max())
    p = Port(n, k)
    p.init(42, 0.0, 0.1)
    p.sgda_begin(sgda_groups(n))
    for e in range(SGDA_EPOCHS):
        p.sgda_epoch(tr, va, 0, SGDA_LR, mn, mx, e > 0)
    key = "sgda/%d/" % k
    assert p.w0.value == wide[key + "w0"]
    assert digest(p.w) + digest(p.v) == wide[key + "wv"]
    assert np.array_equal(p.reg_w, wide[key + "reg_w"])
    assert digest(p.reg_v) == wide[key + "reg_v"]
    assert p.reg_v.max() > 0  # the lambda-steps moved the factor regularisation


@pytest.mark.parametrize("k", WIDE_K_REF)
def test_port_eterms_bit_identical_to_reference(k, wide):
    tr, _, _ = sgd_sets(0)
    n = tr.num_feature
    p = Port(n, k)
    p.init(42, 0.0, 0.1)
    p.set_params(ETERM_W0, eterm_w(n), p.v)
    assert digest(p.mcmc_eterms(tr)) == wide["eterm/%d" % k]


def test_mcmc_records_are_complete(wide):
    """every MCMC / ALS case has its per-iteration record, and the runs moved the model"""
    for name, c in mcmc_cases().items():
        z = mcmc_record(wide, name)
        cfg = z[name + "/cfg"]
        assert int(cfg[1]) == c["k"] and int(cfg[5]) == c["sample"]
        for t in range(MCMC_ITERS):
            for f in ("w0", "w", "v", "hyper", "counters", "pred_this", "pred_sum_all", "pred_sum_all_but5", "line"):
                assert "%s/%d/%s" % (name, t, f) in z
        assert str(z[name + "/0/v"]) != str(z["%s/%d/v" % (name, MCMC_ITERS - 1)])
        assert not z["%s/%d/counters" % (name, MCMC_ITERS - 1)].any()  # no NaN or Inf draw was skipped


# ---- the kernels' width classes -------------------------------------------------------------------------------

def with_kf(k):
    """with_kf<8> (fmb200_internal.h): factors per lane of the one-warp kernels (lane l owns l, l + 32, ...)"""
    assert 0 <= k <= 256
    kf = (k + 31) // 32
    return 1 if kf <= 1 else 2 if kf <= 2 else 4 if kf <= 4 else 8


def ordered_shape(k):
    """fm_ordered.cu::ordered_shape: (GL lanes per example, KF consecutive factors per lane)"""
    if k <= 8:
        return 1, (1 if k <= 1 else 2 if k <= 2 else 4 if k <= 4 else 8)
    g = 2
    while g * 8 < k:
        g <<= 1
    return g, 8


def inorder_slots(k):
    """(full, partial, empty) factor slots j of the one-warp kernels: slot j holds factors 32 j .. 32 j + 31"""
    kf = with_kf(k)
    filled = [min(32, max(0, k - 32 * j)) for j in range(kf)]
    return filled.count(32), sum(0 < c < 32 for c in filled), filled.count(0)


def ordered_lanes(k):
    """(full, partial, empty) lanes of one ORDERED example: lane g holds factors KF g .. KF g + KF - 1"""
    gl, kf = ordered_shape(k)
    filled = [min(kf, max(0, k - kf * g)) for g in range(gl)]
    return filled.count(kf), sum(0 < c < kf for c in filled), filled.count(0)


def test_width_classes_restate_the_kernels():
    assert [with_kf(k) for k in (1, 32, 33, 64, 65, 128, 129, 256)] == [1, 1, 2, 2, 4, 4, 8, 8]
    assert [ordered_shape(k) for k in (1, 2, 3, 5, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 256)] == [
        (1, 1), (1, 2), (1, 4), (1, 8), (1, 8), (2, 8), (2, 8), (4, 8), (4, 8), (8, 8), (8, 8), (16, 8), (16, 8),
        (32, 8), (32, 8)]
    assert inorder_slots(200) == (6, 1, 1)
    assert ordered_lanes(200) == (25, 0, 7)
    assert ordered_lanes(130) == (16, 1, 15)


def test_gpu_widths_reach_every_class_and_edge():
    by_kf, by_gl = {}, {}
    for k in GPU_WIDTHS:
        by_kf.setdefault(with_kf(k), []).append(k)
        by_gl.setdefault(ordered_shape(k)[0], []).append(k)
    assert sorted(by_kf) == [1, 2, 4, 8]
    assert sorted(by_gl) == [1, 2, 4, 8, 16, 32]
    assert set(WIDE_K_REF) <= set(GPU_WIDTHS)
    for kf, ks in by_kf.items():
        assert {k % 2 for k in ks} == {0, 1}, kf
        assert any(inorder_slots(k)[1] for k in ks), kf                      # a partly filled slot
        if kf > 2:  # k > 16 KF is needed, so KF <= 2 never has an idle slot
            assert any(inorder_slots(k)[2] for k in ks), kf                  # a slot with no factor at all
    for gl, ks in by_gl.items():
        assert {k % 2 for k in ks} == {0, 1}, gl                             # odd k pads the record (kw = k + 1)
        assert any(ordered_lanes(k)[1] for k in ks), gl                       # a lane with fewer than KF factors
        if gl > 2:  # k > 4 GL is needed, so GL = 2 never has an idle lane
            assert any(ordered_lanes(k)[2] for k in ks), gl                   # a lane with no factor
    # the one-warp kernels' register cache (rows of <= 8 entries at k <= 32) at its edge widths
    assert 32 in GPU_WIDTHS and 33 in GPU_WIDTHS
