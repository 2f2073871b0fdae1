"""GPU: the fp64 modes at every factor-width class they accept (k up to 256) against the oracle, and MCMC / ALS at
k up to 256 against the reference.

The oracle is pinned to the reference at these widths by tests/test_wide_k.py (tests/golden/reference/wide_k.npz).
Each check holds the bar its mode claims elsewhere (tests/test_parity_gpu.py, tests/test_ordered_gpu.py,
tests/test_sgda_gpu.py, tests/test_mcmc_sweep_gpu.py):
  * INORDER epoch (the one-warp row-at-a-time kernel, KF = 1, 2, 4, 8 factors per lane): bit-exact for regression,
    1e-12 for classification (device exp());
  * evaluate / predict (fm_predict64_kernel) in INORDER and ORDERED: bit-exact regression scores, metrics to 1e-12;
  * ORDERED epoch (GL = 1 .. 32 lanes per example): parameters to 1e-9 relative, RMSE to 1e-9 per epoch; the rows a
    tile of the shared-memory ring cannot hold run row-at-a-time, bit-exact;
  * SGDA (fm_sgda_epoch_kernel): bit-exact parameters and regularisation values, up to the group count the device's
    shared memory holds, and a refusal that names the need beyond it;
  * the MCMC e-terms bit-exact, and every MCMC / ALS iteration bit-identical to the reference's.
The data: ragged rows of 0-12 entries (rows of exactly 8 and 9: the edge of predict_row_exact's register cache at
k = 32 / 33), unsorted and repeated ids, real values, empty rows; a two-field one-hot set for ORDERED's
register-resident paths at k <= 8.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import make_learner
from libfm_b200 import MODE_INORDER, MODE_ORDERED, Data, FmError, synth
from oracle import Port
from test_mcmc_sweep_gpu import _first_difference, _start
from test_wide_k import (GPU_WIDTHS, MCMC_ITERS, SGD_REGS, WIDE_K_REF, GOLDEN, mcmc_cases, mcmc_record, ordered_shape,
                         sgd_sets, with_kf)

pytestmark = pytest.mark.gpu

PARAM_RTOL = 1e-9
ROW_AT_A_TIME = dict(lanes_per_row=32, slots=1, rows_per_tile=1, grid=1, block=32, smem_bytes=0)
CUDA_DEV_ATTR_MAX_SHARED_MEMORY_PER_BLOCK_OPTIN = 97


def _smem_optin(device=0):
    """cudaDeviceGetAttribute(cudaDevAttrMaxSharedMemoryPerBlockOptin): what one block may opt in to"""
    for name in ("libcudart.so.12", "libcudart.so", "/usr/local/cuda/lib64/libcudart.so"):
        try:
            rt = C.CDLL(name)
            break
        except OSError:
            continue
    else:
        raise RuntimeError("libcudart not found")
    v = C.c_int()
    assert rt.cudaDeviceGetAttribute(C.byref(v), CUDA_DEV_ATTR_MAX_SHARED_MEMORY_PER_BLOCK_OPTIN, device) == 0
    return v.value


def _two_field():
    d = synth.two_field(3000, 120, 80, seed=64)
    return Data(d.row_ptr, d.col, d.val, d.target, d.num_feature)


def _setup(d, k, mode, task=0, regs=(0.0, 0.0, 0.0), k0=1, k1=1, lr=0.01, seed=1):
    """a learner and the oracle from the same random state"""
    n = d.num_feature
    r = np.random.default_rng(seed)
    init = (float(r.standard_normal() * 0.1), r.standard_normal(n) * 0.1, r.standard_normal((k, n)) * 0.1)
    mn, mx = float(d.target.min()), float(d.target.max())
    cfg = dict(n=n, k=k, k0=k0, k1=k1, task=task, lr=lr, regs=np.array(regs, dtype=float), min_target=mn,
               max_target=mx)
    p = Port(n, k, k0, k1)
    p.set_params(*init)
    p.reg0, p.regw, p.regv = (float(x) for x in regs)
    return make_learner(cfg, init, mode=mode), p, mn, mx


def _cfg(l, keys=ROW_AT_A_TIME):
    c = l.epoch_config()
    return {key: c[key] for key in keys}


def _close(got, want):
    np.testing.assert_allclose(got, want, rtol=PARAM_RTOL, atol=PARAM_RTOL * 1e-3)


# ---- INORDER epoch: the one-warp row-at-a-time kernel --------------------------------------------------------

INORDER_CASES = [(k, "reg") for k in GPU_WIDTHS] + [(k, "cls") for k in GPU_WIDTHS] + \
                [(k, "no_bias_no_linear") for k in (33, 129, 200)]


@pytest.mark.parametrize("k,case", INORDER_CASES)
def test_inorder_epoch_matches_oracle(k, case, built_lib):
    task = 1 if case == "cls" else 0
    tr, _, _ = sgd_sets(task)
    k0 = k1 = 0 if case == "no_bias_no_linear" else 1
    regs = SGD_REGS if task == 0 else (0.0, 0.0, 0.0)
    l, p, mn, mx = _setup(tr, k, MODE_INORDER, task=task, regs=regs, k0=k0, k1=k1)
    for ep in range(2):
        l.sgd_epoch(tr)
        p.sgd_epoch(tr, task, 0.01, mn, mx)
        assert _cfg(l) == ROW_AT_A_TIME, l.epoch_config()
        l.pull_params()
        if task == 0:
            assert l.fm.w0 == p.w0.value, (k, ep)
            assert np.array_equal(l.fm.w, p.w) and np.array_equal(l.fm.v, p.v), (k, ep)
        else:
            assert abs(l.fm.w0 - p.w0.value) <= 1e-12
            np.testing.assert_allclose(l.fm.w, p.w, rtol=0, atol=1e-12)
            np.testing.assert_allclose(l.fm.v, p.v, rtol=0, atol=1e-12)
    print("\n[wide inorder k=%d %s] KF=%d %s" % (k, case, with_kf(k), l.epoch_config()))
    l.close()


# ---- evaluate / predict: fm_predict64_kernel -----------------------------------------------------------------

@pytest.mark.parametrize("mode", [MODE_INORDER, MODE_ORDERED], ids=["inorder", "ordered"])
@pytest.mark.parametrize("k", GPU_WIDTHS)
def test_evaluate_and_predict_match_oracle(k, mode, built_lib):
    for task in (0, 1):
        tr, _, te = sgd_sets(task)
        l, p, mn, mx = _setup(tr, k, mode, task=task, seed=2)
        for d in (tr, te):
            assert abs(l.evaluate(d) - p.metric(d, task, mn, mx)) <= 1e-12, (k, task)
            raw, out = l.predict(d, transform=False), l.predict(d, transform=True)
            assert np.array_equal(raw, p.predict(d, task, mn, mx, transform=False)), (k, task)
            if task == 0:
                assert np.array_equal(out, p.predict(d, task, mn, mx, transform=True)), (k, task)
            else:
                np.testing.assert_allclose(out, p.predict(d, task, mn, mx, transform=True), rtol=0, atol=1e-12)
        l.close()


# ---- ORDERED epoch: GL lanes x 8 factors per example ---------------------------------------------------------

ORDERED_CASES = [(k, "ragged", t) for k in GPU_WIDTHS for t in ("default", "variant1")] + \
                [(k, "ragged", "threads128") for k in GPU_WIDTHS if ordered_shape(k)[0] <= 4] + \
                [(k, "two_field", t) for k in (5, 7, 8) for t in ("default", "variant1", "threads128")] + \
                [(k, "cls", "default") for k in (33, 130, 256)]


@pytest.mark.parametrize("k,data,tuning", ORDERED_CASES)
def test_ordered_epoch_matches_oracle(k, data, tuning, built_lib):
    task = 1 if data == "cls" else 0
    tr = _two_field() if data == "two_field" else sgd_sets(task)[0]
    regs = SGD_REGS if data == "ragged" else (0.0, 0.0, 0.0)
    l, p, mn, mx = _setup(tr, k, MODE_ORDERED, task=task, regs=regs)
    if tuning == "variant1":
        l.set_tuning(variant=1)
    elif tuning == "threads128":
        l.set_tuning(threads=128)
    gl = ordered_shape(k)[0]
    for ep in range(2):
        l.sgd_epoch(tr)
        p.sgd_epoch(tr, task, 0.01, mn, mx)
        c = l.epoch_config()
        assert c["lanes_per_row"] == gl and c["smem_bytes"] > 0, c   # the ORDERED kernel ran, not the fallback
        got, want = l.evaluate(tr), p.metric(tr, task, mn, mx)
        assert abs(got - want) <= (1e-9 if task == 0 else 0.0), (k, ep, got, want)
    l.pull_params()
    if task == 0:
        _close(l.fm.w0, p.w0.value)
        _close(l.fm.w, p.w)
        _close(l.fm.v, p.v)
    else:
        np.testing.assert_allclose(l.fm.v, p.v, rtol=1e-9, atol=1e-12)
    print("\n[wide ordered k=%d %s %s] GL=%d %s" % (k, data, tuning, gl, l.epoch_config()))
    l.close()


@pytest.mark.parametrize("k_narrow,k_wide", [(64, 128), (128, 256)])
def test_ordered_zero_factors_leave_the_narrower_class_bit_exact(k_narrow, k_wide, built_lib):
    """A factor that starts at 0 stays 0 and adds exactly 0 to every score.  So the GL = 2 G kernel on a model whose
    factors beyond k_narrow are zero must reproduce the GL = G kernel on the narrow model bit for bit: the same
    per-lane sums, the extra lanes' zeros added first in the lane reduction.  This holds without the bias and the
    linear terms only (their chain and lane split depend on the tile and GL), and it pins the wide class at a bar the
    oracle cannot: any change to its arithmetic, however small, shows."""
    tr = sgd_sets(0)[0]
    narrow, p, mn, mx = _setup(tr, k_narrow, MODE_ORDERED, regs=SGD_REGS, k0=0, k1=0, seed=5)
    narrow.pull_params()
    v = np.zeros((k_wide, tr.num_feature))
    v[:k_narrow] = narrow.fm.v
    cfg = dict(n=tr.num_feature, k=k_wide, k0=0, k1=0, task=0, lr=0.01, regs=np.array(SGD_REGS), min_target=mn,
               max_target=mx)
    wide = make_learner(cfg, (0.0, narrow.fm.w.copy(), v), mode=MODE_ORDERED)
    for ep in range(2):
        narrow.sgd_epoch(tr)
        wide.sgd_epoch(tr)
        assert narrow.epoch_config()["lanes_per_row"] * 2 == wide.epoch_config()["lanes_per_row"]
        narrow.pull_params()
        wide.pull_params()
        assert not wide.fm.v[k_narrow:].any(), ep
        diff = np.abs(wide.fm.v[:k_narrow] - narrow.fm.v)
        assert np.array_equal(wide.fm.v[:k_narrow], narrow.fm.v), (ep, np.unravel_index(diff.argmax(), diff.shape))
        p.sgd_epoch(tr, 0, 0.01, mn, mx)
        _close(narrow.fm.v, p.v)
    print("\n[wide ordered k=%d in GL=%d as k=%d in GL=%d] %s" % (k_narrow, wide.epoch_config()["lanes_per_row"],
                                                                  k_narrow, narrow.epoch_config()["lanes_per_row"],
                                                                  wide.epoch_config()))
    narrow.close()
    wide.close()


def _ord_smem_bytes(tr_rows, te, rs):
    """fm_ordered.cuh::ord_smem_bytes: header | 3 CSR stages | 3 record buffers of te entries x rs doubles"""
    rp = ((tr_rows + 2) * 8 + 15) & ~15
    row = ((tr_rows + 4) * 4 + 15) & ~15
    csr = rp + 2 * row + 16 * te + ((te + 15) & ~15)
    return 5632 + 3 * csr + 3 * te * rs * 8


def _longest_ring_row(k, limit):
    """fm_ordered.cu::ordered_geometry at one row per tile (the smallest tile it tries): the longest row whose
    tile of max_row_nnz + 6 entries fits the shared-memory ring.  A longer row leaves no tile that fits."""
    rs = k + (k & 1) + 2
    fits = lambda n_entries: _ord_smem_bytes(1, ((n_entries + 6 + 3) & ~3) + 4, rs) <= limit  # noqa: E731
    L = 0
    while fits(L + 1):
        L += 1
    return L


def _with_long_row(d, length, at, seed):
    """d with one row of `length` entries inserted before row `at` (a repeated id, values != 1)"""
    r = np.random.default_rng(seed)
    col = r.integers(0, d.num_feature, size=length).astype(np.uint32)
    col[-1] = col[0]
    val = (r.standard_normal(length) * 0.5).astype(np.float32)
    a = int(d.row_ptr[at])
    cols = np.concatenate([d.col[:a], col, d.col[a:]])
    vals = np.concatenate([d.val[:a], val, d.val[a:]])
    sizes = np.diff(d.row_ptr.astype(np.int64))
    sizes = np.concatenate([sizes[:at], [length], sizes[at:]])
    rp = np.zeros(sizes.size + 1, np.uint64)
    rp[1:] = np.cumsum(sizes)
    tg = np.concatenate([d.target[:at], [3.0], d.target[at:]]).astype(np.float32)
    return Data(rp, cols, vals, tg, d.num_feature)


def _tile_span32(d):
    """fm_predict.cu's span of a 32-row tile: 4-entry-aligned entries from its first row to past its last"""
    rp = d.row_ptr.astype(np.int64)
    starts = np.arange(0, d.num_cases, 32)
    ends = np.minimum(starts + 32, d.num_cases)
    return int((((rp[ends] + 3) & ~3) - (rp[starts] & ~3)).max())


@pytest.mark.parametrize("over", [0, 1], ids=["longest_that_fits", "one_entry_longer"])
def test_ordered_ring_boundary_at_k256(over, built_lib):
    """At k = 256 a row of L entries still fits one tile of the ring and runs in the GL = 32 kernel (1e-9); a row
    of L + 1 fits no tile, and the epoch runs row-at-a-time instead, bit-exact.  L comes from the device's
    opt-in shared-memory limit."""
    k = 256
    limit = _smem_optin()
    L = _longest_ring_row(k, limit)
    tr = _with_long_row(sgd_sets(0)[0], L + over, 500, seed=65)
    assert _tile_span32(tr) >= L + over + 6   # the one-row tile is sized by the row, not by its 32-row tile
    l, p, mn, mx = _setup(tr, k, MODE_ORDERED, regs=SGD_REGS)
    for ep in range(2):
        l.sgd_epoch(tr)
        p.sgd_epoch(tr, 0, 0.01, mn, mx)
        c = l.epoch_config()
        l.pull_params()
        if over:
            assert _cfg(l) == ROW_AT_A_TIME, c
            assert l.fm.w0 == p.w0.value and np.array_equal(l.fm.w, p.w) and np.array_equal(l.fm.v, p.v), ep
        else:
            assert c["lanes_per_row"] == 32 and c["smem_bytes"] > 0, c
            assert abs(l.evaluate(tr) - p.metric(tr, 0, mn, mx)) <= 1e-9, ep
            _close(l.fm.w0, p.w0.value)
            _close(l.fm.w, p.w)
            _close(l.fm.v, p.v)
    print("\n[wide ordered k=256, a row of %d entries, opt-in limit %d B] %s" % (L + over, limit, l.epoch_config()))
    l.close()


# ---- SGDA: fm_sgda_epoch_kernel -------------------------------------------------------------------------------

def _sgda_run(k, groups, epochs=3):
    tr, va, _ = sgd_sets(0)
    n = tr.num_feature
    group = (np.arange(n) % groups).astype(np.uint32)
    mn, mx = float(tr.target.min()), float(tr.target.max())
    init = (0.0, np.zeros(n), np.random.default_rng(3).standard_normal((k, n)) * 0.1)
    cfg = dict(n=n, k=k, k0=1, k1=1, task=0, lr=0.01, regs=np.zeros(3), min_target=mn, max_target=mx)
    p = Port(n, k)
    p.set_params(*init)
    p.sgda_begin(group)
    l = make_learner(cfg, init, mode=MODE_INORDER)
    l.sgda_begin(group if groups > 1 else None)
    for e in range(epochs):
        l.sgda_epoch(tr, va, e > 0)
        p.sgda_epoch(tr, va, 0, 0.01, mn, mx, e > 0)
    l.pull_params()
    reg_w, reg_v = l.sgda_reg()
    assert l.fm.w0 == p.w0.value and np.array_equal(l.fm.w, p.w) and np.array_equal(l.fm.v, p.v), (k, groups)
    assert np.array_equal(reg_w, p.reg_w) and np.array_equal(reg_v, p.reg_v), (k, groups)
    assert reg_v.max() > 0
    print("\n[wide sgda k=%d, %d groups] KF=%d %s" % (k, groups, with_kf(k), l.epoch_config()))
    l.close()


@pytest.mark.parametrize("groups", [1, 3])
@pytest.mark.parametrize("k", [33, 129, 256])
def test_sgda_matches_oracle(k, groups, built_lib):
    _sgda_run(k, groups)


def test_sgda_group_ceiling_at_k256(built_lib):
    """G groups keep 8 G (2 + 3k) bytes in shared memory: the most the device allows runs bit-exact, one more is
    refused with the need and the limit"""
    k = 256
    limit = _smem_optin()
    per_group = 8 * (2 + 3 * k)
    g_max = limit // per_group
    _sgda_run(k, g_max, epochs=2)
    tr, _, _ = sgd_sets(0)
    n = tr.num_feature
    l, _, _, _ = _setup(tr, k, MODE_INORDER)
    with pytest.raises(FmError, match=r"SGDA with %d groups at num_factor = 256 needs %d bytes of shared memory.*"
                                      r"allows %d: use at most %d groups" % (g_max + 1, (g_max + 1) * per_group,
                                                                             limit, g_max)):
        l.sgda_begin((np.arange(n) % (g_max + 1)).astype(np.uint32))
    print("\n[wide sgda k=256] opt-in limit %d B: at most %d groups" % (limit, g_max))
    l.close()


# ---- MCMC / ALS ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", GPU_WIDTHS)
def test_mcmc_eterms_match_oracle(k, built_lib):
    tr, _, te = sgd_sets(0)
    l, p, _, _ = _setup(tr, k, MODE_INORDER, seed=4)
    for d in (tr, te):
        assert np.array_equal(l.mcmc_eterms(d), p.mcmc_eterms(d)), k
    l.close()


@pytest.mark.parametrize("name", sorted(mcmc_cases()))
def test_mcmc_als_iterations_bit_identical_to_reference(name, built_lib):
    assert int(name.split("_")[0][1:]) in WIDE_K_REF
    z = mcmc_record(np.load(GOLDEN), name)
    l, tr, te = _start(z, name)
    for t in range(MCMC_ITERS):
        m, cnt = l.mcmc_iteration()
        bad = _first_difference(z, name, t, l, te, m, cnt)
        assert bad is None, "%s: iteration %d: %s differs from the reference" % (name, t, bad)
    print("\n[wide %s] %d runs" % (name, l.mcmc_runs()))
    l.close()
