"""CPU: pin the plain-C restatement (oracle/fm_oracle.c) against what the REFERENCE
produced: the golden vectors of tests/golden/*.npz (scripts/make_golden.py) and the
reference's results stored in tests/golden/reference/outputs.npz (scripts/make_ref_golden.py)."""
import ctypes as C

import numpy as np
import pytest

from conftest import GOLDEN_CASES, digest, load_golden
from libfm_b200 import synth
from oracle import Port


def _port_from_golden(z):
    p = Port(int(z["n"]), int(z["k"]), int(z["k0"]), int(z["k1"]))
    p.set_params(float(z["w0_init"]), z["w_init"], z["v_init"])
    p.reg0, p.regw, p.regv = [float(x) for x in z["regs"]]
    return p


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_port_init_matches_reference_draw_order(name):
    z, tr, te = load_golden(name)
    p = Port(int(z["n"]), int(z["k"]))
    p.init(int(z["seed"]), 0.0, float(z["init_stdev"]))
    assert p.w0.value == 0.0 and not p.w.any()
    assert np.array_equal(p.v, z["v_init"])  # bit-exact: same rand() stream, same order


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_port_epochs_bit_exact_vs_golden(name):
    z, tr, te = load_golden(name)
    p = _port_from_golden(z)
    task, lr = int(z["task"]), float(z["lr"])
    mn, mx = float(z["min_target"]), float(z["max_target"])
    for e in range(int(z["epochs"])):
        p.sgd_epoch(tr, task, lr, mn, mx)
        assert p.metric(tr, task, mn, mx) == z["metric_train"][e]
        assert p.metric(te, task, mn, mx) == z["metric_test"][e]
    assert p.w0.value == float(z["w0"])
    assert np.array_equal(p.w, z["w"])
    assert np.array_equal(p.v, z["v"])
    assert np.array_equal(p.predict(te, task, mn, mx, True), z["pred_test"])


def test_port_vs_live_reference_c1_shape(ref_golden):
    tr = synth.plumbing_10k()
    te = synth.plumbing_10k(seed=99, n_rows=2000)
    n, k = max(tr.num_feature, te.num_feature), 8
    port = Port(n, k)
    port.init(42, 0.0, 0.1)
    for _ in range(2):
        port.sgd_epoch(tr, 0, 0.01, tr.min_target, tr.max_target)
    assert port.w0.value == ref_golden["c1_w0"]
    assert digest(port.w) + digest(port.v) == ref_golden["c1_wv_sha"]
    assert port.metric(te, 0, tr.min_target, tr.max_target) == ref_golden["c1_test_metric"]


def test_port_rng_matches_reference(ref_golden):
    p = Port(1, 1)
    p.lib.fmo_srand(C.c_long(123))
    b = [p.lib.fmo_ran_gaussian() for _ in range(1000)]
    assert b == ref_golden["rng_gauss_123"].tolist()


PREDICT_ROW_CASES = [([], []), ([3], [2.5]), ([3, 3], [1.0, -2.0]), ([0, 19, 7], [0.5, 1.5, -1.0])]


def test_port_predict_row_edge_cases(ref_golden):
    n, k = 20, 3
    port = Port(n, k)
    port.set_params(0.25, np.linspace(-1, 1, n), ref_golden["row_v"])
    for i, (col, val) in enumerate(PREDICT_ROW_CASES):
        pp, sp, ssp = port.predict_row(col, val)
        assert pp == ref_golden["row_p"][i]
        assert np.array_equal(sp, ref_golden["row_s"][i]) and np.array_equal(ssp, ref_golden["row_ss"][i])


def _ragged_short_rows(n_rows, n_feat, seed, dup_every=0):
    """rows of 0..4 entries with real-valued x, Zipf-ish ids (many collisions inside 32 rows),
    optionally a repeated id inside a row every `dup_every` rows."""
    from libfm_b200.model import Data
    r = np.random.default_rng(seed)
    sizes = r.integers(0, 5, size=n_rows)
    row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
    row_ptr[1:] = np.cumsum(sizes)
    nnz = int(row_ptr[-1])
    p = 1.0 / np.arange(1, n_feat + 1) ** 0.8
    col = r.choice(n_feat, size=nnz, p=p / p.sum()).astype(np.uint32)
    if dup_every:
        for i in range(0, n_rows, dup_every):
            b, e = int(row_ptr[i]), int(row_ptr[i + 1])
            if e - b >= 2:
                col[e - 1] = col[b]
    val = (r.standard_normal(nnz) * 0.7).astype(np.float32)
    y = r.integers(1, 6, size=n_rows).astype(np.float32)
    return Data(row_ptr, col, val, y, n_feat)


@pytest.mark.parametrize("case", ["c2_shape", "zipf", "ragged", "dups", "classification", "no_bias", "k3_reg"])
def test_wavefront_schedule_is_sequentially_equivalent(case):
    """oracle/wavefront_emul.c replays the schedule of fm_sgd_inorder_wavefront_kernel (conflict-free
    prefixes of 32 examples, addends formed in parallel, bias chain in order, cached scatter).  It must
    leave w0 / w / V bit-identical to the sequential loop -- otherwise the kernel's claim is void."""
    task, k, k0, k1, regs = 0, 8, 1, 1, (0.0, 0.0, 0.0)
    if case == "c2_shape":
        tr = synth.two_field(60_000, 6040, 3706, seed=3)
    elif case == "zipf":
        tr = synth.two_field(40_000, 600, 400, seed=4, zipf=1.1)
    elif case == "ragged":
        tr = _ragged_short_rows(30_000, 500, seed=5)
    elif case == "dups":
        tr = _ragged_short_rows(30_000, 300, seed=6, dup_every=7)
    elif case == "classification":
        tr = synth.two_field(30_000, 800, 500, seed=7)
        tr.target[:] = np.where(tr.target > 3, 1.0, -1.0)
        task = 1
    elif case == "no_bias":
        tr = synth.two_field(30_000, 800, 500, seed=8)
        k0, k1 = 0, 0
    else:
        tr = _ragged_short_rows(20_000, 400, seed=9)
        k, regs = 3, (0.01, 0.02, 0.03)
    n = tr.num_feature
    a, b = Port(n, k, k0, k1), Port(n, k, k0, k1)
    a.init(11, 0.0, 0.1)
    b.set_params(a.w0.value, a.w, a.v)
    a.reg0, a.regw, a.regv = regs
    b.reg0, b.regw, b.regv = regs
    mn, mx = float(tr.target.min()), float(tr.target.max())
    for _ in range(2):
        a.sgd_epoch(tr, task, 0.02, mn, mx)
        steps = b.sgd_epoch_wavefront(tr, task, 0.02, mn, mx)
        assert steps > 0
        assert a.w0.value == b.w0.value
        assert np.array_equal(a.w, b.w) and np.array_equal(a.v, b.v)
    # the schedule is worth having only if prefixes are long: report-level sanity
    if case == "c2_shape":
        assert tr.num_cases / steps > 12, tr.num_cases / steps


def test_wavefront_schedule_refuses_ineligible_shapes():
    tr = synth.multi_field(2000, 6, 300, seed=1)  # 6 entries per row > 4
    p = Port(tr.num_feature, 8)
    assert p.sgd_epoch_wavefront(tr, 0, 0.01, 1.0, 5.0) == 0
    q = Port(100, 16)
    assert q.sgd_epoch_wavefront(synth.two_field(100, 50, 50, seed=1), 0, 0.01, 1.0, 5.0) == 0


MCMC_CASES = ["ragged_unsorted_dups", "two_field", "no_linear", "k0_only"]


def mcmc_case(case):
    """data, n, k, k0, k1, w0, w of one e-term case"""
    k, k0, k1 = 6, 1, 1
    if case == "ragged_unsorted_dups":
        d = synth.ragged(4000, 300, 11, seed=31)   # unsorted ids, repeated ids inside rows, empty rows
    elif case == "two_field":
        d = synth.two_field(6000, 400, 300, seed=32)
        k = 16
    elif case == "no_linear":
        d = synth.ragged(2000, 200, 6, seed=33)
        k1 = 0
    else:
        d = synth.ragged(2000, 200, 6, seed=34)
        k = 0
    n = d.num_feature
    r = np.random.default_rng(5)
    return d, n, k, k0, k1, 0.25, r.standard_normal(n) * 0.1


@pytest.mark.parametrize("case", MCMC_CASES)
def test_mcmc_eterm_port_is_bit_identical_to_reference(case, ref_golden):
    """oracle/fm_oracle.c::fmo_mcmc_eterms against the reference's own e-term pass
    (fm_learn_mcmc::predict_data_and_write_to_eterms, run through its transposed copy of the data)."""
    d, n, k, k0, k1, w0, w = mcmc_case(case)
    p = Port(n, k, k0, k1)
    p.init(42, 0.0, 0.1)  # the reference's draw of V for seed 42
    p.set_params(w0, w, p.v)
    got = p.mcmc_eterms(d)
    assert digest(got) == ref_golden["mcmc_%s_sha" % case]
    # same quantity as fm_model::predict, different association: equal to rounding only
    assert np.max(np.abs(got - p.predict(d, 0, 0, 0, transform=False))) < 1e-12


def sgda_case(task):
    """train, validation, test, attribute groups, n, k, min/max target of one SGDA case"""
    full = synth.two_field(9000, 300, 200, seed=4, planted_k=3)
    tr, rest = synth.split_rows(full, 6000)
    va, te = synth.split_rows(rest, 2000)
    if task == 1:
        for d in (tr, va, te):
            d.target[:] = np.where(d.target > 3, 1.0, -1.0)
    n, k = full.num_feature, 5
    group = (np.arange(n) >= 300).astype(np.uint32)
    return tr, va, te, group, n, k, float(tr.target.min()), float(tr.target.max())


@pytest.mark.parametrize("task", [0, 1])
def test_sgda_port_is_bit_identical_to_reference(task, ref_golden):
    """oracle/fm_oracle_sgda.c against the reference's own fm_learn_sgd_element_adapt_reg::learn
    (4 epochs: the first without lambda-steps, validation cursor wrapping, two attribute groups)."""
    tr, va, te, group, n, k, mn, mx = sgda_case(task)
    p = Port(n, k)
    p.init(42, 0.0, 0.1)  # the reference's initial model for seed 42
    p.sgda_begin(group)
    for e in range(4):
        p.sgda_epoch(tr, va, task, 0.02, mn, mx, e > 0)
    assert p.w0.value == ref_golden["sgda%d_w0" % task]
    assert digest(p.w) + digest(p.v) == ref_golden["sgda%d_wv_sha" % task]
    reg_w, reg_v = ref_golden["sgda%d_reg_w" % task], ref_golden["sgda%d_reg_v" % task]
    assert np.array_equal(reg_w, p.reg_w) and np.array_equal(reg_v, p.reg_v)
    assert reg_w.max() > 0 and reg_v.max() > 0  # the lambda-steps did move the regularisation
