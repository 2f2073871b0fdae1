"""CPU: the fp64 model of the row-group HOGWILD epoch (oracle/rowgroup_model.py) is itself right.

tests/test_rowgroup_model_gpu.py holds fm_sgd_hogwild_kernel to this model, so the model is tied down first,
where no GPU is needed: to the sequential oracle where the two must agree (no damping, no bias), to gamma and a
bias step worked out by hand, to its own preconditions, and to the launcher's geometry rule: the GPU test's
cases must reach every (G, S, class) x DAMP instantiation of the kernel.
"""
import itertools

import numpy as np
import pytest

from libfm_b200 import Data
from oracle import HParams, Port, State, geometry, rowgroup_epoch_model
from oracle import rowgroup_model as gm
from oracle import rowlane_model as rm
from test_rowgroup_model_gpu import MATRIX, make_data, matrix_case, tuning_for


def _state(n, k, seed, w0=0.0):
    r = np.random.default_rng(seed)
    f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
    return State(float(np.float32(w0)), f32(0.05 * r.standard_normal(n)), f32(0.1 * r.standard_normal((k, n))))


def _port_epoch(st, d, hp):
    o = Port(st.w.shape[0], st.v.shape[0], hp.k0, hp.k1)
    o.set_params(st.w0, st.w, st.v)
    o.reg0, o.regw, o.regv = hp.reg0, hp.regw, hp.regv
    o.sgd_epoch(d, hp.task, hp.lr, hp.min_target, hp.max_target)
    return State(o.w0.value, o.w, o.v)


def _one_step(a, b):
    """One fp32 step of an element from a to b: the step rounded to fp32, the sum rounded to fp32."""
    return 0.5 * (rm.ulp32(b - a) + rm.ulp32(np.maximum(np.abs(a), np.abs(b))))


def _with_empty_rows(d, every=7):
    """`d` with an empty row inserted after every `every`-th row."""
    rp = d.row_ptr.astype(np.int64)
    new_rp, tg = [0], []
    for r in range(d.num_cases):
        new_rp.append(int(rp[r + 1]))
        tg.append(d.target[r])
        if r % every == 0:
            new_rp.append(int(rp[r + 1]))
            tg.append(d.target[r])
    return Data(np.array(new_rp), d.col, d.val, np.array(tg), d.num_feature)


FAMILIES = {
    # zero-valued entries (Zipf counts, some in their live entry's row), x != 1 and x < 0, empty rows
    "zeros": dict(live=0.4, regs=(0.0, 0.0, 0.0)),
    # every entry live, all three regularisers on
    "regularised": dict(live=1.0, regs=(0.0, 0.02, 0.03)),
}


@pytest.mark.parametrize("task", [0, 1])
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_undamped_model_is_the_sequential_oracle(family, task):
    """Without damping and without the bias every element takes the one step the sequential loop gives it, from
    the same state: the model equals fm_oracle.c up to its fp32 rounding of the step and the element."""
    f = FAMILIES[family]
    d = _with_empty_rows(make_data(300, 6.0, geometry(8, 300, 1800), seed=3, live=f["live"], task=task))
    assert (d.val == 0).any() == (family == "zeros") and (np.diff(d.row_ptr.astype(np.int64)) == 0).any()
    assert (d.val < 0).any() and ((d.val != 0) & (d.val != 1)).any()
    lr = 0.05
    hp = HParams(task, lr, *f["regs"], -0.8, 0.8, k0=False, k1=True)  # the clamp acts on some rows
    init = _state(d.num_feature, 8, seed=4)
    want = _port_epoch(init, d, hp)
    for damp in (False, True):
        if damp and family == "zeros":
            continue  # damping scales the hot features' steps: not the sequential loop
        got, bud = rowgroup_epoch_model(init, d, hp, 1.0, 1.0, damp, tile_rows=32)
        assert np.all(np.abs(got.w - want.w) <= _one_step(init.w, want.w))
        assert np.all(np.abs(got.v - want.v) <= _one_step(init.v, want.v))
        assert got.w0 == init.w0 and bud.w0 == 0.0
        assert np.abs(got.v - init.v).max() > 1e-3  # the epoch moved the state
        # elements of the features no entry names are neither stepped nor budgeted
        assert np.array_equal(got.v[:, -3:], init.v[:, -3:]) and not bud.v[:, -3:].any()


def test_zero_valued_entries_change_nothing_undamped():
    """The same live entries with and without zero-valued ones: bit-identical, in the model as in the oracle."""
    d = make_data(400, 8.0, geometry(8, 400, 3200), seed=5, live=0.3)
    live = d.val != 0
    erow = np.repeat(np.arange(d.num_cases), np.diff(d.row_ptr.astype(np.int64)))
    rp = np.concatenate([[0], np.cumsum(np.bincount(erow[live], minlength=d.num_cases))])
    d_live = Data(rp, d.col[live], d.val[live], d.target, d.num_feature)
    hp = HParams(0, 0.02, min_target=-3.0, max_target=3.0, k0=False)
    init = _state(d.num_feature, 8, seed=6)
    a, _ = rowgroup_epoch_model(init, d, hp, 1.0, 1.0, False, 32)
    b, _ = rowgroup_epoch_model(init, d_live, hp, 1.0, 1.0, False, 32)
    assert np.array_equal(a.w, b.w) and np.array_equal(a.v, b.v)
    pa, pb = _port_epoch(init, d, hp), _port_epoch(init, d_live, hp)
    assert np.array_equal(pa.w, pb.w) and np.array_equal(pa.v, pb.v)
    # damped, the zero-valued entries raise c_i, and the hottest features' steps shrink far below 1
    c, _ = rowgroup_epoch_model(init, d, hp, 1.0, 1.0, True, 32)
    hot = np.argmax(np.bincount(d.col, minlength=d.num_feature))
    assert abs(c.w[hot] - init.w[hot]) < 0.2 * abs(a.w[hot] - init.w[hot])


def test_gamma_and_the_bias_step_by_hand():
    """One tile of two rows, k = 0, lr = 1/4, reg0 = 1, w0 = 1/2, w = 0, DAMP.  Row 0 names feature 0 (x = 1)
    and, zero-valued, feature 1; row 1 names feature 1 (x = 2) and, zero-valued, feature 0 twice.  Counts 3 and
    2, conc_scale 1: c = 3 and 2.  Targets 1/2 and 2: p = 1/2, mult = 0 and -3/2.

    hrow = xx (no factors): 1 and 4; hjoint = curv (1 + hrow) = 2 and 5.  Feature 1: u = lr 5 = 5/4 >= 1, where
    (1 - u)^c is taken as 0, so gamma(2, 5/4) = 1/(2 5/4) = 2/5 and the step is (2/5)(-lr mult x) = (2/5)(3/4).
    Feature 0: mult = 0, no step.  Bias: M = 0 - 3/2 + T reg0 w0 = -1/2, H = 7, u = lr (H/T + reg0) = 9/8, so
    gamma(2, 9/8) = 4/9 and w0 steps by -lr (4/9) M = 1/18.
    """
    d = Data([0, 2, 5], [0, 1, 1, 0, 0], [1.0, 0.0, 2.0, 0.0, -0.0], [0.5, 2.0], 2)
    hp = HParams(0, 0.25, reg0=1.0, min_target=-100.0, max_target=100.0, k0=True, k1=True)
    init = State(0.5, np.zeros(2), np.zeros((0, 2)))
    got, bud = rowgroup_epoch_model(init, d, hp, conc_scale=1.0, w0_conc=2.0, damp=True, tile_rows=32)
    assert got.w[0] == 0.0
    assert got.w[1] == np.float32(0.3)
    assert got.w0 == np.float32(np.float32(0.5) + np.float32(1.0 / 18.0))
    assert rm.gamma(2.0, 9.0 / 8.0) == pytest.approx(4.0 / 9.0)
    # undamped: hjoint is the loss curvature alone (H = 2), gamma(2, (1/4)(1 + 1)) = (1 - 1/4)/(2 * 1/2) = 3/4,
    # and the features take their plain steps
    got, _ = rowgroup_epoch_model(init, d, hp, 1.0, 2.0, damp=False, tile_rows=32)
    assert got.w[1] == np.float32(0.75)
    assert got.w0 == np.float32(np.float32(0.5) + np.float32(0.25 * 0.75 * 0.5))
    # w0_conc = 1: a lone tile in flight takes the plain bias step
    got, _ = rowgroup_epoch_model(init, d, hp, 1.0, 1.0, damp=False, tile_rows=32)
    assert got.w0 == np.float32(np.float32(0.5) + np.float32(0.25 * 0.5))
    assert bud.w0 > 0.0 and bud.w[1] > 0.0


def test_the_model_refuses_data_a_schedule_could_change():
    hp = HParams(0, 0.01, min_target=-1.0, max_target=1.0, k0=False)
    st = State(0.0, np.zeros(3), np.zeros((4, 3)))
    shared = Data([0, 1, 2], [0, 0], [1.0, 0.5], [0.0, 0.0], 3)
    with pytest.raises(ValueError, match="shares its feature"):
        rowgroup_epoch_model(st, shared, hp, 1.0, 1.0, False, 32)
    zeros = Data([0, 2, 3], [0, 1, 0], [1.0, 1.0, 0.0], [0.0, 0.0], 3)
    rowgroup_epoch_model(st, zeros, hp, 1.0, 1.0, True, 32)  # fine without regularisation
    for regs in [(0.0, 0.01, 0.0), (0.0, 0.0, 0.01)]:
        with pytest.raises(ValueError, match="zero-valued"):
            rowgroup_epoch_model(st, zeros, HParams(0, 0.01, *regs, -1.0, 1.0, k0=False), 1.0, 1.0, True, 32)
    rowgroup_epoch_model(st, zeros, HParams(0, 0.01, 0.5, 0.0, 0.0, -1.0, 1.0, k0=True), 1.0, 2.0, True, 2)
    with pytest.raises(ValueError, match="more than one tile"):
        rowgroup_epoch_model(st, zeros, HParams(0, 0.01, min_target=-1.0, max_target=1.0), 1.0, 2.0, True, 1)


def test_budget_scales_with_the_row():
    """The score's bound grows with the row's length and magnitudes, so a 500-entry row at k = 128 is not
    held to the constants of a 4-entry one."""
    st = _state(2000, 128, seed=1)
    hp = HParams(0, 0.01, min_target=-5.0, max_target=5.0, k0=False)
    short = Data([0, 4], np.arange(4), np.ones(4), [0.0], 2000)
    long = Data([0, 500], np.arange(500), np.ones(500), [0.0], 2000)
    _, dp_s = gm.row_scores(st, short, hp)
    _, dp_l = gm.row_scores(st, long, hp)
    assert dp_l[0] > 100 * dp_s[0]


@pytest.mark.parametrize("k,avg,threads,want", [
    (8, 1.0, 0, (2, 1, -1, 8 * 16 * 4.0)), (8, 39.0, 0, (2, 8, 1, 8 * 2.0)), (64, 39.0, 0, (16, 2, 2, 8.0)),
    (128, 39.0, 96, (32, 1, 3, 3.0)), (100, 2.5, 32, (32, 1, 0, 2.0)), (0, 3.0, 0, (1, 4, -1, 8 * 8 * 4.0))])
def test_geometry_restates_the_launcher(k, avg, threads, want):
    g = geometry(k, 1000, int(avg * 1000), threads)
    assert (g.G, g.S, g.cls, g.rows_per_cta_step) == want
    assert (g.R, g.RW, g.U) == gm.CLASSES[g.cls]


def _instantiations():
    """Every (G, S, class) pick_geometry can return, from its rule over factor widths and row lengths."""
    out = set()
    for k in range(1, 129):
        for avg in np.arange(0.25, 200.0, 0.25):
            g = geometry(k, 1000, int(avg * 1000))
            out.add((g.G, g.S, g.cls))
    return out


def test_matrix_covers_every_instantiation_with_damping_on_and_off():
    reach = _instantiations()
    assert len(reach) == 37
    seen = {}
    for i in range(len(MATRIX)):
        k, d, geo = matrix_case(i)
        key = (geo.G, geo.S, geo.cls)
        assert key not in seen, "MATRIX[%d] drifted onto MATRIX[%d]'s geometry %s" % (i, seen.get(key, -1), key)
        seen[key] = i
        # rows longer than the register caches, so the re-gather loops q >= R and t >= RW run
        longest = int(np.diff(d.row_ptr.astype(np.int64)).max())
        assert longest > geo.R * geo.S and longest > geo.RW * geo.E, (i, key, longest)
        # the row-lane kernel is kept off every shape it could take
        gp = (k + 3) // 4
        assert tuning_for(k, d).get("variant", 0) == (1 if gp <= 2 else 0)
        # live entries name distinct features, zero-valued ones reach concurrencies of hundreds
        live = d.val != 0
        assert np.unique(d.col[live]).size == live.sum()
        assert np.bincount(d.col, minlength=d.num_feature).max() >= 100
    assert set(seen) == reach
    # each with DAMP on and off: test_geometry_matrix is parametrised over both
    from test_rowgroup_model_gpu import test_geometry_matrix
    marks = {m.args[0]: m.args[1] for m in test_geometry_matrix.pytestmark if m.name == "parametrize"}
    assert sorted(marks["damp"]) == [-1, 1] and list(marks["i"]) == list(range(len(MATRIX)))
    assert len(set(itertools.product(seen, marks["damp"]))) == 74
