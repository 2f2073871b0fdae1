"""GPU: the reproducible row-lane HOGWILD epoch computes what the fp64 model of its windows computes.

oracle/rowlane_model.py states the epoch without CTAs, warps, the dealt order or the in-warp merge: every row
of a window reads one state, its steps are damped by gamma, rounded to 2^-32, summed and folded.  Each case
below runs the kernel (fm_sgd_rowlane_kernel, fm_rowlane.cu), reads the geometry the device chose
(epoch_config, epoch_dealt) and feeds exactly that to the model, so no case depends on the SM count and none
skips.  After every epoch each parameter must lie within the model's per-element budget (fp32 row arithmetic,
gamma's fast exponential, quantisation; rowlane_model.py derives it), and each of w0, w and v within a
relative 2-norm of the distance the run has moved it, so that no structural error hides among tiny elements.

The recorded digests (test_rowlane_windows_gpu.py) pin that the bits stay what they were; this pins that they
are right.  tests/test_rowlane_model.py checks the model itself, on the CPU.
"""
import numpy as np
import pytest

from libfm_b200 import Data, FmLearnSgdElement, FmModel, MODE_HOGWILD, synth
from oracle import HParams, State, rowlane_epoch_model
from test_rowlane_deal_gpu import _ragged

pytestmark = pytest.mark.gpu

SMALL = dict(ctas_per_sm=1, threads=32)  # windows of SMs x 32 rows: a few thousand rows make many windows
RAMP_TILES = 4


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pull(l):
    l.pull_params()
    return State(float(l.fm.w0), l.fm.w.copy(), l.fm.v.copy())


def _rel(got, want, init):
    moved = np.linalg.norm(np.ravel(got - init))
    diff = np.linalg.norm(np.ravel(got - want))
    return diff / moved if moved > 0 else (0.0 if diff == 0 else np.inf)


def run_case(name, d, k=8, task=0, regs=(0.0, 0.0, 0.0), k0=True, k1=True, epochs=2, tuning=SMALL, lr=0.01,
             dealt=None, windows=None, aggregate=1e-4):
    """Runs `epochs` epochs on the device and in the model and compares after each.  dealt: the schedule each
    epoch must have run (None: either); windows: the windows epoch 0 must have had.  Returns the worst
    |got - want| / budget and the worst aggregate ratio."""
    fm = FmModel(d.num_feature, k, k0, k1)
    fm.init_stdev = 0.1
    fm.init_numpy(42)
    fm.reg0, fm.regw, fm.regv = regs
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate = task, lr
    l.min_target, l.max_target = d.min_target, d.max_target
    l.push_hparams()
    l.set_tuning(**tuning)
    l.upload(d, 0)
    hp = HParams(task, lr, regs[0], regs[1], regs[2], d.min_target, d.max_target, k0, k1)
    worst, worst_agg = 0.0, 0.0
    try:
        init = _pull(l)  # the fp32 state the device holds
        want, bud = init, None
        for e in range(epochs):
            l.sgd_epoch(d)
            cfg = l.epoch_config()
            assert cfg["lanes_per_row"] == 1, "the row-lane kernel did not run"
            TR, grid = cfg["rows_per_tile"], cfg["grid"]
            n_tiles = (d.num_cases + TR - 1) // TR
            # the bias ramp: the first epoch after set_params, with a bias, unless damping is forced off,
            # on more than 32 tiles; it runs the file-order schedule
            ramp = RAMP_TILES if e == 0 and k0 and tuning.get("damp", 0) >= 0 and n_tiles > 8 * RAMP_TILES else 0
            assert not (ramp and l.epoch_dealt())
            if dealt is not None:
                assert l.epoch_dealt() == dealt[e], "epoch %d" % e
            before = 0 if bud is None else bud.windows
            want, bud = rowlane_epoch_model(want, d, hp, TR, grid, bool(cfg["damp"]), ramp, budget=bud)
            if windows is not None and e == 0:
                assert bud.windows - before == windows
            got = _pull(l)
            b0, bw, bv = bud.bound(want)
            ratio = max(abs(got.w0 - want.w0) / b0, np.max(np.abs(got.w - want.w) / bw),
                        np.max(np.abs(got.v - want.v) / bv))
            agg = max(_rel(got.w0, want.w0, init.w0), _rel(got.w, want.w, init.w), _rel(got.v, want.v, init.v))
            print("rowlane-model %-22s epoch %d  TR %3d grid %3d damp %d dealt %d windows %3d  "
                  "worst/budget %.3f  aggregate %.2e" % (name, e, TR, grid, cfg["damp"], l.epoch_dealt(),
                                                         bud.windows - before, ratio, agg))
            assert ratio < 1.0, "epoch %d: a parameter is %.2f budgets away from the model" % (e, ratio)
            assert agg < aggregate, "epoch %d: relative distance to the model %.2e" % (e, agg)
            if not k0:
                assert got.w0 == init.w0
            if not k1:
                assert np.array_equal(got.w, init.w)
            worst, worst_agg = max(worst, ratio), max(worst_agg, agg)
    finally:
        l.close()
    return worst, worst_agg


def _two_field(n_rows, seed=3):
    return synth.two_field(n_rows, 300, 200, seed=seed)


# ---- one window: no compounding, so a difference is the step or the fold.  These calibrate the budget. ----

@pytest.mark.parametrize("name,k0,damp", [("one_window_plain", False, -1),  # no bias, no gamma: fp32 + quantisation
                                          ("one_window_bias", True, -1),    # the per-tile bias step alone
                                          ("one_window_gamma", False, 1),   # gamma on the features alone
                                          ("one_window_gamma_hot", False, 1)])  # ... at concurrencies up to ~1000
def test_one_window(name, k0, damp, built_lib):
    n_rows = min(4000, _sm_count() * 32)
    d = synth.two_field(n_rows, 50, 40, seed=5, zipf=1.2) if name.endswith("hot") else _two_field(n_rows)
    run_case(name, d, k0=k0, epochs=1, tuning=dict(SMALL, damp=damp), windows=1)


# ---- many windows ----

@pytest.mark.parametrize("threads", [32, 64])
def test_many_windows_ramp_then_dealt(threads, built_lib):
    """Bias ramp and file-order schedule in epoch 0, the dealt schedule after it, a short last window."""
    run_case("two_field_t%d" % threads, _two_field(20_000), epochs=3, tuning=dict(SMALL, threads=threads, damp=1),
             dealt=[False, True, True])


def test_file_order_schedule_after_the_first_epoch(built_lib):
    run_case("file_order", _two_field(20_000), epochs=3, tuning=dict(SMALL, damp=1, variant=5),
             dealt=[False, False, False])


@pytest.mark.parametrize("extra", [0, 1])
def test_last_window_edge(extra, built_lib):
    """The rows fill three windows exactly, or leave one row for a fourth."""
    window = _sm_count() * 32
    d = _two_field(3 * window + extra)
    run_case("exact_multiple+%d" % extra, d, k0=False, tuning=dict(SMALL, damp=1), windows=3 + extra)


@pytest.mark.parametrize("n_rows,windows", [(1000, 1),    # 32 tiles: the grid is clipped to them, no ramp
                                            (1200, 5)])   # 38 tiles: four ramp windows and one short one
def test_few_tiles(n_rows, windows, built_lib):
    assert _sm_count() >= 34
    run_case("tiles_%d" % n_rows, _two_field(n_rows), tuning=dict(SMALL, damp=1), windows=windows)


@pytest.mark.parametrize("k", [1, 4, 5, 8])
def test_factor_widths(k, built_lib):
    """k <= 4 is one float4 per factor row, k <= 8 two; the padding factors take no step."""
    run_case("k%d" % k, _two_field(10_000), k=k, tuning=dict(SMALL, damp=1))


def test_ragged_rows_with_values_and_repeats(built_lib):
    """Rows of 0-4 entries (the four-entry kernel), x != 1, features named twice; empty rows count in a tile's T."""
    d = _ragged(12_000, 300, 200, seed=2, twice=0.05, values=True)
    run_case("ragged", d, tuning=dict(SMALL, damp=1))


def test_one_entry_rows_share_features(built_lib):
    """The one-entry kernel reuses one write-back slot for every row."""
    r = np.random.default_rng(9)
    n = 10_000
    d = Data(np.arange(n + 1), r.integers(0, 50, n), r.uniform(0.5, 1.5, n), r.integers(1, 6, n), 50)
    run_case("one_entry", d, tuning=dict(SMALL, damp=1))


def test_classification(built_lib):
    d = _two_field(10_000)
    d = Data(d.row_ptr, d.col, d.val, np.where(d.target > 3, 1.0, -1.0), d.num_feature)
    run_case("classification", d, task=1, lr=0.05, tuning=dict(SMALL, damp=1))


@pytest.mark.parametrize("name,regs,k0,k1", [("regularised", (0.01, 0.02, 0.03), True, True),
                                             ("no_linear", (0.01, 0.02, 0.03), True, False),
                                             ("no_bias", (0.0, 0.02, 0.03), False, True)])
def test_model_switches_with_shared_features(name, regs, k0, k1, built_lib):
    run_case(name, _two_field(10_000), regs=regs, k0=k0, k1=k1, tuning=dict(SMALL, damp=1))


def test_zipf_hot_features(built_lib):
    """Zipf(1.2) ids over 50 x 40 features: concurrencies in the hundreds, where gamma is far below 1, and the
    in-warp fp32 merge of same-feature steps instead of the dealt schedule."""
    d = synth.two_field(20_000, 50, 40, seed=5, zipf=1.2)
    run_case("zipf", d, epochs=3, tuning=dict(SMALL), dealt=[False, False, False], aggregate=1e-3)


@pytest.mark.parametrize("name,zipf,aggregate", [("c2", 0.0, 1e-4), ("c2_zipf", 1.0, 1e-3)])
def test_c2_full_size_default_geometry(name, zipf, aggregate, built_lib):
    """The configuration the headline number is timed on."""
    d = synth.movielens_1m_shaped(seed=7, zipf=zipf)
    run_case(name, d, epochs=3, tuning={}, aggregate=aggregate)
