"""GPU: the windowed HOGWILD epochs keep their bits.

The reproducible SGD epoch (fm_sgd_window.cu) and the HOGWILD SGDA epoch (fm_sgda_hogwild.cu) compute the same
bits on every run and at every grid size, so what they compute can be pinned exactly.  This recomputes SHA-256
digests of w0, w and V after every epoch (for SGDA also of reg_w, reg_v and the moments) and compares them with
tests/golden/window_digests.json, recorded on an H100 with scripts/make_window_digests.py.  The cases cover both
epochs at every factor class, long rows with repeated features and non-unit values, the bias ramp, classification,
the lambda-steps, one context that runs SGD epochs and then SGDA epochs on the same accumulator and window stamps,
and a diverging run of each.  How close those bits are to the fp64 statement of the windows is
test_sgd_window_gpu.py's and test_sgda_hogwild_gpu.py's business.
"""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, digest
from libfm_b200 import Data, FmLearnSgdElement, FmModel, MODE_HOGWILD, synth
from test_sgd_window_gpu import _long_rows

pytestmark = pytest.mark.gpu

RECORD_PATH = os.path.join(GOLDEN, "window_digests.json")
EPOCHS = 3


def _cls(d):
    return Data(d.row_ptr, d.col, d.val, np.where(d.target > 3, 1.0, -1.0).astype(np.float32), d.num_feature)


def _learner(n, k, task, lr, tuning, stdev=0.05, min_target=1.0, max_target=5.0):
    fm = FmModel(n, k)
    fm.init_stdev = stdev
    fm.init_numpy(42)
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate = task, lr
    l.min_target, l.max_target = min_target, max_target
    l.push_hparams()
    l.set_tuning(**tuning)
    return l


def _theta(l):
    l.pull_params()
    return {"w0": digest(float(l.fm.w0)), "w": digest(l.fm.w), "v": digest(l.fm.v)}


def _sgd_epochs(l, d, epochs):
    out = []
    for _ in range(epochs):
        l.sgd_epoch(d)
        assert l.epoch_config()["lanes_per_row"] == 32, "the windowed epoch did not run"
        out.append(_theta(l))
    return out


def _sgda_epochs(l, train, val, groups, epochs):
    n = train.num_feature
    l.sgda_begin(np.arange(n) % groups if groups > 1 else None)
    out = []
    for e in range(epochs):
        l.sgda_epoch(train, val, e > 0)  # lambda-steps from the second epoch
        rec = _theta(l)
        reg_w, reg_v = l.sgda_reg()
        var_w, var_v = l.sgda_moments()
        rec.update(reg_w=digest(reg_w), reg_v=digest(reg_v), moments=digest(np.append(var_w, var_v)))
        out.append(rec)
    return out


def _sgd(d, k, T=0, B=0, task=0, lr=0.01, damp=0, stdev=0.05):
    l = _learner(d.num_feature, k, task, lr, dict(damp=damp), stdev, d.min_target, d.max_target)
    try:
        l.set_reproducible(True, T, B)
        l.upload(d, 0)
        return _sgd_epochs(l, d, EPOCHS)
    finally:
        l.close()


def _sgda(train, val, k, groups, W=0, lr=0.01):
    l = _learner(train.num_feature, k, 0, lr, dict(rows_per_tile=W))
    try:
        l.upload(train, 0)
        l.upload(val, 1)
        return _sgda_epochs(l, train, val, groups, EPOCHS)
    finally:
        l.close()


def _sgd_then_sgda():
    """One context: reproducible SGD epochs, then fmb200_sgda_begin and SGDA epochs on the same accumulator and
    window stamps."""
    train, val = _long_rows(3000, 500, 30, seed=21), _long_rows(600, 500, 30, seed=22)
    l = _learner(train.num_feature, 16, 0, 0.005, dict(damp=1, rows_per_tile=256))
    try:
        l.set_reproducible(True, 32, 4)
        l.upload(train, 0)
        l.upload(val, 1)
        return _sgd_epochs(l, train, 2) + _sgda_epochs(l, train, val, 3, 2)
    finally:
        l.close()


def _two_field(n_rows, seed):
    return synth.two_field(n_rows, 6040, 3706, seed=seed)


def cases():
    """name -> a function that runs the case and returns one dict of digests per epoch.  Data is made when a case
    runs."""
    return {
        "sgd_c2_zipf": lambda: _sgd(synth.movielens_1m_shaped(seed=7, zipf=1.0), 8),
        "sgd_long_k33": lambda: _sgd(_long_rows(4003, 900, 60, seed=33), 33, T=32, B=4, lr=0.002, damp=1,
                                     stdev=0.02),
        "sgd_long_k100": lambda: _sgd(_long_rows(4003, 900, 60, seed=100), 100, T=32, B=4, lr=0.002, damp=1,
                                      stdev=0.02),
        "sgd_classification": lambda: _sgd(_cls(_long_rows(6000, 500, 20, seed=8)), 16, T=32, B=4, task=1,
                                           lr=0.02, damp=1),
        "sgda_c2_two_groups": lambda: _sgda(*synth.split_rows(_two_field(220_000, 5), 200_000), 8, 2),
        "sgda_long_k48": lambda: _sgda(_long_rows(3000, 600, 60, seed=48), _long_rows(500, 600, 60, seed=49), 48,
                                       3, W=256, lr=0.002),
        "sgda_long_k100": lambda: _sgda(_long_rows(3000, 600, 60, seed=100), _long_rows(500, 600, 60, seed=101),
                                        100, 3, W=256, lr=0.002),
        "sgd_then_sgda": _sgd_then_sgda,
        "sgd_diverging": lambda: _sgd(_long_rows(5000, 200, 30, seed=2), 16, T=32, B=4, lr=50.0, damp=-1,
                                      stdev=0.5),
        "sgda_diverging": lambda: _sgda(*synth.split_rows(synth.two_field(4500, 300, 200, seed=3), 3000), 8, 1,
                                        W=256, lr=50.0),
    }


@pytest.fixture(scope="module")
def record():
    with open(RECORD_PATH) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(cases()))
def test_window_epochs_match_recorded_digests(name, record, built_lib):
    got = cases()[name]()
    want = record["digests"][name]
    assert len(got) == len(want)
    for e, (g, w) in enumerate(zip(got, want)):
        assert g == w, "epoch %d: %s differ" % (e, sorted(key for key in w if g.get(key) != w[key]))
