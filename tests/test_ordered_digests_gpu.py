"""GPU: the ORDERED epoch computes what it computed when its digests were recorded.

The ORDERED epoch is one CTA walking the rows in a fixed order, so what it computes is deterministic and can be
pinned exactly: SHA-256 digests of w0, w and V after two epochs (scripts/make_ordered_digests.py, recorded on an
H100 into tests/golden/ordered_digests.json).  The matrix launches every kernel instantiation the launcher can
pick in every configuration it can run in: with the helper warp (the default for k <= 32) and without (k > 32,
explicit thread counts, variant 1 and 2), the register-resident and the general kernels, both tasks.  The launch
configuration each case reports is pinned with it.
"""
import functools
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, digest, make_learner
from libfm_b200 import MODE_ORDERED, Data, synth
from test_oracle import _ragged_short_rows
from test_ordered_gpu import _cfg, _rand_init, _shape

pytestmark = pytest.mark.gpu

EPOCHS = 2
RECORD_PATH = os.path.join(GOLDEN, "ordered_digests.json")
SHAPES = ["tiny", "c2_shape", "zipf", "ragged", "dups", "classification", "no_bias", "k3_reg", "k16_c4_shape",
          "k64_fields", "k128_long", "two_field_real_values", "one_hot_regularised", "clamp_heavy"]
TUNINGS = {"default": {}, "threads128": {"threads": 128}, "threads256": {"threads": 256},
           "threads1024": {"threads": 1024}, "variant1": {"variant": 1}, "variant2": {"variant": 2}}


@functools.lru_cache(maxsize=None)
def _data(name):
    """(train, native task, k, k0, k1, regs, lr): test_ordered_gpu's shapes plus the ones that reach the
    remaining kernels (rows longer than 4 entries for k in {1, 2, 8}, the register-resident kernels of k = 2 and
    4, GL = 4 and GL = 32) and C2 at full size"""
    if name in SHAPES:
        return _shape(name)
    regs = (0.0, 0.0, 0.0)
    if name in ("k1_long", "k2_long", "k8_long"):
        return synth.ragged(3_000, 800, 12, seed=17), 0, int(name[1]), 1, 1, regs, 0.01
    if name in ("k2_onehot", "k4_onehot"):
        return synth.two_field(20_000, 600, 400, seed=18), 0, int(name[1]), 1, 1, regs, 0.02
    if name in ("k2_short", "k4_short"):
        return _ragged_short_rows(20_000, 500, seed=19), 0, int(name[1]), 1, 1, (0.0, 0.01, 0.02), 0.02
    if name == "k32_ragged":
        return _ragged_short_rows(20_000, 400, seed=15), 0, 32, 1, 1, regs, 0.01
    if name == "k200_ragged":
        return synth.ragged(1_000, 1_500, 20, seed=16), 0, 200, 1, 1, regs, 0.002
    if name == "c2_full":
        return synth.movielens_1m_shaped(seed=7, planted_k=4), 0, 8, 1, 1, regs, 0.01
    raise ValueError(name)


def _matrix():
    ids = ["%s/native/default" % s for s in SHAPES]
    for s in ("zipf", "ragged", "k16_c4_shape", "k32_ragged"):  # k = 8 one-hot, k = 8 ragged, k = 16, k = 32
        ids += ["%s/t%d/%s" % (s, t, tn) for t in (0, 1) for tn in TUNINGS]
    for s in ("k1_long", "k2_long", "k8_long", "k2_onehot", "k4_onehot", "k2_short", "k4_short", "k3_reg"):
        ids += ["%s/t%d/%s" % (s, t, tn) for t in (0, 1) for tn in ("default", "variant1", "variant2")]
    for s in ("k64_fields", "k128_long", "k200_ragged"):
        ids += ["%s/t%d/default" % (s, t) for t in (0, 1)]
    return ids + ["c2_full/native/default"]


MATRIX = _matrix()


def run(case_id):
    """Two ORDERED epochs of one matrix entry: the digests of (w0, w, V) and the launch configuration."""
    name, task_s, tuning = case_id.split("/")
    tr, task, k, k0, k1, regs, lr = _data(name)
    if task_s != "native" and int(task_s[1]) != task:
        task = int(task_s[1])
        if task == 1:  # (a regression case's targets split at their mean; a classification case's stay +-1)
            tr = Data(tr.row_ptr, tr.col, tr.val, np.where(tr.target > tr.target.mean(), 1.0, -1.0), tr.num_feature)
    n = tr.num_feature
    mn, mx = float(tr.target.min()), float(tr.target.max())
    l = make_learner(_cfg(n, k, task=task, lr=lr, regs=regs, k0=k0, k1=k1, mn=mn, mx=mx), _rand_init(n, k, 1),
                     mode=MODE_ORDERED)
    try:
        if TUNINGS[tuning]:
            l.set_tuning(**TUNINGS[tuning])
        for _ in range(EPOCHS):
            l.sgd_epoch(tr)
        l.pull_params()
        return {"w0": digest(float(l.fm.w0)), "w": digest(l.fm.w), "v": digest(l.fm.v), "cfg": l.epoch_config()}
    finally:
        l.close()


@functools.lru_cache(maxsize=None)
def _record():
    with open(RECORD_PATH) as f:
        return json.load(f)


@pytest.mark.parametrize("case_id", MATRIX)
def test_ordered_epochs_match_recorded_digests(case_id, built_lib):
    assert run(case_id) == _record()["digests"][case_id]
