"""GPU: the row-lane HOGWILD epoch keeps its window schedule.

Two runs agreeing with each other (test_hogwild_gpu.py::test_rowlane_epochs_are_reproducible) does not show
that the epoch still draws the same windows: which rows share a window decides which state they read, so a
different schedule would be reproducible and still compute something else.  This pins what the epoch computes
on C2 and C2-Zipf (the bias-ramp epoch and two more) to SHA-256 digests of the parameters recorded on an H100
(scripts/make_rowlane_digests.py), and checks that the epoch is one launch.

The digests were recorded from this kernel, so they pin that its bits stay what they were, on the recorded
geometry; that those bits are right, on any geometry, is pinned by test_rowlane_model_gpu.py, which compares
the epoch with an fp64 model of its windows.
"""
import json
import os

import pytest

from conftest import GOLDEN, digest
from libfm_b200 import FmLearnSgdElement, FmModel, MODE_HOGWILD, synth

pytestmark = pytest.mark.gpu

RECORD = json.load(open(os.path.join(GOLDEN, "rowlane_c2_digests.json")))


@pytest.mark.parametrize("name,zipf", [("c2", 0.0), ("c2_zipf", 1.0)])
def test_rowlane_epochs_match_recorded_digests(name, zipf, built_lib):
    d = synth.movielens_1m_shaped(seed=7, zipf=zipf)
    fm = FmModel(d.num_feature, 8)
    fm.init_stdev = 0.1
    fm.init_numpy(42)
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate = 0, 0.01
    l.min_target, l.max_target = d.min_target, d.max_target
    l.push_hparams()
    l.upload(d, 0)
    try:
        for e, want in enumerate(RECORD["digests"][name]):
            n0 = l.kernel_launches()
            l.sgd_epoch(d)
            assert l.kernel_launches() - n0 == 1, "epoch %d" % e
            cfg = l.epoch_config()
            assert cfg["lanes_per_row"] == 1  # the row-lane kernel ran
            if (cfg["rows_per_tile"], cfg["grid"]) != (RECORD["rows_per_tile"], RECORD["grid"]):
                pytest.skip("digests recorded for windows of %d x %d rows; this device runs %d x %d" % (
                    RECORD["grid"], RECORD["rows_per_tile"], cfg["grid"], cfg["rows_per_tile"]))
            l.pull_params()
            got = {"w0": digest(float(l.fm.w0)), "w": digest(l.fm.w), "v": digest(l.fm.v)}
            assert got == want, "epoch %d" % e
    finally:
        l.close()
