"""GPU: the row-lane epoch's dealt schedule computes what the file-order schedule computes, bit for bit.

The dealt schedule hands each window's rows to the CTAs sorted by the id of their last entry, merges the
gathers and the integer steps of rows that share it, and forms the bias step from the rows of each
file-order tile (fm_rowlane.cu, fm_deal.cu).  Tuning variant 5 forces the file-order schedule on the same
build; three epochs of each must leave identical parameters on every shape below.
"""
import numpy as np
import pytest

from conftest import digest
from libfm_b200 import FmLearnSgdElement, FmModel, MODE_HOGWILD, synth
from libfm_b200.model import Data

pytestmark = pytest.mark.gpu

EPOCHS = 3


def _ragged(n_rows, n_users, n_items, seed, twice=0.0, values=False):
    """(user, item) rows cut to 0-4 entries: some rows empty, some with a second item, some naming a feature
    twice (`twice` of them); the last entry is the item wherever the row has one."""
    rng = np.random.default_rng(seed)
    lens = rng.choice([0, 1, 2, 3, 4], size=n_rows, p=[0.05, 0.15, 0.5, 0.2, 0.1])
    rows = []
    for r in range(n_rows):
        u = int(rng.integers(n_users))
        items = [n_users + int(x) for x in rng.integers(n_items, size=3)]
        row = ([u] + items)[: lens[r]]
        if row and rng.random() < twice:
            row = row[:-1] + [row[-1], row[-1]] if len(row) < 4 else row[:-2] + [row[-1], row[-1]]
        rows.append(row)
    row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
    row_ptr[1:] = np.cumsum([len(x) for x in rows])
    col = np.array([i for x in rows for i in x], dtype=np.uint32)
    val = rng.uniform(0.5, 1.5, size=len(col)).astype(np.float32) if values else np.ones(len(col), np.float32)
    target = rng.integers(1, 6, size=n_rows).astype(np.float32)
    return Data(row_ptr, col, val, target, num_feature=n_users + n_items)


SHAPES = {
    "c2": lambda: synth.movielens_1m_shaped(seed=7),
    # 1-4 entries per row and empty rows; 200 000 rows leave a short last window
    "ragged": lambda: _ragged(200_000, 3000, 900, seed=1),
    # rows that name one feature twice, values other than 1
    "twice": lambda: _ragged(150_000, 2000, 600, seed=2, twice=0.05, values=True),
    # one window of 24 tiles and no bias ramp: every epoch is dealt (few rows per feature: no COMBINE)
    "small": lambda: _ragged(6_000, 300, 800, seed=3),
}


def _run(d, variant, threads):
    fm = FmModel(d.num_feature, 8)
    fm.init_stdev = 0.1
    fm.init_numpy(42)
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate = 0, 0.01
    l.min_target, l.max_target = float(d.target.min()), float(d.target.max())
    l.push_hparams()
    l.set_tuning(threads=threads, variant=variant)
    l.upload(d, 0)
    out = []
    try:
        for _ in range(EPOCHS):
            l.sgd_epoch(d)
            assert l.epoch_config()["lanes_per_row"] == 1  # the row-lane kernel ran
            l.pull_params()
            out.append(({"w0": digest(float(l.fm.w0)), "w": digest(l.fm.w), "v": digest(l.fm.v)}, l.epoch_dealt()))
    finally:
        l.close()
    return out


# 64-row tiles cut far more items' runs at a CTA boundary than 256-row ones
@pytest.mark.parametrize("threads", [256, 64])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_dealt_schedule_is_bit_identical_to_file_order(shape, threads, built_lib):
    d = SHAPES[shape]()
    want = _run(d, 5, threads)
    got = _run(d, 0, threads)
    assert not any(dealt for _, dealt in want)
    assert all(dealt for _, dealt in got[1:]), "the dealt schedule did not run"
    for e in range(EPOCHS):
        assert got[e][0] == want[e][0], "epoch %d" % e
