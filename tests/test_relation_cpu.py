"""CPU: the relational loaders (RelationData.load, RelationJoin.load) and the joined meta table against what the
reference's loaders and libfm.cpp:206-240 made of the same files (tests/golden/reference/mcmc_relation.npz,
scripts/make_relation_golden.py): the block sizes its loader printed, and the joined attr_group / num_attr_per_group.
"""
import os
import sys

import numpy as np
import pytest

from libfm_b200 import Data, FmError, RelationData, RelationJoin
from libfm_b200.model import join_meta

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
from make_relation_golden import write_block_files  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference", "mcmc_relation.npz")


def _cases():
    return sorted({k.split("/")[0] for k in np.load(GOLDEN).files})


def _load_case(z, name, tmp):
    cfg = z[f"{name}/cfg"]
    n_tr, n_te = len(z[f"{name}/tr_row_ptr"]) - 1, len(z[f"{name}/te_row_ptr"]) - 1
    out = []
    for i in range(int(cfg[10])):
        rows, nf, binary = (int(x) for x in z[f"{name}/rel{i}/rows"])
        d = Data(z[f"{name}/rel{i}/row_ptr"], z[f"{name}/rel{i}/col"], z[f"{name}/rel{i}/val"],
                 np.zeros(rows, np.float32), nf)
        g = z[f"{name}/rel{i}/groups"] if f"{name}/rel{i}/groups" in z.files else None
        stem = os.path.join(tmp, f"rel{i}")
        write_block_files(stem, dict(data=d, train=z[f"{name}/rel{i}/train"], test=z[f"{name}/rel{i}/test"],
                                     groups=g, binary=bool(binary)), n_tr, n_te)
        b = RelationData.load(stem)
        out.append((d, b, RelationJoin.load(stem + ".train", n_tr, b), RelationJoin.load(stem + ".test", n_te, b)))
    return out


@pytest.mark.parametrize("name", _cases())
def test_loaders_match_the_reference_loader(name, tmp_path):
    z = np.load(GOLDEN)
    blocks = _load_case(z, name, str(tmp_path))
    loads = list(z[f"{name}/loads"])
    assert len(loads) == len(blocks)
    for i, (d, b, jtr, jte) in enumerate(blocks):
        assert loads[i] == "num_cases=%d\tnum_values=%d\tnum_features=%d" % (b.num_cases, b.num_values, b.num_feature)
        # the .xt read back is the block transposed: every (row, feature, value) once, column by column
        cols = np.repeat(np.arange(b.num_feature), np.diff(b.col_ptr.astype(np.int64)))
        got = sorted(zip(b.row.tolist(), cols.tolist(), b.val.tolist()))
        rows = np.repeat(np.arange(d.num_cases), np.diff(d.row_ptr.astype(np.int64)))
        assert got == sorted(zip(rows.tolist(), d.col.tolist(), d.val.tolist()))
        assert np.array_equal(jtr.rows, z[f"{name}/rel{i}/train"])
        assert np.array_equal(jte.rows, z[f"{name}/rel{i}/test"])


@pytest.mark.parametrize("name", _cases())
def test_joined_meta_table_matches_libfm(name, tmp_path):
    z = np.load(GOLDEN)
    blocks = _load_case(z, name, str(tmp_path))
    cfg = z[f"{name}/cfg"]
    n_main = max(int(cfg[8]), int(cfg[9]))
    meta = z[f"{name}/meta"] if f"{name}/meta" in z.files else None
    n, group, per = join_meta(n_main, meta, [b for _, b, _, _ in blocks])
    assert n == int(cfg[0])
    assert np.array_equal(group, z[f"{name}/group"])
    assert np.array_equal(per, z[f"{name}/per_group"])
    off = n_main
    for _, b, _, _ in blocks:
        assert b.attr_offset == off
        off += b.num_feature


def test_join_load_refuses_a_short_file(tmp_path):
    p = str(tmp_path / "j.train")
    with open(p, "w") as f:
        f.write("0\n1\n")
    with pytest.raises(FmError, match="2 of 3 entries"):
        RelationJoin.load(p, 3)
    with open(p, "wb") as f:
        f.write(np.array([1, 4, 2, 0, 1], np.uint32).tobytes())
    with pytest.raises(FmError, match="2 entries, the data set 3 cases"):
        RelationJoin.load(p, 3)
