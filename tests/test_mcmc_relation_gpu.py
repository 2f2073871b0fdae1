"""GPU: MCMC and ALS on relational data (block structure, fmb200_mcmc_set_relations) against the reference's
fm_learn_mcmc_simultaneous with train.relation / test.relation set as libfm.cpp does, bit for bit.

tests/golden/reference/mcmc_relation.npz (scripts/make_relation_golden.py) holds what the reference leaves after
each of its first iterations.  The blocks are written to files and read back with RelationData.load and
RelationJoin.load (binary and text joins, .groups files), so the loaders feed the learner.  After every iteration
w0, w, v, the hyperparameters, the NaN/Inf counters, the three test prediction vectors and the #Iter Train value
must equal the reference's, in both fp64 modes.
"""
import os
import sys

import numpy as np
import pytest

from libfm_b200 import MODE_INORDER, MODE_ORDERED, Data, FmError, FmLearnSgdElement, FmModel, RelationData, RelationJoin
from libfm_b200.model import XtBlocks, write_transposed
from test_mcmc_sweep_gpu import _digest, _first_difference, _reference_init

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
from make_relation_golden import ITERS, bs_case, write_block_files  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference", "mcmc_relation.npz")


def _z():
    return np.load(GOLDEN)


def _cases():
    return sorted({k.split("/")[0] for k in _z().files})


def _regular(reg, G, k):
    """-regular as libfm.cpp:326-364 spreads it: (reg0, w_lambda[G], v_lambda[G][k])"""
    if len(reg) == 0:
        return 0.0, np.zeros(G), np.zeros((G, k))
    if len(reg) == 1:
        return reg[0], np.full(G, reg[0]), np.full((G, k), reg[0])
    if len(reg) == 3:
        return reg[0], np.full(G, reg[1]), np.full((G, k), reg[2])
    return reg[0], np.array(reg[1:1 + G]), np.repeat(np.array(reg[1 + G:1 + 2 * G])[:, None], k, axis=1)


def _blocks(z, name, tmp, n_tr, n_te):
    """every block of the case written to files and loaded back as the reference's loaders read them"""
    R = int(z[f"{name}/cfg"][10])
    out = []
    for i in range(R):
        rows, nf, binary = (int(x) for x in z[f"{name}/rel{i}/rows"])
        d = Data(z[f"{name}/rel{i}/row_ptr"], z[f"{name}/rel{i}/col"], z[f"{name}/rel{i}/val"],
                 np.zeros(rows, np.float32), nf)
        g = z[f"{name}/rel{i}/groups"] if f"{name}/rel{i}/groups" in z.files else None
        stem = os.path.join(tmp, f"{name}_rel{i}")
        write_block_files(stem, dict(data=d, train=z[f"{name}/rel{i}/train"], test=z[f"{name}/rel{i}/test"],
                                     groups=g, binary=bool(binary)), n_tr, n_te)
        b = RelationData.load(stem)
        out.append((b, RelationJoin.load(stem + ".train", n_tr, b), RelationJoin.load(stem + ".test", n_te, b)))
    return out


def _start(z, name, tmp, mode):
    _, _, _, _, _, _, _, _, tr_nf, te_nf, _ = (int(x) for x in z[f"{name}/cfg"])
    tr = Data(z[f"{name}/tr_row_ptr"], z[f"{name}/tr_col"], z[f"{name}/tr_val"], z[f"{name}/tr_target"], tr_nf)
    te = Data(z[f"{name}/te_row_ptr"], z[f"{name}/te_col"], z[f"{name}/te_val"], z[f"{name}/te_target"], te_nf)
    rel = _blocks(z, name, tmp, tr.num_cases, te.num_cases)
    meta = z[f"{name}/meta"] if f"{name}/meta" in z.files else None
    return _learner(z, name, tr, te, rel, mode, list(z[f"{name}/reg"]), meta) + (rel,)


def _learner(z, name, tr, te, rel, mode, reg, meta=None):
    """a learner started as the reference's libfm.cpp starts it on these tables, with the relations set"""
    n, k, k0, k1, task, sample, ml, seed = (int(x) for x in z[f"{name}/cfg"][:8])
    l = FmLearnSgdElement(FmModel(n, k, k0, k1), mode=mode)
    l.upload(tr, 0)
    l.upload(te, 1)
    l.fm = _reference_init(n, k, k0, k1, seed)
    assert _digest(np.concatenate([[l.fm.w0], l.fm.w, l.fm.v.reshape(-1)])) == str(z[f"{name}/init_digest"])
    l.push_params()
    l.task = task
    l.min_target, l.max_target = (float(x) for x in z[f"{name}/minmax"])
    G = len(z[f"{name}/per_group"])
    reg0, wl, vl = _regular(reg, G, k)
    l.mcmc_begin(tr, te, sample, ml, reg0, wl, vl, relations=rel, main_group=meta)
    return l, tr, te


@pytest.mark.parametrize("mode", [MODE_INORDER, MODE_ORDERED], ids=["inorder", "ordered"])
@pytest.mark.parametrize("name", _cases())
def test_relational_iterations_bit_identical_to_reference(name, mode, tmp_path, built_lib):
    z = _z()
    l, tr, te, _ = _start(z, name, str(tmp_path), mode)
    assert ITERS >= 6   # iteration 5 is the first that pred_sum_all_but5 sums
    for t in range(ITERS):
        m, cnt = l.mcmc_iteration()
        bad = _first_difference(z, name, t, l, te, m, cnt)
        assert bad is None, "%s: iteration %d: %s differs from the reference" % (name, t, bad)
    l.close()


def _plain_run(l, z, name, tr, te):
    """from the reference's initial state, one iteration without relations: (runs, w0, w, v, test predictions)"""
    n, k, k0, k1, _, _, _, seed = (int(x) for x in z[f"{name}/cfg"][:8])
    l.fm = _reference_init(n, k, k0, k1, seed)
    l.push_params()
    l.mcmc_begin(tr, te, True, True, 0.0, np.zeros(1), np.zeros((1, k)))
    runs = l.mcmc_runs()
    l.mcmc_iteration()
    l.pull_params()
    return runs, l.fm.w0, l.fm.w.copy(), l.fm.v.copy(), l.mcmc_pred(te)[0]


def test_relations_apply_to_one_begin(tmp_path, built_lib):
    """the next mcmc_begin without relations runs the plain learner: the same runs and state as a context that
    never saw relations; a _begin that fails consumes the relations too"""
    z = _z()
    name = "main_features_one_block_mcmc"
    l, tr, te, rel = _start(z, name, str(tmp_path), MODE_INORDER)
    l.mcmc_iteration()
    got = _plain_run(l, z, name, tr, te)
    fresh = FmLearnSgdElement(FmModel(l.fm.num_attribute, l.fm.num_factor), mode=MODE_INORDER)
    fresh.upload(tr, 0)
    fresh.upload(te, 1)
    want = _plain_run(fresh, z, name, tr, te)
    assert got[0] == want[0]
    for a, b in zip(got[1:], want[1:]):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
    l.mcmc_set_relations(tr, te, rel)
    with pytest.raises(FmError, match="null w_lambda"):
        l._check(l.lib.fmb200_mcmc_begin(l._ctx, 0, 1, 1, 1, 1, None, None, 0.0, None, None))
    assert _plain_run(l, z, name, tr, te)[0] == want[0]
    fresh.close()
    l.close()


def test_refusals(tmp_path, built_lib):
    """bad join length, out-of-range join id, non-contiguous offsets, the streamed begin: each named"""
    l, tr, te, rel = _start(_z(), "main_features_one_block_mcmc", str(tmp_path), MODE_INORDER)
    b, jtr, jte = rel[0]
    k = l.fm.num_factor
    with pytest.raises(FmError, match="the train join has 1499 entries, the train set 1500 cases"):
        l.mcmc_set_relations(tr, te, [(b, RelationJoin(jtr.rows[:-1], b), jte)])
    bad = jte.rows.copy()
    bad[7] = b.num_cases
    with pytest.raises(FmError, match="the test join maps case 7 to row %d, not below num_cases %d"
                       % (b.num_cases, b.num_cases)):
        l.mcmc_set_relations(tr, te, [(b, jtr, RelationJoin(bad, b))])
    gap = RelationData(b.col_ptr[:2], b.row, b.val, b.num_cases, 1)
    gap.attr_offset = b.attr_offset + b.num_feature + 1   # one id left out between the blocks
    with pytest.raises(FmError, match="relation 1: attr_offset %d does not follow" % gap.attr_offset):
        l.mcmc_set_relations(tr, te, [(b, jtr, jte), (gap, jtr, jte)])
    l.mcmc_set_relations(tr, te, [(b, jtr, jte)])
    path = str(tmp_path / "tr.xt")
    write_transposed(tr, path)
    xb = XtBlocks(path, tr.target, 1 << 20)
    with pytest.raises(FmError, match="relations are not streamed"):
        l.mcmc_begin_xt(xb, te, True, True, 0.0, np.zeros(1), np.zeros((1, k)))
    # begin-time checks: a slot re-uploaded after the relations were set, a main table naming a block's id
    l.mcmc_set_relations(tr, te, [(b, jtr, jte)])
    l.upload(te, 1)
    with pytest.raises(FmError, match="re-uploaded after fmb200_mcmc_set_relations"):
        l.mcmc_begin(tr, te, True, True, 0.0, np.zeros(1), np.zeros((1, k)))
    col = tr.col.copy()
    col[0] = b.attr_offset + 3
    bad_tr = Data(tr.row_ptr, col, tr.val, tr.target, l.fm.num_attribute)
    l.upload(bad_tr, 0)
    l.mcmc_set_relations(bad_tr, te, [(b, jtr, jte)])
    with pytest.raises(FmError, match="slot 0 names attribute %d, which belongs to relation block" % (b.attr_offset + 3)):
        l.mcmc_begin(bad_tr, te, True, True, 0.0, np.zeros(1), np.zeros((1, k)))
    l.close()


BS_GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference", "mcmc_relation_bs.npz")


@pytest.mark.parametrize("mode", [MODE_INORDER, MODE_ORDERED], ids=["inorder", "ordered"])
def test_bs_shape_full_size(mode, tmp_path, built_lib):
    """The full-size BS shape of MovieLens-1M (bs_case: 1 000 209 train cases with empty main rows, a user block
    of 6040 rows carrying each user's rated items with Zipf(1) popularity, rows of up to thousands of entries,
    and an item block): 2 MCMC iterations against digests of the reference's (mcmc_relation_bs.npz)."""
    z = np.load(BS_GOLDEN)
    c = bs_case()
    tr, te = c["train"], c["test"]
    rel = []
    for i, b in enumerate(c["blocks"]):
        stem = str(tmp_path / f"rel{i}")
        write_block_files(stem, b, tr.num_cases, te.num_cases)
        d = RelationData.load(stem)
        rel.append((d, RelationJoin.load(stem + ".train", tr.num_cases, d), RelationJoin.load(stem + ".test", te.num_cases, d)))
    l, tr, te = _learner(z, "bs_mcmc", tr, te, rel, mode, list(c["reg"]))
    for t in range(2):
        m, cnt = l.mcmc_iteration()
        bad = _first_difference(z, "bs_mcmc", t, l, te, m, cnt)
        assert bad is None, "bs_mcmc: iteration %d: %s differs from the reference" % (t, bad)
    l.close()
