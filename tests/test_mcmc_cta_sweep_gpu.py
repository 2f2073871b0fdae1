"""GPU: the launch plan of the segmented MCMC / ALS sweeps.  Each segment's runs are cut into maximal stretches of
narrow runs (at most as many features as the sweeping CTA has warps), swept by one CTA with a CTA barrier between
runs (mcmc_cta_sweep_kernel), and of wide runs, swept by the cooperative grid (mcmc_block_sweep_kernel).

On a case whose run widths are known -- a main table with narrow, wide and narrow stretches and a relation block
with a wide and a narrow stretch, a block column that names a row twice -- the launch count per iteration is the
one the plan states, and w0, w, v, the hyperparameters, the NaN/Inf counters and the test predictions equal those
of a context that sweeps every run with the cooperative kernel (fmb200_set_tuning variant 1), bit for bit, for
MCMC and for ALS with a value whose square overflows (non-finite draws, counted and skipped)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from libfm_b200 import MODE_INORDER, MODE_ORDERED, Data, FmLearnSgdElement, FmModel, RelationData, RelationJoin

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
from make_relation_golden import write_block_files  # noqa: E402

pytestmark = pytest.mark.gpu

N_TR, N_TE, K = 3000, 500, 4
N_MULTI, N_ONEHOT, N_TAIL = 40, 2000, 40      # main table: ids [0, 40) | [40, 2040) | [2040, 2080)
ROWS, N_ITEMS = 300, 50                        # block: its row's id [0, 300), then items [300, 350)


def _rows(rng, n, pick):
    rp, col = [0], []
    for i in range(n):
        col += pick(i)
        rp.append(len(col))
    return np.array(rp, np.uint64), np.array(col, np.uint32)


def _case(huge: bool):
    """main rows: 2 of the first 40 ids, one one-hot id, 2 of the last 40 ids; block rows: the row's id and 3 items
    (row 0 names an item twice).  huge: one block entry of 3e19, whose square overflows float"""
    rng = np.random.default_rng(5)
    n_main = N_MULTI + N_ONEHOT + N_TAIL

    def main(n):
        rp, col = _rows(rng, n, lambda i: [int(x) for x in rng.choice(N_MULTI, 2, replace=False)]
                        + [N_MULTI + int(rng.integers(N_ONEHOT))]
                        + [N_MULTI + N_ONEHOT + int(x) for x in rng.choice(N_TAIL, 2, replace=False)])
        return Data(rp, col, rng.uniform(0.5, 1.5, col.size).astype(np.float32),
                    rng.integers(1, 6, n).astype(np.float32), n_main)

    tr, te = main(N_TR), main(N_TE)

    def block_row(r):
        items = [ROWS + int(x) for x in rng.choice(N_ITEMS, 3, replace=False)]
        return [r] + items + ([items[0]] if r == 0 else [])

    rp, col = _rows(rng, ROWS, block_row)
    val = rng.uniform(0.5, 1.5, col.size).astype(np.float32)
    if huge:
        val[2] = np.float32(3e19)
    blk = Data(rp, col, val, np.zeros(ROWS, np.float32), ROWS + N_ITEMS)
    block = dict(data=blk, train=rng.integers(0, ROWS, N_TR).astype(np.uint32),
                 test=rng.integers(0, ROWS, N_TE).astype(np.uint32), groups=None, binary=True)
    return tr, te, block, n_main


def _runs(rows, seg):
    """the greedy run cut of cut_runs over all ids, with a cut at every segment start; rows: each case's ids"""
    n = seg[-1]
    prev = np.zeros(n, np.int64)
    for ids in rows:
        s = sorted(set(ids))
        for a, b in zip(s, s[1:]):
            prev[b] = max(prev[b], a + 1)
    runs = [0]
    for j in range(1, n):
        if (prev[j] and prev[j] - 1 >= runs[-1]) or j in seg[:-1]:
            runs.append(j)
    return runs + [n]


def _stretches(runs, lo, hi, warps):
    """the plan's launches for the runs that start in [lo, hi)"""
    kinds = [runs[r + 1] - runs[r] <= warps for r in range(len(runs) - 1) if lo <= runs[r] < hi]
    return sum(1 for i, k in enumerate(kinds) if i == 0 or k != kinds[i - 1]), len(kinds)


def _learner(tr, te, block, n_main, tmp, mode, variant, threads, sample):
    stem = os.path.join(tmp, "rel")
    write_block_files(stem, block, N_TR, N_TE)
    b = RelationData.load(stem)
    rel = [(b, RelationJoin.load(stem + ".train", N_TR, b), RelationJoin.load(stem + ".test", N_TE, b))]
    n = n_main + b.num_feature
    l = FmLearnSgdElement(FmModel(n, K), mode=mode)
    l.set_tuning(threads=threads, variant=variant)
    l.upload(tr, 0)
    l.upload(te, 1)
    l.fm.init(42)
    l.fm.w = np.random.default_rng(1).standard_normal(n) * 0.1
    l.push_params()
    l.min_target, l.max_target = 1.0, 5.0
    reg = 0.0 if sample else 0.1
    l.mcmc_begin(tr, te, sample, sample, reg, np.full(2, reg), np.full((2, K), reg), relations=rel)
    return l, b


def _state(l, te):
    l.pull_params()
    h = l.mcmc_hyper()
    return [np.array(x, copy=True) for x in [[l.fm.w0], l.fm.w, l.fm.v] + [h[x] for x in ("alpha", "w_mu", "w_lambda",
                                                                                        "v_mu", "v_lambda")]
            + list(l.mcmc_pred(te))]


@pytest.mark.parametrize("threads", [256, 1024])
def test_plan_launches(threads, tmp_path, built_lib):
    """narrow stretches go to one CTA launch each, wide runs to the cooperative kernel: the extra launches per
    iteration are (1 + k) x (stretches - 1) per segment, the stretches counted from the run widths"""
    tr, te, block, n_main = _case(False)
    rows = [tr.col[tr.row_ptr[c]:tr.row_ptr[c + 1]].tolist() for c in range(N_TR)]
    d = block["data"]
    rows += [[n_main + int(j) for j in d.col[d.row_ptr[r]:d.row_ptr[r + 1]]] for r in range(ROWS)]
    n = n_main + d.num_feature
    runs = _runs(rows, [0, n_main, n])
    main_st, main_runs = _stretches(runs, 0, n_main, threads // 32)
    blk_st, blk_runs = _stretches(runs, n_main, n, threads // 32)
    assert main_st == 3 and blk_st == 2     # narrow, wide, narrow | wide, narrow
    launches = []
    for variant in (0, 1):
        l, _ = _learner(tr, te, block, n_main, str(tmp_path), MODE_INORDER, variant, threads, True)
        assert l.mcmc_runs() == main_runs + blk_runs == len(runs) - 1
        l.mcmc_iteration()
        before = l.kernel_launches()
        l.mcmc_iteration()
        launches.append(l.kernel_launches() - before)
        l.close()
    assert launches[0] - launches[1] == (1 + K) * (main_st - 1 + blk_st - 1)


@pytest.mark.parametrize("mode", [MODE_INORDER, MODE_ORDERED], ids=["inorder", "ordered"])
@pytest.mark.parametrize("method", ["mcmc", "als_nonfinite"])
def test_plan_matches_cooperative_sweep(method, mode, tmp_path, built_lib):
    """the planned sweeps (default CTA width, and 1024 threads) against the cooperative kernel alone, bit for bit
    after every iteration; ALS meets non-finite draws and counts them the same way"""
    sample, huge = method == "mcmc", method != "mcmc"
    tr, te, block, n_main = _case(huge)
    libc = C.CDLL(None)
    got = []
    for v, t in ((1, 0), (0, 0), (0, 1024)):   # the cooperative kernel alone, the default CTA width, 1024 threads
        l = _learner(tr, te, block, n_main, str(tmp_path), mode, v, t, sample)[0]
        libc.srand(7)   # the draws come from the process's rand() stream: each learner starts it afresh
        got.append([(l.mcmc_iteration(), _state(l, te)) for _ in range(4)])
        l.close()
    nonfinite = 0
    for it in range(4):
        (m0, c0), s0 = got[0][it]
        for (m, c), s in (g[it] for g in got[1:]):
            assert np.float64(m).tobytes() == np.float64(m0).tobytes(), it
            assert c.tolist() == c0.tolist(), it
            for i, (a, b) in enumerate(zip(s, s0)):
                assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), "iteration %d: field %d differs" % (it, i)
        nonfinite += int(c0[4:8].sum())
    assert (nonfinite > 0) == huge
