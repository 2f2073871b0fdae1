"""GPU: out-of-core MCMC and ALS (fmb200_mcmc_begin_xt) against the reference, bit for bit.

The data sets of tests/golden/reference/mcmc.npz and mcmc_c4.npz are written as .xt files (write_transposed)
and streamed in the blocks the command line plans under -cache_size (read_xblocks).  Every iteration must equal
the reference's, exactly as the resident runs of test_mcmc_sweep_gpu.py do.  The command line runs of
mcmc_cli.npz are in test_stream_mcmc_cli_gpu.py.
"""
import os

import numpy as np
import pytest

from libfm_b200 import MODE_INORDER, FmError, FmLearnSgdElement, FmModel, synth
from libfm_b200.model import XtBlocks, write_transposed
from test_mcmc_sweep_gpu import ITERS, _cases, _data, _digest, _first_difference, _reference_init, _z

pytestmark = pytest.mark.gpu


def cache_for(path_xt, n_blocks):
    """A -cache_size whose plan of `path_xt` has at least n_blocks blocks (and admits its longest column)."""
    raw = np.fromfile(path_xt, dtype=np.uint32)
    n_rows, words = int(raw[4]), raw[6:]
    longest, pos = 0, 0
    for _ in range(n_rows):
        longest = max(longest, 4 + 8 * int(words[pos]))
        pos += 1 + 2 * int(words[pos])
    return 2 * max(longest, (4 * pos) // n_blocks)


def expected_runs(tr, n, col_lo):
    """The run count of the streamed sweep restated: the greedy cut of mcmc_begin plus one at every block start."""
    prev = np.zeros(n, dtype=np.int64)
    for r in range(tr.num_cases):
        ids = np.unique(tr.col[int(tr.row_ptr[r]):int(tr.row_ptr[r + 1])].astype(np.int64))
        if ids.size > 1:
            prev[ids[1:]] = np.maximum(prev[ids[1:]], ids[:-1] + 1)
    starts = set(int(c) for c in col_lo[1:-1] if 0 < c < n)
    runs = [0]
    for j in range(1, n):
        if (prev[j] != 0 and prev[j] - 1 >= runs[-1]) or j in starts:
            runs.append(j)
    return len(runs)


def _start_xt(z, name, tmp_path, n_blocks, stream_test=True):
    n, k, k0, k1, task, sample, ml, seed, tr_nf, te_nf = (int(x) for x in z[f"{name}/cfg"])
    tr, te = _data(z, name, "tr", tr_nf), _data(z, name, "te", te_nf)
    write_transposed(tr, str(tmp_path / "train.xt"))
    write_transposed(te, str(tmp_path / "test.xt"))
    xtr = XtBlocks(str(tmp_path / "train.xt"), tr.target, cache_for(str(tmp_path / "train.xt"), n_blocks), (2, 4))
    xte = XtBlocks(str(tmp_path / "test.xt"), te.target, cache_for(str(tmp_path / "test.xt"), n_blocks), (3, 5))
    l = FmLearnSgdElement(FmModel(n, k, k0, k1), mode=MODE_INORDER)
    if not stream_test:
        l.upload(te, 1)
    l.fm = _reference_init(n, k, k0, k1, seed)
    assert _digest(np.concatenate([[l.fm.w0], l.fm.w, l.fm.v.reshape(-1)])) == str(z[f"{name}/init_digest"])
    l.push_params()
    l.task = task
    l.min_target, l.max_target = (float(x) for x in z[f"{name}/minmax"])
    l.mcmc_begin_xt(xtr, xte if stream_test else te, sample, ml, float(z[f"{name}/reg0"]), z[f"{name}/wl"],
                    z[f"{name}/vl"], attr_group=z[f"{name}/group"], attr_per_group=z[f"{name}/per_group"])
    return l, tr, te, xtr, xte


def _resident_runs(z, name):
    n, k, k0, k1, *_ = (int(x) for x in z[f"{name}/cfg"])
    tr_nf, te_nf = (int(x) for x in z[f"{name}/cfg"][8:10])
    tr, te = _data(z, name, "tr", tr_nf), _data(z, name, "te", te_nf)
    l = FmLearnSgdElement(FmModel(n, k, k0, k1), mode=MODE_INORDER)
    l.push_params()
    l.mcmc_begin(tr, te, True, True, 0.0, np.zeros(1), np.zeros((1, k)))
    runs = l.mcmc_runs()
    l.close()
    return runs


@pytest.mark.parametrize("n_blocks", [3, 20])
@pytest.mark.parametrize("name", _cases())
def test_streamed_iterations_bit_identical_to_reference(name, n_blocks, tmp_path, built_lib):
    z = _z()
    l, tr, te, xtr, xte = _start_xt(z, name, tmp_path, n_blocks)
    assert xtr.n_blocks >= n_blocks and xte.n_blocks >= n_blocks
    n, k, k0, k1 = (int(x) for x in z[f"{name}/cfg"][:4])
    runs = l.mcmc_runs()
    assert runs == expected_runs(tr, n, xtr.col_lo)  # the resident cut and a cut at every block start
    assert runs >= _resident_runs(z, name)
    # begin: the prev pass and the e-term passes over train, the e-term passes over test
    eterm = k + k1
    assert xtr.fetches == xtr.n_blocks * (1 + eterm) and xte.fetches == xte.n_blocks * eterm
    for t in range(ITERS):
        m, cnt = l.mcmc_iteration()
        bad = _first_difference(z, name, t, l, te, m, cnt)
        assert bad is None, "%s: iteration %d: %s differs from the reference" % (name, t, bad)
    sweep = (1 if (k1 or k) else 0) + k  # DESIGN 3.8: the passes of one iteration
    assert xtr.fetches == xtr.n_blocks * (1 + eterm + ITERS * (sweep + eterm))
    assert xte.fetches == xte.n_blocks * eterm * (1 + ITERS)
    l.close()


def test_streamed_train_resident_test(tmp_path, built_lib):
    """train and test decide independently: a streamed train set beside a resident test set"""
    z = _z()
    name = "ragged_meta_mcmc"
    l, tr, te, _, _ = _start_xt(z, name, tmp_path, 5, stream_test=False)
    for t in range(3):
        m, cnt = l.mcmc_iteration()
        bad = _first_difference(z, name, t, l, te, m, cnt)
        assert bad is None, "%s: iteration %d: %s differs from the reference" % (name, t, bad)
    l.close()


def _corrupt(path, word, value):
    raw = np.fromfile(path, dtype=np.uint32)
    raw[word] = value
    raw.tofile(path)


def test_refuses_a_corrupt_column_header(tmp_path, built_lib):
    z = _z()
    name = "twofield_mcmc"
    n, k, k0, k1, *_ = (int(x) for x in z[f"{name}/cfg"])
    tr = _data(z, name, "tr", int(z[f"{name}/cfg"][8]))
    te = _data(z, name, "te", int(z[f"{name}/cfg"][9]))
    p = str(tmp_path / "train.xt")
    write_transposed(tr, p)
    x = XtBlocks(p, tr.target, cache_for(p, 4))
    # column 0 of block 1: its header word is read into the block as it stands, and disagrees with its size
    lo, _, words, sizes = x.blocks[1]
    words[0] = sizes[0] + 1
    l = FmLearnSgdElement(FmModel(n, k, k0, k1), mode=MODE_INORDER)
    l.push_params()
    with pytest.raises(FmError, match=r"column %d of the \.xt: its header word is not its size" % lo):
        l.mcmc_begin_xt(x, te, True, True, 0.0, np.zeros(1), np.zeros((1, k)))
    l.close()


def test_refuses_a_case_id_out_of_range(tmp_path, built_lib):
    z = _z()
    name = "twofield_mcmc"
    n, k, k0, k1, *_ = (int(x) for x in z[f"{name}/cfg"])
    tr = _data(z, name, "tr", int(z[f"{name}/cfg"][8]))
    te = _data(z, name, "te", int(z[f"{name}/cfg"][9]))
    p = str(tmp_path / "train.xt")
    write_transposed(tr, p)
    x = XtBlocks(p, tr.target, cache_for(p, 4))
    x.blocks[2][2][1] = tr.num_cases  # the first entry's case id of block 2
    l = FmLearnSgdElement(FmModel(n, k, k0, k1), mode=MODE_INORDER)
    l.push_params()
    with pytest.raises(FmError, match=r"case id %d .* out of range" % tr.num_cases):
        l.mcmc_begin_xt(x, te, True, True, 0.0, np.zeros(1), np.zeros((1, k)))
    l.close()


def test_c4_shape_full_size_streamed(tmp_path, built_lib):
    """BASELINE config C4 at full size (10 000 054 cases, k = 16), train streamed in at least 8 blocks and test
    in at least 2: 2 MCMC iterations against digests of the reference's (tests/golden/reference/mcmc_c4.npz)."""
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference", "mcmc_c4.npz"))
    name = "c4_mcmc"
    n, k, k0, k1, task, sample, ml, seed, _, _ = (int(x) for x in z[f"{name}/cfg"])
    tr = synth.two_field(10_000_054, 71_567, 10_681, seed=5)
    te = synth.two_field(200_000, 71_567, 10_681, seed=6)
    write_transposed(tr, str(tmp_path / "train.xt"))
    write_transposed(te, str(tmp_path / "test.xt"))
    xtr = XtBlocks(str(tmp_path / "train.xt"), tr.target, cache_for(str(tmp_path / "train.xt"), 8), (2, 4))
    xte = XtBlocks(str(tmp_path / "test.xt"), te.target, cache_for(str(tmp_path / "test.xt"), 2), (3, 5))
    assert xtr.n_blocks >= 8 and xte.n_blocks >= 2
    l = FmLearnSgdElement(FmModel(n, k, k0, k1), mode=MODE_INORDER)
    l.fm = _reference_init(n, k, k0, k1, seed)
    assert _digest(np.concatenate([[l.fm.w0], l.fm.w, l.fm.v.reshape(-1)])) == str(z[f"{name}/init_digest"])
    l.push_params()
    l.task = task
    l.min_target, l.max_target = (float(x) for x in z[f"{name}/minmax"])
    l.mcmc_begin_xt(xtr, xte, sample, ml, float(z[f"{name}/reg0"]), np.zeros(1), np.zeros((1, k)),
                    attr_per_group=np.array([n], np.uint32))
    assert l.mcmc_runs() >= 2
    for t in range(2):
        m, cnt = l.mcmc_iteration()
        bad = _first_difference(z, name, t, l, te, m, cnt)
        assert bad is None, "%s: iteration %d: %s differs from the reference" % (name, t, bad)
    l.close()
