"""GPU: reuse and release of the library's device buffers.

A slot keeps its buffers across uploads that fit and grows them for one that does not; the ORDERED index and
its scratch, the prediction staging, the per-block partials and the MCMC state are rebuilt or regrown on demand;
fmb200_destroy releases everything a context holds.  Each result below must equal what a fresh context gives.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import make_learner
from libfm_b200 import MODE_HOGWILD, MODE_INORDER, synth
from libfm_b200.model import _LibcRand
from test_ordered_gpu import _cfg, _host_index, _port, _rand_init

pytestmark = pytest.mark.gpu

N, K = 1000, 8  # every set below has ids < N: all of them fit one context


def _sets():
    small = synth.ragged(3_000, N, 6, seed=21)
    large = synth.two_field(60_000, 600, 400, seed=22)
    return small, large


def test_slot_regrows_and_rebuilds_ordered_index(built_lib):
    """slot 0: a large set with its index, a smaller one into the same buffers, then one larger than the first"""
    seq = [synth.two_field(60_000, 600, 400, seed=1), synth.ragged(20_000, N, 6, seed=2),
           synth.two_field(120_000, 600, 400, seed=3)]
    cfg = _cfg(N, K)
    init = _rand_init(N, K, 4)
    l = make_learner(cfg, init, mode=MODE_INORDER)
    for i, d in enumerate(seq):
        l.upload(d, 0)
        link, rowdep = l.ordered_index(d)
        want_link, want_rowdep = _host_index(d)
        assert np.array_equal(link, want_link), i
        assert np.array_equal(rowdep, want_rowdep), i
        l.fm.w0, l.fm.w, l.fm.v = init[0], init[1].copy(), init[2].copy()
        l.push_params()
        p = _port(cfg, init)
        l.sgd_epoch(d)
        p.sgd_epoch(d, 0, cfg["lr"], cfg["min_target"], cfg["max_target"])
        l.pull_params()
        assert l.fm.w0 == p.w0.value and np.array_equal(l.fm.w, p.w) and np.array_equal(l.fm.v, p.v), i
    l.close()


def _outputs(l, d, mode):
    out = [l.evaluate(d), l.last_mae, l.predict(d), l.predict(d, transform=False)]
    if mode == MODE_INORDER:
        out.append(l.mcmc_eterms(d))
    return out


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()


@pytest.mark.parametrize("mode", [MODE_INORDER, MODE_HOGWILD])
def test_scratch_regrows_for_evaluate_predict_eterms(mode, built_lib):
    """small slot, large slot, small slot again: the staging grows and is reused, results do not change"""
    small, large = _sets()
    cfg = _cfg(N, K)
    init = _rand_init(N, K, 5)
    l = make_learner(cfg, init, mode=mode)
    l.upload(small, 0)
    l.upload(large, 1)
    got = [_outputs(l, d, mode) for d in (small, large, small)]
    l.close()
    for d, g in zip((small, large, small), got):
        f = make_learner(cfg, init, mode=mode)
        _same(g, _outputs(f, d, mode))
        f.close()


def _mcmc_run(l, tr, te, seed):
    init = _rand_init(N, K, 6)
    l.fm.w0, l.fm.w, l.fm.v = init[0], init[1].copy(), init[2].copy()
    l.push_params()
    _LibcRand().srand(seed)
    l.mcmc_begin(tr, te, True, True, 0.0, np.full(1, 2.0), np.full((1, K), 2.0))
    runs = l.mcmc_runs()
    m, cnt = l.mcmc_iteration()
    l.pull_params()
    h = l.mcmc_hyper()
    return [runs, m, cnt, l.fm.w0, l.fm.w, l.fm.v, h["alpha"], h["w_mu"], h["w_lambda"], h["v_mu"], h["v_lambda"],
            *l.mcmc_pred(te)]


def test_mcmc_begin_after_reupload(built_lib):
    """mcmc_begin, new data into the train slot, mcmc_begin again: the state is rebuilt for the new data"""
    first = synth.two_field(40_000, 600, 400, seed=7)
    second = synth.ragged(30_000, N, 5, seed=8)
    te = synth.two_field(5_000, 600, 400, seed=9)
    cfg = _cfg(N, K)
    l = make_learner(cfg, _rand_init(N, K, 6), mode=MODE_INORDER)
    l.upload(first, 0)
    l.upload(te, 1)
    _mcmc_run(l, first, te, 11)
    l.upload(second, 0)
    got = _mcmc_run(l, second, te, 12)
    l.close()
    f = make_learner(cfg, _rand_init(N, K, 6), mode=MODE_INORDER)
    f.upload(second, 0)
    f.upload(te, 1)
    want = _mcmc_run(f, second, te, 12)
    f.close()
    _same(got, want)


def test_destroy_with_every_buffer_then_train(built_lib):
    """a context holding two indexed slots, SGDA and MCMC state, the row-lane accumulator and a local peer
    attach is destroyed cleanly; a new context then trains"""
    small, large = _sets()
    cfg = _cfg(N, K)
    a = make_learner(cfg, _rand_init(N, K, 1), mode=MODE_INORDER)
    b = make_learner(cfg, _rand_init(N, K, 2), mode=MODE_HOGWILD)
    a.upload(small, 0)
    a.upload(large, 1)
    a.ordered_index(small)
    a.ordered_index(large)
    a.sgda_begin()
    a.sgda_epoch(large, small, True)
    a.mcmc_begin(large, small, True, True, 0.0, np.full(1, 2.0), np.full((1, K), 2.0))
    a.set_mode(MODE_HOGWILD)
    a.sgd_epoch(large)  # two-field, k = 8: the reproducible row-lane epoch and its accumulator
    assert a.epoch_config()["lanes_per_row"] == 1
    arr = (C.c_void_p * 2)(a._ctx, b._ctx)
    assert a.lib.fmb200_peer_attach_local(a._ctx, 2, 0, arr) == 0, a.lib.fmb200_last_error()
    a.close()
    b.close()
    c = make_learner(cfg, _rand_init(N, K, 3), mode=MODE_HOGWILD)
    before = c.evaluate(large)
    for _ in range(3):
        c.sgd_epoch(large)
    after = c.evaluate(large)
    assert np.isfinite(after) and after < before
    c.close()
