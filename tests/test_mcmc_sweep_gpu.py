"""GPU: MCMC and ALS learning (fmb200_mcmc_*) against the reference's fm_learn_mcmc_simultaneous, bit for bit.

tests/golden/reference/mcmc.npz (scripts/make_mcmc_golden.py) holds what the reference leaves after each of
its first 7 iterations.  Each case seeds libc rand() and initialises the model as libfm.cpp does (fm.init(),
then w ~ N(0, 0.1)) in this process, so the library's draws continue the same stream.  After every iteration
w0, w, v, the hyperparameters, the NaN/Inf counters, the three test prediction vectors and the #Iter Train
value must equal the reference's; a failure names the first iteration and parameter that differ.
Classification also goes through host libm (the truncated normals); a difference there shows up the same way.
"""
import hashlib
import os

import numpy as np
import pytest

from libfm_b200 import MODE_HOGWILD, MODE_INORDER, Data, FmError, FmLearnSgdElement, FmModel, synth
from libfm_b200.model import _LibcRand

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference", "mcmc.npz")
ITERS = 7
COUNTER_NAMES = ["alpha", "w0", "w", "v", "w_mu", "w_lambda", "v_mu", "v_lambda"]


def _z():
    return np.load(GOLDEN)


def _cases():
    return sorted({k.split("/")[0] for k in _z().files})


def _digest(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()


def _data(z, name, p, nf):
    return Data(z[f"{name}/{p}_row_ptr"], z[f"{name}/{p}_col"], z[f"{name}/{p}_val"], z[f"{name}/{p}_target"], nf)


def _reference_init(n, k, k0, k1, seed):
    """srand(seed); fm_model::init; fm.w.init_normal(0, 0.1) (libfm.cpp:115-116,257,283) on this process's rand()"""
    fm = FmModel(n, k, k0, k1)
    fm.init_stdev = 0.1
    fm.init(seed)
    rng = _LibcRand()
    fm.w = np.array([0.0 + 0.1 * rng.gaussian() for _ in range(n)])
    return fm


def _start(z, name, mode=MODE_INORDER):
    n, k, k0, k1, task, sample, ml, seed, tr_nf, te_nf = (int(x) for x in z[f"{name}/cfg"])
    tr, te = _data(z, name, "tr", tr_nf), _data(z, name, "te", te_nf)
    l = FmLearnSgdElement(FmModel(n, k, k0, k1), mode=mode)
    l.upload(tr, 0)   # the device work before the seed: nothing may draw from rand() after srand
    l.upload(te, 1)
    l.fm = _reference_init(n, k, k0, k1, seed)
    state = np.concatenate([[l.fm.w0], l.fm.w, l.fm.v.reshape(-1)])
    assert _digest(state) == str(z[f"{name}/init_digest"]), "model init does not reproduce the reference's"
    l.push_params()
    l.task = task
    l.min_target, l.max_target = (float(x) for x in z[f"{name}/minmax"])
    l.mcmc_begin(tr, te, sample, ml, float(z[f"{name}/reg0"]), z[f"{name}/wl"], z[f"{name}/vl"],
                 attr_group=z[f"{name}/group"], attr_per_group=z[f"{name}/per_group"])
    return l, tr, te


def _first_difference(z, name, t, l, te, train_metric, counters):
    G = l._mcmc_groups
    l.pull_params()
    h = l.mcmc_hyper()
    hyper = np.concatenate([[h["alpha"]], h["w_mu"], h["w_lambda"], h["v_mu"].reshape(-1), h["v_lambda"].reshape(-1)])
    want = z[f"{name}/{t}/hyper"]
    pt, pa, pb = l.mcmc_pred(te)
    checks = [("w0", np.float64(l.fm.w0).tobytes() == np.float64(z[f"{name}/{t}/w0"]).tobytes()),
              ("w", _digest(l.fm.w) == str(z[f"{name}/{t}/w"])),
              ("v", _digest(l.fm.v) == str(z[f"{name}/{t}/v"])),
              ("alpha", hyper[0].tobytes() == want[0].tobytes()),
              ("w_mu", hyper[1:1 + G].tobytes() == want[1:1 + G].tobytes()),
              ("w_lambda", hyper[1 + G:1 + 2 * G].tobytes() == want[1 + G:1 + 2 * G].tobytes()),
              ("v_mu/v_lambda", hyper[1 + 2 * G:].tobytes() == want[1 + 2 * G:].tobytes()),
              ("counters", np.array_equal(counters, z[f"{name}/{t}/counters"])),
              ("pred_this", _digest(pt) == str(z[f"{name}/{t}/pred_this"])),
              ("pred_sum_all", _digest(pa) == str(z[f"{name}/{t}/pred_sum_all"])),
              ("pred_sum_all_but5", _digest(pb) == str(z[f"{name}/{t}/pred_sum_all_but5"])),
              ("#Iter Train", "Train=%g\t" % train_metric in str(z[f"{name}/{t}/line"]))]
    for what, ok in checks:
        if not ok:
            return what
    return None


@pytest.mark.parametrize("name", _cases())
def test_iterations_bit_identical_to_reference(name, built_lib):
    z = _z()
    l, tr, te = _start(z, name)
    for t in range(ITERS):
        m, cnt = l.mcmc_iteration()
        bad = _first_difference(z, name, t, l, te, m, cnt)
        assert bad is None, "%s: iteration %d: %s differs from the reference" % (name, t, bad)
    l.close()


def test_two_field_data_gives_two_runs(built_lib):
    """one-hot (user, item): users never share a case, items never do -> the sweep walks 2 runs"""
    z = _z()
    l, _, _ = _start(z, "twofield_mcmc")
    assert l.mcmc_runs() == 2
    l.close()
    l, _, _ = _start(z, "ragged_meta_mcmc")
    assert l.mcmc_runs() > 2
    l.close()


def test_diverged_sampled_run_stops_with_error(built_lib):
    """A non-finite state gives a draw the reference would skip without consuming a random number: the
    library stops, naming the parameter and the iteration, instead of desynchronising the stream."""
    z = _z()
    l, tr, te = _start(z, "twofield_mcmc")
    l.pull_params()
    l.fm.v[0, int(tr.col[0])] = np.inf
    l.push_params()
    l.mcmc_begin(tr, te, True, True, 0.0, np.zeros(1), np.zeros((1, l.fm.num_factor)))
    with pytest.raises(FmError, match=r"iteration 0: a draw of v\[f=0\].*posterior variance"):
        l.mcmc_iteration()
    l.close()


def test_refuses_fp32_state(built_lib):
    d = synth.two_field(500, 30, 20, seed=3)
    l = FmLearnSgdElement(FmModel(d.num_feature, 4), mode=MODE_HOGWILD)
    with pytest.raises(FmError, match="fp64"):
        l.mcmc_begin(d, d, True, True, 0.0, np.zeros(1), np.zeros((1, 4)))
    l.close()


def test_c4_shape_full_size(built_lib):
    """BASELINE config C4 at full size (10 000 054 cases, 82 248 features, items with tens of thousands of
    cases, k = 16): 2 MCMC iterations against digests of the reference's (tests/golden/reference/mcmc_c4.npz)."""
    z = np.load(os.path.join(os.path.dirname(GOLDEN), "mcmc_c4.npz"))
    name = "c4_mcmc"
    n, k, k0, k1, task, sample, ml, seed, _, _ = (int(x) for x in z[f"{name}/cfg"])
    tr = synth.two_field(10_000_054, 71_567, 10_681, seed=5)
    te = synth.two_field(200_000, 71_567, 10_681, seed=6)
    l = FmLearnSgdElement(FmModel(n, k, k0, k1), mode=MODE_INORDER)
    l.upload(tr, 0)
    l.upload(te, 1)
    l.fm = _reference_init(n, k, k0, k1, seed)
    assert _digest(np.concatenate([[l.fm.w0], l.fm.w, l.fm.v.reshape(-1)])) == str(z[f"{name}/init_digest"])
    l.push_params()
    l.task = task
    l.min_target, l.max_target = (float(x) for x in z[f"{name}/minmax"])
    l.mcmc_begin(tr, te, sample, ml, float(z[f"{name}/reg0"]), np.zeros(1), np.zeros((1, k)),
                 attr_per_group=np.array([n], np.uint32))
    assert l.mcmc_runs() == 2
    for t in range(2):
        m, cnt = l.mcmc_iteration()
        bad = _first_difference(z, name, t, l, te, m, cnt)
        assert bad is None, "%s: iteration %d: %s differs from the reference" % (name, t, bad)
    l.close()
