import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")
GOLDEN_CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); select with -m gpu")


def load_golden(name):
    from libfm_b200 import Data
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    n = int(z["n"])
    tr = Data(z["tr_row_ptr"], z["tr_col"], z["tr_val"], z["tr_target"], n)
    te = Data(z["te_row_ptr"], z["te_col"], z["te_val"], z["te_target"], n)
    return z, tr, te


def digest(a):
    """SHA-256 of an array's bytes: how tests/golden/reference/outputs.npz stores large results."""
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="session")
def ref_golden():
    """What the reference computed for the inputs of the tests that compare against it
    (scripts/make_ref_golden.py)."""
    return np.load(os.path.join(GOLDEN, "reference", "outputs.npz"))


@pytest.fixture(scope="session")
def built_lib():
    """libfmb200.so must exist (built by __graft_entry__.build / libfm_b200.build)."""
    from libfm_b200 import _capi, build
    if not os.path.exists(_capi.LIB_PATH):
        build.build_lib()
    return _capi.load()


def make_learner(z_or_cfg, fm_init, device=0, mode=0):
    """Build an FmLearnSgdElement from a golden record / config dict and initial params."""
    from libfm_b200 import FmLearnSgdElement, FmModel
    n, k = int(z_or_cfg["n"]), int(z_or_cfg["k"])
    fm = FmModel(n, k, bool(z_or_cfg["k0"]), bool(z_or_cfg["k1"]))
    fm.w0, fm.w, fm.v = fm_init
    fm.w = np.array(fm.w, dtype=np.float64)
    fm.v = np.array(fm.v, dtype=np.float64).reshape(k, n)
    regs = z_or_cfg["regs"]
    fm.reg0, fm.regw, fm.regv = float(regs[0]), float(regs[1]), float(regs[2])
    l = FmLearnSgdElement(fm, device=device, mode=mode)
    l.task = int(z_or_cfg["task"])
    l.learn_rate = float(z_or_cfg["lr"])
    l.min_target = float(z_or_cfg["min_target"])
    l.max_target = float(z_or_cfg["max_target"])
    l.push_hparams()
    return l
