"""Record what the SGDA window model (oracle/sgda_window_model.py) computes on long rows as SHA-256 digests.

    python scripts/make_sgda_model_digests.py OUT.json

Two epochs (the first without lambda-steps) of sgda_window_epoch with its default arguments, on rows of 0-60
entries that name features two and three times, at k = 33 and k = 100 with three groups.  After each epoch: a
digest of the state, the SGDA state (stored gradients, reg), the moments and both budgets.
tests/test_sgda_window_model.py recomputes them and compares against tests/golden/sgda_window_model_digests.json,
so a change to the model that moves any of these by one bit at the default arguments fails there.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from conftest import digest  # noqa: E402
from libfm_b200 import Data, synth  # noqa: E402
from oracle import HParams, State  # noqa: E402
from oracle import sgda_window_model as sm  # noqa: E402

# name: (k, task, damp, W, seed)
CASES = {"k33_damped": (33, 0, True, 64, 21), "k100_classification_undamped": (100, 1, False, 50, 22)}


def long_case(name):
    """(train, val, state, sgda, hp, W, damp) of a case: 600 training and 150 validation rows, 150 features."""
    k, task, damp, W, seed = CASES[name]
    train, val = synth.split_rows(synth.long_rows(750, 150, 60, seed=seed), 600)
    if task:
        train, val = [Data(d.row_ptr, d.col, d.val, np.where(d.target > 3, 1.0, -1.0).astype(np.float32),
                           d.num_feature) for d in (train, val)]
    n = train.num_feature
    r = np.random.default_rng(seed)
    v = np.asarray(0.02 * r.standard_normal((k, n)), dtype=np.float32).astype(np.float64)
    hp = HParams(task, 0.002, min_target=1.0, max_target=5.0)
    return train, val, State(0.0, np.zeros(n), v), sm.Sgda.begin(n, k, np.arange(n) % 3), hp, W, damp


def model_digests(name, **kw):
    """[{quantity: digest}] after each of two epochs; kw goes to sgda_window_epoch."""
    train, val, st, sg, hp, W, damp = long_case(name)
    bud = rb = None
    out = []
    for e in range(2):
        st, sg, mom, bud, rb = sm.sgda_window_epoch(st, sg, train, val, hp, W, e > 0, damp=damp, budget=bud,
                                                    reg_budget=rb, **kw)
        out.append({q: digest(np.float64(x) if np.isscalar(x) else x) for q, x in [
            ("w0", st.w0), ("w", st.w), ("v", st.v), ("grad_w", sg.grad_w), ("grad_v", sg.grad_v),
            ("reg_w", sg.reg_w), ("reg_v", sg.reg_v), ("var_w", mom[0]), ("var_v", mom[1]),
            ("budget_w0", bud.w0), ("budget_w", bud.w), ("budget_v", bud.v), ("bound_reg_w", rb.reg_w),
            ("bound_reg_v", rb.reg_v), ("bound_var_w", rb.var_w), ("bound_var_v", rb.var_v)]})
    return out


if __name__ == "__main__":
    with open(sys.argv[1], "w") as f:
        json.dump({name: model_digests(name) for name in CASES}, f, indent=1, sort_keys=True)
        f.write("\n")
