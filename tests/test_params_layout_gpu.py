"""GPU: the packed fp32 state puts w and V on 128-byte lines, and nothing but the parameters is non-zero.

A k = 8 factor row is then exactly one 32-byte L2 sector (fm_rowlane.cu gathers and reduces whole sectors), a
longer row fills the sectors and lines it touches, and the kernels that walk the whole buffer (fold, scale,
peer exchange) find zeros in the padding.
"""
import numpy as np
import pytest
import torch

from libfm_b200 import FmLearnSgdElement, FmModel, MODE_HOGWILD

pytestmark = pytest.mark.gpu


class _DevBuf:
    def __init__(self, ptr, n_floats):
        self.__cuda_array_interface__ = {"shape": (n_floats,), "typestr": "<f4", "data": (ptr, False), "version": 2}


# (features, factors): linear weights one per sector (ws = 8) up to 131 072 features, packed (ws = 1) above;
# feature counts that are no multiple of anything, so that both paddings are non-empty
@pytest.mark.parametrize("n,k,ws", [(9_746, 8, 8), (1_003, 5, 8), (131_075, 8, 1), (140_001, 64, 1)])
def test_w_and_v_start_on_lines_and_params_round_trip(n, k, ws, built_lib):
    fm = FmModel(n, k)
    fm.init_stdev = 0.1
    fm.init_numpy(3)
    rng = np.random.default_rng(5)
    fm.w0 = float(np.float32(0.25))
    fm.w = rng.standard_normal(n).astype(np.float32).astype(np.float64)
    fm.v = np.asarray(fm.v, dtype=np.float32).astype(np.float64)
    w0, w, v = fm.w0, fm.w.copy(), fm.v.copy()
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    try:
        lay = l.params_layout()
        kp = (k + 3) & ~3
        assert (lay["ws"], lay["kp"]) == (ws, kp)
        assert lay["off_w"] * 4 % 128 == 0 and lay["off_v"] * 4 % 128 == 0
        assert lay["off_w"] >= 1 and lay["off_v"] >= lay["off_w"] + n * ws
        ptr, n_floats = l.params_device()
        assert ptr % 256 == 0 and n_floats == lay["off_v"] + n * kp and n_floats % 4 == 0
        state = torch.as_tensor(_DevBuf(ptr, n_floats), device="cuda").cpu().numpy()
        want = np.zeros(n_floats, dtype=np.float32)
        want[0] = w0
        want[lay["off_w"]:lay["off_w"] + n * ws:ws] = w
        want[lay["off_v"]:].reshape(n, kp)[:, :k] = v.T
        assert np.array_equal(state, want)
        l.pull_params()
        assert l.fm.w0 == w0 and np.array_equal(l.fm.w, w) and np.array_equal(l.fm.v, v)
    finally:
        l.close()
