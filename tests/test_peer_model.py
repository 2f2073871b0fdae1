"""CPU: the fp64 model of the peer exchange (oracle/peer_model.py) states the rule it claims to.

gamma's limits and cut, a two-replica combine worked by hand, and agreement with the torch restatement of the
same rule that the NCCL path runs (libfm_b200/dist.py: combine_meanfield_) at world 2, 3 and 4 -- the only
check of worlds above 2, which tests/test_peer_exchange_gpu.py cannot run on one device.
"""
import numpy as np
import pytest
import torch

from libfm_b200 import dist
from oracle import HParams
from oracle import peer_model as pm


def _layout(n, k, ws):
    kp = (k + 3) & ~3
    off_w = 32
    off_v = off_w + ((n * ws + 31) & ~31)
    return {"off_w": off_w, "ws": ws, "off_v": off_v, "kp": kp, "n": n}


def test_gamma_limits_and_cut():
    for G in (2, 3, 4, 8):
        assert pm.gamma(0.0, G) == 1.0
        assert pm.gamma(1e-6, G) == 1.0  # the cut: u <= 1e-6 sums
        just = pm.gamma(1.01e-6, G)
        assert just < 1.0 and abs(1.0 - just - (G - 1) / 2 * 1.01e-6) < 1e-11  # 1 - (G-1) u / 2
        assert abs(pm.gamma(1e-3, G) - (1 - (G - 1) / 2 * 1e-3)) < G * G * 1e-6  # + O(G^2 u^2)
        assert abs(pm.gamma(50.0, G) - 1.0 / G) < 1e-15  # a converged parameter is averaged
        u = np.logspace(-5, 1, 200)
        g = pm.gamma(u, G)
        assert np.all(np.diff(g) < 0) and np.all(g > 1.0 / G) and np.all(g < 1.0)
        # the closed-form derivative against a central difference
        h = u * 1e-4
        fd = (pm.gamma(u + h, G) - pm.gamma(u - h, G)) / (2 * h)
        np.testing.assert_allclose(pm.gamma_prime(u, G), fd, rtol=1e-5, atol=1e-9)
    # G = 2: (1 - e^{-2u}) / (2 (1 - e^{-u})) = (1 + e^{-u}) / 2
    np.testing.assert_allclose(pm.gamma([0.5, 2.0], 2), (1 + np.exp([-0.5, -2.0])) / 2, rtol=1e-15)


def test_mean_combine_is_the_rank_order_fp32_sum():
    a = np.float32([1.0, 3.0, 2.0 ** 24, 0.1])
    b = np.float32([2.0, -3.0, 1.0, 0.2])
    got = pm.mean_combine([a, b])
    assert got.dtype == np.float32
    want = np.float32([1.5, 0.0, 2.0 ** 23, np.float32(np.float32(0.1) + np.float32(0.2)) * np.float32(0.5)])
    assert np.array_equal(got, want)
    c = np.float32([1.0, 1.0, -(2.0 ** 24), 0.3])
    third = np.float32(np.float32(1) / np.float32(3))
    assert np.array_equal(pm.mean_combine([a, b, c]), ((a + b) + c) * third)


def test_two_replicas_by_hand():
    """n = 2 features, k = 1, ws = 8: bias, w[0], w[1], V[0][0], V[1][0]; everything else padding."""
    lay = _layout(2, 1, 8)
    lr, G = 0.5, 2
    hp = HParams(0, lr, reg0=0.0, regw=1.0, regv=0.25)
    th0 = pm.pack(1.0, [0.5, -0.5], np.array([[1.0, 0.0]]), lay, 1)
    r0 = pm.pack(1.5, [1.0, -0.5], np.array([[0.5, 0.0]]), lay, 1)
    r1 = pm.pack(2.0, [0.5, -0.5], np.array([[0.0, 0.0]]), lay, 1)
    r1[3] = 7.0  # a padding word a replica dirtied: gamma 0 keeps theta0's
    hv = pm.hv(th0, lay)
    assert hv == 0.5  # (1^2 + 0^2) / 2
    out, bud, g = pm.meanfield_combine(th0, [r0, r1], [[2, 0], [0, 0]], [4, 2], hv, hp, lay, 1)
    gam = lambda u: (1 - np.exp(-2 * u)) / (2 * (1 - np.exp(-u)))  # noqa: E731
    ow, ov = lay["off_w"], lay["off_v"]
    w0, w, v = out[0], out[[ow, ow + 8]], out[[ov, ov + 4]][None, :]
    assert abs(w0 - (1.0 + gam(lr * 3.0) * 1.5)) < 1e-15         # rows: mean 3; d = 0.5 + 1.0
    assert abs(w[0] - (0.5 + gam(lr * 2.0 * 1.0) * 0.5)) < 1e-15  # cnt 1, (1 + regw) = 2
    assert w[1] == -0.5                                            # d = 0
    assert abs(v[0, 0] - (1.0 + gam(lr * 0.75 * 1.0) * -1.5)) < 1e-15  # hv + regv = 0.75
    assert v[0, 1] == 0.0
    assert out[3] == 0.0 and g[3] == 0.0 and bud[3] == 0.0
    kind, _ = pm.layout_masks(lay, 1, th0.size)
    assert np.all(out[kind == 0] == th0[kind == 0]) and np.all(bud[kind > 0] > 0)
    # the budget: a few ulp of each moved element, not orders of magnitude more
    assert np.all(bud[[0, lay["off_w"], lay["off_v"]]] < 1e-6)


def _stub_allreduce(monkeypatch, sums):
    """torch.distributed.all_reduce(t, SUM) -> t := the next of `sums` (what the ranks' tensors add up to)."""
    import torch.distributed as tdist
    it = iter(sums)

    def all_reduce(t, op=None):
        t.copy_(next(it).to(t.dtype))
    monkeypatch.setattr(tdist, "all_reduce", all_reduce)


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("n,k,ws", [(37, 5, 8), (200, 8, 1), (64, 33, 8)])
def test_agrees_with_the_torch_restatement(world, n, k, ws, monkeypatch):
    """dist.combine_meanfield_ on CPU tensors (hv in fp64, gamma in fp32 torch): within the model's budget,
    with regularisation on and counts from u ~ 0 (cold features) to u >> 1 (hot ones)."""
    rng = np.random.default_rng(world * 1000 + n + k)
    lay = _layout(n, k, ws)
    hp = HParams(0, 0.05, reg0=0.1, regw=0.2, regv=0.3)
    th0 = pm.pack(0.3, rng.standard_normal(n) * 0.1, rng.standard_normal((k, n)) * 0.3, lay, k)
    kind, _ = pm.layout_masks(lay, k, th0.size)
    states = []
    for q in range(world):
        s = th0.copy()
        s[kind > 0] += (rng.standard_normal(int(np.sum(kind > 0))) * 0.01).astype(np.float32)
        states.append(s)
    zipf = (3000.0 / np.arange(1, n + 1) ** 2.5).astype(np.int64)
    counts = [rng.permutation(zipf).astype(np.float64) for _ in range(world)]
    for c in counts:
        c[:3] = 0  # features no shard saw: u = 0 sums
    counts[0][3:6] = 0  # features one shard never saw
    rows = [1000 + 7 * q for q in range(world)]
    hv = pm.hv(th0, lay)
    want, bud, g = pm.meanfield_combine(th0, states, counts, rows, hv, hp, lay, k, hv_rel=0.0)
    assert g[kind > 0].min() < 1.0 / world + 0.05 and g[kind > 0].max() > 0.99  # gamma spans its range

    # what all_reduce returns on every rank: the rank-order fp32 sums of the ranks' delta, counts and rows
    dsum = np.zeros_like(th0)
    for s in states:
        dsum = dsum + (s - th0)
    sums = [torch.from_numpy(dsum), torch.from_numpy(np.sum(np.float32(counts), axis=0)),
            torch.tensor([float(sum(rows))])]
    for r in range(world):
        _stub_allreduce(monkeypatch, sums)
        p = torch.from_numpy(states[r].copy())
        dist.combine_meanfield_(p, torch.from_numpy(th0), torch.from_numpy(counts[r]), rows[r], lay, hp.lr,
                                hp.reg0, hp.regw, hp.regv, world=world)
        got = p.numpy()
        assert np.array_equal(got[kind == 0], th0[kind == 0])
        ratio = pm.combine_ratio(got, want, bud)
        assert ratio < 1.0, "rank %d: %.2f budgets from the model" % (r, ratio)


def test_hv_bound_grows_with_the_partials():
    small = pm.hv_rel_bound(1000, 2, 132)
    big = pm.hv_rel_bound(5_000_000, 2, 132)
    assert 0 < small < big < 1e-4
