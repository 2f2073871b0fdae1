"""GPU: the per-epoch peer exchange (fm_peer.cu) computes what oracle/peer_model.py computes, exchange after
exchange, and the epochs after it train on the combined state.

Two contexts of one process on one device play two ranks (fmb200_peer_attach_local).  Before every exchange
both replicas are read raw (the packed fp32 buffer, padding included) and fed to the model exactly as they are;
theta0 is the raw state at the start of the epoch before.  After every exchange:
  * both replicas are bit-identical;
  * allreduce_mean equals the model bit for bit; allreduce_meanfield is within the model's per-element budget
    (worst element / budget is printed), so exchanges 2 and 3 also check the h_V the previous one left;
  * every word the exchange gives gamma 0 (the words between the bias and w, the stride gaps and tail of w) is
    what theta0 holds, bit for bit -- the cases that dirty those words in one replica before the exchange check
    that no rank's padding leaks into the combination.  V's padding columns share their row's gamma in the
    kernel, so they are only held to stay zero, as every replica keeps them.
Where a case trains on after the exchange, rank 0's combined state is pushed into a fresh context without
peers, and one epoch on both must give the same bits, predict and evaluate too.

World 2 only.  The exchange kernels spin on their peers' flags, and with both ranks on one device that is safe
only while both ranks' spinning grids are resident together: at two ranks and the state sizes here (mean-count
grids of at most one block per SM) they are.  With more ranks their kernels and streams are not guaranteed to
be scheduled together and a correct build could hang the device, so worlds above 2 are checked on the CPU only
(tests/test_peer_model.py, against the torch restatement of the rule).  At world 2 neither rank's slice of the
sliced exchange can be empty (a state is at least 8 float4s); the smallest state gives rank 1 a slice of the
w padding and two one-float V rows.
"""
import numpy as np
import pytest
import torch

from libfm_b200 import Data, FmLearnSgdElement, FmModel, MODE_HOGWILD, MODE_INORDER, synth
from oracle import HParams, geometry
from oracle import peer_model as pm
from test_rowgroup_model_gpu import MATRIX, make_data, tuning_for

pytestmark = pytest.mark.gpu

SLICED, ONE_SHOT = 8, 9  # fmb200_set_tuning variants that force either mean-field kernel


class _DevBuf:
    def __init__(self, ptr, n_floats):
        self.__cuda_array_interface__ = {"shape": (n_floats,), "typestr": "<f4", "data": (ptr, False), "version": 2}


def _dev(l):
    ptr, n = l.params_device()
    return torch.as_tensor(_DevBuf(ptr, n), device="cuda")


def _raw(l):
    """The packed fp32 state the context trains on (fmb200_params_device moves with every exchange)."""
    _sync(l)
    return _dev(l).cpu().numpy().copy()


def _sync(*ls):
    for l in ls:
        assert l.lib.fmb200_sync(l._ctx) == 0, l.lib.fmb200_last_error().decode()


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _learner(n, k, lr, regs, k0, k1, stdev, seed, targets, tuning, reproducible):
    fm = FmModel(n, k, k0, k1)
    fm.init_stdev = stdev
    fm.init_numpy(seed)
    fm.w = np.float32(np.random.default_rng(seed + 1).standard_normal(n) * 0.05).astype(np.float64)
    fm.reg0, fm.regw, fm.regv = regs
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate = 0, lr
    l.min_target, l.max_target = targets
    l.push_hparams()
    l.set_tuning(**tuning)
    if reproducible is not None:
        l.set_reproducible(True, *reproducible)
    return l


class Pair:
    """Two attached ranks, each with its shard in slot 0, and the model's view of them."""

    def __init__(self, shards, k, lr=0.01, regs=(0.0, 0.0, 0.0), k0=True, k1=True, stdev=0.1, variant=0,
                 tuning=None, reproducible=None, poison=False, seed=3):
        import ctypes as C
        self.n = max(d.num_feature for d in shards)
        self.shards = [Data(d.row_ptr, d.col, d.val, d.target, self.n) for d in shards]
        self.k, self.lr, self.regs, self.poison = k, lr, regs, poison
        lo = min(float(np.min(d.target)) for d in self.shards)
        hi = max(float(np.max(d.target)) for d in self.shards)
        self.targets = (lo, hi)
        self.tuning = dict(tuning or {}, variant=variant) if variant else dict(tuning or {})
        self.args = (self.n, k, lr, regs, k0, k1, stdev, seed, self.targets, self.tuning, reproducible)
        self.ls = []
        try:
            for _ in range(2):
                self.ls.append(_learner(*self.args))
            for l, d in zip(self.ls, self.shards):
                l.upload(d, 0)
            arr = (C.c_void_p * 2)(*[l._ctx for l in self.ls])
            for rank, l in enumerate(self.ls):
                assert l.lib.fmb200_peer_attach_local(l._ctx, 2, rank, arr) == 0, \
                    l.lib.fmb200_last_error().decode()
        except BaseException:
            self.close()
            raise
        self.layout = self.ls[0].params_layout()
        self.hp = HParams(0, lr, *regs)
        self.theta0 = None
        self.ratios = []

    def close(self):
        for l in self.ls:
            l.close()

    # every case holds its pair in a `with` block: no failed assertion leaves attached contexts behind
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False

    def reupload(self, rank, d):
        self.shards[rank] = Data(d.row_ptr, d.col, d.val, d.target, self.n)
        self.ls[rank].upload(self.shards[rank], 0)

    def epoch(self):
        self.theta0 = [_raw(l) for l in self.ls]
        for l, d in zip(self.ls, self.shards):
            l.sgd_epoch(d)
        _sync(*self.ls)

    def _exchange(self, fn):
        for l in self.ls:
            assert getattr(l.lib, fn)(l._ctx) == 0, l.lib.fmb200_last_error().decode()
        _sync(*self.ls)
        got = [_raw(l) for l in self.ls]
        assert np.array_equal(_bits(got[0]), _bits(got[1])), "the replicas differ after %s" % fn
        return got[0]

    def mean(self, tag):
        states = [_raw(l) for l in self.ls]
        got = self._exchange("fmb200_allreduce_mean")
        want = pm.mean_combine(states)
        bad = np.flatnonzero(_bits(got) != _bits(want))
        print("peer %-28s mean       bit-exact %s" % (tag, bad.size == 0))
        assert bad.size == 0, "allreduce_mean differs from the rank-order fp32 mean at %s" % bad[:8]

    def _dirty(self, state):
        """Write non-zero values into rank 1's gamma-0 words below V (see the module docstring)."""
        kind, _ = pm.layout_masks(self.layout, self.k, state.size)
        idx = np.flatnonzero(kind[:self.layout["off_v"]] == 0)
        vals = np.float32(0.25 + (idx % 7) * 0.5)
        t = _dev(self.ls[1])
        t[torch.as_tensor(idx, device="cuda")] = torch.as_tensor(vals, device="cuda")
        torch.cuda.synchronize()
        state = state.copy()
        state[idx] = vals
        return state

    def meanfield(self, tag):
        states = [_raw(l) for l in self.ls]
        th0 = self.theta0[0]
        assert np.array_equal(_bits(th0), _bits(self.theta0[1]))
        if self.poison:
            states[1] = self._dirty(states[1])
        got = self._exchange("fmb200_allreduce_meanfield")
        n_vec = th0.size // 4
        want, bud, g = pm.meanfield_combine(
            th0, states, [pm.counts_of(d, self.n) for d in self.shards], [d.num_cases for d in self.shards],
            pm.hv(th0, self.layout), self.hp, self.layout, self.k, hv_rel=pm.hv_rel_bound(n_vec, 2, _sm_count()))
        kind, _ = pm.layout_masks(self.layout, self.k, th0.size)
        pad = kind == 0
        assert np.array_equal(_bits(got[pad]), _bits(th0[pad])), "a gamma-0 word changed at %s" % \
            np.flatnonzero(pad & (_bits(got) != _bits(th0)))[:8]
        ratio = pm.combine_ratio(got, want, bud)
        moved = g[kind > 0]
        print("peer %-28s meanfield  k %3d ws %d n_vec %7d  gamma %.3f..%.3f  worst/budget %.3f" % (
            tag, self.k, self.layout["ws"], n_vec, moved.min(), moved.max(), ratio))
        assert ratio < 1.0, "%s: an element is %.2f budgets from the model" % (tag, ratio)
        self.ratios.append(ratio)
        return got


def _two_field_shards(n_rows, users, items, seed, zipf=0.0, sizes=(0.5,)):
    d = synth.two_field(n_rows, users, items, seed=seed, zipf=zipf)
    cut = int(n_rows * sizes[0])
    return [d.rows(0, cut), d.rows(cut, n_rows)]


def run_meanfield(pair, exchanges=3):
    for e in range(exchanges):
        pair.epoch()
        pair.meanfield("exchange %d" % (e + 1))
    assert max(pair.ratios) > 0.0, "the model matched every element exactly: the budget is never exercised"


# ---- the combines at every state layout ----

@pytest.mark.parametrize("variant", [ONE_SHOT, SLICED])
@pytest.mark.parametrize("k", [1, 5, 8, 33, 64, 128])
def test_meanfield_factor_widths(k, variant, built_lib):
    shards = _two_field_shards(12_000, 700, 500, seed=k, zipf=0.8)
    with Pair(shards, k, lr=0.01, stdev=0.2, variant=variant, poison=True) as p:
        run_meanfield(p)


@pytest.mark.parametrize("variant", [ONE_SHOT, SLICED])
def test_meanfield_packed_linear_weights(variant, built_lib):
    """n > 131 072: w packed at stride 1 (ws = 1); n not a multiple of 32, so w has a padded tail."""
    shards = _two_field_shards(30_000, 100_003, 40_000, seed=11, zipf=0.9)
    with Pair(shards, 8, lr=0.02, stdev=0.2, variant=variant, poison=True) as p:
        assert p.layout["ws"] == 1 and p.n % 32 != 0
        run_meanfield(p)


def test_mean_is_bit_exact(built_lib):
    with Pair(_two_field_shards(8000, 300, 200, seed=2), 5, stdev=0.2) as p:
        for e in range(3):
            p.epoch()
            p.mean("exchange %d" % (e + 1))


@pytest.mark.parametrize("variant", [ONE_SHOT, SLICED])
@pytest.mark.parametrize("name,regs,k0,k1", [("regularised", (0.3, 0.5, 0.7), True, True),
                                             ("no bias", (0.0, 0.2, 0.4), False, True),
                                             ("no linear", (0.1, 0.0, 0.4), True, False)])
def test_meanfield_switches(name, regs, k0, k1, variant, built_lib):
    """reg0, regw and regv enter gamma; regv outweighs h_V here, so V's gamma depends on it."""
    shards = _two_field_shards(10_000, 500, 300, seed=5, zipf=0.8)
    with Pair(shards, 8, lr=0.01, regs=regs, k0=k0, k1=k1, stdev=0.15, variant=variant, poison=True) as p:
        run_meanfield(p)


def test_meanfield_gamma_over_its_range(built_lib):
    """Zipf shards: hot features' u >> 1 (gamma -> 1/2), cold ones' u << 1 (gamma -> 1), V's u in between."""
    shards = _two_field_shards(40_000, 3000, 2000, seed=9, zipf=1.3)
    with Pair(shards, 8, lr=0.02, stdev=0.3, variant=SLICED, poison=True) as p:
        for e in range(3):
            p.epoch()
            p.meanfield("zipf exchange %d" % (e + 1))
        cnt = (pm.counts_of(p.shards[0], p.n) + pm.counts_of(p.shards[1], p.n)) / 2
        u = p.lr * cnt
        assert u.max() > 20 and np.min(u[cnt > 0]) < 0.05
        uv = p.lr * pm.hv(p.theta0[0], p.layout) * cnt
        assert np.any((uv > 0.3) & (uv < 3))  # where gamma leans on h_V hardest


# ---- where the two slices of the sliced exchange meet ----

def _slice_edge(p):
    n_vec = p.layout["off_v"] // 4 + p.n * p.layout["kp"] // 4
    per = (n_vec + 1) // 2
    return n_vec, 4 * per


@pytest.mark.parametrize("name,users,items,k,where", [
    ("edge in w", 6, 4, 8, "w"),                 # n = 10
    ("edge at off_v", 4, 4, 12, "off_v"),        # n = 8, kp = 12
    ("edge inside a V row, n_vec odd", 12, 9, 33, "v odd"),  # n = 21, kp = 36
    ("smallest state", 1, 1, 1, "w"),            # n = 2: rank 1 holds the w tail and both V rows
])
def test_sliced_slice_edges(name, users, items, k, where, built_lib):
    shards = _two_field_shards(3000, users, items, seed=users * 31 + k)
    with Pair(shards, k, lr=0.0004, stdev=0.3, variant=SLICED, poison=True) as p:
        n_vec, edge = _slice_edge(p)
        lay = p.layout
        if where == "w":
            assert lay["off_w"] <= edge < lay["off_v"]
        elif where == "off_v":
            assert edge == lay["off_v"]
        else:
            assert n_vec % 2 == 1 and edge > lay["off_v"] and (edge - lay["off_v"]) % lay["kp"] != 0
        run_meanfield(p)


# ---- the count tables: unequal shards, re-uploads between exchanges ----

@pytest.mark.parametrize("variant", [ONE_SHOT, SLICED])
def test_counts_follow_the_uploads(variant, built_lib):
    """Shards of 3 000 and 9 000 rows.  Between exchanges 1 and 2 rank 1 uploads other rows and rank 0 uploads
    its own again; exchange 3 (the first table's parity again) must see the new counts, exchange 4 too."""
    d = synth.two_field(20_000, 400, 300, seed=21, zipf=1.0)
    with Pair([d.rows(0, 3000), d.rows(3000, 12_000)], 8, lr=0.01, stdev=0.2, variant=variant, poison=True) as p:
        p.epoch()
        p.meanfield("unequal shards 1")
        p.reupload(1, d.rows(12_000, 20_000))
        p.reupload(0, d.rows(0, 3000))
        for e in range(2, 5):
            p.epoch()
            p.meanfield("after re-upload %d" % e)


# ---- theta0: recaptured whenever the state was set another way ----

def test_mean_then_meanfield(built_lib):
    with Pair(_two_field_shards(10_000, 500, 300, seed=4, zipf=0.8), 8, stdev=0.2, poison=True) as p:
        p.epoch()
        p.mean("mean first")
        for e in range(2):
            p.epoch()
            p.meanfield("after the mean %d" % (e + 1))


@pytest.mark.parametrize("variant", [ONE_SHOT, SLICED])
def test_push_params_between_exchanges(variant, built_lib):
    with Pair(_two_field_shards(10_000, 500, 300, seed=6, zipf=0.8), 8, stdev=0.2, variant=variant,
              poison=True) as p:
        p.epoch()
        p.meanfield("before the push")
        w0, w, v = pm.unpack(_raw(p.ls[0]), p.layout, p.k)
        for l in p.ls:
            l.fm.w0, l.fm.w, l.fm.v = w0 * 0.5, w * 0.5, np.float32(v * 1.5).astype(np.float64)
            l.push_params()
        for l in p.ls:  # nothing to combine: no epoch since the state was set
            assert l.lib.fmb200_allreduce_meanfield(l._ctx) != 0
            assert "no epoch has run since the state was last set" in l.lib.fmb200_last_error().decode()
        for e in range(2):
            p.epoch()
            p.meanfield("after the push %d" % (e + 1))


def test_mode_round_trip_between_exchanges(built_lib):
    """HOGWILD -> INORDER -> HOGWILD with one INORDER epoch in between: the state at the next HOGWILD epoch's start
    is no longer what the last exchange left in theta0, so that epoch must capture theta0 (and h_V) afresh.
    Both ranks run the INORDER epoch on the same rows: that epoch is sequential, so they stay identical."""
    d = synth.two_field(12_000, 500, 300, seed=8, zipf=0.8)
    with Pair([d.rows(0, 5000), d.rows(5000, 10_000)], 8, stdev=0.2, variant=SLICED, poison=True) as p:
        p.epoch()
        p.meanfield("before INORDER")
        before = _raw(p.ls[0])
        common = Data(*(getattr(d.rows(10_000, 12_000), a) for a in ("row_ptr", "col", "val", "target")), p.n)
        for l in p.ls:
            l.set_mode(MODE_INORDER)
            l.sgd_epoch(common)
            l.set_mode(MODE_HOGWILD)
            l.release(common)
        after = [_raw(l) for l in p.ls]
        assert np.array_equal(_bits(after[0]), _bits(after[1]))
        assert not np.array_equal(_bits(after[0]), _bits(before)), "the INORDER epoch left the state as it was"
        for e in range(2):
            p.epoch()
            p.meanfield("after INORDER %d" % (e + 1))


# ---- the epochs after an exchange train on the combined buffer ----

def _fresh_twin(p, state):
    """A context without peers holding `state`, past the first-epoch bias ramp: one epoch at learning rate 0,
    which leaves the state as it is."""
    l = _learner(*p.args)
    try:
        w0, w, v = pm.unpack(state, p.layout, p.k)
        l.fm.w0, l.fm.w, l.fm.v = w0, w, v
        l.push_params()
        assert np.array_equal(_bits(_raw(l)), _bits(state))
        l.upload(p.shards[0], 0)
        l.learn_rate = 0.0
        l.push_hparams()
        l.sgd_epoch(p.shards[0])
        assert np.array_equal(_bits(_raw(l)), _bits(state)), "an epoch at learning rate 0 changed the state"
        l.learn_rate = p.lr
        l.push_hparams()
    except BaseException:
        l.close()
        raise
    return l


def run_trains_on(p, test, combine="meanfield", dealt=None, expect_cfg=None):
    for e in range(3):
        p.epoch()
        if combine == "mean":
            p.mean("exchange %d" % (e + 1))
            state = _raw(p.ls[0])
        else:
            state = p.meanfield("exchange %d" % (e + 1))
        twin = _fresh_twin(p, state)
        try:
            assert np.array_equal(p.ls[0].predict(test), twin.predict(test))
            assert p.ls[0].evaluate(test) == twin.evaluate(test)
            p.epoch()  # both ranks train on; rank 0's epoch must equal the twin's
            twin.sgd_epoch(p.shards[0])
            a, b = _raw(p.ls[0]), _raw(twin)
            cfg = p.ls[0].epoch_config()
            assert cfg == twin.epoch_config()
            if expect_cfg is not None:
                expect_cfg(cfg)
            if dealt is not None:
                assert p.ls[0].epoch_dealt() == dealt and twin.epoch_dealt() == dealt
            bad = np.flatnonzero(_bits(a) != _bits(b))
            print("peer trains on the combined buffer after exchange %d: %s" % (
                e + 1, "bit-identical" if bad.size == 0 else "%d words differ" % bad.size))
            assert bad.size == 0, "the epoch after exchange %d did not train on the combined state" % (e + 1)
        finally:
            twin.close()
        if combine != "mean":
            p.meanfield("exchange %d, second" % (e + 1))


def _as(d, n):
    return Data(d.row_ptr, d.col, d.val, d.target, n)


@pytest.mark.parametrize("name,variant,dealt", [("dealt, sliced", SLICED, True),
                                                ("file order, one-shot", 5, False)])
def test_rowlane_epoch_trains_on_the_combined_buffer(name, variant, dealt, built_lib):
    """The reproducible row-lane epoch (C2 shape, k = 8; windows of SMs x 64 rows); variant 5 forces its
    file-order schedule, and then the exchange picks the one-shot kernel for this state size."""
    d = synth.two_field(42_000, 3000, 2000, seed=13)
    with Pair([d.rows(0, 20_000), d.rows(20_000, 40_000)], 8, lr=0.01, stdev=0.1, variant=variant,
              tuning=dict(ctas_per_sm=1, threads=64)) as p:
        assert p.layout["kp"] == 8

        def expect(cfg):
            assert cfg["lanes_per_row"] == 1, "the row-lane kernel did not run"
        run_trains_on(p, _as(d.rows(40_000, 42_000), p.n), dealt=dealt, expect_cfg=expect)


def test_rowlane_epoch_trains_on_the_mean(built_lib):
    d = synth.two_field(22_000, 1000, 800, seed=17)
    with Pair([d.rows(0, 10_000), d.rows(10_000, 20_000)], 8, stdev=0.1,
              tuning=dict(ctas_per_sm=1, threads=64)) as p:
        run_trains_on(p, _as(d.rows(20_000, 22_000), p.n), combine="mean")


def test_windowed_epoch_trains_on_the_combined_buffer(built_lib):
    """set_reproducible(True, 32, 4), k = 33, rows of 0-60 entries, some naming a feature two or three times."""
    shards = [synth.long_rows(1500, 900, 60, seed=s) for s in (1, 2)]
    test = synth.long_rows(300, 900, 60, seed=3)
    with Pair(shards, 33, lr=0.002, stdev=0.05, variant=SLICED, reproducible=(32, 4)) as p:
        def expect(cfg):
            assert cfg["rows_per_tile"] == 32 and cfg["lanes_per_row"] == 32, "the windowed epoch did not run"
        run_trains_on(p, test, expect_cfg=expect)


def test_rowgroup_epoch_trains_on_the_combined_buffer(built_lib):
    """The row-group kernel at MATRIX's (k = 40, 25 entries a row): G = 16, S = 2, class 2; race-free rows
    (every non-zero entry names its own feature), no bias -- its result is a function of its input."""
    k, avg = 40, 25.0
    assert (k, avg) in MATRIX
    n_rows = int(np.clip(30_000 / avg, 400, 40_000))
    geo0 = geometry(k, n_rows, int(avg * n_rows))
    shards = [make_data(n_rows, avg, geo0, seed=s) for s in (31, 32)]
    test = make_data(200, avg, None, seed=33, long_rows=0)
    geo = geometry(k, shards[0].num_cases, shards[0].num_values)
    with Pair(shards, k, lr=0.01, k0=False, stdev=0.1, tuning=tuning_for(k, shards[0])) as p:
        def expect(cfg):
            assert (cfg["lanes_per_row"], cfg["slots"]) == (geo.G, geo.S), "the row-group kernel did not run"
        run_trains_on(p, Data(test.row_ptr, test.col % p.n, test.val, test.target, p.n), expect_cfg=expect)
