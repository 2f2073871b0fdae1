"""GPU: out-of-core SGDA (fmb200_sgda_epoch_x through FmLearnSgdElement.sgda_epoch_x) against the resident epoch
(fmb200_sgda_epoch) on the same data: w0, w, V, reg_w, reg_v and the moments bit for bit after every epoch, the
first epoch without lambda-steps.  The training and validation sets are written as .x files and read in blocks cut
at chosen rows: evenly (3+ and 20+ blocks), at t* and at the validation cursor's restart, or as the command line
plans them under -cache_size; each set also runs resident beside a streamed other."""
import numpy as np
import pytest

from conftest import make_learner
from libfm_b200 import MODE_INORDER, MODE_ORDERED, synth
from libfm_b200.model import XtBlocks, write_binary

pytestmark = pytest.mark.gpu

N = 1500  # training rows
EPOCHS = 3


def make_sets(kind, n_val, seed=4):
    if kind == "long":  # rows of up to 9 entries: the one-warp kernel
        full = synth.ragged(N + n_val, 300, 9, seed=seed, empty_frac=0.05)
    else:  # (user, item) rows: the wavefront kernel at k <= 8
        full = synth.two_field(N + n_val, 300, 200, seed=seed, planted_k=3)
    return synth.split_rows(full, N)


def blocks_at(path_x, target, starts, slots):
    """The .x at path_x as an XtBlocks (transposed=False) cut into blocks that start at rows `starts` (0 first)."""
    x = XtBlocks(path_x, target, 1 << 40, slots, transposed=False)  # one block
    _, n, words, sizes = x.blocks[0]
    off = np.concatenate([[0], np.cumsum(1 + 2 * sizes.astype(np.int64))])
    bounds = sorted(set(starts) | {0}) + [n]
    x.blocks = [(a, b, np.ascontiguousarray(words[off[a]:off[b]]), np.ascontiguousarray(sizes[a:b]))
                for a, b in zip(bounds, bounds[1:])]
    x.col_lo = np.array(bounds, dtype=np.uint32)
    x.nnz = np.array([int(s.sum()) for _, _, _, s in x.blocks], dtype=np.uint64)
    return x


def even(n, n_blocks):
    return [n * b // n_blocks for b in range(n_blocks)]


def t_star(n_val):
    return 0 if N <= n_val else (N - 1) // n_val * n_val


def plan_starts(plan, n_val):
    """(training block starts, validation block starts); None: that set resident"""
    if plan == "t3_v3":
        return even(N, 3), even(n_val, 3)
    if plan == "t22_vres":
        return even(N, 22), None
    if plan == "tres_v4":
        return None, even(n_val, 4)
    if plan == "t21_v20":
        return even(N, 21), even(n_val, 20)
    if plan == "edges":  # training blocks start at t*, at the first restart (t = V) and just after it;
        ts = t_star(n_val)  # validation blocks at row 1 and at the last row, next to the restart
        return sorted({0, 7, min(n_val, N - 1), min(n_val + 1, N - 1), ts, ts + 1} - {N}), [0, 1, n_val - 1]
    raise ValueError(plan)


CASES = {
    "wraps": dict(kind="short", n_val=500),          # V < N: the cursor restarts at t = 500 and t* = 1000
    "val_long": dict(kind="short", n_val=2200),      # V > N: no restart, t* = 0
    "v_eq_n": dict(kind="short", n_val=N),           # V == N
    "odd_wraps": dict(kind="short", n_val=333),      # t* = 1332, four restarts
    "one_group": dict(kind="short", n_val=500, groups=1),
    "cls": dict(kind="short", n_val=500, task=1),
    "long_rows": dict(kind="long", n_val=400, k=12),  # one-warp kernel (rows > 4 entries, k > 8)
    "variant1": dict(kind="short", n_val=500, variant=1),
}
RUNS = [(c, p) for c in ("wraps", "val_long", "v_eq_n", "long_rows") for p in ("t3_v3", "t22_vres", "tres_v4", "edges")]
RUNS += [("odd_wraps", "t21_v20"), ("odd_wraps", "edges"), ("one_group", "t3_v3"), ("cls", "t3_v3"),
         ("cls", "edges"), ("variant1", "t3_v3"), ("variant1", "edges")]


def learners(case, mode):
    cfg = CASES[case]
    task, k, groups = cfg.get("task", 0), cfg.get("k", 5), cfg.get("groups", 3)
    tr, va = make_sets(cfg["kind"], cfg["n_val"])
    if task == 1:
        for d in (tr, va):
            d.target[:] = np.where(d.target > 3, 1.0, -1.0)
    n = tr.num_feature
    group = (np.arange(n) * groups // n).astype(np.uint32)
    init = (0.0, np.zeros(n), np.random.default_rng(2).standard_normal((k, n)) * 0.1)
    lc = dict(n=n, k=k, k0=1, k1=1, task=task, lr=0.02, regs=np.zeros(3), min_target=float(tr.target.min()),
              max_target=float(tr.target.max()))
    out = []
    for _ in range(2):
        l = make_learner(lc, init, mode=mode)
        if cfg.get("variant"):
            l.set_tuning(variant=cfg["variant"])
        l.sgda_begin(group if groups > 1 else None)
        out.append(l)
    return tr, va, out


def state(l):
    l.pull_params()
    reg_w, reg_v = l.sgda_reg()
    var_w, var_v = l.sgda_moments()
    return [np.array([l.fm.w0]), l.fm.w.copy(), l.fm.v.copy(), reg_w, reg_v, np.array([var_w]), var_v]


def assert_same(a, b, what):
    names = ["w0", "w", "v", "reg_w", "reg_v", "var_w", "var_v"]
    for name, x, y in zip(names, a, b):
        assert np.array_equal(x.view(np.uint64), y.view(np.uint64)), (what, name)


@pytest.mark.parametrize("mode", [MODE_INORDER, MODE_ORDERED])
@pytest.mark.parametrize("case,plan", RUNS)
def test_streamed_epochs_bit_identical_to_resident(case, plan, mode, tmp_path, built_lib):
    tr, va, (res, st) = learners(case, mode)
    for d, name in ((tr, "train"), (va, "val")):
        write_binary(d, str(tmp_path / (name + ".x")), str(tmp_path / (name + ".y")))
    t_starts, v_starts = plan_starts(plan, va.num_cases)
    xtr = tr if t_starts is None else blocks_at(str(tmp_path / "train.x"), tr.target, t_starts, (2, 4))
    xva = va if v_starts is None else blocks_at(str(tmp_path / "val.x"), va.target, v_starts, (3, 5))
    for e in range(EPOCHS):
        res.sgda_epoch(tr, va, e > 0)
        st.sgda_epoch_x(xtr, xva, e > 0)
        assert_same(state(st), state(res), "epoch %d" % e)
    assert state(res)[4].max() > 0  # the lambda-steps moved reg_v
    if v_starts is not None:
        assert xva.fetches >= len(xva.blocks)  # the validation blocks went through the device
    res.close()
    st.close()


@pytest.mark.parametrize("mode", [MODE_INORDER, MODE_ORDERED])
def test_cache_size_plan_and_single_blocks(mode, tmp_path, built_lib):
    """Blocks as the command line plans them (read_xblocks), several per set; then a budget past both files: one
    block each, whose epochs launch what the resident ones launch beside the blocks' decoding."""
    tr, va, (res, st) = learners("wraps", mode)
    px, pv = str(tmp_path / "train.x"), str(tmp_path / "val.x")
    write_binary(tr, px, str(tmp_path / "train.y"))
    write_binary(va, pv, str(tmp_path / "val.y"))
    xtr = XtBlocks(px, tr.target, 4000, (2, 4), transposed=False)
    xva = XtBlocks(pv, va.target, 4000, (3, 5), transposed=False)
    assert xtr.n_blocks >= 3 and xva.n_blocks >= 3
    for e in range(EPOCHS):
        res.sgda_epoch(tr, va, e > 0)
        st.sgda_epoch_x(xtr, xva, e > 0)
        assert_same(state(st), state(res), "epoch %d" % e)
    one_tr = XtBlocks(px, tr.target, 1 << 40, (2, 4), transposed=False)
    one_va = XtBlocks(pv, va.target, 1 << 40, (3, 5), transposed=False)
    assert one_tr.n_blocks == one_va.n_blocks == 1
    # the kernels one upload of each block launches (the same shapes into a spare slot)
    decode = []
    for x in (one_tr, one_va):
        n0 = st.kernel_launches()
        _, _, words, sizes = x.blocks[0]
        st.upload_xblock(words, sizes, x.target, 7, asynchronous=True)
        decode.append(st.kernel_launches() - n0)
        st.lib.fmb200_free_data(st._ctx, 7)  # waits for the copy
    for e in range(2):
        lam = e > 0
        r0, s0 = res.kernel_launches(), st.kernel_launches()
        res.sgda_epoch(tr, va, lam)
        st.sgda_epoch_x(one_tr, one_va, lam)
        assert_same(state(st), state(res), "one block, lambda-steps %d" % lam)
        assert st.kernel_launches() - s0 == res.kernel_launches() - r0 + decode[0] + (decode[1] if lam else 0)
        assert res.kernel_launches() - r0 == (3 if lam else 2)  # moments and one launch, or two around t*
    res.close()
    st.close()


def test_refusals(tmp_path, built_lib):
    tr, va, (res, st) = learners("wraps", MODE_INORDER)
    px = str(tmp_path / "train.x")
    write_binary(tr, px, str(tmp_path / "train.y"))
    bad = XtBlocks(px, tr.target, 1 << 40, (2, 2), transposed=False)
    with pytest.raises(Exception, match="the two slots must differ"):
        st.sgda_epoch_x(bad, va, True)
    clash = XtBlocks(px, tr.target, 4000, (2, 4), transposed=False)
    with pytest.raises(Exception, match="must differ from every other slot"):
        st.sgda_epoch_x(clash, XtBlocks(str(tmp_path / "train.x"), tr.target, 4000, (4, 5), transposed=False), True)
    res.close()
    st.close()
