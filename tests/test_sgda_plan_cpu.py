"""CPU: the launch plan of one SGDA epoch (libfm_b200/csrc/fm_sgda_plan.h, driven through tests/sgda_plan_dump.cpp)
against a step-by-step restatement: the reference's epoch walked half-step by half-step, its validation cursor
moved as fm_learn_sgd_element_adapt_reg.h:295-311 moves it, a launch ended wherever the next step reads another
block of a streamed set, the cursor restarts inside a set of several blocks, or the last update_means comes."""
import os
import subprocess

import pytest

from conftest import ROOT


@pytest.fixture(scope="module")
def plan_dump(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("bin") / "sgda_plan_dump")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "libfm_b200", "csrc"),
                    os.path.join(ROOT, "tests", "sgda_plan_dump.cpp"), "-o", exe], check=True)
    return exe


def run_plan(exe, n, v, lam, train_lo, val_lo):
    inp = "%d %d %d\n%s\n%s\n" % (n, v, int(lam), " ".join(map(str, train_lo)), " ".join(map(str, val_lo)))
    r = subprocess.run([exe], input=inp, capture_output=True, text=True, check=True)
    return [tuple(int(x) for x in l.split()) for l in r.stdout.splitlines()]


def block_of(lo, row):
    """The block holding `row` (lo: first rows, then the count); -1 for a resident set."""
    if not lo:
        return -1
    return max(b for b in range(len(lo) - 1) if lo[b] <= row)


def restated_plan(n, v, lam, train_lo, val_lo):
    lam = lam and v > 0
    # the reference's epoch: update_means at the start and at every cursor restart; the last one is the moments
    steps, cursor, last_means = [], 0, 0
    for t in range(n):
        steps.append(("theta", t, None))
        if lam:
            if cursor == v:
                cursor, last_means = 0, t
            steps.append(("lambda", t, cursor))
            cursor += 1
    h_of = {}  # half-step -> (kind, row read)
    for kind, t, s in steps:
        h_of[2 * t + (kind == "lambda")] = (kind, t if kind == "theta" else s)
    cuts = set()
    cur = {"theta": None, "lambda": None}
    for h in sorted(h_of):
        kind, row = h_of[h]
        lo = train_lo if kind == "theta" else val_lo
        b = block_of(lo, row)
        if kind == "lambda" and len(val_lo) > 2 and row == 0 and h > 1:
            cuts.add(h)  # the cursor restarts inside a set of several blocks
        if cur[kind] is not None and b != cur[kind]:
            cuts.add(h)
        cur[kind] = b
    if last_means > 0:
        cuts.add(2 * last_means + 1)
    bounds = sorted({0, 2 * n} | cuts)
    plan = [(0, 0, 0, -1, -1, 1)] if n == 0 else []
    for h0, h1 in zip(bounds, bounds[1:]):
        done = sum(1 for h in h_of if h < h0 and h % 2 == 1)  # lambda-steps before the launch
        vc0 = 0 if done == 0 else (done - 1) % v + 1
        # the blocks the launch reads: its first theta- and lambda-step's, else those the next ones read
        pair = h0 // 2
        tb = block_of(train_lo, pair)
        vb = block_of(val_lo, pair % v) if lam else -1
        moments = (h0 == 0) if last_means == 0 else (h0 == 2 * last_means + 1)
        plan.append((h0, h1, vc0, tb, vb, int(moments)))
    return plan


def check_plan(got, n, v, lam, train_lo, val_lo):
    assert got == restated_plan(n, v, lam, train_lo, val_lo)
    # and what the plan promises: consecutive launches cover [0, 2N), each reads the blocks it names
    if n:
        assert got[0][0] == 0 and got[-1][1] == 2 * n
        assert all(a[1] == b[0] for a, b in zip(got, got[1:]))
    for h0, h1, _, tb, vb, _ in got:
        for h in range(h0, h1):
            t = h // 2
            if h % 2 == 0 and train_lo:
                assert train_lo[tb] <= t < train_lo[tb + 1]
            if h % 2 == 1 and lam and v and len(val_lo) > 2:
                assert val_lo[vb] <= t % v < val_lo[vb + 1]


# (N, V, train block starts, validation block starts): blocks as lists of first rows plus the row count
CASES = [
    (10, 3, [0, 4, 10], [0, 1, 3]),          # V < N: restarts at t = 3, 6, 9 = t*
    (10, 3, [], [0, 1, 3]),                  # resident training set
    (10, 3, [0, 4, 10], []),                 # resident validation set: t* is the only validation cut
    (10, 3, [0, 4, 10], [0, 3]),             # one validation block wraps as a resident set does
    (7, 12, [0, 2, 5, 7], [0, 4, 8, 12]),    # V > N: the cursor never restarts
    (9, 9, [0, 3, 6, 9], [0, 3, 6, 9]),      # V == N, blocks aligned with the training blocks
    (12, 5, [0, 10, 12], [0, 2, 5]),         # a training block boundary at t* = 10
    (11, 5, [0, 5, 6, 11], [0, 2, 4, 5]),    # training boundaries at the restarts t = 5, 10 = t*
    (1, 4, [0, 1], [0, 2, 4]),               # one training row
    (2000, 37, list(range(0, 2000, 91)) + [2000], [0, 5, 6, 20, 37]),  # 22 training blocks, many restarts
]


@pytest.mark.parametrize("n,v,train_lo,val_lo", CASES)
@pytest.mark.parametrize("lam", [False, True])
def test_plan_matches_the_restatement(plan_dump, n, v, train_lo, val_lo, lam):
    got = run_plan(plan_dump, n, v, lam, train_lo, val_lo)
    check_plan(got, n, v, lam, train_lo, val_lo)


def test_resident_plan_is_the_resident_launch_sequence(plan_dump):
    """No blocks: the moments and one launch, or a cut at t* with a full cursor after it"""
    assert run_plan(plan_dump, 10, 3, True, [], []) == [(0, 19, 0, -1, -1, 0), (19, 20, 3, -1, -1, 1)]
    assert run_plan(plan_dump, 10, 3, False, [], []) == [(0, 20, 0, -1, -1, 1)]
    assert run_plan(plan_dump, 3, 10, True, [], []) == [(0, 6, 0, -1, -1, 1)]
    # one block per set plans as resident
    assert [l[:3] + l[5:] for l in run_plan(plan_dump, 10, 3, True, [0, 10], [0, 3])] == [(0, 19, 0, 0), (19, 20, 3, 1)]


def test_cut_at_block_boundaries_wrap_and_t_star(plan_dump):
    got = run_plan(plan_dump, 10, 3, True, [0, 4, 10], [0, 1, 3])
    starts = [l[0] for l in got]
    assert 8 in starts                                   # training block 1 starts at row 4
    assert {3, 9, 15} <= set(starts)                     # validation row 1 starts block 1, at t = 1, 4, 7
    assert {7, 13, 19} <= set(starts)                    # restarts at t = 3, 6, 9
    assert [l[0] for l in got if l[5]] == [19]           # the moments at t* = 9
