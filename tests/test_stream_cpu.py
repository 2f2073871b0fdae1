"""CPU: -cache_size streaming, host side -- the block plan of a binary .x file, the block reader and its
errors (host/sparse_data.h, driven through tests/xblock_dump.cpp), and the command line's plan line."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from libfm_b200 import Data, FmError, synth
from libfm_b200.model import read_xblocks, write_binary


@pytest.fixture(scope="module")
def xblock_dump(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("bin") / "xblock_dump")
    subprocess.run(["g++", "-O2", "-std=c++17", "-pthread", "-I", os.path.join(ROOT, "libfm_b200", "host"),
                    os.path.join(ROOT, "tests", "xblock_dump.cpp"), "-o", exe], check=True)
    return exe


def ragged_with_long_row():
    """Empty rows (10 %), rows of up to 9 entries, and one row of 5000 entries in the middle."""
    d = synth.ragged(3_000, 400, 9, seed=31, empty_frac=0.1)
    sizes = np.diff(d.row_ptr.astype(np.int64))
    r = np.random.default_rng(32)
    at = 1_234
    sizes = np.concatenate([sizes[:at], [5_000], sizes[at:]])
    cols = np.concatenate([d.col[:int(d.row_ptr[at])], r.integers(0, 400, 5_000).astype(np.uint32),
                           d.col[int(d.row_ptr[at]):]])
    vals = np.concatenate([d.val[:int(d.row_ptr[at])], r.standard_normal(5_000).astype(np.float32),
                           d.val[int(d.row_ptr[at]):]])
    tg = np.concatenate([d.target[:at], [3.0], d.target[at:]]).astype(np.float32)
    return Data(np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64), cols, vals, tg, 400)


@pytest.fixture(scope="module")
def ragged_bin(tmp_path_factory):
    d = ragged_with_long_row()
    stem = str(tmp_path_factory.mktemp("ragged") / "train")
    write_binary(d, stem + ".x", stem + ".y")
    return d, stem


def _dump(exe, stem, cache_size, out):
    return subprocess.run([exe, stem, str(cache_size), out], capture_output=True, text=True)


# 5000-entry row = 40004 bytes: budgets just above it, a few rows' worth bigger, and past the whole file
@pytest.mark.parametrize("cache_size", [80_008, 80_009, 100_001, 250_000, 1_000_000])
def test_block_plan_equals_the_rule(xblock_dump, ragged_bin, tmp_path, cache_size):
    d, stem = ragged_bin
    out = str(tmp_path / "dump")
    r = _dump(xblock_dump, stem, cache_size, out)
    assert r.returncode == 0, r.stderr
    x_bytes = 4 * d.num_cases + 8 * d.num_values
    if x_bytes <= cache_size // 2:
        assert r.stdout.split() == ["resident"]
        return
    want = list(read_xblocks(stem + ".x", cache_size))
    got = [tuple(int(t) for t in l.split()) for l in r.stdout.splitlines()]
    assert len(got) == len(want) >= 2
    assert [(a, b) for a, b, _, _ in got] == [(lo, hi) for lo, hi, _, _ in want]
    assert got[-1][1] == d.num_cases
    if cache_size < 2 * (40_004 + 4):  # no other row fits beside the long one
        assert (1234, 1235) in [(lo, hi) for lo, hi, _, _ in want]
    off = 24
    for (lo, hi, nnz, o), (_, _, words, sizes) in zip(got, want):
        assert nnz == int(sizes.sum()) and o == off and 4 * words.size <= cache_size // 2
        off += 4 * words.size
    # what the reader read: the file's bytes, the headers' sizes and the targets, block after block
    assert open(out + ".x", "rb").read() == open(stem + ".x", "rb").read()[24:]
    assert np.array_equal(np.fromfile(out + ".sizes", np.uint32), np.diff(d.row_ptr.astype(np.int64)))
    assert np.array_equal(np.fromfile(out + ".y", np.float32), d.target)


def test_row_larger_than_budget_is_refused(xblock_dump, ragged_bin, tmp_path):
    _, stem = ragged_bin
    r = _dump(xblock_dump, stem, 80_007, str(tmp_path / "o"))
    assert r.returncode == 1
    assert "ERROR: row 1234 of %s.x takes 40004 bytes: -cache_size must be at least 80008" % stem in r.stderr
    with pytest.raises(FmError, match="row 1234 .* at least 80008"):
        list(read_xblocks(stem + ".x", 80_007))


def test_truncated_file_is_refused(xblock_dump, ragged_bin, tmp_path):
    _, stem = ragged_bin
    raw = open(stem + ".x", "rb").read()
    t = str(tmp_path / "t")
    with open(t + ".y", "wb") as f:
        f.write(open(stem + ".y", "rb").read())
    # cut inside the last row's entries: the header's entry count no longer fits the file; then the same
    # file with the count lowered to what fits, so that the walk over the rows meets the cut
    nv = int(np.frombuffer(raw, np.uint64, 1, 8)[0])
    for header_nv in (nv, nv - 1):
        with open(t + ".x", "wb") as f:
            f.write(raw[:8] + np.array([header_nv], np.uint64).tobytes() + raw[16:-6])
        r = _dump(xblock_dump, t, 100_000, str(tmp_path / "o"))
        assert r.returncode == 1 and "ERROR: could not read %s.x" % t in r.stderr, (header_nv, r.stderr)


def test_row_count_disagreeing_with_targets_is_refused(xblock_dump, ragged_bin, tmp_path):
    d, stem = ragged_bin
    t = str(tmp_path / "c")
    with open(t + ".x", "wb") as f:
        f.write(open(stem + ".x", "rb").read())
    with open(t + ".y", "wb") as f:
        f.write(np.array([1, 4, d.num_cases - 1], np.uint32).tobytes() + d.target[:-1].tobytes())
    r = _dump(xblock_dump, t, 100_000, str(tmp_path / "o"))
    assert r.returncode == 1 and "ERROR: row count of %s.x and %s.y differ" % (t, t) in r.stderr


def test_cli_prints_the_plan_line(ragged_bin, tmp_path):
    """Loading needs no GPU: the plan line comes before the learner asks for one."""
    cli = os.path.join(ROOT, "bin", "libFM")
    if not os.path.exists(cli):
        pytest.skip("CLI not built")
    d, stem = ragged_bin
    args = [cli, "-task", "r", "-train", stem, "-test", stem, "-method", "sgd", "-iter", "1", "-learn_rate", "0.01",
            "-seed", "1"]
    r = subprocess.run(args + ["-cache_size", "100001"], capture_output=True, text=True)
    n_blocks = len(list(read_xblocks(stem + ".x", 100_001)))
    longest = max(hi - lo for lo, hi, _, _ in read_xblocks(stem + ".x", 100_001))
    line = "streaming %s.x: %d blocks of at most %d rows and 50000 bytes" % (stem, n_blocks, longest)
    assert r.stdout.splitlines().count(line) == 2, r.stdout  # train and test
    # a budget the file fits in, and text input, print what a run without -cache_size prints
    base = subprocess.run(args, capture_output=True, text=True)
    big = subprocess.run(args + ["-cache_size", "10000000000"], capture_output=True, text=True)
    assert "streaming" not in big.stdout and big.stdout == base.stdout
    import torch
    if not torch.cuda.is_available():
        assert r.returncode != 0 and "no CPU path" in r.stderr and "#Iter" not in r.stdout
