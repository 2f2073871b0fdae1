"""CPU: the host side of out-of-core MCMC and ALS -- the .xt layout (write_transposed, bin/transpose) against what
the stock transpose tool wrote for the same inputs (tests/golden/reference/transpose.json), the block plan of a
.xt (host/sparse_data.h through tests/xtblock_dump.cpp) against the rule read_xblocks states, and the command
line's refusals, which all happen before the GPU is touched."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from libfm_b200 import Data, build, synth
from libfm_b200.model import read_xblocks, write_binary, write_transposed

CLI_GOLDEN = os.path.join(ROOT, "tests", "golden", "reference", "mcmc_cli.npz")
# what the stock reference's tools/transpose.cpp writes for transpose_inputs() (scripts/make_transpose_golden.py)
TRANSPOSE_GOLDEN = os.path.join(ROOT, "tests", "golden", "reference", "transpose.json")
STEMS = ("c1_train", "c1_test", "c1c_train", "c1c_test", "rag_train", "rag_test")


def _bin(tool):
    build.build_cli()
    return os.path.join(ROOT, "bin", tool)


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def ragged_unsorted():
    """unsorted ids, ids repeated within a row, empty rows, and empty columns (ids 400..419 never occur)"""
    d = synth.ragged(3_000, 400, 9, seed=41, empty_frac=0.1)
    r = np.random.default_rng(42)
    col = d.col.copy()
    for row in range(0, d.num_cases, 7):
        a, b = int(d.row_ptr[row]), int(d.row_ptr[row + 1])
        if b - a >= 2:
            col[a:b] = r.permutation(col[a:b])
            col[b - 1] = col[a]  # a repeated id
    return Data(d.row_ptr, col, d.val, d.target, 420)


def transpose_inputs(d):
    """{name: <stem>}: the text inputs of mcmc_cli.npz converted by bin/convert to <stem>.x / <stem>.y, and
    ragged_unsorted() written by write_binary"""
    z = np.load(CLI_GOLDEN)
    for key in z.files:
        if key.startswith("input/"):
            with open(os.path.join(str(d), key[len("input/"):]), "w") as f:
                f.write(str(z[key]))
    out = {}
    for stem in STEMS:
        p = os.path.join(str(d), stem)
        subprocess.run([_bin("convert"), "-ifile", p, "-ofilex", p + ".x", "-ofiley", p + ".y"], check=True,
                       capture_output=True)
        out[stem] = p
    p = os.path.join(str(d), "ragged")
    write_binary(ragged_unsorted(), p + ".x", p + ".y")
    out["ragged"] = p
    return out


def _read_x(path_x, path_y):
    raw = np.fromfile(path_x, dtype=np.uint32)
    n_rows, n_cols, words = int(raw[4]), int(raw[5]), raw[6:]
    rp, col, val, pos = [0], [], [], 0
    for _ in range(n_rows):
        s = int(words[pos])
        pairs = words[pos + 1:pos + 1 + 2 * s].reshape(-1, 2)
        col.append(pairs[:, 0])
        val.append(pairs[:, 1].view(np.float32))
        rp.append(rp[-1] + s)
        pos += 1 + 2 * s
    y = np.fromfile(path_y, dtype=np.float32)[3:]
    cat = (lambda a, t: np.concatenate(a).astype(t)) if col else (lambda a, t: np.zeros(0, t))
    return Data(np.array(rp, np.uint64), cat(col, np.uint32), cat(val, np.float32), y, n_cols)


@pytest.fixture(scope="module")
def stock(tmp_path_factory):
    """the inputs, each checked against the one the stock tool was run on, and the stock tool's .xt digests"""
    with open(TRANSPOSE_GOLDEN) as f:
        g = json.load(f)
    inputs = transpose_inputs(tmp_path_factory.mktemp("inputs"))
    assert sorted(inputs) == sorted(g["x"])
    for name, stem in inputs.items():
        assert _sha(stem + ".x") == g["x"][name], "the input %s is not the one the golden was made from" % name
    return inputs, g["xt"]


def test_write_transposed_equals_stock_transpose(stock, tmp_path):
    inputs, want = stock
    for name, stem in inputs.items():
        out = str(tmp_path / (name + ".xt"))
        write_transposed(_read_x(stem + ".x", stem + ".y"), out)
        assert _sha(out) == want[name], name


@pytest.mark.parametrize("ranges", [1, 3, 7])
def test_bin_transpose_equals_stock_transpose(stock, tmp_path, ranges):
    """at the default cache, and at caches that cut the columns into at least 3 and 7 ranges"""
    inputs, want = stock
    for name, stem in inputs.items():
        raw = np.fromfile(stem + ".x", dtype=np.uint32)
        n_rows, n_cols = int(raw[4]), int(raw[5])
        nnz = (raw.size - 6 - n_rows) // 2
        xt_bytes = 4 * n_cols + 8 * nnz
        args = [] if ranges == 1 else ["-cache_size", str(2 * (xt_bytes // ranges))]
        out = str(tmp_path / (name + ".xt"))
        p = subprocess.run([_bin("transpose"), "-ifile", stem + ".x", "-ofile", out] + args, capture_output=True,
                           text=True)
        assert p.returncode == 0, (name, p.stderr)
        assert _sha(out) == want[name], name


def test_bin_transpose_refuses_bad_input(tmp_path):
    t = _bin("transpose")
    p = subprocess.run([t, "-ifile", str(tmp_path / "missing.x"), "-ofile", str(tmp_path / "o.xt")], capture_output=True,
                       text=True)
    assert p.returncode == 1 and "could not open" in p.stderr
    d = ragged_unsorted()
    stem = str(tmp_path / "r")
    write_binary(d, stem + ".x", stem + ".y")
    raw = np.fromfile(stem + ".x", dtype=np.uint32)
    raw[:-3].tofile(stem + ".cut.x")  # truncated
    bad = raw.copy()
    row = next(r for r in range(d.num_cases) if d.row_ptr[r + 1] > d.row_ptr[r])
    bad[6 + row + 2 * int(d.row_ptr[row]) + 1] = 10_000  # an id past num_cols
    bad.tofile(stem + ".id.x")
    for name in ("cut", "id"):
        p = subprocess.run([t, "-ifile", stem + "." + name + ".x", "-ofile", str(tmp_path / "o.xt")],
                           capture_output=True, text=True)
        assert p.returncode == 1 and "could not read" in p.stderr, (name, p.stderr)
    p = subprocess.run([t, "-ifile", stem + ".x", "-ofile", str(tmp_path / "o.xt"), "-cache_size", "100"],
                       capture_output=True, text=True)
    assert p.returncode == 1 and "-cache_size must be at least" in p.stderr


@pytest.fixture(scope="module")
def xtblock_dump(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("bin") / "xtblock_dump")
    subprocess.run(["g++", "-O2", "-std=c++17", "-pthread", "-I", os.path.join(ROOT, "libfm_b200", "host"),
                    os.path.join(ROOT, "tests", "xtblock_dump.cpp"), "-o", exe], check=True)
    return exe


@pytest.mark.parametrize("cache_size", [2_000, 5_000, 20_000, 10_000_000])
def test_xt_block_plan_equals_the_rule(xtblock_dump, tmp_path, cache_size):
    d = ragged_unsorted()
    stem = str(tmp_path / "train")
    write_binary(d, stem + ".x", stem + ".y")
    write_transposed(d, stem + ".xt")
    out = str(tmp_path / "dump")
    r = subprocess.run([xtblock_dump, stem, str(cache_size), out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    xt_bytes = 4 * d.num_feature + 8 * d.num_values
    if xt_bytes <= cache_size // 2:
        assert r.stdout.split() == ["resident"]
        return
    want = list(read_xblocks(stem + ".xt", cache_size))
    lines = r.stdout.splitlines()
    assert lines[0] == "has x = 0" and lines[1] == "has xt = 1"
    assert lines[2].startswith("data transpose... num_cases=%d\tnum_values=%d\tnum_features=%d\t"
                               % (d.num_cases, d.num_values, d.num_feature))
    assert lines[3] == "streaming %s.xt: %d blocks of at most %d columns and %d bytes" % (
        stem, len(want), max(hi - lo for lo, hi, _, _ in want), cache_size // 2)
    got = [tuple(int(x) for x in ln.split()) for ln in lines[4:]]
    offset = 24
    for (lo, hi, nnz, off), (wlo, whi, words, sizes) in zip(got, want):
        assert (lo, hi, nnz, off) == (wlo, whi, int(sizes.sum()), offset)
        offset += 4 * words.size
    assert len(got) == len(want)
    assert np.fromfile(out + ".xt", dtype=np.uint32).tobytes() == np.fromfile(stem + ".xt", dtype=np.uint32)[6:].tobytes()
    assert np.array_equal(np.fromfile(out + ".sizes", dtype=np.uint32), np.bincount(d.col, minlength=d.num_feature))


def _cli(args, d):
    return subprocess.run([_bin("libFM")] + args, cwd=str(d), capture_output=True, text=True)


def test_streamed_cli_refusals(tmp_path):
    d = ragged_unsorted()
    for s in ("train", "test"):
        write_binary(d, str(tmp_path / s) + ".x", str(tmp_path / s) + ".y")
        write_transposed(d, str(tmp_path / s) + ".xt")
    base = ["-task", "r", "-train", "train", "-test", "test", "-method", "mcmc", "-dim", "1,1,4", "-iter", "2"]
    raw = np.fromfile(str(tmp_path / "train.xt"), dtype=np.uint32)
    sizes = np.bincount(d.col, minlength=d.num_feature)
    at = int(np.argmax(sizes))
    longest = 4 + 8 * int(sizes[at])
    cache = str(2 * ((4 * (raw.size - 6)) // 5))
    # a column longer than B/2 names the budget it needs
    p = _cli(base + ["-mode", "inorder", "-cache_size", str(2 * longest - 2)], tmp_path)
    assert p.returncode == 1
    assert "column %d of train.xt takes %d bytes: -cache_size must be at least %d" % (at, longest, 2 * longest) \
        in p.stderr, p.stderr
    # a corrupted column header word names the column
    bad = raw.copy()
    bad[6] = 0x7fffffff
    bad.tofile(str(tmp_path / "train.xt"))
    p = _cli(base + ["-mode", "inorder", "-cache_size", cache], tmp_path)
    assert p.returncode == 1 and "column 0 of train.xt: its header word 2147483647" in p.stderr, p.stderr
    # a .xt whose case count disagrees with .y
    bad = raw.copy()
    bad[5] += 1
    bad.tofile(str(tmp_path / "train.xt"))
    p = _cli(base + ["-mode", "inorder", "-cache_size", cache], tmp_path)
    assert p.returncode == 1 and "case count of train.xt and train.y differ" in p.stderr, p.stderr
    # -mode hogwild, -gpus > 1 and -relation stay refused, before anything is read
    raw.tofile(str(tmp_path / "train.xt"))
    p = _cli(base + ["-mode", "hogwild", "-cache_size", cache], tmp_path)
    assert p.returncode == 1 and "outside the libfm_b200 scope" in p.stderr
    p = _cli(base + ["-mode", "inorder", "-gpus", "2", "-cache_size", cache], tmp_path)
    assert p.returncode == 1 and "-gpus must be 1" in p.stderr
    p = _cli(base + ["-mode", "inorder", "-relation", "rel", "-cache_size", cache], tmp_path)
    assert p.returncode == 1 and "relations (-relation) are not supported" in p.stderr
