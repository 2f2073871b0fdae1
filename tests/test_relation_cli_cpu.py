"""CPU: the command line's relation loaders (RelationData, RelationJoin in host/sparse_data.h, through
tests/relation_dump.cpp) on blocks written as the reference reads them, and the -relation refusals of bin/libFM,
which all happen before the GPU is touched."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from libfm_b200 import build
from libfm_b200.model import RelationData, RelationJoin

sys.path.insert(0, os.path.join(ROOT, "scripts"))
from make_relation_golden import cases, write_block_files  # noqa: E402

CLI_GOLDEN = os.path.join(ROOT, "tests", "golden", "reference", "mcmc_relation_cli.npz")


@pytest.fixture(scope="module")
def relation_dump(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("bin") / "relation_dump")
    subprocess.run(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "libfm_b200", "host"),
                    os.path.join(ROOT, "tests", "relation_dump.cpp"), "-o", exe], check=True)
    return exe


@pytest.fixture(scope="module")
def cli():
    build.build_cli()
    return os.path.join(ROOT, "bin", "libFM")


def _dump(exe, stem, n_tr, n_te, out):
    p = subprocess.run([exe, stem, str(n_tr), str(n_te), out], capture_output=True, text=True)
    if p.returncode != 0:
        return None, p.stderr
    raw = open(out, "rb").read()
    nc, nf, G, nnz = (int(x) for x in np.frombuffer(raw[:32], np.uint64))
    o = 32
    def take(dt, n):
        nonlocal o
        a = np.frombuffer(raw[o:o + n * np.dtype(dt).itemsize], dt)
        o += n * np.dtype(dt).itemsize
        return a
    r = dict(num_cases=nc, num_feature=nf, num_groups=G, col_ptr=take(np.uint64, nf + 1), row=take(np.uint32, nnz),
             val=take(np.float32, nnz), group=take(np.uint32, nf), train=take(np.uint32, n_tr),
             test=take(np.uint32, n_te))
    assert o == len(raw)
    return r, p.stderr


def _blocks():
    """(name, block, train cases, test cases): binary and text joins, with and without .groups, a row naming an id
    twice, rows no train case joins"""
    out = []
    for name in ("user_item_mcmc", "awkward_mcmc"):
        c = cases()[name]
        for i, b in enumerate(c["blocks"]):
            out.append(("%s_%d" % (name, i), b, c["train"].num_cases, c["test"].num_cases))
    return out


@pytest.mark.parametrize("i", range(4))
def test_loaders_read_what_was_written(i, relation_dump, tmp_path):
    name, b, n_tr, n_te = _blocks()[i]
    stem = str(tmp_path / name)
    write_block_files(stem, b, n_tr, n_te)
    got, err = _dump(relation_dump, stem, n_tr, n_te, str(tmp_path / "dump"))
    assert got is not None, err
    want = RelationData.load(stem)
    d = b["data"]
    assert (got["num_cases"], got["num_feature"]) == (d.num_cases, d.num_feature)
    assert (got["num_cases"], got["num_feature"]) == (want.num_cases, want.num_feature)
    for key, w in (("col_ptr", want.col_ptr), ("row", want.row), ("val", want.val), ("group", want.attr_group)):
        assert got[key].tobytes() == np.asarray(w).tobytes(), key
    assert got["num_groups"] == want.num_attr_groups
    if b["groups"] is None:
        assert got["num_groups"] == 1 and not got["group"].any()
    else:
        assert got["group"].tolist() == list(b["groups"])
    assert got["train"].tolist() == b["train"].tolist()
    assert got["test"].tolist() == b["test"].tolist()
    assert got["train"].tolist() == RelationJoin.load(stem + ".train", n_tr).rows.tolist()


def test_binary_and_text_joins_agree(relation_dump, tmp_path):
    _, b, n_tr, n_te = _blocks()[0]
    res = []
    for binary in (True, False):
        stem = str(tmp_path / ("bin" if binary else "txt"))
        write_block_files(stem, dict(b, binary=binary), n_tr, n_te)
        head = open(stem + ".train", "rb").read(8)
        assert (np.frombuffer(head, np.uint32).tolist() == [1, 4]) == binary
        got, err = _dump(relation_dump, stem, n_tr, n_te, str(tmp_path / "dump"))
        assert got is not None, err
        res.append((got["train"].tolist(), got["test"].tolist()))
    assert res[0] == res[1] == (b["train"].tolist(), b["test"].tolist())


@pytest.mark.parametrize("binary", [True, False], ids=["binary", "text"])
def test_short_join_is_refused(binary, relation_dump, tmp_path):
    _, b, n_tr, n_te = _blocks()[0]
    stem = str(tmp_path / "rel")
    write_block_files(stem, dict(b, binary=binary, train=b["train"][:-1]), n_tr, n_te)
    got, err = _dump(relation_dump, stem, n_tr, n_te, str(tmp_path / "dump"))
    assert got is None
    assert "relations: %s.train maps %d cases, its data set has %d" % (stem, n_tr - 1, n_tr) in err, err


def test_missing_groups_is_one_group(relation_dump, tmp_path):
    _, b, n_tr, n_te = _blocks()[1]   # the item block, written with a .groups file
    stem = str(tmp_path / "rel")
    write_block_files(stem, b, n_tr, n_te)
    with_groups, _ = _dump(relation_dump, stem, n_tr, n_te, str(tmp_path / "dump"))
    assert with_groups["num_groups"] == 2
    os.remove(stem + ".groups")
    got, err = _dump(relation_dump, stem, n_tr, n_te, str(tmp_path / "dump"))
    assert got is not None, err
    assert got["num_groups"] == 1 and not got["group"].any()
    # a short .groups file reads its missing values as group 0
    with open(stem + ".groups", "w") as f:
        f.write("1 1 1\n")
    got, _ = _dump(relation_dump, stem, n_tr, n_te, str(tmp_path / "dump"))
    assert got["num_groups"] == 2 and got["group"].tolist() == [1, 1, 1] + [0] * (b["data"].num_feature - 3)


def test_missing_or_malformed_xt_is_named(relation_dump, tmp_path):
    _, b, n_tr, n_te = _blocks()[0]
    stem = str(tmp_path / "rel")
    write_block_files(stem, b, n_tr, n_te)
    raw = open(stem + ".xt", "rb").read()
    os.remove(stem + ".xt")
    got, err = _dump(relation_dump, stem, n_tr, n_te, str(tmp_path / "dump"))
    assert got is None and "relations: could not open %s.xt" % stem in err, err
    with open(stem + ".xt", "wb") as f:
        f.write(raw[:-5])
    got, err = _dump(relation_dump, stem, n_tr, n_te, str(tmp_path / "dump"))
    assert got is None and "relations: could not read %s.xt" % stem in err, err


def _run_dir(tmp_path, run="mcmc_user_item_r"):
    z = np.load(CLI_GOLDEN)
    ds = str(z[run + "/data"])
    for key in z.files:
        if key.startswith("input/%s/" % ds):
            (tmp_path / key.split("/")[-1]).write_bytes(z[key].tobytes())
    return "-task r -train train -test test -iter 1 -relation ui_rel0,ui_rel1"


def _cli(cli, d, args):
    return subprocess.run([cli] + args.split(), cwd=d, capture_output=True, text=True)


def test_cli_refusals(cli, tmp_path):
    base = _run_dir(tmp_path)
    p = _cli(cli, tmp_path, base + " -method sgd")
    assert p.returncode == 1 and "relations are not supported with SGD" in p.stderr, p.stderr
    p = _cli(cli, tmp_path, base + " -method sgda -validation test -mode inorder")
    assert p.returncode == 1 and "relations (-relation) are not supported with -method sgda" in p.stderr, p.stderr
    for m in ("mcmc", "als"):
        p = _cli(cli, tmp_path, base + " -method %s -mode inorder -cache_size 1000000" % m)
        assert p.returncode == 1 and "relations (-relation) are not supported with -cache_size" in p.stderr
        assert "Loading train" not in p.stdout   # refused before anything is read
        p = _cli(cli, tmp_path, base + " -method %s -mode hogwild" % m)
        assert p.returncode == 1 and "outside the libfm_b200 scope" in p.stderr
        p = _cli(cli, tmp_path, base + " -method %s -mode inorder -gpus 2" % m)
        assert p.returncode == 1 and "-gpus must be 1" in p.stderr


def test_cli_names_missing_relation_files(cli, tmp_path):
    base = _run_dir(tmp_path)
    # a stem without its .xt: -relation is refused before anything is read
    for m in ("mcmc", "als"):
        p = _cli(cli, tmp_path, base.replace("ui_rel1", "nope") + " -method %s -mode inorder" % m)
        assert p.returncode == 1 and "relations (-relation) are not supported with -method %s" % m in p.stderr
        assert "Loading train" not in p.stdout
    # a malformed .xt, a missing join and a short join are named as they load
    raw = (tmp_path / "ui_rel1.xt").read_bytes()
    (tmp_path / "ui_rel1.xt").write_bytes(raw[:-5])
    p = _cli(cli, tmp_path, base + " -method als -mode inorder")
    assert p.returncode == 1 and "relations: could not read ui_rel1.xt" in p.stderr, p.stderr
    assert "#relations: 2" in p.stdout
    (tmp_path / "ui_rel1.xt").write_bytes(raw)
    os.remove(str(tmp_path / "ui_rel1.test"))
    p = _cli(cli, tmp_path, base + " -method mcmc -mode ordered")
    assert p.returncode == 1 and "relations: could not open ui_rel1.test" in p.stderr, p.stderr
    # the joins are read with the case counts of the data sets they join
    (tmp_path / "ui_rel1.test").write_text("0\n1\n")
    p = _cli(cli, tmp_path, base + " -method mcmc -mode ordered")
    assert p.returncode == 1 and "relations: ui_rel1.test maps 2 cases, its data set has 400" in p.stderr, p.stderr
