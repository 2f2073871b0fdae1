"""GPU: bin/libFM -method mcmc|als -cache_size streaming the transposed binary data (.xt from bin/transpose)
against what the stock reference printed and wrote for the same runs (tests/golden/reference/mcmc_cli.npz, the
assertions of test_cli_mcmc_gpu.test_cli_matches_stock_reference) and the resident runs.  The refusals, which
happen before the GPU is touched, are in test_stream_mcmc_cpu.py."""
import os
import re
import subprocess

import numpy as np
import pytest

from libfm_b200 import build
from test_cli_mcmc_gpu import GOLDEN, _inputs, _rlog_without_time

pytestmark = pytest.mark.gpu

RUNS = ["mcmc_default_r", "als_r", "mcmc_c", "als_c", "mcmc_meta_r", "als_meta_r"]


@pytest.fixture(scope="module")
def cli():
    build.build_cli()
    return build.cli_path()


def _binary_inputs(z, d, transpose=True):
    """the text inputs of the runs as .x/.y (bin/convert) and .xt (bin/transpose), the text files removed"""
    _inputs(z, d)
    bindir = os.path.dirname(build.cli_path())
    for stem in ("c1_train", "c1_test", "c1c_train", "c1c_test", "rag_train", "rag_test"):
        p = os.path.join(str(d), stem)
        subprocess.run([os.path.join(bindir, "convert"), "-ifile", p, "-ofilex", p + ".x", "-ofiley", p + ".y"],
                       check=True, capture_output=True)
        if transpose:
            subprocess.run([os.path.join(bindir, "transpose"), "-ifile", p + ".x", "-ofile", p + ".xt"],
                           check=True, capture_output=True)
        os.remove(p)


def _xt_bytes(path):
    raw = np.fromfile(path, dtype=np.uint32)
    return 4 * (raw.size - 6), raw


def _cache(d, train, test):
    """a -cache_size giving at least 4 train and 2 test blocks"""
    tr, _ = _xt_bytes(os.path.join(str(d), train + ".xt"))
    te, _ = _xt_bytes(os.path.join(str(d), test + ".xt"))
    return 2 * min(tr // 5, te // 3)


def _run(cli, d, args):
    return subprocess.run([cli] + args, cwd=d, capture_output=True, text=True)


def _check_against_reference(z, run, p, d):
    assert p.returncode == 0, p.stderr
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("#Iter") or ln.startswith("#nans")]
    want = str(z[run + "/lines"]).splitlines()
    for i, (got, exp) in enumerate(zip(lines, want)):
        assert got == exp, "%s: line %d differs: %r != %r" % (run, i, got, exp)
    assert len(lines) == len(want)
    for f in ("out", "model"):
        exp = str(z[run + "/" + f])
        got = (d / f).read_text() if (d / f).exists() else ""
        assert got == exp, "%s: -%s file differs" % (run, "out" if f == "out" else "save_model")
    exp = str(z[run + "/rlog"])
    got = (d / "rlog").read_text() if (d / "rlog").exists() else ""
    assert _rlog_without_time(got) == _rlog_without_time(exp)


def _blocks(stdout, stem):
    m = re.search(r"streaming %s\.xt: (\d+) blocks of at most \d+ columns and \d+ bytes" % stem, stdout)
    return int(m.group(1)) if m else 0


@pytest.mark.parametrize("run", RUNS)
def test_streamed_cli_matches_stock_reference(run, cli, tmp_path, built_lib):
    z = np.load(GOLDEN)
    _binary_inputs(z, tmp_path)
    args = str(z[run + "/args"]).split()
    train, test = args[args.index("-train") + 1], args[args.index("-test") + 1]
    cache = _cache(tmp_path, train, test)
    p = _run(cli, tmp_path, args + ["-mode", "inorder", "-cache_size", str(cache)])
    assert _blocks(p.stdout, train) >= 4 and _blocks(p.stdout, test) >= 2, p.stdout + p.stderr
    assert "has x = 0" in p.stdout and "data transpose... " in p.stdout
    _check_against_reference(z, run, p, tmp_path)


def test_streamed_cli_ordered_mode(cli, tmp_path, built_lib):
    z = np.load(GOLDEN)
    run = "als_meta_r"
    _binary_inputs(z, tmp_path)
    args = str(z[run + "/args"]).split()
    p = _run(cli, tmp_path, args + ["-mode", "ordered", "-cache_size", str(_cache(tmp_path, "rag_train", "rag_test"))])
    assert _blocks(p.stdout, "rag_train") >= 4
    _check_against_reference(z, run, p, tmp_path)


def _outputs(d):
    return {f: (d / f).read_text() for f in ("out", "model") if (d / f).exists()}


@pytest.mark.parametrize("case", ["no_xt", "budget_covers_file"])
def test_resident_when_not_streamed(case, cli, tmp_path, built_lib):
    """no .xt, or a budget of at least the file: stdout and files exactly as the resident run's"""
    z = np.load(GOLDEN)
    run = "als_r"
    args = str(z[run + "/args"]).split() + ["-mode", "inorder"]
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    _binary_inputs(z, tmp_path / "a", transpose=False)
    _binary_inputs(z, tmp_path / "b", transpose=(case != "no_xt"))
    base = _run(cli, tmp_path / "a", args)
    big = 2 * max(os.path.getsize(str(tmp_path / "b" / s)) for s in ("c1_train.x", "c1_train.xt", "c1_test.xt")
                  if (tmp_path / "b" / s).exists())
    cache = 1000 if case == "no_xt" else big
    p = _run(cli, tmp_path / "b", args + ["-cache_size", str(cache)])
    assert base.returncode == 0 and p.returncode == 0, base.stderr + p.stderr
    assert "streaming" not in p.stdout
    assert p.stdout == base.stdout
    assert _outputs(tmp_path / "b") == _outputs(tmp_path / "a")
    assert _rlog_without_time((tmp_path / "b" / "rlog").read_text()) == _rlog_without_time(
        (tmp_path / "a" / "rlog").read_text())
