"""GPU: bin/libFM -mode inorder -method mcmc|als (and no -method: MCMC is the default) against what the stock
reference command line printed and wrote for the same files and seed (tests/golden/reference/mcmc_cli.npz,
scripts/make_mcmc_cli_golden.py): the #Iter and #nans lines, the -out file, the -rlog file without its
time columns and the ALS -save_model file must be identical.  Also the refusals and the MCMC model-file WARNING."""
import os
import subprocess

import numpy as np
import pytest

from libfm_b200 import build

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference", "mcmc_cli.npz")


@pytest.fixture(scope="module")
def cli():
    build.build_cli()
    return build.cli_path()


def _inputs(z, d):
    for key in z.files:
        if key.startswith("input/"):
            with open(os.path.join(d, key[len("input/"):]), "w") as f:
                f.write(str(z[key]))


def _rlog_without_time(text):
    rows = [ln.split("\t") for ln in text.splitlines()]
    keep = [i for i, h in enumerate(rows[0]) if not h.startswith("time_")] if rows else []
    return [[r[i] for i in keep] for r in rows]


@pytest.mark.parametrize("run", ["mcmc_default_r", "als_r", "mcmc_c", "als_c", "mcmc_meta_r", "als_meta_r"])
def test_cli_matches_stock_reference(run, cli, tmp_path, built_lib):
    z = np.load(GOLDEN)
    _inputs(z, tmp_path)
    p = subprocess.run([cli] + str(z[run + "/args"]).split() + ["-mode", "inorder"], cwd=tmp_path,
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("#Iter") or ln.startswith("#nans")]
    want = str(z[run + "/lines"]).splitlines()
    for i, (got, exp) in enumerate(zip(lines, want)):
        assert got == exp, "%s: line %d differs: %r != %r" % (run, i, got, exp)
    assert len(lines) == len(want)
    assert "Final" not in p.stdout
    for f in ("out", "model"):
        exp = str(z[run + "/" + f])
        got = (tmp_path / f).read_text() if (tmp_path / f).exists() else ""
        assert got == exp, "%s: -%s file differs" % (run, "out" if f == "out" else "save_model")
    exp = str(z[run + "/rlog"])
    got = (tmp_path / "rlog").read_text() if (tmp_path / "rlog").exists() else ""
    assert _rlog_without_time(got) == _rlog_without_time(exp)


def _run(cli, d, args):
    return subprocess.run([cli] + args.split(), cwd=d, capture_output=True, text=True)


def test_cli_mcmc_refusals_and_warning(cli, tmp_path, built_lib):
    z = np.load(GOLDEN)
    _inputs(z, tmp_path)
    base = "-task r -train c1_train -test c1_test -iter 1"
    p = _run(cli, tmp_path, base + " -mode inorder -save_model m")  # libfm.cpp:123-127
    assert p.returncode == 0 and "WARNING: -save_model enabled only for SGD and ALS." in p.stdout
    assert not (tmp_path / "m").exists()
    p = _run(cli, tmp_path, base + " -method mcmc -mode inorder -load_model m")
    assert p.returncode == 0 and "WARNING: -load_model enabled only for SGD and ALS." in p.stdout
    p = _run(cli, tmp_path, base + " -method als")
    assert p.returncode != 0 and "outside the libfm_b200 scope" in p.stderr and "use -mode inorder" in p.stderr
    p = _run(cli, tmp_path, base + " -method mcmc -mode inorder -gpus 2")
    assert p.returncode != 0 and "-gpus must be 1" in p.stderr
    p = _run(cli, tmp_path, base + " -method als -mode inorder -relation rel")
    assert p.returncode != 0 and "relations" in p.stderr
