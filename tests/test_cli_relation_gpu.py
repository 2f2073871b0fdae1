"""GPU: bin/libFM -relation (MCMC and ALS on block-structured data) in -mode inorder and ordered against what the
stock reference command line printed and wrote for the same files and seed (tests/golden/reference/
mcmc_relation_cli.npz, scripts/make_relation_cli_golden.py): the #Iter and #nans lines, the -out file, the -rlog
file without its time columns and the ALS -save_model file must be identical.  The runs cover a user and an item
block over empty main rows (binary and text joins, a .groups file), ALS with per-group -regular, -save_model and
-load_model, classification, and a main table with features and -meta groups ahead of a block's."""
import os
import subprocess

import numpy as np
import pytest

from libfm_b200 import build
from test_cli_mcmc_gpu import _rlog_without_time

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference", "mcmc_relation_cli.npz")
RUNS = ["mcmc_user_item_r", "als_groups_r", "als_load_r", "mcmc_c", "mcmc_meta_r"]


@pytest.fixture(scope="module")
def cli():
    build.build_cli()
    return build.cli_path()


@pytest.mark.parametrize("mode", ["inorder", "ordered"])
@pytest.mark.parametrize("run", RUNS)
def test_relation_cli_matches_stock_reference(run, mode, cli, tmp_path, built_lib):
    z = np.load(GOLDEN)
    ds = str(z[run + "/data"])
    for key in z.files:
        if key.startswith("input/%s/" % ds):
            (tmp_path / key.split("/")[-1]).write_bytes(z[key].tobytes())
    args = str(z[run + "/args"])
    if "-load_model" in args:
        (tmp_path / "als_groups_r.model").write_text(str(z["als_groups_r/model"]))
    p = subprocess.run([cli] + args.split() + ["-mode", mode], cwd=tmp_path, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    assert "#relations: %d" % (args.split("-relation ")[1].split()[0].count(",") + 1) in p.stdout
    assert "WARNING" not in p.stdout
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("#Iter") or ln.startswith("#nans")]
    want = str(z[run + "/lines"]).splitlines()
    for i, (got, exp) in enumerate(zip(lines, want)):
        assert got == exp, "%s: line %d differs: %r != %r" % (run, i, got, exp)
    assert len(lines) == len(want)
    for f in ("out", "model"):
        exp = str(z[run + "/" + f])
        got = (tmp_path / f).read_text() if (tmp_path / f).exists() else ""
        assert got == exp, "%s: -%s file differs" % (run, "out" if f == "out" else "save_model")
    exp = str(z[run + "/rlog"])
    got = (tmp_path / "rlog").read_text() if (tmp_path / "rlog").exists() else ""
    assert _rlog_without_time(got) == _rlog_without_time(exp)
