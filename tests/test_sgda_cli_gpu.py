"""GPU: `bin/libFM -method sgda -mode inorder|ordered` against the stock reference's own runs
(tests/golden/reference/sgda_cli.npz, scripts/make_sgda_cli_golden.py): the learner's stdout lines, the -out and
-save_model files and every -rlog column but the time_* ones.  Regression is byte-identical; classification goes
through the device's exp(), so its printed numbers are compared to within their 6 significant digits."""
import os
import subprocess

import numpy as np
import pytest

from libfm_b200 import build

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference", "sgda_cli.npz")
RUNS = ["reg_wraps", "reg_val_long", "reg_exact", "cls", "load_model", "iter1"]
LEARNER_LINES = ("learnrate=", "learnrates=", "#iterations=", "Training using", "DON'T FORGET", "Using ",
                 "#Iter=", "Final\t", "Writing FM model")


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN)
    return {k: str(z[k]) for k in z.files}


def _learner_lines(stdout):
    return [l for l in stdout.splitlines() if l.startswith(LEARNER_LINES)]


def _rlog_without_time(text):
    rows = [l.split("\t") for l in text.splitlines()]
    keep = [i for i, h in enumerate(rows[0]) if not h.startswith("time_")]
    return [[r[i] for i in keep] for r in rows]


def _numbers_close(a, b):
    """the same tokens, numbers within the last printed digit (6 significant digits)"""
    ta, tb = a.split(), b.split()
    assert len(ta) == len(tb)
    for x, y in zip(ta, tb):
        if x == y:
            continue
        fx, fy = float(x.split("=")[-1]), float(y.split("=")[-1])
        assert abs(fx - fy) <= 2e-6 * max(abs(fx), abs(fy)) + 1e-12, (x, y)


@pytest.mark.parametrize("mode", ["inorder", "ordered"])
@pytest.mark.parametrize("run", RUNS)
def test_sgda_cli_matches_reference(run, mode, golden, tmp_path):
    exe = build.cli_path()
    if not os.path.exists(exe):
        build.build_all()
    for key, text in golden.items():
        if key.startswith("files/"):
            (tmp_path / key[len("files/"):]).write_text(text)
    args = golden[run + "/args"].split()
    p = subprocess.run([exe, "-method", "sgda", "-mode", mode] + args, cwd=tmp_path, capture_output=True,
                       text=True)
    assert p.returncode == 0, p.stderr
    outs = {"out": (tmp_path / "out.txt").read_text(), "model": (tmp_path / "model.txt").read_text()}
    got_lines, ref_lines = _learner_lines(p.stdout), _learner_lines(golden[run + "/stdout"])
    got_rlog = _rlog_without_time((tmp_path / "rlog.txt").read_text())
    ref_rlog = _rlog_without_time(golden[run + "/rlog"])
    assert got_rlog[0] == ref_rlog[0]  # the columns, in the reference's order
    if run != "cls":
        assert got_lines == ref_lines
        assert got_rlog == ref_rlog
        for key in outs:
            assert outs[key] == golden[run + "/" + key], key
    else:
        assert len(got_lines) == len(ref_lines)
        for a, b in zip(got_lines, ref_lines):
            _numbers_close(a, b)
        assert len(got_rlog) == len(ref_rlog)
        for a, b in zip(got_rlog[1:], ref_rlog[1:]):
            _numbers_close(" ".join(a), " ".join(b))
        for key in outs:
            _numbers_close(outs[key], golden[run + "/" + key])
