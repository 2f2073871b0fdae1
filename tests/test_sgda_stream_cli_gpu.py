"""GPU: `bin/libFM -method sgda -cache_size` streaming binary training, test and validation sets (.x/.y from
bin/convert of the text inputs of tests/golden/reference/sgda_cli.npz) against the stock reference's runs on that
data: the learner's stdout lines, the -out and -save_model files and every -rlog column but the time_* ones, under
budgets that give 3+ and 20+ blocks per set.  The reference's results do not depend on how it caches its data, so
the golden of the resident runs is the golden of these.  Regression is byte-identical; classification to within
its 6 printed significant digits (the device's exp()), as in test_sgda_cli_gpu.py."""
import os
import re
import subprocess

import numpy as np
import pytest

from libfm_b200 import build
from test_sgda_cli_gpu import GOLDEN, RUNS, _learner_lines, _numbers_close, _rlog_without_time

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN)
    return {k: str(z[k]) for k in z.files}


def binary_inputs(golden, d):
    """the golden's files in d, every .libfm converted to .libfm.x/.y and removed: the same names load as binary"""
    convert = os.path.join(os.path.dirname(build.cli_path()), "convert")
    for key, text in golden.items():
        if not key.startswith("files/"):
            continue
        p = os.path.join(str(d), key[len("files/"):])
        with open(p, "w") as f:
            f.write(text)
        if p.endswith(".libfm"):
            subprocess.run([convert, "-ifile", p, "-ofilex", p + ".x", "-ofiley", p + ".y"], check=True,
                           capture_output=True)
            os.remove(p)


def cache_for(d, files, n_blocks):
    """a -cache_size that cuts every one of `files` into at least n_blocks blocks"""
    return 2 * min((os.path.getsize(os.path.join(str(d), f + ".x")) - 24) // (n_blocks + 1) for f in files)


def stream_blocks(stdout, f):
    m = re.search(r"streaming %s\.x: (\d+) blocks of at most \d+ rows and \d+ bytes" % re.escape(f), stdout)
    return int(m.group(1)) if m else 0


@pytest.mark.parametrize("n_blocks", [3, 20])
@pytest.mark.parametrize("run", RUNS)
def test_streamed_sgda_cli_matches_reference(run, n_blocks, golden, tmp_path, built_lib):
    exe = build.cli_path()
    if not os.path.exists(exe):
        build.build_all()
    binary_inputs(golden, tmp_path)
    args = golden[run + "/args"].split()
    files = [args[args.index(f) + 1] for f in ("-train", "-test", "-validation")]
    cache = cache_for(tmp_path, files, n_blocks)
    for mode in (["inorder", "ordered"] if n_blocks == 3 and run == "reg_wraps" else ["inorder"]):
        p = subprocess.run([exe, "-method", "sgda", "-mode", mode, "-cache_size", str(cache)] + args, cwd=tmp_path,
                           capture_output=True, text=True)
        assert p.returncode == 0, p.stderr
        for f in files:
            assert stream_blocks(p.stdout, f) >= n_blocks, (f, p.stdout)
        outs = {"out": (tmp_path / "out.txt").read_text(), "model": (tmp_path / "model.txt").read_text()}
        got_lines, ref_lines = _learner_lines(p.stdout), _learner_lines(golden[run + "/stdout"])
        got_rlog = _rlog_without_time((tmp_path / "rlog.txt").read_text())
        ref_rlog = _rlog_without_time(golden[run + "/rlog"])
        assert got_rlog[0] == ref_rlog[0]
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
