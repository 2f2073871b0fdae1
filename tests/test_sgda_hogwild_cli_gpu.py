"""GPU: `bin/libFM -method sgda -validation ...` in the default -mode hogwild (the windowed fp32 epoch) against the
stock reference binary (oracle/_ref/libFM) on a planted data set generated here: the same learner lines as the
-mode inorder run, as many #Iter lines, the same -rlog columns, one -out value per test row, a model file that
-load_model reads back, and a Final test RMSE within 0.05 of the reference's."""
import os
import subprocess

import pytest

from libfm_b200 import build, synth
from oracle.binding import REF_CLI

pytestmark = pytest.mark.gpu

ARGS = ["-task", "r", "-train", "train.libfm", "-test", "test.libfm", "-validation", "val.libfm", "-method", "sgda",
        "-dim", "1,1,8", "-iter", "12", "-learn_rate", "0.01", "-init_stdev", "0.1", "-seed", "3", "-meta", "meta.txt"]
LEARNER_LINES = ("learnrate=", "learnrates=", "#iterations=", "Training using", "DON'T FORGET", "Using ",
                 "#Iter=", "Final\t", "Writing FM model")


def _run(exe, args, cwd):
    return subprocess.run([exe] + args, cwd=cwd, capture_output=True, text=True, timeout=900)


def _lines(stdout):
    return [l for l in stdout.splitlines() if l.startswith(LEARNER_LINES)]


def _final_test(stdout):
    line = [l for l in stdout.splitlines() if l.startswith("Final")][-1]
    return float([t for t in line.split("\t") if t.startswith("Test")][0].split("=")[1])


def test_hogwild_sgda_command_line(tmp_path):
    exe = build.cli_path()
    if not os.path.exists(exe):
        build.build_all()
    if not os.path.exists(REF_CLI):
        pytest.skip("oracle/_ref/libFM not built")
    d = synth.two_field(60_000, 600, 400, seed=5, planted_k=4)
    train, rest = synth.split_rows(d, 40_000)
    val, test = synth.split_rows(rest, 10_000)
    for name, part in [("train", train), ("val", val), ("test", test)]:
        synth.to_libfm_text(part, str(tmp_path / (name + ".libfm")))
    (tmp_path / "meta.txt").write_text("".join("%d\n" % (i >= 600) for i in range(1000)))
    out = ["-rlog", "log.txt", "-out", "out.txt", "-save_model", "model.txt"]
    ours = _run(exe, ARGS + out, tmp_path)
    assert ours.returncode == 0, ours.stderr
    ours_log = (tmp_path / "log.txt").read_text().splitlines()
    n_out = len((tmp_path / "out.txt").read_text().splitlines())
    inorder = _run(exe, ARGS + ["-mode", "inorder", "-rlog", "in_log.txt", "-out", "in_out.txt", "-save_model",
                                "in_model.txt"], tmp_path)
    assert inorder.returncode == 0, inorder.stderr
    ref_out = ["-rlog", "ref_log.txt", "-out", "ref_out.txt", "-save_model", "ref_model.txt"]
    ref = _run(REF_CLI, ARGS + ref_out, tmp_path)
    assert ref.returncode == 0, ref.stderr
    key = lambda l: [p for p in LEARNER_LINES if l.startswith(p)][0]  # noqa: E731
    assert [key(l) for l in _lines(ours.stdout)] == [key(l) for l in _lines(inorder.stdout)]
    assert sum(l.startswith("#Iter=") for l in ours.stdout.splitlines()) == 12
    ref_log = (tmp_path / "ref_log.txt").read_text().splitlines()
    assert ours_log[0].split("\t") == ref_log[0].split("\t")
    assert len(ours_log) == len(ref_log)
    assert n_out == test.num_cases
    a, b = _final_test(ours.stdout), _final_test(ref.stdout)
    print("\n[sgda -mode hogwild] Final Test %.5f, reference %.5f" % (a, b))
    assert abs(a - b) < 0.05, (a, b)
    back = _run(exe, ["-task", "r", "-train", "train.libfm", "-test", "test.libfm", "-dim", "1,1,8", "-iter", "0",
                      "-learn_rate", "0.01", "-load_model", "model.txt", "-method", "sgd", "-mode", "inorder"],
                tmp_path)
    assert back.returncode == 0, back.stderr
