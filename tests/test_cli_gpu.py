"""GPU: the drop-in command line (bin/libFM, C++ host over the C ABI) against what the
stock reference binary printed and wrote on BASELINE config C1 with the same flags
(tests/golden/reference/outputs.npz, scripts/make_ref_golden.py): same stdout lines,
same -out / -save_model / -rlog files.  The tests of integration/ need the reference
binaries themselves (oracle/_ref, built from a checkout of the reference) and skip without them."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, digest
from libfm_b200 import synth
from oracle.binding import REF_CLI, REF_CLI_B200, REF_CONVERT

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "bin", "libFM")
CONVERT = os.path.join(ROOT, "bin", "convert")


def _run(binary, args, cwd):
    r = subprocess.run([binary] + args, capture_output=True, text=True, cwd=cwd, timeout=600)
    return r


def _file_digest(path):
    return digest(np.frombuffer(open(path, "rb").read(), np.uint8))


def write_c1_files(d):
    synth.to_libfm_text(synth.plumbing_10k(), os.path.join(d, "train.libfm"))
    synth.to_libfm_text(synth.plumbing_10k(seed=99, n_rows=2000), os.path.join(d, "test.libfm"))


@pytest.fixture(scope="module")
def c1_files(tmp_path_factory, ref_golden):
    d = tmp_path_factory.mktemp("c1")
    write_c1_files(str(d))
    # the files the reference binary read
    assert _file_digest(str(d / "train.libfm")) == ref_golden["c1_train_sha"]
    assert _file_digest(str(d / "test.libfm")) == ref_golden["c1_test_sha"]
    return d


def _need():
    if not os.path.exists(CLI):
        pytest.skip("CLI binaries not built")


def _need_ref():
    _need()
    if not (os.path.exists(REF_CLI) and os.path.exists(REF_CLI_B200)):
        pytest.skip("oracle/_ref/libFM and libFM_b200 not built")


def _iters(stdout):
    return [l for l in stdout.splitlines() if l.startswith("#Iter=") or l.startswith("Final")]


INORDER_CASES = [("r", []), ("r", ["-regular", "0,0,0.01"]), ("c", ["-dim", "1,1,4"])]


def inorder_args(task, extra):
    base = ["-task", task, "-train", "train.libfm", "-test", "test.libfm", "-method", "sgd",
            "-dim", "1,1,8", "-iter", "3", "-learn_rate", "0.01", "-init_stdev", "0.1", "-seed", "42"]
    if "-dim" in extra:
        base = [a for i, a in enumerate(base) if not (a == "-dim" or (i > 0 and base[i - 1] == "-dim"))]
    return base + extra


@pytest.mark.parametrize("task,extra", INORDER_CASES)
def test_cli_inorder_equals_reference_cli(c1_files, task, extra, ref_golden):
    _need()
    i = INORDER_CASES.index((task, extra))
    g = lambda key: ref_golden["inorder%d_%s" % (i, key)]  # noqa: E731
    ours = _run(CLI, inorder_args(task, extra) + ["-mode", "inorder", "-out", "our_pred.txt", "-save_model",
                                                  "our_model.txt", "-rlog", "our_log.tsv"], c1_files)
    assert ours.returncode == 0, ours.stderr
    assert _iters(ours.stdout) == g("iters").tolist() and len(g("iters")) == 4
    rd = lambda f: open(os.path.join(c1_files, f)).read()  # noqa: E731
    if task == "r":
        assert _file_digest(os.path.join(c1_files, "our_pred.txt")) == g("pred_sha")
        assert _file_digest(os.path.join(c1_files, "our_model.txt")) == g("model_sha")
    else:
        a = np.loadtxt(os.path.join(c1_files, "our_pred.txt"))
        np.testing.assert_allclose(a, g("pred"), atol=2e-6)
    # rlog: same header, same metric columns (time columns differ by construction)
    lo, lr = rd("our_log.tsv").splitlines(), g("log").tolist()
    assert lo[0] == lr[0] and len(lo) == len(lr) == 4
    hdr = lo[0].split("\t")
    for a, b in zip(lo[1:], lr[1:]):
        fa, fb = a.split("\t"), b.split("\t")
        for name, x, y in zip(hdr, fa, fb):
            if not name.startswith("time"):
                assert x == y, (name, x, y)


def test_cli_binary_input_equals_text_input(c1_files):
    _need()
    for stem in ("train", "test"):  # bin/convert writes what the reference's convert writes (test_host_cpu.py)
        r = _run(CONVERT, ["--ifile", stem + ".libfm", "--ofilex", stem + ".bin.x", "--ofiley", stem + ".bin.y"], c1_files)
        assert os.path.exists(os.path.join(c1_files, stem + ".bin.x")), r.stdout + r.stderr
    base = ["-task", "r", "-method", "sgd", "-iter", "2", "-learn_rate", "0.01", "-seed", "7", "-mode", "inorder"]
    t = _run(CLI, base + ["-train", "train.libfm", "-test", "test.libfm"], c1_files)
    b = _run(CLI, base + ["-train", "train.bin", "-test", "test.bin"], c1_files)
    assert t.returncode == 0 and b.returncode == 0, t.stderr + b.stderr
    assert _iters(t.stdout) == _iters(b.stdout) and len(_iters(t.stdout)) == 3


HOGWILD_ARGS = ["-task", "r", "-train", "train.libfm", "-test", "test.libfm", "-method", "sgd",
                "-iter", "5", "-learn_rate", "0.01", "-seed", "42"]


def test_cli_hogwild_tracks_reference(c1_files, ref_golden):
    _need()
    ours = _run(CLI, HOGWILD_ARGS, c1_files)  # default mode: hogwild
    assert ours.returncode == 0, ours.stderr
    val = lambda l: [float(t.split("=")[1]) for t in l.split("\t") if t.startswith(("Train", "Test"))]  # noqa: E731
    a, b = val(_iters(ours.stdout)[-1]), val(str(ref_golden["hogwild_iters"][-1]))
    assert abs(a[0] - b[0]) < 0.05 and abs(a[1] - b[1]) < 0.05, (a, b)


def _gpu_count():
    r = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True)
    return sum(1 for l in r.stdout.splitlines() if l.startswith("GPU ")) if r.returncode == 0 else 0


TWO_GPU_ARGS = ["-task", "r", "-train", "train.libfm", "-test", "test.libfm", "-method", "sgd",
                "-iter", "8", "-learn_rate", "0.01", "-seed", "42"]


def test_cli_two_gpus_row_sharded(c1_files, ref_golden):
    """bin/libFM -gpus 2: the rows are cut into two shards, one context per GPU in ONE process, one exchange of
    w0|w|V per epoch over peer memory (fm_peer.cu).  Runs only where two GPUs are visible."""
    _need()
    if _gpu_count() < 2:
        pytest.skip("needs 2 GPUs")
    ours = _run(CLI, TWO_GPU_ARGS + ["-gpus", "2"], c1_files)
    assert ours.returncode == 0, ours.stderr
    val = lambda l: [float(t.split("=")[1]) for t in l.split("\t") if t.startswith(("Train", "Test"))]  # noqa: E731
    a, b = val(_iters(ours.stdout)[-1]), val(str(ref_golden["two_gpu_iters"][-1]))
    print("\n[cli -gpus 2] final Train/Test %s vs the reference's single stream %s" % (a, b))
    # C1 is uniform-random ratings on 10 k rows (nothing to learn, every feature seen once or twice): the two shard
    # streams memorise the training rows more slowly than one stream
    assert abs(a[0] - b[0]) < 0.15 and abs(a[1] - b[1]) < 0.08, (a, b)


LOAD_MODEL_ARGS = ["-task", "r", "-train", "train.libfm", "-test", "test.libfm", "-method", "sgd",
                   "-learn_rate", "0.01", "-seed", "42"]


def test_cli_load_model_roundtrip(c1_files, ref_golden):
    _need()
    base = LOAD_MODEL_ARGS + ["-mode", "inorder"]
    a = _run(CLI, base + ["-iter", "2", "-save_model", "m2.txt"], c1_files)
    assert a.returncode == 0, a.stderr
    # 0 further epochs from the checkpoint: Final must equal the 6-digit-rounded model's metrics, as the
    # reference binary printed them from its own 2-epoch checkpoint (the in-order checkpoints are identical)
    b = _run(CLI, base + ["-iter", "0", "-load_model", "m2.txt"], c1_files)
    assert b.returncode == 0, b.stderr
    assert _iters(b.stdout) == ref_golden["load_model_iters"].tolist()


@pytest.mark.parametrize("task,fmt", [("r", "text"), ("c", "text"), ("r", "binary")])
def test_reference_main_with_b200_learner(c1_files, task, fmt):
    """The maintainer's binding (integration/fm_learn_sgd_b200.h) compiled INTO the reference's own
    main(): its loader, CMDLine, RLog and writers are untouched, only the passes over the data run
    in libfmb200.  In-order mode must reproduce the stock binary's stdout and files."""
    _need_ref()
    train, test = "train.libfm", "test.libfm"
    if fmt == "binary":  # LargeSparseMatrixHD path -> row-cursor upload
        if not os.path.exists(REF_CONVERT):
            pytest.skip("convert not built")
        for stem in ("train", "test"):
            _run(REF_CONVERT, ["--ifile", stem + ".libfm", "--ofilex", stem + ".hd.x", "--ofiley", stem + ".hd.y"], c1_files)
        train, test = "train.hd", "test.hd"
    base = ["-task", task, "-train", train, "-test", test, "-method", "sgd", "-dim", "1,1,8",
            "-iter", "3", "-learn_rate", "0.01", "-init_stdev", "0.1", "-seed", "42"]
    ref = _run(REF_CLI, base + ["-out", "s_pred.txt", "-save_model", "s_model.txt"], c1_files)
    env = dict(os.environ, FMB200_MODE="inorder")
    ours = subprocess.run([REF_CLI_B200] + base + ["-out", "p_pred.txt", "-save_model", "p_model.txt", "-rlog", "p_log.tsv"],
                          capture_output=True, text=True, cwd=c1_files, timeout=600, env=env)
    assert ours.returncode == 0 and "ERROR" not in ours.stderr, ours.stderr
    assert _iters(ours.stdout) == _iters(ref.stdout) and len(_iters(ref.stdout)) == 4
    rd = lambda f: open(os.path.join(c1_files, f)).read()  # noqa: E731
    if task == "r":
        assert rd("p_pred.txt") == rd("s_pred.txt")
        assert rd("p_model.txt") == rd("s_model.txt")
    else:
        np.testing.assert_allclose(np.loadtxt(os.path.join(c1_files, "p_pred.txt")),
                                   np.loadtxt(os.path.join(c1_files, "s_pred.txt")), atol=2e-6)
    assert len(rd("p_log.tsv").splitlines()) == 4
    # hogwild (the default) through the same binding: tracks the reference
    hw = subprocess.run([REF_CLI_B200] + base, capture_output=True, text=True, cwd=c1_files, timeout=600)
    assert hw.returncode == 0 and "ERROR" not in hw.stderr, hw.stderr
    val = lambda l: [float(t.split("=")[1]) for t in l.split("\t") if t.startswith(("Train", "Test"))]  # noqa: E731
    a, b = val(_iters(hw.stdout)[-1]), val(_iters(ref.stdout)[-1])
    assert abs(a[0] - b[0]) < 0.05 and abs(a[1] - b[1]) < 0.05, (a, b)


@pytest.mark.parametrize("method", ["mcmc", "als"])
def test_reference_mcmc_with_b200_eterm_pass(c1_files, method):
    """SURVEY section 8 f3 through the reference's own main(): integration/fm_mcmc_eterms_b200.h swaps the
    two call sites of fm_learn_mcmc::predict_data_and_write_to_eterms (fm_learn_mcmc_simultaneous.h:69,122)
    for fmb200_mcmc_eterms.  The e-terms are bit-identical, the Gibbs draws are the reference's own code with
    the same rand() stream: every #Iter= line and the -out file equal the stock binary's."""
    _need_ref()
    base = ["-task", "r", "-train", "train.libfm", "-test", "test.libfm", "-method", method, "-dim", "1,1,8",
            "-iter", "5", "-init_stdev", "0.1", "-seed", "42"]
    ref = _run(REF_CLI, base + ["-out", "m_ref.txt"], c1_files)
    assert ref.returncode == 0, ref.stderr
    env = dict(os.environ, FMB200_MCMC_ETERMS="1")
    ours = subprocess.run([REF_CLI_B200] + base + ["-out", "m_b200.txt"], capture_output=True, text=True,
                          cwd=c1_files, timeout=600, env=env)
    assert ours.returncode == 0 and "ERROR" not in ours.stderr, ours.stderr
    assert _iters(ours.stdout) == _iters(ref.stdout) and len(_iters(ref.stdout)) >= 5
    rd = lambda f: open(os.path.join(c1_files, f)).read()  # noqa: E731
    assert rd("m_b200.txt") == rd("m_ref.txt")
