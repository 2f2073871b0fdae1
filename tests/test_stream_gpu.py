"""GPU: -cache_size streaming -- the device decode of .x blocks (fmb200_upload_xblock, fm_upload.cu) and the
command line's streamed SGD passes (host/fm_host.h GpuSgdLearner::pass) against the resident runs and the stock
reference's stored output."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, make_learner
from libfm_b200 import MODE_INORDER, FmError
from libfm_b200.model import pinned_copy, read_xblocks, write_binary
from test_cli_gpu import HOGWILD_ARGS, INORDER_CASES, _file_digest, _iters, inorder_args, write_c1_files
from test_stream_cpu import ragged_with_long_row

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "bin", "libFM")
CONVERT = os.path.join(ROOT, "bin", "convert")


def _learner(n, k=4):
    cfg = dict(n=n, k=k, k0=1, k1=1, task=0, lr=0.01, regs=np.zeros(3), min_target=1.0, max_target=5.0)
    r = np.random.default_rng(0)
    return make_learner(cfg, (0.1, r.standard_normal(n) * 0.1, r.standard_normal((k, n)) * 0.1), mode=MODE_INORDER)


def _same(a, b):
    assert np.array_equal(a.row_ptr, b.row_ptr)
    assert np.array_equal(a.col, b.col)
    assert np.array_equal(a.val.view(np.uint32), b.val.view(np.uint32))
    assert np.array_equal(a.target.view(np.uint32), b.target.view(np.uint32))


@pytest.fixture(scope="module")
def ragged_x(tmp_path_factory):
    d = ragged_with_long_row()
    stem = str(tmp_path_factory.mktemp("xb") / "d")
    write_binary(d, stem + ".x", stem + ".y")
    return d, stem + ".x"


@pytest.mark.parametrize("cache_size", [80_008, 100_001])
def test_xblock_decode_equals_resident_rows(ragged_x, cache_size, built_lib):
    d, path = ragged_x
    l = _learner(d.num_feature)
    l.upload(d, 1)
    whole = l.download(1)
    blocks = list(read_xblocks(path, cache_size))
    assert len(blocks) >= 3 and (cache_size > 80_008 or (1234, 1235) in [(lo, hi) for lo, hi, _, _ in blocks])
    assert any(np.any(s == 0) for _, _, _, s in blocks)
    for lo, hi, words, sizes in blocks:
        want = whole.rows(lo, hi)
        l.upload_xblock(words, sizes, d.target[lo:hi], 2)
        _same(l.download(2), want)
        w, s, t = pinned_copy(words), pinned_copy(sizes), pinned_copy(d.target[lo:hi])
        l.upload_xblock(w, s, t, 3, asynchronous=True)
        _same(l.download(3), want)  # the next call on the slot waits for the upload
    l.close()


def test_xblock_refuses_a_bad_header_and_a_bad_id(ragged_x, built_lib):
    d, path = ragged_x
    lo, hi, words, sizes = next(b for b in read_xblocks(path, 100_001) if b[1] - b[0] > 3)
    bad = words.copy()
    head2 = 2 + 2 * int(sizes[:2].sum())  # row 2's header word
    bad[head2] += 1
    l = _learner(d.num_feature)
    with pytest.raises(FmError, match="row 2 of the .x block"):
        l.upload_xblock(bad, sizes, d.target[lo:hi], 2)
    l.upload_xblock(bad, sizes, d.target[lo:hi], 3, asynchronous=True)
    with pytest.raises(FmError, match="row 2 of the .x block"):
        l.download(3)
    l.close()
    small = _learner(10)  # ids up to 399 >= num_attribute 10
    with pytest.raises(FmError, match="out of range"):
        small.upload_xblock(words, sizes, d.target[lo:hi], 2)
    small.close()


# ---- the command line ---------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def c1_bin(tmp_path_factory, ref_golden):
    if not os.path.exists(CLI):
        pytest.skip("CLI binaries not built")
    d = tmp_path_factory.mktemp("c1s")
    write_c1_files(str(d))
    for stem in ("train", "test"):
        subprocess.run([CONVERT, "--ifile", stem + ".libfm", "--ofilex", stem + ".bin.x", "--ofiley", stem + ".bin.y"],
                       cwd=d, capture_output=True, check=True)
    # train in at least 5 blocks, test (a fifth of its size) in at least 2
    x_bytes = os.path.getsize(str(d / "train.bin.x")) - 24
    return d, 2 * (x_bytes // 6)


def _bin(args):
    return [{"train.libfm": "train.bin", "test.libfm": "test.bin"}.get(a, a) for a in args]


def _run(args, cwd):
    r = subprocess.run([CLI] + args, capture_output=True, text=True, cwd=cwd, timeout=600)
    assert r.returncode == 0, r.stderr
    return r


def _plan(stdout):
    return [int(l.split(": ")[1].split()[0]) for l in stdout.splitlines() if l.startswith("streaming ")]


@pytest.mark.parametrize("task,extra", INORDER_CASES)
def test_streamed_inorder_equals_reference_cli(c1_bin, task, extra, ref_golden):
    d, cache = c1_bin
    i = INORDER_CASES.index((task, extra))
    g = lambda key: ref_golden["inorder%d_%s" % (i, key)]  # noqa: E731
    ours = _run(_bin(inorder_args(task, extra)) + ["-mode", "inorder", "-cache_size", str(cache), "-out", "s_pred.txt",
                                                   "-save_model", "s_model.txt", "-rlog", "s_log.tsv"], d)
    n_train, n_test = _plan(ours.stdout)
    assert n_train >= 5 and n_test >= 2
    assert _iters(ours.stdout) == g("iters").tolist() and len(g("iters")) == 4
    if task == "r":
        assert _file_digest(os.path.join(d, "s_pred.txt")) == g("pred_sha")
        assert _file_digest(os.path.join(d, "s_model.txt")) == g("model_sha")
    else:
        np.testing.assert_allclose(np.loadtxt(os.path.join(d, "s_pred.txt")), g("pred"), atol=2e-6)
    lo, lr = open(os.path.join(d, "s_log.tsv")).read().splitlines(), g("log").tolist()
    assert lo[0] == lr[0] and len(lo) == len(lr) == 4
    hdr = lo[0].split("\t")
    for a, b in zip(lo[1:], lr[1:]):
        for name, x, y in zip(hdr, a.split("\t"), b.split("\t")):
            if not name.startswith("time"):
                assert x == y, (name, x, y)


def _values(stdout):
    return [float(t.split("=")[1]) for l in _iters(stdout) for t in l.split("\t") if t.startswith(("Train", "Test"))]


def test_streamed_ordered_tracks_resident_ordered(c1_bin):
    d, cache = c1_bin
    args = _bin(inorder_args("r", [])) + ["-mode", "ordered"]
    res = _run(args, d)
    st = _run(args + ["-cache_size", str(cache)], d)
    assert len(_plan(st.stdout)) == 2
    a, b = _values(res.stdout), _values(st.stdout)
    assert len(a) == len(b) == 8
    assert max(abs(x - y) for x, y in zip(a, b)) < 1e-9, (a, b)


def test_streamed_hogwild_is_reproducible_and_tracks_reference(c1_bin, ref_golden):
    d, cache = c1_bin
    args = _bin(HOGWILD_ARGS) + ["-cache_size", str(cache)]
    runs = []
    for rep in range(2):
        r = _run(args + ["-out", "h%d_pred.txt" % rep, "-save_model", "h%d_model.txt" % rep], d)
        runs.append(r.stdout.replace("h%d_" % rep, "h_"))
    assert len(_plan(runs[0])) == 2
    assert runs[0] == runs[1]
    for f in ("pred", "model"):
        assert open(os.path.join(d, "h0_%s.txt" % f)).read() == open(os.path.join(d, "h1_%s.txt" % f)).read()
    val = lambda l: [float(t.split("=")[1]) for t in l.split("\t") if t.startswith(("Train", "Test"))]  # noqa: E731
    a, b = val(_iters(runs[0])[-1]), val(str(ref_golden["hogwild_iters"][-1]))
    assert abs(a[0] - b[0]) < 0.05 and abs(a[1] - b[1]) < 0.05, (a, b)


@pytest.mark.parametrize("mode", ["inorder", "hogwild"])
def test_budget_larger_than_the_file_changes_nothing(c1_bin, mode):
    d, _ = c1_bin
    args = _bin(inorder_args("r", [])) + ["-mode", mode]
    a = _run(args + ["-out", "a_pred.txt", "-save_model", "a_model.txt"], d)
    b = _run(args + ["-cache_size", str(1 << 34), "-out", "b_pred.txt", "-save_model", "b_model.txt"], d)
    assert a.stdout.replace("a_model", "b_model") == b.stdout and "streaming" not in b.stdout
    for f in ("pred", "model"):
        assert open(os.path.join(d, "a_%s.txt" % f)).read() == open(os.path.join(d, "b_%s.txt" % f)).read()
