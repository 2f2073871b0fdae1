"""Generate tests/golden/reference/outputs.npz: what the REFERENCE itself computes for the
inputs of the tests that compare against it (oracle/_ref, built by `make -C oracle ref` from
a checkout of the reference):

    python scripts/make_ref_golden.py

The tests rebuild the same seeded inputs and compare the project's result with the values
stored here, so they run without the reference.  Large results are stored as SHA-256
digests of their bytes (see tests/conftest.py::digest); so are the generated input files,
which lets a test tell a changed generator apart from a changed result.
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from conftest import digest  # noqa: E402
from libfm_b200 import synth  # noqa: E402
from oracle import Port, Ref  # noqa: E402
from oracle.binding import REF_CLI, REF_CONVERT  # noqa: E402
import test_cli_gpu as tcli  # noqa: E402
import test_host_cpu as thost  # noqa: E402
import test_oracle as tor  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference", "outputs.npz")


def file_digest(path):
    return digest(np.frombuffer(open(path, "rb").read(), np.uint8))


def csr_digest(csr):
    rp, col, val, tgt = csr[:4]
    return digest(rp) + digest(col) + digest(val) + digest(tgt)


def blank_time_columns(lines):
    """rlog lines with the time_* columns emptied: they differ on every run, the tests ignore them."""
    hdr = lines[0].split("\t")
    out = [lines[0]]
    for line in lines[1:]:
        out.append("\t".join("" if h.startswith("time") else x for h, x in zip(hdr, line.split("\t"))))
    return out


def oracle_outputs(g):
    tr = synth.plumbing_10k()
    te = synth.plumbing_10k(seed=99, n_rows=2000)
    n, k = max(tr.num_feature, te.num_feature), 8
    ref = Ref(n, k, seed=42, init_stdev=0.1)
    ref.learn(tr, te, 0, 0.01, 2, tr.min_target, tr.max_target)
    w0, w, v = ref.get_params()
    g["c1_w0"], g["c1_wv_sha"] = w0, digest(w) + digest(v)
    g["c1_test_metric"] = ref.evaluate(te, 0, tr.min_target, tr.max_target)

    L = Ref.lib()
    L.ref_srand(C.c_long(123))
    g["rng_gauss_123"] = np.array([L.ref_ran_gaussian() for _ in range(1000)])

    ref = Ref(20, 3, seed=5)
    _, _, v = ref.get_params()
    ref.set_params(0.25, np.linspace(-1, 1, 20), v)
    g["row_v"] = v
    out = [ref.predict_row(col, val) for col, val in tor.PREDICT_ROW_CASES]
    g["row_p"] = np.array([o[0] for o in out])
    g["row_s"] = np.array([o[1] for o in out])
    g["row_ss"] = np.array([o[2] for o in out])

    for case in tor.MCMC_CASES:
        d, n, k, k0, k1, w0, w = tor.mcmc_case(case)
        ref = Ref(n, k, k0, k1, seed=42, init_stdev=0.1)
        _, _, v = ref.get_params()
        p = Port(n, k, k0, k1)
        p.init(42, 0.0, 0.1)
        assert np.array_equal(p.v, v)  # the test draws V with the port
        ref.set_params(w0, w, v)
        g["mcmc_%s_sha" % case] = digest(ref.mcmc_eterms(d))

    for task in (0, 1):
        tr, va, te, group, n, k, mn, mx = tor.sgda_case(task)
        ref = Ref(n, k, seed=42, init_stdev=0.1)
        w0, w, v = ref.get_params()
        p = Port(n, k)
        p.init(42, 0.0, 0.1)
        assert p.w0.value == w0 and np.array_equal(p.w, w) and np.array_equal(p.v, v)
        reg_w, reg_v = ref.sgda_learn(tr, va, te, group, task, 0.02, 4, mn, mx)
        a0, aw, av = ref.get_params()
        g["sgda%d_w0" % task], g["sgda%d_wv_sha" % task] = a0, digest(aw) + digest(av)
        g["sgda%d_reg_w" % task], g["sgda%d_reg_v" % task] = reg_w, reg_v


def host_outputs(g, tmp):
    tricky = os.path.join(tmp, "tricky.libfm")
    open(tricky, "w").write(thost.TRICKY)
    rp, col, val, tgt, nf, mn, mx = Ref.load_data(tricky)
    g["tricky_row_ptr"], g["tricky_col"], g["tricky_val"], g["tricky_target"] = rp, col, val, tgt
    g["tricky_meta"] = np.array([nf, mn, mx], dtype=np.float64)

    ref = Ref(37, 5, seed=42, init_stdev=0.1)
    g["init37_w0"], g["init37_w"], g["init37_v"] = ref.get_params()

    fm = thost.checkpoint_model()
    path = os.path.join(tmp, "m.txt")
    fm.saveModel(path)
    ref = Ref(12, 3, seed=1)
    assert ref.load_model(path) == 1
    g["ckpt_w0"], g["ckpt_w"], g["ckpt_v"] = ref.get_params()
    ref.save_model(os.path.join(tmp, "ref.txt"))
    g["ckpt_text"] = np.array(open(os.path.join(tmp, "ref.txt")).read())

    r = subprocess.run([REF_CLI] + thost.cli_loader_args(tricky), capture_output=True, text=True)
    g["cli_loader_lines"] = np.array(thost.loader_lines(r.stdout))

    big = os.path.join(tmp, "big.libfm")
    thost.write_threaded_input(big)
    g["threaded_input_sha"] = file_digest(big)
    want = Ref.load_data(big)
    g["threaded_csr_sha"] = csr_digest(want)
    g["threaded_meta"] = np.array(want[4:], dtype=np.float64)

    big = os.path.join(tmp, "convert_big.libfm")
    thost.write_convert_input(big)
    g["convert_big_input_sha"] = file_digest(big)
    for tag, src in (("tricky", tricky), ("big", big)):
        subprocess.run([REF_CONVERT, "--ifile", src, "--ofilex", os.path.join(tmp, "b.x"), "--ofiley",
                        os.path.join(tmp, "b.y")], capture_output=True, check=True)
        g["convert_%s_sha" % tag] = file_digest(os.path.join(tmp, "b.x")) + file_digest(os.path.join(tmp, "b.y"))

    fz_in, fz_err, fz_csr, fz_meta = [], [], [], []
    for trial, text in enumerate(thost.fuzz_inputs()):
        path = os.path.join(tmp, "f%d.libfm" % trial)
        open(path, "w").write(text)
        fz_in.append(file_digest(path))
        try:
            want = Ref.load_data(path)
        except RuntimeError as e:
            fz_err.append(str(e).strip())
            fz_csr.append("")
            fz_meta.append([0.0, 0.0, 0.0])
            continue
        fz_err.append("")
        fz_csr.append(csr_digest(want))
        fz_meta.append(list(want[4:]))
    g["fuzz_input_sha"], g["fuzz_error"] = np.array(fz_in), np.array(fz_err)
    g["fuzz_csr_sha"], g["fuzz_meta"] = np.array(fz_csr), np.array(fz_meta, dtype=np.float64)


def cli_outputs(g, tmp):
    tcli.write_c1_files(tmp)
    g["c1_train_sha"] = file_digest(os.path.join(tmp, "train.libfm"))
    g["c1_test_sha"] = file_digest(os.path.join(tmp, "test.libfm"))
    run = lambda args: subprocess.run([REF_CLI] + args, capture_output=True, text=True, cwd=tmp, check=True)  # noqa: E731
    rd = lambda f: os.path.join(tmp, f)  # noqa: E731
    for i, (task, extra) in enumerate(tcli.INORDER_CASES):
        r = run(tcli.inorder_args(task, extra) + ["-out", "pred.txt", "-save_model", "model.txt", "-rlog", "log.tsv"])
        g["inorder%d_iters" % i] = np.array(tcli._iters(r.stdout))
        g["inorder%d_pred_sha" % i] = file_digest(rd("pred.txt"))
        g["inorder%d_pred" % i] = np.loadtxt(rd("pred.txt"))
        g["inorder%d_model_sha" % i] = file_digest(rd("model.txt"))
        g["inorder%d_log" % i] = np.array(blank_time_columns(open(rd("log.tsv")).read().splitlines()))
    g["hogwild_iters"] = np.array(tcli._iters(run(tcli.HOGWILD_ARGS).stdout))
    g["two_gpu_iters"] = np.array(tcli._iters(run(tcli.TWO_GPU_ARGS).stdout))
    run(tcli.LOAD_MODEL_ARGS + ["-iter", "2", "-save_model", "m2.txt"])
    g["load_model_iters"] = np.array(tcli._iters(run(tcli.LOAD_MODEL_ARGS + ["-iter", "0", "-load_model", "m2.txt"]).stdout))


def main():
    g = {}
    oracle_outputs(g)
    with tempfile.TemporaryDirectory() as tmp:
        host_outputs(g, tmp)
    with tempfile.TemporaryDirectory() as tmp:
        cli_outputs(g, tmp)
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT), "bytes,", len(g), "entries")


if __name__ == "__main__":
    main()
