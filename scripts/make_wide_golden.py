"""Write tests/golden/reference/wide_k.npz: what the reference itself computes at the factor widths k in
tests/test_wide_k.py::WIDE_K_REF (33 .. 256), on that module's seeded data sets.

Through the reference shim (oracle/_ref/libfm_ref.so, `make -C oracle ref`), per k:
  sgd/<k>/<task>/   2 epochs of fm_learn_sgd_element::learn, regression (regularised) and classification: the
                    per-epoch train / test metrics, w0, digests of w and v, the digest of predict() on the test set
  sgda/<k>/         3 epochs of fm_learn_sgd_element_adapt_reg::learn over 3 attribute groups: w0, digests of w and
                    v, reg_w, the digest of reg_v
  eterm/<k>         the digest of the MCMC e-term pass over the training set
and through scripts/mcmc_ref_probe.cpp (as scripts/make_mcmc_golden.py), the cases k<k>_mcmc and k<k>_als: the
same per-iteration record as tests/golden/reference/mcmc.npz for 4 iterations, without the inputs (they are
regenerated from their seeds; inputs/<set> holds the digests of every generated input).

    python scripts/make_wide_golden.py [--ref /root/reference]

The archive is written with fixed entry timestamps, so a rerun reproduces it byte for byte.
"""
from __future__ import annotations

import argparse
import io
import os
import sys
import tempfile
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from conftest import digest  # noqa: E402
from oracle import Ref  # noqa: E402
import make_mcmc_golden as mg  # noqa: E402
import test_wide_k as tw  # noqa: E402

OUT = tw.GOLDEN


def sgd_records(rec):
    for k in tw.WIDE_K_REF:
        for task in (0, 1):
            tr, _, te = tw.sgd_sets(task)
            n, mn, mx = tr.num_feature, float(tr.target.min()), float(tr.target.max())
            ref = Ref(n, k, seed=42, init_stdev=0.1)
            if task == 0:
                ref.set_reg(*tw.SGD_REGS)
            m_tr, m_te, _ = ref.learn(tr, te, task, tw.SGD_LR, tw.SGD_EPOCHS, mn, mx)
            w0, w, v = ref.get_params()
            key = "sgd/%d/%d/" % (k, task)
            rec[key + "metric_train"], rec[key + "metric_test"] = m_tr, m_te
            rec[key + "w0"], rec[key + "wv"] = np.float64(w0), np.array(digest(w) + digest(v))
            rec[key + "pred"] = np.array(digest(ref.predict(te, task, mn, mx)))
        tr, va, te = tw.sgd_sets(0)
        n, mn, mx = tr.num_feature, float(tr.target.min()), float(tr.target.max())
        ref = Ref(n, k, seed=42, init_stdev=0.1)
        reg_w, reg_v = ref.sgda_learn(tr, va, te, tw.sgda_groups(n), 0, tw.SGDA_LR, tw.SGDA_EPOCHS, mn, mx)
        w0, w, v = ref.get_params()
        key = "sgda/%d/" % k
        rec[key + "w0"], rec[key + "wv"] = np.float64(w0), np.array(digest(w) + digest(v))
        rec[key + "reg_w"], rec[key + "reg_v"] = reg_w, np.array(digest(reg_v))
        ref = Ref(n, k, seed=42, init_stdev=0.1)
        _, _, v = ref.get_params()
        ref.set_params(tw.ETERM_W0, tw.eterm_w(n), v)
        rec["eterm/%d" % k] = np.array(digest(ref.mcmc_eterms(tr)))
        print("k=%d: sgd, sgda, e-terms" % k)


def mcmc_records(rec, ref_dir):
    tr, te = tw.mcmc_sets()
    with tempfile.TemporaryDirectory() as tmp:
        lib = mg.build_probe(ref_dir, tmp)
        for name, c in tw.mcmc_cases().items():
            c = dict(c, train=tr, test=te, n=tr.num_feature, k0=1, k1=1, task=0, multilevel=c["sample"])
            n, k = c["n"], c["k"]
            rec[f"{name}/cfg"] = np.array([n, k, 1, 1, 0, c["sample"], c["multilevel"], c["seed"], tr.num_feature,
                                           te.num_feature], np.int64)
            rec[f"{name}/reg0"] = np.float64(c["reg0"])
            rec[f"{name}/minmax"] = np.array([tr.min_target, tr.max_target])
            for t in range(tw.MCMC_ITERS):
                init, state, hyper, cnt, pred, lines = mg.run(lib, c, t + 1)
                if t == 0:
                    rec[f"{name}/init_digest"] = np.array(tw.fp64_digest(init))
                rec[f"{name}/{t}/w0"] = np.float64(state[0])
                rec[f"{name}/{t}/w"] = np.array(tw.fp64_digest(state[1:1 + n]))
                rec[f"{name}/{t}/v"] = np.array(tw.fp64_digest(state[1 + n:]))   # factor-major [k][n]
                rec[f"{name}/{t}/hyper"] = hyper
                rec[f"{name}/{t}/counters"] = cnt
                for i, p in enumerate(("pred_this", "pred_sum_all", "pred_sum_all_but5")):
                    rec[f"{name}/{t}/{p}"] = np.array(tw.fp64_digest(pred[i]))
                rec[f"{name}/{t}/line"] = np.array(lines[-1])
            print(name, lines[-1])


def save(path, rec):
    """np.savez_compressed with fixed timestamps and entry order"""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for key in sorted(rec):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(rec[key]), allow_pickle=False)
            info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    args = ap.parse_args()
    rec = {"inputs/" + key: np.array(d) for key, d in tw.input_digests().items()}
    sgd_records(rec)
    mcmc_records(rec, args.ref)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    save(OUT, rec)
    print("wrote", OUT, os.path.getsize(OUT), "bytes,", len(rec), "entries")


if __name__ == "__main__":
    main()
