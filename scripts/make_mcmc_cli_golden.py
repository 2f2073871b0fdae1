"""Write tests/golden/reference/mcmc_cli.npz: what the stock reference command line (oracle/_ref/libFM,
built by `make -C oracle ref`) prints and writes for the MCMC / ALS runs tests/test_cli_mcmc_gpu.py replays
through bin/libFM -mode inorder.

Per run the file holds the input files, the arguments, the #Iter and #nans lines, the -out file, the -rlog
file and (ALS) the -save_model file.

    python scripts/make_mcmc_cli_golden.py
"""
from __future__ import annotations

import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from libfm_b200 import Data, synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference", "mcmc_cli.npz")
REF = os.path.join(ROOT, "oracle", "_ref", "libFM")


def inputs(tmp: str) -> dict:
    """name -> text of the input files"""
    c1 = synth.plumbing_10k()
    tr, te = synth.split_rows(c1, 8000)
    cls = lambda d: Data(d.row_ptr, d.col, d.val, np.where(d.target >= 4, 1.0, 0.0), d.num_feature)  # noqa: E731
    d = synth.ragged(2400, 300, 11, seed=21)
    rtr, rte = synth.split_rows(d, 2000)
    files = {"c1_train": tr, "c1_test": te, "c1c_train": cls(tr), "c1c_test": cls(te), "rag_train": rtr,
             "rag_test": rte}
    out = {}
    for name, data in files.items():
        path = os.path.join(tmp, name)
        synth.to_libfm_text(data, path)
        out[name] = open(path).read()
    out["rag_meta"] = "".join("%d\n" % (i % 3) for i in range(300))
    return out


# run name -> arguments (file names are resolved in the run directory); no -method = MCMC, the default
RUNS = {
    "mcmc_default_r": "-task r -train c1_train -test c1_test -dim 1,1,8 -iter 7 -seed 42 -out out -rlog rlog",
    "als_r": "-task r -train c1_train -test c1_test -method als -dim 1,1,8 -iter 7 -seed 42 -regular 0.1 "
             "-out out -rlog rlog -save_model model",
    "mcmc_c": "-task c -train c1c_train -test c1c_test -method mcmc -dim 1,1,4 -iter 7 -seed 3 -out out -rlog rlog",
    "als_c": "-task c -train c1c_train -test c1c_test -method als -dim 1,1,4 -iter 7 -seed 3 -regular 0.1,0.2,0.3 "
             "-out out -save_model model",
    "mcmc_meta_r": "-task r -train rag_train -test rag_test -meta rag_meta -dim 1,1,5 -iter 7 -seed 5 -out out "
                   "-rlog rlog",
    "als_meta_r": "-task r -train rag_train -test rag_test -meta rag_meta -method als -dim 1,1,5 -iter 7 -seed 5 "
                  "-regular 0.2,0.3,0.4,0.5,0.6,0.7,0.8 -out out -rlog rlog -save_model model",
}


def read(path: str) -> str:
    return open(path).read() if os.path.exists(path) else ""


def main():
    rec = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, text in inputs(tmp).items():
            rec["input/" + name] = np.array(text)
        for run, args in RUNS.items():
            d = os.path.join(tmp, run)
            os.makedirs(d)
            for name in ("c1_train", "c1_test", "c1c_train", "c1c_test", "rag_train", "rag_test", "rag_meta"):
                open(os.path.join(d, name), "w").write(str(rec["input/" + name]))
            p = subprocess.run([REF] + args.split(), cwd=d, capture_output=True, text=True, check=True)
            lines = [ln for ln in p.stdout.splitlines() if ln.startswith("#Iter") or ln.startswith("#nans")]
            rec[run + "/args"] = np.array(args)
            rec[run + "/lines"] = np.array("\n".join(lines))
            for f in ("out", "rlog", "model"):
                rec[run + "/" + f] = np.array(read(os.path.join(d, f)))
            print(run, lines[-1])
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
