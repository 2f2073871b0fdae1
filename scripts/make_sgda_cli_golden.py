"""Write tests/golden/reference/sgda_cli.npz: the stock reference's `libFM -method sgda` on small data sets.

  python scripts/make_sgda_cli_golden.py      (needs oracle/_ref/libFM, built by __graft_entry__.build())

For every run the archive holds its input files (<run>/<file>), its command line (<run>/args, file names
relative to the run's directory) and what the reference wrote: stdout, -out, -save_model and -rlog
(<run>/stdout, <run>/out, <run>/model, <run>/rlog).  tests/test_sgda_cli_gpu.py runs bin/libFM on the same
files and compares.  Runs:
  reg_wraps     regression, 3 attribute groups (-meta), 600 train / 250 validation rows (the cursor restarts)
  reg_val_long  regression, 300 train / 500 validation rows (no restart: the moments at the epoch's start)
  reg_exact     regression, N = 2 V (the last restart falls on the last step)
  cls           classification, 3 groups, 600 / 250
  load_model    regression starting from a -load_model file (V kept, w zeroed)
  iter1         -iter 1: no lambda-steps
"""
from __future__ import annotations

import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from libfm_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference", "sgda_cli.npz")
N_USERS, N_ITEMS = 40, 30


def _text(d) -> str:
    with tempfile.NamedTemporaryFile("r", suffix=".libfm", delete=False) as f:
        path = f.name
    synth.to_libfm_text(d, path)
    with open(path) as f:
        s = f.read()
    os.remove(path)
    return s


def _model_text(seed: int, n: int, k: int) -> str:
    """a -save_model file: #global bias W, #unary interactions Wj, #pairwise interactions Vj,f"""
    r = np.random.default_rng(seed)
    lines = ["#global bias W0", "%.6g" % r.standard_normal(), "#unary interactions Wj"]
    lines += ["%.6g" % x for x in r.standard_normal(n)]
    lines.append("#pairwise interactions Vj,f")
    lines += [" ".join("%.6g" % x for x in row) for row in r.standard_normal((n, k)) * 0.1]
    return "\n".join(lines) + "\n"


def runs():
    """(name, {file: text}, args) for every run"""
    full = synth.two_field(1300, N_USERS, N_ITEMS, seed=31, planted_k=2)
    tr, rest = synth.split_rows(full, 600)
    va, te = rest.rows(0, 500), rest.rows(500, 700)
    n = N_USERS + N_ITEMS
    meta = "".join("%d\n" % (0 if i < N_USERS else 1 + (i - N_USERS) % 2) for i in range(n))
    files = {"train.libfm": _text(tr), "test.libfm": _text(te), "val.libfm": _text(va.rows(0, 250)),
             "val_long.libfm": _text(va), "train300.libfm": _text(tr.rows(0, 300)),
             "val300.libfm": _text(va.rows(0, 300)), "groups.meta": meta}
    common = "-test test.libfm -dim 1,1,4 -learn_rate 0.02 -init_stdev 0.1 -seed 7 -out out.txt " \
             "-save_model model.txt -rlog rlog.txt"
    out = [
        ("reg_wraps", "-task r -train train.libfm -validation val.libfm -meta groups.meta -iter 4 " + common),
        ("reg_val_long", "-task r -train train300.libfm -validation val_long.libfm -iter 3 " + common),
        ("reg_exact", "-task r -train train.libfm -validation val300.libfm -meta groups.meta -iter 3 " + common),
        ("cls", "-task c -train train.libfm -validation val.libfm -meta groups.meta -iter 4 " + common),
        ("load_model", "-task r -train train.libfm -validation val.libfm -iter 3 -load_model start.txt " + common),
        ("iter1", "-task r -train train.libfm -validation val.libfm -meta groups.meta -iter 1 " + common),
    ]
    files["start.txt"] = _model_text(5, n, 4)
    return files, out


def main() -> None:
    exe = os.path.join(ROOT, "oracle", "_ref", "libFM")
    if not os.path.exists(exe):
        sys.exit("build oracle/_ref/libFM first (__graft_entry__.build())")
    files, rs = runs()
    g = {}
    for name, args in rs:
        with tempfile.TemporaryDirectory() as d:
            for f, text in files.items():
                with open(os.path.join(d, f), "w") as fh:
                    fh.write(text)
            p = subprocess.run([exe, "-method", "sgda"] + args.split(), cwd=d, capture_output=True, text=True,
                               check=True)
            g[name + "/args"] = np.array(args)
            g[name + "/stdout"] = np.array(p.stdout)
            for key, f in (("out", "out.txt"), ("model", "model.txt"), ("rlog", "rlog.txt")):
                with open(os.path.join(d, f)) as fh:
                    g[name + "/" + key] = np.array(fh.read())
    for f, text in files.items():
        g["files/" + f] = np.array(text)
    np.savez_compressed(OUT, **g)
    print("wrote", OUT, "(%d runs)" % len(rs))


if __name__ == "__main__":
    main()
