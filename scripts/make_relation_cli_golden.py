"""Write tests/golden/reference/mcmc_relation_cli.npz: what the stock reference command line (oracle/_ref/libFM,
built by `make -C oracle ref`) prints and writes for the -relation runs tests/test_cli_relation_gpu.py replays
through bin/libFM -mode inorder and ordered.

The data are cases of make_relation_golden.py, written as files: the main tables as libfm text, each block as
<stem>.xt, <stem>.train, <stem>.test and an optional <stem>.groups (write_block_files).  Per run the file holds the
input files (text, or bytes for the .xt and binary joins), the arguments, the #Iter and #nans lines, the -out file,
the -rlog file and, for ALS, the -save_model file.

    python scripts/make_relation_cli_golden.py
"""
from __future__ import annotations

import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from libfm_b200 import synth  # noqa: E402
from libfm_b200.model import write_binary  # noqa: E402
from make_relation_golden import cases, write_block_files  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference", "mcmc_relation_cli.npz")
REF = os.path.join(ROOT, "oracle", "_ref", "libFM")

# data set name -> the make_relation_golden case it comes from
DATA = {"ui": "user_item_mcmc", "cls": "cls_mcmc", "meta": "main_meta_als"}

# run name -> (data set, arguments; file names are resolved in the run directory).  ui's user block has binary joins,
# its item block text joins and a .groups file (1 + 1 + 2 groups); meta's main table has features and -meta groups
RUNS = {
    "mcmc_user_item_r": ("ui", "-task r -train train -test test -relation ui_rel0,ui_rel1 -dim 1,1,5 -iter 6 "
                               "-seed 42 -out out -rlog rlog"),
    "als_groups_r": ("ui", "-task r -train train -test test -relation ui_rel0,ui_rel1 -method als -dim 1,1,5 "
                           "-iter 6 -seed 42 -regular 0.1,0.2,0.3,0.4,0.5,0.6,0.7,0.8,0.9 -out out -rlog rlog "
                           "-save_model model"),
    "als_load_r": ("ui", "-task r -train train -test test -relation ui_rel0,ui_rel1 -method als -dim 1,1,5 "
                         "-iter 3 -seed 43 -regular 0.1 -load_model als_groups_r.model -out out -save_model model"),
    "mcmc_c": ("cls", "-task c -train train -test test -relation cls_rel0 -method mcmc -dim 1,1,4 -iter 6 -seed 7 "
                      "-out out -rlog rlog"),
    "mcmc_meta_r": ("meta", "-task r -train train -test test -meta meta -relation meta_rel0 -dim 1,1,4 -iter 6 "
                            "-seed 11 -out out -rlog rlog"),
}


def read(path: str) -> str:
    return open(path).read() if os.path.exists(path) else ""


def inputs(tmp: str) -> dict:
    """data set name -> {file name: bytes} of every file its runs read"""
    allc = cases()
    out = {}
    for ds, name in DATA.items():
        c = allc[name]
        d = os.path.join(tmp, ds)
        os.makedirs(d)
        synth.to_libfm_text(c["train"], os.path.join(d, "train"))
        synth.to_libfm_text(c["test"], os.path.join(d, "test"))
        if c["meta"] is not None:
            with open(os.path.join(d, "meta"), "w") as f:
                f.write("\n".join(str(int(x)) for x in c["meta"]) + "\n")
        for i, b in enumerate(c["blocks"]):
            write_block_files(os.path.join(d, f"{ds}_rel{i}"), b, c["train"].num_cases, c["test"].num_cases)
        out[ds] = {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}
    return out


def write_inputs(files: dict, d: str) -> None:
    for f, data in files.items():
        with open(os.path.join(d, f), "wb") as fh:
            fh.write(data)


def main():
    rec = {}
    with tempfile.TemporaryDirectory() as tmp:
        data = inputs(tmp)
        allc = cases()
        for ds, files in data.items():
            for f, b in files.items():
                rec[f"input/{ds}/{f}"] = np.frombuffer(b, np.uint8)
        for run, (ds, args) in RUNS.items():
            d = os.path.join(tmp, "run_" + run)
            os.makedirs(d)
            write_inputs(data[ds], d)
            # the reference's ALS also reads each block's .x (has_x, libfm.cpp:186-190); bin/libFM does not
            for i, b in enumerate(allc[DATA[ds]]["blocks"]):
                write_binary(b["data"], os.path.join(d, f"{ds}_rel{i}.x"), os.path.join(d, f"{ds}_rel{i}.xy"))
            if "-load_model" in args:
                with open(os.path.join(d, "als_groups_r.model"), "w") as f:
                    f.write(str(rec["als_groups_r/model"]))
            p = subprocess.run([REF] + args.split(), cwd=d, capture_output=True, text=True, check=True)
            lines = [ln for ln in p.stdout.splitlines() if ln.startswith("#Iter") or ln.startswith("#nans")]
            rec[run + "/data"] = np.array(ds)
            rec[run + "/args"] = np.array(args)
            rec[run + "/lines"] = np.array("\n".join(lines))
            for f in ("out", "rlog", "model"):
                rec[run + "/" + f] = np.array(read(os.path.join(d, f)))
            print(run, lines[-1])
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
