"""Write tests/golden/cli_transcripts.json: what a bin/libFM prints, writes and returns for a fixed matrix of
command lines (the SGD, MCMC and ALS flows, their files, refusals and flag errors).  tests/test_cli_transcripts.py
replays the matrix and compares.

    python scripts/make_cli_transcripts.py CLI [--out PATH]

Run it on an H100 with the CLI the golden should describe.  Per run the record holds the arguments, stdout,
stderr, the exit code and every file the run wrote.  Parts that are not reproducible are masked: the `time:`
line of -verbosity 1, the time_* columns of -rlog files, and Train=/Test= of HOGWILD runs whose shape does
not take the reproducible row-lane epoch (k <= 8, rows of at most 4 entries).
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile
from typing import NamedTuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from libfm_b200 import Data, FmModel, synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "cli_transcripts.json")
MCMC_CLI = os.path.join(ROOT, "tests", "golden", "reference", "mcmc_cli.npz")
FILE_TEXT_MAX = 4096  # larger files are recorded as SHA-256 and size


class Run(NamedTuple):
    args: str
    device: bool = True         # reaches the GPU (without one the CLI stops with "no CPU path")
    mask_metrics: bool = False  # HOGWILD off the row-lane epoch: Train=/Test= vary from run to run
    rowlane: bool = False       # HOGWILD on the row-lane epoch: reproducible on a device with the same SM count


C1 = "-train train.libfm -test test.libfm -seed 42"
C1C = "-train c1c_train -test c1c_test -seed 3"
MC = "-train c1_train -test c1_test -seed 42"
RAG = "-train rag_train -test rag_test -seed 5"

RUNS = {
    # SGD
    "sgd_inorder_r": Run(C1 + " -task r -method sgd -mode inorder -iter 2 -learn_rate 0.01 -regular 0,0,0.01 "
                         "-rlog rlog -out out -save_model model"),
    "sgd_ordered_c": Run(C1C + " -task c -method sgd -mode ordered -dim 1,1,4 -iter 2 -regular 0.01 "
                         "-learn_rate 0.01,0.02,0.03 -rlog rlog -out out"),
    "sgd_inorder_c": Run(C1C + " -task c -method sgd -mode inorder -dim 1,1,4 -iter 2 -learn_rate 0.01 -out out"),
    "sgd_hogwild_rowlane": Run(C1 + " -task r -method sgd -iter 3 -learn_rate 0.01 -verbosity 1 "
                               "-validation test.libfm -rlog rlog -out out", rowlane=True),
    "sgd_hogwild_tiles": Run(C1 + " -task r -method sgd -mode hogwild -dim 1,1,16 -iter 2 -learn_rate 0.01 "
                             "-regular 0.01", mask_metrics=True),
    "sgd_load_model": Run(RAG + " -task r -method sgd -mode inorder -dim 1,1,4 -iter 1 -learn_rate 0.01 "
                          "-load_model good_model -save_model model"),
    "sgd_load_malformed": Run(RAG + " -task r -method sgd -mode inorder -dim 1,1,4 -iter 1 -learn_rate 0.01 "
                              "-load_model bad_model -out out"),
    "sgd_out_unopenable": Run(RAG + " -task r -method sgd -mode inorder -iter 1 -learn_rate 0.01 -out nodir/out"),
    "sgd_regular_two": Run(RAG + " -task r -method sgd -mode inorder -iter 1 -learn_rate 0.01 -regular 0.1,0.2"),
    "sgd_learn_rate_two": Run(RAG + " -task r -method sgd -mode inorder -iter 1 -learn_rate 0.1,0.2"),
    # MCMC and ALS
    "mcmc_default": Run(MC + " -task r -dim 1,1,4 -iter 3 -mode inorder -rlog rlog -out out"),
    "mcmc_c": Run(C1C + " -task c -method mcmc -dim 1,1,2 -iter 3 -mode inorder -rlog rlog -out out"),
    "mcmc_meta": Run(RAG + " -task r -meta rag_meta -dim 1,1,3 -iter 3 -mode inorder -rlog rlog -out out"),
    "als_meta_groups": Run(RAG + " -task r -method als -meta rag_meta -dim 1,1,3 -iter 3 -mode ordered "
                           "-regular 0.2,0.3,0.4,0.5,0.6,0.7,0.8 -rlog rlog -out out -save_model model"),
    "als_regular3": Run(MC + " -task r -method als -dim 1,1,4 -iter 3 -mode inorder -regular 0.1,0.2,0.3 "
                        "-verbosity 1 -save_model model"),
    "als_load_model": Run(RAG + " -task r -method als -dim 1,1,4 -iter 2 -mode inorder -load_model good_model "
                          "-save_model model"),
    "als_load_malformed": Run(RAG + " -task r -method als -dim 1,1,4 -iter 2 -mode inorder -load_model bad_model "
                              "-out out"),
    "als_regular_two": Run(RAG + " -task r -method als -iter 1 -mode inorder -regular 0.1,0.2"),
    "mcmc_save_model_warning": Run(MC + " -task r -iter 1 -mode inorder -save_model model", device=False),
    "mcmc_load_model_warning": Run(MC + " -task r -method mcmc -iter 1 -mode inorder -load_model good_model",
                                   device=False),
    # refusals and errors
    "sgda": Run(C1 + " -task r -method sgda -iter 1", device=False),
    "method_foo": Run(C1 + " -task r -method foo", device=False),
    "sgd_relation": Run(C1 + " -task r -method sgd -relation rel", device=False),
    "mcmc_relation": Run(MC + " -task r -method mcmc -mode inorder -relation rel", device=False),
    "mcmc_gpus_2": Run(MC + " -task r -method mcmc -mode inorder -gpus 2", device=False),
    "sgd_gpus_0": Run(C1 + " -task r -method sgd -mode inorder -gpus 0", device=False),
    "sgd_gpus_2_inorder": Run(C1 + " -task r -method sgd -mode inorder -gpus 2 -learn_rate 0.01", device=False),
    "sgd_mode_foo": Run(C1 + " -task r -method sgd -mode foo", device=False),
    "mcmc_mode_foo": Run(MC + " -task r -mode foo", device=False),
    "als_mode_default": Run(MC + " -task r -method als", device=False),
    "sgd_dim_two": Run(C1 + " -task r -method sgd -mode inorder -dim 1,8", device=False),
    "mcmc_dim_two": Run(MC + " -task r -mode inorder -dim 1,8", device=False),
    "sgd_task_unknown": Run(C1 + " -task x -method sgd -mode inorder", device=False),
    "sgd_rlog_unopenable": Run(C1 + " -task r -method sgd -mode inorder -rlog nodir/rlog", device=False),
    "mcmc_rlog_unopenable": Run(MC + " -task r -mode inorder -rlog nodir/rlog", device=False),
    "mcmc_meta_unopenable": Run(RAG + " -task r -mode inorder -meta nodir/meta", device=False),
    "flag_unknown": Run("-task r -bogus 1", device=False),
    "flag_repeated": Run("-task r -task c", device=False),
    "help": Run("-help", device=False),
    "no_arguments": Run("", device=False),
}


def write_inputs(d: str) -> None:
    """The C1 files of tests/test_cli_gpu.py (write_c1_files), the inputs of tests/golden/reference/mcmc_cli.npz
    (with a -meta file) and two model files for the ragged set: one it loads, one that is malformed."""
    synth.to_libfm_text(synth.plumbing_10k(), os.path.join(d, "train.libfm"))
    synth.to_libfm_text(synth.plumbing_10k(seed=99, n_rows=2000), os.path.join(d, "test.libfm"))
    z = np.load(MCMC_CLI)
    for key in z.files:
        if key.startswith("input/"):
            with open(os.path.join(d, key[len("input/"):]), "w") as f:
                f.write(str(z[key]))
    n = max(Data.load(os.path.join(d, "rag_train")).num_feature, Data.load(os.path.join(d, "rag_test")).num_feature)
    fm = FmModel(n, 4)
    fm.init_stdev = 0.1
    fm.init(seed=11)
    fm.saveModel(os.path.join(d, "good_model"))
    with open(os.path.join(d, "bad_model"), "w") as f:
        f.write("#global bias W0\n0.5\n#unary interactions Wj\n0.25\n")


def mask_text(text: str, metrics: bool) -> str:
    text = re.sub(r"(?m)^time: .*$", "time: <masked>", text)
    if metrics:
        text = re.sub(r"(Train|Test)=[^\t\n]*", r"\1=<masked>", text)
    return text


def mask_rlog(text: str) -> str:
    head, *rows = [line.split("\t") for line in text.split("\n")]
    timed = {i for i, h in enumerate(head) if h.startswith("time_")}
    rows = [["<masked>" if i in timed else x for i, x in enumerate(r)] if len(r) == len(head) else r for r in rows]
    return "\n".join("\t".join(r) for r in [head] + rows)


def file_record(name: str, data: bytes):
    text = data.decode()
    if name == "rlog":
        text = mask_rlog(text)
    if len(text) <= FILE_TEXT_MAX:
        return text
    return {"sha256": hashlib.sha256(text.encode()).hexdigest(), "bytes": len(text)}


def transcript(cli: str, name: str, inputs: str, work: str) -> dict:
    """Run one entry of RUNS in a fresh directory holding the inputs; what it printed, returned and wrote."""
    run = RUNS[name]
    d = os.path.join(work, name)
    os.makedirs(d)
    given = set(os.listdir(inputs))
    for f in given:
        os.symlink(os.path.join(inputs, f), os.path.join(d, f))
    p = subprocess.run([os.path.abspath(cli)] + run.args.split(), cwd=d, capture_output=True, text=True, timeout=600)
    files = {}
    for f in sorted(set(os.listdir(d)) - given):
        path = os.path.join(d, f)
        if os.path.isfile(path):
            with open(path, "rb") as fh:
                files[f] = file_record(f, fh.read())
    return {"args": run.args, "returncode": p.returncode, "stdout": mask_text(p.stdout, run.mask_metrics),
            "stderr": mask_text(p.stderr, run.mask_metrics), "files": files}


def device() -> dict:
    import torch
    p = torch.cuda.get_device_properties(0)
    return {"name": p.name, "sms": p.multi_processor_count}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("cli", help="the libFM binary the golden describes")
    ap.add_argument("--out", default=OUT)
    a = ap.parse_args()
    rec = {"device": device(), "runs": {}}
    with tempfile.TemporaryDirectory() as work:
        inputs = os.path.join(work, "inputs")
        os.makedirs(inputs)
        write_inputs(inputs)
        for name in RUNS:
            rec["runs"][name] = t = transcript(a.cli, name, inputs, work)
            print(name, t["returncode"], (t["stdout"].strip().splitlines() or [""])[-1][:100], flush=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", a.out)


if __name__ == "__main__":
    main()
