"""Time one MCMC iteration on the full-size BS shape (make_relation_golden.bs_case) two ways.

  python scripts/time_mcmc_relation.py [--reps 3] [--phases] [--threads T] [--no-reference] [--out FILE]

  gpu        fmb200_mcmc_iteration with the two relation blocks (-mode inorder), host wall clock around the call,
             which returns after the iteration's last device work and host step; iterations 2 .. reps + 1 of one
             learner (the first warms up), median reported
  reference  the stock reference's time_learn (user time of its iteration on one host core) for the second
             iteration of oracle/_ref/libFM -method mcmc -relation user,item on the same files, from its -rlog
  phases     (--phases) one more GPU iteration under torch.profiler: the device time of its kernels by phase (block
             sweeps, unsync / resync, q rebuild, e-terms, the rest), from CUDA activity records; the iteration's wall
             time less their sum is host work and launch gaps

FMB200_LIB selects the library (_capi.py), so two builds can be timed in turn.

Data: 1 000 209 train and 100 000 test ratings of MovieLens-1M shape with Zipf(1) popularity and empty main rows; a
user block (6040 rows: the user's id and the items the user rated, 1/sqrt(#items)) and an item block (3706 rows),
k = 8.  Prints the card's name and power limit with the times.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from libfm_b200 import MODE_INORDER, FmLearnSgdElement, FmModel, RelationData, RelationJoin  # noqa: E402
from make_relation_golden import bs_case, write_block_files  # noqa: E402

STEMS = ("user", "item")


def write_files(c, d: str) -> dict:
    """the case as the stock command line reads it: main tables as text (targets only), blocks as files"""
    paths = {}
    for name in ("train", "test"):
        paths[name] = os.path.join(d, name + ".libfm")
        with open(paths[name], "w") as f:
            f.write("".join("%g\n" % y for y in c[name].target))
    for stem, b in zip(STEMS, c["blocks"]):
        write_block_files(os.path.join(d, stem), b, c["train"].num_cases, c["test"].num_cases)
    return paths


# phase -> substrings of the kernel names it takes (fm_mcmc.cu); REL_Q = 0, REL_ETERM = 1
PHASES = (("block sweeps", ("mcmc_block_sweep_kernel", "mcmc_cta_sweep_kernel")),
          ("unsync / resync", ("rel_unsync_kernel", "rel_resync_kernel")),
          ("q rebuild", ("rel_row_kernel<0>", "rel_case_q_kernel")),
          ("e-terms", ("rel_row_kernel<1>", "fm_eterm64_kernel")))


def phase_ms(l) -> tuple[dict, float]:
    """one iteration under torch.profiler: {phase: device ms} (kernels only) and the iteration's wall ms"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        l.mcmc_iteration()
        wall = (time.perf_counter() - t0) * 1e3
    out = {name: 0.0 for name, _ in PHASES}
    out["other kernels"] = 0.0
    n = 0
    for e in prof.events():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if not us or e.name.startswith("cuda") or "Memcpy" in e.name or "Memset" in e.name:
            continue  # kernels only
        n += 1
        name = next((p for p, keys in PHASES if any(k in e.name for k in keys)), "other kernels")
        out[name] += us / 1e3
    if n == 0:
        raise RuntimeError("torch.profiler recorded no kernels of the iteration")
    return out, wall


def gpu_ms(c, d: str, reps: int, phases: bool = False, threads: int = 0):
    tr, te, k = c["train"], c["test"], c["k"]
    rel = []
    for stem in STEMS:
        b = RelationData.load(os.path.join(d, stem))
        rel.append((b, RelationJoin.load(os.path.join(d, stem + ".train"), tr.num_cases, b),
                    RelationJoin.load(os.path.join(d, stem + ".test"), te.num_cases, b)))
    n = sum(b.num_feature for b, _, _ in rel)
    l = FmLearnSgdElement(FmModel(n, k), mode=MODE_INORDER)
    if threads:
        l.set_tuning(threads=threads)  # the width of the CTA that sweeps narrow runs
    l.upload(tr, 0)
    l.upload(te, 1)
    l.fm.init(42)
    l.fm.w = np.random.default_rng(1).standard_normal(n) * 0.1
    l.push_params()
    l.min_target, l.max_target = tr.min_target, tr.max_target
    l.mcmc_begin(tr, te, True, True, 0.0, np.zeros(3), np.zeros((3, k)), relations=rel)
    l.mcmc_iteration()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        l.mcmc_iteration()
        out.append((time.perf_counter() - t0) * 1e3)
    ph = phase_ms(l) if phases else None
    l.close()
    return out, ph


def reference_ms(paths: dict, d: str, k: int) -> float | None:
    exe = os.path.join(ROOT, "oracle", "_ref", "libFM")
    if not os.path.exists(exe):
        return None
    rlog = os.path.join(d, "rlog")
    cmd = [exe, "-task", "r", "-method", "mcmc", "-dim", "1,1,%d" % k, "-iter", "2", "-train", paths["train"],
           "-test", paths["test"], "-relation", ",".join(os.path.join(d, s) for s in STEMS), "-init_stdev", "0.1",
           "-seed", "42", "-rlog", rlog]
    subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    with open(rlog) as f:
        lines = f.read().splitlines()
    head = lines[0].split("\t")
    return float(lines[2].split("\t")[head.index("time_learn")]) * 1e3


def gpu_info() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True)
    except FileNotFoundError:
        return "unknown"
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", help="also write the report to this file")
    ap.add_argument("--reference-only", action="store_true", help="skip the GPU (checks the reference command)")
    ap.add_argument("--no-reference", action="store_true", help="skip the reference run")
    ap.add_argument("--phases", action="store_true", help="also time one iteration's kernels by phase")
    ap.add_argument("--threads", type=int, default=0, help="width of the narrow-run CTA (0: the library's)")
    a = ap.parse_args()
    c = bs_case()
    with tempfile.TemporaryDirectory() as d:
        paths = write_files(c, d)
        g, ph = ([], None) if a.reference_only else gpu_ms(c, d, a.reps, a.phases, a.threads)
        ref = None if a.no_reference else reference_ms(paths, d, c["k"])
    nnz = [b["data"].num_values for b in c["blocks"]]
    lines = ["MCMC iteration, full-size BS shape: %d train / %d test cases, empty main rows, user block %d entries, "
             "item block %d entries, k = %d" % (c["train"].num_cases, c["test"].num_cases, nnz[0], nnz[1], c["k"]),
             "card (name, power limit): %s" % gpu_info(),
             "gpu        %10s ms  (runs: %s)" % ("%.1f" % sorted(g)[len(g) // 2] if g else "n/a",
                                                  ", ".join("%.1f" % x for x in g)),
             "reference  %10s ms  (stock libFM -method mcmc -relation, time_learn of iteration 1, one host core)"
             % ("%.1f" % ref if ref is not None else "n/a"),
             "library    %s%s" % (os.environ.get("FMB200_LIB", "libfm_b200/lib/libfmb200.so"),
                                 ", narrow-run CTA of %d threads" % a.threads if a.threads else "")]
    if ph:
        out, wall = ph
        lines.append("phases of one profiled iteration (device ms of its kernels; wall %.1f ms):" % wall)
        lines += ["  %-16s %8.1f ms" % (name, ms) for name, ms in out.items()]
        lines.append("  %-16s %8.1f ms" % ("host and gaps", wall - sum(out.values())))
    text = "\n".join(lines) + "\n"
    sys.stdout.write(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
