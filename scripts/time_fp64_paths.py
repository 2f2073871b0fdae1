"""Time the fp64 reference-order paths of two or more builds of libfmb200.so, alternating them.

  python scripts/time_fp64_paths.py --lib A/libfmb200.so --lib B/libfmb200.so [--repeats 3] [--out DIR]

Each (repeat, library) pair runs in a child process of its own (the library is picked through
FMB200_LIB), in the order A B A B ..., so that both builds see the same machine state.  A child
times, after a warm-up of each:
  inorder_rows       one C2 in-order epoch with the row-at-a-time kernel (tuning variant 1), k = 8
  inorder_wavefront  one C2 in-order epoch with the wavefront kernel (the default for C2), k = 8
  evaluate64         fmb200_evaluate on C2 in INORDER mode (kernel, per-row errors to the host, row-order sum)
  sgda, sgda_k40     one SGDA epoch with lambda-steps on two shapes of tests/test_sgda_gpu.py (k = 5, k = 40)
  eterms_c4          fmb200_mcmc_eterms on the C4 shape (10 000 054 cases, k = 16), D2H of the terms included
  mcmc_iter_c4       one MCMC iteration (sampling, multilevel) on the C4 shape
Epochs report the library's own CUDA-event time.  The other calls are bracketed by CUDA events
recorded on the library's stream (driver API), so they include what the call does on the host
before its final synchronise.  Prints per workload the range of each library over the repeats, in
ms, and the card's name and power limit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Events:
    """cuEventRecord / cuEventElapsedTime on a given stream (the calling thread holds the library's context)."""

    def __init__(self):
        self.cu = C.CDLL("libcuda.so.1")
        self.a, self.b = C.c_void_p(), C.c_void_p()
        self._ok(self.cu.cuEventCreate(C.byref(self.a), 0))
        self._ok(self.cu.cuEventCreate(C.byref(self.b), 0))

    @staticmethod
    def _ok(rc):
        if rc != 0:
            raise RuntimeError("CUDA driver call failed: %d" % rc)

    def time_ms(self, stream, fn):
        self._ok(self.cu.cuEventRecord(self.a, stream))
        fn()
        self._ok(self.cu.cuEventRecord(self.b, stream))
        self._ok(self.cu.cuEventSynchronize(self.b))
        ms = C.c_float()
        self._ok(self.cu.cuEventElapsedTime(C.byref(ms), self.a, self.b))
        return ms.value


def _stream(l):
    s = C.c_void_p()
    l._check(l.lib.fmb200_stream(l._ctx, C.byref(s)))
    return s


def _median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def child(reps: int) -> dict:
    import numpy as np
    sys.path.insert(0, ROOT)
    from libfm_b200 import MODE_INORDER, FmLearnSgdElement, FmModel, synth

    out = {}
    c2 = synth.movielens_1m_shaped(seed=7)

    def c2_learner():
        fm = FmModel(c2.num_feature, 8)
        fm.init_stdev = 0.1
        fm.init_numpy(42)
        l = FmLearnSgdElement(fm, mode=MODE_INORDER)
        l.task, l.learn_rate = 0, 0.01
        l.min_target, l.max_target = c2.min_target, c2.max_target
        l.push_hparams()
        return l

    for name, variant in (("inorder_rows", 1), ("inorder_wavefront", 0)):
        l = c2_learner()
        l.set_tuning(variant=variant)
        l.sgd_epoch(c2)  # warm-up
        out[name] = _median([l.sgd_epoch(c2) * 1e3 for _ in range(reps)])
        l.close()

    l = c2_learner()
    ev = _Events()  # in the context the learner made current
    st = _stream(l)
    l.evaluate(c2)
    out["evaluate64"] = _median([ev.time_ms(st, lambda: l.evaluate(c2)) for _ in range(reps)])
    l.close()

    # SGDA: the two_groups_reg and k40_ragged cases of tests/test_sgda_gpu.py
    for name, full, k, groups in (("sgda", synth.two_field(12_000, 300, 200, seed=4, planted_k=3), 5, 2),
                                  ("sgda_k40", synth.ragged(5000, 300, 6, seed=14), 40, 3)):
        tr, rest = synth.split_rows(full, full.num_cases * 2 // 3)
        va, _ = synth.split_rows(rest, rest.num_cases // 2)
        n = full.num_feature
        fm = FmModel(n, k)
        fm.v = np.random.default_rng(2).standard_normal((k, n)) * 0.1
        l = FmLearnSgdElement(fm, mode=MODE_INORDER)
        l.task, l.learn_rate = 0, 0.02
        l.min_target, l.max_target = float(tr.target.min()), float(tr.target.max())
        l.push_hparams()
        l.sgda_begin((np.arange(n) * groups // n).astype(np.uint32))
        l.sgda_epoch(tr, va, False)  # warm-up
        out[name] = _median([l.sgda_epoch(tr, va, True) * 1e3 for _ in range(reps)])
        l.close()

    # C4 shape (MovieLens-10M), k = 16
    tr = synth.two_field(10_000_054, 71_567, 10_681, seed=5)
    te = synth.two_field(200_000, 71_567, 10_681, seed=6)
    k = 16
    fm = FmModel(tr.num_feature, k)
    fm.init_stdev = 0.1
    fm.init_numpy(5)
    l = FmLearnSgdElement(fm, mode=MODE_INORDER)
    l.task, l.min_target, l.max_target = 0, tr.min_target, tr.max_target
    l.upload(tr, 0)
    l.upload(te, 1)
    st = _stream(l)
    l.mcmc_eterms(tr)
    out["eterms_c4"] = _median([ev.time_ms(st, lambda: l.mcmc_eterms(tr)) for _ in range(reps)])
    l.mcmc_begin(tr, te, True, True, 0.0, np.zeros(1), np.zeros((1, k)))
    l.mcmc_iteration()
    out["mcmc_iter_c4"] = _median([ev.time_ms(st, l.mcmc_iteration) for _ in range(reps)])
    l.close()
    return out


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lib", action="append", default=[], help="a libfmb200.so to time (give two or more)")
    ap.add_argument("--repeats", type=int, default=3, help="child runs per library, alternating")
    ap.add_argument("--reps", type=int, default=3, help="timed calls per workload in a child (median taken)")
    ap.add_argument("--out", help="directory for times.json")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        print(json.dumps(child(a.reps)))
        return
    if not a.lib:
        ap.error("give --lib at least once")
    libs = [os.path.abspath(p) for p in a.lib]
    runs = {p: [] for p in libs}
    for rep in range(a.repeats):
        for p in libs:
            env = dict(os.environ, FMB200_LIB=p)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--reps", str(a.reps)],
                               env=env, capture_output=True, text=True)
            if r.returncode != 0:
                sys.exit("child failed for %s:\n%s" % (p, r.stderr[-4000:]))
            runs[p].append(json.loads(r.stdout.strip().splitlines()[-1]))
            print("repeat %d %s: %s" % (rep, p, runs[p][-1]), flush=True)
    card = gpu_info()
    print("\n%s (name, power limit)" % card)
    for i, p in enumerate(libs):
        print("lib%d = %s" % (i, p))
    print("%-18s" % "ms" + "".join("%-24s" % ("lib%d min-max" % i) for i in range(len(libs))))
    for w in runs[libs[0]][0]:
        cells = []
        for p in libs:
            xs = [r[w] for r in runs[p]]
            cells.append("%.3f-%.3f" % (min(xs), max(xs)))
        print("%-18s" % w + "".join("%-24s" % c for c in cells))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "times.json"), "w") as f:
            json.dump({"card": card, "libs": libs, "runs": runs}, f, indent=1)


if __name__ == "__main__":
    main()
