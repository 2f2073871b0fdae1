"""Write tests/golden/reference/mcmc.npz: what the reference's MCMC / ALS learner
(fm_learn_mcmc_simultaneous, run through scripts/mcmc_ref_probe.cpp on the unmodified reference headers)
leaves after each of its first ITERS iterations, for the cases tests/test_mcmc_sweep_gpu.py replays.

Per case the file holds the inputs (CSR arrays, groups, regularisation, seed) and, per iteration t,
the exact scalars (w0, hyperparameters, counters, the #Iter line) and SHA-256 digests of w, v and the
three test prediction vectors.  The probe reruns the learner from the seed for every t, so iteration t's
record is the state after t+1 iterations of one run.

    python scripts/make_mcmc_golden.py [--ref /root/reference] [--c4]

--c4 writes tests/golden/reference/mcmc_c4.npz instead: the full-size C4 shape, 2 iterations, digests only
(the inputs are regenerated from their seeds).
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from libfm_b200 import Data, synth  # noqa: E402

ITERS = 7
OUT = os.path.join(ROOT, "tests", "golden", "reference", "mcmc.npz")
OUT_C4 = os.path.join(ROOT, "tests", "golden", "reference", "mcmc_c4.npz")


def digest(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()


def _two_field_split(n_rows, n_users, n_items, seed, n_extra):
    """two-field one-hot train; the test also names n_extra ids beyond the train's (test-only features),
    and num_feature leaves a few ids in neither (empty columns)."""
    d = synth.two_field(n_rows, n_users, n_items, seed=seed)
    tr, te = synth.split_rows(d, n_rows * 4 // 5)
    r = np.random.default_rng(seed + 1)
    col = te.col.copy()
    pick = r.choice(te.num_cases, size=min(n_extra, te.num_cases), replace=False)
    col[2 * pick + 1] = d.num_feature + np.arange(pick.size, dtype=np.uint32)
    n = d.num_feature + pick.size + 3
    te = Data(te.row_ptr, col, te.val, te.target, n)
    tr = Data(tr.row_ptr, tr.col, tr.val, tr.target, d.num_feature)
    return tr, te, n


def cases():
    """name -> dict(train, test, n, k, k0, k1, task, sample, multilevel, group, per_group, reg0, wl, vl, seed)"""
    out = {}

    def add(name, tr, te, n, k, sample, task=0, k0=1, k1=1, group=None, per_group=None, reg=(), seed=7):
        group = np.zeros(n, np.uint32) if group is None else np.asarray(group, np.uint32)
        G = int(group.max()) + 1 if per_group is None else len(per_group)
        if per_group is None:
            per_group = np.bincount(group, minlength=G).astype(np.uint32)
        reg = list(reg)
        if len(reg) == 0:      # libfm.cpp:331-336
            reg0, wl, vl = 0.0, np.zeros(G), np.zeros((G, k))
        elif len(reg) == 1:
            reg0, wl, vl = reg[0], np.full(G, reg[0]), np.full((G, k), reg[0])
        elif len(reg) == 3:
            reg0, wl, vl = reg[0], np.full(G, reg[1]), np.full((G, k), reg[2])
        else:                  # 1 + 2G: per-group values (:349-364)
            reg0, wl = reg[0], np.array(reg[1:1 + G])
            vl = np.repeat(np.array(reg[1 + G:1 + 2 * G])[:, None], k, axis=1)
        if task == 1:  # ratings 4 and 5 are the positive class
            tr.target = np.where(tr.target >= 4, 1.0, 0.0).astype(np.float32)
            te.target = np.where(te.target >= 4, 1.0, 0.0).astype(np.float32)
            tr.binarize_targets()
            te.binarize_targets()
        out[name] = dict(train=tr, test=te, n=n, k=k, k0=k0, k1=k1, task=task, sample=int(sample),
                         multilevel=int(sample), group=group, per_group=np.asarray(per_group, np.uint32),
                         reg0=float(reg0), wl=np.asarray(wl, float), vl=np.asarray(vl, float).reshape(G, k),
                         seed=seed)

    for m, s in (("mcmc", True), ("als", False)):
        c1 = synth.plumbing_10k()
        tr, te = synth.split_rows(c1, 8000)
        add(f"c1_{m}", Data(tr.row_ptr, tr.col, tr.val, tr.target, c1.num_feature),
            Data(te.row_ptr, te.col, te.val, te.target, c1.num_feature), c1.num_feature, 8, s,
            reg=() if s else (0.1,))
        tr, te, n = _two_field_split(3000, 200, 100, 11, 12)
        add(f"twofield_{m}", tr, te, n, 4, s, reg=() if s else (0.05,))
        # ragged: unsorted rows, duplicate ids, one-entry and empty rows; groups interleave the ids (many
        # short runs) and the group list covers only the first 250 ids, as a short -meta file does
        d = synth.ragged(2400, 300, 11, seed=21)
        tr, te = synth.split_rows(d, 2000)
        grp = np.zeros(300, np.uint32)
        grp[:250] = np.arange(250) % 3
        per = np.bincount(grp[:250], minlength=3).astype(np.uint32)
        add(f"ragged_meta_{m}", Data(tr.row_ptr, tr.col, tr.val, tr.target, 300),
            Data(te.row_ptr, te.col, te.val, te.target, 300), 300, 5, s, group=grp, per_group=per,
            reg=() if s else (0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8))
        d = synth.ragged(1500, 120, 6, seed=22)
        tr, te = synth.split_rows(d, 1200)
        add(f"k0_{m}", Data(tr.row_ptr, tr.col, tr.val, tr.target, 120),
            Data(te.row_ptr, te.col, te.val, te.target, 120), 120, 0, s, reg=() if s else (0.1,))
        add(f"nobias_nolinear_{m}", Data(tr.row_ptr, tr.col, tr.val, tr.target, 120),
            Data(te.row_ptr, te.col, te.val, te.target, 120), 120, 4, s, k0=0, k1=0,
            reg=() if s else (0.1,))
        tr, te, n = _two_field_split(2500, 150, 80, 31, 8)
        add(f"cls_{m}", tr, te, n, 4, s, task=1, reg=() if s else (0.1,))
    tr, te, n = _two_field_split(2000, 120, 60, 41, 6)
    add("als_zero_reg", tr, te, n, 3, False)
    # many more features than training cases (n > 2N): the index build's per-feature arrays outgrow the
    # per-case ones
    d = synth.ragged(500, 5000, 4, seed=23)
    tr, te = synth.split_rows(d, 400)
    add("wide_mcmc", Data(tr.row_ptr, tr.col, tr.val, tr.target, 5000),
        Data(te.row_ptr, te.col, te.val, te.target, 5000), 5000, 3, True)
    return out


def c4_case():
    """BASELINE C4 shape: MovieLens-10M-sized two-field train (10 000 054 cases, 71 567 users, 10 681 items,
    items with tens of thousands of cases), k=16, MCMC; 200 000 test cases of the same shape."""
    out = {}
    tr = synth.two_field(10_000_054, 71_567, 10_681, seed=5)
    te = synth.two_field(200_000, 71_567, 10_681, seed=6)
    n = tr.num_feature
    G = 1
    out["c4_mcmc"] = dict(train=tr, test=te, n=n, k=16, k0=1, k1=1, task=0, sample=1, multilevel=1,
                          group=np.zeros(n, np.uint32), per_group=np.array([n], np.uint32), reg0=0.0,
                          wl=np.zeros(G), vl=np.zeros((G, 16)), seed=7)
    return out


def build_probe(ref: str, tmp: str) -> C.CDLL:
    so = os.path.join(tmp, "mcmc_ref_probe.so")
    # -Bsymbolic: the reference defines its own erf (random.h); inside a shared object the call would
    # otherwise bind to libm's erf, which the process has already loaded
    subprocess.run(["g++", "-O3", "-w", "-fPIC", "-shared", "-Wl,-Bsymbolic", "-I", os.path.join(ref, "src"),
                    os.path.join(ROOT, "scripts", "mcmc_ref_probe.cpp"), "-o", so], check=True)
    return C.CDLL(so)


def run(lib, c, iters):
    tr, te, n, k = c["train"], c["test"], c["n"], c["k"]
    G = len(c["per_group"])
    P = lambda a, t: np.ascontiguousarray(a).ctypes.data_as(C.POINTER(t))  # noqa: E731
    init = np.zeros(1 + n + n * k)
    state = np.zeros(1 + n + n * k)
    hyper = np.zeros(1 + 2 * G + 2 * G * k)
    cnt = np.zeros(16, np.uint32)
    pred = np.zeros(3 * max(te.num_cases, 1))
    buf = C.create_string_buffer(1 << 20)
    keep = [tr.row_ptr, tr.col, tr.val, tr.target, te.row_ptr, te.col, te.val, te.target, c["group"],
            c["per_group"], c["wl"], np.ascontiguousarray(c["vl"])]
    rc = lib.probe_mcmc(
        C.c_uint32(n), k, c["k0"], c["k1"], C.c_double(0.1), C.c_long(c["seed"]),
        C.c_uint64(tr.num_cases), P(keep[0], C.c_uint64), P(keep[1], C.c_uint32), P(keep[2], C.c_float),
        P(keep[3], C.c_float), tr.num_feature,
        C.c_uint64(te.num_cases), P(keep[4], C.c_uint64), P(keep[5], C.c_uint32), P(keep[6], C.c_float),
        P(keep[7], C.c_float), te.num_feature, c["task"], c["sample"], c["multilevel"], C.c_uint32(G),
        P(keep[8], C.c_uint32), P(keep[9], C.c_uint32), C.c_double(c["reg0"]), P(keep[10], C.c_double),
        P(keep[11], C.c_double), iters, C.c_double(tr.min_target), C.c_double(tr.max_target),
        P(init, C.c_double), P(state, C.c_double), P(hyper, C.c_double), P(cnt, C.c_uint32), P(pred, C.c_double),
        buf, len(buf))
    if rc != 0:
        raise RuntimeError("reference probe failed")
    lines = [ln for ln in buf.value.decode().splitlines() if ln.startswith("#Iter")]
    return init, state, hyper, cnt, pred[:3 * te.num_cases].reshape(3, te.num_cases), lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    ap.add_argument("--c4", action="store_true",
                    help="write the full-size C4 record (2 iterations, digests only; minutes of CPU) instead")
    args = ap.parse_args()
    rec = {}
    out_path, iters = (OUT_C4, 2) if args.c4 else (OUT, ITERS)
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_probe(args.ref, tmp)
        for name, c in (c4_case() if args.c4 else cases()).items():
            tr, te = c["train"], c["test"]
            for key, val in () if args.c4 else (("tr_row_ptr", tr.row_ptr), ("tr_col", tr.col), ("tr_val", tr.val),
                             ("tr_target", tr.target), ("te_row_ptr", te.row_ptr), ("te_col", te.col),
                             ("te_val", te.val), ("te_target", te.target), ("group", c["group"]),
                             ("per_group", c["per_group"]), ("wl", c["wl"]), ("vl", c["vl"])):
                rec[f"{name}/{key}"] = val
            rec[f"{name}/cfg"] = np.array([c["n"], c["k"], c["k0"], c["k1"], c["task"], c["sample"],
                                           c["multilevel"], c["seed"], tr.num_feature, te.num_feature], np.int64)
            rec[f"{name}/reg0"] = np.float64(c["reg0"])
            rec[f"{name}/minmax"] = np.array([tr.min_target, tr.max_target])
            for t in range(iters):
                init, state, hyper, cnt, pred, lines = run(lib, c, t + 1)
                n, k = c["n"], c["k"]
                if t == 0:
                    rec[f"{name}/init_digest"] = np.array(digest(init))
                rec[f"{name}/{t}/w0"] = np.float64(state[0])
                rec[f"{name}/{t}/w"] = np.array(digest(state[1:1 + n]))
                rec[f"{name}/{t}/v"] = np.array(digest(state[1 + n:]))   # factor-major [k][n]
                rec[f"{name}/{t}/hyper"] = hyper
                rec[f"{name}/{t}/counters"] = cnt
                for i, p in enumerate(("pred_this", "pred_sum_all", "pred_sum_all_but5")):
                    rec[f"{name}/{t}/{p}"] = np.array(digest(pred[i]))
                rec[f"{name}/{t}/line"] = np.array(lines[-1])
            print(name, lines[-1])
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    np.savez_compressed(out_path, **rec)
    print("wrote", out_path)


if __name__ == "__main__":
    main()
