"""Write tests/golden/reference/mcmc_relation.npz: what the reference's MCMC / ALS learner leaves after each of
its first ITERS iterations on relational data (block structure), run through scripts/mcmc_relation_probe.cpp on
the unmodified reference headers.  The blocks are written as files (<stem>.xt, <stem>.train, <stem>.test and an
optional <stem>.groups) and loaded by the reference's own RelationData::load and RelationJoin::load.

Per case the file holds the inputs (main CSR arrays, each block's .xt arrays, joins and groups, the -meta groups,
-regular, the seed), the joined group table, the loader's "num_cases=... num_values=... num_features=..." lines,
and per iteration t the exact scalars (w0, hyperparameters, counters, the #Iter line) and SHA-256 digests of w, v
and the three test prediction vectors, as tests/golden/reference/mcmc.npz does.

    python scripts/make_relation_golden.py [--ref /root/reference] [--bs]

--bs writes tests/golden/reference/mcmc_relation_bs.npz instead: the full-size BS shape of bs_case(), 2 iterations,
digests only (the inputs are regenerated from their seed).
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from libfm_b200 import Data, synth  # noqa: E402
from libfm_b200.model import write_transposed  # noqa: E402
from make_mcmc_golden import digest  # noqa: E402

ITERS = 6   # iteration index 5 is the first that pred_sum_all_but5 sums
OUT = os.path.join(ROOT, "tests", "golden", "reference", "mcmc_relation.npz")
OUT_BS = os.path.join(ROOT, "tests", "golden", "reference", "mcmc_relation_bs.npz")


def _block(rng, rows, nf, per_row, ones=True, dup_rows=0):
    """a relation block as a Data (its rows, its features): per_row distinct ids per row, dup_rows rows that
    name one id twice, values 1 or drawn"""
    rp, col = [0], []
    for r in range(rows):
        m = int(rng.integers(0, per_row + 1))
        ids = list(rng.choice(nf, size=min(m, nf), replace=False))
        if r < dup_rows and ids:
            ids.append(ids[0])
        col += ids
        rp.append(len(col))
    val = np.ones(len(col), np.float32) if ones else rng.uniform(0.2, 2.0, len(col)).astype(np.float32)
    return Data(np.array(rp, np.uint64), np.array(col, np.uint32), val, np.zeros(rows, np.float32), nf)


def _main(rng, n, nf, per_row, task):
    rp, col = [0], []
    for _ in range(n):
        m = int(rng.integers(0, per_row + 1)) if nf else 0
        col += list(rng.choice(nf, size=min(m, nf), replace=False)) if m else []
        rp.append(len(col))
    y = rng.integers(1, 6, n).astype(np.float32)
    if task == 1:
        y = np.where(y >= 4, 1.0, -1.0).astype(np.float32)
    val = rng.uniform(0.5, 1.5, len(col)).astype(np.float32)
    return Data(np.array(rp, np.uint64), np.array(col, np.uint32), val, y, nf)


def cases():
    """name -> dict(main train/test, blocks [(Data, train join, test join, groups or None, binary join)], k, ...)"""
    out = {}

    def add(name, seed, n_tr, n_te, main_nf, blocks, k, sample, task=0, reg=(), k0=1, k1=1, meta=None):
        rng = np.random.default_rng(seed)
        tr, te = _main(rng, n_tr, main_nf, 3, task), _main(rng, n_te, main_nf, 3, task)
        bl = []
        for rows, nf, per_row, ones, dup_rows, groups, binary, test_only in blocks:
            d = _block(rng, rows, nf, per_row, ones, dup_rows)
            # train cases join the first rows - test_only rows; the last few rows only test cases join, and some
            # rows no case joins at all when rows > what the joins reach
            reach = max(1, rows - test_only - 2)
            jtr = rng.integers(0, reach, n_tr).astype(np.uint32)
            jte = rng.integers(0, rows, n_te).astype(np.uint32)
            bl.append(dict(data=d, train=jtr, test=jte, groups=groups, binary=binary))
        out[name] = dict(train=tr, test=te, blocks=bl, k=k, k0=k0, k1=k1, task=task, sample=int(sample),
                         multilevel=int(sample), reg=np.array(reg, float), seed=seed, meta=meta)

    # (rows, nf, per_row, values 1, rows naming an id twice, groups, binary joins, rows only test cases join)
    add("main_features_one_block_mcmc", 3, 1500, 300, 40, [(120, 60, 4, False, 0, None, False, 0)], 4, True)
    for m, s in (("mcmc", True), ("als", False)):
        user = (200, 150, 12, True, 0, None, True, 0)        # a user's implicitly rated items (SVD++ style)
        item = (90, 25, 3, True, 0, np.arange(25) % 2, False, 0)  # item attributes with a .groups file
        add(f"user_item_{m}", 5, 2000, 400, 0, [user, item], 5, s,
            reg=() if s else (0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9))
    add("cls_mcmc", 7, 1200, 300, 30, [(100, 40, 5, True, 0, None, True, 0)], 4, True, task=1)
    add("awkward_mcmc", 9, 900, 250, 20,
        [(150, 50, 6, False, 10, None, True, 15), (60, 12, 3, False, 4, np.array([0, 1, 2] * 4), False, 5)], 3, True)
    add("awkward_als", 9, 900, 250, 20,
        [(150, 50, 6, False, 10, None, False, 15), (60, 12, 3, False, 4, None, True, 5)], 3, False, reg=(0.2,))
    # -meta groups of the main table ahead of the blocks' groups, and per-group -regular (3 + 2 groups)
    add("main_meta_als", 11, 1000, 200, 30, [(80, 20, 4, False, 0, np.arange(20) % 2, False, 0)], 4, False,
        reg=(0.1,) + tuple(0.05 * (g + 1) for g in range(10)), meta=np.arange(30) % 3)
    return out


N_USERS, N_ITEMS = 6040, 3706


def bs_case():
    """The full-size BS shape of MovieLens-1M: 1 000 209 train and 100 000 test ratings with Zipf(1) user and item
    popularity and empty main rows.  The user block carries the user's id and, SVD++ style, every item the user
    rated in train with value 1/sqrt(#items); the item block carries the item's id.  k = 8, MCMC."""
    full = synth.two_field(1_100_209, N_USERS, N_ITEMS, seed=5, zipf=1.0)
    tr_full, te_full = synth.split_rows(full, 1_000_209)

    def joins(d):
        c = d.col.reshape(-1, 2).astype(np.int64)
        return c[:, 0].astype(np.uint32), (c[:, 1] - N_USERS).astype(np.uint32)

    u_tr, i_tr = joins(tr_full)
    u_te, i_te = joins(te_full)
    pairs = np.unique(u_tr.astype(np.int64) * N_ITEMS + i_tr)
    pu, pi = pairs // N_ITEMS, pairs % N_ITEMS
    cnt = np.bincount(pu, minlength=N_USERS)
    rows = np.concatenate([np.arange(N_USERS), pu])
    cols = np.concatenate([np.arange(N_USERS), N_USERS + pi])
    vals = np.concatenate([np.ones(N_USERS, np.float32),
                           (1.0 / np.sqrt(cnt[pu].astype(np.float64))).astype(np.float32)])
    o = np.lexsort((cols, rows))
    user = Data(np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=N_USERS))]).astype(np.uint64),
                cols[o].astype(np.uint32), vals[o], np.zeros(N_USERS, np.float32), N_USERS + N_ITEMS)
    item = Data(np.arange(N_ITEMS + 1, dtype=np.uint64), np.arange(N_ITEMS, dtype=np.uint32),
                np.ones(N_ITEMS, np.float32), np.zeros(N_ITEMS, np.float32), N_ITEMS)
    empty = lambda d: Data(np.zeros(d.num_cases + 1, np.uint64), np.zeros(0, np.uint32),  # noqa: E731
                           np.zeros(0, np.float32), d.target, 0)
    tr, te = empty(tr_full), empty(te_full)
    blocks = [dict(data=user, train=u_tr, test=u_te, groups=None, binary=True),
              dict(data=item, train=i_tr, test=i_te, groups=None, binary=True)]
    return dict(train=tr, test=te, blocks=blocks, k=8, k0=1, k1=1, task=0, sample=1, multilevel=1,
                reg=np.zeros(0), seed=7, meta=None)


def write_block_files(stem, b, n_tr, n_te):
    write_transposed(b["data"], stem + ".xt")
    for side, j in (("train", b["train"]), ("test", b["test"])):
        if b["binary"]:
            with open(f"{stem}.{side}", "wb") as f:
                f.write(np.array([1, 4, j.size], np.uint32).tobytes() + j.astype(np.uint32).tobytes())
        else:
            with open(f"{stem}.{side}", "w") as f:
                f.write("\n".join(str(int(x)) for x in j) + "\n")
    if b["groups"] is not None:
        with open(stem + ".groups", "w") as f:
            f.write("\n".join(str(int(x)) for x in b["groups"]) + "\n")


def build_probe(ref: str, tmp: str) -> C.CDLL:
    so = os.path.join(tmp, "mcmc_relation_probe.so")
    subprocess.run(["g++", "-O3", "-w", "-fPIC", "-shared", "-Wl,-Bsymbolic", "-I", os.path.join(ref, "src"),
                    os.path.join(ROOT, "scripts", "mcmc_relation_probe.cpp"), "-o", so], check=True)
    return C.CDLL(so)


def run(lib, c, stems, iters, meta_file=""):
    tr, te, k = c["train"], c["test"], c["k"]
    P = lambda a, t: np.ascontiguousarray(a).ctypes.data_as(C.POINTER(t))  # noqa: E731
    cap = 1 << 16
    n_out, G_out = C.c_uint32(), C.c_uint32()
    group, per_group = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
    init, state = np.zeros(1 + cap * (k + 1)), np.zeros(1 + cap * (k + 1))
    hyper = np.zeros(cap)
    cnt = np.zeros(16, np.uint32)
    pred = np.zeros(3 * max(te.num_cases, 1))
    buf = C.create_string_buffer(1 << 20)
    keep = [tr.row_ptr, tr.col, tr.val, tr.target, te.row_ptr, te.col, te.val, te.target, c["reg"]]
    rc = lib.probe_mcmc_relation(
        k, c["k0"], c["k1"], C.c_long(c["seed"]),
        C.c_uint64(tr.num_cases), P(keep[0], C.c_uint64), P(keep[1], C.c_uint32), P(keep[2], C.c_float),
        P(keep[3], C.c_float), tr.num_feature,
        C.c_uint64(te.num_cases), P(keep[4], C.c_uint64), P(keep[5], C.c_uint32), P(keep[6], C.c_float),
        P(keep[7], C.c_float), te.num_feature, "\n".join(stems).encode(), len(stems), meta_file.encode(), c["task"],
        c["sample"],
        c["multilevel"], P(keep[8], C.c_double), len(c["reg"]), iters, C.c_double(tr.min_target),
        C.c_double(tr.max_target), C.byref(n_out), C.byref(G_out), P(group, C.c_uint32), P(per_group, C.c_uint32), cap,
        P(init, C.c_double), P(state, C.c_double), P(hyper, C.c_double), len(hyper), P(cnt, C.c_uint32),
        P(pred, C.c_double), buf, len(buf))
    if rc != 0:
        raise RuntimeError("reference probe failed")
    n, G = n_out.value, G_out.value
    text = buf.value.decode()
    lines = [ln for ln in text.splitlines() if ln.startswith("#Iter")]
    loads = [ln for ln in text.splitlines() if ln.startswith("num_cases=")]
    return (n, G, group[:n].copy(), per_group[:G].copy(), init[:1 + n * (k + 1)], state[:1 + n * (k + 1)],
            hyper[:1 + 2 * G + 2 * G * k], cnt, pred[:3 * te.num_cases].reshape(3, te.num_cases), lines, loads)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    ap.add_argument("--bs", action="store_true",
                    help="write the full-size BS record (2 iterations, digests only) instead")
    args = ap.parse_args()
    rec = {}
    out_path, iters = (OUT_BS, 2) if args.bs else (OUT, ITERS)
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_probe(args.ref, tmp)
        for name, c in ({"bs_mcmc": bs_case()} if args.bs else cases()).items():
            tr, te = c["train"], c["test"]
            stems = []
            meta_file = ""
            if c["meta"] is not None:
                meta_file = os.path.join(tmp, f"{name}.meta")
                with open(meta_file, "w") as f:
                    f.write("\n".join(str(int(x)) for x in c["meta"]) + "\n")
                rec[f"{name}/meta"] = np.asarray(c["meta"], np.uint32)
            for i, b in enumerate(c["blocks"]):
                stem = os.path.join(tmp, f"{name}_rel{i}")
                write_block_files(stem, b, tr.num_cases, te.num_cases)
                stems.append(stem)
                if args.bs:
                    continue
                d = b["data"]
                rec[f"{name}/rel{i}/rows"] = np.array([d.num_cases, d.num_feature, int(b["binary"])], np.int64)
                rec[f"{name}/rel{i}/row_ptr"] = d.row_ptr
                rec[f"{name}/rel{i}/col"] = d.col
                rec[f"{name}/rel{i}/val"] = d.val
                rec[f"{name}/rel{i}/train"] = b["train"]
                rec[f"{name}/rel{i}/test"] = b["test"]
                if b["groups"] is not None:
                    rec[f"{name}/rel{i}/groups"] = np.asarray(b["groups"], np.uint32)
            for key, val in (("tr_row_ptr", tr.row_ptr), ("tr_col", tr.col), ("tr_val", tr.val),
                             ("tr_target", tr.target), ("te_row_ptr", te.row_ptr), ("te_col", te.col),
                             ("te_val", te.val), ("te_target", te.target), ("reg", c["reg"])):
                if not args.bs:
                    rec[f"{name}/{key}"] = val
            rec[f"{name}/minmax"] = np.array([tr.min_target, tr.max_target])
            for t in range(iters):
                n, G, group, per_group, init, state, hyper, cnt, pred, lines, loads = run(lib, c, stems, t + 1,
                                                                                          meta_file)
                k = c["k"]
                if t == 0:
                    rec[f"{name}/cfg"] = np.array([n, k, c["k0"], c["k1"], c["task"], c["sample"], c["multilevel"],
                                                   c["seed"], tr.num_feature, te.num_feature, len(stems)], np.int64)
                    rec[f"{name}/group"] = group
                    rec[f"{name}/per_group"] = per_group
                    rec[f"{name}/loads"] = np.array(loads)
                    rec[f"{name}/init_digest"] = np.array(digest(init))
                rec[f"{name}/{t}/w0"] = np.float64(state[0])
                rec[f"{name}/{t}/w"] = np.array(digest(state[1:1 + n]))
                rec[f"{name}/{t}/v"] = np.array(digest(state[1 + n:]))   # factor-major [k][n]
                rec[f"{name}/{t}/hyper"] = hyper
                rec[f"{name}/{t}/counters"] = cnt
                for i, p in enumerate(("pred_this", "pred_sum_all", "pred_sum_all_but5")):
                    rec[f"{name}/{t}/{p}"] = np.array(digest(pred[i]))
                rec[f"{name}/{t}/line"] = np.array(lines[-1])
            print(name, G, lines[-1])
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    np.savez_compressed(out_path, **rec)
    print("wrote", out_path)


if __name__ == "__main__":
    main()
