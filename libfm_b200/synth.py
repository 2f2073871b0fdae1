"""Seeded synthetic inputs in the shapes BASELINE.json names (SURVEY.md section 8d).

No real data set is reachable offline; every generator is a pure function of its
seed.  Rows follow the libFM one-hot convention (value 1.0 per active field).
"""
from __future__ import annotations

import numpy as np

from .model import Data


def _fields_to_data(cols: np.ndarray, target: np.ndarray, num_feature: int) -> Data:
    n_rows, z = cols.shape
    row_ptr = np.arange(0, (n_rows + 1) * z, z, dtype=np.uint64)
    val = np.ones(n_rows * z, dtype=np.float32)
    return Data(row_ptr, cols.reshape(-1).astype(np.uint32), val, target.astype(np.float32),
                num_feature)


def two_field(n_rows: int, n_users: int, n_items: int, seed: int, zipf: float = 0.0,
              planted_k: int = 0, noise: float = 0.5) -> Data:
    """MovieLens-shaped triples: row = user:1 (n_users+item):1, rating in 1..5.

    zipf > 0 draws ids from a Zipf-like popularity law (collision stress).
    planted_k > 0 generates ratings from a hidden FM of that rank plus noise
    (so that learning has signal); otherwise ratings are uniform in {1..5}
    exactly as SURVEY.md specifies for C1/C2.
    """
    r = np.random.default_rng(seed)

    def draw(n_ids):
        if zipf > 0:
            p = 1.0 / np.arange(1, n_ids + 1) ** zipf
            p /= p.sum()
            return r.permutation(n_ids)[r.choice(n_ids, size=n_rows, p=p)]
        return r.integers(0, n_ids, size=n_rows)

    u = draw(n_users)
    i = draw(n_items)
    cols = np.stack([u, n_users + i], axis=1)
    if planted_k > 0:
        bu = 0.5 * r.standard_normal(n_users)
        bi = 0.5 * r.standard_normal(n_items)
        pu = r.standard_normal((n_users, planted_k)) * (0.8 / np.sqrt(planted_k))
        qi = r.standard_normal((n_items, planted_k)) * (0.8 / np.sqrt(planted_k))
        y = 3.0 + bu[u] + bi[i] + (pu[u] * qi[i]).sum(1) + noise * r.standard_normal(n_rows)
        y = np.clip(np.rint(y), 1, 5)
    else:
        y = r.integers(1, 6, size=n_rows)
    return _fields_to_data(cols, y, n_users + n_items)


def split_rows(d: Data, n_first: int):
    """(first n_first rows, the remaining rows) of one data set -- train / held-out rows of the SAME
    planted model (two generator calls with different seeds plant different models)."""
    return d.rows(0, n_first), d.rows(n_first, d.num_cases)


def movielens_1m_planted(n_test: int = 100_000, seed: int = 7, zipf: float = 0.0):
    """C2-shaped train set (1 000 209 rows) + held-out rows drawn from the same planted rank-4 model."""
    full = two_field(1_000_209 + n_test, 6040, 3706, seed, zipf=zipf, planted_k=4)
    return split_rows(full, 1_000_209)


def movielens_1m_shaped(seed: int = 7, zipf: float = 0.0, planted_k: int = 0,
                        n_rows: int = 1_000_209) -> Data:
    """BASELINE config C2: 6040 users x 3706 items, ~1M rows, 2 nnz/row."""
    return two_field(n_rows, 6040, 3706, seed, zipf=zipf, planted_k=planted_k)


def plumbing_10k(seed: int = 1234, n_rows: int = 10_000) -> Data:
    """BASELINE config C1: 10k rows, user in [0,6000), item in [0,4000)."""
    return two_field(n_rows, 6000, 4000, seed)


def multi_field(n_rows: int, n_fields: int, n_features: int, seed: int,
                binary_target: bool = True) -> Data:
    """Criteo-shaped rows (C3/C5): n_features split evenly into n_fields fields,
    one active id per field, value 1, y in {0,1}."""
    r = np.random.default_rng(seed)
    per = n_features // n_fields
    cols = r.integers(0, per, size=(n_rows, n_fields), dtype=np.int64)
    cols += (np.arange(n_fields, dtype=np.int64) * per)[None, :]
    y = r.integers(0, 2, size=n_rows) if binary_target else r.standard_normal(n_rows)
    return _fields_to_data(cols, np.asarray(y, dtype=np.float32), n_features)


def ragged(n_rows: int, num_feature: int, max_nnz: int, seed: int, empty_frac: float = 0.1,
           repeat_ids: bool = True, real_values: bool = True) -> Data:
    """Edge-case generator: empty rows, ragged lengths, non-unit x, repeated ids in a row."""
    r = np.random.default_rng(seed)
    lens = r.integers(0 if empty_frac > 0 else 1, max_nnz + 1, size=n_rows)
    lens[r.random(n_rows) < empty_frac] = 0
    row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
    row_ptr[1:] = np.cumsum(lens)
    nnz = int(row_ptr[-1])
    col = r.integers(0, num_feature, size=nnz).astype(np.uint32)
    if repeat_ids and nnz > 1:
        # force some rows to repeat an id (v re-read at update time, fm_sgd.h:44-50)
        for row in r.choice(n_rows, size=max(1, n_rows // 8), replace=False):
            a, b = int(row_ptr[row]), int(row_ptr[row + 1])
            if b - a >= 2:
                col[a + 1] = col[a]
    val = (r.standard_normal(nnz) if real_values else np.ones(nnz)).astype(np.float32)
    y = r.integers(1, 6, size=n_rows).astype(np.float32)
    return Data(row_ptr, col, val, y, num_feature)


def long_rows(n_rows: int, num_feature: int, max_nnz: int, seed: int, zipf: float = 0.0, twice: float = 0.05,
              thrice: float = 0.05) -> Data:
    """Long-row generator: 0 .. max_nnz entries (5 % of the rows empty), x in [0.5, 1.5], y in 1..5.  A
    fraction `twice` of the rows names its first feature again at a later entry, a fraction `thrice` at two later
    entries.  Ids are uniform, or Zipf(zipf) with feature 0 the hottest."""
    r = np.random.default_rng(seed)
    lens = r.integers(0, max_nnz + 1, size=n_rows)
    lens[r.random(n_rows) < 0.05] = 0
    row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
    row_ptr[1:] = np.cumsum(lens)
    nnz = int(row_ptr[-1])
    if zipf > 0:
        p = 1.0 / np.arange(1, num_feature + 1) ** zipf
        col = r.choice(num_feature, size=nnz, p=p / p.sum()).astype(np.uint32)
    else:
        col = r.integers(0, num_feature, size=nnz).astype(np.uint32)
    for times, frac in ((2, twice), (3, thrice)):
        for row in np.flatnonzero((lens >= times) & (r.random(n_rows) < frac)):
            a = int(row_ptr[row])
            col[a + r.choice(np.arange(1, lens[row]), size=times - 1, replace=False)] = col[a]
    val = r.uniform(0.5, 1.5, size=nnz).astype(np.float32)
    y = r.integers(1, 6, size=n_rows).astype(np.float32)
    return Data(row_ptr, col, val, y, num_feature)


def to_libfm_text(data: Data, path: str) -> None:
    """Write `target id:value ...` lines (the format Data::load parses)."""
    with open(path, "w") as f:
        rp = data.row_ptr
        for r in range(data.num_cases):
            a, b = int(rp[r]), int(rp[r + 1])
            f.write("%g" % data.target[r])
            for j in range(a, b):
                f.write(" %d:%g" % (data.col[j], data.val[j]))
            f.write("\n")
