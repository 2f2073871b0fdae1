"""Python mirror of the reference's interface for the SGD path, over the C ABI.

Names follow the reference so that the parity tests read like its own code:

  Data                ~ class Data               (reference src/libfm/src/Data.h:47-74)
  FmModel             ~ class fm_model           (src/fm_core/fm_model.h:36-66)
  FmLearnSgdElement   ~ class fm_learn_sgd_element (src/libfm/src/fm_learn_sgd_element.h,
                        fm_learn_sgd.h, fm_learn.h)

All compute happens in libfmb200.so on the GPU; this module only marshals
numpy buffers.  The compiled drop-in command line lives in host/ (C++).
"""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np

from . import _capi

TASK_REGRESSION = 0  # fm_learn.h:47
TASK_CLASSIFICATION = 1  # fm_learn.h:48
MODE_INORDER = 0
MODE_HOGWILD = 1
MODE_ORDERED = 2  # sequentially consistent, fp64, parallel over conflict-free runs (fm_ordered.cuh)


class FmError(RuntimeError):
    """The reference throws std::string / const char* (caught at libfm.cpp:436-440)."""


def _p(arr, typ):
    return arr.ctypes.data_as(C.POINTER(typ))


class Data:
    """Row-major sparse design matrix + targets (CSR, SoA)."""

    def __init__(self, row_ptr, col, val, target, num_feature=None):
        self.row_ptr = np.ascontiguousarray(row_ptr, dtype=np.uint64)
        self.col = np.ascontiguousarray(col, dtype=np.uint32)
        self.val = np.ascontiguousarray(val, dtype=np.float32)
        self.target = np.ascontiguousarray(target, dtype=np.float32)
        self.num_cases = int(self.row_ptr.shape[0] - 1)
        if num_feature is None:
            # Data.h:227-229: one more than the largest id seen
            num_feature = int(self.col.max()) + 1 if self.col.size else 0
        self.num_feature = int(num_feature)
        if self.target.size:
            self.min_target = float(self.target.min())  # Data.h:207-208
            self.max_target = float(self.target.max())
        else:
            self.min_target = float(np.finfo(np.float32).max)
            self.max_target = -float(np.finfo(np.float32).max)

    @property
    def num_values(self) -> int:
        return int(self.row_ptr[-1])

    def rows(self, lo, hi) -> "Data":
        """Row shard [lo, hi) -- the multi-GPU partition unit."""
        a, b = int(self.row_ptr[lo]), int(self.row_ptr[hi])
        return Data(self.row_ptr[lo:hi + 1] - self.row_ptr[lo], self.col[a:b], self.val[a:b],
                    self.target[lo:hi], self.num_feature)

    def binarize_targets(self) -> None:
        """libfm.cpp:302-303: classification targets become -1 / +1."""
        self.target = np.where(self.target <= 0.0, -1.0, 1.0).astype(np.float32)

    @staticmethod
    def load(filename: str) -> "Data":
        """libfm text format, as Data::load parses it (Data.h:180-290):
        `target id:value id:value ...`, blank lines and `#` lines skipped."""
        row_ptr = [0]
        col, val, target = [], [], []
        try:
            f = open(filename, "r")
        except OSError:
            raise FmError("unable to open " + filename)
        with f:
            for line in f:
                s = line.strip(" \t\r\n")
                if not s or s[0] == "#":
                    continue
                tok = s.split()
                try:
                    target.append(np.float32(tok[0]))
                    for t in tok[1:]:
                        if t[0] == "#":
                            break
                        i, v = t.split(":")
                        col.append(int(i))
                        val.append(np.float32(v))
                except (ValueError, IndexError):
                    raise FmError('cannot parse line "' + line.rstrip("\n") + '"')
                row_ptr.append(len(col))
        return Data(np.array(row_ptr, dtype=np.uint64), np.array(col, dtype=np.uint32),
                    np.array(val, dtype=np.float32), np.array(target, dtype=np.float32))


def pinned_copy(arr: np.ndarray) -> np.ndarray:
    """Copy `arr` into page-locked memory from fmb200_host_alloc (kept alive by the array)."""
    lib = _capi.load()
    p = C.c_void_p()
    if lib.fmb200_host_alloc(C.byref(p), arr.nbytes) != 0:
        raise FmError(lib.fmb200_last_error().decode())
    buf = (C.c_char * max(arr.nbytes, 1)).from_address(p.value)
    out = np.frombuffer(buf, dtype=arr.dtype, count=arr.size).reshape(arr.shape)
    out[...] = arr
    return out  # never freed explicitly: process-lifetime staging buffers


def _write_matrix(path: str, row_ptr, ids, vals, num_cols: int) -> None:
    """A sparse matrix in the binary format: file_header {uint id = 2, uint float_size = 4, uint64 num_values,
    uint num_rows, uint num_cols} (util/fmatrix.h:44-50) + per row {uint size; size x {uint id; float value}}."""
    row_ptr = np.asarray(row_ptr).astype(np.int64)
    n_rows, nnz = len(row_ptr) - 1, int(row_ptr[-1])
    words = np.empty(n_rows + 2 * nnz, dtype=np.uint32)
    head = np.arange(n_rows, dtype=np.int64) + 2 * row_ptr[:-1]
    words[head] = np.diff(row_ptr).astype(np.uint32)
    ent = np.ones(words.size, dtype=bool)
    ent[head] = False
    pairs = np.empty((nnz, 2), dtype=np.uint32)
    pairs[:, 0] = ids
    pairs[:, 1] = np.asarray(vals, dtype=np.float32).view(np.uint32)
    words[ent] = pairs.reshape(-1)
    with open(path, "wb") as f:
        f.write(np.array([2, 4], np.uint32).tobytes() + np.array([nnz], np.uint64).tobytes()
                + np.array([n_rows, num_cols], np.uint32).tobytes())
        f.write(words.tobytes())


def write_binary(data: Data, path_x: str, path_y: str) -> None:
    """`data` as the reference's convert tool writes it: <file>.x = the binary matrix of its rows (_write_matrix),
    <file>.y = {uint 1, uint 4, uint n} + float[n] (util/matrix.h:364-380)."""
    _write_matrix(path_x, data.row_ptr, data.col, data.val, data.num_feature)
    with open(path_y, "wb") as f:
        f.write(np.array([1, 4, data.num_cases], np.uint32).tobytes() + data.target.astype(np.float32).tobytes())


def write_transposed(data: Data, path_xt: str) -> None:
    """`data` as the reference's transpose tool writes <file>.xt: the binary matrix (_write_matrix) with one row per
    feature (num_rows = num_feature, num_cols = the case count).  Column j holds its (case, value) pairs in case
    order, a case's repeated id in entry order; an empty column is a row of size 0."""
    nf = int(data.num_feature)
    col = np.asarray(data.col, dtype=np.int64)
    if col.size and int(col.max()) >= nf:
        raise FmError("feature id %d is not below num_feature = %d" % (int(col.max()), nf))
    cases = np.repeat(np.arange(data.num_cases, dtype=np.uint32), np.diff(data.row_ptr.astype(np.int64)))
    order = np.argsort(col, kind="stable")
    row_ptr = np.concatenate([[0], np.cumsum(np.bincount(col, minlength=nf))])
    _write_matrix(path_xt, row_ptr, cases[order], np.asarray(data.val, dtype=np.float32)[order], data.num_cases)


class XtBlocks:
    """A data set streamed from its transposed file <file>.xt in the blocks the command line plans under
    -cache_size (read_xblocks: rows are features, ids are cases), for FmLearnSgdElement.mcmc_begin_xt.
    `slots`: the two device slots its blocks pass through.  `fetches` counts the blocks handed to the library.
    transposed=False reads a .x instead, in blocks of rows (cases), for FmLearnSgdElement.sgda_epoch_x."""

    def __init__(self, path_xt: str, target, cache_size: int, slots=(2, 4), transposed: bool = True):
        head = np.fromfile(path_xt, dtype=np.uint32, count=6)
        self.num_feature, self.num_cases = int(head[4]), int(head[5])
        if not transposed:
            self.num_cases, self.num_feature = self.num_feature, self.num_cases
        self.target = np.ascontiguousarray(target, dtype=np.float32)
        if self.target.size != self.num_cases:
            raise FmError("case count of %s and its targets differ" % path_xt)
        self.blocks = [(lo, hi, np.ascontiguousarray(w), np.ascontiguousarray(r))
                       for lo, hi, w, r in read_xblocks(path_xt, cache_size)]
        self.col_lo = np.array([b[0] for b in self.blocks] + [self.blocks[-1][1]], dtype=np.uint32)
        self.nnz = np.array([(b[2].size - (b[1] - b[0])) // 2 for b in self.blocks], dtype=np.uint64)
        self.slots = tuple(slots)
        self.fetches = 0

    @property
    def n_blocks(self) -> int:
        return len(self.blocks)

    def _struct(self):
        def fetch(user, b, words, sizes):
            try:
                blk = self.blocks[b]
                words[0] = blk[2].ctypes.data
                sizes[0] = blk[3].ctypes.data_as(C.POINTER(C.c_uint32))
                self.fetches += 1
                return 0
            except Exception:  # noqa: BLE001 - no exception may cross the C ABI
                return 1
        cb = (_capi.XT_FETCH(fetch), _capi.XT_RELEASE(lambda user, b: None))
        s = _capi.XtBlocksC(self.num_cases, _p(self.target, C.c_float), self.n_blocks, _p(self.col_lo, C.c_uint32),
                            _p(self.nnz, C.c_uint64), (C.c_int * 2)(*self.slots), None, cb[0], cb[1])
        return s, cb


def read_xblocks(path_x: str, cache_size: int):
    """The blocks the command line streams a .x file in under -cache_size: greedy in file order, each block's
    bytes at most cache_size // 2 (so two blocks fit), at least one row per block.  Yields
    (row_lo, row_hi, words, row_size): the block's uint32 words as the file stores them and its rows' sizes."""
    budget = cache_size // 2
    raw = np.fromfile(path_x, dtype=np.uint32)
    n_rows = int(raw[4])
    words = raw[6:]
    sizes = np.empty(n_rows, dtype=np.uint32)
    pos = 0
    for r in range(n_rows):
        sizes[r] = words[pos]
        pos += 1 + 2 * int(sizes[r])
    lo, pos, lo_pos, used = 0, 0, 0, 0
    for r in range(n_rows):
        b = 4 + 8 * int(sizes[r])
        if b > budget:
            raise FmError("row %d of %s takes %d bytes: -cache_size must be at least %d" % (r, path_x, b, 2 * b))
        if used + b > budget:
            yield lo, r, words[lo_pos:pos], sizes[lo:r]
            lo, lo_pos, used = r, pos, 0
        used += b
        pos += b // 4
    if n_rows > lo or n_rows == 0:
        yield lo, n_rows, words[lo_pos:pos], sizes[lo:n_rows]


def _read_matrix(path: str):
    """A whole binary sparse matrix (_write_matrix's format): (row_ptr, ids, vals, num_rows, num_cols, num_values)."""
    try:
        raw = np.fromfile(path, dtype=np.uint32)
    except OSError:
        raise FmError("unable to open " + path)
    if raw.size < 6 or raw[0] != 2 or raw[1] != 4:
        raise FmError(path + " is not a binary sparse matrix of 4-byte floats")
    nnz = int(raw[2]) | (int(raw[3]) << 32)
    n_rows, n_cols = int(raw[4]), int(raw[5])
    words = raw[6:]
    if words.size != n_rows + 2 * nnz:
        raise FmError("%s: %d words of rows, the header promises %d" % (path, words.size, n_rows + 2 * nnz))
    sizes = np.empty(n_rows, dtype=np.int64)
    pos = 0
    for r in range(n_rows):
        sizes[r] = words[pos]
        pos += 1 + 2 * int(sizes[r])
    row_ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    head = np.arange(n_rows, dtype=np.int64) + 2 * row_ptr[:-1].astype(np.int64)
    ent = np.ones(words.size, dtype=bool)
    ent[head] = False
    pairs = words[ent].reshape(-1, 2)
    return row_ptr, pairs[:, 0].copy(), pairs[:, 1].view(np.float32).copy(), n_rows, n_cols, nnz


def _read_groups(path: str, n: int) -> np.ndarray:
    """DataMetaInfo::loadGroupsFromFile (Data.h:84-96): n whitespace-separated group ids of a text file; a short
    file leaves the remaining ids in group 0, as DVector::load leaves its zero-initialised entries."""
    with open(path) as f:
        tok = f.read().split()
    g = np.zeros(n, dtype=np.uint32)
    vals = [int(t) for t in tok[:n]]
    g[:len(vals)] = vals
    return g


class RelationData:
    """relation.h RelationData with has_xt: one relation block read from <stem>.xt (rows = the block's features,
    ids = its rows) and the optional <stem>.groups.  attr_offset is set by join_meta (libfm.cpp:209-213)."""

    def __init__(self, col_ptr, row, val, num_cases: int, num_feature: int, attr_group=None):
        self.col_ptr = np.ascontiguousarray(col_ptr, dtype=np.uint64)
        self.row = np.ascontiguousarray(row, dtype=np.uint32)
        self.val = np.ascontiguousarray(val, dtype=np.float32)
        self.num_cases = int(num_cases)
        self.num_feature = int(num_feature)
        self.attr_group = (np.zeros(self.num_feature, np.uint32) if attr_group is None
                           else np.ascontiguousarray(attr_group, dtype=np.uint32))
        self.num_attr_groups = int(self.attr_group.max()) + 1 if self.attr_group.size else 0
        if attr_group is None:
            self.num_attr_groups = 1  # DataMetaInfo's constructor: one group
        self.attr_offset = 0

    @property
    def num_values(self) -> int:
        return int(self.col_ptr[-1])

    @staticmethod
    def load(stem: str) -> "RelationData":
        col_ptr, row, val, n_rows, n_cols, _ = _read_matrix(stem + ".xt")
        groups = _read_groups(stem + ".groups", n_rows) if os.path.exists(stem + ".groups") else None
        return RelationData(col_ptr, row, val, n_cols, n_rows, groups)


class RelationJoin:
    """relation.h RelationJoin: data_row_to_relation_row of one data set and the block it joins."""

    def __init__(self, rows, data: RelationData):
        self.rows = np.ascontiguousarray(rows, dtype=np.uint32)
        self.data = data

    @staticmethod
    def load(path: str, expected_rows: int, data: RelationData = None) -> "RelationJoin":
        """RelationJoin::load: binary when the file starts with {uint 1, uint 4} (DVector<uint>::saveToBinaryFile:
        + uint n + n uint32), else expected_rows whitespace-separated numbers."""
        try:
            raw = open(path, "rb").read()
        except OSError:
            raise FmError("unable to open " + path)
        head = np.frombuffer(raw[:12], dtype=np.uint32) if len(raw) >= 12 else np.zeros(0, np.uint32)
        if head.size == 3 and head[0] == 1 and head[1] == 4:
            rows = np.frombuffer(raw[12:12 + 4 * int(head[2])], dtype=np.uint32)
            if rows.size != int(head[2]):
                raise FmError("%s: %d of %d entries" % (path, rows.size, int(head[2])))
        else:
            tok = raw.split()
            if len(tok) < expected_rows:
                raise FmError("%s: %d of %d entries" % (path, len(tok), expected_rows))
            rows = np.array([int(t) for t in tok[:expected_rows]], dtype=np.uint32)
        if rows.size != expected_rows:
            raise FmError("%s has %d entries, the data set %d cases" % (path, rows.size, expected_rows))
        return RelationJoin(rows, data)


def join_meta(num_main: int, main_group, blocks):
    """The joined meta table of libfm.cpp:206-240: sets each block's attr_offset and returns
    (num_attribute, attr_group[num_attribute], attr_per_group[G]).  main_group: the -meta groups of the main
    table's num_main ids (None: one group)."""
    mg = np.zeros(num_main, np.uint32) if main_group is None else np.ascontiguousarray(main_group, dtype=np.uint32)
    G = 1 if main_group is None else (int(mg.max()) + 1 if mg.size else 0)
    n = num_main
    for b in blocks:
        b.attr_offset = n
        n += b.num_feature
    group = np.zeros(n, np.uint32)
    group[:num_main] = mg
    for b in blocks:
        group[b.attr_offset:b.attr_offset + b.num_feature] = G + b.attr_group
        G += b.num_attr_groups
    return n, group, np.bincount(group, minlength=G).astype(np.uint32)


class _LibcRand:
    """glibc srand()/rand(): the reference's only entropy source (random.h:172-174)."""

    def __init__(self):
        self.libc = C.CDLL(None)
        self.libc.rand.restype = C.c_int
        self.libc.srand.argtypes = [C.c_uint]

    def srand(self, seed: int) -> None:
        self.libc.srand(C.c_uint(seed & 0xFFFFFFFF))

    def uniform(self) -> float:
        return self.libc.rand() / (2147483647.0 + 1.0)

    def gaussian(self) -> float:
        # Leva's ratio-of-uniforms method, random.h:148-162
        while True:
            u = self.uniform()
            while u == 0.0:
                u = self.uniform()
            v = 1.7156 * (self.uniform() - 0.5)
            x = u - 0.449871
            y = abs(v) + 0.386595
            q = x * x + y * (0.19600 * y - 0.25472 * x)
            if q < 0.27597:
                break
            if not ((q > 0.27846) or ((v * v) > (-4.0 * u * u * math.log(u)))):
                break
        return v / u


class FmModel:
    """Host image of the FM parameters; v is factor-major [num_factor][num_attribute]."""

    def __init__(self, num_attribute: int, num_factor: int, k0: bool = True, k1: bool = True):
        self.num_attribute = int(num_attribute)
        self.num_factor = int(num_factor)
        self.k0, self.k1 = bool(k0), bool(k1)
        self.reg0 = self.regw = self.regv = 0.0
        self.init_mean = 0.0
        self.init_stdev = 0.01  # fm_model.h:72
        self.w0 = 0.0
        self.w = np.zeros(self.num_attribute, dtype=np.float64)
        self.v = np.zeros((self.num_factor, self.num_attribute), dtype=np.float64)

    def init(self, seed: int | None = None) -> None:
        """fm_model::init (fm_model.h:91-99): w0 = 0, w = 0, v ~ N(mean, stdev) drawn
        factor-outer / attribute-inner from libc rand() (matrix.h:398-404)."""
        rng = _LibcRand()
        if seed is not None:
            rng.srand(seed)  # libfm.cpp:115-116
        self.w0 = 0.0
        self.w[:] = 0.0
        if self.init_stdev == 0.0 or math.isnan(self.init_stdev):
            self.v[:] = self.init_mean
            return
        flat = self.v.reshape(-1)
        for i in range(flat.shape[0]):
            flat[i] = self.init_mean + self.init_stdev * rng.gaussian()

    def init_numpy(self, seed: int) -> None:
        """Fast non-reference init for large synthetic benchmarks."""
        r = np.random.default_rng(seed)
        self.w0 = 0.0
        self.w[:] = 0.0
        self.v[:] = self.init_mean + self.init_stdev * r.standard_normal(self.v.shape)

    def saveModel(self, path: str) -> None:
        """fm_model::saveModel text layout (fm_model.h:132-154), %g-style numbers."""
        def g(x):
            return "%g" % x
        with open(path, "w") as f:
            if self.k0:
                f.write("#global bias W0\n" + g(self.w0) + "\n")
            if self.k1:
                f.write("#unary interactions Wj\n")
                for i in range(self.num_attribute):
                    f.write(g(self.w[i]) + "\n")
            f.write("#pairwise interactions Vj,f\n")
            for i in range(self.num_attribute):
                f.write(" ".join(g(self.v[q, i]) for q in range(self.num_factor)) + "\n")


class FmLearnSgdElement:
    """fm_learn_sgd_element on an H100: one libfmb200 context (one GPU)."""

    def __init__(self, fm: FmModel, device: int = 0, mode: int = MODE_HOGWILD):
        self.lib = _capi.load()
        self.fm = fm
        self.task = TASK_REGRESSION
        self.learn_rate = 0.0
        self.num_iter = 100  # libfm.cpp:274
        self.min_target = 0.0
        self.max_target = 0.0
        self.mode = mode
        self._ctx = C.c_void_p()
        self._check(self.lib.fmb200_create(C.byref(self._ctx), device, fm.num_attribute,
                                           fm.num_factor, int(fm.k0), int(fm.k1)))
        self._check(self.lib.fmb200_set_mode(self._ctx, mode))
        self._slots = {}
        self.push_params()

    # -- plumbing ---------------------------------------------------------
    def _check(self, rc: int) -> None:
        if rc != 0:
            raise FmError(self.lib.fmb200_last_error().decode())

    def close(self) -> None:
        if self._ctx:
            self.lib.fmb200_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_mode(self, mode: int) -> None:
        self._check(self.lib.fmb200_set_mode(self._ctx, mode))
        self.mode = mode

    def set_tuning(self, ctas_per_sm=0, rows_per_tile=0, threads=0, damp=0, variant=0) -> None:
        self._check(self.lib.fmb200_set_tuning(self._ctx, ctas_per_sm, rows_per_tile, threads, damp,
                                               variant))

    def set_reproducible(self, on=True, tile_rows=0, window_tiles=0) -> None:
        """HOGWILD SGD epochs as windows of tile_rows x window_tiles rows (0: 256 and 64): the same bits on every run
        and grid (include/fmb200.h, fmb200_set_reproducible)."""
        self._check(self.lib.fmb200_set_reproducible(self._ctx, int(bool(on)), tile_rows, window_tiles))

    def push_hparams(self) -> None:
        self._check(self.lib.fmb200_set_hparams(self._ctx, self.task, self.learn_rate, self.fm.reg0,
                                                self.fm.regw, self.fm.regv, self.min_target,
                                                self.max_target))

    def push_params(self) -> None:
        fm = self.fm
        w = np.ascontiguousarray(fm.w, dtype=np.float64)
        v = np.ascontiguousarray(fm.v, dtype=np.float64)
        self._check(self.lib.fmb200_set_params(self._ctx, float(fm.w0), _p(w, C.c_double),
                                               _p(v, C.c_double)))

    def pull_params(self) -> None:
        fm = self.fm
        w0 = C.c_double()
        w = np.empty(fm.num_attribute, dtype=np.float64)
        v = np.empty((fm.num_factor, fm.num_attribute), dtype=np.float64)
        self._check(self.lib.fmb200_get_params(self._ctx, C.byref(w0), _p(w, C.c_double),
                                               _p(v, C.c_double)))
        fm.w0, fm.w, fm.v = w0.value, w, v

    def upload(self, data: Data, slot: int) -> None:
        self._check(self.lib.fmb200_upload_data(
            self._ctx, slot, data.num_cases, data.num_values, _p(data.row_ptr, C.c_uint64),
            _p(data.col, C.c_uint32), _p(data.val, C.c_float), _p(data.target, C.c_float)))
        # the Data object is kept alive with its slot: id() values are reused after garbage
        # collection, and a recycled id must never map to a stale upload
        for key in [k for k, (s, _) in self._slots.items() if s == slot]:
            del self._slots[key]
        self._slots[id(data)] = (slot, data)

    def upload_onehot(self, data: Data, slot: int) -> None:
        """fmb200_upload_onehot: ids + targets only (rows of a fixed width, every value 1)."""
        z = data.num_values // max(data.num_cases, 1)
        if data.num_values != z * data.num_cases or not np.all(data.val == 1.0) or \
                not np.array_equal(data.row_ptr, np.arange(data.num_cases + 1, dtype=np.uint64) * np.uint64(z)):
            raise FmError("upload_onehot needs fixed-width rows with every value 1")
        self._check(self.lib.fmb200_upload_onehot(self._ctx, slot, data.num_cases, z,
                                                  _p(data.col, C.c_uint32), _p(data.target, C.c_float)))
        for key in [k for k, (s, _) in self._slots.items() if s == slot]:
            del self._slots[key]
        self._slots[id(data)] = (slot, data)

    def upload_aos(self, data: Data, slot: int, contiguous: bool = True) -> None:
        """fmb200_upload_data_aos from a host image of the reference's containers
        (sparse_row[] pointing into sparse_entry[]; util/fmatrix.h:34-42)."""
        ent = np.empty(max(data.num_values, 1), dtype=[("id", np.uint32), ("value", np.float32)])
        ent["id"][:data.num_values] = data.col
        ent["value"][:data.num_values] = data.val
        rows = np.zeros(max(data.num_cases, 1), dtype=[("data", np.uint64), ("size", np.uint32), ("pad", np.uint32)])
        sizes = np.diff(data.row_ptr.astype(np.int64)).astype(np.uint32)
        keep = [ent]
        if contiguous:
            rows["data"][:data.num_cases] = ent.ctypes.data + 8 * data.row_ptr[:-1]
        else:  # every row in its own allocation, as a loader without the block would do
            for r in range(data.num_cases):
                a, b = int(data.row_ptr[r]), int(data.row_ptr[r + 1])
                part = ent[a:b].copy()
                keep.append(part)
                rows["data"][r] = part.ctypes.data
        rows["size"][:data.num_cases] = sizes
        self._check(self.lib.fmb200_upload_data_aos(self._ctx, slot, data.num_cases,
                                                    rows.ctypes.data_as(C.c_void_p), _p(data.target, C.c_float)))
        del keep
        for key in [k for k, (s, _) in self._slots.items() if s == slot]:
            del self._slots[key]
        self._slots[id(data)] = (slot, data)

    def upload_xblock(self, words: np.ndarray, row_size: np.ndarray, target: np.ndarray, slot: int,
                      asynchronous: bool = False) -> None:
        """fmb200_upload_xblock(_async): rows of a .x file as the file stores them (read_xblocks) into `slot`.
        The asynchronous form needs the arrays alive until the slot is next used."""
        words = np.ascontiguousarray(words, dtype=np.uint32)
        row_size = np.ascontiguousarray(row_size, dtype=np.uint32)
        target = np.ascontiguousarray(target, dtype=np.float32)
        nnz = (words.size - row_size.size) // 2
        fn = self.lib.fmb200_upload_xblock_async if asynchronous else self.lib.fmb200_upload_xblock
        self._check(fn(self._ctx, slot, row_size.size, nnz, words.ctypes.data_as(C.c_void_p),
                       _p(row_size, C.c_uint32), _p(target, C.c_float)))
        for key in [k for k, (s, _) in self._slots.items() if s == slot]:
            del self._slots[key]

    def release(self, data: Data) -> None:
        """Free the device copy of `data` and its slot."""
        ent = self._slots.pop(id(data), None)
        if ent is not None:
            self._check(self.lib.fmb200_free_data(self._ctx, ent[0]))

    def _slot_of(self, data: Data) -> int:
        if id(data) not in self._slots:
            used = {s for s, _ in self._slots.values()}
            free = [s for s in range(8) if s not in used]
            if not free:
                raise FmError("all 8 data slots are in use: release() one first")
            self.upload(data, free[0])
        return self._slots[id(data)][0]

    # -- the reference's learner surface -----------------------------------
    def sgd_epoch(self, train: Data) -> float:
        """One pass of the row loop, fm_learn_sgd_element.h:56-67.  Returns device seconds."""
        sec = C.c_double()
        self._check(self.lib.fmb200_sgd_epoch(self._ctx, self._slot_of(train), C.byref(sec)))
        return sec.value

    def evaluate(self, data: Data) -> float:
        """fm_learn::evaluate (fm_learn.h:93-153): RMSE or accuracy."""
        sq, ab, ok = C.c_double(), C.c_double(), C.c_uint64()
        self._check(self.lib.fmb200_evaluate(self._ctx, self._slot_of(data), C.byref(sq),
                                             C.byref(ab), C.byref(ok)))
        self.last_mae = ab.value / max(1, data.num_cases)
        if self.task == TASK_REGRESSION:
            return math.sqrt(sq.value / data.num_cases)
        return ok.value / data.num_cases

    def predict(self, data: Data, transform: bool = True) -> np.ndarray:
        """fm_learn_sgd::predict (fm_learn_sgd.h:76-90)."""
        out = np.empty(data.num_cases, dtype=np.float64)
        self._check(self.lib.fmb200_predict(self._ctx, self._slot_of(data), int(transform),
                                            _p(out, C.c_double)))
        return out

    # -- SGDA: fm_learn_sgd_element_adapt_reg ----------------------------------
    def sgda_begin(self, attr_group=None) -> None:
        if attr_group is None:
            self._sgda_groups = 1
            self._check(self.lib.fmb200_sgda_begin(self._ctx, 1, None))
        else:
            g = np.ascontiguousarray(attr_group, dtype=np.uint32)
            self._sgda_groups = int(g.max()) + 1
            self._check(self.lib.fmb200_sgda_begin(self._ctx, self._sgda_groups, _p(g, C.c_uint32)))

    def sgda_epoch(self, train: Data, validation: Data, lambda_steps: bool) -> float:
        sec = C.c_double()
        self._check(self.lib.fmb200_sgda_epoch(self._ctx, self._slot_of(train), self._slot_of(validation),
                                               int(lambda_steps), C.byref(sec)))
        return sec.value

    def sgda_epoch_x(self, train, validation, lambda_steps: bool) -> float:
        """fmb200_sgda_epoch_x: as sgda_epoch, each of train / validation either a Data (resident in a slot) or an
        XtBlocks over its .x (transposed=False; streamed in its blocks).  Returns device seconds."""
        keep, args = [], []
        for d in (train, validation):
            if isinstance(d, XtBlocks):
                st, cb = d._struct()
                keep.append((st, cb))
                args += [-1, C.pointer(st)]
            else:
                args += [self._slot_of(d), None]
        sec = C.c_double()
        self._check(self.lib.fmb200_sgda_epoch_x(self._ctx, *args, int(lambda_steps), C.byref(sec)))
        return sec.value

    def sgda_reg(self):
        reg_w = np.zeros(self._sgda_groups)
        reg_v = np.zeros((self._sgda_groups, self.fm.num_factor))
        self._check(self.lib.fmb200_sgda_get_reg(self._ctx, _p(reg_w, C.c_double), _p(reg_v, C.c_double)))
        return reg_w, reg_v

    def sgda_moments(self):
        """var_w and var_v[k] of the last epoch's last update_means (fm_learn_sgd_element_adapt_reg.h:250-274),
        the wvar / vvar<f> columns of the reference's rlog (its wmean / vmean<f> are always 0)."""
        var_w = C.c_double()
        var_v = np.zeros(self.fm.num_factor)
        self._check(self.lib.fmb200_sgda_get_moments(self._ctx, C.byref(var_w), _p(var_v, C.c_double)))
        return var_w.value, var_v

    def mcmc_eterms(self, data: Data) -> np.ndarray:
        """fm_learn_mcmc::predict_data_and_write_to_eterms (fm_learn_mcmc.h:148-378) for one data set."""
        out = np.empty(data.num_cases, dtype=np.float64)
        self._check(self.lib.fmb200_mcmc_eterms(self._ctx, self._slot_of(data), _p(out, C.c_double)))
        return out

    # -- MCMC / ALS: fm_learn_mcmc_simultaneous ---------------------------------
    def mcmc_begin(self, train: Data, test: Data, do_sample: bool, do_multilevel: bool, reg0: float,
                   w_lambda, v_lambda, attr_group=None, attr_per_group=None, relations=None,
                   main_group=None) -> None:
        """fm_learn_mcmc::init + the prologue of _learn.  w_lambda [G], v_lambda [G][k] as -regular sets
        them (libfm.cpp:326-364); attr_group / attr_per_group as DataMetaInfo holds them (None: one group).
        relations: [(RelationData, train RelationJoin, test RelationJoin), ...] (libfm.cpp:175-198): the block
        attr_offsets and, when attr_group is None, the groups come from join_meta over the main table's ids and
        main_group, the -meta groups of those ids (None: one group)."""
        if relations:
            n_main = self.fm.num_attribute - sum(b.num_feature for b, _, _ in relations)
            n, grp, per = join_meta(n_main, main_group, [b for b, _, _ in relations])
            if attr_group is None:
                attr_group, attr_per_group = grp, per
            self.mcmc_set_relations(train, test, relations)
        self.push_hparams()
        wl = np.ascontiguousarray(w_lambda, dtype=np.float64)
        self._mcmc_groups = int(wl.shape[0])
        vl = np.ascontiguousarray(v_lambda, dtype=np.float64).reshape(self._mcmc_groups, self.fm.num_factor)
        g = None if attr_group is None else np.ascontiguousarray(attr_group, dtype=np.uint32)
        pg = None if attr_per_group is None else np.ascontiguousarray(attr_per_group, dtype=np.uint32)
        self._check(self.lib.fmb200_mcmc_begin(
            self._ctx, self._slot_of(train), self._slot_of(test), int(do_sample), int(do_multilevel),
            self._mcmc_groups, None if g is None else _p(g, C.c_uint32), None if pg is None else _p(pg, C.c_uint32),
            float(reg0), _p(wl, C.c_double), _p(vl, C.c_double)))

    def mcmc_set_relations(self, train: Data, test: Data, relations) -> None:
        """fmb200_mcmc_set_relations: relations = [(RelationData, train RelationJoin, test RelationJoin), ...], each
        block's attr_offset set (join_meta); [] withdraws them."""
        self._rel_keep = []
        arr = (_capi.RelationC * max(len(relations), 1))()
        for i, (b, jtr, jte) in enumerate(relations):
            keep = (b.col_ptr, b.row, b.val, jtr.rows, jte.rows)
            self._rel_keep.append(keep)
            arr[i] = _capi.RelationC(b.num_cases, b.num_feature, b.attr_offset, _p(keep[0], C.c_uint64),
                                     _p(keep[1], C.c_uint32), _p(keep[2], C.c_float), keep[3].size, keep[4].size,
                                     _p(keep[3], C.c_uint32), _p(keep[4], C.c_uint32))
        self._check(self.lib.fmb200_mcmc_set_relations(self._ctx, self._slot_of(train), self._slot_of(test),
                                                        len(relations), arr))

    def mcmc_begin_xt(self, train, test, do_sample: bool, do_multilevel: bool, reg0: float, w_lambda, v_lambda,
                      attr_group=None, attr_per_group=None) -> None:
        """fmb200_mcmc_begin_xt: as mcmc_begin, each of train / test either a Data (resident in a slot) or an
        XtBlocks (streamed from its .xt on every pass)."""
        self.push_hparams()
        wl = np.ascontiguousarray(w_lambda, dtype=np.float64)
        self._mcmc_groups = int(wl.shape[0])
        vl = np.ascontiguousarray(v_lambda, dtype=np.float64).reshape(self._mcmc_groups, self.fm.num_factor)
        g = None if attr_group is None else np.ascontiguousarray(attr_group, dtype=np.uint32)
        pg = None if attr_per_group is None else np.ascontiguousarray(attr_per_group, dtype=np.uint32)
        self._xt_keep = []  # the structs and callbacks live as long as the learner's MCMC state
        args = []
        for d in (train, test):
            if isinstance(d, XtBlocks):
                st, cb = d._struct()
                self._xt_keep.append((d, st, cb))
                args += [-1, C.pointer(st)]
            else:
                args += [self._slot_of(d), None]
        self._check(self.lib.fmb200_mcmc_begin_xt(
            self._ctx, *args, int(do_sample), int(do_multilevel), self._mcmc_groups,
            None if g is None else _p(g, C.c_uint32), None if pg is None else _p(pg, C.c_uint32),
            float(reg0), _p(wl, C.c_double), _p(vl, C.c_double)))

    def mcmc_iteration(self):
        """One iteration of fm_learn_mcmc_simultaneous::_learn; returns (train metric, counters[16])."""
        m = C.c_double()
        cnt = np.zeros(16, dtype=np.uint32)
        self._check(self.lib.fmb200_mcmc_iteration(self._ctx, C.byref(m), _p(cnt, C.c_uint32)))
        return m.value, cnt

    def mcmc_hyper(self) -> dict:
        G, k = self._mcmc_groups, self.fm.num_factor
        alpha = C.c_double()
        out = {"w_mu": np.zeros(G), "w_lambda": np.zeros(G), "v_mu": np.zeros((G, k)), "v_lambda": np.zeros((G, k))}
        self._check(self.lib.fmb200_mcmc_get_hyper(self._ctx, C.byref(alpha), *[_p(out[n], C.c_double) for n in
                                                                               ("w_mu", "w_lambda", "v_mu", "v_lambda")]))
        out["alpha"] = alpha.value
        return out

    def mcmc_pred(self, test: Data):
        """(pred_this, pred_sum_all, pred_sum_all_but5) over the test set."""
        out = [np.zeros(test.num_cases) for _ in range(3)]
        self._check(self.lib.fmb200_mcmc_get_pred(self._ctx, *[_p(a, C.c_double) for a in out]))
        return tuple(out)

    def mcmc_runs(self) -> int:
        n = C.c_uint32()
        self._check(self.lib.fmb200_mcmc_runs(self._ctx, C.byref(n)))
        return n.value

    def learn(self, train: Data, test: Data, log=None):
        """fm_learn_sgd_element::learn (fm_learn_sgd_element.h:48-78)."""
        self.push_hparams()
        hist = []
        for i in range(self.num_iter):
            t = self.sgd_epoch(train)
            tr, te = self.evaluate(train), self.evaluate(test)
            hist.append((tr, te, t))
            if log is not None:
                log("#Iter=%3d\tTrain=%g\tTest=%g" % (i, tr, te))
        self.pull_params()
        return hist

    # -- extras for bench / multi-GPU ---------------------------------------
    def params_device(self):
        ptr, n = C.c_void_p(), C.c_uint64()
        self._check(self.lib.fmb200_params_device(self._ctx, C.byref(ptr), C.byref(n)))
        return ptr.value, n.value

    def params_layout(self) -> dict:
        off_w, off_v, ws, kp = C.c_uint64(), C.c_uint64(), C.c_int(), C.c_int()
        self._check(self.lib.fmb200_params_layout(self._ctx, C.byref(off_w), C.byref(ws), C.byref(off_v), C.byref(kp)))
        return {"off_w": off_w.value, "ws": ws.value, "off_v": off_v.value, "kp": kp.value,
                "n": self.fm.num_attribute}

    def stream(self) -> int:
        s = C.c_void_p()
        self._check(self.lib.fmb200_stream(self._ctx, C.byref(s)))
        return s.value or 0

    def kernel_launches(self) -> int:
        n = C.c_uint64()
        self._check(self.lib.fmb200_kernel_launches(self._ctx, C.byref(n)))
        return n.value

    def download(self, slot: int) -> Data:
        """The device CSR of a slot, copied back (tests of the upload paths)."""
        nr, nz = C.c_uint64(), C.c_uint64()
        self._check(self.lib.fmb200_download_data(self._ctx, slot, C.byref(nr), C.byref(nz), None, None, None, None))
        rp = np.zeros(nr.value + 1, dtype=np.uint64)
        col = np.zeros(max(nz.value, 1), dtype=np.uint32)
        val = np.zeros(max(nz.value, 1), dtype=np.float32)
        tg = np.zeros(max(nr.value, 1), dtype=np.float32)
        self._check(self.lib.fmb200_download_data(self._ctx, slot, None, None, _p(rp, C.c_uint64),
                                                  _p(col, C.c_uint32), _p(val, C.c_float), _p(tg, C.c_float)))
        return Data(rp, col[:nz.value], val[:nz.value], tg[:nr.value], 0)

    def ordered_index(self, data: Data):
        """(link, rowdep) of fm_ordered.cu for `data` (tests)."""
        link = np.empty(max(data.num_values, 1), dtype=np.uint32)
        rowdep = np.empty(max(data.num_cases, 1), dtype=np.uint32)
        self._check(self.lib.fmb200_ordered_index(self._ctx, self._slot_of(data), _p(link, C.c_uint32),
                                                  _p(rowdep, C.c_uint32)))
        return link[:data.num_values], rowdep[:data.num_cases]

    def epoch_config(self) -> dict:
        v = [C.c_int() for _ in range(7)]
        self._check(self.lib.fmb200_last_epoch_config(self._ctx, *[C.byref(x) for x in v]))
        keys = ["lanes_per_row", "slots", "rows_per_tile", "grid", "block", "smem_bytes", "damp"]
        return dict(zip(keys, [x.value for x in v]))

    def epoch_dealt(self) -> bool:
        """Whether the last epoch ran the row-lane dealt schedule (rows dealt to CTAs by their last id)."""
        v = C.c_int()
        self._check(self.lib.fmb200_last_epoch_dealt(self._ctx, C.byref(v)))
        return bool(v.value)
