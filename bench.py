#!/usr/bin/env python
"""bench.py -- throughput measurement of the libFM SGD hot path.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl reference] [--dump-outputs DIR]

Workload (BASELINE.json configs[1], the configuration `metric` is quoted on):
SGD, k=8, MovieLens-1M-shaped CSR (6040 users x 3706 items, 1,000,209 rows,
2 nnz/row, value 1), regression, lr 0.01, init_stdev 0.1.  A "step" is one pass
of the hot path over the whole data set = one SGD epoch = one fmb200_sgd_epoch
(plus, for N > 1, the per-epoch exchange of w0|w|V).  Weak scaling: every rank owns a full C2-sized row shard.

value  : examples/s with inputs resident in HBM, CUDA events on the library's own
         stream, L2 flushed (256 MiB write) before every timed step, max over ranks.
e2e    : examples/s through the C ABI with HOST (pinned) buffers: every step uploads
         the data set (fmb200_upload_onehot_async: ids + targets, 12 B/row for this one-hot
         shape; two device slots so the copy of the next step overlaps this step's epoch),
         runs the epoch and reads the model back (fmb200_get_params); wall clock.
parity : RMSE trajectory of the timed mode against the sequential oracle on a planted-signal
         C2-shaped set from the same initial model (N == 1).
tolerance_mode : the same workload in FMB200_MODE_ORDERED (sequentially consistent, fp64, inside
         the 1e-5 RMSE gate): examples/s device-timed and end to end, and its parity numbers.
dump   : --dump-outputs DIR writes the model the timed path left after its last timed step, as a caller of
         fmb200_get_params receives it: DIR/w0.npy, DIR/w.npy, DIR/v.npy (float64, v factor-major [k][n]).
         Data and initial model are seeded and the C2 epoch is reproducible, so runs with the same arguments
         write the same values.
extra  : BASELINE configs C3 (k=64, 39 nnz/row, 1M features, 10M rows), C2 with Zipf(1) ids and C4 (the MCMC
         e-term pass, k=16, ML-10M shape), each with its own roofline object (N == 1; --no-extras skips them).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "MovieLens-1M-shaped examples/sec at k=8, SGD"
UNIT = "examples/s"
K_FACTORS = 8
LEARN_RATE = 0.01
WORKLOAD = {
    "workload": "C2: libFM SGD epoch, k=8, MovieLens-1M-shaped CSR (6040 users x 3706 items, "
                "1000209 rows, 2 nnz/row, x=1), -task r -learn_rate 0.01 -init_stdev 0.1",
    "rows_per_gpu": 1_000_209, "k": K_FACTORS, "nnz_per_row": 2, "mode": "hogwild",
    "l2": "flushed before every timed step (256 MiB write)",
}


def env_int(name, default):
    try:
        return int(os.environ.get(name, default))
    except ValueError:
        return default


# --------------------------------------------------------------------------
# reference arm / cpu baseline: the reference's own CPU implementation
# --------------------------------------------------------------------------
def cpu_reference_epochs(data, n_epochs):
    """Time the row loop of fm_learn_sgd_element::learn on the host.

    Uses oracle/_ref (the unmodified reference compiled in place) when present,
    else the C restatement.  Returns (examples_per_sec, kind, per_epoch_seconds).
    The reference is single-threaded, so cores == 1 is all it can use."""
    import numpy as np
    import oracle
    n = data.num_feature
    if oracle.have_ref():
        ref = oracle.Ref(n, K_FACTORS, seed=42, init_stdev=0.1)
        # time_learn = the reference's own user-CPU clock around the row loop
        # (fm_learn_sgd_element.h:55,68); evaluate passes are outside it
        tiny = data.rows(0, 1)
        _, _, tm = ref.learn(data, tiny, 0, LEARN_RATE, n_epochs, data.min_target, data.max_target)
        secs = [float(t) for t in tm]
        kind = "reference"
    else:
        port = oracle.Port(n, K_FACTORS)
        port.init(42, 0.0, 0.1)
        secs = []
        for _ in range(n_epochs):
            t0 = time.process_time()
            port.sgd_epoch(data, 0, LEARN_RATE, data.min_target, data.max_target)
            secs.append(time.process_time() - t0)
        kind = "port"
    best = statistics.median(secs)
    return data.num_cases / best, kind, secs


def run_reference_arm(args):
    rank = env_int("RANK", 0)
    if rank != 0:
        return 0  # the reference has no multi-process path: rank 0 alone measures
    from libfm_b200 import synth
    data = synth.movielens_1m_shaped(seed=7)
    n_ep = args.warmup + args.steps
    t0 = time.time()
    ex_s, kind, secs = cpu_reference_epochs(data, n_ep)
    timed = secs[args.warmup:]
    ms = 1e3 * sum(timed) / len(timed)
    value = data.num_cases / (ms * 1e-3)
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
        "config": dict(WORKLOAD, mode="reference CPU, in-order"),
        "cpu_baseline": {"value": value, "unit": UNIT, "cores": 1, "kind": kind,
                         "sample": "%d full epochs of the 1000209-row workload, the reference's own "
                                   "time_learn (user CPU s around the row loop)" % len(timed)},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0, "wall_s": time.time() - t0,
    }
    print(json.dumps(line), flush=True)
    return 0


# --------------------------------------------------------------------------
# clocks: NVML sampling thread
# --------------------------------------------------------------------------
class ClockSampler(threading.Thread):
    REASONS = {0x2: "applications_clocks_setting", 0x4: "sw_power_cap", 0x8: "hw_slowdown",
               0x10: "sync_boost", 0x20: "sw_thermal_slowdown", 0x40: "hw_thermal_slowdown",
               0x80: "hw_power_brake_slowdown", 0x100: "display_clock_setting"}

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.samples, self.reasons, self.stop_flag = index, [], set(), False
        self.max_mhz = None
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)
        except Exception:
            self.nv = None

    def sample(self):
        if not self.nv:
            return
        try:
            self.samples.append(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM))
            bits = self.nv.nvmlDeviceGetCurrentClocksEventReasons(self.h) \
                if hasattr(self.nv, "nvmlDeviceGetCurrentClocksEventReasons") \
                else self.nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
            for b, name in self.REASONS.items():
                if bits & b:
                    self.reasons.add(name)
        except Exception:
            pass

    def run(self):
        while not self.stop_flag:
            self.sample()
            time.sleep(0.01)

    def summary(self):
        return {"sm_mhz": statistics.median(self.samples) if self.samples else None,
                "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons),
                "samples": len(self.samples)}


class _DevBuf:
    """Expose a raw device pointer to torch through the CUDA array interface."""

    def __init__(self, ptr, n_floats):
        self.__cuda_array_interface__ = {"shape": (n_floats,), "typestr": "<f4",
                                         "data": (ptr, False), "version": 2}


# --------------------------------------------------------------------------
# parity of a mode against the sequential oracle (planted-signal C2 shape)
# --------------------------------------------------------------------------
def parity_run(mode, device, epochs=5, tuning=None):
    """RMSE per epoch (train, held-out) of `mode` and of the oracle from the same initial model."""
    import numpy as np
    from libfm_b200 import FmLearnSgdElement, FmModel, synth
    from oracle import Port
    tr, te = synth.movielens_1m_planted(100_000, seed=7)
    n = tr.num_feature
    v0 = np.random.default_rng(42).standard_normal((K_FACTORS, n)) * 0.1
    port = Port(n, K_FACTORS)
    port.set_params(0.0, np.zeros(n), v0)
    fm = FmModel(n, K_FACTORS)
    fm.v = v0.copy()
    l = FmLearnSgdElement(fm, device=device, mode=mode)
    l.task, l.learn_rate = 0, LEARN_RATE
    l.min_target, l.max_target = tr.min_target, tr.max_target
    l.push_hparams()
    if tuning:
        l.set_tuning(*tuning)
    gpu, ref = [], []
    for _ in range(epochs):
        l.sgd_epoch(tr)
        port.sgd_epoch(tr, 0, LEARN_RATE, tr.min_target, tr.max_target)
        gpu.append([l.evaluate(tr), l.evaluate(te)])
        ref.append([port.metric(tr, 0, tr.min_target, tr.max_target),
                    port.metric(te, 0, tr.min_target, tr.max_target)])
    l.close()
    gap = max(max(abs(g[0] - r[0]), abs(g[1] - r[1])) for g, r in zip(gpu, ref))
    return {"data": "C2-shaped, planted rank-4 signal + noise, 1000209 train / 100000 held-out rows",
            "epochs": epochs, "rmse_gpu": gpu, "rmse_ref": ref, "max_abs_gap": gap,
            "oracle": "oracle/fm_oracle.c (pinned bit-exact to the reference)", "tolerance_north_star": 1e-5}


def timed_epochs(lrn, data, steps, warmup, flush, stream, torch):
    """CUDA-event time per epoch on the library's stream, L2 flushed before every step."""
    lib, ctx = lrn.lib, lrn._ctx
    slot = lrn._slot_of(data)
    with torch.cuda.stream(stream):
        for _ in range(warmup):
            flush.zero_()
            if lib.fmb200_sgd_epoch_async(ctx, slot) != 0:
                raise RuntimeError(lib.fmb200_last_error().decode())
        torch.cuda.synchronize()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for a, b in ev:
            flush.zero_()
            a.record(stream)
            if lib.fmb200_sgd_epoch_async(ctx, slot) != 0:
                raise RuntimeError(lib.fmb200_last_error().decode())
            b.record(stream)
        torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in ev]
    return sum(ms) / len(ms)


def hbm_peak():
    return 3350.0, "H100 SXM data sheet (HBM3, 3.35 TB/s)"


def kernel_name(cfg, mode):
    if mode == "ordered":
        ncompute = cfg["lanes_per_row"] * cfg["slots"]
        if cfg["block"] > ncompute:
            return "fm_sgd_ordered_ws_kernel<GL=%d> (1 CTA: %d compute threads + %d parked / helper threads)" % (
                cfg["lanes_per_row"], ncompute, cfg["block"] - ncompute)
        return "fm_sgd_ordered_kernel<GL=%d> (1 CTA x %d threads)" % (cfg["lanes_per_row"], cfg["block"])
    if cfg["lanes_per_row"] == 1:
        return "fm_sgd_rowlane_kernel<GP=%d,Z=%d,DAMP=%d> (grid %d x %d)" % (
            2 if K_FACTORS > 4 else 1, cfg["slots"], cfg["damp"], cfg["grid"], cfg["block"])
    return "fm_sgd_hogwild_kernel<G=%d,S=%d,DAMP=%d> (grid %d x %d)" % (
        cfg["lanes_per_row"], cfg["slots"], cfg["damp"], cfg["grid"], cfg["block"])


def extra_config(name, data, k, task, device, steps, warmup, flush, stream, torch):
    """One more BASELINE config, device-timed, with its own roofline object."""
    from libfm_b200 import FmLearnSgdElement, FmModel, MODE_HOGWILD
    fm = FmModel(data.num_feature, k)
    fm.init_stdev = 0.1
    fm.init_numpy(42)
    l = FmLearnSgdElement(fm, device=device, mode=MODE_HOGWILD)
    l.task, l.learn_rate = task, LEARN_RATE
    l.min_target, l.max_target = data.min_target, data.max_target
    l.push_hparams()
    l.upload(data, 0)
    launches0 = l.kernel_launches()
    stream = torch.cuda.ExternalStream(l.stream(), device=device)  # this learner's own stream
    ms = timed_epochs(l, data, steps, warmup, flush, stream, torch)
    launches = l.kernel_launches() - launches0
    cfg = l.epoch_config()
    l.close()
    peak, peak_src = hbm_peak()
    z = data.num_values / data.num_cases
    bpe = 2 * k * z * 4
    achieved = data.num_cases * bpe / (ms * 1e-3) / 1e9
    return {"workload": name, "rows": data.num_cases, "k": k, "nnz_per_row": z, "value": data.num_cases / (ms * 1e-3),
            "unit": UNIT, "ms_per_step": ms, "steps": steps, "gpu_launches": int(launches),
            "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                         "traffic": None, "peak_source": peak_src,
                         "algorithmic_bytes_per_example": bpe, "kernel": kernel_name(cfg, "hogwild")},
            "kernel_geometry": cfg}


def extra_c4(device, rows, passes=5):
    """BASELINE config C4: the data-parallel part of -method mcmc, the per-iteration e-term pass
    (fm_learn_mcmc.h:148-378) over a MovieLens-10M-shaped set, k=16, through fmb200_mcmc_eterms with a HOST
    result buffer (the Gibbs draws stay on the host, so the read-back belongs to the step)."""
    import numpy as np
    import oracle
    from libfm_b200 import FmLearnSgdElement, FmModel, MODE_INORDER, synth
    d = synth.two_field(rows, 71_567, 10_681, seed=5)
    k = 16
    fm = FmModel(d.num_feature, k)
    fm.init_stdev = 0.1
    fm.init_numpy(42)
    fm.w = np.random.default_rng(1).standard_normal(d.num_feature) * 0.1
    l = FmLearnSgdElement(fm, device=device, mode=MODE_INORDER)
    l.push_hparams()
    l.upload(d, 0)
    launches0 = l.kernel_launches()
    got = l.mcmc_eterms(d)  # warm-up
    ts = []
    for _ in range(passes):
        t0 = time.perf_counter()
        got = l.mcmc_eterms(d)
        ts.append(time.perf_counter() - t0)
    launches = (l.kernel_launches() - launches0) // (passes + 1)
    l.close()
    # the oracle port (pinned bit-identical to the reference's pass) on a bounded sample, 1 core
    sample = d.rows(0, min(rows, 1_000_000))
    port = oracle.Port(d.num_feature, k)
    port.set_params(fm.w0, fm.w, fm.v)
    t0 = time.perf_counter()
    want = port.mcmc_eterms(sample)
    cpu_s = time.perf_counter() - t0
    ms = 1e3 * statistics.median(ts)
    peak, peak_src = hbm_peak()
    bpe = 2 * k * 2 * 4
    achieved = rows * bpe / (ms * 1e-3) / 1e9
    return {"workload": "C4: MCMC/ALS e-term pass, k=16, MovieLens-10M-shaped CSR (71567 users x 10681 items, "
                        "%d cases, 2 nnz/row); fp64, bit-identical to the reference's accumulation order" % rows,
            "rows": rows, "k": k, "value": rows / (ms * 1e-3), "unit": "cases/s", "ms_per_step": ms, "steps": passes,
            "timing": "wall clock around fmb200_mcmc_eterms incl. the device->host copy of the e-terms",
            "d2h_bytes_per_step": int(got.nbytes), "gpu_launches": int(launches), "dtype": "f64",
            "bit_identical_to_oracle_on_sample": bool(np.array_equal(got[:sample.num_cases], want)),
            "cpu_baseline": {"value": sample.num_cases / cpu_s, "unit": "cases/s", "cores": 1, "kind": "port",
                             "sample": "%d cases" % sample.num_cases},
            "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                         "traffic": None, "peak_source": peak_src, "algorithmic_bytes_per_example": bpe,
                         "kernel": "fm_eterm64_kernel (one thread per case, fp64, --fmad=false)",
                         "note": "the step is bound by the 8 B/case read-back over PCIe, not by HBM"}}


def extra_c5(world, rank, local_rank, dist, torch, flush, rows_total, steps=3):
    """BASELINE config C5: SGD k=128 on a 100M-row synthetic CSR (n = 1M features, 39 one-hot fields, -task c)
    row-sharded across the ranks; per epoch ONE exchange of the 516 MB packed state over NVLink peer memory
    (the sliced mean-field combine: reduce-scatter + all-gather in one kernel, fm_peer.cu).  Every rank
    generates and uploads its own shard; device-timed with CUDA events, max over ranks."""
    import ctypes as C
    import numpy as np
    from libfm_b200 import FmLearnSgdElement, FmModel, MODE_HOGWILD
    k, n, z = 128, 1_000_000, 39
    rows = rows_total // world
    ok, l, err = 1, None, ""
    try:
        r = np.random.default_rng(1000 + rank)
        per = n // z
        ids = r.integers(0, per, size=(rows, z), dtype=np.uint32)
        ids += (np.arange(z, dtype=np.uint32) * np.uint32(per))[None, :]
        tgt = np.where(r.integers(0, 2, size=rows) > 0, 1.0, -1.0).astype(np.float32)
        fm = FmModel(n, k)
        fm.init_stdev = 0.01
        fm.init_numpy(42)  # identical replicas
        l = FmLearnSgdElement(fm, device=local_rank, mode=MODE_HOGWILD)
        l.task, l.learn_rate, l.min_target, l.max_target = 1, LEARN_RATE, -1.0, 1.0
        l.push_hparams()
        P = lambda a, t: a.ctypes.data_as(C.POINTER(t))  # noqa: E731
        if l.lib.fmb200_upload_onehot(l._ctx, 0, rows, z, P(ids, C.c_uint32), P(tgt, C.c_float)) != 0:
            raise RuntimeError(l.lib.fmb200_last_error().decode())
        del ids, tgt
        h = C.create_string_buffer(64)
        if l.lib.fmb200_peer_export(l._ctx, h) != 0:
            raise RuntimeError(l.lib.fmb200_last_error().decode())
    except Exception as exc:  # a rank that cannot set up must not leave the others spinning in the exchange
        ok, err = 0, repr(exc)
    flag = torch.tensor([ok], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if int(flag.item()) == 0:
        if l is not None:
            l.close()
        return {"error": "setup failed on at least one rank" + (": " + err if err else "")}
    handles = [None] * world
    dist.all_gather_object(handles, h.raw)
    ok = 1 if l.lib.fmb200_peer_attach_ipc(l._ctx, world, rank, b"".join(handles)) == 0 else 0
    flag = torch.tensor([ok], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if int(flag.item()) == 0:
        l.close()
        return {"error": "peer attach failed"}
    lib, ctx = l.lib, l._ctx
    stream = torch.cuda.ExternalStream(l.stream(), device=local_rank)

    def step():
        if lib.fmb200_sgd_epoch_async(ctx, 0) != 0 or lib.fmb200_allreduce_meanfield(ctx) != 0:
            raise RuntimeError(lib.fmb200_last_error().decode())

    launches0 = l.kernel_launches()
    with torch.cuda.stream(stream):
        step()  # warm-up (first-epoch bias ramp, lazy loading)
        torch.cuda.synchronize()
        dist.barrier()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        ep = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
        for i, (a, b) in enumerate(ev):
            flush.zero_()
            if lib.fmb200_peer_barrier(ctx) != 0:
                raise RuntimeError(lib.fmb200_last_error().decode())
            a.record(stream)
            if lib.fmb200_sgd_epoch_async(ctx, 0) != 0:
                raise RuntimeError(lib.fmb200_last_error().decode())
            ep[i].record(stream)
            if lib.fmb200_allreduce_meanfield(ctx) != 0:
                raise RuntimeError(lib.fmb200_last_error().decode())
            b.record(stream)
        torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in ev) / steps
    ms_epoch = sum(a.elapsed_time(e) for (a, _), e in zip(ev, ep)) / steps
    t = torch.tensor([ms, ms_epoch], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, ms_epoch = float(t[0].item()), float(t[1].item())
    launches = (l.kernel_launches() - launches0) // (steps + 1)
    cfg = l.epoch_config()
    _, n_floats = l.params_device()
    l.close()
    peak, peak_src = hbm_peak()
    bpe = 2 * k * z * 4
    achieved = rows * bpe / (ms_epoch * 1e-3) / 1e9  # per GPU, the epoch kernel alone
    return {"workload": "C5: SGD k=128, %d-row synthetic CSR (1M features, 39 nnz/row) row-sharded over %d GPUs, "
                        "-task c, Hogwild, one sliced mean-field exchange of the packed state per epoch" % (rows * world, world),
            "rows_per_gpu": rows, "k": k, "nnz_per_row": z, "value": world * rows / (ms * 1e-3), "unit": UNIT,
            "ms_per_step": ms, "ms_epoch_kernel": ms_epoch, "ms_exchange": ms - ms_epoch, "steps": steps,
            "state_bytes_per_gpu": int(n_floats * 4), "gpu_launches_per_step": int(launches),
            "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                         "traffic": None, "peak_source": peak_src, "algorithmic_bytes_per_example": bpe,
                         "scope": "per GPU, epoch kernel", "kernel": kernel_name(cfg, "hogwild")},
            "kernel_geometry": cfg}


def dump_model(lrn, out_dir):
    """The parameters after the last timed step, as fmb200_get_params hands them to a caller."""
    import ctypes as C
    import numpy as np
    n, k = lrn.fm.num_attribute, lrn.fm.num_factor
    w0 = C.c_double()
    w = np.empty(n, dtype=np.float64)
    v = np.empty((k, n), dtype=np.float64)
    P = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    if lrn.lib.fmb200_get_params(lrn._ctx, C.byref(w0), P(w), P(v)) != 0:
        raise RuntimeError(lrn.lib.fmb200_last_error().decode())
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "w0.npy"), np.array([w0.value], dtype=np.float64))
    np.save(os.path.join(out_dir, "w.npy"), w)
    np.save(os.path.join(out_dir, "v.npy"), v)


# --------------------------------------------------------------------------
# the GPU arm
# --------------------------------------------------------------------------
def run_gpu_arm(args):
    import numpy as np
    import torch
    from libfm_b200 import FmLearnSgdElement, FmModel, MODE_HOGWILD, synth

    world = env_int("WORLD_SIZE", 1)
    rank = env_int("RANK", 0)
    local_rank = env_int("LOCAL_RANK", 0)
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device (the product has no CPU path)")
    torch.cuda.set_device(local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))

    # every rank owns its own full-size shard (weak scaling), seeded by rank
    data = synth.movielens_1m_shaped(seed=7 + rank)
    n = data.num_feature
    fm = FmModel(n, K_FACTORS)
    fm.init_stdev = 0.1
    fm.init_numpy(42)  # identical replicas on every rank
    lrn = FmLearnSgdElement(fm, device=local_rank, mode=MODE_HOGWILD)
    lrn.task, lrn.learn_rate = 0, LEARN_RATE
    lrn.min_target, lrn.max_target = data.min_target, data.max_target
    lrn.push_hparams()
    lrn.upload(data, 0)

    stream = torch.cuda.ExternalStream(lrn.stream(), device=local_rank)
    ptr, n_floats = lrn.params_device()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    lib, ctx = lrn.lib, lrn._ctx
    import ctypes as C

    # the per-epoch exchange: one-shot all-reduce over NVLink peer memory (fm_peer.cu),
    # NCCL through torch.distributed as the fallback / comparison
    collective = "none"
    params = None
    if world > 1:
        collective = args.collective
        if collective in ("auto", "p2p"):
            h = C.create_string_buffer(64)
            ok = lib.fmb200_peer_export(ctx, h) == 0
            handles = [None] * world
            dist.all_gather_object(handles, h.raw if ok else b"")
            ok = ok and all(len(x) == 64 for x in handles)
            if ok:
                ok = lib.fmb200_peer_attach_ipc(ctx, world, rank, b"".join(handles)) == 0
            flag = torch.tensor([1 if ok else 0], device="cuda")
            dist.all_reduce(flag, op=dist.ReduceOp.MIN)
            if int(flag.item()) == 1:
                collective = "p2p"
            elif collective == "p2p":
                raise RuntimeError("peer attach failed: " + lib.fmb200_last_error().decode())
            else:
                collective = "nccl"
        if collective == "nccl":
            # fallback exchange through torch.distributed: the same mean-field rule as the peer kernel
            # (libfm_b200/dist.py::combine_meanfield_), or the plain mean with --exchange mean
            from libfm_b200 import dist as fdist
            params = torch.as_tensor(_DevBuf(ptr, n_floats), device=torch.device("cuda", local_rank))
            theta0 = params.clone()
            counts_t = torch.as_tensor(np.bincount(data.col, minlength=n).astype(np.float32), device=params.device)
            layout = lrn.params_layout()

    # the combine rule of the peer exchange: mean-field weighted delta sum (default) or plain mean
    peer_exchange = lib.fmb200_allreduce_meanfield if args.exchange == "meanfield" else lib.fmb200_allreduce_mean

    def step():
        rc = lib.fmb200_sgd_epoch_async(ctx, 0)
        if rc == 0 and collective == "p2p":
            rc = peer_exchange(ctx)
        elif rc == 0 and collective == "nccl":
            rc = nccl_exchange()
        if rc != 0:
            raise RuntimeError(lib.fmb200_last_error().decode())

    def nccl_exchange():
        if args.exchange == "mean":
            dist.all_reduce(params)  # sum over ranks on the library's stream
            return lib.fmb200_scale_params(ctx, 1.0 / world)
        fdist.combine_meanfield_(params, theta0, counts_t, data.num_cases, layout, LEARN_RATE, world=world)
        theta0.copy_(params)
        return 0

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    tick = torch.zeros(1, device="cuda")

    def align():
        # the L2 flush takes a different time on every rank; without re-aligning, the
        # first rank to start its epoch would be charged the other ranks' flush time
        # while it waits in the exchange
        if collective == "p2p":
            if lib.fmb200_peer_barrier(ctx) != 0:
                raise RuntimeError(lib.fmb200_last_error().decode())
        elif collective == "nccl":
            dist.all_reduce(tick)

    sampler = ClockSampler(local_rank)
    with torch.cuda.stream(stream):
        for _ in range(max(args.warmup, 3)):
            flush.zero_()
            step()
        barrier()
        launches0 = lrn.kernel_launches()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
              for _ in range(args.steps)]
        sampler.start()
        wall0 = time.perf_counter()
        for a, b in ev:
            flush.zero_()          # evict the CSR and the parameters from L2 (untimed)
            align()                # N > 1: all ranks enter the step together (untimed)
            a.record(stream)
            step()
            b.record(stream)
        torch.cuda.synchronize()
        sampler.sample()
        wall = time.perf_counter() - wall0
        barrier()
    launches = lrn.kernel_launches() - launches0
    if args.dump_outputs and rank == 0:
        dump_model(lrn, args.dump_outputs)
    step_ms = [a.elapsed_time(b) for a, b in ev]
    total_ms = torch.tensor([sum(step_ms)], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(total_ms, op=dist.ReduceOp.MAX)
    total_ms = float(total_ms.item())
    ms_per_step = total_ms / args.steps
    rows = data.num_cases
    value = world * rows / (ms_per_step * 1e-3)

    # ---- end to end through the C ABI, host buffers ------------------------
    from libfm_b200.model import pinned_copy
    ids_h, tgt_h = pinned_copy(data.col), pinned_copy(data.target)
    w0 = C.c_double()
    w_out = np.empty(n, dtype=np.float64)
    v_out = np.empty((K_FACTORS, n), dtype=np.float64)
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t))  # noqa: E731
    n_e2e = max(3, min(args.steps, 20))
    nnz_per_row = data.num_values // rows

    def upload_async(slot):
        # one-hot shape: ids + targets cross PCIe, offsets / values are materialised on the device
        rc = lib.fmb200_upload_onehot_async(ctx, slot, rows, nnz_per_row, P(ids_h, C.c_uint32), P(tgt_h, C.c_float))
        if rc != 0:
            raise RuntimeError(lib.fmb200_last_error().decode())

    # Two device slots, ping-pong: while the epoch of step i runs on slot A, the inputs of
    # step i+1 are already crossing PCIe into slot B (copy stream).  Every step still
    # pays one full upload, one epoch (+ exchange) and one read-back of the model.
    cur_slot = [2, 3]

    def e2e_step(exchange=True):
        upload_async(cur_slot[1])                 # next step's inputs: host -> device
        rc = lib.fmb200_sgd_epoch_async(ctx, cur_slot[0])   # waits for this slot's upload
        if exchange and rc == 0 and collective == "p2p":
            rc = peer_exchange(ctx)
        elif exchange and rc == 0 and collective == "nccl":
            with torch.cuda.stream(stream):
                rc = nccl_exchange()
        if rc == 0:
            rc = lib.fmb200_get_params(ctx, C.byref(w0), P(w_out, C.c_double), P(v_out, C.c_double))
        if rc != 0:
            raise RuntimeError(lib.fmb200_last_error().decode())
        cur_slot.reverse()

    def e2e_measure(exchange=True):
        upload_async(cur_slot[0])
        for _ in range(2):
            e2e_step(exchange)
        barrier()
        t0 = time.perf_counter()
        for _ in range(n_e2e):
            e2e_step(exchange)
        torch.cuda.synchronize()
        t = torch.tensor([(time.perf_counter() - t0) / n_e2e], dtype=torch.float64, device="cuda")
        if world > 1 and exchange:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        barrier()
        return float(t.item())

    e2e_value = world * rows / e2e_measure()
    h2d = int(ids_h.nbytes + tgt_h.nbytes)
    d2h = int(n_floats * 4)
    cfg = lrn.epoch_config()
    launches_total = lrn.kernel_launches()

    # ---- N > 1: what the sharded epochs LEARN, against one sequential stream over all the rows ---------
    # (examples/s alone would hide an exchange that advances the model 1/N epoch per epoch)
    parity_multi = None
    if world > 1 and collective == "p2p" and not args.no_parity:
        ep_n = 4
        full, te = synth.split_rows(synth.two_field(world * rows + 100_000, 6040, 3706, seed=7, planted_k=4),
                                    world * rows)
        shard = full.rows(rank * rows, (rank + 1) * rows)
        v0 = np.random.default_rng(42).standard_normal((K_FACTORS, n)) * 0.1
        lrn.fm.w0, lrn.fm.w, lrn.fm.v = 0.0, np.zeros(n), v0.copy()
        lrn.min_target, lrn.max_target = full.min_target, full.max_target
        lrn.push_hparams()
        lrn.push_params()
        lrn.upload(shard, 4)
        traj = []
        for _ in range(ep_n):
            rc = lib.fmb200_sgd_epoch_async(ctx, 4)
            if rc == 0:
                rc = peer_exchange(ctx)
            if rc != 0:
                raise RuntimeError(lib.fmb200_last_error().decode())
            traj.append(lrn.evaluate(te))  # every rank: the replicas are bit-identical after the exchange
        if rank == 0:
            from oracle import Port
            port = Port(n, K_FACTORS)
            port.set_params(0.0, np.zeros(n), v0)
            ref = []
            for _ in range(ep_n):
                port.sgd_epoch(full, 0, LEARN_RATE, full.min_target, full.max_target)
                ref.append(port.metric(te, 0, full.min_target, full.max_target))
            parity_multi = {"data": "planted rank-4 signal, %d rows in %d shards of %d, 100000 held-out rows"
                                    % (world * rows, world, rows),
                            "exchange": args.exchange, "epochs": ep_n, "heldout_rmse_gpu": traj,
                            "heldout_rmse_one_sequential_stream": ref,
                            "max_abs_gap": max(abs(g - r) for g, r in zip(traj, ref)),
                            "note": "statistical parity only (HOGWILD inside a shard, one combine per epoch)"}
        del full, te, shard

    # ---- N == 8 (or --c5): BASELINE config C5, 100 M rows of k = 128 sharded over the ranks -------------
    c5 = None
    if world > 1 and collective == "p2p" and (args.c5 or (world == 8 and not args.no_extras)):
        try:
            c5 = extra_c5(world, rank, local_rank, dist, torch, flush, args.c5_rows)
        except Exception as exc:
            c5 = {"error": repr(exc)}

    # ---- the tolerance mode: the same workload, sequentially consistent (N == 1) -------------
    tol = None
    if world == 1 and not args.no_tolerance_mode:
        from libfm_b200 import MODE_ORDERED
        lrn.set_mode(MODE_ORDERED)
        l0 = lrn.kernel_launches()
        o_steps = max(3, min(args.steps, 10))
        o_ms = timed_epochs(lrn, data, o_steps, 2, flush, stream, torch)
        o_launches = lrn.kernel_launches() - l0
        o_cfg = lrn.epoch_config()
        o_e2e = rows / e2e_measure(exchange=False)
        peak, _ = hbm_peak()
        o_ach = rows * (2 * K_FACTORS * 2 * 4) / (o_ms * 1e-3) / 1e9
        tol = {"mode": "ordered (FMB200_MODE_ORDERED: the reference's read/write order on w0/w/V; conflict-free "
                       "runs of rows in parallel, bias chain as one fp64 FMA per row over speculated clamp states; "
                       "fp64 state)",
               "dtype": "f64", "value": rows / (o_ms * 1e-3), "unit": UNIT, "ms_per_step": o_ms, "steps": o_steps,
               "e2e": {"value": o_e2e, "unit": UNIT, "h2d_bytes_per_step": h2d,
                       "d2h_bytes_per_step": int((2 + n + n * K_FACTORS) * 8), "steps": n_e2e},
               "gpu_launches": int(o_launches), "kernel": kernel_name(o_cfg, "ordered"), "kernel_geometry": o_cfg,
               "roofline": {"bound": "latency (one dependency chain: one CTA on one SM)", "achieved": o_ach,
                            "peak": peak, "unit": "GB/s", "frac": o_ach / peak,
                            "note": "the sequential semantics leave one chain; HBM is not what bounds this mode"}}
        if not args.no_parity:
            tol["parity"] = parity_run(MODE_ORDERED, local_rank)
    sampler.sample()
    sampler.stop_flag = True
    lrn.close()
    if rank != 0:
        if dist is not None:
            dist.destroy_process_group()
        return 0

    # ---- roofline of the dominant kernel (the epoch kernel of the timed mode) ----------------
    peak, peak_src = hbm_peak()
    bytes_per_example = 2 * K_FACTORS * 2 * 4  # 2*k*nnz*4 (SURVEY.md section 8d)
    kernel_ms = ms_per_step  # the epoch's launches; N > 1: + the peer exchange kernel
    achieved = rows * bytes_per_example / (kernel_ms * 1e-3) / 1e9
    roofline = {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s",
                "frac": achieved / peak, "traffic": None,
                "peak_source": peak_src, "algorithmic_bytes_per_example": bytes_per_example,
                "kernel": kernel_name(cfg, "hogwild")}

    parity = None
    extra = {}
    if world == 1:
        if not args.no_parity:
            parity = parity_run(MODE_HOGWILD, local_rank)
            parity["mode"] = "hogwild (the timed mode): statistical parity only, NOT inside the 1e-5 gate; " \
                             "see tolerance_mode for the path that is"
        if not args.no_extras:
            try:
                dz = synth.movielens_1m_shaped(seed=7, zipf=1.0)
                extra["c2_zipf"] = extra_config("C2 with Zipf(1) user/item ids (hot-feature stress)", dz, K_FACTORS, 0,
                                                local_rank, 10, 3, flush, stream, torch)
                del dz
                d3 = synth.multi_field(args.c3_rows, 39, 1_000_000, 11)
                d3.binarize_targets()
                extra["c3"] = extra_config("C3: SGD k=64, Criteo-shaped CSR (1M features, 39 nnz/row, %d rows), "
                                           "-task c, Hogwild" % args.c3_rows, d3, 64, 1, local_rank, 5, 3, flush,
                                           stream, torch)
                del d3
                extra["c4"] = extra_c4(local_rank, args.c4_rows)
            except Exception as exc:  # an extra must never cost the headline line
                extra["error"] = repr(exc)

    # ---- CPU baseline on this box's host cores (N == 1 only) ------------------
    cpu = None
    if world == 1 and not args.no_cpu_baseline:
        n_cpu = 40  # ~75 ms of row loop each plus the reference's own evaluate passes: ~10-20 s
        ex_s, kind, secs = cpu_reference_epochs(synth.movielens_1m_shaped(seed=7), n_cpu)
        cpu = {"value": ex_s, "unit": UNIT, "cores": 1, "kind": kind,
               "sample": "%d full epochs of the 1000209-row C2 workload (median time_learn %.1f ms)"
                         % (n_cpu, 1e3 * statistics.median(secs))}

    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps,
        "warmup": max(args.warmup, 3), "ms_per_step": ms_per_step, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": dict(WORKLOAD, parallelism="row-sharded dp%d, per-epoch all-reduce of w0|w|V (%s)" % (
            world, {"p2p": "one-shot %s kernel over NVLink peer memory" % args.exchange, "nccl": "NCCL mean",
                    "none": "single GPU"}[collective]),
                       kernel_geometry=cfg),
        "clocks": sampler.summary(),
        "e2e": {"value": e2e_value, "unit": UNIT, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                "steps": n_e2e, "upload": "fmb200_upload_onehot_async (ids + targets; one-hot rows)"},
        "gpu_launches": int(launches),
        "gpu_launches_whole_run": int(launches_total),
        "roofline": roofline,
        "cpu_baseline": cpu,
        "parity": parity,
        "parity_multi_gpu": parity_multi,
        "tolerance_mode": tol,
        "extra": dict(extra, **({"c5": c5} if c5 is not None else {})),
        "timed_region_wall_s": wall,
    }
    print(json.dumps(line), flush=True)
    if dist is not None:
        dist.destroy_process_group()
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-parity", action="store_true")
    ap.add_argument("--no-extras", action="store_true")
    ap.add_argument("--no-tolerance-mode", action="store_true")
    ap.add_argument("--c3-rows", type=int, default=10_000_000)
    ap.add_argument("--c4-rows", type=int, default=10_000_054)
    ap.add_argument("--c5", action="store_true", help="run BASELINE config C5 at any N > 1 (default: only at N = 8)")
    ap.add_argument("--c5-rows", type=int, default=100_000_000, help="total rows of C5 over all ranks")
    ap.add_argument("--collective", default="auto", choices=["auto", "p2p", "nccl"])
    ap.add_argument("--exchange", default="meanfield", choices=["meanfield", "mean"])
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the model after the last timed step as DIR/{w0,w,v}.npy (float64)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if args.dump_outputs and args.impl == "reference":
        ap.error("--dump-outputs writes what the GPU arm computed; the reference arm has nothing to dump")
    if args.impl == "reference":
        return run_reference_arm(args)
    return run_gpu_arm(args)


if __name__ == "__main__":
    sys.exit(main())
