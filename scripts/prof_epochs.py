"""Kernel table of a few HOGWILD epochs from torch.profiler (development aid).

    python scripts/prof_epochs.py [c2|c2_zipf|c3] [N] [OUT_DIR]

Runs 3 untimed epochs (the first one is the bias-ramp epoch), then N epochs under torch.profiler, each
after the same 256 MiB L2 flush bench.py does, on the library's stream.  Writes OUT_DIR/prof_<workload>.txt
(and the Chrome trace beside it): every kernel with its launch count and summed device time per epoch, and
per epoch the span from the first kernel's start to the last kernel's end, whose remainder after the kernel
times is the gaps between launches.  The epoch time by CUDA events, with the profiler off, is measured
over the same N epochs first.
"""
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from libfm_b200 import FmLearnSgdElement, FmModel, MODE_HOGWILD, synth  # noqa: E402

WARMUP = 3


def learner(which):
    if which in ("c2", "c2_zipf"):
        d, k, task = synth.movielens_1m_shaped(seed=7, zipf=1.0 if which == "c2_zipf" else 0.0), 8, 0
    elif which == "c3":
        d, k, task = synth.multi_field(1_000_000, 39, 1_000_000, 11), 64, 1
        d.binarize_targets()
    else:
        raise SystemExit("unknown workload " + which)
    fm = FmModel(d.num_feature, k)
    fm.init_stdev = 0.1
    fm.init_numpy(42)
    l = FmLearnSgdElement(fm, mode=MODE_HOGWILD)
    l.task, l.learn_rate = task, 0.01
    l.min_target, l.max_target = d.min_target, d.max_target
    l.push_hparams()
    l.upload(d, 0)
    return l


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    which = sys.argv[1] if len(sys.argv) > 1 else "c2"
    n_epochs = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    out_dir = sys.argv[3] if len(sys.argv) > 3 else "."
    os.makedirs(out_dir, exist_ok=True)
    l = learner(which)
    lib, ctx = l.lib, l._ctx
    stream = torch.cuda.ExternalStream(l.stream())
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def epoch():
        flush.zero_()
        if lib.fmb200_sgd_epoch_async(ctx, 0) != 0:
            raise RuntimeError(lib.fmb200_last_error().decode())

    with torch.cuda.stream(stream):
        for _ in range(WARMUP):
            epoch()
        torch.cuda.synchronize()
        # epoch time with the profiler off: CUDA events on the library's stream
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n_epochs)]
        for a, b in ev:
            flush.zero_()
            a.record(stream)
            if lib.fmb200_sgd_epoch_async(ctx, 0) != 0:
                raise RuntimeError(lib.fmb200_last_error().decode())
            b.record(stream)
        torch.cuda.synchronize()
        ev_ms = [a.elapsed_time(b) for a, b in ev]
        launches0 = l.kernel_launches()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n_epochs):
                epoch()
            torch.cuda.synchronize()
        launches = l.kernel_launches() - launches0
    cfg = l.epoch_config()
    l.close()

    trace = os.path.join(out_dir, "prof_%s.pt.trace.json" % which)
    prof.export_chrome_trace(trace)
    kernels = sorted((e for e in json.load(open(trace))["traceEvents"] if e.get("cat") == "kernel"),
                     key=lambda e: e["ts"])
    # the library's kernels between two flushes are one epoch
    epochs, cur = [], []
    for e in kernels:
        if "fmb::" in e["name"]:
            cur.append(e)
        elif cur:
            epochs.append(cur)
            cur = []
    if cur:
        epochs.append(cur)
    if len(epochs) != n_epochs:
        raise SystemExit("found %d epochs in the trace, expected %d" % (len(epochs), n_epochs))

    def short(name):
        return name.split("(")[0].replace("void ", "")

    names = sorted({short(e["name"]) for ep in epochs for e in ep})
    per = {nm: {"launches": 0, "us": 0.0} for nm in names}
    spans = []
    for ep in epochs:
        for e in ep:
            per[short(e["name"])]["launches"] += 1
            per[short(e["name"])]["us"] += e["dur"]
        spans.append(max(e["ts"] + e["dur"] for e in ep) - ep[0]["ts"])
    busy = sum(p["us"] for p in per.values()) / n_epochs
    span = statistics.mean(spans)
    lines = ["workload %s, %d epochs after %d warm-up epochs, geometry %s, GPU %s" % (
                 which, n_epochs, WARMUP, cfg, torch.cuda.get_device_name(0)),
             "library launches per epoch: %g" % (launches / n_epochs),
             "epoch time by CUDA events, profiler off: mean %.1f us (min %.1f, max %.1f)" % (
                 1e3 * statistics.mean(ev_ms), 1e3 * min(ev_ms), 1e3 * max(ev_ms)),
             "",
             "%-70s %12s %14s %12s" % ("kernel", "launches/ep", "us/epoch", "us/launch")]
    for nm in names:
        p = per[nm]
        lines.append("%-70s %12g %14.1f %12.2f" % (nm[:70], p["launches"] / n_epochs, p["us"] / n_epochs,
                                                   p["us"] / p["launches"]))
    lines += ["%-70s %12s %14.1f" % ("sum of kernel durations", "", busy),
              "%-70s %12s %14.1f" % ("span, first kernel start to last kernel end", "", span),
              "%-70s %12s %14.1f" % ("gaps (span - kernels)", "", span - busy)]
    text = "\n".join(lines) + "\n"
    with open(os.path.join(out_dir, "prof_%s.txt" % which), "w") as f:
        f.write(text)
    print(text)


if __name__ == "__main__":
    main()
