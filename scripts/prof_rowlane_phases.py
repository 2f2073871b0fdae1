"""Per-window phase split of the reproducible row-lane epoch (development aid).

    python scripts/prof_rowlane_phases.py [c2|c2_zipf] [N] [OUT_DIR]

Times N epochs by CUDA events with the default kernel (3 untimed epochs first, the first of them the
bias-ramp epoch), then runs N epochs of the instantiation with phase timers (tuning variant 132; 133 times
the file-order schedule instead of the dealt one), whose
thread 0 of every CTA adds the clock64 cycles of each phase of a window to a slot.  The library prints
the sums of each epoch divided by windows x CTAs on stderr; this script collects those lines and writes
OUT_DIR/phases_<workload>.txt: the mean cycles per window of each phase and the same in microseconds at
the card's maximum SM clock, beside the card's name and power limit.  The phases:

  bias+gather  window start to the tile's bias in hand (staged tile, bias fetch, gathers)
  score+issue  scores, quantisation, the bulk reductions issued, bias partials, end-of-tile barrier
  bulk_wait    the bulk reductions' writes complete, proxy fence, the CTA's barrier before it arrives
  barrier1     arrival to the last CTA's arrival seen (the state loads of the fold are issued here)
  fold         the fold of this thread's slice (dealt schedule: and the bias step of the file-order tile)
  barrier2     the grid barrier that publishes the fold
"""
import os
import re
import statistics
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from prof_epochs import WARMUP, learner  # noqa: E402

PHASES = ["bias+gather", "score+issue", "bulk_wait", "barrier1", "fold", "barrier2"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, mhz = (s.strip() for s in q.split(","))
    return name, float(power), float(mhz)


def main():
    import torch

    which = sys.argv[1] if len(sys.argv) > 1 else "c2"
    n_epochs = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    out_dir = sys.argv[3] if len(sys.argv) > 3 else "."
    os.makedirs(out_dir, exist_ok=True)
    name, power, mhz = card()
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
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n_epochs)]
        for a, b in ev:
            flush.zero_()
            a.record(stream)
            if lib.fmb200_sgd_epoch_async(ctx, 0) != 0:
                raise RuntimeError(lib.fmb200_last_error().decode())
            b.record(stream)
        torch.cuda.synchronize()
        ev_ms = [a.elapsed_time(b) for a, b in ev]

        # the timed instantiation prints one line per epoch on fd 2: catch it in a file
        l.set_tuning(variant=132)
        sys.stderr.flush()
        saved = os.dup(2)
        with tempfile.TemporaryFile(mode="w+") as cap:
            os.dup2(cap.fileno(), 2)
            try:
                for _ in range(n_epochs):
                    epoch()
                torch.cuda.synchronize()
            finally:
                os.dup2(saved, 2)
                os.close(saved)
            cap.seek(0)
            lines = [s for s in cap.read().splitlines() if s.startswith("[rowlane phases")]
    cfg = l.epoch_config()
    l.close()
    if len(lines) != n_epochs:
        raise SystemExit("found %d phase lines, expected %d" % (len(lines), n_epochs))
    windows = re.search(r"\((\d+) windows x (\d+) CTAs\)", lines[0]).groups()
    cyc = {p: statistics.mean(float(re.search(re.escape(p) + r"=([0-9.]+)", s).group(1)) for s in lines)
           for p in PHASES}
    total = sum(cyc.values())
    out = ["# python scripts/prof_rowlane_phases.py %s %d, %s, power limit %.0f W, max SM clock %.0f MHz" % (
               which, n_epochs, name, power, mhz),
           "workload %s, geometry %s, %s windows x %s CTAs per epoch" % (which, cfg, *windows),
           "epoch time by CUDA events, default kernel: mean %.1f us (min %.1f, max %.1f)" % (
               1e3 * statistics.mean(ev_ms), 1e3 * min(ev_ms), 1e3 * max(ev_ms)),
           "",
           "per window, CTA thread 0, mean over %d epochs and all CTAs (us at %.0f MHz):" % (n_epochs, mhz),
           "%-14s %10s %8s %7s" % ("phase", "cycles", "us", "share")]
    for p in PHASES:
        out.append("%-14s %10.0f %8.2f %6.1f%%" % (p, cyc[p], cyc[p] / mhz, 100.0 * cyc[p] / total))
    out.append("%-14s %10.0f %8.2f" % ("window", total, total / mhz))
    text = "\n".join(out) + "\n"
    with open(os.path.join(out_dir, "phases_%s.txt" % which), "w") as f:
        f.write(text)
    print(text)


if __name__ == "__main__":
    main()
