"""End-to-end wall time of the drop-in CLI on a C2-shaped text file (development aid; run on the GPU box from the
repo root).

    python scripts/cli_walltime.py                      bin/libFM, then the stock reference CLI (oracle/_ref/libFM)
    python scripts/cli_walltime.py --against CLI [--rounds N]
                                                        bin/libFM and another build of it, alternately, N rounds
"""
import argparse, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from libfm_b200 import synth
ap = argparse.ArgumentParser()
ap.add_argument("--against", help="another libFM binary with the same flags, timed alternately with bin/libFM")
ap.add_argument("--rounds", type=int, help="default: 2 with --against, else 1")
a = ap.parse_args()
OURS = [("hogwild 20 iters", ["-iter", "20", "-verbosity", "1"]), ("inorder  2 iters", ["-iter", "2", "-mode", "inorder"])]
REF = [("20 iters", ["-iter", "20"]), ("2 iters", ["-iter", "2"])]
if a.against:
    cands, rounds = [("ours", "bin/libFM", OURS), ("against", a.against, OURS)], a.rounds or 2
else:
    cands, rounds = [("ours", "bin/libFM", OURS), ("reference", "oracle/_ref/libFM", REF)], a.rounds or 1
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip().splitlines()
print("device:", gpu[0] if gpu else "unknown", flush=True)
d = synth.movielens_1m_shaped(seed=7, planted_k=4)
synth.to_libfm_text(d.rows(0, 900000), "/tmp/tr.libfm")
synth.to_libfm_text(d.rows(900000, d.num_cases), "/tmp/te.libfm")
base = ["-task", "r", "-train", "/tmp/tr.libfm", "-test", "/tmp/te.libfm", "-method", "sgd", "-dim", "1,1,8",
        "-learn_rate", "0.01", "-seed", "42"]
for r in range(rounds):
    for label, exe, configs in cands:
        for name, extra in configs:
            t0 = time.time()
            p = subprocess.run([os.path.join(ROOT, exe)] + base + extra, capture_output=True, text=True)
            dt = time.time() - t0
            fin = [l for l in (p.stdout + p.stderr).splitlines() if l.startswith(("Final", "time:")) or "ERROR" in l]
            print("round %d %-9s %s: rc=%d wall %.2f s :: %s" % (r, label, name, p.returncode, dt,
                                                               " ".join(fin).replace("\t", " ")), flush=True)
