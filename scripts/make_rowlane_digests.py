"""Record the parameters the row-lane HOGWILD epoch computes on C2 and C2-Zipf as SHA-256 digests.

    python scripts/make_rowlane_digests.py OUT.json

Three epochs from the seeded initial model (the first-epoch bias ramp and two full-grid epochs), a digest
of w0, w and V (float64, as fmb200_get_params returns them) after each.  The row-lane epoch is
reproducible, and which rows share a window with which decides what it computes, so these digests pin
its window schedule: tests/test_rowlane_windows_gpu.py compares against tests/golden/rowlane_c2_digests.json,
recorded on an H100 with this script.  FMB200_LIB selects the library build that computes them.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from conftest import digest  # noqa: E402
from libfm_b200 import FmLearnSgdElement, FmModel, MODE_HOGWILD, synth  # noqa: E402

EPOCHS = 3


def run(zipf):
    d = synth.movielens_1m_shaped(seed=7, zipf=zipf)
    fm = FmModel(d.num_feature, 8)
    fm.init_stdev = 0.1
    fm.init_numpy(42)
    l = FmLearnSgdElement(fm, device=0, mode=MODE_HOGWILD)
    l.task, l.learn_rate = 0, 0.01
    l.min_target, l.max_target = d.min_target, d.max_target
    l.push_hparams()
    out = []
    for _ in range(EPOCHS):
        l.sgd_epoch(d)
        l.pull_params()
        out.append({"w0": digest(float(l.fm.w0)), "w": digest(l.fm.w), "v": digest(l.fm.v)})
    cfg = l.epoch_config()
    l.close()
    return out, cfg


def main():
    import torch
    cases, geom = {}, set()
    for name, zipf in (("c2", 0.0), ("c2_zipf", 1.0)):
        cases[name], cfg = run(zipf)
        geom.add((cfg["rows_per_tile"], cfg["grid"]))
    assert len(geom) == 1
    (tr, grid), = geom
    # the window is `grid` tiles of `rows_per_tile` rows: the digests hold for this geometry only
    rec = {"gpu": torch.cuda.get_device_name(0), "epochs": EPOCHS, "rows_per_tile": tr, "grid": grid,
           "digests": cases}
    with open(sys.argv[1], "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
