"""CPU: `bin/libFM -method sgda -cache_size` loads a binary validation set as it loads the training and test sets:
block by block, the plan line naming read_xblocks' blocks, the loader's sizes line carrying what the whole-file
load prints for the same file.  Loading needs no GPU: these lines come before the learner asks for one."""
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from libfm_b200.model import read_xblocks
from test_sgda_stream_cli_gpu import GOLDEN, binary_inputs, cache_for

CLI = os.path.join(ROOT, "bin", "libFM")


def sizes_line(stdout, after):
    """the loader's 'num_cases=... max_target=...' line printed after the line starting with `after`"""
    lines = stdout.splitlines()
    i = next(i for i, l in enumerate(lines) if l.startswith(after))
    return next(l[l.index("num_cases="):] for l in lines[i + 1:] if "num_cases=" in l)


def test_validation_set_streams_with_the_plan_of_its_file(tmp_path):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    z = np.load(GOLDEN)
    binary_inputs({k: str(z[k]) for k in z.files}, tmp_path)
    args = [CLI, "-method", "sgda", "-mode", "inorder", "-task", "r", "-train", "train.libfm", "-test", "test.libfm",
            "-validation", "val.libfm", "-iter", "1", "-learn_rate", "0.02", "-seed", "7"]
    cache = cache_for(tmp_path, ["train.libfm", "test.libfm", "val.libfm"], 3)
    r = subprocess.run(args + ["-cache_size", str(cache)], cwd=tmp_path, capture_output=True, text=True)
    base = subprocess.run(args, cwd=tmp_path, capture_output=True, text=True)
    for f in ("train.libfm", "test.libfm", "val.libfm"):
        blocks = list(read_xblocks(str(tmp_path / (f + ".x")), cache))
        longest = max(hi - lo for lo, hi, _, _ in blocks)
        line = "streaming %s.x: %d blocks of at most %d rows and %d bytes" % (f, len(blocks), longest, cache // 2)
        assert r.stdout.splitlines().count(line) == 1, r.stdout
        assert len(blocks) >= 3
    got = sizes_line(r.stdout, "Loading validation set")
    assert got == sizes_line(base.stdout, "Loading validation set")
    assert re.match(r"num_cases=\d+\tnum_values=\d+\tnum_features=\d+\tmin_target=\S+\tmax_target=\S+$", got)
    import torch
    if not torch.cuda.is_available():
        assert r.returncode != 0 and "#Iter" not in r.stdout
    else:
        assert r.returncode == 0, r.stderr
