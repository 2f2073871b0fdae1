"""GPU: `bin/libFM -method sgd` with FMB200_REPRODUCIBLE=1 runs the windowed HOGWILD epoch: on ragged rows of up to
40 entries with k = 16 (shapes the row-lane epoch does not take), two runs of one command line write the same -out
and -save_model files and print the same #Iter lines, with the data resident and streamed from .x blocks
(-cache_size; windows restart at every block)."""
import os
import subprocess

import numpy as np
import pytest

from libfm_b200 import Data, build, synth

pytestmark = pytest.mark.gpu

ARGS = ["-task", "r", "-train", "train.libfm", "-test", "test.libfm", "-method", "sgd", "-dim", "1,1,16", "-iter", "4",
        "-learn_rate", "0.005", "-init_stdev", "0.05", "-seed", "7"]


def _ragged(n_rows, n_feat, seed):
    r = np.random.default_rng(seed)
    lens = r.integers(0, 41, size=n_rows)
    row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
    row_ptr[1:] = np.cumsum(lens)
    col = r.integers(0, n_feat, size=int(row_ptr[-1])).astype(np.uint32)
    val = r.uniform(0.5, 1.5, size=len(col)).astype(np.float32)
    return Data(row_ptr, col, val, r.integers(1, 6, size=n_rows).astype(np.float32), n_feat)


def _run(args, cwd, env):
    r = subprocess.run([build.cli_path()] + args, cwd=cwd, capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stderr
    return r.stdout


def _iters(stdout):
    return [l for l in stdout.splitlines() if l.startswith("#Iter=")]


@pytest.mark.parametrize("streamed", [False, True])
def test_reproducible_command_line(streamed, tmp_path):
    if not os.path.exists(build.cli_path()):
        build.build_all()
    d = _ragged(120_000, 5000, seed=3)
    train, test = synth.split_rows(d, 100_000)
    synth.to_libfm_text(train, str(tmp_path / "train.libfm"))
    synth.to_libfm_text(test, str(tmp_path / "test.libfm"))
    args = list(ARGS)
    if streamed:
        convert = os.path.join(os.path.dirname(build.cli_path()), "convert")
        for stem in ("train", "test"):
            subprocess.run([convert, "--ifile", stem + ".libfm", "--ofilex", stem + ".bin.x", "--ofiley",
                            stem + ".bin.y"], cwd=tmp_path, capture_output=True, check=True)
        args = [{"train.libfm": "train.bin", "test.libfm": "test.bin"}.get(a, a) for a in args]
        args += ["-cache_size", str((os.path.getsize(str(tmp_path / "train.bin.x")) - 24) // 3)]
    env = dict(os.environ, FMB200_REPRODUCIBLE="1")
    outs = []
    for rep in range(2):
        outs.append(_run(args + ["-out", "out%d.txt" % rep, "-save_model", "model%d.txt" % rep], tmp_path, env))
    if streamed:
        assert sum(l.startswith("streaming ") for l in outs[0].splitlines()) == 2
    assert len(_iters(outs[0])) == 4
    assert _iters(outs[0]) == _iters(outs[1])
    for f in ("out", "model"):
        assert (tmp_path / (f + "0.txt")).read_bytes() == (tmp_path / (f + "1.txt")).read_bytes()
    last = _iters(outs[0])[-1]
    assert "nan" not in last.lower(), last
