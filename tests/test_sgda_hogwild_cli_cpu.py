"""CPU: what `bin/libFM -method sgda` refuses in -mode hogwild, before it loads anything: more than one GPU, and
-cache_size over binary data (streamed SGDA runs in -mode inorder or ordered)."""
import os
import subprocess

import pytest

from libfm_b200 import build, synth
from libfm_b200.model import write_binary


@pytest.fixture(scope="module")
def cli():
    exe = build.cli_path()
    if not os.path.exists(exe):
        build.build_all()
    return exe


def _run(cli, args, cwd):
    return subprocess.run([cli] + args.split(), cwd=cwd, capture_output=True, text=True)


def test_more_gpus_refused(cli, tmp_path):
    p = _run(cli, "-train missing.libfm -test missing.libfm -validation missing.libfm -task r -method sgda -gpus 2",
             tmp_path)
    assert p.returncode == 1 and "-method sgda runs on one GPU: -gpus must be 1" in p.stderr
    assert "Loading train" not in p.stdout


def test_cache_size_on_binary_data_refused(cli, tmp_path):
    d = synth.two_field(100, 10, 10, seed=1)
    write_binary(d, str(tmp_path / "t.x"), str(tmp_path / "t.y"))
    p = _run(cli, "-train t -test t -validation t -task r -method sgda -cache_size 1000", tmp_path)
    assert p.returncode == 1 and "-mode inorder" in p.stderr and "-cache_size" in p.stderr
    assert "Loading train" not in p.stdout
