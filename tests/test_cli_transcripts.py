"""bin/libFM against tests/golden/cli_transcripts.json (scripts/make_cli_transcripts.py): for every command line
of the matrix -- SGD, MCMC and ALS runs with their -out, -save_model, -load_model and -rlog files, refusals and
flag errors -- the same stdout, stderr, exit code and written files, with the non-reproducible parts masked alike.

On an H100 every run is compared whole.  Without a GPU the runs that end before a device is needed are compared
whole, and the others up to the point where the command line stops with "no CPU path"."""
import importlib.util
import json
import os

import pytest

from conftest import GOLDEN, ROOT

_spec = importlib.util.spec_from_file_location("make_cli_transcripts",
                                               os.path.join(ROOT, "scripts", "make_cli_transcripts.py"))
mct = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mct)

RECORD = json.load(open(os.path.join(GOLDEN, "cli_transcripts.json")))
CLI = os.path.join(ROOT, "bin", "libFM")
BEFORE_DEVICE = [name for name, run in mct.RUNS.items() if not run.device]
ON_DEVICE = [name for name, run in mct.RUNS.items() if run.device]


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    d = tmp_path_factory.mktemp("cli_inputs")
    mct.write_inputs(str(d))
    return str(d)


def _same(got, want):
    for key in ("returncode", "stderr", "stdout", "files"):
        assert got[key] == want[key], key


def test_matrix_is_the_recorded_one():
    assert {name: run.args for name, run in mct.RUNS.items()} == {n: t["args"] for n, t in RECORD["runs"].items()}


@pytest.mark.parametrize("name", BEFORE_DEVICE)
def test_transcript_before_device(name, inputs, tmp_path):
    _same(mct.transcript(CLI, name, inputs, str(tmp_path)), RECORD["runs"][name])


@pytest.mark.parametrize("name", ON_DEVICE)
def test_transcript_up_to_device_without_gpu(name, inputs, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: test_transcript_on_gpu compares the whole run")
    got, want = mct.transcript(CLI, name, inputs, str(tmp_path)), RECORD["runs"][name]
    assert got["returncode"] == 1 and "no CPU path" in got["stderr"], got["stderr"]
    assert got["stdout"] and want["stdout"].startswith(got["stdout"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ON_DEVICE)
def test_transcript_on_gpu(name, inputs, tmp_path):
    if mct.RUNS[name].rowlane and mct.device()["sms"] != RECORD["device"]["sms"]:
        pytest.skip("the row-lane epoch's windows span the SMs: recorded on %s" % RECORD["device"]["name"])
    _same(mct.transcript(CLI, name, inputs, str(tmp_path)), RECORD["runs"][name])
