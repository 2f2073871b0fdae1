"""CPU: the wavefront kernels' OWN SOURCE (libfm_b200/csrc/fm_inorder_wavefront.cuh, fm_sgda_wavefront.cuh),
compiled for the host through tests/simt/simt_shim.h and run as 32 threads -- one per lane, pthread barriers
where the kernel has __syncwarp / __ballot_sync / __shfl_sync -- against the sequential oracles
(oracle/fm_oracle.c, oracle/fm_oracle_sgda.c).

 * plain build: the SGD epoch's w0 / w / V bit-identical to fmo_sgd_epoch after two epochs on nine shapes;
   the SGDA epoch's w0 / w / V / grad_w / grad_v / reg_w / reg_v bit-identical to fmo_sgda_epoch after three
   epochs (the first without lambda-steps, each later one cut at the moments step as the launcher cuts it)
   on seven: dense conflicts, validation rows that repeat their own and the next pair's train row, a
   validation cursor that restarts inside windows, repeated ids, x != 1, k in {1, 5, 8}, 1 and 3 groups;
 * -fsanitize=thread build: no data race, i.e. every cross-lane hand-off through "shared" or "global"
   memory in the kernel is ordered by one of its barriers;
 * negative control: the same build with __syncwarp compiled out MUST make ThreadSanitizer complain on the
   SGD cases -- otherwise the check above proves nothing.

What this cannot show is hardware behaviour (caches, real warp scheduling, device exp()); the device run is
tests/test_wavefront_gpu.py and tests/test_sgda_wavefront_gpu.py."""
import os
import shutil
import subprocess

import pytest

from conftest import ROOT

SIMT = os.path.join(ROOT, "tests", "simt")
OUT = os.path.join(SIMT, "_build")
CUDA_INC = "/usr/local/cuda/include"

pytestmark = pytest.mark.skipif(shutil.which("g++") is None or not os.path.isdir(CUDA_INC),
                                reason="needs g++ and the CUDA headers")


@pytest.fixture(scope="module")
def oracle_obj():
    os.makedirs(OUT, exist_ok=True)
    objs = []
    for src in ("fm_oracle.c", "fm_oracle_sgda.c"):
        obj = os.path.join(OUT, src.replace(".c", ".o"))
        subprocess.run(["gcc", "-O1", "-ffp-contract=off", "-c", os.path.join(ROOT, "oracle", src), "-o", obj],
                       check=True)
        objs.append(obj)
    return objs


def _build(name, oracle_obj, extra):
    exe = os.path.join(OUT, name)
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-pthread", "-I" + CUDA_INC] + extra + \
          [os.path.join(SIMT, "wavefront_host.cpp")] + oracle_obj + ["-o", exe, "-lm"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _assert_all_cases_identical(stdout):
    lines = [l for l in stdout.splitlines() if l.strip()]
    sgda = [l for l in lines if l.startswith("sgda_")]
    assert len(lines) == 9 + 7 and len(sgda) == 7, stdout
    assert all("bit-identical" in l for l in lines), stdout


def test_kernel_source_on_host_lanes_is_bit_identical(oracle_obj):
    exe = _build("wavefront_host", oracle_obj, [])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    _assert_all_cases_identical(r.stdout)


def test_kernel_source_is_race_free_under_tsan(oracle_obj):
    exe = _build("wavefront_host_tsan", oracle_obj, ["-fsanitize=thread"])
    r = subprocess.run([exe, "0.25"], capture_output=True, text=True, timeout=900)
    if "FATAL: ThreadSanitizer" in r.stderr:  # e.g. ASLR / personality restrictions of a sandbox
        pytest.skip("ThreadSanitizer cannot run here: " + r.stderr.splitlines()[0])
    assert r.returncode == 0 and "ThreadSanitizer" not in r.stderr, r.stdout + r.stderr[:4000]
    _assert_all_cases_identical(r.stdout)
    # negative control: without the kernel's __syncwarp barriers the tool must see races
    bad = _build("wavefront_host_tsan_nosync", oracle_obj, ["-fsanitize=thread", "-DSIMT_NO_SYNCWARP"])
    r = subprocess.run([bad, "0.1", "sgd"], capture_output=True, text=True, timeout=900)
    assert "ThreadSanitizer: data race" in r.stderr
