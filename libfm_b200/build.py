"""In-tree build of the native pieces (nvcc cross-compiles sm_90a without a GPU).

  libfm_b200/lib/libfmb200.so   CUDA kernels + the C ABI of include/fmb200.h
  bin/libFM                     drop-in C++ command line (host/), links the above
  bin/convert, bin/transpose    drop-ins for the reference's tools (text -> .x/.y, .x -> .xt)

Build products are git-ignored.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
HOST = os.path.join(HERE, "host")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(ROOT, "build", "obj")
BINDIR = os.path.join(ROOT, "bin")

NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
          "-I", os.path.join(ROOT, "include")]

# per-file extra flags: the fp64 sequential-equivalent path must not contract a*b+c
CU_SOURCES = {
    "fm_context.cu": [],
    "fm_hogwild.cu": [],
    "fm_rowlane.cu": [],
    "fm_peer.cu": [],
    "fm_predict.cu": [],
    "fm_inorder.cu": ["--fmad=false"],
    "fm_ordered.cu": [],
    "fm_upload.cu": [],
    "fm_deal.cu": [],
    "fm_sgda_hogwild.cu": [],
    "fm_sgd_window.cu": [],
    "fm_mcmc.cu": ["--fmad=false"],
}
CU_HEADERS = ["fm_device.cuh", "fm_rowgroup.cuh", "fm_hogwild_common.cuh", "fm_window.cuh", "fmb200_internal.h",
              "fm_inorder_wavefront.cuh", "fm_sgda_wavefront.cuh", "fm_sgda_plan.h", "fm_loss.cuh", "fm_ordered.cuh", "fm_roworder.cuh", "ref_random.h"]


def _newer(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd: list[str], log: str | None = None) -> None:
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if log:
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + p.stdout)
    if p.returncode != 0:
        sys.stderr.write(p.stdout)
        raise RuntimeError("build step failed: " + " ".join(cmd))


def lib_path() -> str:
    return os.path.join(LIBDIR, "libfmb200.so")


def cli_path() -> str:
    return os.path.join(BINDIR, "libFM")


def build_lib(force: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in CU_HEADERS] + [os.path.join(ROOT, "include", "fmb200.h")]
    jobs = []
    objs = []
    for src, extra in CU_SOURCES.items():
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJDIR, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _newer(o, [s] + hdrs):
            cmd = [NVCC, *ARCH, *COMMON, *extra, "-c", s, "-o", o]
            jobs.append((cmd, o + ".log"))
    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 2)) as ex:
            list(ex.map(lambda j: _run(*j), jobs))
    out = lib_path()
    if force or jobs or _newer(out, objs):
        _run([NVCC, *ARCH, "-shared", "-o", out, *objs])
    return out


def build_cli(force: bool = False) -> str | None:
    """The drop-in command lines: plain C++ host code (bin/libFM over the C ABI, bin/convert)."""
    main = os.path.join(HOST, "libfm_main.cpp")
    if not os.path.exists(main):
        return None
    os.makedirs(BINDIR, exist_ok=True)
    hdrs = [os.path.join(HOST, f) for f in os.listdir(HOST) if f.endswith(".h")]
    hdrs.append(os.path.join(CSRC, "ref_random.h"))  # fm_host.h includes it
    out = cli_path()
    if force or _newer(out, [main] + hdrs + [lib_path()]):
        cmd = ["g++", "-O2", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), main,
               "-o", out, "-pthread", "-L", LIBDIR, "-lfmb200", "-Wl,-rpath,$ORIGIN/../libfm_b200/lib"]
        nccl = os.environ.get("FMB200_NCCL", "1") == "1" and os.path.exists("/usr/include/nccl.h")
        cuda_inc = "/usr/local/cuda/include"
        if nccl:
            cmd += ["-DFMB200_WITH_NCCL", "-I", cuda_inc, "-lnccl", "-L/usr/local/cuda/lib64", "-lcudart"]
        _run(cmd)
    for tool in ("convert", "transpose"):  # the reference's tools/ (text -> binary, .x -> .xt)
        src = os.path.join(HOST, tool + "_main.cpp")
        exe = os.path.join(BINDIR, tool)
        if os.path.exists(src) and (force or _newer(exe, [src] + hdrs)):
            _run(["g++", "-O2", "-std=c++17", "-Wall", src, "-o", exe, "-pthread"])
    return out


def build_all(force: bool = False) -> None:
    build_lib(force)
    build_cli(force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv)
    print(lib_path())
