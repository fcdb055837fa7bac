"""In-tree native build: sm_90a CUDA kernels (nvcc -> ops/libtepdist_kernels.so, C ABI loaded with
ctypes) and the C++ planner/runtime core (g++ + pybind11 -> tepdist_b200/_C*.so).

Artifacts are built next to the sources (git-ignored), so the package imports from the source tree; nothing is
JIT-cached outside the repository.  `python -m tepdist_b200.build_native [--force]`.
"""
from __future__ import annotations

import glob
import os
import shutil
import subprocess
import sys
import sysconfig

ROOT = os.path.dirname(os.path.abspath(__file__))
OPS_SRC = os.path.join(ROOT, "ops", "csrc")
KERNEL_SO = os.path.join(ROOT, "ops", "libtepdist_kernels.so")
CORE_SRC = os.path.join(ROOT, "csrc")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "--use_fast_math", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
]


def _newer(target: str, sources: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def build_kernels(force: bool = False, verbose: bool = False) -> str:
    cus = sorted(glob.glob(os.path.join(OPS_SRC, "*.cu")))
    hdrs = sorted(glob.glob(os.path.join(OPS_SRC, "*.cuh")))
    objdir = os.path.join(ROOT, "ops", "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for cu in cus:
        obj = os.path.join(objdir, os.path.basename(cu)[:-3] + ".o")
        objs.append(obj)
        if force or _newer(obj, [cu] + hdrs):
            cmd = [_nvcc(), *NVCC_FLAGS, "-I", OPS_SRC, "-c", cu, "-o", obj]
            procs.append((cu, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cu, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            print(out)
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {cu}")
        log = os.path.join(objdir, os.path.basename(cu)[:-3] + ".ptxas.txt")
        with open(log, "w") as f:
            f.write(out)
    if force or procs or not os.path.exists(KERNEL_SO):
        cmd = [_nvcc(), "-shared", "-o", KERNEL_SO, *objs, "-lcudart"]
        subprocess.check_call(cmd)
    return KERNEL_SO


def core_so_path() -> str:
    suffix = sysconfig.get_config_var("EXT_SUFFIX") or ".so"
    return os.path.join(ROOT, "_C" + suffix)


def build_core(force: bool = False, verbose: bool = False) -> str:
    import pybind11

    srcs = sorted(glob.glob(os.path.join(CORE_SRC, "**", "*.cc"), recursive=True))
    hdrs = sorted(glob.glob(os.path.join(CORE_SRC, "**", "*.h"), recursive=True))
    out = core_so_path()
    if not srcs:
        return out
    objdir = os.path.join(CORE_SRC, "build")
    os.makedirs(objdir, exist_ok=True)
    inc = ["-I", CORE_SRC, "-I", pybind11.get_include(), "-I", sysconfig.get_paths()["include"]]
    flags = ["-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-Wall", "-Wno-sign-compare", "-pthread"]
    objs, procs = [], []
    for s in srcs:
        rel = os.path.relpath(s, CORE_SRC).replace(os.sep, "_")
        obj = os.path.join(objdir, rel[:-3] + ".o")
        objs.append(obj)
        if force or _newer(obj, [s] + hdrs):
            cmd = ["g++", *flags, *inc, "-c", s, "-o", obj]
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
            if len(procs) % 8 == 0:
                for _, p in procs[-8:]:
                    p.wait()
    for s, p in procs:
        o, _ = p.communicate()
        if verbose or p.returncode != 0:
            print(o)
        if p.returncode != 0:
            raise RuntimeError(f"g++ failed for {s}")
    if force or procs or not os.path.exists(out):
        subprocess.check_call(["g++", "-shared", "-o", out, *objs, "-pthread"])
    return out


def build_all(force: bool = False, verbose: bool = False) -> None:
    build_core(force, verbose)
    build_kernels(force, verbose)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built:", KERNEL_SO, core_so_path())
