"""Build recipes for the native pieces (in-tree, next to the sources that use them).

  build_cuda() -> cranesched_b200/csrc/libcrane_sched.so   (nvcc, sm_90a; the product)
  build_emu()  -> tests/_emu/libcrane_sched_emu.so         (g++ -DCRANE_EMU; test harness only)
"""
from __future__ import annotations

import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cranesched_b200", "csrc")
SO = os.path.join(CSRC, "libcrane_sched.so")
EMU_SO = os.path.join(ROOT, "tests", "_emu", "libcrane_sched_emu.so")
_SOURCES = ["sched_api.cu", "sched_kernels.cuh", "commit_v2.cuh", "qos_kernels.cuh", "step_kernels.cuh", "running_kernels.cuh",
            "gate_kernels.cuh", "step_resident_kernels.cuh", "compact_kernels.cuh", "algebra.cuh"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100 (Hopper)


def _stale(target: str, extra=()) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    # this file too: a library built with other flags (another architecture) is stale
    deps = [os.path.join(CSRC, s) for s in _SOURCES] + [os.path.join(ROOT, "include", "crane_sched.h"),
                                                         os.path.abspath(__file__)] + list(extra)
    return any(os.path.getmtime(d) > t for d in deps)


def build_cuda(force: bool = False, verbose: bool = False) -> str:
    if force or _stale(SO):
        cmd = ["nvcc", "-O3", "-std=c++17", *ARCH, "-lineinfo",
               "--fmad=false", "-Xcompiler", "-fPIC", "-shared", "-o", SO, os.path.join(CSRC, "sched_api.cu")]
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        subprocess.check_call(cmd)
    return SO


def build_prof(force: bool = True) -> str:
    """Profiling variant (-DCRANE_PROFILE: clock64 phase counters in k_commit); tools only."""
    os.makedirs(os.path.join(ROOT, "tools", "variants"), exist_ok=True)
    so = os.path.join(ROOT, "tools", "variants", "libcrane_sched_prof.so")
    cmd = ["nvcc", "-O3", "-std=c++17", *ARCH, "-lineinfo", "--fmad=false",
           "-DCRANE_PROFILE", "-Xcompiler", "-fPIC", "-shared", "-o", so, os.path.join(CSRC, "sched_api.cu")]
    subprocess.check_call(cmd)
    return so


def build_emu(force: bool = False) -> str:
    emu_h = os.path.join(ROOT, "tests", "cuda_emu", "cuda_emu.h")
    if force or _stale(EMU_SO, [emu_h]):
        os.makedirs(os.path.dirname(EMU_SO), exist_ok=True)
        cmd = ["g++", "-O1", "-g", "-std=c++20", "-DCRANE_EMU", "-ffp-contract=off", "-pthread", "-fPIC", "-shared",
               "-I", os.path.join(ROOT, "tests", "cuda_emu"), "-x", "c++", os.path.join(CSRC, "sched_api.cu"),
               "-o", EMU_SO]
        subprocess.check_call(cmd)
    return EMU_SO


if __name__ == "__main__":
    import sys
    if "prof" in sys.argv:
        print(build_prof())
    elif "emu" in sys.argv:
        print(build_emu(force=True))
    else:
        print(build_cuda(force=True, verbose="-v" in sys.argv))
