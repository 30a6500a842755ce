"""ctypes front-end of oracle/libcrane_step_oracle.so, the CPU oracle of the step
scheduler (TEST INFRASTRUCTURE ONLY)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from cranesched_b200 import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libcrane_step_oracle.so")
_SRC = ("step_oracle.cpp", "crane_step_oracle.h", "crane_oracle.cpp", "crane_oracle.h", "../include/crane_sched.h")
_lib = None


def build(force: bool = False) -> str:
    """g++ with the flags of oracle/Makefile (no reference sources needed)."""
    deps = [os.path.join(_HERE, s) for s in _SRC]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(d) > os.path.getmtime(_SO) for d in deps):
        subprocess.check_call(["g++", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-std=c++20", "-fPIC",
                               "-Wall", "-Wextra", "-Wno-unused-parameter", "-shared", "-o", _SO,
                               os.path.join(_HERE, "step_oracle.cpp")])
    return _SO


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        _lib = C.CDLL(_SO)
        _lib.crane_oracle_schedule_steps.restype = C.c_int
        _lib.crane_oracle_schedule_steps.argtypes = [
            C.POINTER(abi.ClusterC), C.POINTER(abi.StepJobsC), C.POINTER(abi.StepsC),
            C.POINTER(abi.StepPlacementsC), C.c_void_p, C.POINTER(C.c_double)]
    return _lib


def schedule_steps(cluster: abi.Cluster, jobs: abi.StepJobs, steps: abi.Steps, visit=None):
    """Returns (StepPlacements, elapsed_ms of the scheduling loop); jobs.avail is updated in place.
    visit: per (job, node) row, the job-local node positions in walk order (None = index order)."""
    out = abi.StepPlacements.for_steps(jobs, steps)
    v = None if visit is None else np.ascontiguousarray(visit, np.uint32)
    c_cl, c_j, c_s, c_o = cluster.as_c(), jobs.as_c(), steps.as_c(), out.as_c()
    ms = C.c_double(0.0)
    rc = lib().crane_oracle_schedule_steps(C.byref(c_cl), C.byref(c_j), C.byref(c_s), C.byref(c_o),
                                           None if v is None else v.ctypes.data, C.byref(ms))
    if rc != 0:
        raise RuntimeError(f"crane_oracle_schedule_steps rc={rc}")
    return out, ms.value
