"""ctypes front-end of oracle/_ref/libcrane_ref_steps.so — the reference's own
JobInCtld::SchedulePendingSteps compiled from its source text (oracle/ref_step_build.py).
TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C

import numpy as np

from cranesched_b200 import abi
from oracle import ref_step_build

_lib = None


def available() -> bool:
    return ref_step_build.build() is not None


def lib():
    global _lib
    if _lib is None:
        so = ref_step_build.build()
        if so is None:
            raise RuntimeError("oracle/_ref/libcrane_ref_steps.so is not built and /root/reference is absent")
        _lib = C.CDLL(so)
        _lib.crane_ref_schedule_steps.restype = C.c_int
        _lib.crane_ref_schedule_steps.argtypes = [
            C.POINTER(abi.ClusterC), C.POINTER(abi.StepJobsC), C.POINTER(abi.StepsC), C.c_void_p,
            C.POINTER(abi.StepPlacementsC), C.c_void_p, C.POINTER(C.c_double)]
    return _lib


def schedule_steps(cluster: abi.Cluster, jobs: abi.StepJobs, steps: abi.Steps, erased=None):
    """Returns (StepPlacements, visit, elapsed_ms); jobs.avail is updated in place. visit holds, per
    (job, node) row, the job-local node positions in the order the reference walked them."""
    out = abi.StepPlacements.for_steps(jobs, steps)
    visit = np.zeros(int(jobs.node_off[-1]), np.uint32)
    er = None if erased is None else np.ascontiguousarray(erased, np.uint8)
    c_cl, c_j, c_s, c_o = cluster.as_c(), jobs.as_c(), steps.as_c(), out.as_c()
    ms = C.c_double(0.0)
    rc = lib().crane_ref_schedule_steps(C.byref(c_cl), C.byref(c_j), C.byref(c_s),
                                        None if er is None else er.ctypes.data, C.byref(c_o),
                                        visit.ctypes.data, C.byref(ms))
    if rc != 0:
        raise RuntimeError(f"crane_ref_schedule_steps rc={rc}")
    return out, visit, ms.value
