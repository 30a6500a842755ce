"""Host-side mirror of the reference interface for the scheduling hot path.

`GpuScheduler.node_select(now, running, pending)` has the argument meaning and
error behaviour of `SchedulerAlgo::NodeSelect(now, running_jobs, pending_jobs)`
(reference: src/CraneCtld/JobScheduler.h:254-257): per-job failure is a pending
reason, never an exception; malformed input / missing device raises.

The work happens in the C-ABI library cranesched_b200/csrc/libcrane_sched.so
(hand-written sm_90a kernels). There is no CPU path: if the library is missing
or no CUDA device is present, construction fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libcrane_sched.so")
_libs: dict[str, C.CDLL] = {}


class CraneSchedError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"crane_sched error {code}: {msg}")
        self.code = code


def load_library(path: str | None = None) -> C.CDLL:
    path = path or os.environ.get("CRANE_SCHED_LIB") or LIB_PATH  # env override: A/B builds in tools/
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise FileNotFoundError(
            f"{path} not found: build it with `python -m cranesched_b200.build` "
            "(nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(path)
    P = C.POINTER
    lib.crane_sched_create.restype = C.c_int
    lib.crane_sched_create.argtypes = [P(abi.SchedConfig), C.c_int, P(C.c_void_p)]
    lib.crane_sched_destroy.restype = None
    lib.crane_sched_destroy.argtypes = [C.c_void_p]
    lib.crane_sched_last_error.restype = C.c_char_p
    lib.crane_sched_last_error.argtypes = [C.c_void_p]
    lib.crane_sched_set_cluster.restype = C.c_int
    lib.crane_sched_set_cluster.argtypes = [C.c_void_p, P(abi.ClusterC)]
    lib.crane_sched_node_select.restype = C.c_int
    lib.crane_sched_node_select.argtypes = [C.c_void_p, C.c_int64, P(abi.RunningC), P(abi.PendingC), P(abi.PlacementsC)]
    lib.crane_sched_upload.restype = C.c_int
    lib.crane_sched_upload.argtypes = [C.c_void_p, P(abi.RunningC), P(abi.PendingC)]
    lib.crane_sched_run.restype = C.c_int
    lib.crane_sched_run.argtypes = [C.c_void_p, C.c_int64]
    lib.crane_sched_fetch.restype = C.c_int
    lib.crane_sched_fetch.argtypes = [C.c_void_p, P(abi.PlacementsC)]
    lib.crane_sched_sync.restype = C.c_int
    lib.crane_sched_sync.argtypes = [C.c_void_p, P(C.c_float)]
    lib.crane_sched_get_timing.restype = C.c_int
    lib.crane_sched_get_timing.argtypes = [C.c_void_p, P(abi.TimingC)]
    lib.crane_sched_qos_filter.restype = C.c_int
    lib.crane_sched_qos_filter.argtypes = [C.c_void_p, P(abi.QosTableC), C.c_void_p]
    lib.crane_sched_set_reservations.restype = C.c_int
    lib.crane_sched_set_reservations.argtypes = [C.c_void_p, P(abi.ReservationsC)]
    lib.crane_sched_pending_reset.restype = C.c_int
    lib.crane_sched_pending_reset.argtypes = [C.c_void_p]
    lib.crane_sched_pending_append.restype = C.c_int
    lib.crane_sched_pending_append.argtypes = [C.c_void_p, P(abi.PendingC), P(C.c_uint32)]
    lib.crane_sched_pending_erase.restype = C.c_int
    lib.crane_sched_pending_erase.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    lib.crane_sched_set_running.restype = C.c_int
    lib.crane_sched_set_running.argtypes = [C.c_void_p, P(abi.RunningC)]
    lib.crane_sched_pending_rows.restype = C.c_uint32
    lib.crane_sched_pending_rows.argtypes = [C.c_void_p]
    lib.crane_sched_running_append.restype = C.c_int
    lib.crane_sched_running_append.argtypes = [C.c_void_p, P(abi.RunningC), P(C.c_uint32)]
    lib.crane_sched_running_erase.restype = C.c_int
    lib.crane_sched_running_erase.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    lib.crane_sched_start.restype = C.c_int
    lib.crane_sched_start.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, P(C.c_uint32)]
    lib.crane_sched_keep_running.restype = C.c_int
    lib.crane_sched_keep_running.argtypes = [C.c_void_p, P(C.c_float)]
    lib.crane_sched_running_rows.restype = C.c_uint32
    lib.crane_sched_running_rows.argtypes = [C.c_void_p]
    lib.crane_sched_pending_set_gate.restype = C.c_int
    lib.crane_sched_pending_set_gate.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.crane_sched_pending_depend.restype = C.c_int
    lib.crane_sched_pending_depend.argtypes = [C.c_void_p, P(abi.DependenciesC)]
    lib.crane_sched_pending_cancel.restype = C.c_int
    lib.crane_sched_pending_cancel.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int64]
    lib.crane_sched_running_end.restype = C.c_int
    lib.crane_sched_running_end.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.crane_sched_set_shard.restype = C.c_int
    lib.crane_sched_set_shard.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.crane_sched_device_placements.restype = C.c_int
    lib.crane_sched_device_placements.argtypes = [C.c_void_p, P(abi.DevicePlacementsC)]
    lib.crane_sched_debug_bitmap.restype = C.c_int
    lib.crane_sched_debug_bitmap.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, P(C.c_uint32), P(C.c_uint32)]
    lib.crane_sched_debug_profile.restype = C.c_int
    lib.crane_sched_debug_profile.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    lib.crane_sched_schedule_steps.restype = C.c_int
    lib.crane_sched_schedule_steps.argtypes = [C.c_void_p, P(abi.StepJobsC), P(abi.StepsC), P(abi.StepPlacementsC),
                                               P(C.c_float)]
    lib.crane_sched_step_jobs_start.restype = C.c_int
    lib.crane_sched_step_jobs_start.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, P(C.c_uint32)]
    lib.crane_sched_step_jobs_append.restype = C.c_int
    lib.crane_sched_step_jobs_append.argtypes = [C.c_void_p, P(abi.StepJobsC), P(C.c_uint32)]
    lib.crane_sched_step_jobs_erase.restype = C.c_int
    lib.crane_sched_step_jobs_erase.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    lib.crane_sched_steps_append.restype = C.c_int
    lib.crane_sched_steps_append.argtypes = [C.c_void_p, P(abi.StepsC), C.c_void_p, P(C.c_uint32)]
    lib.crane_sched_steps_erase.restype = C.c_int
    lib.crane_sched_steps_erase.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    lib.crane_sched_steps_run.restype = C.c_int
    lib.crane_sched_steps_run.argtypes = [C.c_void_p, P(C.c_uint32), P(C.c_uint32), P(C.c_uint32), P(C.c_float)]
    lib.crane_sched_steps_fetch.restype = C.c_int
    lib.crane_sched_steps_fetch.argtypes = [C.c_void_p, P(abi.StepResultsC)]
    lib.crane_sched_step_jobs_avail.restype = C.c_int
    lib.crane_sched_step_jobs_avail.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, P(C.c_uint32)]
    lib.crane_sched_step_jobs_reset.restype = C.c_int
    lib.crane_sched_step_jobs_reset.argtypes = [C.c_void_p]
    lib.crane_sched_compact.restype = C.c_int
    lib.crane_sched_compact.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.crane_sched_step_rows.restype = C.c_int
    lib.crane_sched_step_rows.argtypes = [C.c_void_p, P(C.c_uint32), P(C.c_uint32), P(C.c_uint32)]
    lib.crane_sched_steps_compact.restype = C.c_int
    lib.crane_sched_steps_compact.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    _libs[path] = lib
    return lib


EXPORTS = ("crane_sched_create", "crane_sched_destroy", "crane_sched_last_error",
           "crane_sched_set_cluster", "crane_sched_set_reservations", "crane_sched_node_select", "crane_sched_upload", "crane_sched_pending_reset", "crane_sched_pending_append", "crane_sched_pending_erase",
           "crane_sched_set_running", "crane_sched_pending_rows", "crane_sched_running_append",
           "crane_sched_running_erase", "crane_sched_start", "crane_sched_keep_running", "crane_sched_running_rows",
           "crane_sched_run", "crane_sched_fetch", "crane_sched_sync", "crane_sched_get_timing",
           "crane_sched_qos_filter", "crane_sched_set_shard", "crane_sched_device_placements",
           "crane_sched_debug_bitmap", "crane_sched_debug_profile", "crane_sched_schedule_steps",
           "crane_sched_pending_set_gate", "crane_sched_pending_depend", "crane_sched_pending_cancel",
           "crane_sched_running_end", "crane_sched_step_jobs_start", "crane_sched_step_jobs_append",
           "crane_sched_step_jobs_erase", "crane_sched_steps_append", "crane_sched_steps_erase", "crane_sched_steps_run",
           "crane_sched_steps_fetch", "crane_sched_step_jobs_avail", "crane_sched_step_jobs_reset",
           "crane_sched_compact", "crane_sched_step_rows", "crane_sched_steps_compact")


class GpuScheduler:
    """One handle per GPU; owns the device-resident node, job and timeline tables."""

    def __init__(self, cfg: abi.Config, device: int = 0, lib_path: str | None = None):
        self._lib = load_library(lib_path)
        self._h = C.c_void_p()
        c_cfg = cfg.as_c()
        rc = self._lib.crane_sched_create(C.byref(c_cfg), device, C.byref(self._h))
        if rc != 0:
            raise CraneSchedError(rc, "crane_sched_create failed (no CUDA device?)" if rc == abi.ENODEV else "crane_sched_create")
        self.cfg = cfg
        self._keep = []

    def close(self):
        if self._h:
            self._lib.crane_sched_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            raise CraneSchedError(rc, (self._lib.crane_sched_last_error(self._h) or b"").decode())

    def set_cluster(self, cluster: abi.Cluster):
        c = cluster.as_c()
        self._check(self._lib.crane_sched_set_cluster(self._h, C.byref(c)))
        self.cluster = cluster

    def set_reservations(self, resv: "abi.Reservations | None"):
        """ResvMeta snapshot (JobScheduler.cpp:5655-5713); after set_cluster."""
        c = resv.as_c() if resv is not None else None
        self._check(self._lib.crane_sched_set_reservations(self._h, C.byref(c) if c is not None else None))

    # --- the NodeSelect call, host buffers in / host buffers out ------------
    def node_select(self, now: int, running: abi.Running, pending: abi.Pending,
                    out: abi.Placements | None = None) -> abi.Placements:
        out = out if out is not None else abi.Placements.for_pending(pending)
        c_rn, c_pd, c_out = running.as_c(), pending.as_c(), out.as_c()
        self._check(self._lib.crane_sched_node_select(self._h, now, C.byref(c_rn), C.byref(c_pd), C.byref(c_out)))
        return out

    # --- the same call split at the PCIe boundary ----------------------------
    def upload(self, running: abi.Running, pending: abi.Pending):
        c_rn, c_pd = running.as_c(), pending.as_c()
        self._keep = [running, pending]
        self._check(self._lib.crane_sched_upload(self._h, C.byref(c_rn), C.byref(c_pd)))

    # --- the pending table resident on the device across ticks ---------------------
    def pending_reset(self):
        self._check(self._lib.crane_sched_pending_reset(self._h))

    def pending_append(self, rows: abi.Pending) -> int:
        """Submit (JobScheduler.cpp:4254): returns the index of the first new row."""
        c, first = rows.as_c(), C.c_uint32(0)
        self._check(self._lib.crane_sched_pending_append(self._h, C.byref(c), C.byref(first)))
        return first.value

    def pending_erase(self, rows):
        r = np.ascontiguousarray(rows, np.uint32)
        self._check(self._lib.crane_sched_pending_erase(self._h, r.ctypes.data, len(r)))

    def set_running(self, running: abi.Running):
        c = running.as_c()
        self._check(self._lib.crane_sched_set_running(self._h, C.byref(c)))

    def pending_rows(self) -> int:
        return int(self._lib.crane_sched_pending_rows(self._h))

    # --- the running table resident on the device across ticks ----------------------
    def running_append(self, rows: abi.Running) -> int:
        """Running jobs from the host (recovery, jobs started elsewhere): returns the
        index of the first new row."""
        c, first = rows.as_c(), C.c_uint32(0)
        self._check(self._lib.crane_sched_running_append(self._h, C.byref(c), C.byref(first)))
        return first.value

    def running_erase(self, rows):
        """Jobs that ended or were cancelled (FreeResourceFromNode): their rows become tombstones."""
        r = np.ascontiguousarray(rows, np.uint32)
        self._check(self._lib.crane_sched_running_erase(self._h, r.ctypes.data, len(r)))

    def start(self, pending_rows) -> int:
        """Moves pending rows the last run starts now into the running table, on the device
        (JobScheduler.cpp:1273-1305); returns the running row of the first one."""
        r = np.ascontiguousarray(pending_rows, np.uint32)
        first = C.c_uint32(0)
        self._check(self._lib.crane_sched_start(self._h, r.ctypes.data, len(r), C.byref(first)))
        return first.value

    def keep_running(self) -> float:
        """The next run uses the running table as it stands on the device; returns the
        device ms of the regroup."""
        ms = C.c_float(0.0)
        self._check(self._lib.crane_sched_keep_running(self._h, C.byref(ms)))
        return ms.value

    def running_rows(self) -> int:
        return int(self._lib.crane_sched_running_rows(self._h))

    # --- the gate of the resident pending table: hold, begin time, dependencies --------
    def pending_set_gate(self, rows, held=None, begin_time=None):
        """Hold flag and / or begin time of resident rows (None = unchanged)."""
        r = np.ascontiguousarray(rows, np.uint32)
        hd = None if held is None else np.ascontiguousarray(held, np.uint8)
        bt = None if begin_time is None else np.ascontiguousarray(begin_time, np.int64)
        for a in (hd, bt):
            if a is not None and len(a) != len(r):
                raise ValueError("pending_set_gate: one value per row")
        self._check(self._lib.crane_sched_pending_set_gate(self._h, r.ctypes.data, len(r),
                                                           None if hd is None else hd.ctypes.data,
                                                           None if bt is None else bt.ctypes.data))

    def pending_depend(self, deps: abi.Dependencies):
        """Dependency lists of pending rows (SetDependency + AddDependent at submit)."""
        c = deps.as_c()
        self._check(self._lib.crane_sched_pending_depend(self._h, C.byref(c)))

    def pending_cancel(self, rows, cancel_time: int):
        """pending_erase of cancelled jobs plus their dependency events."""
        r = np.ascontiguousarray(rows, np.uint32)
        self._check(self._lib.crane_sched_pending_cancel(self._h, r.ctypes.data, len(r), cancel_time))

    def running_end(self, rows, end_time, exit_code):
        """running_erase of ended jobs plus their dependency events."""
        r = np.ascontiguousarray(rows, np.uint32)
        t = np.ascontiguousarray(end_time, np.int64)
        c = np.ascontiguousarray(exit_code, np.uint32)
        if len(t) != len(r) or len(c) != len(r):
            raise ValueError("running_end: one end time and one exit code per row")
        self._check(self._lib.crane_sched_running_end(self._h, r.ctypes.data, len(r), t.ctypes.data, c.ctypes.data))

    def compact(self, maps: bool = True) -> tuple[np.ndarray | None, np.ndarray | None]:
        """Drops the erased rows of the resident pending and running tables and the resolved
        dependency entries, on the device. Returns (pending_map, running_map): uint32, the
        new row of every old row or abi.ROW_NONE for an erased one (None, None when `maps`
        is false: the call then passes NULL maps)."""
        pm = np.zeros(self.pending_rows(), np.uint32) if maps else None
        rm = np.zeros(self.running_rows(), np.uint32) if maps else None
        self._check(self._lib.crane_sched_compact(self._h, None if pm is None else pm.ctypes.data,
                                                  None if rm is None else rm.ctypes.data))
        return pm, rm

    def run(self, now: int):
        self._check(self._lib.crane_sched_run(self._h, now))

    def sync(self) -> float:
        """Waits for the handle's stream; returns the device ms of the last run."""
        ms = C.c_float(0.0)
        self._check(self._lib.crane_sched_sync(self._h, C.byref(ms)))
        return ms.value

    def fetch(self, out: abi.Placements) -> abi.Placements:
        c_out = out.as_c()
        self._check(self._lib.crane_sched_fetch(self._h, C.byref(c_out)))
        return out

    # --- one queue over several GPUs (include/crane_sched.h: crane_sched_set_shard) ---
    def set_shard(self, rank: int, n_ranks: int, part_owner):
        import numpy as np
        owner = np.ascontiguousarray(part_owner, np.uint32) if part_owner is not None else None
        self._check(self._lib.crane_sched_set_shard(self._h, rank, n_ranks, owner.ctypes.data if owner is not None else None))

    def device_placements(self) -> "abi.DevicePlacementsC":
        d = abi.DevicePlacementsC()
        self._check(self._lib.crane_sched_device_placements(self._h, C.byref(d)))
        return d

    def qos_filter(self, qos: abi.QosTable, reason: np.ndarray) -> np.ndarray:
        """CheckAndMallocQosResource pass of the commit loop (JobScheduler.cpp:1262)
        over the placements of the last run; updates `reason` and qos.*_usage."""
        c_q = qos.as_c()
        self._check(self._lib.crane_sched_qos_filter(self._h, C.byref(c_q), reason.ctypes.data))
        return reason

    # --- the step scheduler of running jobs ------------------------------------------
    def schedule_steps(self, jobs: abi.StepJobs, steps: abi.Steps,
                       out: abi.StepPlacements | None = None) -> tuple[abi.StepPlacements, float]:
        """JobInCtld::SchedulePendingSteps for every job of `jobs` (CtldPublicDefs.cpp:1877-1998),
        after set_cluster (its gres dictionary). jobs.avail is updated in place.
        Returns (placements, device ms of the step kernel)."""
        out = out if out is not None else abi.StepPlacements.for_steps(jobs, steps)
        c_j, c_s, c_o, ms = jobs.as_c(), steps.as_c(), out.as_c(), C.c_float(0.0)
        self._check(self._lib.crane_sched_schedule_steps(self._h, C.byref(c_j), C.byref(c_s), C.byref(c_o), C.byref(ms)))
        return out, ms.value

    # --- the step state of running jobs kept resident on the device -------------------
    def step_jobs_start(self, running_rows) -> int:
        """Running rows become step jobs whose avail is their allocation
        (SetStepResAvail, JobScheduler.cpp:1277); returns the first new step-job row."""
        r = np.ascontiguousarray(running_rows, np.uint32)
        first = C.c_uint32(0)
        self._check(self._lib.crane_sched_step_jobs_start(self._h, r.ctypes.data, len(r), C.byref(first)))
        return first.value

    def step_jobs_append(self, jobs: abi.StepJobs) -> int:
        """Step jobs from host rows (a crun primary, a job started elsewhere, recovery);
        jobs.step_off is not sent. Returns the first new step-job row."""
        c, first = jobs.as_c(), C.c_uint32(0)
        c.step_off = None
        self._check(self._lib.crane_sched_step_jobs_append(self._h, C.byref(c), C.byref(first)))
        return first.value

    def step_jobs_erase(self, rows):
        """Jobs that left the running map: they and their steps go, nothing is released."""
        r = np.ascontiguousarray(rows, np.uint32)
        self._check(self._lib.crane_sched_step_jobs_erase(self._h, r.ctypes.data, len(r)))

    def steps_append(self, steps: abi.Steps, job_row) -> int:
        """AddStep: pending steps at the tail of their jobs' queues; returns the first new step row."""
        j = np.ascontiguousarray(job_row, np.uint32)
        if len(j) != steps.n:
            raise ValueError("steps_append: one job row per step")
        c, first = steps.as_c(), C.c_uint32(0)
        self._check(self._lib.crane_sched_steps_append(self._h, C.byref(c), j.ctypes.data, C.byref(first)))
        return first.value

    def steps_erase(self, rows):
        """EraseStep: pending rows leave their queue, scheduled rows give their allocation back."""
        r = np.ascontiguousarray(rows, np.uint32)
        self._check(self._lib.crane_sched_steps_erase(self._h, r.ctypes.data, len(r)))

    def steps_run(self) -> tuple[abi.StepResults, float]:
        """One pass of the step scheduler over the resident tables, then its results.
        Returns (results, device ms of the pass's kernels)."""
        n, nr, tr, ms = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0), C.c_float(0.0)
        self._check(self._lib.crane_sched_steps_run(self._h, C.byref(n), C.byref(nr), C.byref(tr), C.byref(ms)))
        out = abi.StepResults.sized(n.value, nr.value, tr.value)
        c = out.as_c()
        self._check(self._lib.crane_sched_steps_fetch(self._h, C.byref(c)))
        return out, ms.value

    def step_jobs_avail(self, rows) -> np.ndarray:
        """The avail rows of step jobs `rows`, one job after another."""
        r = np.ascontiguousarray(rows, np.uint32)
        n = C.c_uint32(0)
        self._check(self._lib.crane_sched_step_jobs_avail(self._h, r.ctypes.data, len(r), None, C.byref(n)))
        dst = np.zeros(n.value, abi.RES_IN_NODE)
        self._check(self._lib.crane_sched_step_jobs_avail(self._h, r.ctypes.data, len(r), dst.ctypes.data, None))
        return dst

    def step_jobs_reset(self):
        self._check(self._lib.crane_sched_step_jobs_reset(self._h))

    def step_rows(self) -> tuple[int, int, int]:
        """(step jobs, steps, allocation-pool rows) of the resident step tables, tombstones included."""
        j, s, a = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
        self._check(self._lib.crane_sched_step_rows(self._h, C.byref(j), C.byref(s), C.byref(a)))
        return j.value, s.value, a.value

    def steps_compact(self, maps: bool = True) -> tuple[np.ndarray | None, np.ndarray | None]:
        """Drops the erased step jobs, the erased steps and the steps of erased jobs, and
        the allocation rows of the steps that go, on the device; running steps keep their
        allocation. Returns (step_job_map, step_map): uint32, the new row of every old row
        or abi.ROW_NONE (None, None when `maps` is false: the call then passes NULL maps)."""
        j, s, _ = self.step_rows()
        jm = np.zeros(j, np.uint32) if maps else None
        sm = np.zeros(s, np.uint32) if maps else None
        self._check(self._lib.crane_sched_steps_compact(self._h, None if jm is None else jm.ctypes.data,
                                                        None if sm is None else sm.ctypes.data))
        return jm, sm

    def timing(self) -> dict:
        t = abi.TimingC()
        self._check(self._lib.crane_sched_get_timing(self._h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in abi.TimingC._fields_}

    def debug_profile(self):
        import numpy as np
        buf = np.zeros((self.cluster.n_partitions, 16), np.uint64)
        self._check(self._lib.crane_sched_debug_profile(self._h, buf.ctypes.data, buf.size))
        return buf

    def debug_bitmap(self):
        import numpy as np
        rows, wpr = C.c_uint32(0), C.c_uint32(0)
        self._check(self._lib.crane_sched_debug_bitmap(self._h, None, 0, C.byref(rows), C.byref(wpr)))
        buf = np.zeros((rows.value, wpr.value), np.uint32)
        if buf.size:
            self._check(self._lib.crane_sched_debug_bitmap(self._h, buf.ctypes.data, buf.size, C.byref(rows), C.byref(wpr)))
        return buf
