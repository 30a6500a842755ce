"""ctypes / numpy mirror of include/crane_sched.h.

Pure layout definitions: no CUDA, no oracle. The structs here are the POD types
that cross the C-ABI boundary which replaces SchedulerAlgo::NodeSelect
(reference: src/CraneCtld/JobScheduler.h:254-257, JobScheduler.cpp:1141).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

CORE_WORDS = 4
GRES_ENTRIES = 8
GRES_NAMES = 8
MAX_SLOTS = 16

OK = 0
EINVAL = -22
ENOMEM = -12
ENODEV = -19
ECUDA = -5
ENOSYS = -38

REASON_NONE = 0
REASON_PRIORITY = 1
REASON_RESOURCE = 2
REASON_RESERVED = 3
REASON_PART_NOT_FOUND = 4
REASON_RESV_NOT_FOUND = 5
REASON_HELD = 7
REASON_BEGIN_TIME = 8
REASON_DEPENDENCY = 9
REASON_DEPENDENCY_NEVER = 10
REASON_ERASED = 255  # a row removed from the device-resident pending table
ROW_NONE = 0xFFFFFFFF  # crane_sched_compact: the map entry of an erased row
REASON_QOS_CPU = 16
REASON_QOS_JOBS = 17
REASON_QOS_WALL = 18
REASON_QOS_MEM = 19
REASON_QOS_GRES = 20
REASON_QOS_INVALID = 21
REASON_STR = {
    0: "",
    1: "Priority",
    2: "Resource",
    3: "Resource Reserved",
    4: "Partition Not Found",
    7: "Held",
    8: "BeginTime",
    9: "Dependency",
    10: "DependencyNeverSatisfied",
    16: "QosCpuResourceLimit",
    17: "QosJobsResourceLimit",
    18: "QosWallTimeLimit",
    19: "QosMemResourceLimit",
    20: "QosGresResourceLimit",
    21: "InvalidQOS",
}

# ResourceInNodeV3 as bit masks (PublicHeader.h:562-615) -- 72 bytes
RES_IN_NODE = np.dtype(
    [
        ("cpu_raw", "<i8"),
        ("mem", "<u8"),
        ("mem_sw", "<u8"),
        ("core", "<u8", (CORE_WORDS,)),
        ("gres", "<u2", (GRES_ENTRIES,)),
    ]
)
# ResourceView as counts (PublicHeader.h:671-737) -- 56 bytes
RES_VIEW = np.dtype(
    [
        ("cpu_raw", "<i8"),
        ("mem", "<u8"),
        ("mem_sw", "<u8"),
        ("gres_total", "<u2", (GRES_NAMES,)),
        ("gres_spec", "<u2", (GRES_ENTRIES,)),
    ]
)
assert RES_IN_NODE.itemsize == 72 and RES_VIEW.itemsize == 56
# crane_tres_limit_t: a ResourceView limit of struct Qos (Account/AccountDefs.h:27-50) -- 64 bytes
TRES_LIMIT = np.dtype(
    [
        ("view", RES_VIEW),
        ("gres_name_present", "u1"),
        ("gres_spec_present", "u1"),
        ("pad", "u1", (6,)),
    ]
)
# crane_meta_resource_t: MetaResource (Accounting/AccountMetaContainer.h:30-47) -- 104 bytes
META_RESOURCE = np.dtype(
    [
        ("cpu_raw", "<i8"),
        ("mem", "<u8"),
        ("mem_sw", "<u8"),
        ("gres_total", "<u4", (GRES_NAMES,)),
        ("gres_spec", "<u4", (GRES_ENTRIES,)),
        ("jobs_count", "<u4"),
        ("pad", "<u4"),
        ("wall_time", "<i8"),
    ]
)
assert TRES_LIMIT.itemsize == 64 and META_RESOURCE.itemsize == 104

_p = C.c_void_p


class SchedConfig(C.Structure):
    _fields_ = [
        ("priority_type", C.c_uint32),
        ("favor_small", C.c_uint32),
        ("max_age_s", C.c_uint64),
        ("weight_age", C.c_uint32),
        ("weight_fair_share", C.c_uint32),
        ("weight_job_size", C.c_uint32),
        ("weight_partition", C.c_uint32),
        ("weight_qos", C.c_uint32),
        ("scheduled_batch_size", C.c_uint32),
        ("max_jobs_per_node", C.c_uint32),
        ("cost_policy", C.c_uint32),
        ("max_time_window_s", C.c_int64),
    ]


class ClusterC(C.Structure):
    _fields_ = [
        ("n_nodes", C.c_uint32),
        ("res_total", _p),
        ("alive", _p),
        ("drain", _p),
        ("n_partitions", C.c_uint32),
        ("part_off", _p),
        ("part_nodes", _p),
        ("n_gres_entries", C.c_uint32),
        ("gres_entry_name", C.c_uint8 * GRES_ENTRIES),
    ]


class RunningC(C.Structure):
    _fields_ = [
        ("n", C.c_uint32),
        ("start_time", _p),
        ("end_time", _p),
        ("node_num", _p),
        ("partition_priority", _p),
        ("qos_priority", _p),
        ("account", _p),
        ("view_cpu_raw", _p),
        ("view_mem", _p),
        ("alloc_off", _p),
        ("alloc_node", _p),
        ("alloc_res", _p),
        ("reservation", _p),
    ]


class PendingC(C.Structure):
    _fields_ = [
        ("n", C.c_uint32),
        ("partition", _p),
        ("time_limit", _p),
        ("submit_time", _p),
        ("node_num", _p),
        ("ntasks", _p),
        ("ntasks_per_node_min", _p),
        ("ntasks_per_node_max", _p),
        ("exclusive", _p),
        ("partition_priority", _p),
        ("qos_priority", _p),
        ("account", _p),
        ("qos", _p),
        ("user", _p),
        ("mandated_priority", _p),
        ("req_node", _p),
        ("req_task", _p),
        ("req_total", _p),
        ("incl_off", _p),
        ("incl_nodes", _p),
        ("excl_off", _p),
        ("excl_nodes", _p),
        ("reservation", _p),
    ]


class PlacementsC(C.Structure):
    _fields_ = [
        ("reason", _p),
        ("priority", _p),
        ("start_time", _p),
        ("end_time", _p),
        ("n_alloc", _p),
        ("alloc_off", _p),
        ("alloc_node", _p),
        ("alloc_ntasks", _p),
        ("alloc_res", _p),
    ]


class QosTableC(C.Structure):
    _fields_ = [
        ("n_qos", C.c_uint32),
        ("n_users", C.c_uint32),
        ("n_accounts", C.c_uint32),
        ("valid", _p),
        ("max_jobs_per_user", _p),
        ("max_jobs_per_account", _p),
        ("max_jobs", _p),
        ("max_cpus_per_user_raw", _p),
        ("max_wall", _p),
        ("max_tres_per_user", _p),
        ("max_tres_per_account", _p),
        ("max_tres", _p),
        ("chain_off", _p),
        ("chain_acct", _p),
        ("user_usage", _p),
        ("account_usage", _p),
        ("qos_usage", _p),
    ]


class TimingC(C.Structure):
    _fields_ = [
        ("h2d_ms", C.c_float),
        ("init_ms", C.c_float),
        ("priority_ms", C.c_float),
        ("feas_ms", C.c_float),
        ("commit_ms", C.c_float),
        ("d2h_ms", C.c_float),
        ("total_ms", C.c_float),
        ("kernel_launches", C.c_uint32),
        ("qos_ms", C.c_float),
    ]


def _ptr(a):
    return None if a is None else a.ctypes.data


def _arr(a, dtype, n=None):
    a = np.ascontiguousarray(a, dtype=dtype)
    if n is not None and a.shape[0] != n:
        raise ValueError(f"expected length {n}, got {a.shape[0]}")
    return a


# ---------------------------------------------------------------------------
# SoA tables (host side). Field names follow the reference structs.
# ---------------------------------------------------------------------------
@dataclass
class Config:
    """Config::Priority + ScheduledBatchSize + JobScheduler.h:262-264."""

    priority_type: int = 1
    favor_small: bool = True
    max_age_s: int = 7 * 24 * 3600
    weight_age: int = 1000
    weight_fair_share: int = 0
    weight_job_size: int = 0
    weight_partition: int = 0
    weight_qos: int = 0
    scheduled_batch_size: int = 100_000
    max_jobs_per_node: int = 1000
    cost_policy: int = 0
    max_time_window_s: int = 7 * 24 * 3600

    def as_c(self) -> SchedConfig:
        return SchedConfig(
            self.priority_type, int(self.favor_small), self.max_age_s,
            self.weight_age, self.weight_fair_share, self.weight_job_size,
            self.weight_partition, self.weight_qos, self.scheduled_batch_size,
            self.max_jobs_per_node, self.cost_policy, self.max_time_window_s,
        )


@dataclass
class Cluster:
    res_total: np.ndarray  # RES_IN_NODE [M]
    alive: np.ndarray
    drain: np.ndarray
    part_off: np.ndarray
    part_nodes: np.ndarray
    n_gres_entries: int = 0
    gres_entry_name: tuple = ()

    def __post_init__(self):
        self.res_total = _arr(self.res_total, RES_IN_NODE)
        m = self.res_total.shape[0]
        self.alive = _arr(self.alive, np.uint8, m)
        self.drain = _arr(self.drain, np.uint8, m)
        self.part_off = _arr(self.part_off, np.uint32)
        self.part_nodes = _arr(self.part_nodes, np.uint32)

    @property
    def n_nodes(self):
        return self.res_total.shape[0]

    @property
    def n_partitions(self):
        return self.part_off.shape[0] - 1

    def as_c(self) -> ClusterC:
        names = (C.c_uint8 * GRES_ENTRIES)(*list(self.gres_entry_name) + [0] * (GRES_ENTRIES - len(self.gres_entry_name)))
        return ClusterC(
            self.n_nodes, _ptr(self.res_total), _ptr(self.alive), _ptr(self.drain),
            self.n_partitions, _ptr(self.part_off), _ptr(self.part_nodes),
            self.n_gres_entries, names,
        )


@dataclass
class Running:
    start_time: np.ndarray
    end_time: np.ndarray
    node_num: np.ndarray
    partition_priority: np.ndarray
    qos_priority: np.ndarray
    account: np.ndarray
    view_cpu_raw: np.ndarray
    view_mem: np.ndarray
    alloc_off: np.ndarray
    alloc_node: np.ndarray
    alloc_res: np.ndarray
    reservation: np.ndarray | None = None  # index into Reservations, 0xFFFFFFFF = none

    @staticmethod
    def empty() -> "Running":
        z = lambda dt: np.zeros(0, dt)
        return Running(z(np.int64), z(np.int64), z(np.uint32), z(np.uint32), z(np.uint32),
                       z(np.uint32), z(np.int64), z(np.uint64), np.zeros(1, np.uint32),
                       z(np.uint32), z(RES_IN_NODE))

    def __post_init__(self):
        n = len(self.start_time)
        self.start_time = _arr(self.start_time, np.int64, n)
        self.end_time = _arr(self.end_time, np.int64, n)
        self.node_num = _arr(self.node_num, np.uint32, n)
        self.partition_priority = _arr(self.partition_priority, np.uint32, n)
        self.qos_priority = _arr(self.qos_priority, np.uint32, n)
        self.account = _arr(self.account, np.uint32, n)
        self.view_cpu_raw = _arr(self.view_cpu_raw, np.int64, n)
        self.view_mem = _arr(self.view_mem, np.uint64, n)
        self.alloc_off = _arr(self.alloc_off, np.uint32, n + 1)
        self.alloc_node = _arr(self.alloc_node, np.uint32)
        self.alloc_res = _arr(self.alloc_res, RES_IN_NODE)
        if self.reservation is not None:
            self.reservation = _arr(self.reservation, np.uint32, n)

    @property
    def n(self):
        return len(self.start_time)

    def take(self, idx) -> "Running":
        """Rows `idx` (in the given order) as a table of their own."""
        idx = np.asarray(idx, np.int64)
        nn = (self.alloc_off[1:] - self.alloc_off[:-1]).astype(np.int64)[idx]
        off = np.zeros(len(idx) + 1, np.uint32)
        off[1:] = np.cumsum(nn)
        ent = np.repeat(self.alloc_off[:-1][idx].astype(np.int64) - off[:-1], nn) + np.arange(int(off[-1]))
        return Running(self.start_time[idx], self.end_time[idx], self.node_num[idx], self.partition_priority[idx],
                       self.qos_priority[idx], self.account[idx], self.view_cpu_raw[idx], self.view_mem[idx], off,
                       self.alloc_node[ent], self.alloc_res[ent],
                       None if self.reservation is None else self.reservation[idx])

    @staticmethod
    def concat(a: "Running", b: "Running") -> "Running":
        """The rows of `a`, then the rows of `b`."""
        cols = {f: np.concatenate([getattr(a, f), getattr(b, f)])
                for f in a.__dataclass_fields__ if f not in ("alloc_off", "reservation")}
        cols["alloc_off"] = np.concatenate([a.alloc_off, a.alloc_off[-1] + b.alloc_off[1:]])
        if a.reservation is not None or b.reservation is not None:
            none = lambda t: np.full(t.n, 0xFFFFFFFF, np.uint32)
            cols["reservation"] = np.concatenate([none(a) if a.reservation is None else a.reservation,
                                                  none(b) if b.reservation is None else b.reservation])
        return Running(**cols)

    @staticmethod
    def started(pending: "Pending", placements: "Placements", rows) -> "Running":
        """The running jobs that pending rows `rows` (in this order) become when a run
        with `placements` starts them (JobScheduler.cpp:1273-1305): start / end time from
        the placement, node_num, partition_priority, qos_priority, account and
        reservation from the pending row, the placement rows as the allocation and
        their sum as the view (allocated_res_view += AllocatedRes())."""
        rows = np.asarray(rows, np.int64)
        nn = pending.node_num[rows].astype(np.int64)
        off = np.zeros(len(rows) + 1, np.uint32)
        off[1:] = np.cumsum(nn)
        ent = np.repeat(placements.alloc_off[rows].astype(np.int64) - off[:-1], nn) + np.arange(int(off[-1]))
        res = placements.alloc_res[ent]
        job = np.repeat(np.arange(len(rows)), nn)
        cpu = np.zeros(len(rows), np.int64)
        mem = np.zeros(len(rows), np.uint64)
        np.add.at(cpu, job, res["cpu_raw"])
        np.add.at(mem, job, res["mem"])
        return Running(placements.start_time[rows], placements.end_time[rows], pending.node_num[rows],
                       pending.partition_priority[rows], pending.qos_priority[rows], pending.account[rows],
                       cpu, mem, off, placements.alloc_node[ent], res,
                       None if pending.reservation is None else pending.reservation[rows])

    def as_c(self) -> RunningC:
        return RunningC(
            self.n, _ptr(self.start_time), _ptr(self.end_time), _ptr(self.node_num),
            _ptr(self.partition_priority), _ptr(self.qos_priority), _ptr(self.account),
            _ptr(self.view_cpu_raw), _ptr(self.view_mem), _ptr(self.alloc_off),
            _ptr(self.alloc_node), _ptr(self.alloc_res), _ptr(self.reservation),
        )


@dataclass
class Pending:
    partition: np.ndarray
    time_limit: np.ndarray
    submit_time: np.ndarray
    node_num: np.ndarray
    ntasks: np.ndarray
    ntasks_per_node_min: np.ndarray
    ntasks_per_node_max: np.ndarray
    exclusive: np.ndarray
    partition_priority: np.ndarray
    qos_priority: np.ndarray
    account: np.ndarray
    qos: np.ndarray
    user: np.ndarray
    mandated_priority: np.ndarray
    req_node: np.ndarray
    req_task: np.ndarray
    req_total: np.ndarray
    incl_off: np.ndarray | None = None
    incl_nodes: np.ndarray | None = None
    excl_off: np.ndarray | None = None
    excl_nodes: np.ndarray | None = None
    reservation: np.ndarray | None = None  # index into Reservations, 0xFFFFFFFF = none

    def __post_init__(self):
        n = len(self.partition)
        u32 = lambda a: _arr(a, np.uint32, n)
        self.partition = u32(self.partition)
        self.time_limit = _arr(self.time_limit, np.int64, n)
        self.submit_time = _arr(self.submit_time, np.int64, n)
        self.node_num = u32(self.node_num)
        self.ntasks = u32(self.ntasks)
        self.ntasks_per_node_min = u32(self.ntasks_per_node_min)
        self.ntasks_per_node_max = u32(self.ntasks_per_node_max)
        self.exclusive = _arr(self.exclusive, np.uint8, n)
        self.partition_priority = u32(self.partition_priority)
        self.qos_priority = u32(self.qos_priority)
        self.account = u32(self.account)
        self.qos = u32(self.qos)
        self.user = u32(self.user)
        self.mandated_priority = _arr(self.mandated_priority, np.float64, n)
        self.req_node = _arr(self.req_node, RES_VIEW, n)
        self.req_task = _arr(self.req_task, RES_VIEW, n)
        self.req_total = _arr(self.req_total, RES_VIEW, n)
        for k in ("incl", "excl"):
            off = getattr(self, k + "_off")
            if off is not None:
                setattr(self, k + "_off", _arr(off, np.uint32, n + 1))
                setattr(self, k + "_nodes", _arr(getattr(self, k + "_nodes"), np.uint32))
        if self.reservation is not None:
            self.reservation = _arr(self.reservation, np.uint32, n)

    @property
    def n(self):
        return len(self.partition)

    def take(self, idx) -> "Pending":
        """Rows `idx` (ascending) as a table of their own."""
        idx = np.asarray(idx, np.int64)
        cols = {}
        for f in self.__dataclass_fields__:
            v = getattr(self, f)
            if v is None or f in ("incl_off", "incl_nodes", "excl_off", "excl_nodes"):
                continue
            cols[f] = v[idx]
        for k in ("incl", "excl"):
            off = getattr(self, k + "_off")
            if off is not None:
                nodes = getattr(self, k + "_nodes")
                new_off, new_nodes = [0], []
                for j in idx:
                    new_nodes += nodes[off[j]:off[j + 1]].tolist()
                    new_off.append(len(new_nodes))
                cols[k + "_off"] = np.array(new_off, np.uint32)
                cols[k + "_nodes"] = np.array(new_nodes, np.uint32)
        return Pending(**cols)

    def as_c(self) -> PendingC:
        return PendingC(
            self.n, _ptr(self.partition), _ptr(self.time_limit), _ptr(self.submit_time),
            _ptr(self.node_num), _ptr(self.ntasks), _ptr(self.ntasks_per_node_min),
            _ptr(self.ntasks_per_node_max), _ptr(self.exclusive),
            _ptr(self.partition_priority), _ptr(self.qos_priority), _ptr(self.account),
            _ptr(self.qos), _ptr(self.user), _ptr(self.mandated_priority),
            _ptr(self.req_node), _ptr(self.req_task), _ptr(self.req_total),
            _ptr(self.incl_off), _ptr(self.incl_nodes), _ptr(self.excl_off),
            _ptr(self.excl_nodes), _ptr(self.reservation),
        )


@dataclass
class Placements:
    """What NodeSelect writes into PdJobInScheduler (JobScheduler.h:116-132)."""

    reason: np.ndarray
    priority: np.ndarray
    start_time: np.ndarray
    end_time: np.ndarray
    n_alloc: np.ndarray
    alloc_off: np.ndarray
    alloc_node: np.ndarray
    alloc_ntasks: np.ndarray
    alloc_res: np.ndarray

    @staticmethod
    def for_pending(pending: Pending, pinned: bool = False) -> "Placements":
        n = pending.n
        total = int(pending.node_num.astype(np.int64).sum())
        mk = _pinned_empty if pinned else (lambda shape, dt: np.zeros(shape, dt))
        return Placements(
            mk(n, np.uint8), mk(n, np.float64), mk(n, np.int64), mk(n, np.int64),
            mk(n, np.uint32), mk(n + 1, np.uint32), mk(total, np.uint32),
            mk(total, np.uint32), mk(total, RES_IN_NODE),
        )

    def as_c(self) -> PlacementsC:
        return PlacementsC(
            _ptr(self.reason), _ptr(self.priority), _ptr(self.start_time),
            _ptr(self.end_time), _ptr(self.n_alloc), _ptr(self.alloc_off),
            _ptr(self.alloc_node), _ptr(self.alloc_ntasks), _ptr(self.alloc_res),
        )

    def nbytes(self) -> int:
        return sum(getattr(self, f).nbytes for f in self.__dataclass_fields__)

    def diff(self, other: "Placements") -> list[str]:
        """Field-by-field bit-exact comparison; returns mismatch descriptions."""
        out = []
        for f in self.__dataclass_fields__:
            a, b = getattr(self, f), getattr(other, f)
            if a.shape != b.shape:
                out.append(f"{f}: shape {a.shape} vs {b.shape}")
                continue
            if f == "priority":
                a, b = a.view(np.uint64), b.view(np.uint64)
            if a.dtype.names:
                neq = np.zeros(a.shape, bool)
                for name in a.dtype.names:
                    x, y = a[name], b[name]
                    d = x != y
                    neq |= d.reshape(len(a), -1).any(axis=1) if d.ndim > 1 else d
            else:
                neq = a != b
            if neq.any():
                idx = np.flatnonzero(neq)
                out.append(f"{f}: {len(idx)} mismatches, first at {idx[:5].tolist()}: "
                           f"{getattr(self, f)[idx[0]]} vs {getattr(other, f)[idx[0]]}")
        return out


@dataclass
class QosTable:
    """struct Qos limits (Account/AccountDefs.h:27-50), the pending jobs' account
    chains and the usage maps of AccountMetaContainer (m_user_meta_map_,
    m_account_meta_map_, m_qos_meta_map_) as dense tables."""

    n_users: int
    n_accounts: int
    valid: np.ndarray
    max_jobs_per_user: np.ndarray
    max_jobs_per_account: np.ndarray
    max_jobs: np.ndarray
    max_cpus_per_user_raw: np.ndarray
    max_wall: np.ndarray
    max_tres_per_user: np.ndarray
    max_tres_per_account: np.ndarray
    max_tres: np.ndarray
    chain_off: np.ndarray
    chain_acct: np.ndarray
    user_usage: np.ndarray | None = None
    account_usage: np.ndarray | None = None
    qos_usage: np.ndarray | None = None

    def __post_init__(self):
        q = len(self.valid)
        self.valid = _arr(self.valid, np.uint8, q)
        self.max_jobs_per_user = _arr(self.max_jobs_per_user, np.uint32, q)
        self.max_jobs_per_account = _arr(self.max_jobs_per_account, np.uint32, q)
        self.max_jobs = _arr(self.max_jobs, np.uint32, q)
        self.max_cpus_per_user_raw = _arr(self.max_cpus_per_user_raw, np.int64, q)
        self.max_wall = _arr(self.max_wall, np.int64, q)
        self.max_tres_per_user = _arr(self.max_tres_per_user, TRES_LIMIT, q)
        self.max_tres_per_account = _arr(self.max_tres_per_account, TRES_LIMIT, q)
        self.max_tres = _arr(self.max_tres, TRES_LIMIT, q)
        self.chain_off = _arr(self.chain_off, np.uint32)
        self.chain_acct = _arr(self.chain_acct, np.uint32)
        if self.user_usage is None:
            self.user_usage = np.zeros(self.n_users * q, META_RESOURCE)
        if self.account_usage is None:
            self.account_usage = np.zeros(self.n_accounts * q, META_RESOURCE)
        if self.qos_usage is None:
            self.qos_usage = np.zeros(q, META_RESOURCE)
        self.user_usage = _arr(self.user_usage, META_RESOURCE, self.n_users * q)
        self.account_usage = _arr(self.account_usage, META_RESOURCE, self.n_accounts * q)
        self.qos_usage = _arr(self.qos_usage, META_RESOURCE, q)

    @property
    def n_qos(self):
        return len(self.valid)

    def copy(self) -> "QosTable":
        import copy

        return copy.deepcopy(self)

    def as_c(self) -> QosTableC:
        return QosTableC(
            self.n_qos, self.n_users, self.n_accounts, _ptr(self.valid),
            _ptr(self.max_jobs_per_user), _ptr(self.max_jobs_per_account), _ptr(self.max_jobs),
            _ptr(self.max_cpus_per_user_raw), _ptr(self.max_wall), _ptr(self.max_tres_per_user),
            _ptr(self.max_tres_per_account), _ptr(self.max_tres), _ptr(self.chain_off),
            _ptr(self.chain_acct), _ptr(self.user_usage), _ptr(self.account_usage),
            _ptr(self.qos_usage),
        )


def _pinned_empty(shape, dt):
    """Page-locked host buffer (torch is plumbing for pinned memory only)."""
    import torch

    dt = np.dtype(dt)
    n = int(np.prod(shape)) if not isinstance(shape, int) else shape
    t = torch.zeros(max(n * dt.itemsize, 1), dtype=torch.uint8)
    try:
        t = t.pin_memory()
    except Exception:
        pass
    a = t.numpy()[: n * dt.itemsize].view(dt)
    return a.reshape(shape)  # the ndarray keeps `t` alive through .base


class DevicePlacementsC(C.Structure):
    """crane_device_placements_t: device pointers of the placement columns."""
    _fields_ = [("reason", C.c_void_p), ("start_time", C.c_void_p), ("end_time", C.c_void_p), ("n_alloc", C.c_void_p),
                ("alloc_node", C.c_void_p), ("alloc_ntasks", C.c_void_p), ("alloc_res", C.c_void_p),
                ("n_jobs", C.c_uint64), ("n_rows", C.c_uint64)]


class ReservationsC(C.Structure):
    """crane_reservations_t"""
    _fields_ = [("n", C.c_uint32), ("start_time", C.c_void_p), ("end_time", C.c_void_p), ("node_off", C.c_void_p),
                ("node", C.c_void_p), ("res", C.c_void_p)]


@dataclass
class Reservations:
    """ResvMeta table (Node/NodeDefs.h:81-97): start, end, (node, reserved resources) pairs."""
    start_time: np.ndarray
    end_time: np.ndarray
    node_off: np.ndarray
    node: np.ndarray
    res: np.ndarray

    def __post_init__(self):
        n = len(self.start_time)
        self.start_time = _arr(self.start_time, np.int64, n)
        self.end_time = _arr(self.end_time, np.int64, n)
        self.node_off = _arr(self.node_off, np.uint32, n + 1)
        self.node = _arr(self.node, np.uint32)
        self.res = _arr(self.res, RES_IN_NODE)

    @property
    def n(self):
        return len(self.start_time)

    def as_c(self) -> ReservationsC:
        return ReservationsC(self.n, _ptr(self.start_time), _ptr(self.end_time), _ptr(self.node_off),
                             _ptr(self.node), _ptr(self.res))


# ---------------------------------------------------------------------------
# The gate of the resident pending table: hold, begin time, dependencies
# ---------------------------------------------------------------------------
TIME_PAST = -(2 ** 63)     # absl::InfinitePast
TIME_FUTURE = 2 ** 63 - 1  # absl::InfiniteFuture
DEP_AFTER, DEP_AFTER_ANY, DEP_AFTER_OK, DEP_AFTER_NOT_OK = 0, 1, 2, 3  # DependencyType (PublicDefs.proto:136-141)
DEPENDEE_PENDING, DEPENDEE_RUNNING, DEPENDEE_EVENT = 0, 1, 2


class DependenciesC(C.Structure):
    """crane_dependencies_t"""
    _fields_ = [("n", C.c_uint32), ("row", _p), ("is_or", _p), ("dep_off", _p), ("kind", _p), ("dependee", _p),
                ("type", _p), ("delay_s", _p), ("event_time", _p)]


@dataclass
class Dependencies:
    """Dependency lists of pending rows: row k is pending row `row[k]`, its entries are
    [dep_off[k], dep_off[k+1]) of (kind, dependee row, type, delay, event time)."""
    row: np.ndarray
    is_or: np.ndarray
    dep_off: np.ndarray
    kind: np.ndarray
    dependee: np.ndarray
    type: np.ndarray
    delay_s: np.ndarray
    event_time: np.ndarray

    def __post_init__(self):
        n = len(self.row)
        self.row = _arr(self.row, np.uint32, n)
        self.is_or = _arr(self.is_or, np.uint8, n)
        self.dep_off = _arr(self.dep_off, np.uint32, n + 1)
        m = int(self.dep_off[-1])
        self.kind = _arr(self.kind, np.uint8, m)
        self.dependee = _arr(self.dependee, np.uint32, m)
        self.type = _arr(self.type, np.uint8, m)
        self.delay_s = _arr(self.delay_s, np.uint64, m)
        self.event_time = _arr(self.event_time, np.int64, m)

    @staticmethod
    def from_lists(rows, is_or, entries) -> "Dependencies":
        """entries[k] = list of (kind, dependee, type, delay_s, event_time) of rows[k]."""
        off = np.zeros(len(rows) + 1, np.uint32)
        off[1:] = np.cumsum([len(e) for e in entries]) if len(entries) else []
        flat = [x for e in entries for x in e]
        col = lambda i, dt: np.array([x[i] for x in flat], dt)  # noqa: E731
        return Dependencies(rows, is_or, off, col(0, np.uint8), col(1, np.uint32), col(2, np.uint8),
                            col(3, np.uint64), col(4, np.int64))

    @property
    def n(self):
        return len(self.row)

    def as_c(self) -> DependenciesC:
        return DependenciesC(self.n, _ptr(self.row), _ptr(self.is_or), _ptr(self.dep_off), _ptr(self.kind),
                             _ptr(self.dependee), _ptr(self.type), _ptr(self.delay_s), _ptr(self.event_time))


# ---------------------------------------------------------------------------
# The step scheduler of running jobs (JobInCtld::SchedulePendingSteps)
# ---------------------------------------------------------------------------
class StepJobsC(C.Structure):
    """crane_step_jobs_t"""
    _fields_ = [("n_jobs", C.c_uint32), ("node_off", _p), ("node", _p), ("avail", _p), ("step_off", _p)]


class StepsC(C.Structure):
    """crane_steps_t"""
    _fields_ = [("n", C.c_uint32), ("node_num", _p), ("ntasks", _p), ("ntasks_per_node_min", _p),
                ("ntasks_per_node_max", _p), ("req_node", _p), ("req_task", _p), ("incl_off", _p),
                ("incl_nodes", _p), ("excl_off", _p), ("excl_nodes", _p)]


class StepPlacementsC(C.Structure):
    """crane_step_placements_t"""
    _fields_ = [("placed", _p), ("scheduled", _p), ("node_off", _p), ("alloc_node", _p), ("alloc_ntasks", _p),
                ("alloc_res", _p), ("task_off", _p), ("task_node", _p), ("task_res", _p)]


@dataclass
class StepJobs:
    """Running jobs with pending steps: their nodes, step_res_avail_ (one row per
    (job, node), updated in place by the scheduler) and the CSR of their FIFO steps."""
    node_off: np.ndarray
    node: np.ndarray
    avail: np.ndarray
    step_off: np.ndarray

    def __post_init__(self):
        self.node_off = _arr(self.node_off, np.uint32)
        n = len(self.node_off) - 1
        self.node = _arr(self.node, np.uint32, int(self.node_off[-1]))
        self.avail = _arr(self.avail, RES_IN_NODE, int(self.node_off[-1]))
        self.step_off = _arr(self.step_off, np.uint32, n + 1)

    @property
    def n_jobs(self):
        return len(self.node_off) - 1

    def copy(self) -> "StepJobs":
        return StepJobs(self.node_off.copy(), self.node.copy(), self.avail.copy(), self.step_off.copy())

    def as_c(self) -> StepJobsC:
        return StepJobsC(self.n_jobs, _ptr(self.node_off), _ptr(self.node), _ptr(self.avail), _ptr(self.step_off))


@dataclass
class Steps:
    """The fields of CommonStepInCtld the step scheduler reads, one row per step."""
    node_num: np.ndarray
    ntasks: np.ndarray
    ntasks_per_node_min: np.ndarray
    ntasks_per_node_max: np.ndarray
    req_node: np.ndarray
    req_task: np.ndarray
    incl_off: np.ndarray | None = None
    incl_nodes: np.ndarray | None = None
    excl_off: np.ndarray | None = None
    excl_nodes: np.ndarray | None = None

    def __post_init__(self):
        n = len(self.node_num)
        for f in ("node_num", "ntasks", "ntasks_per_node_min", "ntasks_per_node_max"):
            setattr(self, f, _arr(getattr(self, f), np.uint32, n))
        self.req_node = _arr(self.req_node, RES_VIEW, n)
        self.req_task = _arr(self.req_task, RES_VIEW, n)
        for k in ("incl", "excl"):
            off = getattr(self, k + "_off")
            if off is not None:
                setattr(self, k + "_off", _arr(off, np.uint32, n + 1))
                setattr(self, k + "_nodes", _arr(getattr(self, k + "_nodes"), np.uint32))

    @property
    def n(self):
        return len(self.node_num)

    def as_c(self) -> StepsC:
        return StepsC(self.n, _ptr(self.node_num), _ptr(self.ntasks), _ptr(self.ntasks_per_node_min),
                      _ptr(self.ntasks_per_node_max), _ptr(self.req_node), _ptr(self.req_task),
                      _ptr(self.incl_off), _ptr(self.incl_nodes), _ptr(self.excl_off), _ptr(self.excl_nodes))


@dataclass
class StepPlacements:
    """What SchedulePendingSteps writes: per job the steps placed at the head of its
    queue, per step `scheduled`, node rows (node-index order) and task rows (task-id order)."""
    placed: np.ndarray
    scheduled: np.ndarray
    node_off: np.ndarray
    alloc_node: np.ndarray
    alloc_ntasks: np.ndarray
    alloc_res: np.ndarray
    task_off: np.ndarray
    task_node: np.ndarray
    task_res: np.ndarray

    @staticmethod
    def for_steps(jobs: StepJobs, steps: Steps) -> "StepPlacements":
        nr = int(steps.node_num.astype(np.int64).sum())
        tr = int(steps.ntasks.astype(np.int64).sum())
        z = np.zeros
        return StepPlacements(z(jobs.n_jobs, np.uint32), z(steps.n, np.uint8), z(steps.n + 1, np.uint32),
                              z(nr, np.uint32), z(nr, np.uint32), z(nr, RES_IN_NODE), z(steps.n + 1, np.uint32),
                              z(tr, np.uint32), z(tr, RES_IN_NODE))

    def as_c(self) -> StepPlacementsC:
        return StepPlacementsC(*[_ptr(getattr(self, f)) for f in self.__dataclass_fields__])

    def diff(self, other: "StepPlacements") -> list[str]:
        """Field-by-field bit-exact comparison; returns mismatch descriptions."""
        out = []
        for f in self.__dataclass_fields__:
            a, b = getattr(self, f), getattr(other, f)
            if a.shape != b.shape:
                out.append(f"{f}: shape {a.shape} vs {b.shape}")
                continue
            neq = a.view(np.uint8).reshape(len(a), -1) != b.view(np.uint8).reshape(len(b), -1)
            bad = np.flatnonzero(neq.any(axis=1)) if len(a) else np.zeros(0, int)
            if len(bad):
                out.append(f"{f}: {len(bad)} mismatches, first at {bad[:5].tolist()}: {a[bad[0]]} vs {b[bad[0]]}")
        return out

    def digest(self) -> str:
        import hashlib
        h = hashlib.sha256()
        for f in self.__dataclass_fields__:
            h.update(np.ascontiguousarray(getattr(self, f)).tobytes())
        return h.hexdigest()


# ---------------------------------------------------------------------------
# The step state of running jobs kept resident on the device (crane_sched_steps_run)
# ---------------------------------------------------------------------------
class StepResultsC(C.Structure):
    """crane_step_results_t"""
    _fields_ = [("step_row", _p), ("node_off", _p), ("alloc_node", _p), ("alloc_ntasks", _p), ("alloc_res", _p),
                ("task_off", _p), ("task_node", _p), ("task_res", _p)]


@dataclass
class StepResults:
    """What one resident pass scheduled: the step rows (ascending), their node rows
    (node-index order) and task rows (task-id order), offsets over the returned steps."""
    step_row: np.ndarray
    node_off: np.ndarray
    alloc_node: np.ndarray
    alloc_ntasks: np.ndarray
    alloc_res: np.ndarray
    task_off: np.ndarray
    task_node: np.ndarray
    task_res: np.ndarray

    @staticmethod
    def sized(n_scheduled: int, n_node_rows: int, n_task_rows: int) -> "StepResults":
        z = np.zeros
        return StepResults(z(n_scheduled, np.uint32), z(n_scheduled + 1, np.uint32), z(n_node_rows, np.uint32),
                           z(n_node_rows, np.uint32), z(n_node_rows, RES_IN_NODE), z(n_scheduled + 1, np.uint32),
                           z(n_task_rows, np.uint32), z(n_task_rows, RES_IN_NODE))

    @property
    def n(self):
        return len(self.step_row)

    def as_c(self) -> StepResultsC:
        return StepResultsC(*[_ptr(getattr(self, f)) for f in self.__dataclass_fields__])

    def diff(self, other: "StepResults") -> list[str]:
        return StepPlacements.diff(self, other)

    def digest(self) -> str:
        return StepPlacements.digest(self)

    def expand(self, step_rows, job_step_off, steps: Steps) -> StepPlacements:
        """The StepPlacements crane_sched_schedule_steps writes for `steps`, whose row s
        is resident step row step_rows[s] and whose jobs own the rows
        [job_step_off[j], job_step_off[j+1]): steps outside the results are not scheduled
        (their rows zero), `placed` counts a job's scheduled steps."""
        step_rows = np.asarray(step_rows, np.int64)
        job_step_off = np.asarray(job_step_off, np.int64)
        out = StepPlacements.for_steps(StepJobs(np.zeros(len(job_step_off), np.uint32), np.zeros(0, np.uint32),
                                                np.zeros(0, RES_IN_NODE), job_step_off), steps)
        out.node_off[1:] = np.cumsum(steps.node_num, dtype=np.int64)
        out.task_off[1:] = np.cumsum(steps.ntasks, dtype=np.int64)
        at = np.searchsorted(self.step_row, step_rows)
        hit = (at < self.n) & (self.step_row[np.minimum(at, max(self.n - 1, 0))] == step_rows) if self.n else \
            np.zeros(len(step_rows), bool)
        if int(hit.sum()) != self.n:
            raise ValueError("StepResults.expand: a returned step is not in the given step set")
        out.scheduled[hit] = 1
        for s in np.flatnonzero(hit):
            r = at[s]
            d0, n0, n1 = out.node_off[s], self.node_off[r], self.node_off[r + 1]
            out.alloc_node[d0:d0 + n1 - n0] = self.alloc_node[n0:n1]
            out.alloc_ntasks[d0:d0 + n1 - n0] = self.alloc_ntasks[n0:n1]
            out.alloc_res[d0:d0 + n1 - n0] = self.alloc_res[n0:n1]
            d0, t0, t1 = out.task_off[s], self.task_off[r], self.task_off[r + 1]
            out.task_node[d0:d0 + t1 - t0] = self.task_node[t0:t1]
            out.task_res[d0:d0 + t1 - t0] = self.task_res[t0:t1]
        job = np.repeat(np.arange(len(job_step_off) - 1), np.diff(job_step_off))
        np.add.at(out.placed, job[hit], 1)
        return out
