"""NodeSelect at the size limits of the scheduling kernels, against the oracle.

Above each limit k_commit2 or the host layout takes another code path:
  * a job of more than 32 (job, node) tasks leaves the batch path for the one-job path;
  * a placed job of more than 64 nodes re-sorts the whole cost order instead of re-keying;
  * general task distribution: top-K heaps of up to 127 nodes, 128 refused at upload;
  * nodes of res_total class >= 4 get no per-batch cost delta, a partition of more
    than 16 classes leaves the rest unclassed (the kernel reads slot_total);
  * cores 128-255 in words 2-3 and gres entries 4-7 in the second half of the packed rows;
  * a partition near the shared-memory budget gets a job ring shallower than 64.
The cases come from synth.edge_case, whose oracle is pinned to the reference's own
NodeSelect at these shapes (tests/test_edge_ref_pin.py). Every case also checks, from
its inputs and outputs, that it reaches the path it is there for.
"""
import os
import re

import numpy as np
import pytest

from cranesched_b200 import abi, synth
from tests.helpers import assert_same, check_invariants, run_sched

KMAXT = 32
KRK = 64


# ---- what a case reaches -------------------------------------------------------------
def _general(pd):
    t = pd.ntasks_per_node_min.astype(np.int64)
    return (pd.ntasks_per_node_max != pd.ntasks_per_node_min) | (t * pd.node_num != pd.ntasks)


def _order(case, out):
    cfg, pd = case[0], case[3]
    return np.arange(pd.n) if cfg.priority_type == 0 else np.argsort(-out.priority, kind="stable")


def wide_between_batches(case, out, wider_than):
    """Placed jobs of more than `wider_than` nodes with placed batch jobs (at most 32 nodes,
    uniform tasks) of the same partition both before and after them in priority order."""
    pd = case[3]
    batchable = (out.n_alloc > 0) & (pd.node_num <= KMAXT) & ~_general(pd)
    hits = []
    for p in np.unique(pd.partition):
        seq = [j for j in _order(case, out) if pd.partition[j] == p and out.n_alloc[j] > 0]
        b = np.array([batchable[j] for j in seq], bool)
        for i, j in enumerate(seq):
            if out.n_alloc[j] > wider_than and b[:i].any() and b[i + 1:].any():
                hits.append(j)
    return hits


def placed_general(case, out, nodes):
    pd = case[3]
    return np.flatnonzero((out.n_alloc == nodes) & _general(pd))


def usable_shapes(cl):
    """Distinct res_total rows among the usable nodes of every partition."""
    ok = (cl.alive == 1) & (cl.drain == 0)
    return [len({cl.res_total[n].tobytes() for n in cl.part_nodes[cl.part_off[p]:cl.part_off[p + 1]] if ok[n]})
            for p in range(cl.n_partitions)]


def placed_rows(case, out):
    pd = case[3]
    return np.repeat(out.n_alloc > 0, pd.node_num)


def high_alloc(case, out):
    """(placement rows holding cores of words 2-3, placement rows holding slots of entries 4-7)."""
    res = out.alloc_res[placed_rows(case, out)]
    return int((res["core"][:, 2:] != 0).any(1).sum()), int((res["gres"][:, 4:] != 0).any(1).sum())


def running_high_under_started(case, out):
    """Nodes where a running job ending inside the backfill window holds cores of words 2-3
    (resp. slots of entries 5-7) and a pending job was started now."""
    cfg, cl, rn, pd, now = case
    job = np.repeat(np.arange(rn.n), np.diff(rn.alloc_off.astype(np.int64)))
    ends = rn.end_time[job] < now + cfg.max_time_window_s
    started = np.repeat(out.reason == abi.REASON_NONE, pd.node_num)
    busy = set(out.alloc_node[started].tolist())
    core = {int(n) for n in rn.alloc_node[ends & (rn.alloc_res["core"][:, 2:] != 0).any(1)]} & busy
    gres = {int(n) for n in rn.alloc_node[ends & (rn.alloc_res["gres"][:, 5:] != 0).any(1)]} & busy
    return core, gres


def check_running_disjoint(case, out):
    """Cores and slots started now never overlap what running jobs hold on the node."""
    rn, pd = case[2], case[3]
    held_c = np.zeros((case[1].n_nodes, abi.CORE_WORDS), np.uint64)
    held_g = np.zeros((case[1].n_nodes, abi.GRES_ENTRIES), np.uint16)
    for n, r in zip(rn.alloc_node, rn.alloc_res):
        held_c[n] |= r["core"]
        held_g[n] |= r["gres"]
    started = np.repeat(out.reason == abi.REASON_NONE, pd.node_num)
    for n, r in zip(out.alloc_node[started], out.alloc_res[started]):
        assert not (held_c[n] & r["core"]).any(), f"node {n}: a core held by a running job started again"
        assert not (held_g[n] & r["gres"]).any(), f"node {n}: a slot held by a running job started again"


def _match(oracle, lib, case, resv=None):
    cfg, cl, rn, pd, now = case
    ref, _, _ = oracle.node_select(cfg, cl, rn, pd, now, resv=resv)
    got, _ = run_sched(case, lib, resv=resv)
    assert_same(ref, got)
    check_invariants(case, got)
    if resv is None:
        check_running_disjoint(case, got)
    return got


# ---- emulated kernels (CPU) ---------------------------------------------------------------
def test_emulated_wide_jobs_between_batches(oracle, emu_lib):
    """Jobs of 33-100 nodes between batches of narrow ones in one partition of 20 node shapes:
    the one-job path, the full re-sort after a placement of more than 64 nodes and the batches
    that follow it on the re-sorted order; unclassed nodes (class 0xff) and classes without a
    cost delta; cores of words 2-3 and entries 4-7 handed out next to running jobs holding them."""
    case = synth.edge_case(11, n_jobs=150, parts=((100, 20),), n_running=30, p_wide=0.12, p_general=0.2)
    got = _match(oracle, emu_lib, case)
    assert max(usable_shapes(case[1])) > 16
    assert wide_between_batches(case, got, KRK), "no job wider than 64 nodes placed between batch jobs"
    assert wide_between_batches(case, got, KMAXT)
    c, g = high_alloc(case, got)
    assert c > 0 and g > 0, "no allocation in core words 2-3 (%d) or gres entries 4-7 (%d)" % (c, g)
    core, gres = running_high_under_started(case, got)
    assert core and gres, "no running job holds cores of words 2-3 and slots of entries 5-7 where a job started"


def test_emulated_general_127_nodes(oracle, emu_lib):
    """A job of 127 nodes with a ntasks_per_node range (the widest top-K heap) placed in a
    partition of 8 node shapes (classes 4-7: no per-batch cost delta) beside one of 3 shapes,
    the layout with several gres types per name, FIFO."""
    case = synth.edge_case(33, n_jobs=110, parts=((134, 8), (24, 3)), n_running=20, wide=(127, 100, 65, 33),
                           p_wide=0.1, p_general=0.7, p_down=0.01, fifo=True)
    got = _match(oracle, emu_lib, case)
    shapes = usable_shapes(case[1])
    assert 5 <= shapes[0] <= 16 and shapes[1] <= 4
    assert len(placed_general(case, got, 127)), "no general job of 127 nodes placed"
    c, g = high_alloc(case, got)
    assert c > 0 and g > 0, "no allocation in core words 2-3 (%d) or gres entries 4-7 (%d)" % (c, g)


def test_emulated_bestfit_one_type_per_name(oracle, emu_lib):
    """BestFit (keys move down) with 17 shapes and the reference pin's gres layout (one type per
    name), short limits so that running jobs end inside the window and backfills land on them."""
    case = synth.edge_case(37, n_jobs=130, parts=((90, 17),), n_running=30, p_wide=0.12, cost_policy=1,
                           one_type_per_name=True, short=True)
    got = _match(oracle, emu_lib, case)
    assert usable_shapes(case[1])[0] == 17
    assert wide_between_batches(case, got, KMAXT), "no job wider than a batch placed between batch jobs"
    assert (got.n_alloc > KRK).any(), "no job wider than 64 nodes placed"
    core, gres = running_high_under_started(case, got)
    assert core and gres, "no running job holds cores of words 2-3 and slots of entries 5-7 where a job started"


# ---- refusals at the boundary -----------------------------------------------------------
def _resize(pd, j, nodes, ntasks, tmin, tmax):
    """Job j of `pd` with another shape; its total request follows (node * nodes + task * ntasks)."""
    pd.node_num[j], pd.ntasks[j] = nodes, ntasks
    pd.ntasks_per_node_min[j], pd.ntasks_per_node_max[j] = tmin, tmax
    for f in ("cpu_raw", "mem", "mem_sw"):
        pd.req_total[f][j] = int(pd.req_node[f][j]) * nodes + int(pd.req_task[f][j]) * ntasks
    for f in ("gres_total", "gres_spec"):
        pd.req_total[f][j] = pd.req_node[f][j].astype(np.int64) * nodes + pd.req_task[f][j].astype(np.int64) * ntasks


def _scheduler(lib, case):
    from cranesched_b200.scheduler import GpuScheduler
    s = GpuScheduler(case[0], 0, lib)
    s.set_cluster(case[1])
    return s


def test_general_job_of_128_nodes_is_refused(emu_lib):
    """The top-K heaps hold 127 nodes: a general job of 127 uploads, one of 128 gets CRANE_ENOSYS
    naming its row."""
    from cranesched_b200.scheduler import CraneSchedError
    base = synth.edge_case(5, n_jobs=6, parts=((140, 2),), n_running=0, p_wide=0.0, p_general=0.0, p_down=0.0)
    cfg, cl, rn, pd, now = base
    for nodes, ok in ((127, True), (128, False)):
        pd2 = pd.take(np.arange(pd.n))
        _resize(pd2, 3, nodes, nodes + 50, 1, 3)
        s = _scheduler(emu_lib, base)
        try:
            if ok:
                s.upload(rn, pd2)
            else:
                with pytest.raises(CraneSchedError) as e:
                    s.upload(rn, pd2)
                assert e.value.code == abi.ENOSYS and "pending[3]" in str(e.value), str(e.value)
        finally:
            s.close()


def test_uniform_job_wider_than_its_partition(oracle, emu_lib):
    """A uniform job of more nodes than its partition has (or has usable) gets reason Resource,
    as in the oracle; the jobs around it are placed."""
    case = synth.edge_case(7, n_jobs=12, parts=((40, 5), (20, 3)), n_running=4, p_wide=0.0, p_general=0.0)
    cfg, cl, rn, pd, now = case
    usable = [int(((cl.alive == 1) & (cl.drain == 0))[cl.part_off[p]:cl.part_off[p + 1]].sum()) for p in range(2)]
    for j, nodes in ((2, 41), (5, usable[0] + 1), (8, 21)):
        pd.partition[j] = 0 if nodes > 21 else 1
        _resize(pd, j, nodes, nodes, 1, 1)
    got = _match(oracle, emu_lib, case)
    assert (got.reason[[2, 5, 8]] == abi.REASON_RESOURCE).all() and (got.n_alloc[[2, 5, 8]] == 0).all()
    assert (got.n_alloc > 0).sum() >= 6


# ---- the per-SM state budget --------------------------------------------------------------
def _header_constants():
    src = open(os.path.join(os.path.dirname(synth.__file__), "csrc", "commit_v2.cuh")).read()
    return {k: int(re.search(r"constexpr int %s = (\d+);" % k, src).group(1)) for k in ("kBlk", "kRingMax", "kMaxJ")}


def _words(mp):
    return max(4, ((mp + 31) // 32 + 3) // 4 * 4)


def _fixed_bytes(mp, k):
    """commit2_fixed_bytes of a single-partition scheduler with gres."""
    nblk = (mp + k["kBlk"] - 1) // k["kBlk"]
    return mp * 8 * 3 + nblk * 8 * 3 + (mp + 4) * 4 + mp * 2 * 4 + mp * 2 + 256


def _one_partition(n):
    names = tuple(range(abi.GRES_ENTRIES))
    return synth.make_cluster([(n, synth.node_row(64, 256 * synth.GiB, {0: 8, 7: 16}))], gres_entry_name=names)


def largest_partition(lib):
    """Bisect the node count of a single-partition cluster set_cluster accepts. Returns (largest
    accepted, the refusal of one node more)."""
    from cranesched_b200.scheduler import CraneSchedError, GpuScheduler

    def accepted(n):
        s = GpuScheduler(synth.config1()[0], 0, lib)
        try:
            s.set_cluster(_one_partition(n))
            return None
        except CraneSchedError as e:
            return e
        finally:
            s.close()

    lo, hi = 64, 65000
    assert accepted(lo) is None and accepted(hi) is not None
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if accepted(mid) is None:
            lo = mid
        else:
            hi = mid
    return lo, accepted(lo + 1)


def ring_bounds(m):
    """Any budget with m nodes accepted and m + 1 refused gives m a ring depth in [lo, hi]."""
    k = _header_constants()
    need = k["kMaxJ"] + 4
    b_lo = _fixed_bytes(m, k) + need * _words(m) * 4
    b_hi = _fixed_bytes(m + 1, k) + need * _words(m + 1) * 4 - 1
    ring = lambda b: min((b - _fixed_bytes(m, k)) // (_words(m) * 4), k["kRingMax"])
    return ring(b_lo), ring(b_hi), k


def _check_boundary(lib):
    m, err = largest_partition(lib)
    assert err is not None and err.code == abi.ENOSYS and "per-SM state budget" in str(err), err
    lo, hi, k = ring_bounds(m)
    assert k["kMaxJ"] + 4 <= lo <= hi < k["kRingMax"], (m, lo, hi)
    return m, hi


def test_partition_budget_boundary_emulated(emu_lib):
    """One node above the largest partition set_cluster accepts is refused with CRANE_ENOSYS; the
    largest one runs with a ring below kRingMax (host work only)."""
    _check_boundary(emu_lib)


# ---- GPU ----------------------------------------------------------------------------------
SWEEP = [
    # (n_jobs, parts, extra edge_case knobs, what else: None / "resv" / "overlap")
    (300, ((80, 20),), {}, None),
    (600, ((200, 24), (80, 3)), {}, None),
    (900, ((300, 6), (150, 18)), dict(one_type_per_name=True), None),
    (800, ((300, 30),), dict(p_wide=0.06), None),
    (2000, ((240, 40),), dict(p_wide=0.04, short=True), None),
    (800, ((160, 4), (160, 17), (100, 9)), dict(fifo=True), None),
    (700, ((250, 20),), dict(cost_policy=1), None),
    (1000, ((200, 12), (200, 25)), dict(cost_policy=1, one_type_per_name=True), None),
    (500, ((130, 16), (130, 17)), dict(fifo=True, cost_policy=1), None),
    (1000, ((200, 20), (120, 2)), dict(p_general=0.8), None),
    (600, ((140, 5), (140, 22)), dict(short=True, limit=450), None),
    (900, ((300, 19),), dict(p_full=0.02), None),
    (600, ((120, 18), (100, 4)), {}, "resv"),
    (900, ((240, 20),), dict(fifo=True), "resv"),
    (700, ((150, 10), (150, 20)), dict(cost_policy=1), "resv"),
    (800, ((100, 20), (100, 3), (100, 12)), {}, "overlap"),
    (700, ((200, 24), (160, 8)), dict(fifo=True), "overlap"),
    (600, ((120, 17), (120, 17)), dict(cost_policy=1, short=True), "overlap"),
    (1200, ((90, 4), (200, 30), (110, 6)), dict(one_type_per_name=True), "overlap"),
    (400, ((128, 20),), dict(p_wide=0.2, n_running=80), None),
    (700, ((450, 26), (150, 5)), dict(n_running=120), None),
    (500, ((96, 3),), dict(p_wide=0.15), None),
    (1000, ((260, 20), (260, 4)), dict(p_general=0.7, fifo=True), None),
    (700, ((200, 17),), dict(cost_policy=1, p_wide=0.1, short=True), "resv"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(SWEEP)))
def test_edge_sweep(oracle, gpu_lib, i):
    n_jobs, parts, kw, extra = SWEEP[i]
    kw = dict(kw)
    kw.setdefault("n_running", 40)
    case = synth.edge_case(9000 + i, n_jobs=n_jobs, parts=parts, **kw)
    resv = None
    if extra == "resv":
        resv, pd2, rn2 = synth.random_reservations(9000 + i, case, n_resv=5)
        case = (case[0], case[1], rn2, pd2, case[4])
    elif extra == "overlap":
        case = synth.overlap_partitions(case, 9000 + i, frac=0.3)
    got = _match(oracle, gpu_lib, case, resv)
    if extra != "overlap":
        assert usable_shapes(case[1]) == [s for _, s in parts]
    assert wide_between_batches(case, got, KMAXT), "no job wider than a batch placed between batch jobs"
    c, g = high_alloc(case, got)
    assert c > 0 and g > 0, "no allocation in core words 2-3 (%d) or gres entries 4-7 (%d)" % (c, g)


@pytest.mark.gpu
def test_shallow_ring_partition(oracle, gpu_lib):
    """The largest single partition the device's shared memory takes: one node more is refused,
    the largest one runs ~1500 jobs with a ring below kRingMax and matches the oracle."""
    m, ring = _check_boundary(gpu_lib)
    print("largest partition %d nodes, ring depth at most %d" % (m, ring))
    case = synth.edge_case(9100, n_jobs=1500, parts=((m, 12),), n_running=60, p_down=0.0, p_wide=0.05)
    assert usable_shapes(case[1]) == [12] and case[1].n_nodes == m
    got = _match(oracle, gpu_lib, case)
    assert wide_between_batches(case, got, KRK)
