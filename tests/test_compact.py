"""crane_sched_compact: the resident pending and running tables and the dependency entries
compacted on the device.

  - twin trajectories: two handles get the same calls (submits with holds, begin times and
    dependency lists, recovery EVENT entries, starts on the device, ends, cancels, erases of
    rows that have dependents, holds and releases, running rows appended from the host, a
    drain part-way); handle b compacts at several ticks (twice in a row, on a table without
    tombstones, right after set_cluster, right after start before keep_running), handle a
    never does. After every tick every output column of b equals a's at the mapped rows,
    byte for byte, and on some ticks the oracle's NodeSelect over the eligible rows;
  - the maps: strictly increasing over the live rows, CRANE_ROW_NONE on erased ones, the
    identity without tombstones, NULL maps accepted;
  - calls after compaction address the new rows (step_jobs_start, pending_depend, start
    with AFTER dependents);
  - the argument codes, and one 2-rank gloo case.
Through the emulator here, on the GPU in the `gpu`-marked twins."""
import dataclasses
import os
import sys
import types
from collections import Counter

import numpy as np
import pytest

from cranesched_b200 import abi, synth
from cranesched_b200.scheduler import GpuScheduler
from oracle.pygate import AFTER, AFTER_ANY, AFTER_OK
from tests import test_gate
from tests.test_gate import _case, _code, _compare, _Trajectory

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = abi.ROW_NONE


def _check_map(m, dead):
    """m = the map of a table whose erased rows are `dead`."""
    assert m.dtype == np.uint32 and len(m) == len(dead)
    assert (m[dead] == NONE).all()
    assert np.array_equal(m[~dead], np.arange(int((~dead).sum())))


class _Twin:
    """Two handles given the same calls: `a` never compacts, `b` compacts when asked. Rows
    passed in and returned are a's; b's rows are a's through the composed maps."""

    def __init__(self, cfg, device=0, lib=None):
        self.a = GpuScheduler(cfg, device, lib)
        self.b = GpuScheduler(cfg, device, lib)
        self.pmap = np.zeros(0, np.int64)   # a's pending row -> b's, or NONE
        self.rmap = np.zeros(0, np.int64)   # a's running row -> b's, or NONE
        self.pdead = np.zeros(0, bool)      # a's erased pending rows
        self.rdead = np.zeros(0, bool)
        self.nn = np.zeros(0, np.int64)     # node_num of a's pending rows
        self.compact_after_start = False
        self.seen = Counter()

    def _p(self, rows):
        r = self.pmap[np.asarray(rows, np.int64)]
        assert (r != NONE).all()
        return r.astype(np.uint32)

    def _r(self, rows):
        r = self.rmap[np.asarray(rows, np.int64)]
        assert (r != NONE).all()
        return r.astype(np.uint32)

    def compact(self):
        bdead = np.zeros(self.b.pending_rows(), bool)
        bdead[self.pmap[(self.pmap != NONE) & self.pdead]] = True
        brdead = np.zeros(self.b.running_rows(), bool)
        brdead[self.rmap[(self.rmap != NONE) & self.rdead]] = True
        pm, rm = self.b.compact()
        _check_map(pm, bdead)
        _check_map(rm, brdead)
        if not bdead.any():
            self.seen["compactions without pending tombstones"] += 1
        keep = self.pmap != NONE
        self.pmap[keep] = pm[self.pmap[keep]]
        self.pmap[self.pmap == NONE] = NONE
        keep = self.rmap != NONE
        self.rmap[keep] = rm[self.rmap[keep]]
        assert self.b.pending_rows() == int((~self.pdead).sum())
        assert self.b.running_rows() == int((~self.rdead).sum())
        self.seen["compactions"] += 1

    # ---- the calls of the trajectory, on both handles ----
    def set_cluster(self, cl):
        self.a.set_cluster(cl)
        self.b.set_cluster(cl)

    def set_reservations(self, r):
        self.a.set_reservations(r)
        self.b.set_reservations(r)

    def pending_append(self, pd):
        fa, fb = self.a.pending_append(pd), self.b.pending_append(pd)
        assert fa == len(self.pmap)
        self.pmap = np.concatenate([self.pmap, fb + np.arange(pd.n)])
        self.pdead = np.concatenate([self.pdead, np.zeros(pd.n, bool)])
        self.nn = np.concatenate([self.nn, pd.node_num.astype(np.int64)])
        return fa

    def running_append(self, rn):
        fa, fb = self.a.running_append(rn), self.b.running_append(rn)
        self.rmap = np.concatenate([self.rmap, fb + np.arange(rn.n)])
        self.rdead = np.concatenate([self.rdead, np.zeros(rn.n, bool)])
        return fa

    def pending_set_gate(self, rows, held=None, begin_time=None):
        self.a.pending_set_gate(rows, held, begin_time)
        self.b.pending_set_gate(self._p(rows), held, begin_time)

    def pending_depend(self, d):
        self.a.pending_depend(d)
        dep = d.dependee.astype(np.int64)
        p, r = d.kind == abi.DEPENDEE_PENDING, d.kind == abi.DEPENDEE_RUNNING
        dep[p] = self._p(dep[p])
        dep[r] = self._r(dep[r])
        self.b.pending_depend(abi.Dependencies(self._p(d.row), d.is_or, d.dep_off, d.kind, dep, d.type, d.delay_s,
                                               d.event_time))

    def start(self, rows):
        rows = np.asarray(rows, np.int64)
        fa, fb = self.a.start(rows), self.b.start(self._p(rows))
        self.pdead[rows] = True
        self.rmap = np.concatenate([self.rmap, fb + np.arange(len(rows))])
        self.rdead = np.concatenate([self.rdead, np.zeros(len(rows), bool)])
        if self.compact_after_start:
            self.compact_after_start = False
            self.compact()
            self.seen["compactions after start"] += 1
        return fa

    def pending_erase(self, rows):
        self.a.pending_erase(rows)
        self.b.pending_erase(self._p(rows))
        self.pdead[np.asarray(rows, np.int64)] = True

    def pending_cancel(self, rows, t):
        self.a.pending_cancel(rows, t)
        self.b.pending_cancel(self._p(rows), t)
        self.pdead[np.asarray(rows, np.int64)] = True

    def running_erase(self, rows):
        self.a.running_erase(rows)
        self.b.running_erase(self._r(rows))
        self.rdead[np.asarray(rows, np.int64)] = True

    def running_end(self, rows, t, code):
        self.a.running_end(rows, t, code)
        self.b.running_end(self._r(rows), t, code)
        self.rdead[np.asarray(rows, np.int64)] = True

    def keep_running(self):
        self.a.keep_running()
        self.b.keep_running()

    def run(self, now):
        self.a.run(now)
        self.b.run(now)

    def fetch(self, out):
        """a's placements into `out`; b's must equal them at every live row of a."""
        self.a.fetch(out)
        held = np.flatnonzero(self.pmap != NONE)  # a's rows still in b, in b's row order
        assert np.array_equal(self.pmap[held], np.arange(len(held))) and self.b.pending_rows() == len(held)
        got = self.b.fetch(abi.Placements.for_pending(types.SimpleNamespace(n=len(held), node_num=self.nn[held])))
        live = ~self.pdead[held]
        ref = abi.Placements(out.reason[held][live], out.priority[held][live], out.start_time[held][live],
                             out.end_time[held][live], out.n_alloc[held][live], None,
                             out.alloc_node[np.repeat(~self.pdead, self.nn)],
                             out.alloc_ntasks[np.repeat(~self.pdead, self.nn)],
                             out.alloc_res[np.repeat(~self.pdead, self.nn)])
        _compare(got, live, self.nn[held], ref, "compacted")
        self.seen["rows compared"] += int(live.sum())
        return out

    def step_jobs_start(self, rows):
        fa, fb = self.a.step_jobs_start(rows), self.b.step_jobs_start(self._r(rows))
        return fa, fb

    def close(self):
        self.a.close()
        self.b.close()


def _drain(cl, rng):
    drain = cl.drain.copy()
    drain[rng.choice(cl.n_nodes, max(1, cl.n_nodes // 10), replace=False)] = 1
    return dataclasses.replace(cl, drain=drain)


def _extra_events(tr, tw, rng):
    """Erases of rows that have dependents (their entries never fire) and running rows of
    jobs started elsewhere."""
    dm = tr.dm
    wanted = {d for j in dm.jobs.values() if j.state == "pending" for d in j.deps.deps}
    pend = [int(j) for j in tr.rows_job if dm.jobs[int(j)].state == "pending" and int(j) in wanted]
    if pend:
        j = pend[int(rng.integers(len(pend)))]
        tw.pending_erase([tr.pd_row[j]])
        dm.jobs[j].state = "ended"  # gone without events: its dependents wait forever
        tw.seen["pending erased with dependents"] += 1
    run = [k for k, j in enumerate(tr.rjob) if int(j) in wanted]
    if run:
        k = run[int(rng.integers(len(run)))]
        tw.running_erase([tr.ids[k]])
        dm.jobs[int(tr.rjob[k])].state = "ended"
        keep = np.delete(np.arange(tr.host.n), k)
        tr.host, tr.ids, tr.rjob = tr.host.take(keep), tr.ids[keep], tr.rjob[keep]
        tw.seen["running erased with dependents"] += 1
    # a job started elsewhere: a running row from the host
    cand = [int(j) for j in tr.rows_job if dm.jobs[int(j)].state == "pending" and not dm.jobs[int(j)].held]
    if cand and tr.host.n:
        j = cand[0]
        r = tr.pd_row[j]
        tw.pending_erase([r])  # (it left the pending map without a start here)
        dm.jobs[j].state = "ended"
        one = tr.host.take([0])
        one_id = -10 ** 6 - tw.seen["appended"]
        first = tw.running_append(one)
        dm.running(one_id, int(one.start_time[0]))
        tr.host = abi.Running.concat(tr.host, one)
        tr.ids = np.concatenate([tr.ids, [first]])
        tr.rjob = np.concatenate([tr.rjob, [one_id]])
        tr.run_row[one_id] = first
        tw.seen["appended"] += 1


def _twin_run(lib, case, resv, seed, n_ticks=9, oracle=None, oracle_every=3):
    """A trajectory of test_gate's on a _Twin; b compacts at ticks 2, 3, 3 (twice in a row),
    after the drain, after a start and on a table it has just compacted."""
    pd = case[3]
    cuts = sorted({pd.n // 2, (5 * pd.n) // 8, (3 * pd.n) // 4, (7 * pd.n) // 8, pd.n})
    made = []

    def factory(cfg, device, lib_):
        made.append(_Twin(cfg, device, lib_))
        return made[-1]

    orig = test_gate.GpuScheduler
    test_gate.GpuScheduler = factory
    try:
        tr = _Trajectory(lib, case, resv, seed)
    finally:
        test_gate.GpuScheduler = orig
    tw = made[0]
    rng = np.random.Generator(np.random.PCG64(seed + 1))
    drain_at = n_ticks // 2
    try:
        tr.submit(np.arange(cuts[0]), recovery=True)
        for t in range(n_ticks):
            if t == drain_at:
                cl = _drain(tr.cl, rng)
                tw.set_cluster(cl)
                if resv is not None:
                    tw.set_reservations(resv)
                tr.cl = cl
                tw.compact()  # right after set_cluster
            if t in (2, 3, 6):
                tw.compact()
            if t == 3:
                tw.compact()  # twice in a row: nothing left to drop
            got = tr.tick(None, oracle if t % oracle_every == 0 else None)
            tw.compact_after_start = t in (4, 7)
            tr.advance(got)
            if t % 2:
                _extra_events(tr, tw, rng)
            nxt = next((c for c in cuts if c > tr.n_sub), tr.n_sub)
            if nxt > tr.n_sub:
                tr.submit(np.arange(tr.n_sub, nxt))
        tr.tick(None, oracle)
    finally:
        tw.close()
    seen = tr.seen + tw.seen
    for what in ("compactions", "compactions after start", "compactions without pending tombstones",
                 "pending erased with dependents", "running erased with dependents", "appended", "started",
                 "cancelled", "Dependency", "rows compared"):
        assert seen[what] > 0, (what, dict(seen))
    return seen


EMU_CASES = {
    "multifactor": dict(seed=81, n_jobs=90, n_nodes=20, n_parts=2, n_running=12, short=True),
    "fifo_resv": dict(seed=82, n_jobs=90, n_nodes=24, n_parts=3, n_running=10, short=True, fifo=True, resv=True,
                      limit=40),
}


@pytest.mark.parametrize("name", sorted(EMU_CASES))
def test_compact_twin_trajectory_emulated(oracle, emu_lib, name):
    kw = dict(EMU_CASES[name])
    case, resv = _case(**kw)
    _twin_run(emu_lib, case, resv, kw["seed"], oracle=oracle)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [120, 121])
def test_compact_twin_trajectory_gpu(oracle, gpu_lib, seed):
    """600 jobs a seed, the second with reservations."""
    case, resv = _case(seed, n_jobs=600, n_nodes=90, n_parts=2, n_running=60, short=True, resv=seed % 2 == 1,
                       limit=300)
    _twin_run(gpu_lib, case, resv, seed, oracle=oracle, oracle_every=4)


@pytest.mark.gpu
def test_compact_twin_trajectory_gpu_4000(gpu_lib):
    """4 000 jobs, as the resident running table's large case (no oracle at this size)."""
    case, resv = _case(123, n_jobs=4000, n_nodes=400, n_parts=4, n_running=300, short=True)
    _twin_run(gpu_lib, case, resv, 123, n_ticks=8)


# ---- the maps and calls after compaction ----------------------------------------------------

def _small(lib, seed=90):
    cfg, cl, rn, pd, now = synth.random_case(seed, n_jobs=40, n_nodes=12, n_parts=1, n_running=8, short=True)
    s = GpuScheduler(cfg, 0, lib)
    s.set_cluster(cl)
    return s, cfg, cl, rn, pd, now


def test_compact_maps(emu_lib):
    s, cfg, cl, rn, pd, now = _small(emu_lib)
    try:
        pm, rm = s.compact()  # empty tables
        assert len(pm) == 0 and len(rm) == 0
        s.pending_append(pd)
        s.running_append(rn)
        pm, rm = s.compact()  # no tombstones: the identity
        assert np.array_equal(pm, np.arange(pd.n)) and np.array_equal(rm, np.arange(rn.n))
        s.pending_erase([0, 5, 6, pd.n - 1])
        s.running_erase([2])
        assert s.compact(maps=False) == (None, None)  # NULL maps
        assert s.pending_rows() == pd.n - 4 and s.running_rows() == rn.n - 1
        s.pending_erase([1, 3])
        pm, rm = s.compact()
        dead = np.zeros(pd.n - 4, bool)
        dead[[1, 3]] = True
        _check_map(pm, dead)
        assert np.all(np.diff(pm[~dead].astype(np.int64)) == 1)
        assert np.array_equal(rm, np.arange(rn.n - 1))
        s.keep_running()
        s.run(now)
        keep = np.setdiff1d(np.arange(pd.n), [0, 5, 6, pd.n - 1])
        keep = np.delete(keep, [1, 3])
        got = s.fetch(abi.Placements.for_pending(pd.take(keep)))
        u = GpuScheduler(cfg, 0, emu_lib)
        u.set_cluster(cl)
        u.upload(rn.take(np.delete(np.arange(rn.n), 2)), pd.take(keep))
        u.run(now)
        ref = u.fetch(abi.Placements.for_pending(pd.take(keep)))
        u.close()
        assert not ref.diff(got), ref.diff(got)[:4]
    finally:
        s.close()


def test_calls_after_compaction_address_new_rows(emu_lib):
    cfg, cl, rn, pd, now = synth.random_case(91, n_jobs=40, n_nodes=16, n_parts=1, n_running=8, short=True)
    tw = _Twin(cfg, 0, emu_lib)
    P, R = abi.DEPENDEE_PENDING, abi.DEPENDEE_RUNNING
    D = abi.Dependencies.from_lists
    try:
        tw.set_cluster(cl)
        tw.pending_append(pd)
        tw.running_append(rn)
        dependee = [0, 1, 4, 7, 8]
        tw.pending_depend(D([10, 11, 12, 13, 14], [0] * 5, [[(P, r, AFTER, 30, 0)] for r in dependee]))
        tw.running_end([0, 1], [now - 10, now - 5], [0, 1])
        tw.pending_cancel([2, 3], now)
        tw.compact()
        # a new list on a remapped row, and "already has its list" is still refused for one
        tw.pending_depend(D([6], [1], [[(P, 5, AFTER_OK, 0, 0), (R, 3, AFTER_ANY, 0, 0)]]))
        assert _code(tw.b.pending_depend, D(tw._p([10]), [0], [[]])) == abi.EINVAL
        assert _code(tw.b.pending_depend, D(tw._p([6]), [0], [[]])) == abi.EINVAL
        tw.keep_running()
        tw.run(now)
        out = tw.fetch(abi.Placements.for_pending(pd))
        # start of a new row fires AFTER on its dependents as in a
        started = np.flatnonzero(out.reason == abi.REASON_NONE)
        assert np.isin(dependee, started).any()
        first = tw.start(started)
        tw.compact()
        # step jobs on the new running rows: the same avail as a's on the old ones
        ja, jb = tw.step_jobs_start(first + np.arange(len(started)))
        rows = np.arange(len(started))
        assert tw.a.step_jobs_avail(ja + rows).tobytes() == tw.b.step_jobs_avail(jb + rows).tobytes()
        tw.keep_running()
        tw.run(now + 40)
        tw.fetch(abi.Placements.for_pending(pd))
    finally:
        tw.close()


def test_compact_argument_codes(emu_lib):
    from cranesched_b200.scheduler import load_library
    lib = load_library(emu_lib)
    assert lib.crane_sched_compact(None, None, None) == abi.EINVAL
    cfg, cl, rn, pd, now = synth.random_case(92, n_jobs=20, n_nodes=8, n_parts=1, n_running=4, short=True)
    cfg.priority_type = 1
    s = GpuScheduler(cfg, 0, emu_lib)
    try:
        assert _code(s.compact) == abi.EINVAL  # before set_cluster
        s.set_cluster(cl)
        s.upload(rn, pd)
        s.run(now)
        s.compact()
        out = abi.Placements.for_pending(pd)
        assert _code(s.fetch, out) == abi.EINVAL  # the run is void
        assert _code(s.start, [0]) == abi.EINVAL
        assert _code(s.qos_filter, synth.random_qos(92, cl, pd), out.reason.copy()) == abi.EINVAL
        s.keep_running()
        s.run(now)
        s.fetch(out)
    finally:
        s.close()


# ---- one queue over two ranks ---------------------------------------------------------------

def _shard_worker(rank, world, port, emu_lib, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from cranesched_b200 import sharding
    cfg, cl, rn, pd, now = synth.random_case(77, n_jobs=90, n_nodes=30, n_parts=4, n_running=16, limit=60)
    owner = sharding.deal_partitions(pd, cl.n_partitions, world, cl)
    res = []
    for compact in (False, True):
        s = GpuScheduler(cfg, 0, emu_lib)
        s.set_cluster(cl)
        s.set_shard(rank, world, owner)
        test_gate._gate_calls(s, pd, rn, now)
        if compact:
            pm, rm = s.compact()
            s.keep_running()
        s.run(now)
        rows = s.pending_rows()
        out = abi.Placements.for_pending(pd.take(np.flatnonzero(pm != NONE)) if compact else pd)
        s.fetch(out)
        s.close()
        res.append((out, rows, pm if compact else None))
    (a, _, _), (b, nb, pm) = res
    live = np.flatnonzero(pm != NONE)
    mask = np.repeat(pm != NONE, pd.node_num)
    d = []
    for f in ("reason", "start_time", "end_time", "n_alloc"):
        if not np.array_equal(getattr(a, f)[live], getattr(b, f)):
            d.append(f)
    if a.priority[live].view(np.uint64).tolist() != b.priority.view(np.uint64).tolist():
        d.append("priority")
    for f in ("alloc_node", "alloc_ntasks"):
        if not np.array_equal(getattr(a, f)[mask], getattr(b, f)):
            d.append(f)
    if a.alloc_res[mask].tobytes() != b.alloc_res.tobytes():
        d.append("alloc_res")
    q.put((rank, d, nb, len(live), pd.n))
    dist.destroy_process_group()


def test_compact_sharded_rank_equals_uncompacted_gloo(emu_lib):
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + os.getpid() % 2000
    procs = [ctx.Process(target=_shard_worker, args=(r, world, port, emu_lib, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=900) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, d, nb, n_live, n in res:
        assert not d, f"rank {rank}: the compacted rank's columns differ: {d}"
        assert nb == n_live < n
