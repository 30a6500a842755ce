"""The gate of the resident pending table: held jobs, jobs whose begin time is ahead and
jobs whose dependencies are not met stay resident and sit the run out
(crane_sched_pending_set_gate / _pending_depend / _pending_cancel / _running_end, and the
dependency events of crane_sched_start).

  - oracle/pygate.py (the daemon's DependenciesInJob and its call sites) on hand-derived
    cases;
  - the argument codes, on the kernel-emulation library;
  - trajectories of ticks with submits (holds, begin times, AFTER / AFTER_ANY / AFTER_OK /
    AFTER_NOT_OK lists, AND and OR), a recovery with EVENT entries, holds and releases,
    starts on the device, ends with zero and non-zero exit codes, cancels and a
    compaction. Every tick: (a) a gated row carries pygate's reason and no placement,
    (b) every output column of the eligible rows is byte-identical to a second handle
    given a fresh upload of only the eligible rows, (c) and equals the oracle's NodeSelect
    over them (priority compared as bits). Through the emulator here, on the GPU in the
    `gpu`-marked twins;
  - one 2-rank gloo case: a gated, sharded tick equals the unsplit one."""
import os
import sys
from collections import Counter

import numpy as np
import pytest

from cranesched_b200 import abi, synth
from cranesched_b200.scheduler import CraneSchedError, GpuScheduler
from oracle import pygate
from oracle.pygate import AFTER, AFTER_ANY, AFTER_NOT_OK, AFTER_OK, FUTURE, PAST

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _code(fn, *args, **kw):
    try:
        fn(*args, **kw)
        return 0
    except CraneSchedError as e:
        return e.code


# ---- pygate by hand ------------------------------------------------------------------------

def test_pygate_types_and_call_sites():
    d = pygate.Daemon()
    for j in (1, 2, 3, 4):
        d.submit(j)
    d.submit(10, [(1, AFTER, 5)])
    d.submit(11, [(2, AFTER_ANY, 0)])
    d.submit(12, [(3, AFTER_OK, 0)])
    d.submit(13, [(4, AFTER_NOT_OK, 0)])
    d.submit(14, [(3, AFTER_NOT_OK, 0)])
    now = 1000
    assert [d.reason(j, now) for j in (10, 11, 12, 13, 14)] == [pygate.DEPENDENCY] * 5
    d.start(1, 990)  # AFTER: start + delay
    assert d.reason(10, 994) == pygate.DEPENDENCY and d.reason(10, 995) == pygate.NONE
    d.cancel(2, 900)  # AFTER_ANY at the cancel time
    assert d.reason(11, now) == pygate.NONE
    d.start(3, 950)
    assert d.reason(12, now) == pygate.DEPENDENCY  # AFTER_OK waits for the end
    d.end(3, 980, 0)
    assert d.reason(12, now) == pygate.NONE
    assert d.reason(14, now) == pygate.DEPENDENCY_NEVER  # AFTER_NOT_OK on a job that exited 0
    d.start(4, 950)
    d.end(4, 990, 1)
    assert d.reason(13, now) == pygate.NONE


def test_pygate_and_or_and_edges():
    d = pygate.Daemon()
    for j in (1, 2):
        d.submit(j)
    d.submit(10, [(1, AFTER_OK, 0), (2, AFTER_OK, 0)])              # AND
    d.submit(11, [(1, AFTER_OK, 0), (2, AFTER_OK, 0)], is_or=True)  # OR
    d.submit(12, [], is_or=True)                                     # an OR with no entries
    assert d.reason(12, 0) == pygate.DEPENDENCY_NEVER
    d.cancel(1, 100)  # AFTER_OK of a cancelled job: InfiniteFuture
    assert d.reason(10, 10 ** 9) == pygate.DEPENDENCY_NEVER  # AND: failed at once
    assert d.reason(11, 10 ** 9) == pygate.DEPENDENCY        # OR: the other may still come
    d.start(2, 200)
    d.end(2, 300, 0)
    assert d.reason(11, 300) == pygate.NONE and d.reason(10, 10 ** 9) == pygate.DEPENDENCY_NEVER
    # begin_time == now is eligible; hold overrides a met dependency; the filter order
    d.submit(20, begin=500)
    assert d.reason(20, 499) == pygate.BEGIN_TIME and d.reason(20, 500) == pygate.NONE
    d.submit(21, [(2, AFTER_ANY, 0)], held=True, resolved={2: 300})
    assert d.reason(21, 400) == pygate.HELD
    d.set_held(21, False)
    assert d.reason(21, 400) == pygate.NONE
    d.submit(22, [(1, AFTER, 0)], held=True, begin=10 ** 6, resolved={1: 100})
    assert d.reason(22, 0) == pygate.HELD
    d.set_held(22, False)
    assert d.reason(22, 0) == pygate.BEGIN_TIME
    # a running dependee: AFTER fires at once at its start time, the others register
    d.running(30, 700)
    d.submit(31, [(30, AFTER, 10)])
    d.submit(32, [(30, AFTER_ANY, 0)])
    assert d.reason(31, 709) == pygate.DEPENDENCY and d.reason(31, 710) == pygate.NONE
    assert d.reason(32, 10 ** 9) == pygate.DEPENDENCY
    # missing or ended dependees are rejected; an event for an unknown id is ignored
    with pytest.raises(pygate.MissingDependency):
        d.submit(40, [(99, AFTER, 0)])
    with pytest.raises(pygate.MissingDependency):
        d.submit(40, [(1, AFTER, 0)])  # cancelled
    x = pygate.Deps(False, {5: (AFTER, 0)})
    assert not x.update(6, 10) and x.deps
    # saturation: an infinite event time stays infinite whatever the delay
    y = pygate.Deps(True, {5: (AFTER_OK, 100)})
    y.update(5, FUTURE)
    assert y.ready == FUTURE and y.is_failed()


# ---- argument codes ---------------------------------------------------------------------------

def test_depend_argument_codes(emu_lib):
    case = synth.random_case(61, n_jobs=30, n_nodes=10, n_parts=1, n_running=4)
    cfg, cl, rn, pd, now = case
    s = GpuScheduler(cfg, 0, emu_lib)
    D = abi.Dependencies.from_lists
    P, R, E = abi.DEPENDEE_PENDING, abi.DEPENDEE_RUNNING, abi.DEPENDEE_EVENT
    try:
        assert _code(s.pending_depend, D([0], [0], [[(P, 1, AFTER, 0, 0)]])) == abi.EINVAL  # before set_cluster
        s.set_cluster(cl)
        s.pending_append(pd)
        s.running_append(rn)
        s.pending_erase([5])
        s.running_erase([1])
        bad = {
            "row out of range": D([pd.n], [0], [[]]),
            "row erased": D([5], [0], [[]]),
            "row listed twice": D([2, 2], [0, 0], [[], []]),
            "pending dependee out of range": D([0], [0], [[(P, pd.n, AFTER, 0, 0)]]),
            "pending dependee erased": D([0], [0], [[(P, 5, AFTER, 0, 0)]]),
            "running dependee out of range": D([0], [0], [[(R, rn.n, AFTER, 0, 0)]]),
            "running dependee ended": D([0], [0], [[(R, 1, AFTER_ANY, 0, 0)]]),
            "depends on itself": D([3], [0], [[(P, 3, AFTER, 0, 0)]]),
            "dependee twice": D([0], [0], [[(P, 1, AFTER, 0, 0), (P, 1, AFTER_OK, 0, 0)]]),
            "running dependee twice": D([0], [1], [[(R, 0, AFTER, 0, 0), (R, 0, AFTER_OK, 0, 0)]]),
            "type > 3": D([0], [0], [[(P, 1, 4, 0, 0)]]),
            "kind > 2": D([0], [0], [[(3, 1, AFTER, 0, 0)]]),
            "delay >= 2^62": D([0], [0], [[(P, 1, AFTER, 2 ** 62, 0)]]),
        }
        for what, deps in bad.items():
            assert _code(s.pending_depend, deps) == abi.EINVAL, what
        # the same dependee as a pending and as an EVENT entry, and EVENT entries twice, are fine
        ok = D([0, 4], [0, 1], [[(P, 1, AFTER, 0, 0), (E, 0, AFTER_OK, 0, 5), (E, 0, AFTER_OK, 0, 6)],
                                [(R, 0, AFTER, 2 ** 62 - 1, 0)]])
        assert _code(s.pending_depend, ok) == 0
        assert _code(s.pending_depend, D([0], [0], [[]])) == abi.EINVAL  # a row already has a list
        assert _code(s.pending_depend, D([4], [0], [[]])) == abi.EINVAL
        assert _code(s.pending_set_gate, [pd.n], [1]) == abi.EINVAL
        assert _code(s.pending_cancel, [pd.n], now) == abi.EINVAL
        assert _code(s.running_end, [rn.n], [now], [0]) == abi.EINVAL
        s.pending_reset()  # clears the lists
        s.pending_append(pd)
        assert _code(s.pending_depend, D([0], [0], [[(P, 1, AFTER, 0, 0)]])) == 0
    finally:
        s.close()


def test_event_time_plus_delay_saturates(emu_lib):
    """A finite event time whose sum with the delay leaves the int64 range is InfiniteFuture,
    as absl::Time + Duration saturates: the dependency can never be met (it must not wrap
    round to a time in the past)."""
    case = synth.random_case(62, n_jobs=12, n_nodes=8, n_parts=1, n_running=0)
    cfg, cl, rn, pd, now = case
    s = GpuScheduler(cfg, 0, emu_lib)
    E = abi.DEPENDEE_EVENT
    try:
        s.set_cluster(cl)
        s.pending_append(pd)
        big = FUTURE - 2 ** 61
        s.pending_depend(abi.Dependencies.from_lists(
            [0, 1, 2], [0, 1, 0], [[(E, 0, AFTER_OK, 2 ** 62 - 1, big)],   # AND: failed
                                   [(E, 0, AFTER_OK, 2 ** 62 - 1, big)],   # OR, nothing left: failed
                                   [(E, 0, AFTER_OK, 2 ** 61 - 1, big)]]))  # FUTURE - 1: finite, not met
        s.set_running(rn)
        s.run(now)
        out = s.fetch(abi.Placements.for_pending(pd))
        assert out.reason[:3].tolist() == [abi.REASON_DEPENDENCY_NEVER, abi.REASON_DEPENDENCY_NEVER,
                                           abi.REASON_DEPENDENCY]
        d = pygate.Daemon()
        d.submit(0, [(99, AFTER_OK, 2 ** 62 - 1)], resolved={99: big})
        d.submit(2, [(99, AFTER_OK, 2 ** 61 - 1)], resolved={99: big})
        assert [d.reason(0, now), d.reason(2, now)] == [pygate.DEPENDENCY_NEVER, pygate.DEPENDENCY]
    finally:
        s.close()


# ---- trajectories ---------------------------------------------------------------------------

def _compare(got, mask, node_num, ref, what):
    for f in ("reason", "start_time", "end_time", "n_alloc"):
        assert np.array_equal(getattr(ref, f), getattr(got, f)[mask]), (what, f)
    assert np.array_equal(ref.priority.view(np.uint64), got.priority[mask].view(np.uint64)), (what, "priority")
    rows = np.repeat(mask, node_num)
    assert np.array_equal(ref.alloc_node, got.alloc_node[rows]), (what, "alloc_node")
    assert np.array_equal(ref.alloc_ntasks, got.alloc_ntasks[rows]), (what, "alloc_ntasks")
    assert ref.alloc_res.tobytes() == got.alloc_res[rows].tobytes(), (what, "alloc_res")


class _Trajectory:
    """One gated resident handle `b`, the daemon model `dm` and the bookkeeping that maps
    job ids (pending row of the drawn case; running jobs known at start: -1, -2, ...) to
    the rows of `b`."""

    def __init__(self, lib, case, resv, seed, dt=900, dep_frac=0.35):
        self.cfg, self.cl, rn0, self.pd, self.now = case
        self.resv, self.dt, self.dep_frac = resv, dt, dep_frac
        self.rng = np.random.Generator(np.random.PCG64(seed))
        self.dm = pygate.Daemon()
        self.seen = Counter()
        self.b = GpuScheduler(self.cfg, 0, lib)
        self.b.set_cluster(self.cl)
        if resv is not None:
            self.b.set_reservations(resv)
        self.rows_job = np.zeros(0, np.int64)     # job of every pending row of b
        self.pd_row = {}                          # job -> pending row
        self.host = rn0                           # live running rows in row order
        self.ids = np.arange(rn0.n)               # their running rows in b
        self.rjob = -1 - np.arange(rn0.n)         # their jobs
        self.run_row = {int(j): int(r) for j, r in zip(self.rjob, self.ids)}
        for j, t in zip(self.rjob, rn0.start_time):
            self.dm.running(int(j), int(t))
        assert self.b.running_append(rn0) == 0
        self.n_sub = 0

    def pdb(self):
        return self.pd.take(self.rows_job)

    def _entry(self, dep, ty, dl, resolved):
        if dep in resolved:
            return (abi.DEPENDEE_EVENT, 0, ty, dl, resolved[dep])
        if self.dm.jobs[dep].state == "pending":
            return (abi.DEPENDEE_PENDING, self.pd_row[dep], ty, dl, 0)
        return (abi.DEPENDEE_RUNNING, self.run_row[dep], ty, dl, 0)

    def submit(self, jobs, recovery=False):
        rng, now, dm = self.rng, self.now, self.dm
        first = self.b.pending_append(self.pd.take(jobs))
        self.rows_job = np.concatenate([self.rows_job, jobs])
        for k, j in enumerate(jobs):
            self.pd_row[int(j)] = first + k
        held = (rng.random(len(jobs)) < 0.08).astype(np.uint8)
        begin = np.full(len(jobs), PAST, np.int64)
        late = rng.random(len(jobs)) < 0.12
        begin[late] = now + self.dt * rng.integers(0, 3, int(late.sum()))  # (0: eligible from the next tick on)
        begin[rng.random(len(jobs)) < 0.03] = now - 5
        gated = np.flatnonzero(held.astype(bool) | (begin != PAST))
        if len(gated):
            self.b.pending_set_gate(first + gated, held=held[gated], begin_time=begin[gated])
        rows, is_or, entries = [], [], []
        for k, j in enumerate(int(x) for x in jobs):
            deps, resolved, orr = [], {}, bool(rng.random() < 0.3)
            if rng.random() < self.dep_frac:
                cand = [x for x, v in dm.jobs.items() if v.state != "ended"]
                for dep in rng.choice(cand, min(len(cand), int(rng.integers(1, 4))), replace=False):
                    deps.append((int(dep), int(rng.integers(0, 4)), int(rng.choice([0, 0, 60, 3600, 2 ** 40]))))
                if recovery and rng.random() < 0.5:  # a dependee that ended before the restart
                    gone = 10 ** 9 + j
                    deps.append((gone, int(rng.integers(0, 4)), int(rng.choice([0, 300]))))
                    resolved[gone] = FUTURE if rng.random() < 0.3 else now - int(rng.integers(0, 5000))
                    self.seen["event entries"] += 1
            elif rng.random() < 0.02:
                orr = True  # an OR with no entries: never met
            else:
                orr = False
            dm.submit(j, deps, orr, bool(held[k]), int(begin[k]), resolved)
            if deps or orr:
                rows.append(first + k)
                is_or.append(int(orr))
                entries.append([self._entry(d, ty, dl, resolved) for d, ty, dl in deps])
                self.seen["dependency lists"] += 1
        if rows:
            self.b.pending_depend(abi.Dependencies.from_lists(rows, is_or, entries))
        self.n_sub = max(self.n_sub, int(jobs[-1]) + 1)

    def compact(self):
        """A fresh pending table of the live rows with their gate state re-sent: one EVENT
        entry at ready_time for what was resolved, the open entries as they stand."""
        dm = self.dm
        keep = np.array([j for j in self.rows_job if dm.jobs[int(j)].state == "pending"], np.int64)
        self.b.pending_reset()
        self.rows_job = np.zeros(0, np.int64)
        self.pd_row = {}
        if not len(keep):
            return
        first = self.b.pending_append(self.pd.take(keep))
        self.rows_job = keep
        self.pd_row = {int(j): first + k for k, j in enumerate(keep)}
        jobs = [dm.jobs[int(j)] for j in keep]
        self.b.pending_set_gate(np.arange(len(keep)), held=[int(x.held) for x in jobs],
                                begin_time=[x.begin for x in jobs])
        rows, is_or, entries = [], [], []
        for k, x in enumerate(jobs):
            dp = x.deps
            if not dp.is_or and not dp.deps and dp.ready == PAST:
                continue
            ent = []
            if dp.ready != (FUTURE if dp.is_or else PAST):
                ent.append((abi.DEPENDEE_EVENT, 0, AFTER_ANY, 0, dp.ready))
            ent += [self._entry(d, ty, dl, {}) for d, (ty, dl) in dp.deps.items()]
            rows.append(k)
            is_or.append(int(dp.is_or))
            entries.append(ent)
        if rows:
            self.b.pending_depend(abi.Dependencies.from_lists(rows, is_or, entries))
        self.seen["compactions"] += 1

    def tick(self, twin=None, oracle=None):
        b, dm, now = self.b, self.dm, self.now
        b.keep_running()
        b.run(now)
        pdb = self.pdb()
        got = b.fetch(abi.Placements.for_pending(pdb))
        alive = np.array([dm.jobs[int(j)].state == "pending" for j in self.rows_job], bool)
        want = np.array([dm.reason(int(j), now) if a else abi.REASON_ERASED for j, a in zip(self.rows_job, alive)],
                        np.uint8).reshape(-1)
        gated = alive & (want != 0)
        assert np.array_equal(got.reason[gated | ~alive], want[gated | ~alive]), "gate reasons differ from pygate"
        assert not got.start_time[gated].any() and not got.end_time[gated].any() and not got.n_alloc[gated].any()
        grows = np.repeat(gated, pdb.node_num)
        assert not got.alloc_node[grows].any() and not got.alloc_res[grows].tobytes().strip(b"\0")
        self.seen.update(abi.REASON_STR[int(c)] for c in want[gated])
        elig = alive & (want == 0)
        ejobs = self.rows_job[elig]
        if twin is not None:  # a fresh upload of only the eligible rows
            twin.pending_reset()
            twin.pending_append(self.pd.take(ejobs))
            twin.set_running(self.host)
            twin.run(now)
            _compare(got, elig, pdb.node_num, twin.fetch(abi.Placements.for_pending(self.pd.take(ejobs))), "twin")
        if oracle is not None:
            ref, _, _ = oracle.node_select(self.cfg, self.cl, self.host, self.pd.take(ejobs), now, resv=self.resv)
            _compare(got, elig, pdb.node_num, ref, "oracle")
        return got

    def advance(self, got):
        """The commit loop starts most start-now rows; time passes; jobs end and are
        cancelled; holds change; the next batch is submitted."""
        b, dm, rng = self.b, self.dm, self.rng
        now_rows = np.flatnonzero(got.reason == abi.REASON_NONE)
        sel = rng.permutation(now_rows[rng.random(len(now_rows)) < 0.8])
        first = b.start(sel)
        for k, r in enumerate(sel):
            j = int(self.rows_job[r])
            dm.start(j, int(got.start_time[r]))
            self.run_row[j] = first + k
        self.host = abi.Running.concat(self.host, abi.Running.started(self.pdb(), got, sel))
        self.ids = np.concatenate([self.ids, first + np.arange(len(sel))])
        self.rjob = np.concatenate([self.rjob, self.rows_job[sel]])
        self.seen["started"] += len(sel)
        self.now += self.dt
        now = self.now
        ended = ((self.host.end_time < now + 1) & (rng.random(self.host.n) < 0.6)) | (rng.random(self.host.n) < 0.05)
        if ended.any():
            t_end = np.maximum(np.minimum(self.host.end_time[ended], now - rng.integers(0, self.dt, int(ended.sum()))),
                               self.host.start_time[ended])
            code = (rng.random(int(ended.sum())) < 0.3).astype(np.uint32)
            b.running_end(self.ids[ended], t_end, code)
            for j, t, c in zip(self.rjob[ended], t_end, code):
                dm.end(int(j), int(t), int(c))
            self.seen["ended, exit 0"] += int((code == 0).sum())
            self.seen["ended, exit != 0"] += int((code != 0).sum())
            keep = np.flatnonzero(~ended)
            self.host, self.ids, self.rjob = self.host.take(keep), self.ids[keep], self.rjob[keep]
        live = np.flatnonzero([dm.jobs[int(j)].state == "pending" for j in self.rows_job])
        if len(live) > 4:
            gone = rng.choice(live, len(live) // 20, replace=False)
            b.pending_cancel(gone, now)
            for r in gone:
                dm.cancel(int(self.rows_job[r]), now)
            self.seen["cancelled"] += len(gone)
            live = np.setdiff1d(live, gone)
        flip = rng.choice(live, min(len(live), 1 + len(live) // 15), replace=False) if len(live) else []
        if len(flip):
            held = np.array([not dm.jobs[int(self.rows_job[r])].held for r in flip], np.uint8)
            b.pending_set_gate(flip, held=held)
            for r, h in zip(flip, held):
                dm.set_held(int(self.rows_job[r]), bool(h))
            self.seen["hold / release"] += len(flip)

    def close(self):
        self.b.close()


def _run(lib, case, resv, seed, n_ticks=6, oracle=None, twin=True, compact_at=4):
    pd = case[3]
    cuts = sorted({pd.n // 2, (5 * pd.n) // 8, (3 * pd.n) // 4, (7 * pd.n) // 8, pd.n})
    tr = _Trajectory(lib, case, resv, seed)
    a = GpuScheduler(case[0], 0, lib) if twin else None
    try:
        if a is not None:
            a.set_cluster(case[1])
            if resv is not None:
                a.set_reservations(resv)
        tr.submit(np.arange(cuts[0]), recovery=True)
        for t in range(n_ticks):
            if t == compact_at:
                tr.compact()
            got = tr.tick(a, oracle)
            tr.advance(got)
            nxt = next((c for c in cuts if c > tr.n_sub), tr.n_sub)
            if nxt > tr.n_sub:
                tr.submit(np.arange(tr.n_sub, nxt))
        tr.tick(a, oracle)
    finally:
        tr.close()
        if a is not None:
            a.close()
    return tr.seen


def _case(seed, resv=False, **kw):
    case = synth.random_case(seed, **kw)
    r = None
    if resv:
        r, pd, rn = synth.random_reservations(seed, case, n_resv=4)
        case = (case[0], case[1], rn, pd, case[4])
    return case, r


def _check_seen(seen):
    for what in ("Held", "BeginTime", "Dependency", "DependencyNeverSatisfied", "started", "ended, exit 0",
                 "ended, exit != 0", "cancelled", "hold / release", "compactions", "event entries"):
        assert seen[what] > 0, (what, dict(seen))


EMU_CASES = {
    "multifactor": dict(seed=71, n_jobs=100, n_nodes=20, n_parts=2, n_running=12, short=True),
    "multifactor_resv": dict(seed=72, n_jobs=100, n_nodes=24, n_parts=2, n_running=10, short=True, resv=True),
    "fifo": dict(seed=73, n_jobs=100, n_nodes=20, n_parts=2, n_running=12, short=True, fifo=True, limit=50),
    "fifo_resv": dict(seed=74, n_jobs=100, n_nodes=24, n_parts=3, n_running=10, short=True, fifo=True, resv=True),
}


@pytest.mark.parametrize("name", sorted(EMU_CASES))
def test_gated_trajectory_emulated(oracle, emu_lib, name):
    kw = dict(EMU_CASES[name])
    case, resv = _case(**kw)
    _check_seen(_run(emu_lib, case, resv, kw["seed"], oracle=oracle))


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(110, 116))
def test_gated_trajectory_gpu(oracle, gpu_lib, seed):
    """500+ jobs a seed; the last one has a dependency graph of over a thousand rows."""
    n_jobs = 1400 if seed == 115 else 600
    case, resv = _case(seed, n_jobs=n_jobs, n_nodes=80 + 10 * (seed % 3), n_parts=1 + seed % 3, n_running=60,
                       short=True, fifo=seed % 3 == 0, limit=400 if seed % 2 else None, resv=seed % 2 == 0)
    seen = _run(gpu_lib, case, resv, seed, oracle=oracle if seed % 2 else None)
    _check_seen(seen)
    if seed == 115:
        assert seen["dependency lists"] >= 400


# ---- one queue over two ranks ---------------------------------------------------------------

def _gate_calls(s, pd, rn, now):
    """The same gate calls on any handle: holds, begin times, dependency lists, a cancel
    and an end."""
    rng = np.random.Generator(np.random.PCG64(5))
    s.pending_append(pd)
    s.running_append(rn)
    rows = np.arange(pd.n)
    s.pending_set_gate(rows[::9], held=np.ones(len(rows[::9]), np.uint8))
    s.pending_set_gate(rows[4::11], begin_time=now + rng.integers(-10, 10, len(rows[4::11])))
    dep_rows = rows[2::5]
    entries = [[(abi.DEPENDEE_PENDING, int(r) - 1, int(rng.integers(0, 4)), 0, 0)] if k % 2 else
               [(abi.DEPENDEE_RUNNING, k % rn.n, int(rng.integers(0, 4)), 0, 0)] for k, r in enumerate(dep_rows)]
    s.pending_depend(abi.Dependencies.from_lists(dep_rows, (dep_rows % 3 == 0).astype(np.uint8), entries))
    s.pending_cancel(dep_rows[1:4] - 1, now - 50)
    s.running_end([0, 1], [now - 20, now - 10], [0, 1])
    s.keep_running()


def _shard_worker(rank, world, port, emu_lib, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from cranesched_b200 import sharding
    cfg, cl, rn, pd, now = synth.random_case(76, n_jobs=90, n_nodes=30, n_parts=4, n_running=16, limit=60)
    owner = sharding.deal_partitions(pd, cl.n_partitions, world, cl)
    s = GpuScheduler(cfg, 0, emu_lib)
    s.set_cluster(cl)
    s.set_shard(rank, world, owner)
    _gate_calls(s, pd, rn, now)
    got = sharding.sharded_tick(s, now, rn, pd, owner, dist, on_gpu=False, upload=False)
    s.close()
    u = GpuScheduler(cfg, 0, emu_lib)
    u.set_cluster(cl)
    _gate_calls(u, pd, rn, now)
    u.run(now)
    ref = u.fetch(abi.Placements.for_pending(pd))
    u.close()
    d = ref.diff(got)
    gated = int(np.isin(ref.reason, [abi.REASON_HELD, abi.REASON_BEGIN_TIME, abi.REASON_DEPENDENCY,
                                     abi.REASON_DEPENDENCY_NEVER]).sum())
    q.put((rank, d[:3], gated))
    dist.destroy_process_group()


def test_gated_sharded_tick_equals_unsplit_gloo(emu_lib):
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_shard_worker, args=(r, world, port, emu_lib, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=900) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, d, gated in res:
        assert not d, f"rank {rank}: the gated sharded tick differs from the unsplit one: {d}"
        assert gated > 10
