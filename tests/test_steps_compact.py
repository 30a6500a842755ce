"""crane_sched_steps_compact: the resident step tables and the allocation pool of running
steps compacted on the device.

Two handles get the same calls; `a` never compacts, `b` compacts at several points (right
after a pass that scheduled steps, twice in a row, on tables without tombstones, right
after step_jobs_start, after erasing jobs with running steps). The caller translates a's
rows through the composed maps. After every pass b's fetched results equal a's byte for
byte at the mapped step rows, step_jobs_avail is equal, and on some passes b's results
equal the step oracle; steps that were running when b compacted later end on both handles
and give back the same avail. Also: exact maps and row counts on a hand-built table
(CRANE_ROW_NONE, a job without nodes, steps without lists, an unknown host in an include
list), calls at mapped rows, argument codes, and isolation from NodeSelect and from
crane_sched_compact. On the emulator here and on the GPU in the `gpu`-marked tests; the
emulated twins take their step jobs from running_append rows rather than from a NodeSelect
run, which keeps the emulated part of this file to about half a minute."""
import numpy as np
import pytest

from cranesched_b200 import abi, synth
from cranesched_b200.scheduler import GpuScheduler
from tests.test_steps_resident import _Model, _arrive, _code, _one_job, _steps

NONE = abi.ROW_NONE


@pytest.fixture(scope="module")
def steps_oracle():
    from oracle import pystep
    pystep.build()
    return pystep


def _compose(m, new):
    """a's rows -> b's rows, after b compacted with map `new`"""
    out = m.copy()
    ok = out != NONE
    out[ok] = new[out[ok]]
    return out


def _same_results(ra, rb, sm):
    assert rb.step_row.tolist() == sm[ra.step_row.astype(np.int64)].tolist()
    for f in ("node_off", "alloc_node", "alloc_ntasks", "alloc_res", "task_off", "task_node", "task_res"):
        assert getattr(ra, f).tobytes() == getattr(rb, f).tobytes(), f


class _Twin:
    """Handles a (never compacts) and b (compacts); jm / sm map a's step-job / step rows to b's."""

    def __init__(self, a, b):
        self.a, self.b = a, b
        self.jm = np.zeros(0, np.int64)
        self.sm = np.zeros(0, np.int64)
        self.compactions = 0

    def J(self, rows):
        return self.jm[np.asarray(rows, np.int64)]

    def S(self, rows):
        return self.sm[np.asarray(rows, np.int64)]

    def step_jobs_start(self, rows):
        fa, fb = self.a.step_jobs_start(rows), self.b.step_jobs_start(rows)
        self.jm = np.concatenate([self.jm, fb + np.arange(len(rows))])
        return fa

    def step_jobs_append(self, jobs):
        fa, fb = self.a.step_jobs_append(jobs), self.b.step_jobs_append(jobs)
        self.jm = np.concatenate([self.jm, fb + np.arange(jobs.n_jobs)])
        return fa

    def steps_append(self, steps, rows):
        fa, fb = self.a.steps_append(steps, rows), self.b.steps_append(steps, self.J(rows))
        self.sm = np.concatenate([self.sm, fb + np.arange(steps.n)])
        return fa

    def steps_erase(self, rows):
        self.a.steps_erase(rows)
        self.b.steps_erase(self.S(rows))

    def step_jobs_erase(self, rows):
        self.a.step_jobs_erase(rows)
        self.b.step_jobs_erase(self.J(rows))

    def compact(self, live=None):
        """With live = (a's live step-job rows, a's live step rows), NULL maps: the maps
        are then the ranks of those rows among b's, since kept rows keep their order."""
        before = self.b.step_rows()
        jm, sm = self.b.steps_compact(live is None)
        self.compactions += 1
        if live is not None:
            assert (jm, sm) == (None, None)
            jm, sm = np.full(before[0], NONE, np.int64), np.full(before[1], NONE, np.int64)
            for m, rows in ((jm, self.J(live[0])), (sm, self.S(live[1]))):
                m[np.sort(rows)] = np.arange(len(rows))
            assert self.b.step_rows()[:2] == (len(live[0]), len(live[1]))
        assert len(jm) == before[0] and len(sm) == before[1]
        self.jm, self.sm = _compose(self.jm, jm), _compose(self.sm, sm)
        return jm, sm

    def run(self):
        ra, _ = self.a.steps_run()
        rb, _ = self.b.steps_run()
        _same_results(ra, rb, self.sm)
        return ra, rb

    def check_avail(self, live):
        live = sorted(live)
        assert self.a.step_jobs_avail(live).tobytes() == self.b.step_jobs_avail(self.J(live)).tobytes()

    def close(self):
        self.a.close()
        self.b.close()


def _follow(model, a, res):
    """The model takes a pass's results (a's rows) and a's avail."""
    got = set(res.step_row.tolist())
    at = {int(s): k for k, s in enumerate(res.step_row)}
    for j, jb in model.jobs.items():
        q, k = jb["queue"], 0
        while k < len(q) and q[k] in got:
            r = at[q[k]]
            n0, n1 = res.node_off[r], res.node_off[r + 1]
            model.running[q[k]] = (j, res.alloc_node[n0:n1].copy(), res.alloc_res[n0:n1].copy())
            k += 1
        jb["queue"] = q[k:]
    live = sorted(model.jobs)
    if live:
        av = a.step_jobs_avail(live)
        at = 0
        for j in live:
            n = len(model.jobs[j]["nodes"])
            model.jobs[j]["avail"] = av[at:at + n].copy()
            at += n


def _start_twins(lib, case, seed, via_run=True):
    """Two handles with the same running rows; half of them become step jobs now, the rest
    are returned for a later step_jobs_start. via_run: the rows a NodeSelect run starts
    (crane_sched_start); else the case's running jobs (running_append) next to its pending
    table, which spares the emulator the run."""
    cfg, cl, rn, pd, now = case
    rng = np.random.Generator(np.random.PCG64(seed))
    a, b = GpuScheduler(cfg, 0, lib), GpuScheduler(cfg, 0, lib)
    got = None
    for s in (a, b):
        s.set_cluster(cl)
        if not via_run:
            s.pending_append(pd)
            s.running_append(rn)
            continue
        s.upload(rn, pd)
        s.run(now)
        g = s.fetch(abi.Placements.for_pending(pd))
        assert got is None or not got.diff(g)
        got = g
    if via_run:
        sel = rng.permutation(np.flatnonzero(got.reason == abi.REASON_NONE))
        first = a.start(sel)
        assert b.start(sel) == first
        started = abi.Running.started(pd, got, sel)
    else:
        sel, first, started = rng.permutation(rn.n), 0, rn
    tw, model = _Twin(a, b), _Model()
    half = len(sel) // 2

    def start(ks):
        ks = list(ks)
        j0 = tw.step_jobs_start(first + np.asarray([sel[k] for k in ks] if not via_run else ks, np.int64))
        for i, k in enumerate(ks):
            r = k if via_run else sel[k]
            x, y = started.alloc_off[r], started.alloc_off[r + 1]
            model.add_job(j0 + i, started.alloc_node[x:y], started.alloc_res[x:y], started.alloc_res[x:y])

    start(range(half))
    return tw, model, cl, lambda: start(range(half, len(sel)))


def _twin_trajectory(lib, case, seed, n_passes=7, steps_oracle=None, oracle_every=3, via_run=True):
    """Returns (steps scheduled, steps running at a compaction that ended later, jobs
    erased with running steps)."""
    rng = np.random.Generator(np.random.PCG64(seed + 7))
    tw, model, cl, start_rest = _start_twins(lib, case, seed, via_run)
    seen = np.zeros(3, np.int64)
    held = set()  # a's step rows that were running when b compacted
    try:
        jm, sm = tw.compact()  # no tombstones yet: identity, nothing moves
        assert np.array_equal(jm, np.arange(len(jm))) and np.array_equal(sm, np.arange(len(sm)))
        for p in range(n_passes):
            _arrive(tw, model, cl, seed * 100 + p)
            if p == 2:
                start_rest()
                tw.compact()  # right after step_jobs_start
                _arrive(tw, model, cl, seed * 100 + 50 + p)
            pend = [q for j in model.jobs for q in model.jobs[j]["queue"]]
            heads = [model.jobs[j]["queue"][0] for j in model.jobs if model.jobs[j]["queue"]]
            gone = set(rng.choice(heads, min(len(heads), 2), replace=False).tolist()) if p and heads else set()
            gone |= {q for q in pend if rng.random() < 0.05}
            if gone:
                tw.steps_erase(sorted(gone))
                for j in model.jobs:
                    model.jobs[j]["queue"] = [q for q in model.jobs[j]["queue"] if q not in gone]
            ended = [q for q in sorted(model.running) if rng.random() < 0.4]
            if ended:
                tw.steps_erase(rng.permutation(ended))
                for q in ended:
                    model.release(q)
                seen[1] += len(held & set(ended))
            if p % 2 == 1 and len(model.jobs) > 4:
                busy = sorted({v[0] for v in model.running.values()})
                out = rng.choice(busy, min(2, len(busy)), replace=False).tolist() if busy else []
                out = (out + [j for j in sorted(model.jobs) if j not in out])[:2]
                seen[2] += sum(1 for j in out if j in busy)
                tw.step_jobs_erase(out)
                for j in out:
                    del model.jobs[int(j)]
                model.running = {q: v for q, v in model.running.items() if v[0] in model.jobs}
                # after erasing jobs with running steps; once with NULL maps
                steps = sorted(model.running) + [q for jb in model.jobs.values() for q in jb["queue"]]
                tw.compact(live=(sorted(model.jobs), steps) if p == 3 else None)
            # the pass; on some passes b's results against the oracle over every job with pending steps
            check = steps_oracle is not None and p % oracle_every == 0
            if check:
                rows, tj, ts, srows = model.twin_tables()
                ref, _ = steps_oracle.schedule_steps(cl, tj, ts)
            ra, rb = tw.run()
            if check:
                got = rb.expand(tw.S(srows), tj.step_off, ts)
                assert not ref.diff(got), (p, ref.diff(got)[:4])
            _follow(model, tw.a, ra)
            seen[0] += ra.n
            tw.check_avail(model.jobs)
            if p in (1, 3) and ra.n:  # right after a pass that scheduled steps, twice in a row at p == 3
                held |= set(model.running)
                tw.compact()
                if p == 3:
                    tw.compact()
                tw.check_avail(model.jobs)
        # the steps still running end on both handles: the same avail comes back
        if model.running:
            ended = sorted(model.running)
            seen[1] += len(held & set(ended))
            tw.steps_erase(ended)
            model.running = {}
        tw.check_avail(model.jobs)
        ra, rb = tw.run()
        _follow(model, tw.a, ra)
        # the compacted pool holds exactly the node rows of the steps this last pass scheduled
        tw.compact()
        n_pending = sum(len(jb["queue"]) for jb in model.jobs.values())
        assert tw.b.step_rows() == (len(model.jobs), n_pending + ra.n, int(ra.node_off[-1]))
        assert tw.compactions >= 6
    finally:
        tw.close()
    return seen


EMU_SEEDS = [31, 32, 33]


@pytest.mark.parametrize("seed", EMU_SEEDS)
def test_steps_compact_twin_emulated(steps_oracle, emu_lib, seed):
    case = synth.random_case(seed, n_jobs=40, n_nodes=16, n_running=24, ntpn_range=True,
                             one_type_per_name=bool(seed & 1))
    seen = _twin_trajectory(emu_lib, case, seed, n_passes=6, steps_oracle=steps_oracle, via_run=False)
    assert (seen > 0).all(), seen


@pytest.mark.gpu
@pytest.mark.parametrize("seed", EMU_SEEDS + [34, 35, 36])
def test_steps_compact_twin_gpu(steps_oracle, gpu_lib, seed):
    case = synth.random_case(seed, n_jobs=800, n_nodes=96, n_running=30, ntpn_range=True,
                             one_type_per_name=bool(seed & 1))
    seen = _twin_trajectory(gpu_lib, case, seed, n_passes=9, steps_oracle=steps_oracle)
    assert (seen > 0).all(), seen


# ---- a hand-built table -------------------------------------------------------------------

def _hand(lib):
    """Jobs 0: nodes 0, 1; 1: nodes 2, 3; 2: no nodes; 3: nodes 4, 5 (4 cores each).
    Steps 0 (job 0), 1 (job 1), 2 (job 3, two nodes) are scheduled by the first pass;
    3 (job 0), 4 (job 3), 5 (job 1) ask for 8 cpus and block their jobs; 6 (job 0, behind
    3) has the include list [unknown host, node 1]."""
    cl = synth.make_cluster([(6, synth.node_row(8, 64 * synth.GiB))])
    s = GpuScheduler(abi.Config(), 0, lib)
    s.set_cluster(cl)
    nodes = [[0, 1], [2, 3], [], [4, 5]]
    off = np.zeros(5, np.uint32)
    off[1:] = np.cumsum([len(n) for n in nodes])
    avail = np.stack([synth.node_row(4, 8 * synth.GiB)] * int(off[-1]))
    assert s.step_jobs_append(abi.StepJobs(off, np.array(sum(nodes, []), np.uint32), avail, np.zeros(5, np.uint32))) == 0
    rows = [(1, 1, 1, 1, 1), (1, 1, 1, 1, 1), (2, 2, 1, 1, 1), (1, 1, 1, 1, 8), (1, 1, 1, 1, 8), (1, 1, 1, 1, 8),
            (1, 1, 1, 1, 1)]
    incl = [[], [], [], [], [], [], [0xFFFFFFFF, 1]]
    assert s.steps_append(_steps(rows, incl), [0, 1, 3, 0, 3, 1, 0]) == 0
    res, _ = s.steps_run()
    assert res.step_row.tolist() == [0, 1, 2]
    return s


def test_steps_compact_maps_and_rows(emu_lib):
    a, b = _hand(emu_lib), _hand(emu_lib)
    try:
        assert b.step_rows() == (4, 7, 4)
        # nothing erased: identity maps, nothing moves; NULL maps too
        jm, sm = b.steps_compact()
        assert jm.tolist() == [0, 1, 2, 3] and sm.tolist() == list(range(7))
        assert b.steps_compact(maps=False) == (None, None)
        assert b.step_rows() == (4, 7, 4)
        for s in (a, b):
            s.steps_erase([3, 2])     # a pending head (job 0) and a scheduled step (job 3) end
            s.step_jobs_erase([1])    # job 1 goes with its scheduled step 1 and pending step 5
        assert b.step_rows() == (4, 7, 4)
        jm, sm = b.steps_compact()
        assert jm.tolist() == [0, NONE, 1, 2]
        assert sm.tolist() == [0, NONE, NONE, NONE, 1, NONE, 2]
        assert b.step_rows() == (3, 3, 1)  # the pool keeps step 0's node row only
        tw = _Twin(a, b)
        tw.jm, tw.sm = jm.astype(np.int64), sm.astype(np.int64)
        tw.check_avail([0, 2, 3])
        # job 0 is dirty (its head went): step 6 with the unknown host in its include list
        ra, rb = tw.run()
        tw.check_avail([0, 2, 3])
        # step 0 was running at compaction: erased at its new row, it gives the same rows back
        tw.steps_erase([0])
        tw.check_avail([0, 2, 3])
        ra, rb = tw.run()
        tw.check_avail([0, 2, 3])
        # everything erased
        tw.step_jobs_erase([0, 2, 3])
        jm, sm = b.steps_compact()
        assert (jm == NONE).all() and (sm == NONE).all() and b.step_rows() == (0, 0, 0)
        res, _ = b.steps_run()
        assert res.n == 0
        assert b.step_jobs_append(_one_job([0, 1], [4, 4])) == 0
    finally:
        a.close()
        b.close()


def test_steps_compact_no_step_scheduled(emu_lib):
    """n_alloc == 0, steps without include / exclude lists, a job without nodes"""
    s = GpuScheduler(abi.Config(), 0, emu_lib)
    try:
        s.set_cluster(synth.make_cluster([(4, synth.node_row(8, 64 * synth.GiB))]))
        s.step_jobs_append(abi.StepJobs([0, 0, 2], [0, 1], np.stack([synth.node_row(4, 8 * synth.GiB)] * 2), [0, 0, 0]))
        s.steps_append(_steps([(1, 1, 1, 1, 8), (1, 1, 1, 1, 1), (1, 1, 1, 1, 1)]), [1, 1, 0])
        s.steps_erase([1])
        jm, sm = s.steps_compact()
        assert jm.tolist() == [0, 1] and sm.tolist() == [0, NONE, 1] and s.step_rows() == (2, 2, 0)
        s.steps_erase([0])  # the blocking head goes
        res, _ = s.steps_run()
        assert res.n == 0  # step 1 belongs to the job without nodes
        s.steps_append(_steps([(1, 1, 1, 1, 1)]), [1])
        res, _ = s.steps_run()
        assert res.step_row.tolist() == [2] and s.step_rows() == (2, 3, 1)
    finally:
        s.close()


def test_calls_after_compaction_use_new_rows(emu_lib):
    a, b = _hand(emu_lib), _hand(emu_lib)
    tw = _Twin(a, b)
    tw.jm, tw.sm = np.arange(4), np.arange(7)
    try:
        tw.steps_erase([3])
        tw.step_jobs_erase([2])
        tw.compact()
        assert tw.J([0, 1, 3]).tolist() == [0, 1, 2] and tw.S([0, 1, 2, 6]).tolist() == [0, 1, 2, 5]
        # old rows past the new end
        assert _code(b.step_jobs_avail, [3]) == abi.EINVAL
        assert _code(b.steps_erase, [6]) == abi.EINVAL
        assert _code(b.step_jobs_erase, [3]) == abi.EINVAL
        assert _code(b.steps_append, _steps([(1, 1, 1, 1, 1)]), [3]) == abi.EINVAL
        # the same calls at the mapped rows act as on the uncompacted twin
        assert tw.steps_append(_steps([(1, 1, 1, 1, 1), (1, 1, 1, 1, 1)]), [3, 1]) == 7
        assert b.step_rows()[1] == 8
        tw.steps_erase([1])      # scheduled: its node row goes back to job 1
        tw.check_avail([0, 1, 3])
        tw.run()
        tw.check_avail([0, 1, 3])
        tw.step_jobs_erase([1])
        tw.check_avail([0, 3])
        tw.run()
        tw.compact()
        tw.run()
        tw.check_avail([0, 3])
        # steps_run after compaction appends its node rows at the compacted end of the pool
        n_alloc = b.step_rows()[2]
        tw.steps_append(_steps([(1, 1, 1, 1, 1)]), [0])
        _, rb = tw.run()
        assert rb.n == 1 and b.step_rows()[2] == n_alloc + 1
        tw.steps_erase([9])
        tw.check_avail([0, 3])
    finally:
        tw.close()


# ---- argument codes and isolation -----------------------------------------------------------

def test_steps_compact_arguments(emu_lib):
    s = GpuScheduler(abi.Config(), 0, emu_lib)
    try:
        assert s.step_rows() == (0, 0, 0)
        assert _code(s.steps_compact) == abi.EINVAL  # set_cluster first
        assert s._lib.crane_sched_steps_compact(None, None, None) == abi.EINVAL
        assert s._lib.crane_sched_step_rows(None, None, None, None) == abi.EINVAL
        assert s._lib.crane_sched_step_rows(s._h, None, None, None) == 0
    finally:
        s.close()
    s = _hand(emu_lib)
    try:
        s.steps_compact()  # voids the fetch
        out = abi.StepResults.sized(0, 0, 0)
        assert s._lib.crane_sched_steps_fetch(s._h, out.as_c()) == abi.EINVAL
    finally:
        s.close()


def _ticks(lib, case, seed, with_steps, n_ticks=2):
    """Resident NodeSelect ticks; with_steps puts step calls and steps_compact between
    every fetch and start and after every start. Returns the fetched ticks."""
    cfg, cl, rn, pd, now = case
    rng = np.random.Generator(np.random.PCG64(seed))
    s = GpuScheduler(cfg, 0, lib)
    outs = []
    try:
        s.set_cluster(cl)
        s.pending_append(pd)
        s.running_append(rn)
        jobs = set()
        for t in range(n_ticks):
            s.keep_running()
            s.run(now)
            got = s.fetch(abi.Placements.for_pending(pd))
            outs.append(got)
            if with_steps and jobs:
                live = sorted(jobs)
                s.steps_append(_steps([(1, 1, 1, 1, 1)] * len(live)), live)
                res, _ = s.steps_run()
                if res.n:
                    s.steps_erase(res.step_row[:1])
                s.step_jobs_erase(live[:1])
                jm, _ = s.steps_compact()
                jobs = {int(jm[j]) for j in live[1:]}
            sel = rng.permutation(np.flatnonzero(got.reason == abi.REASON_NONE))[:20]
            first = s.start(sel)  # after a fetch, with step calls and steps_compact between
            if with_steps:
                j0 = s.step_jobs_start(first + np.arange(len(sel)))
                jobs |= set(range(j0, j0 + len(sel)))
                s.steps_compact()
            now += 600
            if t % 2:
                s.running_erase(rng.choice(s.running_rows(), 3, replace=False))
    finally:
        s.close()
    return outs


def test_steps_compact_leaves_node_select_alone(emu_lib):
    case = synth.random_case(41, n_jobs=30, n_nodes=8, n_parts=2, n_running=4, short=True)
    a = _ticks(emu_lib, case, 41, with_steps=False)
    b = _ticks(emu_lib, case, 41, with_steps=True)
    for t, (x, y) in enumerate(zip(a, b)):
        assert not x.diff(y), (t, x.diff(y)[:4])


def test_compactions_leave_each_other_alone(emu_lib):
    """crane_sched_compact and steps_compact, in either order, touch disjoint tables: each
    leaves the other's row counts alone, and both orders end in the same state."""
    case = synth.random_case(42, n_jobs=30, n_nodes=8, n_running=12)
    cfg, cl, rn, pd, now = case
    outs = []
    for order in (0, 1):
        tw, model, _, _ = _start_twins(emu_lib, case, 42, via_run=False)
        try:
            _arrive(tw, model, cl, 7)
            ra, _ = tw.run()
            _follow(model, tw.a, ra)
            live = sorted(model.jobs)
            tw.step_jobs_erase(live[:1])
            del model.jobs[live[0]]
            model.running = {q: v for q, v in model.running.items() if v[0] != live[0]}
            n_pending = sum(len(jb["queue"]) for jb in model.jobs.values())
            for s in (tw.a, tw.b):
                s.pending_erase([0, 1])
                s.running_erase([0])
            if order:
                rows = (tw.b.pending_rows(), tw.b.running_rows())
                tw.compact()
                assert (tw.b.pending_rows(), tw.b.running_rows()) == rows
                pm, rm = tw.b.compact()
            else:
                steps = tw.b.step_rows()
                pm, rm = tw.b.compact()
                assert tw.b.step_rows() == steps
                tw.compact()
            assert pm[0] == pm[1] == rm[0] == NONE and tw.b.step_rows()[:2] == (len(live) - 1, len(model.running) + n_pending)
            tw.check_avail(live[1:])
            if model.running:
                tw.steps_erase(sorted(model.running))
            tw.check_avail(live[1:])
            tw.run()
            tw.b.keep_running()
            tw.b.run(now)
            outs.append((tw.b.fetch(abi.Placements.for_pending(pd.take(np.flatnonzero(pm != NONE)))), pm, rm,
                         tw.b.step_jobs_avail(tw.J(live[1:]))))
        finally:
            tw.close()
    (x, pm0, rm0, av0), (y, pm1, rm1, av1) = outs
    assert not x.diff(y) and np.array_equal(pm0, pm1) and np.array_equal(rm0, rm1) and av0.tobytes() == av1.tobytes()


# ---- config 2 -------------------------------------------------------------------------------

@pytest.mark.gpu
def test_steps_compact_config2(gpu_lib):
    """The jobs GPU NodeSelect starts on config 2 and the steps of step_case(2): a pass,
    some jobs and steps erased, compaction, then half the running steps end. The avail
    and the next pass equal a never-compacted twin's."""
    case = synth.config2()
    cfg, cl, rn, pd, now = case
    rng = np.random.Generator(np.random.PCG64(2))
    a, b = GpuScheduler(cfg, 0, gpu_lib), GpuScheduler(cfg, 0, gpu_lib)
    tw = _Twin(a, b)
    try:
        for s in (a, b):
            s.set_cluster(cl)
            s.upload(rn, pd)
            s.run(now)
        got = a.fetch(abi.Placements.for_pending(pd))
        assert not got.diff(b.fetch(abi.Placements.for_pending(pd)))
        _, jobs, steps = synth.step_case(2, lambda *c: got, base=case)
        started = np.flatnonzero(got.reason == abi.REASON_NONE)
        first = a.start(started)
        assert b.start(started) == first
        j0 = tw.step_jobs_start(first + np.arange(len(started)))
        owner = np.repeat(np.arange(jobs.n_jobs), np.diff(jobs.step_off)) + j0
        s0 = tw.steps_append(steps, owner)
        ra, _ = tw.run()
        assert ra.n > 1000
        sched = ra.step_row.astype(np.int64)
        sched_set = set(sched.tolist())
        pending = np.array([s0 + i for i in range(steps.n) if s0 + i not in sched_set], np.int64)
        gone_jobs = rng.choice(jobs.n_jobs, jobs.n_jobs // 10, replace=False) + j0
        tw.step_jobs_erase(gone_jobs)
        gone = set(gone_jobs.tolist())
        alive = lambda rows: np.array([r for r in rows if int(owner[r - s0]) not in gone], np.int64)
        sched, pending = alive(sched), alive(pending)
        tw.steps_erase(np.concatenate([rng.choice(sched, len(sched) // 5, replace=False),
                                       rng.choice(pending, len(pending) // 5, replace=False)]))
        before = b.step_rows()
        tw.compact()
        after = b.step_rows()
        assert after[0] < before[0] and after[1] < before[1] and after[2] < before[2]
        live = np.array(sorted(set(range(j0, j0 + jobs.n_jobs)) - gone), np.int64)
        tw.check_avail(live)
        still = np.array([r for r in sched if tw.sm[r] != NONE], np.int64)
        tw.steps_erase(rng.choice(still, len(still) // 2, replace=False))
        tw.check_avail(live)
        ra, rb = tw.run()
        assert ra.n > 0
        rb.step_row = ra.step_row  # (tw.run checked rb's rows are ra's, mapped)
        assert rb.digest() == ra.digest()
        tw.check_avail(live)
    finally:
        tw.close()
