"""The step state of running jobs kept resident on the device (crane_sched_step_jobs_* /
crane_sched_steps_*).

Trajectories of passes over jobs an emulated NodeSelect run starts (crane_sched_start,
then step_jobs_start) and jobs appended from host rows (one with a crun primary taken
from its avail). Each pass has step arrivals, erases of pending steps (a blocked queue
head among them), erases of scheduled steps (their allocation goes back), job erases,
and one pass compacts the tables (reset, then the live jobs and their pending steps
again). A host model keeps every job's avail and FIFO queue; after every pass
  - the fetched results, expanded to the StepPlacements of all the model's jobs with
    pending steps, are byte-identical to a twin handle's crane_sched_schedule_steps over
    those jobs (so skipping clean jobs changes nothing), and on some passes to the oracle;
  - step_jobs_avail equals the model's avail.
Also: an idle pass, isolation from NodeSelect, and the argument checks. On the emulator
here and on the GPU in the `gpu`-marked twins."""
import dataclasses

import numpy as np
import pytest

from cranesched_b200 import abi, synth
from cranesched_b200.scheduler import CraneSchedError, GpuScheduler


@pytest.fixture(scope="module")
def steps_oracle():
    from oracle import pystep
    pystep.build()
    return pystep


def _code(fn, *args):
    try:
        fn(*args)
        return 0
    except CraneSchedError as e:
        return e.code


def _steps_of(refs):
    """A Steps table of the rows refs = [(Steps, row), ...], in this order."""
    cols = {f: [] for f in ("node_num", "ntasks", "ntasks_per_node_min", "ntasks_per_node_max", "req_node", "req_task")}
    lists = {"incl": ([0], []), "excl": ([0], [])}
    for t, i in refs:
        for f in cols:
            cols[f].append(getattr(t, f)[i])
        for k, (off, nodes) in lists.items():
            o = getattr(t, k + "_off")
            nodes += getattr(t, k + "_nodes")[o[i]:o[i + 1]].tolist()
            off.append(len(nodes))
    return abi.Steps(np.array(cols["node_num"], np.uint32), np.array(cols["ntasks"], np.uint32),
                     np.array(cols["ntasks_per_node_min"], np.uint32), np.array(cols["ntasks_per_node_max"], np.uint32),
                     np.array(cols["req_node"], abi.RES_VIEW).reshape(-1), np.array(cols["req_task"], abi.RES_VIEW).reshape(-1),
                     np.array(lists["incl"][0], np.uint32), np.array(lists["incl"][1], np.uint32),
                     np.array(lists["excl"][0], np.uint32), np.array(lists["excl"][1], np.uint32))


def _row_add(a, b):
    """ResourceInNodeV3 += (EraseStep: step_res_avail_ += AllocatedRes())"""
    for f in ("cpu_raw", "mem", "mem_sw"):
        a[f] += b[f]
    a["core"] |= b["core"]
    a["gres"] |= b["gres"]


class _Model:
    """The daemon's step state of its running jobs, on the host."""

    def __init__(self):
        self.jobs = {}   # step-job row -> dict(nodes, avail, alloc, queue)
        self.ref = {}    # step row -> (Steps, row)
        self.running = {}  # step row -> (job row, node rows, res rows)

    def add_job(self, row, nodes, avail, alloc):
        self.jobs[row] = dict(nodes=np.array(nodes, np.uint32), avail=np.array(avail).copy(), alloc=np.array(alloc).copy(),
                              queue=[])

    def release(self, s):
        j, nodes, res = self.running.pop(s)
        jb = self.jobs[j]
        for n, r in zip(nodes, res):
            _row_add(jb["avail"][int(np.searchsorted(jb["nodes"], n))], r)

    def twin_tables(self):
        """StepJobs + Steps of every job with pending steps (row order), and each step's row."""
        rows = [j for j in sorted(self.jobs) if self.jobs[j]["queue"]]
        node_off, step_off, steps = [0], [0], []
        for j in rows:
            node_off.append(node_off[-1] + len(self.jobs[j]["nodes"]))
            steps += self.jobs[j]["queue"]
            step_off.append(len(steps))
        cat = lambda k, dt: np.concatenate([self.jobs[j][k] for j in rows]) if rows else np.zeros(0, dt)
        jobs = abi.StepJobs(np.array(node_off, np.uint32), cat("nodes", np.uint32), cat("avail", abi.RES_IN_NODE),
                            np.array(step_off, np.uint32))
        return rows, jobs, _steps_of([self.ref[s] for s in steps]), np.array(steps, np.int64)


def _crun_primary(avail):
    """avail after a crun primary took one cpu of its first node (InitPrimaryStepFromJob)."""
    a = avail.copy()
    core = int(a["core"][0, 0])
    if core and a["cpu_raw"][0] >= 256:
        a["core"][0, 0] = core & (core - 1)
        a["cpu_raw"][0] -= 256
        a["mem"][0] //= 2
    return a


def _start_jobs(lib, case, seed, n_host=3, select_frac=0.7):
    """A handle with a NodeSelect run; a subset of its start-now rows started through
    crane_sched_start + step_jobs_start, a few more appended from host rows (the first of
    them as a crun primary). Returns (handle, model, cluster)."""
    cfg, cl, rn, pd, now = case
    rng = np.random.Generator(np.random.PCG64(seed))
    s = GpuScheduler(cfg, 0, lib)
    s.set_cluster(cl)
    s.upload(rn, pd)
    s.run(now)
    got = s.fetch(abi.Placements.for_pending(pd))
    now_rows = rng.permutation(np.flatnonzero(got.reason == abi.REASON_NONE))
    host_rows, sel = now_rows[:n_host], now_rows[n_host:]
    sel = sel[rng.random(len(sel)) < select_frac]
    first = s.start(sel)
    model = _Model()
    started = abi.Running.started(pd, got, sel)
    j0 = s.step_jobs_start(first + np.arange(len(sel)))
    for k in range(len(sel)):
        a, b = started.alloc_off[k], started.alloc_off[k + 1]
        model.add_job(j0 + k, started.alloc_node[a:b], started.alloc_res[a:b], started.alloc_res[a:b])
    other = abi.Running.started(pd, got, host_rows)
    avail = other.alloc_res.copy()
    if len(host_rows):
        a, b = other.alloc_off[0], other.alloc_off[1]
        avail[a:b] = _crun_primary(avail[a:b])
    j1 = s.step_jobs_append(abi.StepJobs(other.alloc_off, other.alloc_node, avail, np.zeros(len(host_rows) + 1, np.uint32)))
    for k in range(len(host_rows)):
        a, b = other.alloc_off[k], other.alloc_off[k + 1]
        model.add_job(j1 + k, other.alloc_node[a:b], avail[a:b], other.alloc_res[a:b])
    return s, model, cl


def _arrive(s, model, cl, seed):
    live = sorted(model.jobs)
    if not live:
        return 0
    node_off = np.zeros(len(live) + 1, np.int64)
    node_off[1:] = np.cumsum([len(model.jobs[j]["nodes"]) for j in live])
    node = np.concatenate([model.jobs[j]["nodes"] for j in live])
    alloc = np.concatenate([model.jobs[j]["alloc"] for j in live])
    owner, steps = synth.step_pass_stream(seed, node_off, node, alloc, range(len(live)), cl)
    if not steps.n:
        return 0
    rows = np.array(live, np.int64)[owner]
    first = s.steps_append(steps, rows)
    for i in range(steps.n):
        model.ref[first + i] = (steps, i)
        model.jobs[int(rows[i])]["queue"].append(first + i)
    return steps.n


def _compact(s, model):
    """step_jobs_reset, then the live jobs from host rows and their pending steps again
    (the scheduled ones end first)."""
    if model.running:
        ended = sorted(model.running)
        s.steps_erase(ended)
        for st in ended:
            model.release(st)
    old = model.jobs
    s.step_jobs_reset()
    model.jobs, model.ref = {}, {k: v for k, v in model.ref.items()}
    live = sorted(old)
    if not live:
        return
    off = np.zeros(len(live) + 1, np.uint32)
    off[1:] = np.cumsum([len(old[j]["nodes"]) for j in live])
    j0 = s.step_jobs_append(abi.StepJobs(off, np.concatenate([old[j]["nodes"] for j in live]),
                                         np.concatenate([old[j]["avail"] for j in live]), np.zeros(len(live) + 1, np.uint32)))
    refs, owner = [], []
    for k, j in enumerate(live):
        model.add_job(j0 + k, old[j]["nodes"], old[j]["avail"], old[j]["alloc"])
        refs += [model.ref[q] for q in old[j]["queue"]]
        owner += [j0 + k] * len(old[j]["queue"])
    model.ref = {}
    if refs:
        first = s.steps_append(_steps_of(refs), owner)
        for i, j in enumerate(owner):
            model.ref[first + i] = refs[i]
            model.jobs[j]["queue"].append(first + i)


def _trajectory(lib, case, seed, n_passes=8, steps_oracle=None, oracle_every=3, compact_at=5):
    """Returns (steps scheduled, pending erased, scheduled erased, jobs erased) over the passes."""
    cfg = case[0]
    rng = np.random.Generator(np.random.PCG64(seed + 7))
    s, model, cl = _start_jobs(lib, case, seed)
    twin = GpuScheduler(cfg, 0, lib)
    twin.set_cluster(cl)
    seen = np.zeros(4, np.int64)
    try:
        for p in range(n_passes):
            _arrive(s, model, cl, seed * 100 + p)
            if p == compact_at:
                _compact(s, model)
            # pending steps leave: a blocked head (the queue stays blocked behind it otherwise) and a few others
            pend = [(j, q) for j in model.jobs for q in model.jobs[j]["queue"]]
            heads = [model.jobs[j]["queue"][0] for j in model.jobs if model.jobs[j]["queue"]]
            gone = set(rng.choice(heads, min(len(heads), 2), replace=False).tolist()) if p and heads else set()
            gone |= {q for j, q in pend if rng.random() < 0.05}
            if gone:
                s.steps_erase(sorted(gone))
                for j in model.jobs:
                    model.jobs[j]["queue"] = [q for q in model.jobs[j]["queue"] if q not in gone]
                seen[1] += len(gone)
            # scheduled steps end: their allocation goes back
            ended = [q for q in sorted(model.running) if rng.random() < 0.4]
            if ended:
                s.steps_erase(rng.permutation(ended))
                for q in ended:
                    model.release(q)
                seen[2] += len(ended)
            # jobs end
            if p % 3 == 2 and len(model.jobs) > 4:
                out = rng.choice(sorted(model.jobs), 2, replace=False)
                s.step_jobs_erase(out)
                for j in out:
                    del model.jobs[int(j)]
                model.running = {q: v for q, v in model.running.items() if v[0] in model.jobs}
                seen[3] += 2
            # the pass, and its twin over every job with pending steps
            res, ms = s.steps_run()
            assert ms >= 0
            rows, tj, ts, srows = model.twin_tables()
            ref_jobs = tj.copy()
            want, _ = twin.schedule_steps(tj, ts)
            got = res.expand(srows, tj.step_off, ts)
            d = want.diff(got)
            assert not d, f"pass {p}: resident pass differs from schedule_steps:\n" + "\n".join(d[:8])
            assert want.digest() == got.digest()
            if steps_oracle is not None and p % oracle_every == 0:
                ref, _ = steps_oracle.schedule_steps(cl, ref_jobs, ts)
                assert not ref.diff(got), (p, ref.diff(got)[:4])
                assert ref_jobs.avail.tobytes() == tj.avail.tobytes()
            # the model follows the twin
            for k, j in enumerate(rows):
                jb = model.jobs[j]
                jb["avail"] = tj.avail[tj.node_off[k]:tj.node_off[k + 1]].copy()
                placed = int(want.placed[k])
                for i in range(tj.step_off[k], tj.step_off[k] + placed):
                    n0, n1 = want.node_off[i], want.node_off[i + 1]
                    model.running[int(srows[i])] = (j, want.alloc_node[n0:n1].copy(), want.alloc_res[n0:n1].copy())
                jb["queue"] = jb["queue"][placed:]
            seen[0] += res.n
            live = sorted(model.jobs)
            if live:
                want_avail = np.concatenate([model.jobs[j]["avail"] for j in live])
                assert s.step_jobs_avail(live).tobytes() == want_avail.tobytes(), p
        # an idle pass right after: nothing scheduled, avail unchanged
        live = sorted(model.jobs)
        before = s.step_jobs_avail(live)
        res, _ = s.steps_run()
        assert res.n == 0 and s.step_jobs_avail(live).tobytes() == before.tobytes()
    finally:
        s.close()
        twin.close()
    return seen


EMU_SEEDS = [11, 12, 13]


@pytest.mark.parametrize("seed", EMU_SEEDS)
def test_resident_steps_trajectory_emulated(steps_oracle, emu_lib, seed):
    case = synth.random_case(seed, n_jobs=120, n_nodes=24, n_running=6, ntpn_range=True,
                             one_type_per_name=bool(seed & 1))
    seen = _trajectory(emu_lib, case, seed, steps_oracle=steps_oracle)
    assert (seen > 0).all(), seen


@pytest.mark.gpu
@pytest.mark.parametrize("seed", EMU_SEEDS + [14, 15, 16])
def test_resident_steps_trajectory_gpu(steps_oracle, gpu_lib, seed):
    case = synth.random_case(seed, n_jobs=800, n_nodes=96, n_running=30, ntpn_range=True,
                             one_type_per_name=bool(seed & 1))
    seen = _trajectory(gpu_lib, case, seed, steps_oracle=steps_oracle)
    assert (seen > 0).all(), seen


@pytest.mark.gpu
def test_resident_steps_config2_digest(steps_oracle, gpu_lib):
    """The jobs GPU NodeSelect starts on config 2 become step jobs through step_jobs_start;
    one resident pass over the steps of step_case(2) reproduces the oracle's digest."""
    case = synth.config2()
    cfg, cl, rn, pd, now = case
    s = GpuScheduler(cfg, 0, gpu_lib)
    try:
        s.set_cluster(cl)
        s.upload(rn, pd)
        s.run(now)
        got = s.fetch(abi.Placements.for_pending(pd))
        cl2, jobs, steps = synth.step_case(2, lambda *c: got, base=case)
        started = np.flatnonzero(got.reason == abi.REASON_NONE)
        first = s.start(started)
        j0 = s.step_jobs_start(first + np.arange(len(started)))
        owner = np.repeat(np.arange(jobs.n_jobs), np.diff(jobs.step_off)) + j0
        s0 = s.steps_append(steps, owner)
        res, _ = s.steps_run()
        ref_jobs = jobs.copy()
        ref, _ = steps_oracle.schedule_steps(cl, ref_jobs, steps)
        out = res.expand(s0 + np.arange(steps.n), jobs.step_off, steps)
        assert ref.digest() == out.digest(), ref.diff(out)[:6]
        assert s.step_jobs_avail(j0 + np.arange(jobs.n_jobs)).tobytes() == ref_jobs.avail.tobytes()
        assert jobs.n_jobs > 1000 and 0 < res.n < steps.n
    finally:
        s.close()


# ---- isolation from NodeSelect ------------------------------------------------------------

def _node_select_ticks(lib, case, seed, with_steps, n_ticks=4):
    """Resident NodeSelect ticks (fetch, start, erase, keep_running); with_steps puts step
    calls between every fetch and start and after every start. Returns the fetched ticks."""
    cfg, cl, rn, pd, now = case
    rng = np.random.Generator(np.random.PCG64(seed))
    s = GpuScheduler(cfg, 0, lib)
    outs = []
    try:
        s.set_cluster(cl)
        s.pending_append(pd)
        s.running_append(rn)
        model = _Model()
        for t in range(n_ticks):
            s.keep_running()
            s.run(now)
            got = s.fetch(abi.Placements.for_pending(pd))
            outs.append(got)
            if with_steps and model.jobs:
                _arrive(s, model, cl, seed * 10 + t)
                res, _ = s.steps_run()
                if res.n:
                    s.steps_erase(res.step_row[:1])
            sel = rng.permutation(np.flatnonzero(got.reason == abi.REASON_NONE))[:20]
            first = s.start(sel)
            if with_steps:
                j0 = s.step_jobs_start(first + np.arange(len(sel)))
                st = abi.Running.started(pd, got, sel)
                for k in range(len(sel)):
                    a, b = st.alloc_off[k], st.alloc_off[k + 1]
                    model.add_job(j0 + k, st.alloc_node[a:b], st.alloc_res[a:b], st.alloc_res[a:b])
                _arrive(s, model, cl, seed * 10 + t + 5)
                s.steps_run()
            now += 600
            if t % 2:
                s.running_erase(rng.choice(s.running_rows(), 3, replace=False))
    finally:
        s.close()
    return outs


def test_step_calls_leave_node_select_alone(emu_lib):
    case = synth.random_case(21, n_jobs=100, n_nodes=20, n_parts=2, n_running=8, short=True)
    a = _node_select_ticks(emu_lib, case, 21, with_steps=False)
    b = _node_select_ticks(emu_lib, case, 21, with_steps=True)
    for t, (x, y) in enumerate(zip(a, b)):
        assert not x.diff(y), (t, x.diff(y)[:4])


def test_start_after_fetch_with_step_calls_between(emu_lib):
    """Step calls after a run's fetch leave it startable (the stage does not drop)."""
    case = synth.random_case(22, n_jobs=60, n_nodes=12, n_running=4)
    s, model, cl = _start_jobs(emu_lib, case, 22)
    cfg, _, rn, pd, now = case
    try:
        s.keep_running()
        s.run(now)
        got = s.fetch(abi.Placements.for_pending(pd))
        _arrive(s, model, cl, 5)
        s.steps_run()
        s.step_jobs_avail(sorted(model.jobs))
        rows = np.flatnonzero(got.reason == abi.REASON_NONE)
        assert len(rows)
        s.start(rows[:1])
    finally:
        s.close()


# ---- arguments ----------------------------------------------------------------------------

def _steps(rows, incl=None):
    n = len(rows)
    vt = np.zeros(n, abi.RES_VIEW)
    vt["cpu_raw"] = [int(r[4] * 256) for r in rows]
    kw = {}
    if incl is not None:
        off = np.zeros(n + 1, np.uint32)
        off[1:] = np.cumsum([len(x) for x in incl])
        kw = dict(incl_off=off, incl_nodes=np.array(sum(incl, []), np.uint32))
    return abi.Steps([r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows], [r[3] for r in rows],
                     np.zeros(n, abi.RES_VIEW), vt, **kw)


def _one_job(nodes, cores):
    return abi.StepJobs([0, len(nodes)], nodes, np.stack([synth.node_row(c, 8 * synth.GiB) for c in cores]), [0, 0])


def test_argument_checks(emu_lib):
    cl = synth.make_cluster([(6, synth.node_row(8, 64 * synth.GiB))])
    s = GpuScheduler(abi.Config(), 0, emu_lib)
    try:
        ok = _steps([(1, 1, 1, 1, 1)])
        # every call needs set_cluster
        for fn, args in ((s.step_jobs_append, (_one_job([0, 1], [4, 4]),)), (s.step_jobs_start, ([],)),
                         (s.steps_append, (ok, [0])), (s.steps_erase, ([],)), (s.step_jobs_erase, ([],)),
                         (s.steps_run, ()), (s.step_jobs_avail, ([],)), (s.step_jobs_reset, ())):
            assert _code(fn, *args) == abi.EINVAL, fn.__name__
        s.set_cluster(cl)
        # host rows: the node checks of schedule_steps, and no step_off
        for bad in (([0, 6], [4, 4]), ([1, 1], [4, 4]), ([2, 1], [4, 4])):
            assert _code(s.step_jobs_append, _one_job(*bad)) == abi.EINVAL
        c = _one_job([0, 1], [4, 4]).as_c()
        assert s._lib.crane_sched_step_jobs_append(s._h, c, None) == abi.EINVAL  # step_off given
        assert s.step_jobs_append(_one_job([0, 1], [4, 4])) == 0
        assert s.step_jobs_append(_one_job([2, 3], [4, 4])) == 1
        # steps: the answers of schedule_steps, then the job row
        for bad, code in (((0, 1, 1, 1, 1), abi.EINVAL), ((2, 1, 1, 1, 1), abi.EINVAL), ((1, 2, 3, 2, 1), abi.EINVAL),
                          ((128, 128, 1, 1, 1), abi.ENOSYS), ((1, 1, 0, 1, 1), abi.ENOSYS)):
            assert _code(s.steps_append, _steps([bad]), [0]) == code, bad
        assert _code(s.steps_append, _steps([(1, 1, 1, 1, 1)], incl=[[7]]), [0]) == abi.EINVAL
        neg = _steps([(1, 1, 1, 1, 1)])
        neg.req_task["cpu_raw"] = -1
        assert _code(s.steps_append, neg, [0]) == abi.EINVAL
        assert _code(s.steps_append, ok, [2]) == abi.EINVAL  # job row out of range
        assert s.steps_append(_steps([(1, 1, 1, 1, 1), (1, 1, 1, 1, 8), (1, 1, 1, 1, 1)]), [0, 1, 1]) == 0
        res, _ = s.steps_run()
        assert res.step_row.tolist() == [0]  # step 1 blocks step 2
        # erases: out of range, listed twice, already erased, job erased
        assert _code(s.steps_erase, [3]) == abi.EINVAL
        assert _code(s.steps_erase, [1, 1]) == abi.EINVAL
        s.steps_erase([0])
        assert _code(s.steps_erase, [0]) == abi.EINVAL
        assert _code(s.steps_erase, [2, 0]) == abi.EINVAL  # refused as a whole: row 2 is still pending
        s.steps_erase([1])  # the blocked head leaves: row 2 runs next pass
        assert s.steps_run()[0].step_row.tolist() == [2]
        assert _code(s.step_jobs_erase, [2]) == abi.EINVAL
        assert _code(s.step_jobs_erase, [0, 0]) == abi.EINVAL
        s.step_jobs_erase([1])
        assert _code(s.step_jobs_erase, [1]) == abi.EINVAL
        assert _code(s.steps_erase, [2]) == abi.EINVAL      # its job was erased
        assert _code(s.steps_append, ok, [1]) == abi.EINVAL  # erased job row
        assert _code(s.step_jobs_avail, [1]) == abi.EINVAL
        # the fetch is void after any later step call
        s.steps_run()
        s.step_jobs_avail([0])
        out = abi.StepResults.sized(0, 0, 0)
        assert s._lib.crane_sched_steps_fetch(s._h, out.as_c()) == abi.EINVAL
        # step_jobs_start: rows out of range, erased, listed twice, unordered allocations
        case = synth.random_case(23, n_jobs=40, n_nodes=12, n_running=6)
        cfg, cl2, rn, pd, now = case
        s.set_cluster(cl2)
        s.running_append(rn)
        assert _code(s.step_jobs_start, [rn.n]) == abi.EINVAL
        assert _code(s.step_jobs_start, [0, 0]) == abi.EINVAL
        multi = [j for j in range(rn.n) if rn.alloc_off[j + 1] - rn.alloc_off[j] > 1]
        assert multi
        rev = rn.take([multi[0]])
        rev = dataclasses.replace(rev, alloc_node=rev.alloc_node[::-1].copy(), alloc_res=rev.alloc_res[::-1].copy())
        r = s.running_append(rev)
        n_sj = 2
        assert _code(s.step_jobs_start, [0, r]) == abi.EINVAL
        assert s.step_jobs_start([0]) == n_sj  # the refused call appended nothing
        s.running_erase([1])
        assert _code(s.step_jobs_start, [1]) == abi.EINVAL
        s.step_jobs_reset()
        assert s.step_jobs_start([0]) == 0
    finally:
        s.close()
