"""The running table kept resident on the device across ticks (crane_sched_start /
_running_append / _running_erase / _keep_running).

Ticks with submits, starts (a random subset of the start-now rows in a random order,
as if the rest were refused), jobs started elsewhere (running_append), ended and
cancelled jobs (running_erase) and a set_cluster that drains a node part-way:
  - every output column of a handle that keeps its running table on the device is
    byte-identical to a second handle given set_running with the host table of the
    live rows in row order;
  - the trajectory equals the oracle's NodeSelect over host tables kept with
    abi.Running.started (priority compared as bits).
Both through the kernel-emulation library here and on the GPU in the `gpu`-marked
twins; the argument codes on the emulator."""
import dataclasses

import numpy as np
import pytest

from cranesched_b200 import abi, synth
from cranesched_b200.scheduler import CraneSchedError, GpuScheduler


def _code(fn, *args):
    try:
        fn(*args)
        return 0
    except CraneSchedError as e:
        return e.code


def _drained(cl, host, rng):
    """The cluster with one more node drained: a node that holds a live allocation if any."""
    busy = np.unique(host.alloc_node)
    busy = busy[(cl.alive[busy] == 1) & (cl.drain[busy] == 0)]
    node = int(rng.choice(busy)) if len(busy) else 0
    drain = cl.drain.copy()
    drain[node] = 1
    return dataclasses.replace(cl, drain=drain)


def _ticks(lib, case, resv, seed, n_ticks=6, dt=900, oracle=None, twin=True, drain_at=3, elsewhere_at=2):
    """Runs the ticks; returns the number of (start-now, rows started on the device,
    running rows erased, live rows past their end time) seen over all ticks."""
    cfg, cl, rn0, pd, now = case
    rng = np.random.Generator(np.random.PCG64(seed))
    cuts = sorted({pd.n // 2, (3 * pd.n) // 4, pd.n})
    b = GpuScheduler(cfg, 0, lib)
    a = GpuScheduler(cfg, 0, lib) if twin else None
    both = [s for s in (b, a) if s is not None]
    seen = np.zeros(4, np.int64)
    try:
        for s in both:
            s.set_cluster(cl)
            if resv is not None:
                s.set_reservations(resv)
        n_sub = cuts[0]
        for s in both:
            assert s.pending_append(pd.take(np.arange(n_sub))) == 0
        pd_alive = np.zeros(pd.n, bool)
        pd_alive[:n_sub] = True
        # running jobs known at start (recovery): two appends
        k = rn0.n // 2
        assert b.running_append(rn0.take(np.arange(k))) == 0
        assert b.running_append(rn0.take(np.arange(k, rn0.n))) == k
        host, ids = rn0, np.arange(rn0.n)  # live rows in row order, and their row indices
        for t in range(n_ticks):
            if t == drain_at:
                cl = _drained(cl, host, rng)
                for s in both:
                    s.set_cluster(cl)
                    if resv is not None:
                        s.set_reservations(resv)
            b.keep_running()
            b.run(now)
            got = b.fetch(abi.Placements.for_pending(pd.take(np.arange(n_sub))))
            if a is not None:
                a.set_running(host)
                a.run(now)
                want = a.fetch(abi.Placements.for_pending(pd.take(np.arange(n_sub))))
                d = want.diff(got)
                assert not d, f"tick {t}: resident running table differs from set_running:\n" + "\n".join(d[:8])
            if oracle is not None:
                alive = np.flatnonzero(pd_alive)
                ref, _, _ = oracle.node_select(cfg, cl, host, pd.take(alive), now, resv=resv)
                assert (got.reason[~pd_alive[:n_sub]] == abi.REASON_ERASED).all()
                for f in ("reason", "start_time", "end_time", "n_alloc"):
                    assert np.array_equal(getattr(ref, f), getattr(got, f)[alive]), (t, f)
                assert np.array_equal(ref.priority.view(np.uint64), got.priority[alive].view(np.uint64)), t
                rows = np.isin(np.repeat(np.arange(n_sub), pd.node_num[:n_sub]), alive)
                assert np.array_equal(ref.alloc_node, got.alloc_node[rows]), t
                assert np.array_equal(ref.alloc_ntasks, got.alloc_ntasks[rows]), t
                assert ref.alloc_res.tobytes() == got.alloc_res[rows].tobytes(), t
            # the commit loop starts a random subset of the start-now rows, in a random order
            now_rows = np.flatnonzero(got.reason == abi.REASON_NONE)
            sel = rng.permutation(now_rows[rng.random(len(now_rows)) < 0.8])
            seen[0] += len(now_rows)
            other = np.zeros(0, np.int64)
            if t == elsewhere_at and len(sel) > 2:  # some of them are started by another path
                other, sel = np.sort(sel[: len(sel) // 3]), sel[len(sel) // 3:]
            first = b.start(sel)
            assert b.running_rows() == first + len(sel)
            host = abi.Running.concat(host, abi.Running.started(pd, got, sel))
            ids = np.concatenate([ids, first + np.arange(len(sel))])
            seen[1] += len(sel)
            if len(other):
                b.pending_erase(other)
                assert b.running_append(abi.Running.started(pd, got, other)) == first + len(sel)
                host = abi.Running.concat(host, abi.Running.started(pd, got, other))
                ids = np.concatenate([ids, first + len(sel) + np.arange(len(other))])
            gone = np.concatenate([sel, other]).astype(np.int64)
            if a is not None and len(gone):
                a.pending_erase(gone)
            pd_alive[gone] = False
            # jobs end: most of those past their end time, and a few cancelled ones; the
            # rest of the overdue ones stay and meet the end >= now + 1 clamp
            now += dt
            over = host.end_time < now + 1
            ended = (over & (rng.random(host.n) < 0.6)) | (rng.random(host.n) < 0.05)
            seen[2] += int(ended.sum())
            seen[3] += int((over & ~ended).sum())
            b.running_erase(ids[ended])
            host, ids = host.take(np.flatnonzero(~ended)), ids[~ended]
            # cancelled pending jobs, then new submits
            live = np.flatnonzero(pd_alive)
            if len(live) > 4:
                gone = rng.choice(live, len(live) // 20, replace=False)
                for s in both:
                    s.pending_erase(gone)
                pd_alive[gone] = False
            nxt = next((c for c in cuts if c > n_sub), n_sub)
            if nxt > n_sub:
                for s in both:
                    assert s.pending_append(pd.take(np.arange(n_sub, nxt))) == n_sub
                pd_alive[n_sub:nxt] = True
                n_sub = nxt
        # compaction: set_running with the live rows gives the same tick as the tombstoned table
        b.keep_running()
        b.run(now)
        before = b.fetch(abi.Placements.for_pending(pd.take(np.arange(n_sub))))
        b.set_running(host)
        assert b.running_rows() == host.n
        b.run(now)
        after = b.fetch(abi.Placements.for_pending(pd.take(np.arange(n_sub))))
        assert not before.diff(after)
    finally:
        for s in both:
            s.close()
    return seen


def _case(seed, resv=False, overlap=False, **kw):
    case = synth.random_case(seed, **kw)
    if overlap:
        case = synth.overlap_partitions(case, seed, frac=0.4)
    r = None
    if resv:
        r, pd, rn = synth.random_reservations(seed, case, n_resv=4)
        case = (case[0], case[1], rn, pd, case[4])
    return case, r


EMU_CASES = {
    "plain": dict(seed=81, n_jobs=90, n_nodes=20, n_parts=2, n_running=12, short=True),
    "reservations": dict(seed=82, n_jobs=90, n_nodes=24, n_parts=2, n_running=10, short=True, resv=True),
    "overlap": dict(seed=83, n_jobs=90, n_nodes=24, n_parts=3, n_running=10, short=True, overlap=True, resv=True),
    "fifo": dict(seed=84, n_jobs=90, n_nodes=20, n_parts=2, n_running=12, short=True, fifo=True, limit=50),
}


@pytest.mark.parametrize("name", sorted(EMU_CASES))
def test_resident_running_equals_set_running_emulated(emu_lib, name):
    kw = dict(EMU_CASES[name])
    case, resv = _case(**kw)
    seen = _ticks(emu_lib, case, resv, kw["seed"], n_ticks=5)
    assert seen[1] > 0 and seen[2] > 0


@pytest.mark.parametrize("name", ["reservations", "overlap"])
def test_resident_running_trajectory_oracle_emulated(oracle, emu_lib, name):
    kw = dict(EMU_CASES[name])
    case, resv = _case(**kw)
    seen = _ticks(emu_lib, case, resv, kw["seed"] + 100, n_ticks=5, oracle=oracle, twin=False)
    assert seen[1] > 0 and seen[2] > 0 and seen[3] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(90, 96))
def test_resident_running_equals_set_running_gpu(gpu_lib, seed):
    case, resv = _case(seed, n_jobs=1500, n_nodes=150, n_parts=1 + seed % 4, n_running=80, short=bool(seed % 2),
                       fifo=seed % 3 == 0, limit=900 if seed % 2 else None, resv=seed % 3 != 2,
                       overlap=seed % 2 == 0, ntpn_range=seed % 3 == 1)
    seen = _ticks(gpu_lib, case, resv, seed, n_ticks=6)
    assert seen[1] > 0 and seen[2] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("seed,kw", [(97, dict(n_jobs=4000, n_nodes=400, n_parts=3, n_running=200, resv=True)),
                                     (98, dict(n_jobs=1200, n_nodes=120, n_parts=3, n_running=60, overlap=True,
                                               resv=True, ntpn_range=True))])
def test_resident_running_trajectory_oracle_gpu(oracle, gpu_lib, seed, kw):
    case, resv = _case(seed, short=True, **kw)
    seen = _ticks(gpu_lib, case, resv, seed, n_ticks=6, oracle=oracle, twin=False)
    assert seen[1] > 0 and seen[2] > 0 and seen[3] > 0


# ---- arguments --------------------------------------------------------------------------------

def _ran(emu_lib, case, resv=None):
    cfg, cl, rn, pd, now = case
    s = GpuScheduler(cfg, 0, emu_lib)
    s.set_cluster(cl)
    if resv is not None:
        s.set_reservations(resv)
    s.upload(rn, pd)
    s.run(now)
    return s, s.fetch(abi.Placements.for_pending(pd))


def test_start_refuses_rows_without_a_start_now_placement(emu_lib):
    """Every kind of row that does not start now: "Priority" (batch limit), "Resource",
    a backfill reservation, "Partition Not Found", "Reservation Not Found", a QoS refusal,
    an erased row; also rows out of range and listed twice. A refused start changes
    nothing: the run can still be fetched."""
    case, resv = _case(86, n_jobs=120, n_nodes=16, n_parts=2, n_running=10, limit=70, resv=True)
    cfg, cl, rn, pd, now = case
    s, out = _ran(emu_lib, case, resv)
    try:
        kinds = {}
        for code in (abi.REASON_PRIORITY, abi.REASON_RESOURCE, abi.REASON_PART_NOT_FOUND, abi.REASON_RESV_NOT_FOUND):
            rows = np.flatnonzero(out.reason == code)
            assert len(rows), code
            kinds[code] = int(rows[0])
        backfill = np.flatnonzero((out.reason != abi.REASON_NONE) & (out.n_alloc > 0))
        assert len(backfill)
        kinds["backfill"] = int(backfill[0])
        ok = np.flatnonzero(out.reason == abi.REASON_NONE)
        assert len(ok) >= 3
        for kind, row in kinds.items():
            assert _code(s.start, [int(ok[0]), row]) == abi.EINVAL, kind
        assert _code(s.start, [pd.n]) == abi.EINVAL
        assert _code(s.start, [int(ok[0]), int(ok[1]), int(ok[0])]) == abi.EINVAL
        again = s.fetch(abi.Placements.for_pending(pd))  # nothing moved
        assert not out.diff(again) and s.running_rows() == rn.n
        # QoS-refused rows (crane_sched_qos_filter rewrites the reasons on the device)
        table = synth.random_qos(86, cl, pd, tight=0.3)
        reason = out.reason.copy()
        s.qos_filter(table, reason)
        refused = np.flatnonzero((out.reason == abi.REASON_NONE) & (reason != abi.REASON_NONE))
        passed = np.flatnonzero(reason == abi.REASON_NONE)
        assert len(refused) and len(passed)
        assert _code(s.start, [int(refused[0])]) == abi.EINVAL
        assert s.start(passed[:1]) == rn.n
        # the started row is erased from the pending table, and the run is void
        assert _code(s.fetch, abi.Placements.for_pending(pd)) == abi.EINVAL
        assert _code(s.run, now) == abi.EINVAL  # the running table must follow
        assert _code(s.start, passed[1:2]) == abi.EINVAL  # no completed run
        s.keep_running()
        s.run(now)
        out2 = s.fetch(abi.Placements.for_pending(pd))
        assert out2.reason[passed[0]] == abi.REASON_ERASED
        assert _code(s.start, passed[:1]) == abi.EINVAL  # erased
    finally:
        s.close()


def test_start_before_a_run_and_on_a_sharded_handle(emu_lib):
    case = synth.random_case(86, n_jobs=40, n_nodes=12, n_parts=2, n_running=4)
    cfg, cl, rn, pd, now = case
    s = GpuScheduler(cfg, 0, emu_lib)
    try:
        assert _code(s.keep_running) == abi.EINVAL  # before any cluster
        assert _code(s.running_append, rn) == abi.EINVAL
        s.set_cluster(cl)
        s.upload(rn, pd)
        assert _code(s.start, [0]) == abi.EINVAL  # before a run
        s.run(now)
        out = s.fetch(abi.Placements.for_pending(pd))
        s.set_shard(0, 2, np.zeros(cl.n_partitions, np.uint32))
        s.upload(rn, pd)
        s.run(now)
        assert _code(s.start, np.flatnonzero(out.reason == 0)[:1]) == abi.ENOSYS
    finally:
        s.close()


def test_running_rows_and_node_range(emu_lib):
    """running_erase checks its rows; appended rows are checked as set_running checks
    them; keep_running refuses live rows on nodes a smaller cluster does not have, and
    ignores erased ones."""
    case = synth.random_case(87, n_jobs=40, n_nodes=12, n_parts=1, n_running=6)
    cfg, cl, rn, pd, now = case
    s = GpuScheduler(cfg, 0, emu_lib)
    try:
        s.set_cluster(cl)
        s.pending_append(pd)
        assert s.running_append(rn) == 0
        assert _code(s.running_erase, [rn.n]) == abi.EINVAL
        bad = dataclasses.replace(rn, alloc_node=np.full_like(rn.alloc_node, cl.n_nodes))
        assert _code(s.running_append, bad) == abi.EINVAL
        assert s.running_rows() == rn.n
        s.keep_running()
        s.run(now)
        # a cluster of the first m nodes: the rows on nodes >= m must go first
        m = int(rn.alloc_node.min()) + 1
        small = abi.Cluster(cl.res_total[:m], cl.alive[:m], cl.drain[:m], np.array([0, m], np.uint32),
                            np.arange(m, dtype=np.uint32), cl.n_gres_entries, cl.gres_entry_name)
        pd_small = dataclasses.replace(pd.take(np.arange(pd.n)), incl_off=None, incl_nodes=None, excl_off=None,
                                       excl_nodes=None)
        s.set_cluster(small)
        s.pending_reset()
        s.pending_append(pd_small)
        assert _code(s.keep_running) == abi.EINVAL
        far = [j for j in range(rn.n) if (rn.alloc_node[rn.alloc_off[j]:rn.alloc_off[j + 1]] >= m).any()]
        s.running_erase(far)
        s.keep_running()
        s.run(now)
        got = s.fetch(abi.Placements.for_pending(pd_small))
        keep = np.setdiff1d(np.arange(rn.n), far)
        t = GpuScheduler(cfg, 0, emu_lib)
        try:
            t.set_cluster(small)
            want = t.node_select(now, rn.take(keep), pd_small)
        finally:
            t.close()
        assert not want.diff(got)
    finally:
        s.close()
