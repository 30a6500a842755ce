"""Ticks at config-2 scale with held, not-yet-begun and dependent jobs: the gated
resident pending table against re-uploading the eligible rows.

A share of the submits carry AFTER_OK / AFTER_ANY lists on earlier jobs (AND and OR),
some are held and released later, some begin a few ticks ahead; running jobs end with
zero and non-zero exit codes and some pending jobs are cancelled. The daemon's own
bookkeeping (oracle/pygate.py) decides which jobs are eligible. Two handles follow the
same trajectory in one process, in alternating order:

  A (re-upload)  the only option without a gate: the pending table holds the eligible
                 rows in job-id order; rows that left are erased, newer eligible jobs are
                 appended, and any other change (a release, a begin time passing, a
                 dependency met) is a pending_reset + pending_append of every eligible row;
  B (gated)      every job is appended at submit with set_gate / pending_depend; ends,
                 cancels, holds and starts go through running_end, pending_cancel,
                 set_gate and start, and the run's k_gate leaves the gated rows out.

Both keep their running table on the device (start, running_erase / running_end,
keep_running). Per arm and tick: host -> device bytes of the job-table calls, host wall
time of the tick beyond the run's device time. Each arm's timed window holds every
library call the arm makes for that tick and the building of the tables those calls
upload:
  A: running_erase, pending_reset + pending_append or pending_erase + pending_append of
     the changed eligible rows, keep_running, run, fetch, start;
  B: the pending_cancel, set_gate (holds / releases) and submit calls (pending_append,
     set_gate, pending_depend) since its last tick, running_end, keep_running, run, fetch,
     start.
Outside both windows: the daemon model, A's eligibility filter and the diff of its
eligible set (the daemon's host work, left out in A's favour), the row bookkeeping of the
harness, the output buffers and the byte counts. The placements of A and B are
byte-compared on the eligible rows every tick. A separate profiled pass over B's last
tick reports the device time of k_gate and k_dep_fire (torch.profiler, CUDA activities).

    python tools/bench_gate.py [--ticks 8] [--jobs 100000] [--submit 5000] [--dt 300]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cranesched_b200 import abi, synth  # noqa: E402
from cranesched_b200.scheduler import GpuScheduler  # noqa: E402
from oracle import pygate  # noqa: E402
from tools.bench_ticks import card  # noqa: E402

ROW_EXTRA = 4 + 1  # alloc_off and tombstone flag of every appended row


def rows_bytes(p: abi.Pending) -> int:
    return sum(getattr(p, f).nbytes for f in p.__dataclass_fields__ if getattr(p, f) is not None) + ROW_EXTRA * p.n


class World:
    """The trajectory: jobs by id (= row of the drawn table), the daemon model, the
    running jobs (host table in row order for the running ids of both arms)."""

    def __init__(self, args):
        n_all = args.jobs + args.submit * args.ticks
        self.cfg, self.cl, _, self.pd, self.now = synth.config2(n_jobs=n_all, n_nodes=args.nodes, limit=args.jobs)
        self.rng = np.random.Generator(np.random.PCG64(args.seed))
        self.args = args
        self.dm = pygate.Daemon()
        self.n_sub = 0
        self.running = np.zeros(0, np.int64)  # jobs running, in running-row order of both arms
        self.run_end = np.zeros(0, np.int64)

    def draw_submits(self, n):
        """Gate and dependency lists of the next n jobs: (held, begin, is_or, deps) per job."""
        rng, now, dt = self.rng, self.now, self.args.dt
        out = []
        pend = [j for j in range(max(0, self.n_sub - 20000), self.n_sub) if self.dm.jobs[j].state == "pending"]
        for j in range(self.n_sub, self.n_sub + n):
            held = rng.random() < 0.02
            begin = now + dt * int(rng.integers(1, 4)) if rng.random() < 0.03 else pygate.PAST
            deps, orr = [], False
            if rng.random() < self.args.dep_frac and (pend or len(self.running)):
                pool = pend if (pend and rng.random() < 0.7) or not len(self.running) else list(self.running[-2000:])
                k = int(rng.integers(1, 4))
                for d in rng.choice(pool, min(k, len(pool)), replace=False):
                    deps.append((int(d), int(rng.choice([pygate.AFTER_OK, pygate.AFTER_ANY])), int(rng.choice([0, 0, 60]))))
                orr = bool(rng.random() < 0.3)
            out.append((j, held, begin, orr, deps))
            pend.append(j)
        return out

    def eligible(self):
        dm, now = self.dm, self.now
        return np.array([j for j in range(self.n_sub) if dm.jobs[j].state == "pending" and dm.reason(j, now) == 0],
                        np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=8)
    ap.add_argument("--jobs", type=int, default=100_000)
    ap.add_argument("--nodes", type=int, default=10_000)
    ap.add_argument("--submit", type=int, default=5000)
    ap.add_argument("--dep-frac", type=float, default=0.15, help="share of submits with a dependency list")
    ap.add_argument("--end-frac", type=float, default=0.05)
    ap.add_argument("--cancel-frac", type=float, default=0.002)
    ap.add_argument("--dt", type=int, default=300)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--profile-ticks", type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    print(f"card: {name}, power limit: {power}", flush=True)
    res = trajectory(args, profile=False)
    prof = trajectory(argparse.Namespace(**{**vars(args), "ticks": args.profile_ticks}), profile=True)
    print(json.dumps({"card": name, "power_limit": power, **res, "profiled_B": prof}), flush=True)


def trajectory(args, profile):
    w = World(args)
    pd, dm = w.pd, w.dm
    a, b = GpuScheduler(w.cfg, 0), GpuScheduler(w.cfg, 0)
    for s in (a, b):
        s.set_cluster(w.cl)
    a_jobs = np.zeros(0, np.int64)          # job of every row of A's pending table (tombstones included)
    a_live = np.zeros(0, np.int64)          # jobs with a live row in A
    a_row = {}                              # job -> pending row of A
    b_jobs = []                             # job of every row of B's pending table
    b_row = {}                              # job -> pending row of B
    b_run = {}                              # running job -> running row (the same in both arms)
    b_calls = []                            # B's calls since its last tick, run inside its next timed window
    rows, kern = [], {"k_gate": [], "k_dep_fire": []}

    def b_submit(batch):
        """Queues B's append + set_gate + depend of a batch of submits. Each queued call
        returns what it copied to the device, counted after the timed window."""
        jobs = np.array([x[0] for x in batch], np.int64)
        first = len(b_jobs)
        for k, j in enumerate(jobs):  # (harness bookkeeping: the rows the append will give)
            b_row[int(j)] = first + k
            b_jobs.append(int(j))
        kinds = [[abi.DEPENDEE_PENDING if d not in dm.jobs or dm.jobs[d].state == "pending" else abi.DEPENDEE_RUNNING
                  for d, _, _ in x[4]] for x in batch]

        def call():
            table = pd.take(jobs)
            assert b.pending_append(table) == first
            up = [table]
            g = [k for k, x in enumerate(batch) if x[1] or x[2] != pygate.PAST]
            if g:
                held = np.array([int(batch[k][1]) for k in g], np.uint8)
                begin = np.array([batch[k][2] for k in g], np.int64)
                b.pending_set_gate(first + np.array(g, np.uint32), held=held, begin_time=begin)
                up += [np.array(g, np.uint32), held, begin]
            lst, orr, ent = [], [], []
            for k, x in enumerate(batch):
                if x[4]:
                    lst.append(first + k)
                    orr.append(int(x[3]))
                    ent.append([(kd, b_row[d] if kd == abi.DEPENDEE_PENDING else b_run[d], ty, dl, 0)
                                for kd, (d, ty, dl) in zip(kinds[k], x[4])])
            if lst:
                deps = abi.Dependencies.from_lists(lst, orr, ent)
                b.pending_depend(deps)
                up.append(deps)
            return up
        b_calls.append(call)

    def model_submit(batch):
        for j, held, begin, o, deps in batch:
            dm.submit(j, deps, o, held, begin)
        w.n_sub += len(batch)

    # the first submits
    batch = w.draw_submits(args.jobs)
    b_submit(batch)
    model_submit(batch)
    for t in range(args.ticks):
        if profile and t == args.ticks - 1:  # the last tick of B, its queued calls included
            from torch.profiler import ProfilerActivity, profile as tprof
            w.prof = tprof(activities=[ProfilerActivity.CUDA])
            w.prof.__enter__()
        rec = {"tick": t + 1}
        ended = np.zeros(len(w.running), bool)
        if t:  # jobs that ended since the last tick
            ended = (w.run_end <= w.now) | (w.rng.random(len(w.running)) < args.end_frac)
        t_end = np.minimum(w.run_end[ended], w.now)
        codes = (w.rng.random(int(ended.sum())) < 0.2).astype(np.uint32)
        for j, te, c in zip(w.running[ended], t_end, codes):
            dm.end(int(j), int(te), int(c))
        ended_rows = np.array([b_run[int(j)] for j in w.running[ended]], np.uint32)
        # A's plan (the daemon's host filter, not timed): which rows leave, which arrive
        elig = w.eligible()
        gone = np.setdiff1d(a_live, elig)
        new = np.setdiff1d(elig, a_live)
        reset = len(a_jobs) == 0 or (len(new) and new.min() < a_jobs.max())
        a_next = elig.copy() if reset else np.concatenate([a_jobs, new])
        out_a = abi.Placements.for_pending(pd.take(a_next))
        out_b = abi.Placements.for_pending(pd.take(np.array(b_jobs, np.int64)))
        outs = {}
        for arm in (("A", "B") if t % 2 == 0 else ("B", "A")):
            s = a if arm == "A" else b
            up = []
            t0 = time.perf_counter()
            if arm == "A":
                s.running_erase(ended_rows)
                if reset:
                    s.pending_reset()
                    table = pd.take(elig)
                    if len(elig):
                        s.pending_append(table)
                    up.append(table)
                else:
                    if len(gone):
                        er = np.array([a_row[int(j)] for j in gone], np.uint32)
                        s.pending_erase(er)
                        up.append(er)
                    if len(new):
                        table = pd.take(new)
                        s.pending_append(table)
                        up.append(table)
                s.keep_running()
                s.run(w.now)
                out = s.fetch(out_a)
            else:
                for call in b_calls:
                    up += call()
                if len(ended_rows):
                    s.running_end(ended_rows, t_end, codes)
                    up += [t_end, codes]
                s.keep_running()
                s.run(w.now)
                out = s.fetch(out_b)
            started = np.flatnonzero(out.reason == abi.REASON_NONE)
            s.start(started)
            wall = (time.perf_counter() - t0) * 1e3
            outs[arm] = (out, started)
            h2d = up_bytes(up) + ended_rows.nbytes + (started.astype(np.uint32).nbytes + 4 if len(started) else 0)
            rec[arm] = {"host_ms": round(wall, 3), "h2d_bytes": int(h2d), "run_device_ms": round(s.timing()["total_ms"], 3)}
        b_calls.clear()
        a_jobs = a_next
        a_live = elig.copy()
        a_row = {int(j): k for k, j in enumerate(a_jobs)}
        bj = np.array(b_jobs, np.int64)
        # the placements of the eligible rows, byte for byte
        (oa, sa), (ob, sb) = outs["A"], outs["B"]
        sa, sb = a_jobs[sa], bj[sb]
        ia = np.array([a_row[int(j)] for j in elig], np.int64)
        ib = np.array([b_row[int(j)] for j in elig], np.int64)
        equal = np.array_equal(sa, sb)
        for f in ("reason", "start_time", "end_time", "n_alloc"):
            equal &= np.array_equal(getattr(oa, f)[ia], getattr(ob, f)[ib])
        equal &= np.array_equal(oa.priority[ia].view(np.uint64), ob.priority[ib].view(np.uint64))

        def alloc_rows(idx, jobs):  # allocation rows of the table's rows `idx`, in row order
            sel = np.zeros(len(jobs), bool)
            sel[idx] = True
            return np.repeat(sel, pd.node_num[jobs].astype(np.int64))

        ra_rows, rb_rows = alloc_rows(ia, a_jobs), alloc_rows(ib, bj)
        equal &= oa.alloc_res[ra_rows].tobytes() == ob.alloc_res[rb_rows].tobytes()
        equal &= np.array_equal(oa.alloc_node[ra_rows], ob.alloc_node[rb_rows])
        rec["equal"] = bool(equal)
        rec["eligible"] = int(len(elig))
        rec["gated"] = int(sum(dm.jobs[j].state == "pending" for j in range(w.n_sub)) - len(elig))
        rec["started"] = int(len(sa))
        # the model follows the starts
        keep = ~ended
        w.running, w.run_end = w.running[keep], w.run_end[keep]
        base = b.running_rows() - len(sb)
        for k, j in enumerate(sb):
            dm.start(int(j), w.now)
            b_run[int(j)] = base + k
        w.running = np.concatenate([w.running, sb])
        w.run_end = np.concatenate([w.run_end, ob.end_time[[b_row[int(j)] for j in sb]] if len(sb) else []]).astype(np.int64)
        a_live = np.setdiff1d(a_live, sa)
        rows.append(rec)
        print(json.dumps(rec), flush=True)
        if t == args.ticks - 1:
            break
        # until the next tick: cancels, holds / releases, submits. The model follows at once;
        # B's calls are queued for its next timed window, A sees them as a changed eligible set.
        w.now += args.dt
        pend = [j for j in b_row if dm.jobs[j].state == "pending"]
        if pend:
            cancel = w.rng.choice(pend, max(1, int(len(pend) * args.cancel_frac)), replace=False)
            c_rows, c_now = np.array([b_row[int(j)] for j in cancel], np.uint32), w.now
            b_calls.append(lambda r=c_rows, tc=c_now: (b.pending_cancel(r, tc), [r])[1])
            for j in cancel:
                dm.cancel(int(j), w.now)
            flip = [j for j in pend if dm.jobs[j].held] + list(w.rng.choice(pend, 20, replace=False))
            flip = [int(j) for j in dict.fromkeys(flip) if dm.jobs[int(j)].state == "pending"]
            held = np.array([int(not dm.jobs[j].held) for j in flip], np.uint8)
            f_rows = np.array([b_row[j] for j in flip], np.uint32)
            b_calls.append(lambda r=f_rows, hd=held: (b.pending_set_gate(r, held=hd), [r, hd])[1])
            for j, h in zip(flip, held):
                dm.set_held(j, bool(h))
        batch = w.draw_submits(args.submit)
        b_submit(batch)
        model_submit(batch)
    if profile and hasattr(w, "prof"):
        import torch
        torch.cuda.synchronize()
        w.prof.__exit__(None, None, None)
        for ev in w.prof.events():
            for k in kern:
                if k + "(" in ev.name:
                    kern[k].append(getattr(ev, "device_time_total", 0.0) / 1e3)
    for s in (a, b):
        s.close()
    later = rows[1:] or rows
    med = lambda arm, f: round(float(np.median([f(r[arm]) for r in later])), 3)  # noqa: E731
    summary = {arm: {"h2d_bytes": med(arm, lambda x: x["h2d_bytes"]),
                     "host_minus_run_ms": med(arm, lambda x: x["host_ms"] - x["run_device_ms"]),
                     "run_device_ms": med(arm, lambda x: x["run_device_ms"])} for arm in ("A", "B")}
    res = {"ticks": len(rows), "all_equal": all(r["equal"] for r in rows), "median_after_tick1": summary}
    if profile:
        res = {"kernel_ms": {k: [round(x, 4) for x in v] for k, v in kern.items()}, "all_equal": res["all_equal"]}
    return res


def up_bytes(up) -> int:
    """Host -> device bytes of what a tick's calls uploaded: pending tables (every column,
    alloc_off and the tombstone flag of each row), dependency lists, plain arrays."""
    n = 0
    for x in up:
        if isinstance(x, abi.Pending):
            n += rows_bytes(x)
        elif isinstance(x, abi.Dependencies):
            n += sum(getattr(x, f).nbytes for f in x.__dataclass_fields__)
        else:
            n += np.asarray(x).nbytes
    return n


if __name__ == "__main__":
    main()
