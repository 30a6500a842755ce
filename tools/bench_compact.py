"""Compaction of the resident tables at config-2 scale: crane_sched_compact against the host
re-send it replaces.

Two handles follow the same trajectory of bench_gate.py's traffic (its World: submits with
holds, begin times and AFTER_OK / AFTER_ANY lists, running jobs ending with zero and
non-zero exit codes, cancels, holds and releases, starts on the device) and never compact
until the tables carry several times more erased rows than live ones. Then, per round and
in alternating order:

  C (compact)   crane_sched_compact on handle 1;
  R (re-send)   on handle 2: pending_reset + pending_append of the live rows + set_gate +
                pending_depend with the model's state (one EVENT entry at ready_time for
                what was resolved, the open entries as they stand) + set_running with the
                live running rows.

Both leave the same rows in the same order, so the handles stay row for row alike. Per arm:
host wall time of the call(s), bytes in each direction (C: the maps; R: every table it
sends), device time (torch.profiler, CUDA activities, in a profiled round of its own).
Around the first round: keep_running + run + fetch time and fetch bytes, and one
pending_cancel's k_dep_fire, before and after. The placements of both handles are
compared byte for byte after every round, and a few ticks of traffic run between rounds.

    python tools/bench_compact.py [--warm-ticks 12] [--rounds 4] [--jobs 20000] [--submit 5000]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cranesched_b200 import abi  # noqa: E402
from cranesched_b200.scheduler import GpuScheduler  # noqa: E402
from oracle import pygate  # noqa: E402
from tools.bench_gate import World, up_bytes  # noqa: E402
from tools.bench_ticks import card  # noqa: E402


class Pair:
    """Two handles given the same calls; the row bookkeeping of both (they stay alike)."""

    def __init__(self, w: World):
        self.w = w
        self.h = [GpuScheduler(w.cfg, 0), GpuScheduler(w.cfg, 0)]
        for s in self.h:
            s.set_cluster(w.cl)
        self.jobs = np.zeros(0, np.int64)  # job of every pending row (tombstones included)
        self.row = {}                      # pending job -> row
        self.rjobs = np.zeros(0, np.int64)  # job of every running row
        self.rrow = {}                     # running job -> row
        self.host_run = None               # live running rows, row order (for the re-send)
        self.last = None

    def each(self, fn):
        return [fn(s) for s in self.h]

    def submit(self, batch):
        w, dm = self.w, self.w.dm
        jobs = np.array([x[0] for x in batch], np.int64)
        first = len(self.jobs)
        table = w.pd.take(jobs)
        self.each(lambda s: s.pending_append(table))
        self.jobs = np.concatenate([self.jobs, jobs])
        for k, j in enumerate(jobs):
            self.row[int(j)] = first + k
        g = [k for k, x in enumerate(batch) if x[1] or x[2] != pygate.PAST]
        if g:
            held = np.array([int(batch[k][1]) for k in g], np.uint8)
            begin = np.array([batch[k][2] for k in g], np.int64)
            self.each(lambda s: s.pending_set_gate(first + np.array(g, np.uint32), held=held, begin_time=begin))
        for j, held, begin, o, deps in batch:
            dm.submit(j, deps, o, held, begin)
        w.n_sub += len(batch)
        lst, orr, ent = [], [], []
        for k, x in enumerate(batch):
            if x[4]:
                lst.append(first + k)
                orr.append(int(x[3]))
                ent.append([self._entry(d, ty, dl) for d, ty, dl in x[4]])
        if lst:
            d = abi.Dependencies.from_lists(lst, orr, ent)
            self.each(lambda s: s.pending_depend(d))

    def _entry(self, d, ty, dl):
        if self.w.dm.jobs[d].state == "pending":
            return (abi.DEPENDEE_PENDING, self.row[d], ty, dl, 0)
        return (abi.DEPENDEE_RUNNING, self.rrow[d], ty, dl, 0)

    def tick(self, compare=True):
        """keep_running + run + fetch on both; the outputs must be equal. Returns handle 0's
        placements, its run + fetch wall ms and fetch bytes."""
        w = self.w
        outs, ms = [], []
        for s in self.h:
            out = abi.Placements.for_pending(w.pd.take(self.jobs))
            t0 = time.perf_counter()
            s.keep_running()
            s.run(w.now)
            s.fetch(out)
            ms.append((time.perf_counter() - t0) * 1e3)
            outs.append(out)
        if compare:
            d = outs[0].diff(outs[1])
            assert not d, "the handles' placements differ: " + "; ".join(d[:3])
        self.last = outs[0]
        return outs[0], ms[0], outs[0].nbytes()

    def advance(self, out, args):
        """Starts, then time passes: ends, cancels, holds / releases, submits."""
        w, dm, rng = self.w, self.w.dm, self.w.rng
        started = np.flatnonzero(out.reason == abi.REASON_NONE)
        first = self.each(lambda s: s.start(started))[0]
        run = abi.Running.started(w.pd.take(self.jobs), out, started)
        self.host_run = run if self.host_run is None else abi.Running.concat(self.host_run, run)
        for k, r in enumerate(started):
            j = int(self.jobs[r])
            dm.start(j, w.now)
            self.rrow[j] = first + k
            del self.row[j]
        self.rjobs = np.concatenate([self.rjobs, self.jobs[started]])
        w.now += args.dt
        live = np.array([j for j in self.rjobs if dm.jobs[int(j)].state == "running"], np.int64)
        assert len(live) == self.host_run.n
        ended = (self.host_run.end_time <= w.now) | (rng.random(len(live)) < args.end_frac)
        if ended.any():
            t_end = np.minimum(self.host_run.end_time[ended], w.now)
            codes = (rng.random(int(ended.sum())) < 0.2).astype(np.uint32)
            rows = np.array([self.rrow[int(j)] for j in live[ended]], np.uint32)
            self.each(lambda s: s.running_end(rows, t_end, codes))
            for j, te, c in zip(live[ended], t_end, codes):
                dm.end(int(j), int(te), int(c))
                del self.rrow[int(j)]
            self.host_run = self.host_run.take(np.flatnonzero(~ended))
        pend = [j for j in self.row if dm.jobs[j].state == "pending"]
        if pend:
            cancel = rng.choice(pend, max(1, int(len(pend) * args.cancel_frac)), replace=False)
            rows = np.array([self.row[int(j)] for j in cancel], np.uint32)
            self.each(lambda s: s.pending_cancel(rows, w.now))
            for j in cancel:
                dm.cancel(int(j), w.now)
                del self.row[int(j)]
            flip = [int(j) for j in rng.choice(pend, min(len(pend), 20), replace=False) if int(j) in self.row]
            held = np.array([int(not dm.jobs[j].held) for j in flip], np.uint8)
            if flip:
                self.each(lambda s: s.pending_set_gate(np.array([self.row[j] for j in flip], np.uint32), held=held))
            for j, h in zip(flip, held):
                dm.set_held(j, bool(h))
        w.running = np.array(list(self.rrow), np.int64)  # (the dependees draw_submits may pick)
        self.submit(w.draw_submits(args.submit))

    # ---- the two arms ----
    def compact(self, s):
        """C: returns (host ms, h2d bytes, d2h bytes, pending map, running map)."""
        t0 = time.perf_counter()
        pm, rm = s.compact()
        return (time.perf_counter() - t0) * 1e3, 0, pm.nbytes + rm.nbytes + 4, pm, rm

    def resend(self, s, live_jobs, new_row, new_rrow):
        """R: returns (host ms, h2d bytes, d2h bytes); the model's state is read inside the window."""
        dm, pd = self.w.dm, self.w.pd
        t0 = time.perf_counter()
        up = []
        s.pending_reset()
        table = pd.take(live_jobs)
        if len(live_jobs):
            s.pending_append(table)
        up.append(table)
        xs = [dm.jobs[int(j)] for j in live_jobs]
        g = np.flatnonzero([x.held or x.begin != pygate.PAST for x in xs])
        if len(g):
            held = np.array([int(xs[k].held) for k in g], np.uint8)
            begin = np.array([xs[k].begin for k in g], np.int64)
            s.pending_set_gate(g.astype(np.uint32), held=held, begin_time=begin)
            up += [g.astype(np.uint32), held, begin]
        rows, is_or, entries = [], [], []
        for k, x in enumerate(xs):
            dp = x.deps
            if not dp.is_or and not dp.deps and dp.ready == pygate.PAST:
                continue
            ent = []
            if dp.ready != (pygate.FUTURE if dp.is_or else pygate.PAST):
                ent.append((abi.DEPENDEE_EVENT, 0, pygate.AFTER_ANY, 0, dp.ready))
            for d, (ty, dl) in dp.deps.items():
                st = dm.jobs[d].state
                if st == "pending":
                    ent.append((abi.DEPENDEE_PENDING, new_row[d], ty, dl, 0))
                elif st == "running":
                    ent.append((abi.DEPENDEE_RUNNING, new_rrow[d], ty, dl, 0))
            rows.append(k)
            is_or.append(int(dp.is_or))
            entries.append(ent)
        s.set_running(self.host_run)
        if rows:
            d = abi.Dependencies.from_lists(rows, is_or, entries)
            s.pending_depend(d)
            up.append(d)
        h2d = up_bytes(up) + sum(getattr(self.host_run, f).nbytes for f in self.host_run.__dataclass_fields__
                                 if getattr(self.host_run, f) is not None)
        return (time.perf_counter() - t0) * 1e3, h2d, 0

    def round(self, order, profile=False):
        """One compaction of handle 0 and one re-send of handle 1, in `order`."""
        dm = self.w.dm
        keep = np.array([int(j) in self.row for j in self.jobs])
        live_jobs = self.jobs[keep]
        new_row = {int(j): k for k, j in enumerate(live_jobs)}
        rkeep = np.array([int(j) in self.rrow for j in self.rjobs], bool)
        new_rrow = {int(j): k for k, j in enumerate(self.rjobs[rkeep])}
        res, dev = {}, {}
        rows_before = (len(self.jobs), len(self.rjobs))
        for arm in order:
            if profile:
                from torch.profiler import ProfilerActivity, profile as tprof
                p = tprof(activities=[ProfilerActivity.CUDA])
                p.__enter__()
            if arm == "C":
                ms, h2d, d2h, pm, rm = self.compact(self.h[0])
            else:
                ms, h2d, d2h = self.resend(self.h[1], live_jobs, new_row, new_rrow)
            if profile:
                import torch
                torch.cuda.synchronize()
                p.__exit__(None, None, None)
                dev[arm] = round(sum(getattr(e, "device_time_total", 0.0) for e in p.events()
                                     if str(getattr(e, "device_type", "")).endswith("CUDA")) / 1e3, 4)
            res[arm] = {"host_ms": round(ms, 3), "h2d_bytes": int(h2d), "d2h_bytes": int(d2h)}
        assert np.array_equal(np.flatnonzero(pm != abi.ROW_NONE), np.flatnonzero(keep))
        assert np.array_equal(np.flatnonzero(rm != abi.ROW_NONE), np.flatnonzero(rkeep))
        self.jobs, self.row = live_jobs, new_row
        self.rjobs, self.rrow = self.rjobs[rkeep], new_rrow
        assert all(dm.jobs[j].state == "pending" for j in self.row)
        return {"rows_before": rows_before, "rows_after": (len(self.jobs), len(self.rjobs)), **res,
                **({"device_ms": dev} if profile else {})}

    def dep_fire_ms(self):
        """One pending_cancel of one live row on both handles; k_dep_fire's device ms on handle 0."""
        from torch.profiler import ProfilerActivity, profile as tprof
        import torch
        dm, w = self.w.dm, self.w
        j = next(iter(self.row))
        r = np.array([self.row[j]], np.uint32)
        with tprof(activities=[ProfilerActivity.CUDA]) as p:
            self.h[0].pending_cancel(r, w.now)
            torch.cuda.synchronize()
        self.h[1].pending_cancel(r, w.now)
        dm.cancel(j, w.now)
        del self.row[j]
        return round(sum(e.device_time_total for e in p.events() if "k_dep_fire(" in e.name) / 1e3, 4)

    def close(self):
        self.each(lambda s: s.close())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warm-ticks", type=int, default=12, help="ticks before the first compaction")
    ap.add_argument("--between", type=int, default=2, help="ticks between rounds")
    ap.add_argument("--rounds", type=int, default=4, help="rounds; the last one is profiled")
    ap.add_argument("--jobs", type=int, default=20_000)
    ap.add_argument("--nodes", type=int, default=10_000)
    ap.add_argument("--submit", type=int, default=5000)
    ap.add_argument("--dep-frac", type=float, default=0.15)
    ap.add_argument("--end-frac", type=float, default=0.2)
    ap.add_argument("--cancel-frac", type=float, default=0.1)
    ap.add_argument("--dt", type=int, default=300)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    args.ticks = args.warm_ticks + args.rounds * (args.between + 1) + 2
    name, power = card()
    print(f"card: {name}, power limit: {power}", flush=True)
    w = World(args)
    pr = Pair(w)
    pr.submit(w.draw_submits(args.jobs))
    for _ in range(args.warm_ticks):
        out, _, _ = pr.tick()
        pr.advance(out, args)
    live = (len(pr.row), len(pr.rrow))
    print(json.dumps({"before_compaction": {"pending_rows": len(pr.jobs), "pending_live": live[0],
                                            "running_rows": len(pr.rjobs), "running_live": live[1]}}), flush=True)
    # run + fetch and k_dep_fire before, one compaction round, the same after
    before = [pr.tick()[1:] for _ in range(3)][1:]
    fire_before = pr.dep_fire_ms()
    rounds = [pr.round(("C", "R"))]
    after = [pr.tick()[1:] for _ in range(3)][1:]
    fire_after = pr.dep_fire_ms()
    rf = {"before": {"run_fetch_ms": [round(x[0], 3) for x in before], "fetch_bytes": before[-1][1],
                     "k_dep_fire_ms": fire_before},
          "after": {"run_fetch_ms": [round(x[0], 3) for x in after], "fetch_bytes": after[-1][1],
                    "k_dep_fire_ms": fire_after}}
    print(json.dumps({"run_fetch": rf}), flush=True)
    for k in range(1, args.rounds):
        for _ in range(args.between):
            out, _, _ = pr.tick()
            pr.advance(out, args)
        rounds.append(pr.round(("C", "R") if k % 2 == 0 else ("R", "C"), profile=k == args.rounds - 1))
        pr.tick()  # the placements of both handles, byte for byte
        print(json.dumps(rounds[-1]), flush=True)
    pr.close()
    med = lambda arm, f: round(float(np.median([r[arm][f] for r in rounds[:-1] if arm in r])), 3)  # noqa: E731
    print(json.dumps({"card": name, "power_limit": power, "all_equal": True, "run_fetch": rf,
                      "median_unprofiled": {arm: {f: med(arm, f) for f in ("host_ms", "h2d_bytes", "d2h_bytes")}
                                            for arm in ("C", "R")},
                      "profiled_round": rounds[-1]}), flush=True)


if __name__ == "__main__":
    main()
