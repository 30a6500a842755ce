"""Steady-state NodeSelect ticks at config-2 scale, with the running table rebuilt on
the host every tick against the running table kept on the device.

Tick 1 starts from an empty running table (config 2: 100 000 jobs on 10 000 nodes).
Every later tick: the running jobs past their end time and a share of the others end,
new jobs are submitted, the tick runs and every job it starts now moves into the
running table. Two handles follow the same trajectory in one process, in alternating
order:

  A (host table)   rebuild a host crane_running_t of the live jobs (the flattening of
                   RnJobInScheduler), set_running, run, fetch, pending_erase of the
                   started rows and their host rows built from the placements;
  B (resident)     running_erase, keep_running, run, fetch, start.

Per arm and tick: host wall time from the first running-table call until the
started jobs have moved (fetch and start both end with a synchronise), keep_running's
device time (B), and the bytes the running-table calls copy host -> device (the
submits are the same in both arms and are left out). The
placements of A and B are byte-compared on every tick.

    python tools/bench_ticks.py [--ticks 8] [--submit 5000] [--end-frac 0.05] [--dt 300]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cranesched_b200 import abi, synth  # noqa: E402
from cranesched_b200.scheduler import GpuScheduler  # noqa: E402

# what the running-table calls copy host -> device
JOB_BYTES = 48 + 4 + 4 + 1                 # A: the columns, alloc_off, reservation, tombstone flag, per job
ENTRY_BYTES = 4 + abi.RES_IN_NODE.itemsize  # A: alloc_node + alloc_res, per (job, node)
START_BYTES = 4 + 4 + 1                     # B: pending row, alloc_off, tombstone flag, per started job


def card():
    try:
        import torch
        name = torch.cuda.get_device_name(0)
    except Exception:
        name = "unknown"
    try:
        o = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        o = "unknown"
    return name, o


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=8)
    ap.add_argument("--jobs", type=int, default=100_000)
    ap.add_argument("--nodes", type=int, default=10_000)
    ap.add_argument("--submit", type=int, default=5000, help="jobs submitted before every tick after the first")
    ap.add_argument("--end-frac", type=float, default=0.05, help="share of the running jobs not yet due that end")
    ap.add_argument("--dt", type=int, default=300, help="seconds between ticks")
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()

    cfg, cl, _, pd, now = synth.config2(n_jobs=args.jobs + args.submit * (args.ticks - 1), n_nodes=args.nodes,
                                        limit=args.jobs)
    rng = np.random.Generator(np.random.PCG64(args.seed))
    name, power = card()
    print(f"card: {name}, power limit: {power}")

    arms = {"A": GpuScheduler(cfg, 0), "B": GpuScheduler(cfg, 0)}
    for s in arms.values():
        s.set_cluster(cl)
    n_sub = args.jobs
    for s in arms.values():
        s.pending_append(pd.take(np.arange(n_sub)))
    host = abi.Running.empty()  # the live jobs, in row order (A's host table)
    ids = np.zeros(0, np.int64)  # their rows in B's resident table
    rows = []
    for t in range(args.ticks):
        if t:
            now += args.dt
        ended = (host.end_time <= now) | (rng.random(host.n) < args.end_frac)
        rec = {"tick": t + 1, "ended": int(ended.sum())}
        outs = {}
        for arm in (("A", "B") if t % 2 == 0 else ("B", "A")):
            s = arms[arm]
            out = abi.Placements.for_pending(pd.take(np.arange(n_sub)))
            t0 = time.perf_counter()
            if arm == "A":
                table = host.take(np.flatnonzero(~ended))
                s.set_running(table)
                s.run(now)
                s.fetch(out)
                started = np.flatnonzero(out.reason == abi.REASON_NONE)
                if len(started):
                    s.pending_erase(started)
                host_next = abi.Running.concat(table, abi.Running.started(pd, out, started))
                h2d = table.n * JOB_BYTES + 4 + len(table.alloc_node) * ENTRY_BYTES + 4 * len(started)
                kr_ms = None
            else:
                s.running_erase(ids[ended])
                kr_ms = s.keep_running()
                s.run(now)
                s.fetch(out)
                started = np.flatnonzero(out.reason == abi.REASON_NONE)
                first = s.start(started)
                ids_next = np.concatenate([ids[~ended], first + np.arange(len(started))])
                h2d = 4 * int(ended.sum()) + (START_BYTES * len(started) + 4 if len(started) else 0)
            wall = (time.perf_counter() - t0) * 1e3
            rec[arm] = {"host_ms": round(wall, 3), "h2d_bytes": int(h2d), "run_device_ms": round(s.timing()["total_ms"], 3)}
            if kr_ms is not None:
                rec[arm]["keep_running_ms"] = round(kr_ms, 4)
            outs[arm] = out
        host, ids = host_next, ids_next
        d = outs["A"].diff(outs["B"])
        rec["equal"] = not d
        rec["started"] = int(len(started))
        rec["running"] = int(host.n)
        print(json.dumps(rec), flush=True)
        if d:
            print("A and B differ:\n" + "\n".join(d[:8]))
        rows.append(rec)
        # submits of the next tick (not timed: the same in both arms)
        if t + 1 < args.ticks:
            for s in arms.values():
                s.pending_append(pd.take(np.arange(n_sub, n_sub + args.submit)))
            n_sub += args.submit
    for s in arms.values():
        s.close()
    # the run's device time differs from tick to tick with the queue: the host wall time
    # beyond it is what the running-table path costs
    later = rows[1:] or rows
    med = lambda arm, f: round(float(np.median([f(r[arm]) for r in later])), 3)
    summary = {arm: {"host_ms": med(arm, lambda x: x["host_ms"]),
                     "host_minus_run_ms": med(arm, lambda x: x["host_ms"] - x["run_device_ms"]),
                     "h2d_bytes": med(arm, lambda x: x["h2d_bytes"])} for arm in ("A", "B")}
    summary["B"]["keep_running_ms"] = med("B", lambda x: x["keep_running_ms"])
    print(json.dumps({"card": name, "power_limit": power, "ticks": len(rows),
                      "all_equal": all(r["equal"] for r in rows), "median_after_tick1": summary}))


if __name__ == "__main__":
    main()
