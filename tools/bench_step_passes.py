"""Steady-state passes of the step scheduler on one GPU: host tables per pass against the
resident step state.

The jobs config 2 starts now (GPU NodeSelect over 100k x 10k) become step jobs. Every pass
then has step arrivals (synth.step_pass_stream), a share of the scheduled steps ending
(their allocation goes back), and a few jobs ending and as many starting. Two arms on two
handles see the same events, alternating which goes first:
  A  crane_sched_schedule_steps with host tables of every job that has pending steps, as
     the adaptor does today;
  B  the resident tables: steps_append, steps_erase, step_jobs_erase / _append, steps_run
     and steps_fetch.
Each arm's timed window holds every library call of the pass and the building of the
tables those calls upload. Per pass: host-to-device and device-to-host bytes (computed from
the tables), host wall time beyond device time, device time per arm, and a check that the
scheduled steps and the avail rows are equal. Prints one JSON line with medians and
spread, and the card and its power limit read in the same run. Needs a CUDA device.

    python tools/bench_step_passes.py [--passes 12] [--warmup 2]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cranesched_b200 import abi, synth  # noqa: E402
from cranesched_b200.scheduler import GpuScheduler  # noqa: E402
from tools.bench_steps import _card  # noqa: E402

V, R = abi.RES_VIEW.itemsize, abi.RES_IN_NODE.itemsize


def _csr_take(off, idx):
    """(new offsets, entry indices) of CSR rows idx."""
    idx = np.asarray(idx, np.int64)
    n = (off[idx + 1] - off[idx]).astype(np.int64)
    new = np.zeros(len(idx) + 1, np.int64)
    new[1:] = np.cumsum(n)
    ent = np.repeat(off[idx].astype(np.int64) - new[:-1], n) + np.arange(int(new[-1]))
    return new, ent


class Steps:
    """Every step ever appended, one global table (row = step id = resident step row)."""

    def __init__(self):
        self.t = None

    def add(self, s):
        if self.t is None:
            self.t = s
            return
        t = self.t
        cat = lambda f: np.concatenate([getattr(t, f), getattr(s, f)])
        lists = {}
        for k in ("incl", "excl"):
            o, n = getattr(t, k + "_off"), getattr(t, k + "_nodes")
            lists[k + "_off"] = np.concatenate([o, o[-1] + getattr(s, k + "_off")[1:]])
            lists[k + "_nodes"] = np.concatenate([n, getattr(s, k + "_nodes")])
        self.t = abi.Steps(cat("node_num"), cat("ntasks"), cat("ntasks_per_node_min"), cat("ntasks_per_node_max"),
                           cat("req_node"), cat("req_task"), **lists)

    def take(self, idx):
        t = self.t
        kw = {}
        for k in ("incl", "excl"):
            off, ent = _csr_take(getattr(t, k + "_off"), idx)
            kw[k + "_off"], kw[k + "_nodes"] = off.astype(np.uint32), getattr(t, k + "_nodes")[ent]
        return abi.Steps(t.node_num[idx], t.ntasks[idx], t.ntasks_per_node_min[idx], t.ntasks_per_node_max[idx],
                         t.req_node[idx], t.req_task[idx], **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--p-job", type=float, default=0.1, help="share of jobs that get new steps in a pass")
    ap.add_argument("--end-share", type=float, default=0.4, help="share of running steps that end in a pass")
    ap.add_argument("--job-churn", type=int, default=50, help="jobs that end (and start) per pass")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_step_passes: no CUDA device")
    rng = np.random.Generator(np.random.PCG64(2))
    case = synth.config2()
    cfg, cl, rn, pd, now = case
    A, B = GpuScheduler(cfg, 0), GpuScheduler(cfg, 0)
    try:
        for s in (A, B):
            s.set_cluster(cl)
        B.upload(rn, pd)
        B.run(now)
        got = B.fetch(abi.Placements.for_pending(pd))
        started = np.flatnonzero(got.reason == abi.REASON_NONE)
        st = abi.Running.started(pd, got, started)
        # the model (the daemon's state): per job its node range in one avail pool
        n0 = len(started)
        job_off = st.alloc_off.astype(np.int64)          # grows as jobs start: node ranges in the pools
        job_node, alloc = st.alloc_node.copy(), st.alloc_res.copy()
        avail = alloc.copy()
        alive = np.ones(n0, bool)
        j0 = B.step_jobs_start(B.start(started) + np.arange(n0))
        assert j0 == 0
        queue = [[] for _ in range(n0)]   # pending step ids per job, FIFO
        running = {}                      # step id -> (job, pool positions of its nodes, res rows)
        dirty = set(range(n0))
        steps = Steps()
        n_steps = 0
        rows = {k: [] for k in ("A_e2e", "A_dev", "B_e2e", "B_dev", "A_h2d", "A_d2h", "B_h2d", "B_d2h", "sched", "visited")}
        for p in range(a.warmup + a.passes):
            # ---- the pass's events (drawn outside both windows) ----------------------------
            live = np.flatnonzero(alive)
            gone = rng.choice(live, min(a.job_churn, len(live)), replace=False)
            owner, new = synth.step_pass_stream(1000 + p, job_off, job_node, alloc, np.setdiff1d(live, gone), cl,
                                                p_job=a.p_job)
            ended = [q for q in running if rng.random() < a.end_share]
            came = rng.choice(np.flatnonzero(~alive) if (~alive).any() else live, len(gone))  # re-run as new jobs
            # ---- the model applies them (the daemon's own work, in neither window) --------
            for q in ended:
                j, pos, res = running.pop(q)
                for f in ("cpu_raw", "mem", "mem_sw"):
                    avail[f][pos] += res[f]
                avail["core"][pos] |= res["core"]
                avail["gres"][pos] |= res["gres"]
                dirty.add(j)
            for j in gone:
                alive[j] = False
                queue[j] = []
            running = {q: v for q, v in running.items() if alive[v[0]]}
            base = len(alive)
            new_off, ent = _csr_take(job_off, came)
            job_off = np.concatenate([job_off, job_off[-1] + new_off[1:]])
            job_node = np.concatenate([job_node, job_node[ent]])
            alloc = np.concatenate([alloc, alloc[ent]])
            avail = np.concatenate([avail, alloc[len(avail):]])
            alive = np.concatenate([alive, np.ones(len(came), bool)])
            queue += [[] for _ in came]
            dirty |= set(range(base, base + len(came)))
            for i, j in enumerate(owner):
                queue[j].append(n_steps + i)
                dirty.add(int(j))
            if new.n:
                steps.add(new)
            first_new = n_steps
            n_steps += new.n
            has = [j for j in range(len(alive)) if alive[j] and queue[j]]
            visited = [j for j in sorted(dirty) if alive[j] and queue[j]]
            dirty = set()
            # ---- arm A: host tables of every job with pending steps ------------------------
            def arm_a():
                t0 = time.perf_counter()
                jobs_idx = np.array(has, np.int64)
                noff, ent = _csr_take(job_off, jobs_idx)
                sids = np.concatenate([queue[j] for j in has]).astype(np.int64) if has else np.zeros(0, np.int64)
                soff = np.zeros(len(has) + 1, np.uint32)
                soff[1:] = np.cumsum([len(queue[j]) for j in has])
                jb = abi.StepJobs(noff.astype(np.uint32), job_node[ent], avail[ent], soff)
                ts = steps.take(sids)
                out, dev = A.schedule_steps(jb, ts)
                t1 = time.perf_counter()
                E, S, J = len(ent), ts.n, len(has)
                nr, tr = int(ts.node_num.astype(np.int64).sum()), int(ts.ntasks.astype(np.int64).sum())
                lists = int(ts.incl_off[-1]) + int(ts.excl_off[-1])
                h2d = 4 * (3 * J + E + 4 * S + 2 * (S + 1) + lists + 2 * (S + 1) + 2) + R * E + 2 * V * S
                d2h = 4 * J + S + nr * (8 + R) + tr * (4 + R) + R * E
                return (t1 - t0) * 1e3, dev, h2d, d2h, (jb, ts, sids, soff, ent, out)
            # ---- arm B: the resident tables -------------------------------------------------
            def arm_b():
                t0 = time.perf_counter()
                if ended:
                    B.steps_erase(ended)
                B.step_jobs_erase(gone)
                if len(came):
                    B.step_jobs_append(abi.StepJobs(new_off.astype(np.uint32), job_node[job_off[base]:],
                                                    alloc[job_off[base]:], np.zeros(len(came) + 1, np.uint32)))
                if new.n:
                    assert B.steps_append(new, owner) == first_new
                res, dev = B.steps_run()
                t1 = time.perf_counter()
                Sv = sum(len(queue[j]) for j in visited)
                lists = int(new.incl_off[-1]) + int(new.excl_off[-1]) if new.n else 0
                h2d = (4 * len(ended) * 3 + 4 * len(gone) + (4 * (len(came) + 1) + (4 + R) * int(new_off[-1]))
                       + new.n * (5 * 4 + 2 * V + 8) + 4 * lists + 4 * (len(visited) + Sv) + 8 * Sv)
                d2h = Sv + res.n * 0 + int(res.node_off[-1]) * (8 + R) + int(res.task_off[-1]) * (4 + R)
                return (t1 - t0) * 1e3, dev, h2d, d2h, res
            if p % 2:
                eb, db, hb, xb, res = arm_b()
                ea, da, ha, xa, ra = arm_a()
            else:
                ea, da, ha, xa, ra = arm_a()
                eb, db, hb, xb, res = arm_b()
            jb, ts, sids, soff, ent, out = ra
            # ---- equal results, then the model follows ------------------------------------
            exp = res.expand(sids, soff, ts)
            assert exp.digest() == out.digest(), f"pass {p}: resident results differ: {out.diff(exp)[:4]}"
            avail[ent] = jb.avail
            for k, j in enumerate(has):
                for i in range(int(soff[k]), int(soff[k]) + int(out.placed[k])):
                    a0, a1 = int(out.node_off[i]), int(out.node_off[i + 1])
                    nodes = job_node[job_off[j]:job_off[j + 1]]
                    pos = job_off[j] + np.searchsorted(nodes, out.alloc_node[a0:a1])
                    running[int(sids[i])] = (j, pos, out.alloc_res[a0:a1].copy())
                queue[j] = queue[j][int(out.placed[k]):]
            live = np.flatnonzero(alive)
            if p == a.warmup + a.passes - 1 or p == a.warmup:
                idx = np.concatenate([np.arange(job_off[j], job_off[j + 1]) for j in live])
                assert B.step_jobs_avail(live).tobytes() == avail[idx].tobytes(), f"pass {p}: avail differs"
            if p >= a.warmup:
                for k, v in zip(("A_e2e", "A_dev", "A_h2d", "A_d2h", "B_e2e", "B_dev", "B_h2d", "B_d2h"),
                                (ea, da, ha, xa, eb, db, hb, xb)):
                    rows[k].append(v)
                rows["sched"].append(res.n)
                rows["visited"].append(len(visited))
    finally:
        A.close()
        B.close()
    name, power = _card()
    med = lambda k: round(float(np.median(rows[k])), 4)
    spread = lambda k: [round(float(np.min(rows[k])), 4), round(float(np.max(rows[k])), 4)]
    host = {arm: [e - d for e, d in zip(rows[arm + "_e2e"], rows[arm + "_dev"])] for arm in "AB"}
    print(json.dumps({
        "metric": "step_passes", "gpu": name, "power_limit": power, "jobs": int(n0), "passes": a.passes,
        "steps_scheduled_median": med("sched"), "jobs_visited_median": med("visited"),
        "A_e2e_ms_median": med("A_e2e"), "A_e2e_ms_range": spread("A_e2e"),
        "B_e2e_ms_median": med("B_e2e"), "B_e2e_ms_range": spread("B_e2e"),
        "A_device_ms_median": med("A_dev"), "B_device_ms_median": med("B_dev"),
        "A_host_ms_beyond_device_median": round(float(np.median(host["A"])), 4),
        "B_host_ms_beyond_device_median": round(float(np.median(host["B"])), 4),
        "A_h2d_bytes_median": med("A_h2d"), "B_h2d_bytes_median": med("B_h2d"),
        "A_d2h_bytes_median": med("A_d2h"), "B_d2h_bytes_median": med("B_d2h"),
        "results_equal_every_pass": True,
    }))


if __name__ == "__main__":
    main()
