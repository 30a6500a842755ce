"""Compaction of the resident step tables at config-2 scale (crane_sched_steps_compact).

The jobs config 2 starts now (GPU NodeSelect over 100k x 10k) become step jobs on two
handles. Both then see bench_step_passes.py's traffic (step arrivals, a share of the
running steps ending, jobs ending and as many starting) for --passes passes without
compacting. Handle B then compacts after every further round of --round-passes passes;
handle A never does. Reported:
  - rows and bytes of the step-job table, the step table and the allocation pool on B
    before and after its first compaction (A keeps them all);
  - host wall time of steps_compact (the call ends in a stream synchronise) and its device
    time (torch.profiler, kernels and copies, in a separate last round), medians;
  - steps_run end to end and device time on B over the --round-passes passes before the
    first compaction and over the passes after it, with A's over the same passes;
  - that B's scheduled steps (at the mapped rows) and avail equal A's on every pass.
There is no host re-send arm: step_jobs_reset + re-append cannot carry a running step's
allocation, so no equal comparison exists. Prints one JSON line with the card, its power
limit and SM clocks read in the same run. Needs a CUDA device.

    python tools/bench_step_compact.py [--passes 12] [--rounds 5] [--round-passes 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cranesched_b200 import abi, synth  # noqa: E402
from cranesched_b200.scheduler import GpuScheduler  # noqa: E402
from tools.bench_step_passes import Steps, _csr_take  # noqa: E402

V, R = abi.RES_VIEW.itemsize, abi.RES_IN_NODE.itemsize
NONE = abi.ROW_NONE


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    except Exception as e:  # the numbers are still reported, with the card unknown
        return [f"unknown ({e})", "unknown", "unknown", "unknown"]


def _bytes(jobs, node_rows, steps, list_entries, alloc_rows):
    """Device bytes of the step tables: node pool CSR, step columns + list CSRs, allocation pool"""
    return {"step_jobs": 4 * (jobs + 1) + (4 + R) * node_rows,
            "steps": steps * (7 * 4 + 2 * V) + 4 * 2 * (steps + 1) + 4 * list_entries,
            "alloc_pool": (4 + R) * alloc_rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=12, help="passes before the first compaction")
    ap.add_argument("--rounds", type=int, default=5, help="compactions of B (the last one profiled)")
    ap.add_argument("--round-passes", type=int, default=3, help="passes between compactions")
    ap.add_argument("--p-job", type=float, default=0.1)
    ap.add_argument("--end-share", type=float, default=0.4)
    ap.add_argument("--job-churn", type=int, default=50)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_step_compact: no CUDA device")
    rng = np.random.Generator(np.random.PCG64(2))
    case = synth.config2()
    cfg, cl, rn, pd, now = case
    A, B = GpuScheduler(cfg, 0), GpuScheduler(cfg, 0)
    out = {"metric": "step_compact"}
    try:
        for s in (A, B):
            s.set_cluster(cl)
            s.upload(rn, pd)
            s.run(now)
        got = A.fetch(abi.Placements.for_pending(pd))
        assert not got.diff(B.fetch(abi.Placements.for_pending(pd)))
        started = np.flatnonzero(got.reason == abi.REASON_NONE)
        st = abi.Running.started(pd, got, started)
        n0 = len(started)
        for s in (A, B):
            s.step_jobs_start(s.start(started) + np.arange(n0))
        job_off, job_node, alloc = st.alloc_off.astype(np.int64), st.alloc_node.copy(), st.alloc_res.copy()
        alive = np.ones(n0, bool)
        jm, sm = np.arange(n0, dtype=np.int64), np.zeros(0, np.int64)  # A's rows -> B's
        running = set()  # A's step rows scheduled and not ended
        steps = Steps()
        timing = {k: [] for k in ("A_e2e", "A_dev", "B_e2e", "B_dev")}

        def one_pass(p, record):
            nonlocal job_off, job_node, alloc, alive, jm, sm, running
            live = np.flatnonzero(alive)
            gone = rng.choice(live, min(a.job_churn, len(live)), replace=False)
            owner, new = synth.step_pass_stream(1000 + p, job_off, job_node, alloc, np.setdiff1d(live, gone), cl,
                                                p_job=a.p_job)
            ended = sorted(q for q in running if rng.random() < a.end_share)
            came = rng.choice(np.flatnonzero(~alive) if (~alive).any() else live, len(gone))
            alive[gone] = False
            base = len(alive)
            new_off, ent = _csr_take(job_off, came)
            job_off = np.concatenate([job_off, job_off[-1] + new_off[1:]])
            job_node = np.concatenate([job_node, job_node[ent]])
            alloc = np.concatenate([alloc, alloc[ent]])
            alive = np.concatenate([alive, np.ones(len(came), bool)])
            jobs_new = abi.StepJobs(new_off.astype(np.uint32), job_node[job_off[base]:], alloc[job_off[base]:],
                                    np.zeros(len(came) + 1, np.uint32))
            if new.n:
                steps.add(new)
            res = {}
            order = (A, B) if p % 2 == 0 else (B, A)
            for s in order:
                J = (lambda r: np.asarray(r, np.int64)) if s is A else (lambda r: jm[np.asarray(r, np.int64)])
                S = (lambda r: np.asarray(r, np.int64)) if s is A else (lambda r: sm[np.asarray(r, np.int64)])
                if ended:
                    s.steps_erase(S(ended))
                s.step_jobs_erase(J(gone))
                f = s.step_jobs_append(jobs_new)
                if s is B:
                    jm = np.concatenate([jm, f + np.arange(len(came))])
                if new.n:
                    f = s.steps_append(new, J(owner))
                    if s is B:
                        sm = np.concatenate([sm, f + np.arange(new.n)])
                t0 = time.perf_counter()
                r, dev = s.steps_run()
                e2e = (time.perf_counter() - t0) * 1e3
                res[s is A] = r
                if record:
                    k = "A" if s is A else "B"
                    timing[k + "_e2e"].append(e2e)
                    timing[k + "_dev"].append(dev)
            ra, rb = res[True], res[False]
            assert rb.step_row.tolist() == sm[ra.step_row.astype(np.int64)].tolist(), f"pass {p}: rows differ"
            for fld in ("node_off", "alloc_node", "alloc_ntasks", "alloc_res", "task_off", "task_node", "task_res"):
                assert getattr(ra, fld).tobytes() == getattr(rb, fld).tobytes(), f"pass {p}: {fld} differs"
            dead_jobs = set(np.flatnonzero(~alive).tolist())
            ended_set = set(ended)
            running = {q for q in running if q not in ended_set} | set(ra.step_row.tolist())
            owner_all = getattr(one_pass, "owner_all", np.zeros(0, np.int64))
            owner_all = np.concatenate([owner_all, np.asarray(owner, np.int64)])
            one_pass.owner_all = owner_all
            running = {q for q in running if int(owner_all[q]) not in dead_jobs}

        def check_avail(p):
            live = np.flatnonzero(alive)
            assert A.step_jobs_avail(live).tobytes() == B.step_jobs_avail(jm[live]).tobytes(), f"pass {p}: avail"

        def compact():
            nonlocal jm, sm
            t0 = time.perf_counter()
            njm, nsm = B.steps_compact()
            host = (time.perf_counter() - t0) * 1e3
            for m, new in ((jm, njm), (sm, nsm)):
                ok = m != NONE
                m[ok] = new[m[ok]]
            return host

        def table(s, jobs_live=None):
            j, n, al = s.step_rows()
            if jobs_live is None:
                node_rows, lists = int(job_off[-1]), int(steps.t.incl_off[-1]) + int(steps.t.excl_off[-1])
            else:
                node_rows = int(sum(job_off[k + 1] - job_off[k] for k in jobs_live))
                kept = np.flatnonzero(sm != NONE)
                lists = int(sum(steps.t.incl_off[q + 1] - steps.t.incl_off[q] + steps.t.excl_off[q + 1]
                                - steps.t.excl_off[q] for q in kept))
            return {"rows": {"step_jobs": j, "steps": n, "alloc_pool": al}, "bytes": _bytes(j, node_rows, n, lists, al)}

        p = 0
        for _ in range(a.passes):
            one_pass(p, record=p >= a.passes - a.round_passes)
            p += 1
        check_avail(p)
        out["before"] = table(B)
        host_ms = [compact()]
        out["after"] = table(B, jobs_live=np.flatnonzero(alive))
        check_avail(p)
        before = {k: list(v) for k, v in timing.items()}
        for v in timing.values():
            v.clear()
        for rnd in range(1, a.rounds):
            for _ in range(a.round_passes):
                one_pass(p, record=rnd == 1)
                p += 1
            check_avail(p)
            if rnd < a.rounds - 1:
                host_ms.append(compact())
            else:  # the device time of one compaction, profiled on its own
                from torch.profiler import ProfilerActivity, profile
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    compact()
                    torch.cuda.synchronize()
                dev_us = 0.0
                for e in prof.events():
                    if str(e.device_type).endswith("CUDA"):
                        dev_us += float(getattr(e, "self_device_time_total", 0) or getattr(e, "self_cuda_time_total", 0))
                out["compact_device_ms_profiled"] = round(dev_us / 1e3, 4)
            check_avail(p)
        # the pass right after the last compaction
        one_pass(p, record=False)
        check_avail(p + 1)
        med = lambda v: round(float(np.median(v)), 4) if v else None
        out["compact_host_ms_median"] = med(host_ms)
        out["compact_host_ms_range"] = [round(min(host_ms), 4), round(max(host_ms), 4)]
        out["compactions_timed"] = len(host_ms)
        out["steps_run_before"] = {k + "_median": med(v) for k, v in before.items()}
        out["steps_run_after"] = {k + "_median": med(v) for k, v in timing.items()}
        out["A_rows_at_end"] = dict(zip(("step_jobs", "steps", "alloc_pool"), A.step_rows()))
        out["B_rows_at_end"] = dict(zip(("step_jobs", "steps", "alloc_pool"), B.step_rows()))
        out["results_and_avail_equal_every_pass"] = True
    finally:
        A.close()
        B.close()
    name, power, sm_clk, sm_max = _card()
    out.update({"gpu": name, "power_limit": power, "clocks_sm": sm_clk, "clocks_max_sm": sm_max, "jobs": int(n0),
                "passes_before_first": a.passes, "rounds": a.rounds, "round_passes": a.round_passes})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
