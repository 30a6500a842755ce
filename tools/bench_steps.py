"""Measures the step scheduler of running jobs (crane_sched_schedule_steps) on one GPU.

The jobs config 2 starts now (GPU NodeSelect over 100k x 10k) become running jobs
with 0..6 FIFO steps each (synth.step_case); every repetition schedules all of them
from the same starting tables. Prints one JSON line: device ms of the step kernel
(CUDA events), end-to-end ms of the blocking call (H2D + kernel + D2H), steps placed
per second, the card and its power limit read in this run, and the single-thread CPU
time of the reference's own SchedulePendingSteps loop (oracle/_ref; the oracle's
restatement when that is not built) on the same tables, with its kind.
Needs a CUDA device; there is no CPU path.

    python tools/bench_steps.py [--steps 20] [--warmup 3] [--max-steps 6]
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

from cranesched_b200 import synth  # noqa: E402
from cranesched_b200.scheduler import GpuScheduler  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # the number is still reported, with the card unknown
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-steps", type=int, default=6)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_steps: no CUDA device")
    case = synth.config2()
    cfg = case[0]
    s = GpuScheduler(cfg, 0)
    try:
        s.set_cluster(case[1])
        cl, jobs, steps = synth.step_case(2, lambda c, cl_, rn, pd, now: s.node_select(now, rn, pd), base=case,
                                          max_steps=a.max_steps)
        dev, e2e, placed = [], [], 0
        for i in range(a.warmup + a.steps):
            j = jobs.copy()
            t0 = time.perf_counter()
            out, ms = s.schedule_steps(j, steps)
            t1 = time.perf_counter()
            if i >= a.warmup:
                dev.append(ms)
                e2e.append((t1 - t0) * 1e3)
                placed = int(out.scheduled.sum())
    finally:
        s.close()
    cpu_ms, cpu_impl = None, None
    try:
        from oracle import pyref_steps
        if pyref_steps.available():  # the reference's own SchedulePendingSteps (oracle/_ref)
            _, _, cpu_ms = pyref_steps.schedule_steps(cl, jobs.copy(), steps)
            cpu_impl = "reference"
        else:
            from oracle import pystep
            pystep.build()
            ref, cpu_ms = pystep.schedule_steps(cl, jobs.copy(), steps)
            cpu_impl = "oracle"
            assert not ref.diff(out), "GPU step placements differ from the oracle"
    except (ImportError, OSError, subprocess.CalledProcessError) as e:
        cpu_impl = f"unavailable ({e})"
    name, power = _card()
    med_dev, med_e2e = float(np.median(dev)), float(np.median(e2e))
    print(json.dumps({
        "metric": "schedule_steps", "gpu": name, "power_limit": power,
        "jobs": jobs.n_jobs, "steps": steps.n, "steps_placed": placed,
        "device_ms_median": round(med_dev, 4), "device_ms_min": round(float(np.min(dev)), 4),
        "e2e_ms_median": round(med_e2e, 4), "e2e_ms_min": round(float(np.min(e2e)), 4),
        "steps_placed_per_s": round(placed / (med_e2e / 1e3), 1),
        "cpu_single_thread_ms": None if cpu_ms is None else round(cpu_ms, 3), "cpu_impl": cpu_impl,
        "reps": a.steps, "warmup": a.warmup,
    }))


if __name__ == "__main__":
    main()
