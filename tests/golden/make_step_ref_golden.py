"""Writes tests/golden/step_ref_pin.json: the reference's own JobInCtld::SchedulePendingSteps
(oracle/_ref/libcrane_ref_steps.so, built from its source text by oracle/ref_step_build.py) on
24 synth.step_case draws. Per case: the order in which the reference walked each job's
step_res_avail_ (a std::unordered_map) and digests of what it wrote. No reference text is stored.

    python tests/golden/make_step_ref_golden.py
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from cranesched_b200 import synth  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "step_ref_pin.json")


def cases():
    """(seed, random_case arguments): one gres type per name on a node, so the reference's
    unordered_map walk over a node's types has one possible order (as in the NodeSelect pin)."""
    for seed in range(1, 25):
        yield seed, dict(n_jobs=120 + 10 * (seed % 5), n_nodes=24 + 4 * (seed % 4), n_parts=1 + seed % 3,
                         n_running=6 + seed % 7, ntpn_range=True, one_type_per_name=True)


def make(seed, kw, select):
    return synth.step_case(seed, select, base=synth.random_case(seed, **kw), max_steps=4 + seed % 4)


def digest(out, jobs) -> str:
    h = hashlib.sha256(out.digest().encode())
    h.update(jobs.avail.tobytes())
    return h.hexdigest()


def main():
    from oracle import pyoracle, pyref_steps
    select = lambda *c: pyoracle.node_select(*c)[0]  # noqa: E731
    rows = []
    for seed, kw in cases():
        cl, jobs, steps = make(seed, kw, select)
        j = jobs.copy()
        out, visit, _ = pyref_steps.schedule_steps(cl, j, steps)
        rows.append(dict(seed=seed, kw=kw, n_jobs=jobs.n_jobs, n_steps=steps.n, scheduled=int(out.scheduled.sum()),
                         placed=int(out.placed.sum()), visit=visit.tolist(), digest=digest(out, j)))
        print(seed, steps.n, rows[-1]["scheduled"])
    with open(OUT, "w") as f:
        json.dump({"source": "JobInCtld::SchedulePendingSteps, CtldPublicDefs.cpp:1877-1998 (oracle/_ref)",
                   "cases": rows}, f, indent=0)


if __name__ == "__main__":
    main()
