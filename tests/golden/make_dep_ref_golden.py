"""Writes tests/golden/dep_ref_pin.json: the reference's own DependenciesInJob
(oracle/_ref/libcrane_ref_deps.so, built from its source text by oracle/ref_dep_build.py)
on 300 random dependency lists and event sequences: AND and OR, 0-6 entries, zero and
large delays, InfiniteFuture events, finite events whose sum with the delay leaves the
int64 range, events for ids not in the list and repeated events.
Per case the inputs and the reference's answers (is_met at several `now`, is_failed,
ready_time, entries left, events ignored). No reference text is stored.

    python tests/golden/make_dep_ref_golden.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dep_ref_pin.json")
FUTURE = 2 ** 63 - 1
T0 = 1_700_000_000


def cases(n=300, seed=2024):
    rng = np.random.Generator(np.random.PCG64(seed))
    for k in range(n):
        is_or = int(rng.random() < 0.5)
        ids = [int(x) for x in rng.choice(np.arange(1, 40), int(rng.integers(0, 7)), replace=False)]
        delays = [0, 0, 1, 60, 3600, 2 ** 40, 2 ** 62 - 1]
        deps = [(i, int(rng.integers(0, 4)), int(delays[rng.integers(0, len(delays))])) for i in ids]
        events = []
        for _ in range(int(rng.integers(0, 9))):
            u = rng.random()
            if ids and u < 0.7:
                i = int(rng.choice(ids))          # an entry (again, if it was resolved before)
            else:
                i = int(rng.integers(40, 60))     # an id not in the list
            v = rng.random()
            if v < 0.15:
                t = FUTURE
            elif v < 0.25:  # finite, but t + a large delay leaves the int64 range
                t = FUTURE - int(rng.integers(1, 2 ** 62))
            else:
                t = T0 + int(rng.integers(-5000, 5000))
            events.append((i, t))
        nows = [-(2 ** 63), 0, T0 - 5000, T0, T0 + 4000, T0 + 10 ** 6, 2 ** 62, FUTURE - 1, FUTURE]
        yield dict(case=k, is_or=is_or, deps=deps, events=events, nows=nows)


def main():
    from oracle import ref_dep_build
    if not ref_dep_build.build():
        raise SystemExit("the reference's DependenciesInJob could not be built")
    rows = []
    for c in cases():
        met, failed, ready, left, ignored = ref_dep_build.run(c["is_or"], c["deps"], c["events"], c["nows"])
        rows.append(dict(c, met=met, failed=failed, ready=ready, left=left, ignored=ignored))
    with open(OUT, "w") as f:
        json.dump({"source": "DependenciesInJob, CtldPublicDefs.h:413-428 + CtldPublicDefs.cpp:144-159 (oracle/_ref)",
                   "cases": rows}, f, separators=(",", ":"))
        f.write("\n")
    print(len(rows), "cases ->", OUT)


if __name__ == "__main__":
    main()
