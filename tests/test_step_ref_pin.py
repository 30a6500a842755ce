"""The step oracle held to the reference's own JobInCtld::SchedulePendingSteps text.

tests/golden/step_ref_pin.json stores, for 24 step_case draws, the order in which the
reference walked each job's step_res_avail_ (std::unordered_map, libstdc++ hash order)
and a digest of what it wrote (tests/golden/make_step_ref_golden.py). Fed that order, the
oracle must write the same bytes; the GPU path is then held to the oracle in node-index
order (deviation D8: the walk order is the only difference)."""
import json
import os

import numpy as np
import pytest

from tests.golden.make_step_ref_golden import cases, digest, make

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "step_ref_pin.json")
PIN = {c["seed"]: c for c in json.load(open(GOLDEN))["cases"]}


@pytest.fixture(scope="module")
def steps_oracle():
    from oracle import pystep
    pystep.build()
    return pystep


@pytest.mark.parametrize("seed,kw", list(cases()), ids=[f"seed{s}" for s, _ in cases()])
def test_oracle_matches_reference_under_its_walk(oracle, steps_oracle, seed, kw):
    pin = PIN[seed]
    assert pin["kw"] == kw
    cl, jobs, steps = make(seed, kw, lambda *c: oracle.node_select(*c)[0])
    assert (jobs.n_jobs, steps.n) == (pin["n_jobs"], pin["n_steps"])
    j = jobs.copy()
    out, _ = steps_oracle.schedule_steps(cl, j, steps, np.array(pin["visit"], np.uint32))
    assert int(out.scheduled.sum()) == pin["scheduled"] and int(out.placed.sum()) == pin["placed"]
    assert digest(out, j) == pin["digest"]


def test_walk_order_is_observable(oracle, steps_oracle):
    """D8 is a real deviation: in node-index order some pinned cases place steps differently."""
    differ = 0
    for seed, kw in list(cases())[:6]:
        cl, jobs, steps = make(seed, kw, lambda *c: oracle.node_select(*c)[0])
        j = jobs.copy()
        out, _ = steps_oracle.schedule_steps(cl, j, steps)
        differ += digest(out, j) != PIN[seed]["digest"]
    assert differ > 0


def test_reference_live(oracle, steps_oracle):
    """When oracle/_ref is built: the reference run now reproduces the stored walk and digest."""
    from oracle import pyref_steps
    if not pyref_steps.available():
        pytest.skip("oracle/_ref/libcrane_ref_steps.so not built (no reference source)")
    for seed, kw in list(cases())[:4]:
        cl, jobs, steps = make(seed, kw, lambda *c: oracle.node_select(*c)[0])
        j = jobs.copy()
        out, visit, _ = pyref_steps.schedule_steps(cl, j, steps)
        assert visit.tolist() == PIN[seed]["visit"] and digest(out, j) == PIN[seed]["digest"]
