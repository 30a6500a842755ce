"""Pins the oracle to the reference's own NodeSelect and resource algebra at the
kernels' size limits, where tests/test_edges.py compares the kernels with the oracle:
partitions of up to 24 node shapes, cores up to 256 (words 1-3, not always a prefix),
all eight gres entries with up to 16 slots, jobs of 31-127 nodes and whole partitions,
general task distributions of up to 127 nodes, running jobs holding high cores and
slots, reservations and overlapping partitions. tests/golden/edge_ref_pin.json holds the
reference's digests (tests/golden/make_edge_ref_golden.py regenerates it where the
reference is present); this test runs the oracle only.
"""
import functools
import json

import numpy as np
import pytest

from cranesched_b200 import abi
from tests.golden import make_edge_ref_golden as g
from tests.golden.make_ref_golden import algebra_results, placement_digests

with open(g.GOLDEN) as _f:
    REF = json.load(_f)


@functools.lru_cache(maxsize=None)
def _oracle_run(oracle, name):
    case, resv = g.node_select_case(name)
    return case, oracle.node_select(*case[:4], case[4], resv=resv)[0]


@pytest.mark.parametrize("name", sorted(g.DRAWS))
def test_edge_node_select_matches_reference(oracle, name):
    (cfg, cl, rn, pd, now), a = _oracle_run(oracle, name)
    assert cfg.priority_type == 0 or len(np.unique(a.priority)) == pd.n, "priorities must be distinct"
    have, want = placement_digests(a), REF["node_select"][name]
    bad = [f for f in abi.Placements.__dataclass_fields__ if have[f] != want[f]]
    assert not bad, "oracle differs from the reference's own NodeSelect in %s (reasons %s, reference %s)" % (
        bad, have["reason_hist"], want["reason_hist"])
    # the draw reaches the wide paths the kernels are tested on
    assert (a.n_alloc > 32).any()


def test_edge_draws_reach_their_shapes(oracle):
    """Across the pinned draws: jobs of more than 64 nodes and general jobs of 127 placed, partitions
    of more than 16 and of 5-16 usable shapes, allocations in core words 2-3 and entries 4-7."""
    from tests.test_edges import high_alloc, placed_general, usable_shapes
    seen = dict(wide=0, general127=0, over16=0, mid=0, core=0, gres=0)
    for name in g.DRAWS:
        case, a = _oracle_run(oracle, name)
        sh = usable_shapes(case[1])
        c, gr = high_alloc(case, a)
        for k, v in (("wide", (a.n_alloc > 64).sum()), ("general127", len(placed_general(case, a, 127))),
                     ("over16", max(sh) > 16), ("mid", any(5 <= s <= 16 for s in sh)), ("core", c), ("gres", gr)):
            seen[k] += int(v)
    assert all(seen.values()), seen


def test_edge_resource_algebra_matches_reference(oracle):
    """GetFeasibleResourceInNode with its pick, Ckmin and operator<= on rows over all four core
    words, all eight gres entries and full 16-slot masks."""
    have = algebra_results(oracle, *g.algebra_draws())
    bad = [k for k in have if have[k] != REF["algebra"][k]]
    assert not bad, "oracle differs from the reference's own resource algebra in %s" % bad
