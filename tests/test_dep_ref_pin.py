"""oracle/pygate.Deps held to the reference's own DependenciesInJob text.

tests/golden/dep_ref_pin.json stores, for 300 dependency lists and event sequences, what
the reference's struct answered (tests/golden/make_dep_ref_golden.py): is_met at several
`now`, is_failed, ready_time, the entries left and the events it ignored. pygate must give
the same answers; the library is then held to pygate (tests/test_gate.py)."""
import json
import os

import pytest

from oracle import pygate
from tests.golden.make_dep_ref_golden import cases

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dep_ref_pin.json")
PIN = json.load(open(GOLDEN))["cases"]


def _pygate(c):
    d = pygate.Deps(c["is_or"], {i: (ty, dl) for i, ty, dl in c["deps"]})
    ignored = sum(not d.update(i, t) for i, t in c["events"])
    return [int(d.is_met(n)) for n in c["nows"]], int(d.is_failed()), d.ready, len(d.deps), ignored


def test_pin_inputs_are_the_generated_ones():
    assert [dict(case=c["case"], is_or=c["is_or"], deps=[list(x) for x in c["deps"]],
                 events=[list(x) for x in c["events"]], nows=c["nows"]) for c in PIN] == \
           [dict(c, deps=[list(x) for x in c["deps"]], events=[list(x) for x in c["events"]]) for c in cases()]


@pytest.mark.parametrize("block", range(6))
def test_pygate_matches_reference(block):
    for c in PIN[block * 50:(block + 1) * 50]:
        want = (c["met"], c["failed"], c["ready"], c["left"], c["ignored"])
        assert _pygate(c) == want, c["case"]


def test_pin_covers_the_edges():
    assert any(c["is_or"] and not c["deps"] for c in PIN)                        # an OR with no entries
    assert any(not c["is_or"] and c["failed"] and c["left"] for c in PIN)         # AND failed with entries left
    assert any(c["ready"] == pygate.FUTURE for c in PIN) and any(c["ready"] == pygate.PAST for c in PIN)
    assert sum(c["ignored"] for c in PIN) > 0
    assert any(dl >= 2 ** 40 for c in PIN for _, _, dl in c["deps"])
    # a finite event time whose sum with the entry's delay saturates to InfiniteFuture
    assert any(t != pygate.FUTURE and t + dict((i, dl) for i, _, dl in c["deps"])[i] > pygate.FUTURE
               for c in PIN for i, t in c["events"] if i in {d[0] for d in c["deps"]})


def test_reference_live():
    """When oracle/_ref is built: the reference run now reproduces the stored answers."""
    from oracle import ref_dep_build
    if not ref_dep_build.available():
        pytest.skip("oracle/_ref/libcrane_ref_deps.so not built (no reference source)")
    for c in PIN[:60]:
        assert list(ref_dep_build.run(c["is_or"], c["deps"], c["events"], c["nows"])) == \
               [c["met"], c["failed"], c["ready"], c["left"], c["ignored"]], c["case"]
