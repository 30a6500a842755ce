"""The reference's own answers at the kernels' size limits (synth.edge_case draws and
resource rows over all four core words, all eight gres entries and 16-slot masks),
stored in tests/golden/edge_ref_pin.json so that tests/test_edge_ref_pin.py runs
without the reference.

    python -m tests.golden.make_edge_ref_golden      (from the repo root; needs oracle/_ref, oracle/ref_build.py)

Digests as in make_ref_golden.py. Every NodeSelect draw has one gres type per name
and all-distinct priorities, the two conditions under which the reference's own
result does not depend on hash or sort order (see tests/test_ref_pin.py); the cost
policy is the reference's own (MinCpuTimeRatioFirst).
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from cranesched_b200 import abi, synth  # noqa: E402
from tests.golden.make_ref_golden import algebra_results, placement_digests  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "edge_ref_pin.json")

# name -> (n_jobs, parts, edge_case knobs, "resv" / "overlap" / None)
DRAWS = {
    "wide_20_shapes": (220, ((120, 20),), dict(p_wide=0.12), None),
    "wide_17_shapes_short": (200, ((100, 17),), dict(p_wide=0.12, short=True), None),
    "general_127": (180, ((134, 8), (30, 3)), dict(wide=(127, 100, 65, 33), p_general=0.7, p_down=0.01), None),
    "general_127_fifo": (180, ((132, 12),), dict(wide=(127, 64, 33), p_general=0.6, p_down=0.01, fifo=True), None),
    "shapes_24_and_3": (240, ((110, 24), (50, 3)), {}, None),
    "shapes_16_and_4": (220, ((90, 16), (60, 4)), dict(short=True), None),
    "shapes_5_9_18": (240, ((50, 5), (50, 9), (60, 18)), dict(p_general=0.6), None),
    "full_partition": (200, ((80, 20),), dict(p_full=0.04), None),
    "many_running": (200, ((100, 20),), dict(n_running=90, short=True), None),
    "fifo_batch_limit": (240, ((120, 20),), dict(fifo=True, limit=170), None),
    "wide_only": (150, ((128, 19),), dict(p_wide=0.3, p_general=0.5), None),
    "small_partitions": (200, ((40, 17), (36, 6), (20, 2)), {}, None),
    "reservations": (200, ((100, 20),), {}, "resv"),
    "reservations_two_partitions": (200, ((70, 10), (50, 17)), dict(fifo=True), "resv"),
    "overlapping": (220, ((80, 20), (60, 4)), {}, "overlap"),
    "overlapping_three": (220, ((60, 18), (50, 7), (40, 3)), dict(short=True), "overlap"),
}


def node_select_case(name):
    """(case, reservations or None) of draw `name`."""
    n_jobs, parts, kw, extra = DRAWS[name]
    seed = 7700 + sorted(DRAWS).index(name)
    kw = dict(kw)
    kw.setdefault("n_running", 40)
    case = synth.edge_case(seed, n_jobs=n_jobs, parts=parts, one_type_per_name=True, **kw)
    if extra == "resv":
        # one node per reservation: inside one the reference orders equal-cost nodes by node-state addresses
        resv, pd2, rn2 = synth.random_reservations(seed, case, n_resv=5, single_node=True)
        return (case[0], case[1], rn2, pd2, case[4]), resv
    if extra == "overlap":
        return synth.overlap_partitions(case, seed, frac=0.3), None
    return case, None


def algebra_draws():
    """500 (request, availability, other) rows over cores 0-255, eight gres entries (one name each)
    and 16-slot masks."""
    rng = np.random.default_rng(77)
    cl = synth.make_cluster([(1, synth.node_row(256, 1 << 40))], gres_entry_name=tuple(range(abi.GRES_ENTRIES)))
    u64 = lambda: rng.integers(0, 1 << 64, abi.CORE_WORDS, dtype=np.uint64, endpoint=False)

    def cores():
        c = u64()
        c[rng.random(abi.CORE_WORDS) < 0.2] = np.uint64(0xFFFFFFFFFFFFFFFF)
        c[rng.random(abi.CORE_WORDS) < 0.2] = 0
        return c

    def slots():
        g = rng.integers(0, 1 << 16, abi.GRES_ENTRIES).astype(np.uint16)
        g[rng.random(abi.GRES_ENTRIES) < 0.25] = 0xFFFF
        g[rng.random(abi.GRES_ENTRIES) < 0.25] = 0
        return g

    draws = []
    for _ in range(500):
        avail = np.zeros((), abi.RES_IN_NODE)
        avail["core"] = cores()
        avail["cpu_raw"] = int(rng.integers(0, 257)) * 256 - (128 if rng.random() < 0.2 else 0)
        avail["mem"] = avail["mem_sw"] = int(rng.integers(0, 1 << 20))
        avail["gres"] = slots()
        req = np.zeros((), abi.RES_VIEW)
        req["cpu_raw"] = int(rng.integers(0, 200)) * 256 + (int(rng.choice([0, 64, 128])) if rng.random() < 0.3 else 0)
        req["mem"] = req["mem_sw"] = int(rng.integers(0, 1 << 20))
        for e in range(abi.GRES_ENTRIES):
            if rng.random() < 0.5:
                sp = int(rng.integers(0, 17)) if rng.random() < 0.6 else 0
                req["gres_spec"][e] = sp
                req["gres_total"][e] = sp + (int(rng.integers(0, 4)) if rng.random() < 0.4 else 0)
        other = avail.copy()
        other["cpu_raw"] = int(rng.integers(0, 257)) * 256
        other["core"] = cores()
        other["gres"] = slots()
        draws.append((req, avail, other))
    return cl, draws


def main():
    from oracle import pyref
    if not pyref.available():
        raise SystemExit("oracle/_ref/libcrane_ref.so is not built")
    res = {"node_select": {}}
    for name in DRAWS:
        (cfg, cl, rn, pd, now), resv = node_select_case(name)
        ex = None
        if resv is not None:
            ex = pyref.RefExtra(resv_start=resv.start_time, resv_end=resv.end_time, resv_off=resv.node_off,
                                resv_node=resv.node, resv_res=resv.res, pd_resv=pd.reservation, rn_resv=rn.reservation)
        out, _ = pyref.node_select(cfg, cl, rn, pd, now, ex)
        assert cfg.priority_type == 0 or len(np.unique(out.priority)) == pd.n, name
        res["node_select"][name] = placement_digests(out)
    res["algebra"] = algebra_results(pyref, *algebra_draws())
    with open(GOLDEN, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    main()
