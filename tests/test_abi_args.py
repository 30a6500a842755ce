"""Argument checks of the C-ABI host layer, on the CPU kernel-emulation library:
the CSR offsets of every input table (they start at 0 and never decrease), the
include / exclude node lists, the order the entry points must be called in, and
the return of a handle's gres dictionary slot when it is closed."""
import dataclasses

import numpy as np
import pytest

from cranesched_b200 import abi, synth
from cranesched_b200.scheduler import CraneSchedError, GpuScheduler
from tests.helpers import assert_same

PAD = 0  # a valid entry put before the first row when the offsets are made to start at 1


def _code(fn, *args):
    try:
        fn(*args)
        return 0
    except CraneSchedError as e:
        return e.code


def _shifted(off, items, pad):
    """The same rows with one entry `pad` in front of them: off[0] == 1."""
    return np.asarray(off, np.uint32) + 1, np.concatenate([np.asarray([pad], items.dtype), items])


def _with_lists(pd, lead, **lists):
    """`pd` whose include / exclude lists get `lists[k]` (a list of nodes) prepended to
    job 0's; lead=True puts one extra entry before all lists, so that offsets start at 1."""
    kw = {}
    for k, first in lists.items():
        off = getattr(pd, k + "_off") + np.uint32(len(first))
        off[0] = 0
        nodes = np.concatenate([np.asarray(first, np.uint32), getattr(pd, k + "_nodes")])
        if lead:
            off, nodes = _shifted(off, nodes, 5)
        kw[k + "_off"], kw[k + "_nodes"] = off, nodes
    return dataclasses.replace(pd, **kw)


def _open(emu_lib, case):
    s = GpuScheduler(case[0], 0, emu_lib)
    s.set_cluster(case[1])
    return s


def _list_case():
    return synth.random_case(6, n_jobs=40, n_nodes=8, n_parts=1, n_running=0)


def test_pending_list_offsets_start_at_0(oracle, emu_lib):
    """Job 0 may run on node 0 only. With the lists' offsets starting at 0 the device
    agrees with the oracle; with one entry (node 5) before the lists and offsets
    starting at 1, upload and pending_append refuse the table."""
    cfg, cl, rn, pd, now = _list_case()
    good = _with_lists(pd, False, incl=[0])
    ref, _, _ = oracle.node_select(cfg, cl, rn, good, now)
    assert ref.alloc_node[ref.alloc_off[0]:ref.alloc_off[1]].tolist() == [0]
    s = _open(emu_lib, (cfg, cl))
    try:
        assert_same(ref, s.node_select(now, rn, good))
        for k in ("incl", "excl"):
            bad = _with_lists(pd, True, **{k: [0]})
            assert bad.incl_off[0] == (k == "incl") and bad.excl_off[0] == (k == "excl")
            assert _code(s.upload, rn, bad) == abi.EINVAL
            s.pending_reset()
            assert _code(s.pending_append, bad) == abi.EINVAL
    finally:
        s.close()


@pytest.mark.parametrize("k", ["incl", "excl"])
def test_pending_listed_node_out_of_range(emu_lib, k):
    """A listed node is a node index or 0xFFFFFFFF (a host the cluster does not know)."""
    cfg, cl, rn, pd, now = _list_case()
    s = _open(emu_lib, (cfg, cl))
    try:
        assert _code(s.upload, rn, _with_lists(pd, False, **{k: [0xFFFFFFFF]})) == 0
        assert _code(s.upload, rn, _with_lists(pd, False, **{k: [cl.n_nodes]})) == abi.EINVAL
        assert _code(s.pending_append, _with_lists(pd, False, **{k: [cl.n_nodes]})) == abi.EINVAL
    finally:
        s.close()


# ---- one malformed-offset case per table: offsets that start at 1 ------------------------------

def _cluster_call(emu_lib, bad):
    cfg, cl, rn, pd, now = synth.random_case(7, n_jobs=30, n_nodes=12, n_parts=2, n_running=4)
    if bad:
        off, nodes = _shifted(cl.part_off, cl.part_nodes, PAD)
        cl = dataclasses.replace(cl, part_off=off, part_nodes=nodes)
    s = GpuScheduler(cfg, 0, emu_lib)
    try:
        return _code(s.set_cluster, cl)
    finally:
        s.close()


def _reservations_call(emu_lib, bad):
    case = synth.random_case(501, n_jobs=40, n_nodes=26, n_parts=1, n_running=6)
    resv, _, _ = synth.random_reservations(501, case, n_resv=3)
    if bad:
        off, node = _shifted(resv.node_off, resv.node, PAD)
        res = np.concatenate([resv.res[:1], resv.res])
        resv = dataclasses.replace(resv, node_off=off, node=node, res=res)
    s = _open(emu_lib, case)
    try:
        return _code(s.set_reservations, resv)
    finally:
        s.close()


def _running_call(emu_lib, bad):
    cfg, cl, rn, pd, now = case = synth.random_case(8, n_jobs=30, n_nodes=12, n_parts=2, n_running=6)
    if bad:
        off, node = _shifted(rn.alloc_off, rn.alloc_node, PAD)
        res = np.concatenate([rn.alloc_res[:1], rn.alloc_res])
        rn = dataclasses.replace(rn, alloc_off=off, alloc_node=node, alloc_res=res)
    s = _open(emu_lib, case)
    try:
        return _code(s.upload, rn, pd)
    finally:
        s.close()


def _qos_call(emu_lib, bad):
    cfg, cl, rn, pd, now = case = synth.random_case(21, n_jobs=40, n_nodes=16, n_running=4)
    table = synth.random_qos(21, cl, pd)
    if bad:
        table.chain_off, table.chain_acct = _shifted(table.chain_off, table.chain_acct, PAD)
    s = _open(emu_lib, case)
    try:
        out = s.node_select(now, rn, pd)
        return _code(s.qos_filter, table, out.reason)
    finally:
        s.close()


def _step_tables(bad_node_off=False, bad_step_off=False, bad_list=None):
    """One job on nodes 0, 1 with one step (two steps when step_off starts at 1)."""
    node_off, node = np.array([0, 2], np.uint32), np.array([0, 1], np.uint32)
    avail = np.stack([synth.node_row(4, 8 * synth.GiB)] * 2)
    if bad_node_off:
        node_off, node = _shifted(node_off, node, PAD)
        avail = np.concatenate([avail[:1], avail])
    n_steps = 2 if bad_step_off else 1
    step_off = np.array([int(bad_step_off), n_steps], np.uint32)
    lists = {}
    for k in ("incl", "excl"):
        off, nodes = np.array([0] + [1] * n_steps, np.uint32), np.array([1 if k == "incl" else 0], np.uint32)
        if k == bad_list:
            off, nodes = _shifted(off, nodes, PAD)
        lists[k + "_off"], lists[k + "_nodes"] = off, nodes
    view = np.zeros(n_steps, abi.RES_VIEW)
    view["cpu_raw"] = 256
    one = [1] * n_steps
    return abi.StepJobs(node_off, node, avail, step_off), abi.Steps(one, one, one, one, view, view.copy(), **lists)


def _steps_call(emu_lib, **bad):
    cl = synth.make_cluster([(6, synth.node_row(8, 64 * synth.GiB))])
    jobs, steps = _step_tables(**bad)
    s = GpuScheduler(abi.Config(), 0, emu_lib)
    try:
        s.set_cluster(cl)
        return _code(s.schedule_steps, jobs, steps)
    finally:
        s.close()


TABLES = {
    "cluster.part_off": _cluster_call,
    "reservations.node_off": _reservations_call,
    "running.alloc_off": _running_call,
    "qos.chain_off": _qos_call,
    "step_jobs.node_off": lambda lib, bad: _steps_call(lib, bad_node_off=bad),
    "step_jobs.step_off": lambda lib, bad: _steps_call(lib, bad_step_off=bad),
    "steps.incl_off": lambda lib, bad: _steps_call(lib, bad_list="incl" if bad else None),
    "steps.excl_off": lambda lib, bad: _steps_call(lib, bad_list="excl" if bad else None),
}


@pytest.mark.parametrize("table", sorted(TABLES))
def test_offsets_start_at_0(emu_lib, table):
    assert TABLES[table](emu_lib, False) == 0
    assert TABLES[table](emu_lib, True) == abi.EINVAL


# ---- the order of the calls -------------------------------------------------------------------

def _overlapping_case():
    """More than 8 partitions in one connected group: set_cluster fails with CRANE_ENOSYS."""
    return synth.overlap_partitions(synth.random_case(610, n_jobs=20, n_nodes=40, n_parts=10, n_running=0), 610, 1.0)


def test_call_order(emu_lib):
    cfg, cl, rn, pd, now = case = synth.random_case(9, n_jobs=30, n_nodes=12, n_parts=2, n_running=4)
    s = GpuScheduler(cfg, 0, emu_lib)
    try:
        assert _code(s.upload, rn, pd) == abi.EINVAL
        s.set_cluster(cl)
        assert _code(s.run, now) == abi.EINVAL  # run before upload
        s.node_select(now, rn, pd)
        s.pending_append(pd.take([0]))
        out = abi.Placements.for_pending(pd)
        assert _code(s.fetch, out) == abi.EINVAL  # the appended rows void the run
        assert _code(s.device_placements) == abi.EINVAL
        assert _code(s.run, now) == abi.EINVAL  # and the running table must follow
        # a failed set_cluster voids the previous cluster
        assert _code(s.set_cluster, _overlapping_case()[1]) == abi.ENOSYS
        assert _code(s.upload, rn, pd) == abi.EINVAL
        # the step scheduler needs the cluster only
        s.set_cluster(cl)
        jobs, steps = _step_tables()
        assert _code(s.schedule_steps, jobs, steps) == 0
    finally:
        s.close()


def test_closed_handles_return_their_slot(emu_lib):
    """A device has 16 gres dictionary slots; 48 handles opened and closed one after
    the other, half of them after a failed set_cluster, all get one."""
    case = _overlapping_case()
    for i in range(48):
        s = GpuScheduler(case[0], 0, emu_lib)
        if i % 2:
            assert _code(s.set_cluster, case[1]) == abi.ENOSYS
        s.close()
