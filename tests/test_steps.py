"""The step scheduler of running jobs (JobInCtld::SchedulePendingSteps,
CtldPublicDefs.cpp:1877-1998) without a GPU: hand-derived answers on the CPU
oracle, the real kernel source under tests/cuda_emu against the oracle, and the
argument checks of crane_sched_schedule_steps."""
import numpy as np
import pytest

from cranesched_b200 import abi, synth
from cranesched_b200.scheduler import CraneSchedError, GpuScheduler

GiB = synth.GiB


@pytest.fixture(scope="module")
def steps_oracle():
    from oracle import pystep
    pystep.build()
    return pystep


def _cluster(n=6):
    return synth.make_cluster([(n, synth.node_row(8, 64 * GiB))])


def _avail(cores):
    """step_res_avail_ rows: node k holds cores {0 .. cores[k]-1}, 8 GiB."""
    return np.stack([synth.node_row(c, 8 * GiB) for c in cores])


def _steps(rows, incl=None, excl=None):
    """rows: (node_num, ntasks, ntpn_min, ntpn_max, task cpus)."""
    n = len(rows)
    vt = np.zeros(n, abi.RES_VIEW)
    vt["cpu_raw"] = [int(r[4] * 256) for r in rows]
    kw = {}
    for k, lists in (("incl", incl), ("excl", excl)):
        if lists is not None:
            off = np.zeros(n + 1, np.uint32)
            off[1:] = np.cumsum([len(x) for x in lists])
            kw[k + "_off"], kw[k + "_nodes"] = off, np.array(sum(lists, []), np.uint32)
    return abi.Steps([r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows], [r[3] for r in rows],
                     np.zeros(n, abi.RES_VIEW), vt, **kw)


def _one_job(nodes, cores, n_steps):
    return abi.StepJobs([0, len(nodes)], nodes, _avail(cores), [0, n_steps])


def _rows(out, s, what):
    off = out.node_off if what == "node" else out.task_off
    sl = slice(int(off[s]), int(off[s + 1]))
    if what == "node":
        return out.alloc_node[sl].tolist(), out.alloc_ntasks[sl].tolist(), out.alloc_res[sl]
    return out.task_node[sl].tolist(), out.task_res[sl]


def test_head_of_line_blocking(steps_oracle):
    """A step that fits nowhere keeps every later step of its job pending, even one that would fit."""
    cl = _cluster()
    jobs = _one_job([0, 1], [4, 4], 2)
    before = jobs.avail.copy()
    out, _ = steps_oracle.schedule_steps(cl, jobs, _steps([(1, 1, 1, 1, 6), (1, 1, 1, 1, 1)]))
    assert out.placed.tolist() == [0] and out.scheduled.tolist() == [0, 0]
    assert (jobs.avail == before).all()
    assert not out.alloc_res["cpu_raw"].any() and not out.task_res["cpu_raw"].any()


def test_ntpn_min_rejects_a_node(steps_oracle):
    """Node 2 holds 2 tasks < ntasks_per_node_min = 3 and is skipped; node 4 takes all 3."""
    cl = _cluster()
    jobs = _one_job([2, 4], [2, 5], 1)
    out, _ = steps_oracle.schedule_steps(cl, jobs, _steps([(1, 3, 3, 3, 1)]))
    assert out.placed.tolist() == [1]
    nodes, ntasks, res = _rows(out, 0, "node")
    assert nodes == [4] and ntasks == [3]
    assert res["cpu_raw"].tolist() == [3 * 256] and int(res["core"][0, 0]) == 0b111
    tnode, tres = _rows(out, 0, "task")
    assert tnode == [4, 4, 4] and [int(x) for x in tres["core"][:, 0]] == [1, 2, 4]
    assert int(jobs.avail["core"][1, 0]) == 0b11000 and int(jobs.avail["cpu_raw"][1]) == 2 * 256
    assert int(jobs.avail["cpu_raw"][0]) == 2 * 256  # untouched


def test_heap_overflow_rest_distribution_and_task_ids(steps_oracle):
    """node_num = 2, ntasks = 6, ntasks_per_node <= 3; nodes hold 1, 3, 3, 3 tasks.
    Walk: 10 (1 task), 11 (3) -> sum 4 < 6; 12 (3) overflows the heap, the top (10,
    fewest tasks) is popped, sum 6 -> stop; node 13 is never visited. Heap pop order
    11, 12 (equal counts: libstdc++ order); rest = 4: node 11 gets min(4, 2) + 1 = 3
    tasks (ids 0-2), rest 2; node 12 gets 3 (ids 3-5)."""
    cl = _cluster(16)
    jobs = _one_job([10, 11, 12, 13], [1, 3, 3, 3], 1)
    out, _ = steps_oracle.schedule_steps(cl, jobs, _steps([(2, 6, 1, 3, 1)]))
    nodes, ntasks, _ = _rows(out, 0, "node")
    assert nodes == [11, 12] and ntasks == [3, 3]
    tnode, _ = _rows(out, 0, "task")
    assert tnode == [11, 11, 11, 12, 12, 12]
    assert jobs.avail["cpu_raw"].tolist() == [256, 0, 0, 3 * 256]


def test_uneven_rest_and_ties(steps_oracle):
    """Three nodes of 4 tasks each tie; node_num = 3, ntasks = 7: the heap stops after the
    third push (sum 12 >= 7) and pops in push order (ties keep libstdc++'s order); rest = 4:
    min(4, 3) + 1 = 4 tasks (ids 0-3) on the first, rest 1; min(1, 3) + 1 = 2 (ids 4, 5) on
    the second, rest 0; 1 (id 6) on the third."""
    cl = _cluster()
    jobs = _one_job([1, 3, 5], [4, 4, 4], 1)
    out, _ = steps_oracle.schedule_steps(cl, jobs, _steps([(3, 7, 1, 4, 1)]))
    nodes, ntasks, _ = _rows(out, 0, "node")
    assert nodes == [1, 3, 5] and ntasks == [4, 2, 1]
    assert _rows(out, 0, "task")[0] == [1, 1, 1, 1, 3, 3, 5]


def test_lists_and_carry_over(steps_oracle):
    """Exclude / include lists (an unknown host in an include list counts as a member of a
    non-empty list); each step sees what the earlier steps left."""
    cl = _cluster()
    jobs = _one_job([0, 1, 2], [2, 2, 2], 3)
    steps = _steps([(1, 2, 1, 2, 1), (1, 2, 1, 2, 1), (1, 1, 1, 1, 1)],
                   incl=[[], [0xFFFFFFFF, 2], [0xFFFFFFFF]], excl=[[0], [], []])
    out, _ = steps_oracle.schedule_steps(cl, jobs, steps)
    assert out.placed.tolist() == [2] and out.scheduled.tolist() == [1, 1, 0]
    assert _rows(out, 0, "node")[0] == [1] and _rows(out, 1, "node")[0] == [2]
    assert jobs.avail["cpu_raw"].tolist() == [512, 0, 0]


def test_visit_order_changes_the_pick(steps_oracle):
    """The walk order decides which of equal nodes is taken (the reference's unordered_map order)."""
    cl = _cluster()
    steps = _steps([(1, 1, 1, 1, 1)])
    a, _ = steps_oracle.schedule_steps(cl, _one_job([0, 1], [4, 4], 1), steps)
    b, _ = steps_oracle.schedule_steps(cl, _one_job([0, 1], [4, 4], 1), steps, visit=[1, 0])
    assert _rows(a, 0, "node")[0] == [0] and _rows(b, 0, "node")[0] == [1]


def _emu_run(emu_lib, cl, jobs, steps, cfg=None):
    s = GpuScheduler(cfg or abi.Config(), 0, emu_lib)
    try:
        s.set_cluster(cl)
        return s.schedule_steps(jobs, steps)[0]
    finally:
        s.close()


@pytest.mark.parametrize("seed", [1, 2, 5, 8, 13])
def test_emulated_step_kernel_matches_oracle(oracle, steps_oracle, emu_lib, seed):
    case = synth.random_case(seed, n_jobs=150, n_nodes=30, n_running=8, ntpn_range=True,
                             one_type_per_name=bool(seed & 1))
    cl, jobs, steps = synth.step_case(seed, lambda *c: oracle.node_select(*c)[0], base=case)
    assert steps.n > 50
    ja, jb = jobs.copy(), jobs.copy()
    ref, _ = steps_oracle.schedule_steps(cl, ja, steps)
    got = _emu_run(emu_lib, cl, jb, steps, case[0])
    assert not ref.diff(got), ref.diff(got)
    assert ja.avail.tobytes() == jb.avail.tobytes()
    assert 0 < int(ref.scheduled.sum()) < steps.n


def test_emulated_hand_cases(steps_oracle, emu_lib):
    """The hand-derived cases above through the emulated kernel, as one table of jobs."""
    cl = _cluster(16)
    jobs = abi.StepJobs([0, 2, 4, 8, 11], [0, 1, 2, 4, 10, 11, 12, 13, 1, 3, 5],
                        _avail([4, 4, 2, 5, 1, 3, 3, 3, 4, 4, 4]), [0, 2, 3, 4, 5])
    steps = _steps([(1, 1, 1, 1, 6), (1, 1, 1, 1, 1), (1, 3, 3, 3, 1), (2, 6, 1, 3, 1), (3, 7, 1, 4, 1)])
    ja, jb = jobs.copy(), jobs.copy()
    ref, _ = steps_oracle.schedule_steps(cl, ja, steps)
    got = _emu_run(emu_lib, cl, jb, steps)
    assert ref.placed.tolist() == [0, 1, 1, 1]
    assert not ref.diff(got), ref.diff(got)
    assert ja.avail.tobytes() == jb.avail.tobytes()


def _code(emu_lib, cl, jobs, steps, set_cluster=True):
    s = GpuScheduler(abi.Config(), 0, emu_lib)
    try:
        if set_cluster:
            s.set_cluster(cl)
        s.schedule_steps(jobs, steps)
        return 0
    except CraneSchedError as e:
        return e.code
    finally:
        s.close()


def test_argument_checks(emu_lib):
    cl = _cluster()
    ok = _steps([(1, 1, 1, 1, 1)])
    assert _code(emu_lib, cl, _one_job([0, 1], [4, 4], 1), ok) == 0
    assert _code(emu_lib, cl, _one_job([0, 1], [4, 4], 1), ok, set_cluster=False) == abi.EINVAL
    assert _code(emu_lib, cl, _one_job([0, 6], [4, 4], 1), ok) == abi.EINVAL       # node out of range
    assert _code(emu_lib, cl, _one_job([1, 1], [4, 4], 1), ok) == abi.EINVAL       # repeated node
    assert _code(emu_lib, cl, _one_job([2, 1], [4, 4], 1), ok) == abi.EINVAL       # not ascending
    for bad in ((0, 1, 1, 1, 1), (2, 1, 1, 1, 1), (1, 2, 3, 2, 1)):                # node_num 0, ntasks < node_num, min > max
        assert _code(emu_lib, cl, _one_job([0, 1], [4, 4], 1), _steps([bad])) == abi.EINVAL
    assert _code(emu_lib, cl, _one_job([0, 1], [4, 4], 1), _steps([(128, 128, 1, 1, 1)])) == abi.ENOSYS
    assert _code(emu_lib, cl, _one_job([0, 1], [4, 4], 1), _steps([(1, 1, 0, 1, 1)])) == abi.ENOSYS
    assert _code(emu_lib, cl, _one_job([0, 1], [4, 4], 1), _steps([(1, 1, 1, 1, 1)], incl=[[7]])) == abi.EINVAL
    assert _code(emu_lib, cl, _one_job([0, 1], [4, 4], 1), _steps([(127, 127, 1, 1, 1)])) == 0  # blocks, no error
