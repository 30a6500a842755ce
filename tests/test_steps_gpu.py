"""The step scheduler on the H100: the sm_90a kernel against the CPU oracle over many
seeds, behind the GPU NodeSelect pass (NodeSelect -> started jobs -> steps), and one
large case (the jobs config 2 starts, each with a queue of steps) compared by digest."""
import numpy as np
import pytest

from cranesched_b200 import synth
from cranesched_b200.scheduler import GpuScheduler

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def steps_oracle():
    from oracle import pystep
    pystep.build()
    return pystep


def _gpu_select(gpu_lib):
    def select(cfg, cl, rn, pd, now):
        s = GpuScheduler(cfg, 0, gpu_lib)
        try:
            s.set_cluster(cl)
            return s.node_select(now, rn, pd)
        finally:
            s.close()
    return select


def _gpu_steps(gpu_lib, cfg, cl, jobs, steps):
    s = GpuScheduler(cfg, 0, gpu_lib)
    try:
        s.set_cluster(cl)
        return s.schedule_steps(jobs, steps)
    finally:
        s.close()


@pytest.mark.parametrize("seed", range(40))
def test_gpu_steps_match_oracle(oracle, steps_oracle, gpu_lib, seed):
    case = synth.random_case(seed, n_jobs=300, n_nodes=48, n_running=20, ntpn_range=True,
                             one_type_per_name=bool(seed & 1))
    cl, jobs, steps = synth.step_case(seed, lambda *c: oracle.node_select(*c)[0], base=case)
    ja, jb = jobs.copy(), jobs.copy()
    ref, _ = steps_oracle.schedule_steps(cl, ja, steps)
    got, ms = _gpu_steps(gpu_lib, case[0], cl, jb, steps)
    assert not ref.diff(got), ref.diff(got)[:6]
    assert ja.avail.tobytes() == jb.avail.tobytes()
    assert ms >= 0


@pytest.mark.parametrize("seed", [3, 7])
def test_gpu_chain_node_select_then_steps(oracle, steps_oracle, gpu_lib, seed):
    """Running jobs taken from the GPU NodeSelect pass itself (checked against the oracle first)."""
    case = synth.random_case(seed, n_jobs=400, n_nodes=64, n_running=30, ntpn_range=True)
    pl_gpu = _gpu_select(gpu_lib)(*case[:4], case[4])
    assert not oracle.node_select(*case[:4], case[4])[0].diff(pl_gpu)
    cl, jobs, steps = synth.step_case(seed, lambda *c: pl_gpu, base=case, max_steps=8)
    ja, jb = jobs.copy(), jobs.copy()
    ref, _ = steps_oracle.schedule_steps(cl, ja, steps)
    got, _ = _gpu_steps(gpu_lib, case[0], cl, jb, steps)
    assert not ref.diff(got), ref.diff(got)[:6]
    assert ja.avail.tobytes() == jb.avail.tobytes()


def test_gpu_steps_config2_digest(steps_oracle, gpu_lib):
    """The jobs config 2 starts (GPU NodeSelect over 100k x 10k) with up to 6 steps each."""
    case = synth.config2()
    cl, jobs, steps = synth.step_case(2, _gpu_select(gpu_lib), base=case)
    assert jobs.n_jobs > 1000 and steps.n > 1000
    ja, jb = jobs.copy(), jobs.copy()
    ref, _ = steps_oracle.schedule_steps(cl, ja, steps)
    got, _ = _gpu_steps(gpu_lib, case[0], cl, jb, steps)
    assert ref.digest() == got.digest(), ref.diff(got)[:6]
    assert ja.avail.tobytes() == jb.avail.tobytes()
    assert 0 < int(got.scheduled.sum()) < steps.n
