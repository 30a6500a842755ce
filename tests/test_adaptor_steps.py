"""The step scheduler through the C++ adaptor (SchedulerAlgo::SchedulePendingSteps) with
reference-style objects: queued ids of removed steps, the reference's popped_count, the
fields written back into the steps and step_res_avail_."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build_and_run(lib_path, exe):
    libdir, libname = os.path.split(lib_path)
    out = os.path.join(ROOT, "tests", "_emu", exe)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    cmd = ["g++", "-O1", "-g", "-std=c++17", os.path.join(ROOT, "tests", "adaptor", "test_adaptor_steps.cpp"),
           os.path.join(ROOT, "cranesched_b200", "adaptor", "crane_adaptor.cpp"),
           "-L" + libdir, "-l:" + libname, "-Wl,-rpath," + libdir, "-pthread", "-o", out]
    subprocess.check_call(cmd)
    return subprocess.run([out], capture_output=True, text=True, timeout=600)


def test_adaptor_steps_on_emulated_kernels(emu_lib):
    r = _build_and_run(emu_lib, "test_adaptor_steps_emu")
    assert r.returncode == 0, r.stdout + r.stderr
    assert "adaptor steps: 0 mismatches" in r.stdout


@pytest.mark.gpu
def test_adaptor_steps_on_gpu(gpu_lib):
    r = _build_and_run(gpu_lib, "test_adaptor_steps_gpu")
    assert r.returncode == 0, r.stdout + r.stderr
    assert "adaptor steps: 0 mismatches" in r.stdout
