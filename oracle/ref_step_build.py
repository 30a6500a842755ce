"""Builds oracle/_ref/libcrane_ref_steps.so: the REFERENCE's own
JobInCtld::SchedulePendingSteps (src/CraneCtld/CtldPublicDefs.cpp:1877-1998).

TEST INFRASTRUCTURE ONLY (same rules as the rest of oracle/). Uses the slicing
recipe of oracle/ref_build.py (anchors, `_find` / `_func_end`; its resource-algebra
slices ph_h.inc / ph_cpp.inc) and adds one more slice, steps_cpp.inc, compiled
unmodified between the shim declarations of oracle/ref_step_shim/step_shim.h.
"""
from __future__ import annotations

import os
import subprocess
import sys

from oracle import ref_build

HERE = os.path.dirname(os.path.abspath(__file__))
SHIM = os.path.join(HERE, "ref_step_shim")
SO = os.path.join(ref_build.OUT, "libcrane_ref_steps.so")


def extract():
    c = ref_build._lines("src/CraneCtld/CtldPublicDefs.cpp")
    a = ref_build._find(c, r"^uint32_t JobInCtld::SchedulePendingSteps\(")
    ref_build._write("steps_cpp.inc", "src/CraneCtld/CtldPublicDefs.cpp", c[a:ref_build._func_end(c, a) + 1])


def build(force: bool = False) -> str | None:
    """Returns the .so path, or None when /root/reference is absent and nothing prebuilt exists."""
    have_ref = os.path.isdir(os.path.join(ref_build.REF, "src", "CraneCtld"))
    srcs = [os.path.join(SHIM, f) for f in sorted(os.listdir(SHIM))] + [
        os.path.abspath(__file__), os.path.join(HERE, "crane_ref_steps.h"), os.path.join(ref_build.HERE, "ref_shim", "ctld_shim.h")]
    if os.path.exists(SO) and not force:
        if not have_ref or all(os.path.getmtime(s) <= os.path.getmtime(SO) for s in srcs):
            return SO
    if not have_ref:
        return SO if os.path.exists(SO) else None
    ref_build.extract()
    extract()
    cmd = ["g++", "-std=c++23", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fPIC", "-shared", "-w",
           "-I", SHIM, "-I", os.path.join(HERE, "ref_shim"), "-I", ref_build.GEN, "-I", os.path.join(HERE, ".."),
           os.path.join(SHIM, "ref_steps_harness.cpp"), "-o", SO]
    subprocess.check_call(cmd)
    return SO


if __name__ == "__main__":
    p = build(force="-f" in sys.argv)
    print(p or "no /root/reference and no prebuilt oracle/_ref/libcrane_ref_steps.so")
