"""Builds oracle/_ref/libcrane_ref_deps.so: the REFERENCE's own DependenciesInJob
(struct at src/CraneCtld/CtldPublicDefs.h:413-428, update at CtldPublicDefs.cpp:144-159).

TEST INFRASTRUCTURE ONLY (same rules as the rest of oracle/). Uses the slicing recipe
of oracle/ref_build.py (anchors, `_find` / `_func_end`): two slices, deps_h.inc and
deps_cpp.inc, compiled unmodified between the shim declarations of
oracle/ref_dep_shim/dep_shim.h. `run` calls it for one job's dependency list and event
sequence.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

from oracle import ref_build

HERE = os.path.dirname(os.path.abspath(__file__))
SHIM = os.path.join(HERE, "ref_dep_shim")
SO = os.path.join(ref_build.OUT, "libcrane_ref_deps.so")
_lib = None


def extract():
    os.makedirs(ref_build.GEN, exist_ok=True)
    h = ref_build._lines("src/CraneCtld/CtldPublicDefs.h")
    a = ref_build._find(h, r"^struct DependenciesInJob \{")
    ref_build._write("deps_h.inc", "src/CraneCtld/CtldPublicDefs.h", h[a:ref_build._func_end(h, a) + 1])
    c = ref_build._lines("src/CraneCtld/CtldPublicDefs.cpp")
    a = ref_build._find(c, r"^void DependenciesInJob::update\(")
    ref_build._write("deps_cpp.inc", "src/CraneCtld/CtldPublicDefs.cpp", c[a:ref_build._func_end(c, a) + 1])


def build(force: bool = False) -> str | None:
    """Returns the .so path, or None when /root/reference is absent and nothing prebuilt exists."""
    have_ref = os.path.isdir(os.path.join(ref_build.REF, "src", "CraneCtld"))
    srcs = [os.path.join(SHIM, f) for f in sorted(os.listdir(SHIM))] + [os.path.abspath(__file__)]
    if os.path.exists(SO) and not force:
        if not have_ref or all(os.path.getmtime(s) <= os.path.getmtime(SO) for s in srcs):
            return SO
    if not have_ref:
        return SO if os.path.exists(SO) else None
    extract()
    cmd = ["g++", "-std=c++20", "-O2", "-fPIC", "-shared", "-w", "-I", SHIM, "-I", ref_build.GEN,
           os.path.join(SHIM, "ref_dep_harness.cpp"), "-o", SO]
    subprocess.check_call(cmd)
    return SO


def available() -> bool:
    return os.path.exists(SO)


def run(is_or, deps, events, nows):
    """deps: (id, type, delay) triples; events: (id, time) pairs applied in order.
    Returns (is_met per now, is_failed, ready_time, entries left, events ignored)."""
    global _lib
    if _lib is None:
        _lib = C.CDLL(SO)
    ids = np.array([d[0] for d in deps], np.uint32)
    ty = np.array([d[1] for d in deps], np.uint8)
    dl = np.array([d[2] for d in deps], np.uint64)
    ev_id = np.array([e[0] for e in events], np.uint32)
    ev_t = np.array([e[1] for e in events], np.int64)
    nw = np.array(nows, np.int64)
    met = np.zeros(len(nw), np.uint8)
    failed, ready, left, ignored = C.c_uint8(), C.c_int64(), C.c_uint32(), C.c_uint32()
    p = lambda a: a.ctypes.data  # noqa: E731
    _lib.crane_ref_dep_run(C.c_uint8(int(is_or)), C.c_uint32(len(ids)), C.c_void_p(p(ids)), C.c_void_p(p(ty)),
                           C.c_void_p(p(dl)), C.c_uint32(len(ev_id)), C.c_void_p(p(ev_id)), C.c_void_p(p(ev_t)),
                           C.c_uint32(len(nw)), C.c_void_p(p(nw)), C.c_void_p(p(met)), C.byref(failed),
                           C.byref(ready), C.byref(left), C.byref(ignored))
    return [int(x) for x in met], int(failed.value), int(ready.value), int(left.value), int(ignored.value)


if __name__ == "__main__":
    p = build(force="-f" in sys.argv)
    print(p or "no /root/reference and no prebuilt oracle/_ref/libcrane_ref_deps.so")
