"""Aux build descriptions with COUPLED_RECURRENCE groups (kind 8, its k - 1 COUPLED_MEMBER columns kind 9: a[i+1] = M_i a[i] + t_i
over E^k, 2 <= k <= 4) for the tests: tests/rational_builds.py's builder with a `group(k, inits)` helper and emitters
`t(r, reg)` (OUT r) and `m(r, c, reg)` (OUT 4 + 4r + c) on the group's leader, and the CPU reference of the build semantics for
every kind (tests/coupled_build_ref.cpp, compiled on first use into a temporary directory on top of the oracle's field
arithmetic)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import rational_builds
from airs import OUT, P
from rational_builds import (LINEAR_RECURRENCE, POINTWISE, RATIONAL_RECURRENCE, RUNNING_PRODUCT,  # noqa: F401  (re-exported)
                             RUNNING_SUM)

COUPLED_RECURRENCE, COUPLED_MEMBER = 8, 9   # kinds 3, 5 and 7 are not kinds

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")


class _Column(rational_builds._Column):
    def t(self, r, reg): self.prog.append((OUT, r, reg, 0))                 # t_r of a group
    def m(self, r, c, reg): self.prog.append((OUT, 4 + 4 * r + c, reg, 0))   # M[r][c] of a group


class _Member(rational_builds._Column):
    """a COUPLED_MEMBER entry: {9, init, 0, 0}"""

    def __init__(self, b, init):
        super().__init__(b, COUPLED_MEMBER, init)
        self.next_reg = 0


class AuxBuild(rational_builds.AuxBuild):
    """rational_builds.AuxBuild with COUPLED_RECURRENCE groups."""

    def column(self, kind, init=(0, 0, 0)):
        c = _Column(self, kind, tuple(int(v) % P for v in init))
        self.cols.append(c)
        return c

    def member(self, init=(0, 0, 0)):
        m = _Member(self, tuple(int(v) % P for v in init))
        self.cols.append(m)
        return m

    def group(self, k, inits):
        """A leader and k - 1 members with inits[r] for column r of the group; returns the leader, whose program gives the step."""
        lead = self.column(COUPLED_RECURRENCE, inits[0])
        for r in range(1, k):
            self.member(inits[r])
        return lead


_ref = None


def _ref_lib():
    global _ref
    if _ref is None:
        out = tempfile.mkdtemp(prefix="wf_coupled_build_ref_")
        so = os.path.join(out, "libwf_coupled_build_ref.so")
        try:
            subprocess.check_call(["/usr/bin/g++", "-O3", "-march=x86-64-v2", "-fopenmp", "-fPIC", "-std=c++17", "-shared",
                                   "-I", _ORACLE, "-o", so, os.path.join(_HERE, "coupled_build_ref.cpp")])
            _ref = C.CDLL(so)
        finally:
            shutil.rmtree(out, ignore_errors=True)   # the loaded library stays mapped
    return _ref


def reference(desc, build, trace, rand):
    """Aux columns [aw, n, d] of the build description `build` (any kind) for AIR `desc` (tests/coupled_build_ref.cpp): main
    trace [w, n], random elements rand [nr, d]."""
    u64p = C.POINTER(C.c_uint64)
    d_ = np.ascontiguousarray(desc, dtype=np.uint64)
    b_ = np.ascontiguousarray(build, dtype=np.uint64)
    t_ = np.ascontiguousarray(trace, dtype=np.uint64)
    r_ = np.ascontiguousarray(rand, dtype=np.uint64)
    n, d = t_.shape[1], r_.shape[-1]
    out = np.zeros((int(b_[0]), n, d), dtype=np.uint64)
    rc = _ref_lib().wfr_coupled_build(d_.ctypes.data_as(u64p), C.c_size_t(d_.size), b_.ctypes.data_as(u64p), C.c_size_t(b_.size),
                                      t_.ctypes.data_as(u64p), C.c_size_t(n), C.c_int(d), r_.ctypes.data_as(u64p), out.ctypes.data_as(u64p))
    if rc != 0:
        raise ValueError(f"the reference rejected the aux build description ({rc})")
    return out
