"""Aux build descriptions with RATIONAL_RECURRENCE columns (kind 6: a[i+1] = (m_i a[i] + n_i) / (c_i a[i] + d_i), inv(0) = 0)
for the tests: tests/linrec_builds.py's builder with a `den_multiplier(reg)` emitter for OUT 3 (c_i), and the CPU reference of
the build semantics for every kind (tests/rational_build_ref.cpp, compiled on first use into a temporary directory on top of
the oracle's field arithmetic). In a RATIONAL_RECURRENCE column `num` emits n_i (OUT 0), `den` d_i (OUT 1, default 1) and
`multiplier` m_i (OUT 2)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import linrec_builds
from airs import OUT, P
from linrec_builds import LINEAR_RECURRENCE, POINTWISE, RUNNING_PRODUCT, RUNNING_SUM  # noqa: F401  (re-exported)

RATIONAL_RECURRENCE = 6   # kinds 3 and 5 are not kinds

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")


class _Column(linrec_builds._Column):
    def den_multiplier(self, reg): self.prog.append((OUT, 3, reg, 0))   # c_i of a RATIONAL_RECURRENCE column


class AuxBuild(linrec_builds.AuxBuild):
    """linrec_builds.AuxBuild whose columns also emit OUT 3, the denominator multiplier of a RATIONAL_RECURRENCE column."""

    def column(self, kind, init=(0, 0, 0)):
        c = _Column(self, kind, tuple(int(v) % P for v in init))
        self.cols.append(c)
        return c


_ref = None


def _ref_lib():
    global _ref
    if _ref is None:
        out = tempfile.mkdtemp(prefix="wf_rational_build_ref_")
        so = os.path.join(out, "libwf_rational_build_ref.so")
        try:
            subprocess.check_call(["/usr/bin/g++", "-O3", "-march=x86-64-v2", "-fopenmp", "-fPIC", "-std=c++17", "-shared",
                                   "-I", _ORACLE, "-o", so, os.path.join(_HERE, "rational_build_ref.cpp")])
            _ref = C.CDLL(so)
        finally:
            shutil.rmtree(out, ignore_errors=True)   # the loaded library stays mapped
    return _ref


def reference(desc, build, trace, rand):
    """Aux columns [aw, n, d] of the build description `build` (any kind) for AIR `desc` (tests/rational_build_ref.cpp): main
    trace [w, n], random elements rand [nr, d]."""
    u64p = C.POINTER(C.c_uint64)
    d_ = np.ascontiguousarray(desc, dtype=np.uint64)
    b_ = np.ascontiguousarray(build, dtype=np.uint64)
    t_ = np.ascontiguousarray(trace, dtype=np.uint64)
    r_ = np.ascontiguousarray(rand, dtype=np.uint64)
    n, d = t_.shape[1], r_.shape[-1]
    out = np.zeros((int(b_[0]), n, d), dtype=np.uint64)
    rc = _ref_lib().wfr_rational_build(d_.ctypes.data_as(u64p), C.c_size_t(d_.size), b_.ctypes.data_as(u64p), C.c_size_t(b_.size),
                                       t_.ctypes.data_as(u64p), C.c_size_t(n), C.c_int(d), r_.ctypes.data_as(u64p), out.ctypes.data_as(u64p))
    if rc != 0:
        raise ValueError(f"the reference rejected the aux build description ({rc})")
    return out
