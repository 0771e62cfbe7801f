"""Aux build descriptions (wf_aux_build / wf_prove_air_aux_built) for the tests: a builder that emits the flat format, perm_rap's
aux columns as a description, and the CPU reference of the build semantics (tests/aux_build_ref.cpp, compiled on first use into
a temporary directory on top of the oracle's field arithmetic)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from airs import ADD, CONST, MUL, OUT, P, PERM_RAP_AUX_WIDTH, SUB

POINTWISE, RUNNING_PRODUCT, RUNNING_SUM = 0, 1, 2

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")


class AuxBuild:
    """Aux build description: per aux column a kind, an init in E and a program whose OUT 0 is the row's numerator and OUT 1
    its denominator. Registers as in airs.AuxSegment: main cur/next, aux cur/next, periodic values, random elements,
    temporaries — all in E."""

    def __init__(self, w, aw, num_periodic, nr):
        self.w, self.aw, self.np, self.nr = w, aw, num_periodic, nr
        self.consts, self.cols = [], []

    def column(self, kind, init=(0, 0, 0)):
        """Starts the next column's program; returns the builder for it."""
        c = _Column(self, kind, tuple(int(v) % P for v in init))
        self.cols.append(c)
        return c

    def build(self):
        d = [self.aw, len(self.consts)] + self.consts
        for c in self.cols:
            d += [c.kind, *c.init, c.next_reg, len(c.prog)]
            for ins in c.prog:
                d += list(ins)
        return np.array(d, dtype=np.uint64)


class _Column:
    def __init__(self, b, kind, init):
        self.b, self.kind, self.init, self.prog = b, kind, init, []
        self.next_reg = 2 * b.w + 2 * b.aw + b.np + b.nr

    def cur(self, c): return c
    def nxt(self, c): return self.b.w + c
    def acur(self, c): return 2 * self.b.w + c
    def anxt(self, c): return 2 * self.b.w + self.b.aw + c
    def per(self, j): return 2 * self.b.w + 2 * self.b.aw + j
    def rnd(self, j): return 2 * self.b.w + 2 * self.b.aw + self.b.np + j

    def op(self, code, a, b):
        d = self.next_reg
        self.next_reg += 1
        self.prog.append((code, d, a, b))
        return d

    def add(self, a, b): return self.op(ADD, a, b)
    def sub(self, a, b): return self.op(SUB, a, b)
    def mul(self, a, b): return self.op(MUL, a, b)

    def const(self, v):
        self.b.consts.append(int(v) % P)
        return self.op(CONST, len(self.b.consts) - 1, 0)

    def num(self, reg): self.prog.append((OUT, 0, reg, 0))
    def den(self, reg): self.prog.append((OUT, 1, reg, 0))


def perm_rap_build():
    """airs.perm_rap's aux columns as a build description (the same columns as its builder):
        p: running product, init 1, term (x0 + gamma) / (b + gamma)
        q: running sum, init 0, term alpha * k * x1 * p
        c: running sum, init 5, term 1"""
    B = AuxBuild(3, PERM_RAP_AUX_WIDTH, 1, 2)
    p = B.column(RUNNING_PRODUCT, (1, 0, 0))
    p.num(p.add(p.cur(0), p.rnd(0)))
    p.den(p.add(p.cur(2), p.rnd(0)))
    q = B.column(RUNNING_SUM)
    q.num(q.mul(q.mul(q.rnd(1), q.per(0)), q.mul(q.cur(1), q.acur(0))))
    c = B.column(RUNNING_SUM, (5, 0, 0))
    c.num(c.const(1))
    return B.build()


_ref = None


def _ref_lib():
    global _ref
    if _ref is None:
        out = tempfile.mkdtemp(prefix="wf_aux_build_ref_")
        so = os.path.join(out, "libwf_aux_build_ref.so")
        try:
            subprocess.check_call(["/usr/bin/g++", "-O3", "-march=x86-64-v2", "-fopenmp", "-fPIC", "-std=c++17", "-shared",
                                   "-I", _ORACLE, "-o", so, os.path.join(_HERE, "aux_build_ref.cpp")])
            _ref = C.CDLL(so)
        finally:
            shutil.rmtree(out, ignore_errors=True)   # the loaded library stays mapped
    return _ref


def reference(desc, build, trace, rand):
    """Aux columns [aw, n, d] of the build description `build` for AIR `desc` (tests/aux_build_ref.cpp): main trace [w, n],
    random elements rand [nr, d]."""
    u64p = C.POINTER(C.c_uint64)
    d_ = np.ascontiguousarray(desc, dtype=np.uint64)
    b_ = np.ascontiguousarray(build, dtype=np.uint64)
    t_ = np.ascontiguousarray(trace, dtype=np.uint64)
    r_ = np.ascontiguousarray(rand, dtype=np.uint64)
    n, d = t_.shape[1], r_.shape[-1]
    out = np.zeros((int(b_[0]), n, d), dtype=np.uint64)
    rc = _ref_lib().wfr_aux_build(d_.ctypes.data_as(u64p), C.c_size_t(d_.size), b_.ctypes.data_as(u64p), C.c_size_t(b_.size),
                                  t_.ctypes.data_as(u64p), C.c_size_t(n), C.c_int(d), r_.ctypes.data_as(u64p), out.ctypes.data_as(u64p))
    if rc != 0:
        raise ValueError(f"the reference rejected the aux build description ({rc})")
    return out
