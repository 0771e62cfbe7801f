"""An AIR whose aux segment needs LINEAR_RECURRENCE columns (a[i+1] = m_i * a[i] + t_i), for the tests of the device build.

Main columns: a value v, a 0/1 selector f (constraint f * (f - 1) = 0), a lookup column x. Random elements alpha, gamma.
Aux columns, all built by the description of linrec():
    D  running product of x + alpha                         D' = D (x + alpha),      D[0] = 1
    N  LINEAR_RECURRENCE, m = x + alpha, t = D               N' = N (x + alpha) + D,  N[0] = 0
       (N / D = sum over earlier rows of 1 / (x + alpha): a fraction sum kept as numerator / denominator, projective LogUp)
    H  LINEAR_RECURRENCE, m = gamma, t = v                   H' = gamma H + v,        H[0] = 0   (Horner fingerprint of v)
    R  LINEAR_RECURRENCE, m = 1 - f, t = v                   R' = (1 - f) R + v,      R[0] = 0   (sum of v restarting after f = 1)
"""
import numpy as np

import airs
import linrec_builds as ab

P = airs.P
LINREC_AUX_WIDTH, LINREC_NUM_RANDS = 4, 2


def linrec_trace(n, seed=11):
    rng = np.random.default_rng(seed)
    tr = np.zeros((3, n), dtype=np.uint64)
    tr[0] = rng.integers(0, P, size=n, dtype=np.uint64)
    tr[1] = (rng.integers(0, 5, size=n) == 0).astype(np.uint64)   # blocks of about five rows
    tr[2] = rng.integers(0, 1 << 20, size=n, dtype=np.uint64)
    return tr


def linrec_desc(tr):
    """The AIR description for trace tr (its one main assertion is v[0])."""
    A = airs.AirBuilder(3)
    A.constraint(A.mul(A.cur(1), A.sub(A.cur(1), A.const(1))), 2)
    A.assert_single(0, 0, int(tr[0, 0]))
    X = A.aux(LINREC_AUX_WIDTH, LINREC_NUM_RANDS)
    alpha, gamma = X.rnd(0), X.rnd(1)
    xa = X.add(X.cur(2), alpha)
    X.constraint(X.sub(X.anxt(0), X.mul(X.acur(0), xa)), 2)
    X.constraint(X.sub(X.anxt(1), X.add(X.mul(X.acur(1), xa), X.acur(0))), 2)
    X.constraint(X.sub(X.anxt(2), X.add(X.mul(gamma, X.acur(2)), X.cur(0))), 1)
    X.constraint(X.sub(X.anxt(3), X.add(X.mul(X.sub(X.const(1), X.cur(1)), X.acur(3)), X.cur(0))), 2)
    X.assert_single(0, 0, (1, 0, 0))
    for c in (1, 2, 3):
        X.assert_single(c, 0, (0, 0, 0))
    return A.build()


def linrec_build():
    B = ab.AuxBuild(3, LINREC_AUX_WIDTH, 0, LINREC_NUM_RANDS)
    d = B.column(ab.RUNNING_PRODUCT, (1, 0, 0))
    d.num(d.add(d.cur(2), d.rnd(0)))
    nn = B.column(ab.LINEAR_RECURRENCE)
    nn.multiplier(nn.add(nn.cur(2), nn.rnd(0)))
    nn.num(nn.acur(0))
    h = B.column(ab.LINEAR_RECURRENCE)
    h.multiplier(h.rnd(1))
    h.num(h.cur(0))
    r = B.column(ab.LINEAR_RECURRENCE)
    r.multiplier(r.sub(r.const(1), r.cur(1)))
    r.num(r.cur(0))
    return B.build()


def linrec(n, seed=11):
    """(description, main trace [3, n], build description, host builder rand [2, d] -> aux [4, n, d]); the host builder
    returns the CPU reference's columns (tests/linrec_build_ref.cpp)."""
    tr = linrec_trace(n, seed)
    desc, build = linrec_desc(tr), linrec_build()
    return desc, tr, build, lambda rand: ab.reference(desc, build, tr, rand)
