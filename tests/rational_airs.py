"""An AIR whose aux segment needs RATIONAL_RECURRENCE columns (a[i+1] = (m_i a[i] + n_i) / (c_i a[i] + d_i)), for the tests of
the device build.

Main columns: a value v, a multiplier x, a denominator multiplier s, a denominator u, a row counter k (k' = k + 1). Random
elements alpha, beta.
Aux columns, all built by the description of rational_build():
    F  RATIONAL_RECURRENCE, m = alpha, n = v, c = 1, d = beta     F' (F + beta) = alpha F + v,   F[0] = 0
       (a fractional fingerprint of v held in one column)
    G  RATIONAL_RECURRENCE, m = x, n = v, c = s, d = u             G' (s G + u) = x G + v,         G[0] = 1
       (driven by the main trace alone, so a trace can place a vanishing denominator s_i G[i] + u_i on any row)
    H  RUNNING_SUM of F G                                          H' = H + F G,                   H[0] = 0
Where a denominator vanishes the column's next value is 0 (inv(0) = 0): G's constraint then holds only if the numerator vanishes
too (a 0/0 row)."""
import numpy as np

import airs
import rational_builds as rb

P = airs.P
RATIONAL_AUX_WIDTH, RATIONAL_NUM_RANDS = 3, 2


def g_column(tr):
    """G over the base field, as Python integers (it reads no random element)"""
    v, x, s, u = ([int(e) for e in tr[c]] for c in range(4))
    g, a = [], 1
    for i in range(tr.shape[1]):
        g.append(a)
        den = (s[i] * a + u[i]) % P
        a = (x[i] * a + v[i]) * pow(den, P - 2, P) % P if den else 0
    return g


def rational_trace(n, seed=13, zeros=(), zero_zero=()):
    """Main trace [5, n]; the rows in `zeros` get s_i G[i] + u_i = 0 (a vanishing denominator; G's constraint then fails there),
    the rows in `zero_zero` also x_i G[i] + v_i = 0 (0/0: the constraint holds)."""
    rng = np.random.default_rng(seed)
    tr = rng.integers(0, P, size=(5, n), dtype=np.uint64)
    tr[4] = np.arange(n, dtype=np.uint64)
    aimed = sorted(set(zeros) | set(zero_zero))
    for i in aimed:   # in row order: G[i] depends on rows < i only
        gi = g_column(tr[:, : i + 1])[i]
        tr[3, i] = (-int(tr[2, i]) * gi) % P
        if i in zero_zero:
            tr[0, i] = (-int(tr[1, i]) * gi) % P
    return tr


def rational_desc(tr):
    """The AIR description for trace tr (its one main assertion is v[0])."""
    A = airs.AirBuilder(5)
    A.constraint(A.sub(A.sub(A.nxt(4), A.cur(4)), A.const(1)), 1)
    A.assert_single(0, 0, int(tr[0, 0]))
    X = A.aux(RATIONAL_AUX_WIDTH, RATIONAL_NUM_RANDS)
    alpha, beta = X.rnd(0), X.rnd(1)
    X.constraint(X.sub(X.mul(X.anxt(0), X.add(X.acur(0), beta)), X.add(X.mul(alpha, X.acur(0)), X.cur(0))), 2)
    X.constraint(X.sub(X.mul(X.anxt(1), X.add(X.mul(X.cur(2), X.acur(1)), X.cur(3))), X.add(X.mul(X.cur(1), X.acur(1)), X.cur(0))), 3)
    X.constraint(X.sub(X.anxt(2), X.add(X.acur(2), X.mul(X.acur(0), X.acur(1)))), 2)
    X.assert_single(0, 0, (0, 0, 0))
    X.assert_single(1, 0, (1, 0, 0))
    X.assert_single(2, 0, (0, 0, 0))
    return A.build()


def rational_build():
    B = rb.AuxBuild(5, RATIONAL_AUX_WIDTH, 0, RATIONAL_NUM_RANDS)
    f = B.column(rb.RATIONAL_RECURRENCE)
    f.multiplier(f.rnd(0))
    f.num(f.cur(0))
    f.den_multiplier(f.const(1))
    f.den(f.rnd(1))
    g = B.column(rb.RATIONAL_RECURRENCE, (1, 0, 0))
    g.multiplier(g.cur(1))
    g.num(g.cur(0))
    g.den_multiplier(g.cur(2))
    g.den(g.cur(3))
    h = B.column(rb.RUNNING_SUM)
    h.num(h.mul(h.acur(0), h.acur(1)))
    return B.build()


def rational(n, seed=13, zeros=(), zero_zero=()):
    """(description, main trace [5, n], build description, host builder rand [2, d] -> aux [3, n, d]); the host builder
    returns the CPU reference's columns (tests/rational_build_ref.cpp)."""
    tr = rational_trace(n, seed, zeros, zero_zero)
    desc, build = rational_desc(tr), rational_build()
    return desc, tr, build, lambda rand: rb.reference(desc, build, tr, rand)
