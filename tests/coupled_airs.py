"""An AIR whose aux segment needs COUPLED_RECURRENCE groups (a[i+1] = M_i a[i] + t_i over several columns), for the tests of the
device build.

Main columns: v, p, q, x and a row counter s (s' = s + 1). Random elements alpha, beta, gamma.
Aux columns, all built by the description of coupled_build():
    W        POINTWISE 1 / (x + alpha)                             W (x + alpha) = 1
    (A, B)   2-group, the second-order recurrence u[i+2] = p_i u[i+1] + q_i u[i] + v_i held as (u[i+1], u[i]):
             M = [[p, q], [1, 0]], t = (v, 0)                      A' = p A + q B + v,  B' = A,      (A, B)[0] = (1, 2)
    (Y0, Y1, Y2)  3-group with a full matrix of random elements, main columns and W at rows i and i + 1:
             Y0' = alpha Y0 + x Y1 + W Y2 + v
             Y1' = Y0 + beta Y1 + p Y2 + W'
             Y2' = W' Y0 + q Y1 + gamma Y2                          (Y0, Y1, Y2)[0] = (3, 4, 5)
    H        RUNNING_SUM of A Y1 + Y2                              H' = H + A Y1 + Y2,   H[0] = 0"""
import numpy as np

import airs
import coupled_builds as cb

P = airs.P
COUPLED_AUX_WIDTH, COUPLED_NUM_RANDS = 7, 3
W, A, B, Y0, Y1, Y2, H = range(7)
INITS = {A: 1, B: 2, Y0: 3, Y1: 4, Y2: 5, H: 0}


def coupled_trace(n, seed=17):
    rng = np.random.default_rng(seed)
    tr = rng.integers(0, P, size=(5, n), dtype=np.uint64)
    tr[4] = np.arange(n, dtype=np.uint64)
    return tr


def coupled_desc(tr):
    """The AIR description for trace tr (its one main assertion is v[0])."""
    Ab = airs.AirBuilder(5)
    Ab.constraint(Ab.sub(Ab.sub(Ab.nxt(4), Ab.cur(4)), Ab.const(1)), 1)
    Ab.assert_single(0, 0, int(tr[0, 0]))
    X = Ab.aux(COUPLED_AUX_WIDTH, COUPLED_NUM_RANDS)
    alpha, beta, gamma = X.rnd(0), X.rnd(1), X.rnd(2)
    v, p, q, x = X.cur(0), X.cur(1), X.cur(2), X.cur(3)
    a, an = X.acur, X.anxt
    X.constraint(X.sub(X.mul(a(W), X.add(x, alpha)), X.const(1)), 2)
    X.constraint(X.sub(an(A), X.add(X.add(X.mul(p, a(A)), X.mul(q, a(B))), v)), 2)
    X.constraint(X.sub(an(B), a(A)), 1)
    y0 = X.add(X.add(X.mul(alpha, a(Y0)), X.mul(x, a(Y1))), X.add(X.mul(a(W), a(Y2)), v))
    X.constraint(X.sub(an(Y0), y0), 2)
    y1 = X.add(X.add(a(Y0), X.mul(beta, a(Y1))), X.add(X.mul(p, a(Y2)), an(W)))
    X.constraint(X.sub(an(Y1), y1), 2)
    y2 = X.add(X.add(X.mul(an(W), a(Y0)), X.mul(q, a(Y1))), X.mul(gamma, a(Y2)))
    X.constraint(X.sub(an(Y2), y2), 2)
    X.constraint(X.sub(an(H), X.add(a(H), X.add(X.mul(a(A), a(Y1)), a(Y2)))), 2)
    for col, val in INITS.items():
        X.assert_single(col, 0, (val, 0, 0))
    return Ab.build()


def coupled_build(broken_at=None):
    """The build of the columns above; with broken_at = i, W = (s - i) / ((x + alpha)(s - i)), 0 at row i, and the 2-group's
    t_0 = v W (x + alpha), 0 at row i: columns that break W's and A's constraints at step i and nowhere else."""
    Bd = cb.AuxBuild(5, COUPLED_AUX_WIDTH, 0, COUPLED_NUM_RANDS)
    w = Bd.column(cb.POINTWISE)
    xa = w.add(w.cur(3), w.rnd(0))
    if broken_at is None:
        w.num(w.const(1))
        w.den(xa)
    else:
        sd = w.sub(w.cur(4), w.const(broken_at))
        w.num(sd)
        w.den(w.mul(xa, sd))
    u = Bd.group(2, [(INITS[A], 0, 0), (INITS[B], 0, 0)])
    u.m(0, 0, u.cur(1))
    u.m(0, 1, u.cur(2))
    u.m(1, 0, u.const(1))
    u.t(0, u.cur(0) if broken_at is None else u.mul(u.mul(u.cur(0), u.acur(W)), u.add(u.cur(3), u.rnd(0))))
    y = Bd.group(3, [(INITS[Y0], 0, 0), (INITS[Y1], 0, 0), (INITS[Y2], 0, 0)])
    for r, row in enumerate(((y.rnd(0), y.cur(3), y.acur(W)), (y.const(1), y.rnd(1), y.cur(1)), (y.anxt(W), y.cur(2), y.rnd(2)))):
        for c, reg in enumerate(row):
            y.m(r, c, reg)
    y.t(0, y.cur(0))
    y.t(1, y.anxt(W))
    h = Bd.column(cb.RUNNING_SUM, (INITS[H], 0, 0))
    h.num(h.add(h.mul(h.acur(A), h.acur(Y1)), h.acur(Y2)))
    return Bd.build()


def coupled(n, seed=17):
    """(description, main trace [5, n], build description, host builder rand [3, d] -> aux [7, n, d]); the host builder
    returns the CPU reference's columns (tests/coupled_build_ref.cpp)."""
    tr = coupled_trace(n, seed)
    desc, build = coupled_desc(tr), coupled_build()
    return desc, tr, build, lambda rand: cb.reference(desc, build, tr, rand)
