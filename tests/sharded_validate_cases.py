"""Traces with planted violations for the sharded prover's trace checks (tests/sharded_validate_worker.py and
tests/test_sharded_validate_cases.py). A case is a JSON dictionary: the fixture keys of sharded_air_worker.air_of, plus
"plant", the violation, and "at", where a planted transition fails: "0", "edge-1" (step n/G - 1, whose next row is the next
rank's first row), "edge" (step n/G, the next rank's first step) or "last" (step n - exemptions - 1). `want` gives the first
violation the reference's Trace::validate or validate_transition_degrees reports for it, and `where` the rank or boundary
the case is aimed at, so the CPU test can show that each case hits the shard edge it names."""
import numpy as np

import airs
import aux_builds as ab
import trace_validate_ref as R
from airs import P
from sharded_air_worker import air_of


def bump(t, col, row, by=1):
    t[col, row] = (int(t[col, row]) + by) % P


def step_of(at, n, world, exemptions=1):
    return {"0": 0, "edge-1": n // world - 1, "edge": n // world, "last": n - exemptions - 1}[at]


def fib_reversed(k, n):
    """FibSmall x k with its assertions listed from the last pair to the first: assertion 0 is on the highest column pair,
    which the last column-owning rank holds, and the highest indices are on rank 0's columns."""
    d, tr = airs.fib_small_x(k, n)
    A = R.Air(d)
    words = [int(v) for v in d]
    head = 2 + sum(2 + len(c) for _, c in A.degrees)
    head += 1 + sum(1 + len(c) for c in A.periodic)
    head += 1 + len(A.consts) + 1 + 1 + 4 * len(A.prog)
    groups = [A.asserts[3 * j:3 * j + 3] for j in range(k)][::-1]
    body = [len(A.asserts)]
    for g in groups:
        for col, first, stride, vals in g:
            body += [col, first, stride, len(vals)] + [v[0] for v in vals]
    skip = 1 + sum(4 + len(v) for _, _, _, v in A.asserts)
    return np.array(words[:head] + body + words[head + skip:], dtype=np.uint64), tr


def perm_rap_wide(n, aux1_degree=(2, [4])):
    """perm_rap with a third main constraint (x1' = x1 + x0' stated twice), so that with ext 3 the columns of aux constraint 1
    in the degree check are 6, 7 and 8: they straddle the first 8-column segment. aux1_degree: its declared degree."""
    d, tr, builder = airs.perm_rap(n)
    A = airs.AirBuilder(3)
    A.periodic = [[1, 2, 3, 4]]
    A.pub = [int(tr[1, n - 1])]
    A.constraint(A.sub(A.nxt(0), A.add(A.cur(0), A.cur(1))), 1)
    A.constraint(A.sub(A.nxt(1), A.add(A.cur(1), A.nxt(0))), 1)
    A.constraint(A.sub(A.nxt(1), A.add(A.cur(1), A.nxt(0))), 1)
    A.assert_single(0, 0, 1)
    A.assert_single(1, 0, 1)
    A.assert_single(1, n - 1, int(tr[1, n - 1]))
    X = A.aux(airs.PERM_RAP_AUX_WIDTH, 2)
    gamma, alpha = X.rnd(0), X.rnd(1)
    X.constraint(X.sub(X.mul(X.anxt(0), X.add(X.cur(2), gamma)), X.mul(X.acur(0), X.add(X.cur(0), gamma))), 2)
    term = X.mul(X.mul(alpha, X.per(0)), X.mul(X.cur(1), X.acur(0)))
    X.constraint(X.sub(X.anxt(1), X.add(X.acur(1), term)), aux1_degree[0], aux1_degree[1])
    X.assert_single(0, 0, (1, 0, 0))
    X.assert_single(0, n - 1, (1, 0, 0))
    X.assert_single(1, 0, (0, 0, 0))
    X.constraint(X.sub(X.anxt(2), X.add(X.acur(2), X.const(1))), 1)
    X.assert_sequence(2, 1, n // 4, [(5 + 1 + k * (n // 4), 0, 0) for k in range(4)])
    return A.build(), tr, builder


def perm_rap_build(init_p=1, c_term="one"):
    """perm_rap's build description (aux_builds.perm_rap_build), with p's init and c's term open to change:
    c_term "one" (the right term), "two", or "gated": 1 + (x1' - x1 - x0'), which is 1 wherever the main transition
    x1' = x1 + x0' holds and differs from it on exactly the steps where that main constraint fails."""
    B = ab.AuxBuild(3, airs.PERM_RAP_AUX_WIDTH, 1, 2)
    p = B.column(ab.RUNNING_PRODUCT, (init_p, 0, 0))
    p.num(p.add(p.cur(0), p.rnd(0)))
    p.den(p.add(p.cur(2), p.rnd(0)))
    q = B.column(ab.RUNNING_SUM)
    q.num(q.mul(q.mul(q.rnd(1), q.per(0)), q.mul(q.cur(1), q.acur(0))))
    c = B.column(ab.RUNNING_SUM, (5, 0, 0))
    if c_term == "gated":
        c.num(c.add(c.const(1), c.sub(c.sub(c.nxt(1), c.cur(1)), c.nxt(0))))
    else:
        c.num(c.const(2 if c_term == "two" else 1))
    return B.build()


def fib_exempt2(n):
    """FibSmall x 2 with two exemptions and no last-step assertion: steps n-2 and n-1 are not checked, so rows n-1 of the
    first pair may hold anything."""
    tr = airs.fib_small_x(2, n)[1]
    A = airs.AirBuilder(4)
    A.exemptions = 2
    for j in range(2):
        A.constraint(A.sub(A.nxt(2 * j), A.add(A.cur(2 * j), A.cur(2 * j + 1))), 1)
        A.constraint(A.sub(A.nxt(2 * j + 1), A.add(A.cur(2 * j + 1), A.nxt(2 * j))), 1)
        A.assert_single(2 * j, 0, j + 1)
        A.assert_single(2 * j + 1, 0, j + 1)
    return A.build(), tr


def make(case, n, world):
    """(description, trace, aux build, values_fn, num_rands, num_values) of a case, its violation planted."""
    plant = case.get("plant")
    if plant is None:
        return air_of(case, n)
    s = step_of(case.get("at", "0"), n, world)
    if plant == "assert_last_rank":      # FibSmall x 16 reversed: assertion 2 is column 31's last-step value
        d, t = fib_reversed(16, n)
        t = t.copy(); bump(t, 31, n - 1)
        return d, t, None, None, 0, 0
    if plant == "asserts_two_ranks":     # column 31 (the last owning rank, assertion 1) and column 0 (rank 0, assertion 45)
        d, t = fib_reversed(16, n)
        t = t.copy(); bump(t, 0, 0); bump(t, 31, 0)
        return d, t, None, None, 0, 0
    if plant == "sequence_two_steps":    # sequence_mix's sequence assertion on column 0: values 3 and 2^(log_n - 3)
        d, t = airs.sequence_mix(n)
        t = t.copy(); bump(t, 0, 1 + 4 * (n // 8)); bump(t, 0, 1 + 4 * 3)
        return d, t, None, None, 0, 0
    if plant == "main_transition":       # FibSmall x 8: x2 at row s + 1, so constraint 2 fails first at step s
        d, t = airs.fib_small_x(8, n)
        t = t.copy(); bump(t, 2, s + 1)
        return d, t, None, None, 0, 0
    if plant == "exempt_rows":           # rows n-1 of the first pair: only the exempt steps read them
        d, t = fib_exempt2(n)
        t = t.copy(); bump(t, 0, n - 1, 5); bump(t, 1, n - 1, 7)
        return d, t, None, None, 0, 0
    if plant == "two_ranks":             # constraint 4 at step 1 (rank 0), constraint 2 at the last rank's first step
        d, t = airs.fib_small_x(8, n)
        t = t.copy(); bump(t, 4, 2); bump(t, 2, (world - 1) * (n // world) + 1)
        return d, t, None, None, 0, 0
    if plant == "main_and_aux_same_step":   # x1 at row s + 1: main constraint 1 and, through the gated term, aux 2 at step s
        d, t, _ = airs.perm_rap(n)
        t = t.copy(); bump(t, 1, s + 1)
        return d, t, perm_rap_build(c_term="gated"), None, 2, 7
    if plant == "aux_init":
        d, t, _ = airs.perm_rap(n)
        return d, t, perm_rap_build(init_p=2), None, 2, 7
    if plant == "aux_term":
        d, t, _ = airs.perm_rap(n)
        return d, t, perm_rap_build(c_term="two"), None, 2, 7
    if plant == "aux_dyn_value":         # the callback's q[n-1] is one off
        d, t, b = airs.perm_rap(n, dyn_last_q=True)

        def wrong(rand, values):
            out = b.values_fn(rand, values)
            out[3, 0] = (int(out[3, 0]) + 1) % P
            return out
        return d, t, ab.perm_rap_build(), wrong, 2, b.num_values
    from test_trace_validate_oracle import cycled, redeclared
    if plant == "degree_low":
        d, t = airs.mulfib2(n)
        return redeclared(lambda: d, [(1, []), (2, [])]), t, None, None, 0, 0
    if plant == "degree_high":
        d, t = airs.fib_small_x(1, n)
        return redeclared(lambda: d, [(1, []), (2, [])]), t, None, None, 0, 0
    if plant == "cycled":
        d, t = cycled(n, 4)
        return d, t, None, None, 0, 0
    if plant == "periodic_mix":
        d, t = airs.periodic_mix(n)
        return d, t, None, None, 0, 0
    if plant == "aux_degree_straddle":   # aux constraint 1 declared (3, [4]) instead of (2, [4]); its columns 6, 7, 8
        d, t, _ = perm_rap_wide(n, (3, [4]))
        return d, t, ab.perm_rap_build(), None, 2, 7
    raise ValueError(plant)


# the violations, with what the whole-trace check must report first: (check, kind, index, step or None, where)
#   where: "rank:last_owner" (the column's owner is the last rank that owns columns), "ranks" (failures on rank 0 and the last
#   rank), "edge-1" / "edge" / "0" / "last" (the step), "exempt", "degrees"
PLANTS = {
    "assert_last_rank": ("trace", R.MAIN_ASSERTION, 2, None, "rank:last_owner"),
    "asserts_two_ranks": ("trace", R.MAIN_ASSERTION, 1, 0, "ranks"),
    "sequence_two_steps": ("trace", R.MAIN_ASSERTION, 3, None, "steps"),
    "main_transition": ("trace", R.MAIN_TRANSITION, 2, "at", "at"),
    "exempt_rows": ("trace", R.VALID, 0, None, "exempt"),
    "two_ranks": ("trace", R.MAIN_TRANSITION, 4, 1, "ranks"),
    "main_and_aux_same_step": ("trace", R.MAIN_TRANSITION, 1, "at", "at"),
    "degree_low": ("degrees", R.DEGREES, 0, None, "degrees"),
    "degree_high": ("degrees", R.DEGREES, 0, None, "degrees"),
    "cycled": ("degrees", R.DEGREES, 0, None, "degrees"),
    "periodic_mix": ("degrees", R.DEGREES, 0, None, "degrees"),
    "aux_degree_straddle": ("degrees", R.DEGREES, 0, None, "straddle"),
}
