"""CPU tests of the trace checks' restatement (tests/trace_validate_ref.py), which the GPU tests compare wf_trace_validate
with: valid fixtures pass, and planted violations are reported where changing one cell must make the reference panic first
(derived from the constraint each fixture states, not from the evaluator)."""
import numpy as np
import pytest

import airs
import trace_validate_ref as R
from airs import P

N = 32


def fixtures(n=N, ext=2):
    """(name, desc, trace, aux, rand) of every fixture of tests/airs.py with its valid trace."""
    from oracle import oracle as O
    out = [("fib_small_x2", *airs.fib_small_x(2, n), None, None), ("mulfib2", *airs.mulfib2(n), None, None),
           ("periodic_mix", *airs.periodic_mix(n), None, None), ("sequence_mix", *airs.sequence_mix(n), None, None),
           ("rescue_like", *airs.rescue_like(n), None, None)]
    desc, tr, builder = airs.perm_rap(n)
    rand = O.rand_elems((2, ext), 77)
    out.append(("perm_rap", desc, tr, builder(rand), rand))
    return out


@pytest.mark.parametrize("i", range(6))
def test_valid_fixtures_pass_the_trace_check(oracle, i):
    name, desc, tr, aux, rand = fixtures()[i]
    rep = R.check_trace(desc, tr, aux, rand, 2)
    assert rep["kind"] == R.VALID, (name, rep["msg"])
    assert all(s is None for s in rep["first_failing_step"])


def planted(n=N):
    """(name, desc, trace, aux, rand, expected (kind, index, step, column)) for one or two changed cells."""
    from oracle import oracle as O
    cases = []
    d, t = airs.fib_small_x(2, n)
    t1 = t.copy(); t1[3, n - 1] = 5      # the last-step assertion of pair 1 (assertion 5); transitions hold: row n-1 only
    cases.append(("main_single", d, t1, None, None, (R.MAIN_ASSERTION, 5, n - 1, 3)))   # enters constraint 3 at step n-2
    d, t = airs.periodic_mix(n)
    t1 = t.copy(); t1[2, 16] = 0         # flag at step 2 * cycle: the periodic assertion (assertion 2)
    cases.append(("main_periodic", d, t1, None, None, (R.MAIN_ASSERTION, 2, 16, 2)))
    d, t = airs.sequence_mix(n)
    t1 = t.copy(); t1[0, 1 + 3 * 4] = (int(t[0, 13]) + 1) % P   # value 3 of the sequence assertion on column 0 (assertion 3)
    cases.append(("main_sequence", d, t1, None, None, (R.MAIN_ASSERTION, 3, 13, 0)))
    d, t = airs.fib_small_x(2, n)
    t1 = t.copy(); t1[2, 9] = (int(t[2, 9]) + 1) % P   # x2' = x2 + x3 fails at step 8 (constraint 2), x3' = x3 + x2' too
    cases.append(("main_transition", d, t1, None, None, (R.MAIN_TRANSITION, 2, 8, 0)))
    d, t = airs.periodic_mix(n)
    t1 = t.copy(); t1[2, n - 1] = 5; t1[2, n - 2] = 6   # flag * (flag - 1) at steps n-2 and n-1: both exempt (2 exemptions)
    cases.append(("exempt_rows", d, t1, None, None, (R.VALID, 0, 0, 0)))
    d, t = airs.fib_small_x(2, n)
    t1 = t.copy(); t1[2, 9] = 1; t1[1, 0] = 7         # a transition at step 8 and an assertion: the assertion first
    cases.append(("two_assertion_first", d, t1, None, None, (R.MAIN_ASSERTION, 1, 0, 1)))
    d, tr, builder = airs.perm_rap(n)
    rand = O.rand_elems((2, 2), 5)
    aux = builder(rand)
    a1 = aux.copy(); a1[1, 0, 1] = 3     # q[0] = 0 (aux assertion 2); enters the aux transitions at step 0 as well
    cases.append(("aux_single", d, tr, a1, rand, (R.AUX_ASSERTION, 2, 0, 1)))
    a1 = aux.copy(); a1[2, 1 + n // 4, 0] = 1   # c at the sequence's second step (aux assertion 3)
    cases.append(("aux_sequence", d, tr, a1, rand, (R.AUX_ASSERTION, 3, 1 + n // 4, 2)))
    a1 = aux.copy(); a1[2, 3, 0] = 1     # c' = c + 1 fails at steps 2 and 3 (aux constraint 2)
    cases.append(("aux_transition", d, tr, a1, rand, (R.AUX_TRANSITION, 2, 2, 0)))
    t1 = tr.copy(); t1[0, 6] = 1         # x0 feeds main constraint 0 at step 5 and the running product at step 6; aux c at step 2
    a1 = aux.copy(); a1[2, 3, 0] = 1
    cases.append(("two_aux_earlier", d, t1, a1, rand, (R.AUX_TRANSITION, 2, 2, 0)))
    a1 = aux.copy(); a1[2, 6, 0] = 1     # aux constraint 2 fails at step 5 too: main comes first within a step
    cases.append(("two_same_step", d, t1, a1, rand, (R.MAIN_TRANSITION, 0, 5, 0)))
    return cases


@pytest.mark.parametrize("i", range(11))
def test_planted_violation_is_reported_first(oracle, i):
    name, desc, tr, aux, rand, want = planted()[i]
    rep = R.check_trace(desc, tr, aux, rand, 2)
    assert (rep["kind"], rep["index"], rep["step"], rep["column"]) == want, (name, rep["msg"])


def test_messages_use_the_reference_wording(oracle):
    _, d, t, _, _, _ = planted()[0]
    want = int(airs.fib_small_x(2, N)[1][3, N - 1])
    assert R.check_trace(d, t)["msg"] == f"trace does not satisfy assertion main_trace(3, {N - 1}) == {want}"
    _, d, t, _, _, _ = planted()[3]
    assert R.check_trace(d, t)["msg"] == "main transition constraint 2 did not evaluate to ZERO at step 8"


def redeclared(desc_fn, degrees):
    """The description of desc_fn() with its main constraint degrees replaced (same program)."""
    d = [int(v) for v in desc_fn()]
    A = R.Air(d)
    out = [d[0], len(degrees)]
    for base, cyc in degrees:
        out += [base, len(cyc)] + list(cyc)
    skip = 2 + sum(2 + len(c) for _, c in A.degrees)
    return np.array(out + d[skip:], dtype=np.uint64)


def test_fib_small_passes_the_degree_check(oracle):
    d, t = airs.fib_small_x(1, 64)
    e, a, kind, _ = R.check_degrees(d, t)
    assert kind == R.VALID and e == a == [0, 0]


def test_degree_declared_too_low_and_too_high(oracle):
    n = 64
    d, t = airs.mulfib2(n)
    low = redeclared(lambda: d, [(1, []), (2, [])])
    e, a, kind, msg = R.check_degrees(low, t)
    assert kind == R.DEGREES and e == [0, n - 1] and a == [n - 1, n - 1]
    assert msg == f"transition constraint degrees didn't match\nexpected: [  0, {n - 1:>3}]\nactual:   [{n - 1:>3}, {n - 1:>3}]"
    d, t = airs.fib_small_x(1, n)
    high = redeclared(lambda: d, [(1, []), (2, [])])
    e, a, kind, _ = R.check_degrees(high, t)
    assert kind == R.DEGREES and e == [0, n - 1] and a == [0, 0]


def cycled(n, declared_cycle, true_cycle=8):
    """s0' = s0 * k0 with k0 periodic of length true_cycle, declared with a cycle of declared_cycle."""
    A = airs.AirBuilder(1)
    A.periodic = [[(3 * i + 2) % P for i in range(true_cycle)]]
    A.constraint(A.sub(A.nxt(0), A.mul(A.cur(0), A.per(0))), 1, [declared_cycle])
    t = np.zeros((1, n), dtype=np.uint64)
    v = 1
    for i in range(n):
        t[0, i] = v
        v = v * A.periodic[0][i % true_cycle] % P
    A.assert_single(0, 0, 1)
    return A.build(), t


def test_wrong_periodic_cycle(oracle):
    n = 64
    d, t = cycled(n, 8)
    e, a, kind, _ = R.check_degrees(d, t)
    assert kind == R.VALID and e == a == [n // 8 * 7]
    d, t = cycled(n, 4)
    e, a, kind, _ = R.check_degrees(d, t)
    assert kind == R.DEGREES and e == [n // 4 * 3] and a == [n // 8 * 7]


def test_periodic_mix_overdeclares_two_constraints(oracle):
    # Constraint 1 declares a cycle-4 factor although k1 enters only additively, and flag * (flag - 1) vanishes on more of
    # the domain than a degree-2 constraint would: the reference's debug build refuses this fixture as well.
    n, cyc = 64, 8
    d, t = airs.periodic_mix(n, cyc)
    e, a, kind, _ = R.check_degrees(d, t)
    assert kind == R.DEGREES
    assert e[1] == 3 * (n - 1) + 3 * n // 4 - (n - 2) and a[1] == 3 * (n - 1) - (n - 2)
    assert e[2] == n and a[2] == n - 2 * n // cyc + 2
    assert e[0] == a[0]
