"""Cases of the standalone sharded trace check, wf_trace_validate_sharded (tests/sharded_trace_validate_worker.py and
tests/test_sharded_trace_validate_cases.py), on top of the planted violations of tests/sharded_validate_cases.py. Unlike
the prover, the validator reports every constraint's first failing step and the degrees even when a check fails, so these
cases aim at what only that report shows:
  * "ranks_first_fail": three constraints whose first failures sit on three different ranks (the last, rank 1 and rank 0),
    so every entry of first_failing_step comes from a different rank's share and only their minimum gives the report;
  * "last_step_only": a transition that fails on the last checked step, n - exemptions - 1, and nowhere else;
  * "violation_with_degrees": a failing transition in an AIR whose declared degrees are also wrong: the report names the
    transition and still carries the expected and actual degrees.
`make` gives (description, trace, aux build, values_fn, num_rands, num_values), as sharded_validate_cases.make; `aux_of`
gives the host aux columns of a two-segment case (the CPU reference of its build)."""
import numpy as np

import airs
import sharded_validate_cases as S

# the new violations, as sharded_validate_cases.PLANTS: (check, kind, index, step or None, where)
import trace_validate_ref as R

PLANTS = {
    "ranks_first_fail": ("trace", R.MAIN_TRANSITION, 6, 2, "ranks"),
    "last_step_only": ("trace", R.MAIN_TRANSITION, 2, "last", "last"),
    "violation_with_degrees": ("trace", R.MAIN_TRANSITION, 0, 3, "degrees"),
}


def ranks_first_fail_steps(n, world):
    """the steps at which FibSmall x 8's constraints 2, 4 and 6 first fail: on the last rank, rank 1 and rank 0"""
    nt = n // world
    return {2: (world - 1) * nt + 5, 4: nt + 3, 6: 2}


def make(case, n, world):
    plant = case.get("plant")
    if plant == "ranks_first_fail":     # x_c at row s + 1 breaks constraint c first at step s (and c + 1 with it)
        d, t = airs.fib_small_x(8, n)
        t = t.copy()
        for c, s in ranks_first_fail_steps(n, world).items():
            S.bump(t, c, s + 1)
        return d, t, None, None, 0, 0
    if plant == "last_step_only":       # row n - 1 of x2: only step n - 2 reads it as a next row; step n - 1 is exempt
        d, t = airs.fib_small_x(4, n)
        t = t.copy()
        S.bump(t, 2, n - 1)
        return d, t, None, None, 0, 0
    if plant == "violation_with_degrees":   # mulfib2 declared (1, 2) instead of its degrees, and x0 wrong at row 4
        from test_trace_validate_oracle import redeclared
        d, t = airs.mulfib2(n)
        t = t.copy()
        S.bump(t, 0, 4)
        return redeclared(lambda: d, [(1, []), (2, [])]), t, None, None, 0, 0
    if case.get("air") in ("linrec", "rational", "coupled"):
        mod = __import__(case["air"] + "_airs")
        desc, tr, build, _ = getattr(mod, case["air"])(n)
        return desc, tr, build, None, getattr(mod, case["air"].upper() + "_NUM_RANDS"), 0
    return S.make(case, n, world)


def aux_of(case, desc, tr, build, rand):
    """the aux segment [aw, n, ext] the build gives for these random elements (the CPU reference of each build kind)"""
    air = case.get("air")
    if air in ("linrec", "rational", "coupled"):
        mod = __import__(air + "_airs")
        return np.ascontiguousarray(getattr(mod, air)(tr.shape[1])[3](rand), dtype=np.uint64)
    import aux_builds as ab
    return np.ascontiguousarray(ab.reference(desc, build, tr, rand), dtype=np.uint64)
