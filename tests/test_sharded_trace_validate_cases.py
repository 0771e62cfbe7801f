"""The new cases of the standalone sharded trace check (tests/sharded_trace_validate_cases.py), on the CPU: the whole-trace
restatement of the reference's checks (tests/trace_validate_ref.py) gives the report each case names, and the failures sit
where the case says at every world size, so that the GPU test's comparison with the one-GPU validator exercises the
min-combine of the ranks' first failing steps, the last checked step and the degree report of a failing trace."""
import pytest

import sharded_trace_validate_cases as T
import trace_validate_ref as R

LOG_N = 10
WORLDS = (2, 4, 8)


def report(case, world):
    n = 1 << LOG_N
    desc, tr, build, _, _, _ = T.make(case, n, world)
    assert build is None
    return desc, tr, R.validate(desc, tr)


@pytest.mark.parametrize("world", WORLDS)
def test_first_failures_on_three_ranks(oracle, world):
    n, nt = 1 << LOG_N, (1 << LOG_N) // world
    desc, _, rep = report({"plant": "ranks_first_fail"}, world)
    steps = T.ranks_first_fail_steps(n, world)
    ff = rep["first_failing_step"]
    assert (rep["kind"], rep["index"], rep["step"]) == (R.MAIN_TRANSITION, 6, steps[6])
    for c, s in steps.items():
        assert ff[c] == s and ff[c + 1] == s   # x_c' is wrong in both constraints of its pair at step s
    assert [steps[c] // nt for c in (2, 4, 6)] == [world - 1, 1, 0]
    # the first failures lie in different ranks' shares (three ranks, two at world 2, where rank 1 is the last), so no
    # single rank's results give first_failing_step
    assert len({ff[c] // nt for c in (2, 4, 6)}) == min(3, world)


@pytest.mark.parametrize("world", WORLDS)
def test_failure_only_on_the_last_checked_step(oracle, world):
    n = 1 << LOG_N
    desc, _, rep = report({"plant": "last_step_only"}, world)
    s = n - R.Air(desc).exemptions - 1
    assert (rep["kind"], rep["index"], rep["step"]) == (R.MAIN_TRANSITION, 2, s)
    assert {v for v in rep["first_failing_step"] if v is not None} == {s}
    assert s // (n // world) == world - 1   # on the last rank, whose next row is its own last row, not a halo row


@pytest.mark.parametrize("world", WORLDS)
def test_failing_trace_keeps_its_degree_report(oracle, world):
    desc, tr, rep = report({"plant": "violation_with_degrees"}, world)
    _, kind, index, step, _ = T.PLANTS["violation_with_degrees"]
    assert (rep["kind"], rep["index"], rep["step"]) == (kind, index, step)
    assert rep["msg"] == f"main transition constraint {index} did not evaluate to ZERO at step {step}"
    e, a = rep["expected_degrees"], rep["actual_degrees"]
    assert e is not None and a is not None and e != a   # the degree check ran and disagrees, but the trace check's report stands
    assert R.check_degrees(desc, tr)[2] == R.DEGREES


def test_plants_table_matches_the_reports(oracle):
    for plant, (_, kind, index, step, _) in T.PLANTS.items():
        n = 1 << LOG_N
        _, _, rep = report({"plant": plant}, 2)
        want = n - 2 if step == "last" else step
        assert (rep["kind"], rep["index"], rep["step"]) == (kind, index, want), plant
