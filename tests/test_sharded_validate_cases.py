"""The planted violations of the sharded trace-check GPU test (tests/sharded_validate_cases.py), on the CPU: the whole-trace
restatement of the reference's checks (tests/trace_validate_ref.py) reports the intended first violation, and it sits where
the case says at every world size: on a shard boundary, on the intended rank, or in columns that straddle two ranks' blocks.
This is what makes the GPU cases exercise the shard edges."""
import numpy as np
import pytest

import aux_builds as ab
import sharded_validate_cases as S
import trace_validate_ref as R

LOG_N = 10
WORLDS = (2, 4, 8)


def owner(col, width, world):
    """the rank whose column block holds `col` (wf_shard_columns: whole 8-column segments, the first ranks one more)"""
    segs = (width + 7) // 8
    base, extra = divmod(segs, world)
    starts = [r * base + min(r, extra) for r in range(world + 1)]
    return max(r for r in range(world) if starts[r] <= col // 8)


def last_owner(width, world):
    return min((width + 7) // 8, world) - 1


def reports(case, world, ext=3):
    n = 1 << LOG_N
    desc, tr, build, _, _, _ = S.make(case, n, world)
    aux = rand = None
    if build is not None:
        from oracle import oracle as O
        rand = O.rand_elems((2, ext), 9)
        aux = ab.reference(desc, build, tr, rand)
    return desc, tr, aux, rand, R.check_trace(desc, tr, aux, rand, ext)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("at", ["0", "edge-1", "edge", "last"])
def test_main_transition_lands_on_the_shard_edge(oracle, world, at):
    n, nt = 1 << LOG_N, (1 << LOG_N) // world
    _, _, _, _, rep = reports({"plant": "main_transition", "at": at}, world)
    s = S.step_of(at, n, world)
    assert (rep["kind"], rep["index"], rep["step"]) == (R.MAIN_TRANSITION, 2, s)
    rank = s // nt
    if at == "0":
        assert rank == 0
    elif at == "edge-1":   # the last step of rank 0: its next row is rank 1's first row, the halo row
        assert rank == 0 and (s + 1) % nt == 0
    elif at == "edge":     # the first step of rank 1
        assert rank == 1 and s % nt == 0
    else:                  # the last checked step, on the last rank
        assert rank == world - 1 and s == n - 2


@pytest.mark.parametrize("world", WORLDS)
def test_assertion_on_the_last_owning_rank(oracle, world):
    desc, tr, _, _, rep = reports({"plant": "assert_last_rank"}, world)
    assert (rep["kind"], rep["index"], rep["step"], rep["column"]) == (R.MAIN_ASSERTION, 2, (1 << LOG_N) - 1, 31)
    assert owner(31, tr.shape[0], world) == last_owner(tr.shape[0], world) > 0


@pytest.mark.parametrize("world", WORLDS)
def test_two_assertions_higher_rank_owns_the_lower_index(oracle, world):
    desc, tr, _, _, rep = reports({"plant": "asserts_two_ranks"}, world)
    assert (rep["kind"], rep["index"], rep["step"], rep["column"]) == (R.MAIN_ASSERTION, 1, 0, 31)
    A = R.Air(desc)
    assert A.asserts[45][:2] == (0, 0) and A.asserts[1][:2] == (31, 0)
    assert owner(0, tr.shape[0], world) == 0 < owner(31, tr.shape[0], world)
    # without column 31's failure, column 0's assertion (the highest index planted) is the one reported
    t = tr.copy()
    S.bump(t, 31, 0, -1)
    assert R.check_trace(desc, t)["index"] == 45


def test_sequence_assertion_failing_at_two_steps(oracle):
    desc, tr, _, _, rep = reports({"plant": "sequence_two_steps"}, 2)
    assert (rep["kind"], rep["index"], rep["step"], rep["column"]) == (R.MAIN_ASSERTION, 3, 13, 0)


def test_changed_cells_on_exempt_rows_pass(oracle):
    desc, tr, _, _, rep = reports({"plant": "exempt_rows"}, 2)
    assert rep["kind"] == R.VALID
    assert R.check_degrees(desc, tr)[2] == R.VALID
    assert (tr != S.fib_exempt2(1 << LOG_N)[1]).sum() == 2


@pytest.mark.parametrize("world", WORLDS)
def test_failures_on_two_ranks(oracle, world):
    n, nt = 1 << LOG_N, (1 << LOG_N) // world
    _, _, _, _, rep = reports({"plant": "two_ranks"}, world)
    assert (rep["kind"], rep["index"], rep["step"]) == (R.MAIN_TRANSITION, 4, 1)
    ff = rep["first_failing_step"]
    assert ff[4] // nt == 0 and ff[2] // nt == world - 1 and ff[2] == (world - 1) * nt


@pytest.mark.parametrize("world", WORLDS)
def test_main_and_aux_failing_at_the_same_step(oracle, world):
    n = 1 << LOG_N
    desc, _, _, _, rep = reports({"plant": "main_and_aux_same_step", "at": "edge-1"}, world)
    s = S.step_of("edge-1", n, world)
    assert (rep["kind"], rep["index"], rep["step"]) == (R.MAIN_TRANSITION, 1, s)
    n_mtr = len(R.Air(desc).degrees)
    assert rep["first_failing_step"][n_mtr + 2] == s   # the aux counter, through the gated build term, at the same step
    assert rep["first_failing_step"][1] == s


@pytest.mark.parametrize("plant", ["degree_low", "degree_high", "cycled", "periodic_mix", "aux_degree_straddle"])
def test_degree_cases(oracle, plant):
    ext = 3
    desc, tr, aux, rand, rep = reports({"plant": plant}, 2, ext)
    assert rep["kind"] == R.VALID, rep["msg"]
    e, a, kind, msg = R.check_degrees(desc, tr, aux, rand, ext)
    assert kind == R.DEGREES and msg.startswith("transition constraint degrees didn't match")
    if plant == "aux_degree_straddle":
        A = R.Air(desc)
        n_mtr = len(A.degrees)
        wrong = [j for j in range(len(e)) if e[j] != a[j]]
        assert wrong == [n_mtr + 1]
        cols = [n_mtr + ext + q for q in range(ext)]   # aux constraint 1's columns in the degree check
        ncols = n_mtr + len(A.aux_degrees) * ext
        for world in WORLDS:
            assert owner(cols[0], ncols, world) == 0 and owner(cols[-1], ncols, world) == 1
        # the valid declaration passes
        d2, t2, _ = S.perm_rap_wide(1 << LOG_N)
        assert R.check_degrees(d2, t2, aux, rand, ext)[2] == R.VALID


def test_fixtures_of_the_valid_cases_pass_both_checks(oracle):
    n = 1 << LOG_N
    for case in ({"air": "fib_small_x", "k": 8}, {"air": "fib_small_x", "k": 10}, {"air": "fib_small_x", "k": 16}, {"air": "mulfib2"},
                 {"air": "sequence_mix"}, {"air": "rescue_like"}):
        desc, tr, _, _, _, _ = S.make(case, n, 2)
        assert R.validate(desc, tr)["kind"] == R.VALID, case
    desc, tr, build, _, _, _ = S.make({"air": "perm_rap"}, n, 2)
    from oracle import oracle as O
    rand = O.rand_elems((2, 3), 9)
    assert R.validate(desc, tr, ab.reference(desc, build, tr, rand), rand, 3)["kind"] == R.VALID
    assert np.array_equal(S.perm_rap_build(), ab.perm_rap_build())
