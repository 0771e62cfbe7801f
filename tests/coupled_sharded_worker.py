"""One rank of the sharded proofs of the example AIR of tests/coupled_airs.py (tests/test_gpu_aux_coupled.py): the ranks, cases
and checks of tests/sharded_air_worker.py, with the AIR "coupled" added to the ones it knows, and a case key "validation" that
turns the provers' trace checks on for the case (the sharded proof and the one-GPU proof it is compared with)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sharded_air_worker as w  # noqa: E402

_air_of = w.air_of
_run_case = w.run_case


def run_case(ctx, comm, case, rank, world):
    ctx.set_validation(case.get("validation", 0))
    try:
        return _run_case(ctx, comm, case, rank, world)
    finally:
        ctx.set_validation(0)


def air_of(case, n):
    if case["air"] == "coupled":
        import coupled_airs as ca
        desc, tr, build, _ = ca.coupled(n)
        return desc, tr, build, None, ca.COUPLED_NUM_RANDS, 0
    return _air_of(case, n)


w.air_of = air_of
w.run_case = run_case

if __name__ == "__main__":
    w.main()
