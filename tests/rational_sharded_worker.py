"""One rank of the sharded proofs of the example AIR of tests/rational_airs.py (tests/test_gpu_aux_rational.py): the ranks, cases
and checks of tests/sharded_air_worker.py, with the AIR "rational" added to the ones it knows."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sharded_air_worker as w  # noqa: E402

_air_of = w.air_of


def air_of(case, n):
    if case["air"] == "rational":
        import rational_airs as ra
        desc, tr, build, _ = ra.rational(n)
        return desc, tr, build, None, ra.RATIONAL_NUM_RANDS, 0
    return _air_of(case, n)


w.air_of = air_of

if __name__ == "__main__":
    w.main()
