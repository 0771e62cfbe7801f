"""Regenerates tests/golden/invalid_proof_digests.json: SHA-256 and length of the proofs the DEVICE prover emits for traces that
do not satisfy their AIR (one cell of a valid trace changed). For such a trace the constraint evaluations are not those of a
polynomial of degree < kc * n, so the composition polynomial depends on which CE rows it is interpolated from: the prover
interpolates it from the rows of the sub-coset 7 <w_m> (m = the power of two >= kc * n), where the reference's size-ce
transform would keep the low coefficients of all ce rows. These fixtures pin that choice, and with it the bytes the prover
gave before it stopped evaluating the CE rows outside the sub-coset. Needs a GPU.
    python tests/golden/make_invalid_proof_digests.py [OUT.json]        (from the repository root)"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import airs  # noqa: E402
from oracle import oracle as O  # noqa: E402  (trace builder and options only: the proofs are the device's)

CASES = [  # kind, name / k, log2 n, options, (column, step) of the changed cell
    ("fib", 1, 7, dict(num_queries=28, blowup=8, grinding=0, ext=1, folding=4, rem_max_deg=7, hash_id=1), (1, 40)),
    ("fib", 4, 10, dict(num_queries=32, blowup=8, grinding=4, ext=3, folding=4, rem_max_deg=31, hash_id=0), (5, 1023)),
    ("fib", 32, 12, dict(num_queries=32, blowup=8, grinding=0, ext=3, folding=4, rem_max_deg=31, batch_c=2, batch_d=2, hash_id=0), (63, 0)),
    ("fib", 2, 8, dict(num_queries=20, blowup=16, grinding=0, ext=2, folding=8, rem_max_deg=15, hash_id=0), (0, 77)),
    ("air", "mulfib2", 8, dict(num_queries=24, blowup=8, grinding=2, ext=1, folding=4, rem_max_deg=15, hash_id=0), (1, 100)),
    ("air", "periodic_mix", 9, dict(num_queries=24, blowup=8, grinding=2, ext=3, folding=4, rem_max_deg=15, batch_c=1, batch_d=1,
                                    hash_id=0), (1, 3)),
    ("air", "sequence_mix", 8, dict(num_queries=20, blowup=8, grinding=1, ext=2, folding=4, rem_max_deg=7, hash_id=0), (0, 255)),
]


def prove(ctx, case):
    """the device proof of the case's trace with its one changed cell"""
    kind, name, log_n, kw, (col, step) = case
    n = 1 << log_n
    if kind == "fib":
        trace, res = O.build_fib_trace(name, n)
    else:
        desc, trace = getattr(airs, name)(n)
    trace = trace.copy()
    trace[col, step] = (int(trace[col, step]) + 1) % airs.P
    opts = O.make_opts(**kw)
    return ctx.prove_fib(trace, res, opts) if kind == "fib" else ctx.prove_air(desc, trace, opts)


if __name__ == "__main__":
    import winterfell_b200 as wf
    ctx = wf.Context(0)
    recs = []
    for case in CASES:
        proof = prove(ctx, case)
        kind, name, log_n, kw, cell = case
        recs.append({"kind": kind, "name": name, "log_n": log_n, "opts": kw, "cell": list(cell), "bytes": len(proof),
                     "sha256": hashlib.sha256(proof).hexdigest()})
    ctx.close()
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "invalid_proof_digests.json")
    with open(out, "w") as f:
        json.dump(recs, f, indent=1)
    print(f"wrote {len(recs)} digests to {out}")
