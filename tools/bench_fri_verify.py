"""Times wf_fri_verify_batch on the FRI-only sweep's shapes (BASELINE configs[4]: codewords of 2^20, 2^22, 2^24 and 2^26 points,
blowup 8, folding 4, remainder max degree 31, 32 queries, Blake3_256), in the base field and the cubic extension, plus Rp64_256
at 2^22, for B in {1, 16, 256, 1024} proofs per call. The proofs come from the device prover's default channel
(wf_fri_build_layers_default_channel + wf_fri_build_proof at draw_query_positions(0)). Per batch: wall ms (host clock around
the call, which ends in a synchronise), the host part against the device part (the library's stage events), launches,
proofs/s, verdict parity with the CPU restatement's wfr_fri_verify (tests/fri_ref.cpp) on every distinct proof, and
wfr_fri_verify in a loop ("C++ restatement, 1 thread"). One JSON line per (shape, B), to stdout and to --out; the card's name,
power limit and max SM clock are read in the same run. Run on an H100: python tools/bench_fri_verify.py --out /tmp/bench_fri_verify.jsonl"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import winterfell_b200 as wf  # noqa: E402
from fri_cases import default_positions, fri_verify  # noqa: E402
from oracle import oracle as O  # noqa: E402

SHAPES = [("blake3_256", wf.HASH_BLAKE3_256, lg, d) for lg in (20, 22, 24, 26) for d in (1, 3)] + [("rp64_256", wf.HASH_RP64_256, 22, 1),
                                                                                                   ("rp64_256", wf.HASH_RP64_256, 22, 3)]
FOLD, REM, BLOWUP, QUERIES = 4, 31, 8, 32


def make_proof(ctx, h, log_len, d, seed):
    """A proof of a random polynomial of degree < L / 8 over 2^log_len points: (proof, commitments, positions, evaluations)"""
    L = 1 << log_len
    poly = np.random.default_rng(seed).integers(0, wf.P, size=(d, L // BLOWUP), dtype=np.uint64)
    m = ctx.mat_from_host_columns(poly)
    cw = m.lde(3)
    f, roots = ctx.fri_build_layers_default(h, cw, d, FOLD, REM, BLOWUP)
    pos = default_positions(h, roots, d, L, QUERIES)
    proof = f.build_proof(pos)
    ev = cw.read_rows([int(p) for p in pos]).reshape(-1, d)
    for x in (f, m, cw):
        x.free()
    return proof, roots, pos, np.ascontiguousarray(ev, dtype=np.uint64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batches", default="1,16,256,1024")
    ap.add_argument("--distinct", type=int, default=2, help="distinct proofs per shape; a batch repeats them")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    O.set_threads(1)
    ctx = wf.Context(0)
    lines = []
    for hname, h, log_len, d in SHAPES:
        L = 1 << log_len
        max_deg = L // BLOWUP - 1
        proofs = [make_proof(ctx, h, log_len, d, 7 * log_len + 31 * j + d) for j in range(a.distinct)]
        oracle_v = [fri_verify(h, d, FOLD, REM, BLOWUP, max_deg, p, cm, pos, ev) for p, cm, pos, ev in proofs]
        assert oracle_v == [0] * a.distinct
        t = time.perf_counter()
        for p, cm, pos, ev in proofs:
            fri_verify(h, d, FOLD, REM, BLOWUP, max_deg, p, cm, pos, ev)
        cpu_ms = (time.perf_counter() - t) * 1e3 / a.distinct
        for B in [int(x) for x in a.batches.split(",")]:
            sel = [proofs[j % a.distinct] for j in range(B)]
            args = (h, d, FOLD, REM, BLOWUP, max_deg, [s[0] for s in sel], [s[1] for s in sel], [s[2] for s in sel], [s[3] for s in sel])
            ctx.fri_verify_batch(*args)    # warm-up
            ts, split, launches = [], None, None
            for _ in range(a.reps):
                ctx.set_profiling(1)
                l0 = ctx.launches
                t = time.perf_counter()
                v = ctx.fri_verify_batch(*args)
                ts.append((time.perf_counter() - t) * 1e3)
                launches = ctx.launches - l0
                split = dict(ctx.stage_times())
                ctx.set_profiling(0)
                assert v == [oracle_v[j % a.distinct] for j in range(B)]
            best = min(ts)
            row = {"hash": hname, "log_len": log_len, "ext": d, "folding": FOLD, "rem_max_deg": REM, "queries": QUERIES,
                   "proof_bytes": len(proofs[0][0]), "batch": B, "wall_ms": round(best, 3), "wall_ms_all": [round(x, 3) for x in ts],
                   "host_ms": round(split.get("verify_host", float("nan")), 3),
                   "device_ms": round(split.get("verify_device", float("nan")), 3), "launches": launches,
                   "proofs_per_s": round(B / best * 1e3, 1), "parity": "all verdicts equal the C++ restatement's",
                   "cpu_ms_per_proof": round(cpu_ms, 3), "cpu": f"C++ restatement, 1 thread, {os.cpu_count()} cores on the host",
                   "gpu": gpu}
            print(json.dumps(row), flush=True)
            lines.append(row)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
