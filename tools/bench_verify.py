"""Times wf_verify_air_batch on the cfg1 shape (fib_small, 2^16 rows, base field, 28 queries, blowup 8, folding 8, remainder
31, grinding 16) with Blake3_256 and with Rp64_256, for B in {1, 16, 256, 1024} proofs per call. Per batch: wall ms (host
clock around the call, which ends in a synchronise), the host part against the device part (the library's stage events),
launches, proofs/s, verdict parity with the oracle's verifier on every proof, and the oracle's CPU verifier on the same proofs
in a loop ("C++ restatement, 1 thread"). One JSON line per (hasher, B), to stdout and to --out; the card's name and power
limit are read in the same run. Run on an H100: python tools/bench_verify.py --out /tmp/bench_verify.jsonl

--security-arm times the three AcceptableOptions policies instead, at B in {1, 1024}: OptionSet (wf_verify_air_batch with the
proofs' own options as the set), MinConjecturedSecurity(95) and MinProvenSecurity(95) (wf_verify_air_batch_min_security),
which refuse the cfg1 proofs (63 conjectured bits), and the two at the proofs' own estimate, which accept them and so run the
whole verifier behind the estimate.
Each line carries the policy, the verdicts it gave and the host time of one security estimate (wf_security_estimate, the
wf_proof_security: the context read and the m search, through ctypes)."""
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

import airs  # noqa: E402
import winterfell_b200 as wf  # noqa: E402
from oracle import oracle as O  # noqa: E402

P = wf.P


def fib_pair(n, a0, b0):
    """fib_small from (a0, b0): one AIR structure, different assertion values and public result per proof"""
    tr = np.zeros((2, n), dtype=np.uint64)
    a, b = a0, b0
    for i in range(n):
        tr[0, i], tr[1, i] = a, b
        a = (a + b) % P
        b = (b + a) % P
    A = airs.AirBuilder(2)
    A.pub = [int(tr[1, n - 1])]
    A.constraint(A.sub(A.nxt(0), A.add(A.cur(0), A.cur(1))), 1)
    A.constraint(A.sub(A.nxt(1), A.add(A.cur(1), A.nxt(0))), 1)
    A.assert_single(0, 0, a0)
    A.assert_single(1, 0, b0)
    A.assert_single(1, n - 1, int(tr[1, n - 1]))
    return A.build(), tr


def security_arm(a, ctx, hname, h, n, opts, descs, proofs, oracle_v, gpu):
    """host / device ms of one batch under each AcceptableOptions policy"""
    reps = 200
    t = time.perf_counter()
    for _ in range(reps):
        est = wf.proof_security(h, proofs[0])
    estimate_us = (time.perf_counter() - t) * 1e6 / reps
    def min_security(regime, bits):
        return lambda ds, ps: ctx.verify_air_batch_min_security(ds, ps, h, regime, bits)
    proven = max(est[1], est[2])
    policies = [("OptionSet", lambda ds, ps: (ctx.verify_air_batch(ds, ps, h, acceptable=[opts]), None)),
                (f"MinConjecturedSecurity({a.min_bits})", min_security(wf.SECURITY_CONJECTURED, a.min_bits)),
                (f"MinProvenSecurity({a.min_bits})", min_security(wf.SECURITY_PROVEN, a.min_bits)),
                (f"MinConjecturedSecurity({est[0]})", min_security(wf.SECURITY_CONJECTURED, est[0])),
                (f"MinProvenSecurity({proven})", min_security(wf.SECURITY_PROVEN, proven))]
    rows = []
    for B in [int(x) for x in a.batches.split(",")]:
        ds = [descs[j % a.distinct] for j in range(B)]
        ps = [proofs[j % a.distinct] for j in range(B)]
        for name, run in policies:
            run(ds, ps)    # warm-up
            ts, hosts, split = [], [], None
            for _ in range(a.reps):
                ctx.set_profiling(1)
                l0 = ctx.launches
                t = time.perf_counter()
                v, bits = run(ds, ps)
                ts.append((time.perf_counter() - t) * 1e3)
                launches = ctx.launches - l0
                split = dict(ctx.stage_times())
                hosts.append(split.get("verify_host", float("nan")))
                ctx.set_profiling(0)
            codes = sorted(set(int(x) for x in v))
            if codes == [0]:
                assert list(v) == [oracle_v[j % a.distinct] for j in range(B)]
            row = {"hash": hname, "rows": n, "batch": B, "policy": name, "verdicts": codes,
                   "security_bits": None if bits is None else int(bits[0]), "estimate": {"conjectured": est[0], "ldr": est[1], "udr": est[2]},
                   "estimate_us": round(estimate_us, 2), "wall_ms": round(min(ts), 3), "host_ms": round(min(hosts), 3),
                   "host_ms_all": [round(x, 3) for x in hosts], "device_ms": round(split.get("verify_device", float("nan")), 3),
                   "launches": launches, "gpu": gpu}
            print(json.dumps(row), flush=True)
            rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batches", default="1,16,256,1024")
    ap.add_argument("--distinct", type=int, default=16, help="distinct proofs per hasher; a batch repeats them")
    ap.add_argument("--out", default=None)
    ap.add_argument("--security-arm", action="store_true", help="time the AcceptableOptions policies at B = 1 and 1024")
    ap.add_argument("--min-bits", type=int, default=95)
    a = ap.parse_args()
    if a.security_arm:
        a.batches = "1,1024"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ctx = wf.Context(0)
    n = 1 << 16
    lines = []
    for hname, h in (("blake3_256", wf.HASH_BLAKE3_256), ("rp64_256", wf.HASH_RP64_256)):
        opts = O.make_opts(num_queries=28, blowup=8, grinding=16, ext=1, folding=8, rem_max_deg=31, hash_id=h)
        inputs = [fib_pair(n, 1 + j, 2 + 3 * j) for j in range(a.distinct)]
        descs = [d for d, _ in inputs]
        proofs = ctx.prove_air_batch(descs, [t for _, t in inputs], opts)
        oracle_v = [O.verify_air(d, p, h) for d, p in zip(descs, proofs)]
        assert oracle_v == [0] * a.distinct
        t = time.perf_counter()
        for d, p in zip(descs, proofs):
            O.verify_air(d, p, h)
        cpu_ms = (time.perf_counter() - t) * 1e3 / a.distinct
        if a.security_arm:
            lines += security_arm(a, ctx, hname, h, n, opts, descs, proofs, oracle_v, gpu)
            continue
        for B in [int(x) for x in a.batches.split(",")]:
            ds = [descs[j % a.distinct] for j in range(B)]
            ps = [proofs[j % a.distinct] for j in range(B)]
            ctx.verify_air_batch(ds, ps, h)    # warm-up
            ts, split = [], None
            for _ in range(a.reps):
                ctx.set_profiling(1)
                l0 = ctx.launches
                t = time.perf_counter()
                v = ctx.verify_air_batch(ds, ps, h)
                ts.append((time.perf_counter() - t) * 1e3)
                launches = ctx.launches - l0
                split = dict(ctx.stage_times())
                ctx.set_profiling(0)
                assert list(v) == [oracle_v[j % a.distinct] for j in range(B)]
            best = min(ts)
            row = {"hash": hname, "rows": n, "batch": B, "wall_ms": round(best, 3), "wall_ms_all": [round(x, 3) for x in ts],
                   "host_ms": round(split.get("verify_host", float("nan")), 3),
                   "device_ms": round(split.get("verify_device", float("nan")), 3), "launches": launches,
                   "proofs_per_s": round(B / best * 1e3, 1), "parity": "all verdicts equal the oracle's",
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
