"""Many small proofs of one AIR: wf_prove_air_batch against a loop of wf_prove_air over the same traces, in the same process.

Shapes (BASELINE.json): cfg1 = fib_small, 2^16 rows x 2 columns, Blake3_256, base field, 28 queries, blowup 8, folding 8,
remainder degree 31, grinding 16, at B in {1, 8, 64, 256}; cfg2 = FibSmall x 4, 2^20 rows x 8 columns, same options, at
B in {1, 4, 16}. Proof j of a batch proves pairs [k j, k (j + 1)) of one FibSmall x (k B) trace, so every proof has its own
starting values, assertion values and public inputs. Per B: proofs per second and ms per batch of both arms (median of
--reps), launches per batch, and the check that both arms return the same bytes. Also the stage split of one proof
(wf_ctx_set_profiling) and the device memory one proof of each shape holds (wf_ctx_mem_stats), with the card's name and
power limit. One JSON object per line on stdout, and appended to --out when given."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import airs  # noqa: E402
import winterfell_b200 as wf  # noqa: E402

SHAPES = {"cfg1": (1, 16, [1, 8, 64, 256]), "cfg2": (4, 20, [1, 4, 16])}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    name, watts = [s.strip() for s in out.rsplit(",", 1)]
    return {"name": name, "power_limit_w": float(watts)}


def fib_desc(trace, k):
    """FibSmall x k over the pairs of `trace` ([2k, n]), asserting their own starting values and results"""
    n = trace.shape[1]
    A = airs.AirBuilder(2 * k)
    A.pub = [int(trace[2 * q + 1, n - 1]) for q in range(k)]
    for q in range(k):
        A.constraint(A.sub(A.nxt(2 * q), A.add(A.cur(2 * q), A.cur(2 * q + 1))), 1)
        A.constraint(A.sub(A.nxt(2 * q + 1), A.add(A.cur(2 * q + 1), A.nxt(2 * q))), 1)
        A.assert_single(2 * q, 0, int(trace[2 * q, 0]))
        A.assert_single(2 * q + 1, 0, int(trace[2 * q + 1, 0]))
        A.assert_single(2 * q + 1, n - 1, int(trace[2 * q + 1, n - 1]))
    return A.build()


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="cfg1,cfg2")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = wf.Context(0)
    info = card()
    opts = np.array([28, 8, 16, 1, 8, 31, 0, 0, wf.HASH_BLAKE3_256], dtype=np.uint32)
    for shape in args.shapes.split(","):
        k, log_n, batches = SHAPES[shape]
        n = 1 << log_n
        full, _ = wf.build_fib_trace(k * max(batches), n)
        traces = [full[2 * k * j: 2 * k * (j + 1)] for j in range(max(batches))]
        descs = [fib_desc(t, k) for t in traces]
        # device memory of one proof: the pool after one proof on a fresh context holds every buffer the proof needed at once
        c1 = wf.Context(0)
        c1.prove_air(descs[0], traces[0], opts)
        live, _, pooled = c1.mem_stats()
        c1.set_profiling(True)
        t = time.perf_counter()
        c1.prove_air(descs[0], traces[0], opts)
        wall = (time.perf_counter() - t) * 1e3
        stages = {s: round(v, 3) for s, v in c1.stage_times()}
        c1.close()
        emit({"shape": shape, "card": info, "rows": n, "columns": 2 * k, "opts": [int(x) for x in opts],
              "device_bytes_one_proof": pooled, "live_after": live, "profiled_proof_wall_ms": round(wall, 3), "stage_ms": stages}, args.out)
        for B in batches:
            d, tr = descs[:B], traces[:B]
            got = ctx.prove_air_batch(d, tr, opts)        # warm-up of both arms (pool, twiddles, constraint kernel)
            ref = [ctx.prove_air(d[j], tr[j], opts) for j in range(B)]
            assert got == ref, f"{shape} B={B}: batch and loop differ"
            t_batch, t_loop = [], []
            for _ in range(args.reps):
                l0 = ctx.launches
                t = time.perf_counter()
                got = ctx.prove_air_batch(d, tr, opts)
                t_batch.append(time.perf_counter() - t)
                l1 = ctx.launches
                t = time.perf_counter()
                ref = [ctx.prove_air(d[j], tr[j], opts) for j in range(B)]
                t_loop.append(time.perf_counter() - t)
                l2 = ctx.launches
                assert got == ref, f"{shape} B={B}: batch and loop differ"
            mb, ml = statistics.median(t_batch), statistics.median(t_loop)
            emit({"shape": shape, "B": B, "card": info, "outputs_equal": True,
                  "batch": {"ms_per_batch": round(mb * 1e3, 2), "proofs_per_s": round(B / mb, 1), "launches_per_batch": l1 - l0},
                  "loop": {"ms_per_batch": round(ml * 1e3, 2), "proofs_per_s": round(B / ml, 1), "launches_per_batch": l2 - l1},
                  "ms_batch_all": [round(x * 1e3, 2) for x in t_batch], "ms_loop_all": [round(x * 1e3, 2) for x in t_loop]}, args.out)
    ctx.close()


if __name__ == "__main__":
    main()
