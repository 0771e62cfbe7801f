"""Times wf_trace_validate (trace check alone; with the degree check) against wf_prove_air on the same input, and a proof with
wf_ctx_set_validation on against off, for the cfg2 shape (FibSmall x 4, 2^20 rows), the widest FibSmall description the
interpreter's 160 registers accept at the cfg3 length (FibSmall x 16, 2^22 rows, cubic extension; x 32 needs 256 registers)
and rescue_like (2^20 rows). One JSON line per shape, written to stdout and to --out; peak pooled bytes are
read from wf_ctx_mem_stats after each part. Run on an H100: python tools/bench_validate.py --out /tmp/bench_validate.jsonl"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import airs  # noqa: E402
import winterfell_b200 as wf  # noqa: E402
from oracle import oracle as O  # noqa: E402


def wall(fn, reps):
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return min(ts), sorted(ts)[len(ts) // 2]


def fib_small(k, n):
    """airs.fib_small_x(k, n) with the trace from the library's C builder (the Python loop takes minutes at 2^22 x 32)."""
    tr, res = wf.build_fib_trace(k, n)
    A = airs.AirBuilder(2 * k)
    A.pub = [int(v) for v in res]
    for j in range(k):
        A.constraint(A.sub(A.nxt(2 * j), A.add(A.cur(2 * j), A.cur(2 * j + 1))), 1)
        A.constraint(A.sub(A.nxt(2 * j + 1), A.add(A.cur(2 * j + 1), A.nxt(2 * j))), 1)
        A.assert_single(2 * j, 0, j + 1)
        A.assert_single(2 * j + 1, 0, j + 1)
        A.assert_single(2 * j + 1, n - 1, int(res[j]))
    return A.build(), tr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--shapes", default="cfg2,cfg3,rescue")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ctx = wf.Context(0)
    shapes = {"cfg2": (lambda: fib_small(4, 1 << 20), 2, 8), "cfg3": (lambda: fib_small(16, 1 << 22), 3, 8),
              "rescue": (lambda: airs.rescue_like(1 << 20), 2, 8)}
    lines = []
    for name in a.shapes.split(","):
        make, ext, blowup = shapes[name]
        desc, tr = make()
        opts = O.make_opts(num_queries=28, blowup=blowup, grinding=0, ext=ext, folding=4, rem_max_deg=31)
        row = {"shape": name, "rows": tr.shape[1], "width": tr.shape[0], "ext": ext, "gpu": gpu}
        ctx.prove_air(desc, tr, opts)   # warm-up: modules, twiddles, pool
        row["prove_ms"] = wall(lambda: ctx.prove_air(desc, tr, opts), a.reps)
        row["pooled_after_prove"] = ctx.mem_stats()[2]
        rep = ctx.trace_validate(desc, tr, ext, check_degrees=False)
        assert rep["kind"] == wf.VALID, rep["msg"]
        row["trace_check_ms"] = wall(lambda: ctx.trace_validate(desc, tr, ext, check_degrees=False), a.reps)
        rep = ctx.trace_validate(desc, tr, ext)
        assert rep["kind"] == wf.VALID, rep["msg"]
        row["trace_and_degree_check_ms"] = wall(lambda: ctx.trace_validate(desc, tr, ext), a.reps)
        row["pooled_after_check"] = ctx.mem_stats()[2]
        ctx.set_validation(1)
        on = ctx.prove_air(desc, tr, opts)
        row["prove_validation_on_ms"] = wall(lambda: ctx.prove_air(desc, tr, opts), a.reps)
        ctx.set_validation(0)
        assert on == ctx.prove_air(desc, tr, opts)
        row["pooled_after_prove_on"] = ctx.mem_stats()[2]
        print(json.dumps(row), flush=True)
        lines.append(row)
        del tr
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
