"""Times RATIONAL_RECURRENCE aux columns (a[i+1] = (m_i a[i] + n_i) / (c_i a[i] + d_i)) built on the device, at 2^22 rows and
the cubic extension unless told otherwise:
  - one column alone (wf_aux_build, host clock around a device synchronise), the same x + alpha program in each: a
    RUNNING_PRODUCT column (term x + alpha), a LINEAR_RECURRENCE column (m = x + alpha, t = v) and a RATIONAL_RECURRENCE column
    (m = x + alpha, n = v, c = 1, d = beta), and the time of each kernel of the three builds (torch.profiler, CUDA activities);
  - one proof of the example AIR of tests/rational_airs.py through wf_prove_air_aux_built (host and device trace) against
    wf_prove_air_aux with a host builder of the same columns (the CPU reference of the build semantics,
    tests/rational_build_ref.cpp).
One JSON line per part, with the card's name, power limit and max SM clock read in the same run, to stdout and to --out.
Run on an H100: python tools/bench_aux_rational.py --out /tmp/bench_aux_rational.jsonl"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import airs  # noqa: E402
import rational_airs as ra  # noqa: E402
import rational_builds as rb  # noqa: E402
import winterfell_b200 as wf  # noqa: E402
from bench_aux_build import kernel_ms, stages, wall  # noqa: E402
from oracle import oracle as O  # noqa: E402


def one_column(kind):
    """an AIR of the example's main trace and ONE aux column of `kind`, with its build; every kind evaluates x + alpha"""
    A = airs.AirBuilder(5)
    A.constraint(A.sub(A.nxt(0), A.cur(0)), 1)
    A.assert_single(0, 0, 0)
    X = A.aux(1, ra.RATIONAL_NUM_RANDS)
    X.constraint(X.sub(X.anxt(0), X.acur(0)), 1)
    X.assert_single(0, 0, (1, 0, 0))
    B = rb.AuxBuild(5, 1, 0, ra.RATIONAL_NUM_RANDS)
    c = B.column(kind, (1, 0, 0))
    xa = c.add(c.cur(1), c.rnd(0))
    if kind == rb.RUNNING_PRODUCT:
        c.num(xa)
    else:
        c.multiplier(xa)
        c.num(c.cur(0))
        if kind == rb.RATIONAL_RECURRENCE:
            c.den_multiplier(c.const(1))
            c.den(c.rnd(1))
    return A.build(), B.build()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22)
    ap.add_argument("--ext", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    n, ext = 1 << a.log_n, a.ext
    ctx = wf.Context(0)
    opts = O.make_opts(num_queries=28, blowup=8, grinding=8, ext=ext, folding=8, rem_max_deg=31, batch_c=2, batch_d=2, hash_id=0)
    lines = []

    def emit(row):
        row.update(gpu=gpu, log_n=a.log_n, ext=ext)
        print(json.dumps(row), flush=True)
        lines.append(row)

    # 1. one column per kind, the same x + alpha program
    desc, tr, build, builder = ra.rational(n)
    rand = O.rand_elems((ra.RATIONAL_NUM_RANDS, ext), 1)
    main_m = ctx.mat_from_host_columns(tr)
    row = {"part": "one_column"}
    for name, kind in (("running_product", rb.RUNNING_PRODUCT), ("linear_recurrence", rb.LINEAR_RECURRENCE),
                       ("rational_recurrence", rb.RATIONAL_RECURRENCE)):
        d_, b_ = one_column(kind)

        def run():
            m = ctx.aux_build(d_, b_, main_m, rand, ext)
            ctx.sync()
            m.free()
        run()
        row[name + "_ms"] = wall(run, a.reps)
        row[name + "_kernels_ms"] = kernel_ms(ctx, run, a.reps)
    row["term_buffer_mib"] = {"running_product": n * ext * 8 / 2**20, "linear_recurrence": n * 2 * ext * 8 / 2**20,
                              "rational_recurrence": n * 4 * ext * 8 / 2**20}
    main_m.free()
    emit(row)

    # 2. one proof of the example AIR: device build (host / device trace) against the host builder
    import torch
    dev = torch.from_numpy(np.ascontiguousarray(tr).view(np.int64)).cuda()
    torch.cuda.synchronize()
    ctx.prove_air_aux_built(desc, build, tr, opts)   # warm-up: modules, twiddles, pool
    got = ctx.prove_air_aux_built(desc, build, tr, opts)
    ref = ctx.prove_air_aux(desc, tr, opts, builder, ra.RATIONAL_AUX_WIDTH, ra.RATIONAL_NUM_RANDS)
    assert got == ref and ctx.prove_air_aux_built(desc, build, dev.data_ptr(), opts, n=n) == ref
    assert O.verify_air(desc, got, 0) == 0
    row = {"part": "proof", "columns": "2 RATIONAL_RECURRENCE + RUNNING_SUM", "proof_bytes": len(got),
           "built_host_trace_ms": wall(lambda: ctx.prove_air_aux_built(desc, build, tr, opts), 3),
           "built_device_trace_ms": wall(lambda: ctx.prove_air_aux_built(desc, build, dev.data_ptr(), opts, n=n), 3),
           "host_builder_ms": wall(lambda: ctx.prove_air_aux(desc, tr, opts, builder, ra.RATIONAL_AUX_WIDTH, ra.RATIONAL_NUM_RANDS), 2),
           "built_host_trace_stages_ms": stages(ctx, lambda: ctx.prove_air_aux_built(desc, build, tr, opts))}
    emit(row)
    assert ctx.mem_stats()[0] == 0
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
