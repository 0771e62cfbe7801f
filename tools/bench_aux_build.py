"""Times the aux segment built on the device with LINEAR_RECURRENCE columns (a[i+1] = m_i * a[i] + t_i), at 2^22 rows and
the cubic extension unless told otherwise:
  - the aux_build stage of one proof (wf_prove_air_aux_built, stage events on) of the example AIR of tests/linrec_airs.py
    (a running product and three linear recurrences) against perm_rap's (a running product and two running sums);
  - one column alone (wf_aux_build, host clock around a device synchronise): a LINEAR_RECURRENCE column with m = x + alpha,
    t = v against a RUNNING_PRODUCT column whose term is the same x + alpha, and the time of each kernel of both builds
    (torch.profiler, CUDA activities);
  - one proof of the example AIR through wf_prove_air_aux_built (host and device trace) against wf_prove_air_aux with a host
    builder of the same columns (the CPU reference of the build semantics, tests/linrec_build_ref.cpp).
One JSON line per part, with the card's name, power limit and max SM clock read in the same run, to stdout and to --out.
Run on an H100: python tools/bench_aux_build.py --out /tmp/bench_aux_build.jsonl"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import airs  # noqa: E402
import linrec_builds as ab  # noqa: E402
import linrec_airs as la  # noqa: E402
import winterfell_b200 as wf  # noqa: E402
from oracle import oracle as O  # noqa: E402


def wall(fn, reps):
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return {"min": round(min(ts), 3), "median": round(sorted(ts)[len(ts) // 2], 3)}


def stages(ctx, fn):
    """{stage: ms} of one call with the stage events on"""
    ctx.set_profiling(True)
    try:
        fn()
        return {k: round(v, 3) for k, v in ctx.stage_times()}
    finally:
        ctx.set_profiling(False)


def stage_ms(ctx, fn):
    return stages(ctx, fn)["aux_build"]


def one_column(kind):
    """an AIR of the example's main trace and ONE aux column, with its build: RUNNING_PRODUCT of x + alpha, or
    LINEAR_RECURRENCE with m = x + alpha, t = v"""
    A = airs.AirBuilder(3)
    A.constraint(A.sub(A.nxt(0), A.cur(0)), 1)
    A.assert_single(0, 0, 0)
    X = A.aux(1, la.LINREC_NUM_RANDS)
    X.constraint(X.sub(X.anxt(0), X.acur(0)), 1)
    X.assert_single(0, 0, (1, 0, 0))
    B = ab.AuxBuild(3, 1, 0, la.LINREC_NUM_RANDS)
    c = B.column(kind, (1, 0, 0))
    xa = c.add(c.cur(2), c.rnd(0))
    if kind == ab.LINEAR_RECURRENCE:
        c.multiplier(xa)
        c.num(c.cur(0))
    else:
        c.num(xa)
    return A.build(), B.build()


def kernel_ms(ctx, fn, reps):
    """mean device time per call of each kernel fn launches (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        ctx.sync()
    out = {}
    for e in prof.key_averages():
        if e.key.startswith("_Z") or "aux_" in e.key:
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            out[e.key] = round(t / 1e3 / reps, 4)
    return out


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

    # 1. the aux_build stage of one proof: the example AIR against perm_rap
    desc, tr, build, builder = la.linrec(n)
    pdesc, ptr, _ = airs.perm_rap(n)
    pbuild = ab.perm_rap_build()
    row = {"part": "aux_build_stage"}
    for name, (d_, t_, b_) in (("linrec", (desc, tr, build)), ("perm_rap", (pdesc, ptr, pbuild))):
        ctx.prove_air_aux_built(d_, b_, t_, opts)   # warm-up: modules, twiddles, pool
        row[name + "_stage_ms"] = sorted(stage_ms(ctx, lambda: ctx.prove_air_aux_built(d_, b_, t_, opts)) for _ in range(3))
    row["linrec_columns"] = "RUNNING_PRODUCT + 3 LINEAR_RECURRENCE"
    row["perm_rap_columns"] = "RUNNING_PRODUCT + 2 RUNNING_SUM"
    emit(row)

    # 2. one column per kind, the same x + alpha program
    rand = O.rand_elems((la.LINREC_NUM_RANDS, ext), 1)
    main_m = ctx.mat_from_host_columns(tr)
    row = {"part": "one_column"}
    for name, kind in (("running_product", ab.RUNNING_PRODUCT), ("linear_recurrence", ab.LINEAR_RECURRENCE)):
        d_, b_ = one_column(kind)

        def run():
            m = ctx.aux_build(d_, b_, main_m, rand, ext)
            ctx.sync()
            m.free()
        run()
        row[name + "_ms"] = wall(run, a.reps)
        row[name + "_kernels_ms"] = kernel_ms(ctx, run, a.reps)
    row["term_buffer_mib"] = {"running_product": n * ext * 8 / 2**20, "linear_recurrence": n * 2 * ext * 8 / 2**20}
    main_m.free()
    emit(row)

    # 3. one proof of the example AIR: device build (host / device trace) against the host builder
    import torch
    dev = torch.from_numpy(np.ascontiguousarray(tr).view(np.int64)).cuda()
    torch.cuda.synchronize()
    got = ctx.prove_air_aux_built(desc, build, tr, opts)
    ref = ctx.prove_air_aux(desc, tr, opts, builder, la.LINREC_AUX_WIDTH, la.LINREC_NUM_RANDS)
    assert got == ref and ctx.prove_air_aux_built(desc, build, dev.data_ptr(), opts, n=n) == ref
    assert O.verify_air(desc, got, 0) == 0
    row = {"part": "proof", "proof_bytes": len(got),
           "built_host_trace_ms": wall(lambda: ctx.prove_air_aux_built(desc, build, tr, opts), 3),
           "built_device_trace_ms": wall(lambda: ctx.prove_air_aux_built(desc, build, dev.data_ptr(), opts, n=n), 3),
           "host_builder_ms": wall(lambda: ctx.prove_air_aux(desc, tr, opts, builder, la.LINREC_AUX_WIDTH, la.LINREC_NUM_RANDS), 2),
           "built_host_trace_stages_ms": stages(ctx, lambda: ctx.prove_air_aux_built(desc, build, tr, opts)),
           # the host builder runs inside the stage that follows the main commitment (no aux_build mark of its own)
           "host_builder_stages_ms": stages(ctx, lambda: ctx.prove_air_aux(desc, tr, opts, builder, la.LINREC_AUX_WIDTH,
                                                                           la.LINREC_NUM_RANDS))}
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
