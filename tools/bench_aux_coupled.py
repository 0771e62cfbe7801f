"""Times COUPLED_RECURRENCE groups (a[i+1] = M_i a[i] + t_i over k aux columns) built on the device, at 2^22 rows and the cubic
extension unless told otherwise:
  - one group alone for k = 2, 3, 4 (wf_aux_build, host clock around a device synchronise) with a full matrix of main columns
    and random elements, and the time of each of its kernels (torch.profiler, CUDA activities); the term buffer's bytes and
    the pool's high-water mark (a fresh context's live + pooled bytes after one build: the pool keeps every buffer it handed
    out); next to it the same group with a diagonal program and the k LINEAR_RECURRENCE columns that compute the same values;
  - one proof of the example AIR of tests/coupled_airs.py through wf_prove_air_aux_built (host and device trace) against
    wf_prove_air_aux with a host builder of the same columns (the CPU reference of the build semantics,
    tests/coupled_build_ref.cpp).
One JSON line per part, with the card's name, power limit and max SM clock read in the same run, to stdout and to --out.
Run on an H100: python tools/bench_aux_coupled.py --out /tmp/bench_aux_coupled.jsonl"""
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
import coupled_airs as ca  # noqa: E402
import coupled_builds as cb  # noqa: E402
import winterfell_b200 as wf  # noqa: E402
from bench_aux_build import kernel_ms, stages, wall  # noqa: E402
from oracle import oracle as O  # noqa: E402

W_MAIN, NR = 5, 2


def _air(aw):
    A = airs.AirBuilder(W_MAIN)
    A.constraint(A.sub(A.nxt(0), A.cur(0)), 1)
    A.assert_single(0, 0, 0)
    X = A.aux(aw, NR)
    X.constraint(X.sub(X.anxt(0), X.acur(0)), 1)
    X.assert_single(0, 0, (1, 0, 0))
    return A.build()


def group(k, diagonal=False):
    """an AIR with k aux columns and the build of one k-group: M[r][c] = x_((r + c) mod 5) + alpha (only r = c when diagonal),
    t_r = x_r beta"""
    B = cb.AuxBuild(W_MAIN, k, 0, NR)
    g = B.group(k, [(r + 1, 0, 0) for r in range(k)])
    for r in range(k):
        for c in range(k):
            if c == r or not diagonal:
                g.m(r, c, g.add(g.cur((r + c) % W_MAIN), g.rnd(0)))
        g.t(r, g.mul(g.cur(r), g.rnd(1)))
    return _air(k), B.build()


def linear(k):
    """the k LINEAR_RECURRENCE columns equal to group(k, diagonal=True)"""
    B = cb.AuxBuild(W_MAIN, k, 0, NR)
    for r in range(k):
        c = B.column(cb.LINEAR_RECURRENCE, (r + 1, 0, 0))
        c.multiplier(c.add(c.cur((2 * r) % W_MAIN), c.rnd(0)))
        c.num(c.mul(c.cur(r), c.rnd(1)))
    return _air(k), B.build()


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
    tr = O.rand_elems((W_MAIN, n), 1)
    rand = O.rand_elems((NR, ext), 2)
    lines = []

    def emit(row):
        row.update(tool="bench_aux_coupled.py", gpu=gpu, log_n=a.log_n, ext=ext)
        print(json.dumps(row), flush=True)
        lines.append(row)

    # 1. one group alone per k, and the diagonal group next to k linear recurrences
    for k in (2, 3, 4):
        row = {"part": "one_group", "k": k, "term_buffer_bytes": n * k * (k + 1) * ext * 8}
        for name, (d_, b_) in (("group", group(k)), ("diagonal_group", group(k, True)), ("linear_recurrences", linear(k))):
            ctx = wf.Context(0)   # fresh: its pool after the first build is that build's high-water mark
            main_m = ctx.mat_from_host_columns(tr)
            base = sum(ctx.mem_stats()[1:])

            def run():
                m = ctx.aux_build(d_, b_, main_m, rand, ext)
                ctx.sync()
                m.free()
            l0 = ctx.launches
            run()
            row[name + "_launches"] = ctx.launches - l0
            row[name + "_pool_high_water_bytes"] = sum(ctx.mem_stats()[1:]) - base
            row[name + "_ms"] = wall(run, a.reps)
            row[name + "_kernels_ms"] = kernel_ms(ctx, run, a.reps)
            if name == "diagonal_group":
                dg = ctx.aux_build(d_, b_, main_m, rand, ext)
                diag = dg.to_columns()
                dg.free()
            elif name == "linear_recurrences":
                lr = ctx.aux_build(d_, b_, main_m, rand, ext)
                assert np.array_equal(diag, lr.to_columns()), "the diagonal group differs from the linear recurrences"
                lr.free()
            main_m.free()
            assert ctx.mem_stats()[0] == 0
            ctx.close()
        emit(row)

    # 2. one proof of the example AIR: device build (host / device trace) against the host builder
    import torch
    ctx = wf.Context(0)
    opts = O.make_opts(num_queries=28, blowup=8, grinding=8, ext=ext, folding=8, rem_max_deg=31, batch_c=2, batch_d=2, hash_id=0)
    desc, tr, build, builder = ca.coupled(n)
    dev = torch.from_numpy(np.ascontiguousarray(tr).view(np.int64)).cuda()
    torch.cuda.synchronize()
    ctx.prove_air_aux_built(desc, build, tr, opts)   # warm-up: modules, twiddles, pool
    got = ctx.prove_air_aux_built(desc, build, tr, opts)
    ref = ctx.prove_air_aux(desc, tr, opts, builder, ca.COUPLED_AUX_WIDTH, ca.COUPLED_NUM_RANDS)
    assert got == ref and ctx.prove_air_aux_built(desc, build, dev.data_ptr(), opts, n=n) == ref
    assert O.verify_air(desc, got, 0) == 0
    row = {"part": "proof", "columns": "POINTWISE + 2-group + 3-group + RUNNING_SUM", "proof_bytes": len(got),
           "built_host_trace_ms": wall(lambda: ctx.prove_air_aux_built(desc, build, tr, opts), 3),
           "built_device_trace_ms": wall(lambda: ctx.prove_air_aux_built(desc, build, dev.data_ptr(), opts, n=n), 3),
           "host_builder_ms": wall(lambda: ctx.prove_air_aux(desc, tr, opts, builder, ca.COUPLED_AUX_WIDTH, ca.COUPLED_NUM_RANDS), 2),
           "built_host_trace_stages_ms": stages(ctx, lambda: ctx.prove_air_aux_built(desc, build, tr, opts)),
           "pooled_bytes": ctx.mem_stats()[2]}
    emit(row)
    assert ctx.mem_stats()[0] == 0
    ctx.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
