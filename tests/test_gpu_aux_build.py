"""The aux segment built on the device from a build description (wf_aux_build, wf_prove_air_aux_built):
- column for column against the CPU reference of the build semantics (tests/aux_build_ref.cpp), for every kind, D in {1, 2, 3}
  and n from 8 to 2^22 rows, with zero denominators, reads of earlier aux columns at rows i and i + 1, periodic columns and the
  wrap row n - 1;
- perm_rap proofs through the new entry point, from a host trace and from a device trace, byte-identical to wf_prove_air_aux with
  the host builder and to the oracle's proof, and accepted by the restated verifier;
- invalid input fails with WF_ERR_INVALID and leaves no device buffer behind."""
import ctypes as C
import json
import os
import subprocess
import time

import numpy as np
import pytest

import airs
import aux_builds as ab
import winterfell_b200 as wf

pytestmark = pytest.mark.gpu
P = wf.P


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


def _mixed(oracle, n, d, seed):
    """A two-segment AIR shape (3 main columns, periodic columns of 4 and 8 values, 4 aux columns, 2 random elements) with a
    build of every kind. gamma lies in the base field so that main values -gamma make denominators zero."""
    trace = oracle.rand_elems((3, n), seed)
    rand = oracle.rand_elems((2, d), seed + 1)
    rand[0, 1:] = 0
    g = int(rand[0, 0])
    trace[2, n - 1] = (P - g) % P                        # product column: zero denominator on the wrap row (its term is unused)
    for i in {0, 5 % n, n // 2, n - 1}:
        trace[1, i] = (P - g) % P                        # sum and pointwise columns: zero denominators inside the column
    A = airs.AirBuilder(3)
    A.periodic = [[(7 * i + 3) % P for i in range(4)], oracle.rand_elems((8,), seed + 2)]
    A.constraint(A.sub(A.nxt(0), A.cur(0)), 1)
    A.assert_single(0, 0, int(trace[0, 0]))
    X = A.aux(4, 2)
    X.constraint(X.sub(X.anxt(0), X.acur(0)), 1)
    X.assert_single(0, 0, (1, 0, 0))
    B = ab.AuxBuild(3, 4, 2, 2)
    c0 = B.column(ab.RUNNING_PRODUCT, (1, 0, 0))
    c0.num(c0.add(c0.cur(0), c0.rnd(0)))
    c0.den(c0.add(c0.cur(2), c0.rnd(0)))
    init1 = [int(v) for v in oracle.rand_elems((d,), seed + 3)] + [0] * (3 - d)
    c1 = B.column(ab.RUNNING_SUM, init1)
    c1.num(c1.add(c1.mul(c1.mul(c1.rnd(1), c1.per(0)), c1.mul(c1.cur(1), c1.acur(0))), c1.anxt(0)))
    c1.den(c1.add(c1.cur(1), c1.rnd(0)))
    c2 = B.column(ab.POINTWISE)
    c2.num(c2.add(c2.add(c2.mul(c2.acur(1), c2.nxt(2)), c2.per(1)), c2.const(7)))
    c2.den(c2.mul(c2.add(c2.cur(1), c2.rnd(0)), c2.sub(c2.anxt(1), c2.acur(0))))
    c3 = B.column(ab.RUNNING_SUM, (5, 0, 0))
    c3.num(c3.const(1))
    return A.build(), B.build(), trace, rand


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("log_n", [3, 10, 16, 22])
def test_aux_build_matches_reference(ctx, oracle, d, log_n):
    n = 1 << log_n
    desc, build, trace, rand = _mixed(oracle, n, d, 10 * log_n + d)
    assert wf.aux_build_check(desc, build, log_n) == (0, "")
    main = ctx.mat_from_host_columns(trace)
    l0 = ctx.launches
    aux = ctx.aux_build(desc, build, main, rand, d)
    assert ctx.launches - l0 == 4 + 3 * 3                 # a term kernel per column, three scan kernels per running column
    got = aux.to_columns().reshape(4, d, n).transpose(0, 2, 1)
    want = ab.reference(desc, build, trace, rand)
    for j in range(4):
        assert np.array_equal(got[j], want[j]), (j, np.argwhere(got[j] != want[j])[:4])
    # the zero denominators took effect: the sum column skips those rows' terms, the pointwise column is 0 there
    assert not want[2, n // 2].any() and want[0, n - 1].any()
    main.free()
    aux.free()


def _dev_trace(trace):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(trace).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


@pytest.mark.parametrize("ext,hash_id", [(1, 0), (2, 0), (3, 0), (1, 1), (2, 1), (3, 1)])
def test_perm_rap_proof_equals_host_builder_and_oracle(ctx, oracle, ext, hash_id):
    n = 256
    desc, trace, builder = airs.perm_rap(n)
    build = ab.perm_rap_build()
    opts = oracle.make_opts(num_queries=20, blowup=8, grinding=2, ext=ext, folding=4, rem_max_deg=7, batch_c=2, batch_d=1, hash_id=hash_id)
    ref = ctx.prove_air_aux(desc, trace, opts, builder, airs.PERM_RAP_AUX_WIDTH, 2)
    got = ctx.prove_air_aux_built(desc, build, trace, opts)
    assert got == ref
    assert got == oracle.prove_air_aux(desc, trace, opts, builder, airs.PERM_RAP_AUX_WIDTH, 2)
    assert oracle.verify_air(desc, got, hash_id) == 0
    dev = _dev_trace(trace)
    assert ctx.prove_air_aux_built(desc, build, dev.data_ptr(), opts, n=n) == ref


def test_perm_rap_proof_with_aux_assertion_callback(ctx, oracle):
    n = 512
    desc, trace, builder = airs.perm_rap(n, dyn_last_q=True)
    opts = oracle.make_opts(num_queries=24, blowup=8, grinding=0, ext=3, folding=8, rem_max_deg=15, hash_id=0)
    ref = ctx.prove_air_aux_dyn(desc, trace, opts, builder, builder.values_fn, airs.PERM_RAP_AUX_WIDTH, 2, builder.num_values)
    got = ctx.prove_air_aux_built(desc, ab.perm_rap_build(), trace, opts, values_fn=builder.values_fn, num_rands=2,
                                  num_values=builder.num_values)
    assert got == ref
    assert oracle.verify_air_dyn(desc, got, 0, builder.values_fn, 2, builder.num_values, 3) == 0


def test_evaluate_keeps_the_segment_width_of_pipelined_coefficients(ctx, oracle):
    # a host trace of 3 columns at 2^12 rows goes through the chunked upload pipeline in chunks of 2 columns: its coefficient
    # matrix has 2-wide segments, and the forward transform the aux build applies to it must keep them
    trace = oracle.rand_elems((3, 1 << 12), 77)
    polys, lde = ctx.trace_lde_from_host(trace, 3)
    ev = polys.evaluate()
    assert np.array_equal(ev.to_columns(), trace)
    for m in (polys, lde, ev):
        m.free()


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, watts = [s.strip() for s in out.rsplit(",", 1)]
        return {"name": name, "power_limit_w": float(watts)}
    except Exception as e:  # the record still carries the timings
        return {"name": None, "power_limit_w": None, "failed": str(e)}


@pytest.mark.parametrize("log_n,ext,hash_id", [(18, 2, 1), (22, 3, 0)])
def test_perm_rap_large(ctx, oracle, log_n, ext, hash_id):
    n = 1 << log_n
    desc, trace, builder = airs.perm_rap(n)
    build = ab.perm_rap_build()
    opts = oracle.make_opts(num_queries=28, blowup=8, grinding=8, ext=ext, folding=8, rem_max_deg=31, batch_c=2, batch_d=2, hash_id=hash_id)
    got = ctx.prove_air_aux_built(desc, build, trace, opts)
    assert oracle.verify_air(desc, got, hash_id) == 0
    t0 = time.perf_counter()
    ref = ctx.prove_air_aux(desc, trace, opts, builder, airs.PERM_RAP_AUX_WIDTH, 2)   # the oracle's C builder as callback
    ref_wall = (time.perf_counter() - t0) * 1e3
    assert got == ref
    dev = _dev_trace(trace)
    assert ctx.prove_air_aux_built(desc, build, dev.data_ptr(), opts, n=n) == ref
    if os.environ.get("WF_REPORT"):
        # warm pool; wall times with the stage events off, then one run with them on for the aux_build stage
        def wall(fn, reps):
            ts = []
            for _ in range(reps):
                t = time.perf_counter()
                fn()
                ts.append((time.perf_counter() - t) * 1e3)
            return ts
        new_host = wall(lambda: ctx.prove_air_aux_built(desc, build, trace, opts), 3)
        new_dev = wall(lambda: ctx.prove_air_aux_built(desc, build, dev.data_ptr(), opts, n=n), 3)
        old = wall(lambda: ctx.prove_air_aux(desc, trace, opts, builder, airs.PERM_RAP_AUX_WIDTH, 2), 2) + [ref_wall]
        t = time.perf_counter()
        builder(np.zeros((2, ext), dtype=np.uint64))
        cpu_builder_ms = (time.perf_counter() - t) * 1e3
        stages = {}
        for name, arg in (("host_trace", trace), ("device_trace", dev.data_ptr())):
            ctx.set_profiling(True)
            ctx.prove_air_aux_built(desc, build, arg, opts, n=n)
            stages[name] = {k: round(v, 3) for k, v in ctx.stage_times()}
            ctx.set_profiling(False)
        ctx.set_profiling(True)
        ctx.prove_air_aux(desc, trace, opts, builder, airs.PERM_RAP_AUX_WIDTH, 2)
        stages["host_builder"] = {k: round(v, 3) for k, v in ctx.stage_times()}
        ctx.set_profiling(False)
        rec = {"air": "perm_rap (3 main + 3 aux columns, 2 random elements)", "log_n": log_n, "opts": [int(x) for x in opts],
               "card": _card(), "proof_bytes": len(got),
               "wall_ms_built_host_trace": [round(x, 2) for x in new_host],
               "wall_ms_built_device_trace": [round(x, 2) for x in new_dev],
               "wall_ms_prove_air_aux_c_builder": [round(x, 2) for x in old],
               "c_builder_alone_ms": round(cpu_builder_ms, 2), "stage_ms": stages}
        with open(os.environ["WF_REPORT"], "a") as f:
            f.write(json.dumps(rec) + "\n")


def test_invalid_input_fails_and_leaves_no_buffers(oracle):
    c = wf.Context(0)
    try:
        n = 64
        desc, trace, _ = airs.perm_rap(n)
        build = ab.perm_rap_build()
        opts = oracle.make_opts(num_queries=8, blowup=8, grinding=0, ext=2, folding=4, rem_max_deg=7, hash_id=0)

        def rejected(fn, why):
            with pytest.raises(wf.WfError, match="error -2"):
                fn()
            assert why in c.L.wf_last_error(c.h).decode()
            assert c.mem_stats()[0] == 0

        bad = build.copy(); bad[3] = 7
        rejected(lambda: c.prove_air_aux_built(desc, bad, trace, opts), "unknown aux column kind")
        bad = build.copy(); bad[0] = 4
        rejected(lambda: c.prove_air_aux_built(desc, bad, trace, opts), "width does not match")
        bad = build.copy(); bad[5] = 9                        # init word 1 with ext 1
        rejected(lambda: c.prove_air_aux_built(desc, bad, trace, oracle.make_opts(num_queries=8, ext=1)), "beyond the extension degree")
        dev = _dev_trace(trace)
        d_, b_, o_ = (np.ascontiguousarray(x, dtype=t) for x, t in ((desc, np.uint64), (build, np.uint64), (opts, np.uint32)))
        ptrs = (wf.u64p * 3)(*[np.ascontiguousarray(trace[j]).ctypes.data_as(wf.u64p) for j in range(3)])
        buf = np.zeros(1 << 20, dtype=np.uint8)
        for host, devp in ((ptrs, C.c_void_p(dev.data_ptr())), (None, None)):
            ln = C.c_size_t(buf.size)
            rc = c.L.wf_prove_air_aux_built(c.h, d_.ctypes.data_as(wf.u64p), d_.size, b_.ctypes.data_as(wf.u64p), b_.size, host, devp, 0, 6,
                                           o_.ctypes.data_as(C.POINTER(C.c_uint32)), wf.AUX_BUILDER(), None, buf.ctypes.data_as(wf.u8p), C.byref(ln))
            assert rc == -2 and "exactly one of" in c.L.wf_last_error(c.h).decode()
            assert c.mem_stats()[0] == 0
        # the step entry: main matrix of the wrong width, random elements that are not canonical
        for cols, rand, why in ((trace[:2], np.ones((2, 2), dtype=np.uint64), "main trace shape"),
                                (trace, np.full((2, 2), P, dtype=np.uint64), "not a canonical")):
            main = c.mat_from_host_columns(cols)
            with pytest.raises(wf.WfError, match="error -2"):
                c.aux_build(desc, build, main, rand, 2)
            assert why in c.L.wf_last_error(c.h).decode()
            assert c.mem_stats()[0] == 1                      # the matrix the test holds
            main.free()
        assert c.mem_stats()[0] == 0
    finally:
        c.close()
