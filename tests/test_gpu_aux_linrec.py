"""LINEAR_RECURRENCE aux columns (a[i+1] = m_i * a[i] + t_i) built on the device:
- column for column against the CPU reference (tests/linrec_build_ref.cpp) for D in {1, 2, 3} and n from 8 rows (below one scan
  tile) through 2^11 (one tile) to 2^22, with m = 0 on single rows at tile edges, on every row and m = p - 1, zero
  denominators, an init non-zero in every word, reads of an earlier column at rows i and i + 1 and the wrap row;
- bit for bit the RUNNING_SUM column when m = 1, and the RUNNING_PRODUCT column when t = 0 and m is the term;
- one term launch and three scan launches per column;
- proofs of the example AIR (tests/linrec_airs.py) through every entry point that builds an aux segment: wf_prove_air_aux_built
  from a host and a device trace, wf_prove_air_batch, wf_prove_air_sharded, the provers' validation switch, byte-identical to
  wf_prove_air_aux with a host builder and to the oracle, accepted by the oracle verifier and wf_verify_air_batch;
- wf_trace_validate with the build, and invalid builds."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import airs
import linrec_builds as ab
import linrec_airs as la
import trace_validate_ref as R
import winterfell_b200 as wf

pytestmark = pytest.mark.gpu
P = wf.P
AW, NR = la.LINREC_AUX_WIDTH, la.LINREC_NUM_RANDS


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


def _edges(oracle, n, d, seed):
    """A two-segment AIR shape (3 main columns, 4 aux columns, 2 random elements) whose build has four LINEAR_RECURRENCE columns:
        0: m = main column 1, zero at row 0, the last row of the first tile (2047), the first of the next (2048) and n - 2;
           t = v / (x + gamma) with zero denominators; init non-zero in every word
        1: m = p - 1, t = a0[i] a0[i + 1] + beta (row n - 1 reads row 0)
        2: m = 0 on every row, t = v: a[i + 1] = v[i]
        3: m = beta (an element of E), t = a1[i + 1] - a0[i], and its own init"""
    trace = oracle.rand_elems((3, n), seed)
    rand = oracle.rand_elems((2, d), seed + 1)
    rand[0, 1:] = 0
    g = int(rand[0, 0])
    for i in {0, 2047, 2048, n - 2}:
        if i < n:
            trace[1, i] = 0
    for i in {1, 5 % n, n // 2, n - 1}:
        trace[2, i] = (P - g) % P
    A = airs.AirBuilder(3)
    A.constraint(A.sub(A.nxt(0), A.cur(0)), 1)
    A.assert_single(0, 0, int(trace[0, 0]))
    X = A.aux(AW, NR)
    X.constraint(X.sub(X.anxt(0), X.acur(0)), 1)
    X.assert_single(0, 0, (1, 0, 0))
    B = ab.AuxBuild(3, AW, 0, NR)
    init = lambda s: [int(v) for v in oracle.rand_elems((d,), s)] + [0] * (3 - d)   # noqa: E731
    c0 = B.column(ab.LINEAR_RECURRENCE, init(seed + 3))
    c0.multiplier(c0.cur(1))
    c0.num(c0.cur(0))
    c0.den(c0.add(c0.cur(2), c0.rnd(0)))
    c1 = B.column(ab.LINEAR_RECURRENCE, init(seed + 4))
    c1.multiplier(c1.const(P - 1))
    c1.num(c1.add(c1.mul(c1.acur(0), c1.anxt(0)), c1.rnd(1)))
    c2 = B.column(ab.LINEAR_RECURRENCE, init(seed + 5))
    c2.multiplier(c2.const(0))
    c2.num(c2.cur(0))
    c3 = B.column(ab.LINEAR_RECURRENCE, init(seed + 6))
    c3.multiplier(c3.rnd(1))
    c3.num(c3.sub(c3.anxt(1), c3.acur(0)))
    return A.build(), B.build(), trace, rand


def _build(ctx, desc, build, trace, rand, d):
    n = trace.shape[1]
    main = ctx.mat_from_host_columns(trace)
    l0 = ctx.launches
    aux = ctx.aux_build(desc, build, main, rand, d)
    launches = ctx.launches - l0
    got = aux.to_columns().reshape(AW, d, n).transpose(0, 2, 1)
    main.free()
    aux.free()
    return got, launches


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("log_n", [3, 11, 12, 16, 22])
def test_linrec_columns_match_reference(ctx, oracle, d, log_n):
    n = 1 << log_n
    desc, build, trace, rand = _edges(oracle, n, d, 10 * log_n + d)
    assert wf.aux_build_check(desc, build, log_n) == (0, "")
    got, launches = _build(ctx, desc, build, trace, rand, d)
    assert launches == AW * (1 + 3)                       # a term kernel and three scan kernels per column
    want = ab.reference(desc, build, trace, rand)
    for j in range(AW):
        assert np.array_equal(got[j], want[j]), (j, np.argwhere(got[j] != want[j])[:4])
    # the inputs reach their cases: after a row with m = 0 column 0 holds that row's term alone (0 where its denominator is
    # zero), and column 2 (m = 0 everywhere) holds v of the row before
    emb = lambda v: np.array([int(v)] + [0] * (d - 1), dtype=np.uint64)   # noqa: E731
    for i in sorted({0, 2047, 2048, n - 2}):
        if i < n - 1:
            den = (int(trace[2, i]) + int(rand[0, 0])) % P
            t = oracle.ext_mul(emb(trace[0, i]), oracle.ext_inv(emb(den))) if den else emb(0)
            assert np.array_equal(want[0, i + 1], t), i
    assert np.array_equal(want[2, 1:, 0], trace[0, :-1]) and not want[2, 1:, 1:].any()
    assert np.array_equal(want[0, 2], oracle.ext_mul(emb(trace[1, 1]), want[0, 1]))   # row 1: zero denominator, t_1 = 0
    assert ctx.mem_stats()[0] == 0


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("log_n", [12, 16])
def test_linrec_equals_running_kinds(ctx, oracle, d, log_n):
    n = 1 << log_n
    trace = oracle.rand_elems((3, n), log_n + d)
    rand = oracle.rand_elems((2, d), 5 * d)
    rand[0, 1:] = 0
    trace[2, 7] = (P - int(rand[0, 0])) % P               # a zero denominator in the sum columns
    A = airs.AirBuilder(3)
    A.constraint(A.sub(A.nxt(0), A.cur(0)), 1)
    A.assert_single(0, 0, int(trace[0, 0]))
    X = A.aux(AW, NR)
    X.constraint(X.sub(X.anxt(0), X.acur(0)), 1)
    X.assert_single(0, 0, (1, 0, 0))
    B = ab.AuxBuild(3, AW, 0, NR)
    init = [int(v) for v in oracle.rand_elems((d,), 9)] + [0] * (3 - d)
    s = B.column(ab.RUNNING_SUM, init)                   # t = v / (x + gamma)
    s.num(s.cur(0))
    s.den(s.add(s.cur(2), s.rnd(0)))
    ls = B.column(ab.LINEAR_RECURRENCE, init)             # m = 1, the same t
    ls.multiplier(ls.const(1))
    ls.num(ls.cur(0))
    ls.den(ls.add(ls.cur(2), ls.rnd(0)))
    p = B.column(ab.RUNNING_PRODUCT, init)               # term (v + gamma) * beta
    p.num(p.mul(p.add(p.cur(0), p.rnd(0)), p.rnd(1)))
    lp = B.column(ab.LINEAR_RECURRENCE, init)             # t = 0, m = the term
    lp.multiplier(lp.mul(lp.add(lp.cur(0), lp.rnd(0)), lp.rnd(1)))
    lp.num(lp.const(0))
    desc, build = A.build(), B.build()
    got, launches = _build(ctx, desc, build, trace, rand, d)
    assert launches == AW * 4
    assert np.array_equal(got[0], got[1])
    assert np.array_equal(got[2], got[3])
    assert np.array_equal(got, ab.reference(desc, build, trace, rand))


def _dev_trace(trace):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(trace).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


@pytest.mark.parametrize("ext,hash_id", [(1, 0), (2, 0), (3, 0), (1, 1), (2, 1), (3, 1)])
def test_example_air_proofs(ctx, oracle, ext, hash_id):
    n = 256
    desc, trace, build, builder = la.linrec(n)
    opts = oracle.make_opts(num_queries=20, blowup=8, grinding=2, ext=ext, folding=4, rem_max_deg=7, batch_c=2, batch_d=1, hash_id=hash_id)
    ref = ctx.prove_air_aux(desc, trace, opts, builder, AW, NR)
    got = ctx.prove_air_aux_built(desc, build, trace, opts)
    assert got == ref
    assert got == oracle.prove_air_aux(desc, trace, opts, builder, AW, NR)
    assert oracle.verify_air(desc, got, hash_id) == 0
    assert list(ctx.verify_air_batch([desc], [got], hash_id)) == [wf.VERIFY_ACCEPT]
    dev = _dev_trace(trace)
    assert ctx.prove_air_aux_built(desc, build, dev.data_ptr(), opts, n=n) == ref
    assert ctx.mem_stats()[0] == 0


def test_example_air_batch(ctx, oracle):
    n = 512
    cases = [la.linrec(n, seed=s) for s in (1, 2, 3)]
    build = cases[0][2]
    opts = oracle.make_opts(num_queries=24, blowup=8, grinding=0, ext=3, folding=8, rem_max_deg=15, hash_id=1)
    singles = [ctx.prove_air_aux_built(desc, build, tr, opts) for desc, tr, _, _ in cases]
    got = ctx.prove_air_batch([c[0] for c in cases], [c[1] for c in cases], opts, aux_build=build)
    assert got == singles
    import torch
    dev = torch.from_numpy(np.stack([c[1] for c in cases]).view(np.int64)).cuda().contiguous()
    assert ctx.prove_air_batch([c[0] for c in cases], dev, opts, aux_build=build, device=True) == singles
    assert list(ctx.verify_air_batch([c[0] for c in cases], got, 1)) == [wf.VERIFY_ACCEPT] * 3
    assert ctx.mem_stats()[0] == 0


def _sharded(world, cases):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    here = os.path.dirname(os.path.abspath(__file__))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(here, "linrec_sharded_worker.py"), json.dumps(cases)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ))
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-6000:]
    for i in range(len(cases)):
        assert f"case {i} ok" in r.stdout, out[-6000:]


def test_example_air_sharded_world_2():
    _sharded(2, [{"air": "linrec", "log_n": 12, "ext": 3, "fri_min_log": 5},
                 {"air": "linrec", "log_n": 11, "ext": 2, "hash": 1, "trace": "device"},
                 {"air": "linrec", "log_n": 11, "ext": 1, "trace": "mont"}])


def test_example_air_sharded_world_4():
    _sharded(4, [{"air": "linrec", "log_n": 12, "ext": 2, "fri_min_log": 5},
                 {"air": "linrec", "log_n": 11, "ext": 3, "hash": 1, "trace": "device"}])


@pytest.mark.parametrize("ext", [1, 2, 3])
def test_example_air_validation(ctx, oracle, ext):
    n = 64
    desc, tr, build, _ = la.linrec(n)
    rand = oracle.rand_elems((NR, ext), 70 + ext)
    want = R.validate(desc, tr, ab.reference(desc, build, tr, rand), rand, ext)
    assert want["kind"] == R.VALID
    rep = ctx.trace_validate(desc, tr, ext, rand=rand, aux_build=build)
    assert rep["kind"] == wf.VALID and rep["expected_degrees"] == rep["actual_degrees"] == want["actual_degrees"]
    # a selector that is not 0/1 breaks the main transition at that step only (the aux columns are built from the changed trace)
    bad = tr.copy()
    bad[1, 37] = 2
    want = R.validate(desc, bad, ab.reference(desc, build, bad, rand), rand, ext)
    assert (want["kind"], want["index"], want["step"]) == (R.MAIN_TRANSITION, 0, 37)
    rep = ctx.trace_validate(desc, bad, ext, rand=rand, aux_build=build)
    for k in ("kind", "index", "step", "column", "first_failing_step", "expected_degrees", "actual_degrees", "msg"):
        assert rep[k] == want[k], (k, rep[k], want[k])
    # the provers' validation switch: the same bytes for a valid trace, the reference's message for the broken one
    o = oracle.make_opts(num_queries=20, blowup=8, grinding=0, ext=ext, folding=4, rem_max_deg=7)
    off = ctx.prove_air_aux_built(desc, build, tr, o)
    ctx.set_validation(1)
    try:
        assert ctx.prove_air_aux_built(desc, build, tr, o) == off
        assert ctx.prove_air_batch([desc, desc], [tr, tr], o, aux_build=build) == [off, off]
        with pytest.raises(wf.WfError) as e:
            ctx.prove_air_aux_built(la.linrec_desc(bad), build, bad, o)
        assert "main transition constraint 0 did not evaluate to ZERO at step 37" in str(e.value)
    finally:
        ctx.set_validation(0)
    assert ctx.prove_air_aux_built(desc, build, tr, o) == off
    assert ctx.mem_stats()[0] == 0


def test_invalid_linrec_builds_fail_and_leave_no_buffers(oracle):
    c = wf.Context(0)
    try:
        n = 64
        desc, trace, build, _ = la.linrec(n)
        opts = oracle.make_opts(num_queries=8, blowup=8, grinding=0, ext=2, folding=4, rem_max_deg=7, hash_id=0)

        def col1(fn):
            B = ab.AuxBuild(3, AW, 0, NR)
            dd = B.column(ab.RUNNING_PRODUCT, (1, 0, 0))
            dd.num(dd.add(dd.cur(2), dd.rnd(0)))
            fn(B.column(ab.LINEAR_RECURRENCE))
            for _ in (2, 3):
                x = B.column(ab.LINEAR_RECURRENCE)
                x.multiplier(x.rnd(1))
                x.num(x.cur(0))
            return B.build()

        main = c.mat_from_host_columns(trace)
        rand = oracle.rand_elems((NR, 2), 3)
        for b, why in ((col1(lambda x: x.num(x.cur(0))), "has no multiplier (OUT 2)"),
                       (col1(lambda x: (x.multiplier(x.cur(1)), x.multiplier(x.cur(1)), x.num(x.cur(0)))), "more than one multiplier"),
                       (col1(lambda x: (x.multiplier(x.cur(1)), x.num(x.cur(0)), x.prog.append((airs.OUT, 3, x.cur(0), 0)))),
                        "nor multiplier (2)")):
            for fn in (lambda: c.prove_air_aux_built(desc, b, trace, opts), lambda: c.aux_build(desc, b, main, rand, 2),
                       lambda: c.prove_air_batch([desc], [trace], opts, aux_build=b),
                       lambda: c.trace_validate(desc, trace, 2, rand=rand, aux_build=b)):
                with pytest.raises(wf.WfError, match="error -2"):
                    fn()
                assert why in c.L.wf_last_error(c.h).decode()
                assert c.mem_stats()[0] == 1                  # the main matrix the test holds
        bad = build.copy()
        bad[3 + 6 + 8 + 2] = 5                                # column 1's init word 1 with ext 1
        with pytest.raises(wf.WfError, match="error -2"):
            c.prove_air_aux_built(desc, bad, trace, oracle.make_opts(num_queries=8, ext=1))
        assert "beyond the extension degree" in c.L.wf_last_error(c.h).decode()
        main.free()
        assert c.mem_stats()[0] == 0
    finally:
        c.close()
