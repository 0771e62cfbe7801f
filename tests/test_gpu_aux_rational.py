"""RATIONAL_RECURRENCE aux columns (a[i+1] = (m_i a[i] + n_i) / (c_i a[i] + d_i), inv(0) = 0) built on the device:
- column for column against the CPU reference (tests/rational_build_ref.cpp) for D in {1, 2, 3} and n from 8 rows (below one scan
  tile) through 2^11 (one tile) to 2^22, with maps driven by random elements and main columns, an init non-zero in every word,
  and reads of an earlier column at rows i and i + 1;
- bit for bit the LINEAR_RECURRENCE column when c = 0 and d = 1;
- aimed zero denominators: at row 0, around and on tile edges, on consecutive rows, at row n - 1 (no effect), a 0/0 row and 64
  scattered rows;
- one term launch and three scan launches per column, three more per rescan after a vanishing denominator;
- proofs of the example AIR (tests/rational_airs.py) through every entry point that builds an aux segment, byte-identical to
  wf_prove_air_aux with the CPU reference as host builder and to the oracle, accepted by the oracle verifier and
  wf_verify_air_batch, also for traces with a vanishing denominator;
- wf_trace_validate with the build, and invalid builds."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import airs
import rational_airs as ra
import rational_builds as rb
import trace_validate_ref as R
import winterfell_b200 as wf

pytestmark = pytest.mark.gpu
P = wf.P
AW, NR = ra.RATIONAL_AUX_WIDTH, ra.RATIONAL_NUM_RANDS
TILE = 2048   # AUX_SCAN_TILE


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


def _air(w, aw, nr):
    A = airs.AirBuilder(w)
    A.constraint(A.sub(A.nxt(0), A.cur(0)), 1)
    A.assert_single(0, 0, 0)
    X = A.aux(aw, nr)
    X.constraint(X.sub(X.anxt(0), X.acur(0)), 1)
    X.assert_single(0, 0, (1, 0, 0))
    return A.build()


def _init(oracle, d, s): return [int(v) for v in oracle.rand_elems((d,), s)] + [0] * (3 - d)


def _random_maps(oracle, n, d, seed):
    """3 main columns, 3 aux columns, 2 random elements (alpha, beta); the build:
        0: m = alpha, n = v, c = x, d = beta   (a fractional fingerprint, extension-valued), init non-zero in every word
        1: m = a0[i + 1], n = beta, c = a0[i], d = v + x   (reads column 0 at rows i and i + 1; the wrap row too)
        2: m = x, n = a1[i], c = alpha, no denominator (d = 1)"""
    trace = oracle.rand_elems((3, n), seed)
    rand = oracle.rand_elems((NR, d), seed + 1)
    B = rb.AuxBuild(3, AW, 0, NR)
    c0 = B.column(rb.RATIONAL_RECURRENCE, _init(oracle, d, seed + 2))
    c0.multiplier(c0.rnd(0))
    c0.num(c0.cur(0))
    c0.den_multiplier(c0.cur(1))
    c0.den(c0.rnd(1))
    c1 = B.column(rb.RATIONAL_RECURRENCE, _init(oracle, d, seed + 3))
    c1.multiplier(c1.anxt(0))
    c1.num(c1.rnd(1))
    c1.den_multiplier(c1.acur(0))
    c1.den(c1.add(c1.cur(0), c1.cur(1)))
    c2 = B.column(rb.RATIONAL_RECURRENCE, _init(oracle, d, seed + 4))
    c2.multiplier(c2.cur(1))
    c2.num(c2.acur(1))
    c2.den_multiplier(c2.rnd(0))
    return _air(3, AW, NR), B.build(), trace, rand


def _build(ctx, desc, build, trace, rand, d, aw=AW):
    n = trace.shape[1]
    main = ctx.mat_from_host_columns(trace)
    l0 = ctx.launches
    aux = ctx.aux_build(desc, build, main, rand, d)
    launches = ctx.launches - l0
    got = aux.to_columns().reshape(aw, d, n).transpose(0, 2, 1)
    main.free()
    aux.free()
    return got, launches


def _assert_columns(got, want):
    for j in range(want.shape[0]):
        assert np.array_equal(got[j], want[j]), (j, np.argwhere(got[j] != want[j])[:4])


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("log_n", [3, 11, 12, 16, 22])
def test_rational_columns_match_reference(ctx, oracle, d, log_n):
    n = 1 << log_n
    desc, build, trace, rand = _random_maps(oracle, n, d, 10 * log_n + d)
    assert wf.aux_build_check(desc, build, log_n) == (0, "")
    got, launches = _build(ctx, desc, build, trace, rand, d)
    want = rb.reference(desc, build, trace, rand)
    _assert_columns(got, want)
    assert launches == AW * (1 + 3)                       # a term kernel and three scan kernels per column, no rescan
    assert want[0, :, 1:].any() if d > 1 else True         # extension-valued
    assert ctx.mem_stats()[0] == 0


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("log_n", [12, 16])
def test_rational_equals_linear_recurrence(ctx, oracle, d, log_n):
    n = 1 << log_n
    trace = oracle.rand_elems((3, n), log_n + d)
    rand = oracle.rand_elems((NR, d), 5 * d)
    init = _init(oracle, d, 9)
    B = rb.AuxBuild(3, 2, 0, NR)
    lin = B.column(rb.LINEAR_RECURRENCE, init)        # a' = (x + alpha) a + v
    lin.multiplier(lin.add(lin.cur(1), lin.rnd(0)))
    lin.num(lin.cur(0))
    rat = B.column(rb.RATIONAL_RECURRENCE, init)      # the same with c = 0, d = 1
    rat.multiplier(rat.add(rat.cur(1), rat.rnd(0)))
    rat.num(rat.cur(0))
    rat.den_multiplier(rat.const(0))
    desc, build = _air(3, 2, NR), B.build()
    got, launches = _build(ctx, desc, build, trace, rand, d, aw=2)
    assert launches == 2 * 4
    assert np.array_equal(got[0], got[1])
    assert np.array_equal(got, rb.reference(desc, build, trace, rand))


def _aimed(oracle, n, d, rows, zero_zero, seed):
    """An AIR with 5 main columns and 2 aux columns; column 0 is base-valued (m = x, n = v, c = s, d = u, all main columns), so
    setting u_i = -s_i a[i] makes its denominator vanish at row i; at the rows of zero_zero v_i = -x_i a[i] too (0/0). Column 1
    (m = alpha, n = a0[i + 1], c = a0[i], d = beta) reads it, extension-valued. Zeros are placed in row order, each against the
    reference of the trace so far."""
    trace = oracle.rand_elems((5, n), seed)
    rand = oracle.rand_elems((NR, d), seed + 1)
    B = rb.AuxBuild(5, 2, 0, NR)
    c0 = B.column(rb.RATIONAL_RECURRENCE, (7, 0, 0))
    c0.multiplier(c0.cur(1))
    c0.num(c0.cur(0))
    c0.den_multiplier(c0.cur(2))
    c0.den(c0.cur(3))
    c1 = B.column(rb.RATIONAL_RECURRENCE, _init(oracle, d, seed + 2))
    c1.multiplier(c1.rnd(0))
    c1.num(c1.anxt(0))
    c1.den_multiplier(c1.acur(0))
    c1.den(c1.rnd(1))
    desc, build = _air(5, 2, NR), B.build()
    rows = sorted(set(rows) | set(zero_zero))
    # column 0 alone, over the base field, to aim the zeros
    ref = lambda: rb.reference(desc, build, trace, rand[:, :1] if d > 1 else rand)[0, :, 0]   # noqa: E731
    a0 = ref()
    for i in rows:
        trace[3, i] = (-int(trace[2, i]) * int(a0[i])) % P
        if i in zero_zero:
            trace[0, i] = (-int(trace[1, i]) * int(a0[i])) % P
        a0 = ref()
    return desc, build, trace, rand


AIMS = {
    "row0": ([0], []),
    "tile_edges": ([TILE - 2, TILE - 1, 2 * TILE, 2 * TILE + 1, 3 * TILE - 1], []),
    "consecutive": ([100, 101, 102, 103], []),
    "last_row": ([-1], []),
    "zero_zero": ([], [TILE + 5]),
    "zero_zero_row0": ([], [0]),
    "scattered64": (None, []),
}


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("aim", list(AIMS))
def test_aimed_zero_denominators(ctx, oracle, d, aim):
    log_n = 16 if aim == "scattered64" else 13
    n = 1 << log_n
    rows, zz = AIMS[aim]
    if rows is None:
        rows = sorted(np.random.default_rng(d).choice(n - 1, size=64, replace=False).tolist())
    rows = [r % n for r in rows]
    desc, build, trace, rand = _aimed(oracle, n, d, rows, zz, 300 + d)
    want = rb.reference(desc, build, trace, rand)
    # the zeros are where they were aimed: a0 is 0 on the row after each one (and only there, row n - 1 has no successor)
    zeros = {i + 1 for i in rows + zz if i + 1 < n}
    assert {i for i in range(n) if not want[0, i].any()} == zeros
    got, launches = _build(ctx, desc, build, trace, rand, d, aw=2)
    _assert_columns(got, want)
    # column 0: one rescan per aimed row before n - 1 (each from the zero on); column 1 has no zero
    assert launches == 2 * 4 + 3 * len(zeros)
    if aim == "last_row":
        b = trace.copy()
        b[3, n - 1] = (int(b[3, n - 1]) + 1) % P
        assert np.array_equal(want, rb.reference(desc, build, b, rand))
    assert ctx.mem_stats()[0] == 0


def _dev_trace(trace):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(trace).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


@pytest.mark.parametrize("ext,hash_id", [(1, 0), (2, 0), (3, 0), (1, 1), (2, 1), (3, 1)])
def test_example_air_proofs(ctx, oracle, ext, hash_id):
    n = 256
    desc, trace, build, builder = ra.rational(n)
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


@pytest.mark.parametrize("ext", [1, 2, 3])
def test_example_air_proofs_with_vanishing_denominators(ctx, oracle, ext):
    # a 0/0 row keeps the trace valid; a plain zero breaks G's constraint, and the proof is still the host builder's
    n = 256
    opts = oracle.make_opts(num_queries=20, blowup=8, grinding=0, ext=ext, folding=4, rem_max_deg=7, hash_id=0)
    for zeros, zz in (((), (0, 63, 64)), ((17, 18), (100,))):
        desc, trace, build, builder = ra.rational(n, zeros=zeros, zero_zero=zz)
        ref = ctx.prove_air_aux(desc, trace, opts, builder, AW, NR)
        got = ctx.prove_air_aux_built(desc, build, trace, opts)
        assert got == ref == oracle.prove_air_aux(desc, trace, opts, builder, AW, NR)
        assert (oracle.verify_air(desc, got, 0) == 0) == (not zeros)
    assert ctx.mem_stats()[0] == 0


def test_example_air_batch(ctx, oracle):
    n = 512
    cases = [ra.rational(n, seed=1), ra.rational(n, seed=2, zero_zero=(40,)), ra.rational(n, seed=3, zeros=(7,))]
    build = cases[0][2]
    opts = oracle.make_opts(num_queries=24, blowup=8, grinding=0, ext=3, folding=8, rem_max_deg=15, hash_id=1)
    singles = [ctx.prove_air_aux_built(desc, build, tr, opts) for desc, tr, _, _ in cases]
    assert singles == [ctx.prove_air_aux(desc, tr, opts, b, AW, NR) for desc, tr, _, b in cases]
    got = ctx.prove_air_batch([c[0] for c in cases], [c[1] for c in cases], opts, aux_build=build)
    assert got == singles
    import torch
    dev = torch.from_numpy(np.stack([c[1] for c in cases]).view(np.int64)).cuda().contiguous()
    assert ctx.prove_air_batch([c[0] for c in cases], dev, opts, aux_build=build, device=True) == singles
    assert list(ctx.verify_air_batch([c[0] for c in cases], got, 1))[:2] == [wf.VERIFY_ACCEPT] * 2
    assert ctx.mem_stats()[0] == 0


def _sharded(world, cases):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    here = os.path.dirname(os.path.abspath(__file__))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(here, "rational_sharded_worker.py"), json.dumps(cases)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ))
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-6000:]
    for i in range(len(cases)):
        assert f"case {i} ok" in r.stdout, out[-6000:]


def test_example_air_sharded_world_2():
    _sharded(2, [{"air": "rational", "log_n": 12, "ext": 3, "fri_min_log": 5},
                 {"air": "rational", "log_n": 11, "ext": 2, "hash": 1, "trace": "device"},
                 {"air": "rational", "log_n": 11, "ext": 1, "trace": "mont"}])


def test_example_air_sharded_world_4():
    _sharded(4, [{"air": "rational", "log_n": 12, "ext": 2, "fri_min_log": 5},
                 {"air": "rational", "log_n": 11, "ext": 3, "hash": 1, "trace": "device"}])


@pytest.mark.parametrize("ext", [1, 2, 3])
def test_example_air_validation(ctx, oracle, ext):
    n = 64
    rand = oracle.rand_elems((NR, ext), 70 + ext)
    o = oracle.make_opts(num_queries=20, blowup=8, grinding=0, ext=ext, folding=4, rem_max_deg=7)
    for zeros, zz in (((), ()), ((), (9,)), ((37,), ())):
        desc, tr, build, _ = ra.rational(n, zeros=zeros, zero_zero=zz)
        want = R.validate(desc, tr, rb.reference(desc, build, tr, rand), rand, ext)
        assert (want["kind"] == R.VALID) == (not zeros)
        rep = ctx.trace_validate(desc, tr, ext, rand=rand, aux_build=build)
        for k in ("kind", "index", "step", "column", "first_failing_step", "expected_degrees", "actual_degrees", "msg"):
            assert rep[k] == want[k], (k, rep[k], want[k])
        if zeros:
            assert (want["kind"], want["index"], want["step"]) == (R.AUX_TRANSITION, 1, 37)
        # the provers' validation switch: the same bytes for a valid trace, the reference's message for the broken one
        off = ctx.prove_air_aux_built(desc, build, tr, o)
        ctx.set_validation(1)
        try:
            if zeros:
                with pytest.raises(wf.WfError) as e:
                    ctx.prove_air_aux_built(desc, build, tr, o)
                assert "did not evaluate to ZERO at step 37" in str(e.value)
            else:
                assert ctx.prove_air_aux_built(desc, build, tr, o) == off
                assert ctx.prove_air_batch([desc, desc], [tr, tr], o, aux_build=build) == [off, off]
        finally:
            ctx.set_validation(0)
    assert ctx.mem_stats()[0] == 0


def test_invalid_rational_builds_fail_and_leave_no_buffers(oracle):
    c = wf.Context(0)
    try:
        n = 64
        desc, trace, build, _ = ra.rational(n)
        opts = oracle.make_opts(num_queries=8, blowup=8, grinding=0, ext=2, folding=4, rem_max_deg=7, hash_id=0)

        def col1(fn):
            B = rb.AuxBuild(5, AW, 0, NR)
            f = B.column(rb.RATIONAL_RECURRENCE)
            f.multiplier(f.rnd(0))
            f.num(f.cur(0))
            f.den_multiplier(f.const(1))
            f.den(f.rnd(1))
            fn(B.column(rb.RATIONAL_RECURRENCE))
            h = B.column(rb.RUNNING_SUM)
            h.num(h.mul(h.acur(0), h.acur(1)))
            return B.build()

        main = c.mat_from_host_columns(trace)
        rand = oracle.rand_elems((NR, 2), 3)
        for b, why in ((col1(lambda x: (x.multiplier(x.cur(1)), x.num(x.cur(0)))), "has no denominator multiplier (OUT 3)"),
                       (col1(lambda x: (x.den_multiplier(x.cur(1)), x.num(x.cur(0)))), "has no multiplier (OUT 2)"),
                       (col1(lambda x: (x.multiplier(x.cur(1)), x.den_multiplier(x.cur(2)), x.den_multiplier(x.cur(2)),
                                        x.num(x.cur(0)))), "more than one denominator multiplier"),
                       (col1(lambda x: (x.multiplier(x.cur(1)), x.den_multiplier(x.cur(2)), x.num(x.cur(0)),
                                        x.prog.append((airs.OUT, 4, x.cur(0), 0)))), "nor denominator multiplier (3)")):
            for fn in (lambda: c.prove_air_aux_built(desc, b, trace, opts), lambda: c.aux_build(desc, b, main, rand, 2),
                       lambda: c.prove_air_batch([desc], [trace], opts, aux_build=b),
                       lambda: c.trace_validate(desc, trace, 2, rand=rand, aux_build=b)):
                with pytest.raises(wf.WfError, match="error -2"):
                    fn()
                assert why in c.L.wf_last_error(c.h).decode()
                assert c.mem_stats()[0] == 1                  # the main matrix the test holds
        bad = build.copy()
        bad[3 + 6 + 20 + 2] = 5                               # column 1's init word 1 with ext 1
        with pytest.raises(wf.WfError, match="error -2"):
            c.prove_air_aux_built(desc, bad, trace, oracle.make_opts(num_queries=8, ext=1))
        assert "beyond the extension degree" in c.L.wf_last_error(c.h).decode()
        main.free()
        assert c.mem_stats()[0] == 0
    finally:
        c.close()
