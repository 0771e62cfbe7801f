"""COUPLED_RECURRENCE groups (a[i+1] = M_i a[i] + t_i over k = 2..4 aux columns) built on the device:
- the columns against the CPU reference (tests/coupled_build_ref.cpp) for k in {2, 3, 4}, D in {1, 2, 3} and n from 8 rows
  (below one scan tile) through 2^11 (one tile) to 2^22, with maps of main columns, random elements and an earlier column at
  rows i and i + 1, unwritten (zero) slots, and inits non-zero in every word;
- a diagonal M bit for bit k LINEAR_RECURRENCE columns; a 2-group with t = 0 and init (a0, 1) is the projective form of the
  RATIONAL_RECURRENCE column of the same map (y_i r_i = x_i);
- aimed structure: zero maps at row 0, on and around tile edges and at row n - 1, identity maps over runs, singular M;
- one term launch and three scan launches per group, no buffer live after any return;
- proofs of the example AIR (tests/coupled_airs.py) through every entry point that builds an aux segment, byte-identical to
  wf_prove_air_aux with the CPU reference as host builder and to the oracle, accepted by the oracle verifier and
  wf_verify_air_batch;
- wf_trace_validate with the build, and invalid builds."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import airs
import coupled_airs as ca
import coupled_builds as cb
import trace_validate_ref as R
import winterfell_b200 as wf
from test_aux_coupled_check import generic_group, trivial_air
from test_aux_linrec_check import e_mul

pytestmark = pytest.mark.gpu
P = wf.P
AW, NR = ca.COUPLED_AUX_WIDTH, ca.COUPLED_NUM_RANDS
TILE = 2048   # AUX_SCAN_TILE


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


def _inits(oracle, k, d, s):
    """k inits, non-zero in every one of their d words"""
    v = oracle.rand_elems((k, d), s)
    v[v == 0] = 1
    return [tuple(int(x) for x in row) + (0,) * (3 - d) for row in v]


def _build(ctx, desc, build, trace, rand, d, aw):
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


CASES = [(k, d, log_n) for k in (2, 3, 4) for d in (1, 2, 3) for log_n in (3, 11, 12, 16)] + [(2, 1, 22), (4, 3, 22)]


@pytest.mark.parametrize("k,d,log_n", CASES)
def test_coupled_columns_match_reference(ctx, oracle, k, d, log_n):
    n = 1 << log_n
    inits = _inits(oracle, k, d, 7 * k + d)
    desc, build = generic_group(k, inits)
    assert wf.aux_build_check(desc, build, log_n) == (0, "")
    trace = oracle.rand_elems((4, n), 10 * log_n + k + d)
    rand = oracle.rand_elems((2, d), 3 * k + d)
    got, launches = _build(ctx, desc, build, trace, rand, d, k + 2)
    want = cb.reference(desc, build, trace, rand)
    _assert_columns(got, want)
    assert launches == 1 + 4 + 4          # POINTWISE: a term kernel; the group and the running sum: a term and three scans each
    assert ctx.mem_stats()[0] == 0


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("k", [2, 3, 4])
def test_diagonal_group_equals_linear_recurrences(ctx, oracle, k, d):
    n = 1 << 12
    trace = oracle.rand_elems((5, n), 40 + k + d)
    rand = oracle.rand_elems((2, d), 50 + k + d)
    inits = _inits(oracle, k, d, 60 + k + d)
    Bd = cb.AuxBuild(5, 2 * k, 0, 2)
    g = Bd.group(k, inits)
    for r in range(k):                     # a_r' = (x_r + alpha) a_r + x_{r+1} beta
        g.m(r, r, g.add(g.cur(r), g.rnd(0)))
        g.t(r, g.mul(g.cur(r + 1), g.rnd(1)))
    for r in range(k):
        c = Bd.column(cb.LINEAR_RECURRENCE, inits[r])
        c.multiplier(c.add(c.cur(r), c.rnd(0)))
        c.num(c.mul(c.cur(r + 1), c.rnd(1)))
    desc, build = trivial_air(5, 2 * k, 2), Bd.build()
    got, launches = _build(ctx, desc, build, trace, rand, d, 2 * k)
    assert launches == 4 + 4 * k
    assert np.array_equal(got[:k], got[k:])
    assert np.array_equal(got, cb.reference(desc, build, trace, rand))


@pytest.mark.parametrize("d", [1, 2, 3])
def test_projective_pair_matches_rational_recurrence(ctx, oracle, d):
    # (x, y)' = [[m, n], [c, d]] (x, y), (x, y)[0] = (a0, 1): the projective pair of r' = (m r + n) / (c r + d), r[0] = a0, so
    # y_i r_i = x_i while no denominator vanishes (random maps: none does)
    n = 1 << 13
    trace = oracle.rand_elems((4, n), 70 + d)
    rand = oracle.rand_elems((1, d), 80 + d)
    a0 = _inits(oracle, 1, d, 90 + d)[0]
    Bd = cb.AuxBuild(4, 3, 0, 1)
    g = Bd.group(2, [a0, (1, 0, 0)])
    regs = [g.add(g.cur(0), g.rnd(0)), g.cur(1), g.cur(2), g.mul(g.cur(3), g.rnd(0))]
    for s, reg in enumerate(regs):
        g.m(s // 2, s % 2, reg)
    r = Bd.column(cb.RATIONAL_RECURRENCE, a0)
    r.multiplier(r.add(r.cur(0), r.rnd(0)))
    r.num(r.cur(1))
    r.den_multiplier(r.cur(2))
    r.den(r.mul(r.cur(3), r.rnd(0)))
    desc, build = trivial_air(4, 3, 1), Bd.build()
    got, launches = _build(ctx, desc, build, trace, rand, d, 3)
    assert launches == 4 + 4                # no rescan: no denominator vanishes
    assert np.array_equal(got, cb.reference(desc, build, trace, rand))
    for i in range(n):
        y, rr = tuple(int(v) for v in got[1, i]), tuple(int(v) for v in got[2, i])
        assert e_mul(y, rr) == tuple(int(v) for v in got[0, i]), i
    assert ctx.mem_stats()[0] == 0


def _aimed(oracle, n, k, d, zero_rows, id_rows, seed):
    """main columns x0..x3, s, e; the group's map at row i is s_i (the generic map) + e_i (I, t = 0): s = e = 0 a zero map
    (a[i+1] = 0), s = 0, e = 1 the identity (a[i+1] = a[i])"""
    trace = oracle.rand_elems((6, n), seed)
    trace[4] = 1
    trace[5] = 0
    for i in zero_rows:
        trace[4, i] = 0
    for i in id_rows:
        trace[4, i], trace[5, i] = 0, 1
    rand = oracle.rand_elems((2, d), seed + 1)
    Bd = cb.AuxBuild(6, k, 0, 2)
    g = Bd.group(k, _inits(oracle, k, d, seed + 2))
    s, e = g.cur(4), g.cur(5)
    for r in range(k):
        for c in range(k):
            v = g.mul(s, g.add(g.cur((r + 2 * c) % 4), g.rnd((r + c) % 2)))
            g.m(r, c, g.add(v, e) if r == c else v)
        g.t(r, g.mul(s, g.cur(r % 4)))
    return trivial_air(6, k, 2), Bd.build(), trace, rand


AIMS = {
    "zero_row0": ([0], []),
    "zero_tile_edges": ([TILE - 2, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 3 * TILE - 1], []),
    "zero_consecutive": (list(range(100, 110)), []),
    "zero_last_row": ([-1], []),
    "identity_runs": ([], list(range(5, 300)) + list(range(TILE - 3, TILE + 4)) + list(range(3 * TILE - 40, 3 * TILE + 40))),
    "identity_all": ([], None),
}


@pytest.mark.parametrize("d", [1, 3])
@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("aim", list(AIMS))
def test_aimed_structure(ctx, oracle, aim, k, d):
    n = 1 << 13
    zr, ir = AIMS[aim]
    zr = [i % n for i in zr]
    ir = list(range(n)) if ir is None else ir
    desc, build, trace, rand = _aimed(oracle, n, k, d, zr, ir, 500 + k + d)
    want = cb.reference(desc, build, trace, rand)
    for i in zr:                            # a zero map: the state after it is 0 (row n - 1 has no successor)
        if i + 1 < n:
            assert not want[:, i + 1].any()
    for i in ir:                            # the identity: the state carries over
        if i + 1 < n:
            assert np.array_equal(want[:, i + 1], want[:, i])
    got, launches = _build(ctx, desc, build, trace, rand, d, k)
    _assert_columns(got, want)
    assert launches == 4
    assert ctx.mem_stats()[0] == 0


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("k", [2, 3, 4])
def test_singular_maps(ctx, oracle, k, d):
    # M_i = u_i w_i^T (rank one) on every row: the state lies on the line of u after the first row
    n = 1 << 12
    trace = oracle.rand_elems((4, n), 600 + k + d)
    rand = oracle.rand_elems((2, d), 610 + k + d)
    Bd = cb.AuxBuild(4, k, 0, 2)
    g = Bd.group(k, _inits(oracle, k, d, 620 + k + d))
    u = [g.add(g.cur(r % 4), g.rnd(r % 2)) for r in range(k)]
    w = [g.cur((c + 1) % 4) for c in range(k)]
    for r in range(k):
        for c in range(k):
            g.m(r, c, g.mul(u[r], w[c]))
    desc, build = trivial_air(4, k, 2), Bd.build()
    got, _ = _build(ctx, desc, build, trace, rand, d, k)
    assert np.array_equal(got, cb.reference(desc, build, trace, rand))


def _dev_trace(trace):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(trace).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


@pytest.mark.parametrize("ext,hash_id", [(1, 0), (2, 0), (3, 0), (1, 1), (2, 1), (3, 1)])
def test_example_air_proofs(ctx, oracle, ext, hash_id):
    n = 256
    desc, trace, build, builder = ca.coupled(n)
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
    cases = [ca.coupled(n, seed=s) for s in (1, 2, 3)]
    build = cases[0][2]
    opts = oracle.make_opts(num_queries=24, blowup=8, grinding=0, ext=3, folding=8, rem_max_deg=15, hash_id=1)
    singles = [ctx.prove_air_aux_built(desc, build, tr, opts) for desc, tr, _, _ in cases]
    assert singles == [ctx.prove_air_aux(desc, tr, opts, b, AW, NR) for desc, tr, _, b in cases]
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
           "--master-port", str(port), os.path.join(here, "coupled_sharded_worker.py"), json.dumps(cases)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ))
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-6000:]
    for i in range(len(cases)):
        assert f"case {i} ok" in r.stdout, out[-6000:]


def test_example_air_sharded_world_2():
    _sharded(2, [{"air": "coupled", "log_n": 12, "ext": 3, "fri_min_log": 5},
                 {"air": "coupled", "log_n": 12, "ext": 3, "fri_min_log": 5, "validation": 1},
                 {"air": "coupled", "log_n": 11, "ext": 2, "hash": 1, "trace": "device", "validation": 1},
                 {"air": "coupled", "log_n": 11, "ext": 1, "trace": "mont"}])


def test_example_air_sharded_world_4():
    _sharded(4, [{"air": "coupled", "log_n": 12, "ext": 2, "fri_min_log": 5, "validation": 1},
                 {"air": "coupled", "log_n": 11, "ext": 3, "hash": 1, "trace": "device"}])


def _col_start(build, j):
    q = 2 + int(build[1])
    for _ in range(j):
        q += 6 + 4 * int(build[q + 5])
    return q


@pytest.mark.parametrize("ext", [1, 2, 3])
def test_example_air_validation(ctx, oracle, ext):
    n = 64
    rand = oracle.rand_elems((NR, ext), 70 + ext)
    o = oracle.make_opts(num_queries=20, blowup=8, grinding=0, ext=ext, folding=4, rem_max_deg=7)
    desc, tr, build, _ = ca.coupled(n)
    for b, broken in ((build, False), (ca.coupled_build(broken_at=37), True)):
        aux = cb.reference(desc, b, tr, rand)
        if broken:
            good = cb.reference(desc, build, tr, rand)
            assert [i for i in range(n) if not np.array_equal(aux[:, i], good[:, i])][:1] == [37]
        want = R.validate(desc, tr, aux, rand, ext)
        assert (want["kind"] == R.VALID) == (not broken)
        rep = ctx.trace_validate(desc, tr, ext, rand=rand, aux_build=b)
        for k in ("kind", "index", "step", "column", "first_failing_step", "expected_degrees", "actual_degrees", "msg"):
            assert rep[k] == want[k], (k, rep[k], want[k])
        if broken:
            assert (want["kind"], want["step"]) == (R.AUX_TRANSITION, 37)
        off = ctx.prove_air_aux_built(desc, b, tr, o)
        ctx.set_validation(1)
        try:
            if broken:
                with pytest.raises(wf.WfError) as e:
                    ctx.prove_air_aux_built(desc, b, tr, o)
                assert "did not evaluate to ZERO at step 37" in str(e.value)
            else:
                assert ctx.prove_air_aux_built(desc, b, tr, o) == off
                assert ctx.prove_air_batch([desc, desc], [tr, tr], o, aux_build=b) == [off, off]
        finally:
            ctx.set_validation(0)
    assert ctx.mem_stats()[0] == 0


def test_invalid_coupled_builds_fail_and_leave_no_buffers(oracle):
    c = wf.Context(0)
    try:
        n = 64
        desc, trace, build, _ = ca.coupled(n)
        opts = oracle.make_opts(num_queries=8, blowup=8, grinding=0, ext=2, folding=4, rem_max_deg=7, hash_id=0)
        lead, member = _col_start(build, ca.A), _col_start(build, ca.B)

        def patched(at, v):
            b = build.copy()
            b[at] = v
            return b
        bad_slot = build.copy()
        bad_slot[lead + 6 + 1] = 4 + 4 * 2   # the leader's first OUT (M[0][0]) -> M[2][0] in a 2-group
        assert build[lead + 6] == airs.OUT
        cases = [(patched(member, cb.POINTWISE), "fewer than 2 or more than 4 columns"),   # (A, B) -> a group of one
                 (patched(_col_start(build, ca.W), cb.COUPLED_MEMBER), "does not follow a COUPLED_RECURRENCE column"),
                 (patched(member + 4, 1), "has registers or instructions"),
                 (bad_slot, "outside the group's t")]
        main = c.mat_from_host_columns(trace)
        rand = oracle.rand_elems((NR, 2), 3)
        for b, why in cases:
            for fn in (lambda: c.prove_air_aux_built(desc, b, trace, opts), lambda: c.aux_build(desc, b, main, rand, 2),
                       lambda: c.prove_air_batch([desc], [trace], opts, aux_build=b),
                       lambda: c.trace_validate(desc, trace, 2, rand=rand, aux_build=b)):
                with pytest.raises(wf.WfError, match="error -2"):
                    fn()
                assert why in c.L.wf_last_error(c.h).decode()
                assert c.mem_stats()[0] == 1                  # the main matrix the test holds
        bad = build.copy()
        bad[member + 2] = 5                                   # the member's init word 1 with ext 1
        with pytest.raises(wf.WfError, match="error -2"):
            c.prove_air_aux_built(desc, bad, trace, oracle.make_opts(num_queries=8, ext=1))
        assert "beyond the extension degree" in c.L.wf_last_error(c.h).decode()
        main.free()
        assert c.mem_stats()[0] == 0
    finally:
        c.close()
