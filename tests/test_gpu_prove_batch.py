"""wf_prove_air_batch: proofs of one AIR structure in one call.
- every proof of a batch is byte-identical to the single-proof entry point on its own inputs (wf_prove_air, or
  wf_prove_air_aux_built for perm_rap) and to the oracle's prover, and the oracle's verifier accepts it; batches of 1, 2, 3 and
  17 proofs, ext 1 / 2 / 3, all five hashers, partitions, folding 2 / 4 / 8 / 16, the three batching methods, grinding,
  blowup 2 to 16, 2^3 to 2^13 rows, host traces, device traces and Montgomery input;
- the proofs are independent: reversing the batch reverses the output, swapping one trace changes only that proof;
- a batch compiles its constraint kernel once; that its launches do not grow with the batch is checked as an expected failure
  (the proofs of a batch still run one after another);
- a refused batch (structure mismatch, too small a proof buffer) writes nothing and leaves no device buffer live."""
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


def fib_pair(n, a0, b0):
    """examples/src/fibonacci/fib_small with the starting pair (a0, b0): the assertion values and the public result differ
    per starting pair, the structure does not"""
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


def sequence_var(n, a0, b0, stride=4):
    """airs.sequence_mix from the starting pair (a0, b0): different sequence-assertion values per proof"""
    tr = np.zeros((3, n), dtype=np.uint64)
    a, b = a0, b0
    for i in range(n):
        tr[0, i], tr[1, i], tr[2, i] = a, b, 7 if i % stride == 1 else (i % 5)
        a = (a * a + b) % P
        b = (b + a) % P
    A = airs.AirBuilder(3)
    A.pub = [int(tr[1, n - 1])]
    A.constraint(A.sub(A.nxt(0), A.add(A.mul(A.cur(0), A.cur(0)), A.cur(1))), 2)
    A.constraint(A.sub(A.nxt(1), A.add(A.cur(1), A.nxt(0))), 1)
    A.assert_single(0, 0, a0)
    A.assert_single(1, 0, b0)
    A.assert_single(1, n - 1, int(tr[1, n - 1]))
    A.assert_sequence(0, 1, stride, [int(v) for v in tr[0, 1::stride]])
    A.assert_periodic(2, 1, stride, 7)
    A.assert_sequence(2, 0, n // 2, [int(tr[2, 0]), int(tr[2, n // 2])])
    return A.build(), tr


def _inputs(air, batch, n):
    """[(desc, trace)] * batch; the structure is shared, the values differ where the AIR allows it"""
    if air == "fib":
        return [fib_pair(n, 1 + 3 * j, 2 + 5 * j) for j in range(batch)]
    if air == "sequence":
        return [sequence_var(n, 2 + j, 3 + 7 * j) for j in range(batch)]
    if air == "perm_rap":
        return [airs.perm_rap(n, seed=5 + j)[:2] for j in range(batch)]
    one = getattr(airs, air)(n)[:2]
    return [one] * batch


def _to_mont(trace):
    L = wf.lib()
    return np.vectorize(lambda v: L.wf_host_canonical_to_mont(int(v)), otypes=[np.uint64])(trace)


def _dev(traces):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(np.stack(traces)).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return t


# (air, batch, log_n, options, trace input)
CASES = [
    ("fib", 1, 3, dict(ext=1, hash_id=wf.HASH_BLAKE3_256, folding=2, rem_max_deg=3, blowup=8, num_queries=16), "host"),
    ("fib", 2, 6, dict(ext=2, hash_id=wf.HASH_RP64_256, folding=4, rem_max_deg=7, blowup=4, grinding=6, batch_c=1, batch_d=2), "mont"),
    ("fib", 3, 13, dict(ext=3, hash_id=wf.HASH_BLAKE3_192, folding=8, rem_max_deg=31, blowup=8, grinding=8), "device"),
    ("fib", 17, 5, dict(ext=1, hash_id=wf.HASH_SHA3_256, folding=16, rem_max_deg=15, blowup=16, num_partitions=2, hash_rate=1), "host"),
    ("mulfib2", 2, 6, dict(ext=2, hash_id=wf.HASH_RPJIVE64_256, folding=4, rem_max_deg=7, blowup=2, batch_c=2), "host"),
    ("periodic_mix", 2, 7, dict(ext=3, hash_id=wf.HASH_BLAKE3_256, folding=2, rem_max_deg=7, blowup=16, batch_d=1), "device"),
    ("sequence", 3, 8, dict(ext=2, hash_id=wf.HASH_BLAKE3_256, folding=8, rem_max_deg=7, blowup=8, grinding=5, batch_c=2), "host"),
    ("rescue_like", 2, 6, dict(ext=1, hash_id=wf.HASH_RP64_256, folding=4, rem_max_deg=7, blowup=8, num_partitions=2, hash_rate=8), "mont"),
    ("perm_rap", 3, 7, dict(ext=3, hash_id=wf.HASH_BLAKE3_256, folding=4, rem_max_deg=7, blowup=8, grinding=3, batch_c=1), "host"),
    ("perm_rap", 2, 12, dict(ext=2, hash_id=wf.HASH_RP64_256, folding=8, rem_max_deg=31, blowup=8, grinding=4, num_partitions=2, hash_rate=8),
     "device"),
]


@pytest.mark.parametrize("air,batch,log_n,kw,mode", CASES, ids=[f"{c[0]}-B{c[1]}-n{c[2]}-{c[4]}" for c in CASES])
def test_batch_equals_single_proofs_and_oracle(ctx, oracle, air, batch, log_n, kw, mode):
    n = 1 << log_n
    kw = dict(kw)
    kw.setdefault("num_queries", 24)
    opts = oracle.make_opts(**kw)
    inputs = _inputs(air, batch, n)
    descs = [d for d, _ in inputs]
    traces = [t for _, t in inputs]
    assert wf.air_batch_check(descs, log_n, kw["blowup"]) == (0, "")
    build = ab.perm_rap_build() if air == "perm_rap" else None
    if mode == "device":
        got = ctx.prove_air_batch(descs, _dev(traces), opts, aux_build=build, device=True)
    elif mode == "mont":
        got = ctx.prove_air_batch(descs, [_to_mont(t) for t in traces], opts, mont=True, aux_build=build)
    else:
        got = ctx.prove_air_batch(descs, traces, opts, aux_build=build)
    assert len(got) == batch
    for j, (d, t) in enumerate(inputs):
        if build is not None:
            single = ctx.prove_air_aux_built(d, build, t, opts)
            _, _, builder = airs.perm_rap(n, seed=5 + j)
            want = oracle.prove_air_aux(d, t, opts, builder, airs.PERM_RAP_AUX_WIDTH, 2)
        else:
            single = ctx.prove_air(d, t, opts)
            want = oracle.prove_air(d, t, opts)
        assert got[j] == single, j
        assert got[j] == want, j
        assert oracle.verify_air(d, got[j], kw["hash_id"]) == 0, j
    if kw.get("grinding", 0) and air in ("fib", "sequence", "perm_rap") and batch > 1:
        assert len({p[-8:] for p in got}) > 1          # the nonces are each proof's own
    assert ctx.mem_stats()[0] == 0


def test_proofs_are_independent(ctx, oracle):
    n = 64
    opts = oracle.make_opts(num_queries=20, ext=2, folding=4, rem_max_deg=7, grinding=2)
    inputs = _inputs("fib", 4, n)
    descs, traces = [d for d, _ in inputs], [t for _, t in inputs]
    fwd = ctx.prove_air_batch(descs, traces, opts)
    assert len(set(fwd)) == 4
    assert ctx.prove_air_batch(descs[::-1], traces[::-1], opts) == fwd[::-1]
    d2, t2 = fib_pair(n, 11, 13)
    swapped = ctx.prove_air_batch(descs[:2] + [d2] + descs[3:], traces[:2] + [t2] + traces[3:], opts)
    assert swapped[:2] == fwd[:2] and swapped[3] == fwd[3] and swapped[2] != fwd[2]
    assert swapped[2] == ctx.prove_air(d2, t2, opts)


def test_batch_compiles_its_constraint_kernel_once(oracle):
    c = wf.Context(0)
    try:
        opts = oracle.make_opts(num_queries=20, ext=2, folding=4, rem_max_deg=7, grinding=0)
        inputs = _inputs("sequence", 4, 256)
        s0 = c.jit_stats()
        c.prove_air_batch([d for d, _ in inputs], [t for _, t in inputs], opts)
        s1 = c.jit_stats()
        assert s1["compiled"] - s0["compiled"] + s1["fallbacks"] - s0["fallbacks"] == 1   # one kernel for the whole batch
        if s1["compiled"] > s0["compiled"]:
            assert s1["cache_hits"] - s0["cache_hits"] == 3
    finally:
        c.close()


@pytest.mark.xfail(strict=True, reason="the proofs of a batch run one after another: launches grow with the batch until the "
                                       "lockstep orchestration is built (DESIGN section 8)")
def test_launches_per_batch_do_not_grow_with_the_batch(ctx, oracle):
    opts = oracle.make_opts(num_queries=20, ext=2, folding=4, rem_max_deg=7, grinding=0)
    inputs = _inputs("fib", 32, 64)
    ctx.prove_air_batch([inputs[0][0]], [inputs[0][1]], opts)   # tables and constraint kernel of this shape
    launches = {}
    for B in (1, 4, 32):
        l0 = ctx.launches
        ctx.prove_air_batch([d for d, _ in inputs[:B]], [t for _, t in inputs[:B]], opts)
        launches[B] = ctx.launches - l0
    assert launches[1] == launches[4] == launches[32], launches


def test_refused_batches_write_nothing_and_free_everything(ctx, oracle):
    n = 64
    opts = oracle.make_opts(num_queries=20, ext=2, folding=4, rem_max_deg=7)
    (d0, t0), (d1, t1) = _inputs("fib", 2, n)
    good = ctx.prove_air_batch([d0, d1], [t0, t1], opts)
    assert ctx.mem_stats()[0] == 0
    dm, tm = airs.mulfib2(n)
    with pytest.raises(wf.WfError, match="proof 1 differs from proof 0"):
        ctx.prove_air_batch([d0, dm], [t0, tm], opts)
    assert ctx.mem_stats()[0] == 0
    with pytest.raises(wf.WfError, match="proof 0: proof buffer too small"):
        ctx.prove_air_batch([d0, d1], [t0, t1], opts, proof_cap=len(good[0]) - 1)
    assert ctx.mem_stats()[0] == 0
    desc, trace, _ = airs.perm_rap(n)
    with pytest.raises(wf.WfError, match="builds its aux segments from aux_build"):
        ctx.prove_air_batch([desc], [trace], opts)
    assert ctx.mem_stats()[0] == 0
    assert ctx.prove_air_batch([d0, d1], [t0, t1], opts) == good
