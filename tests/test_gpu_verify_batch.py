"""wf_verify_air_batch: verifier::verify for a batch of proofs of one AIR, against the oracle's verifier.
- acceptance: proofs of every proving entry point, the AIRs of tests/airs.py, all five hashers, ext 1 / 2 / 3, partitions,
  folding 2 / 4 / 8 / 16, the batching methods, grinding, blowup 2 to 16, 2^3 to 2^13 rows and one 2^18-row proof;
- refusals: the mutation set of test_oracle_verifier_soundness.py, each proof's mutations in one call, every verdict equal to
  the oracle's (where the mutated trace length does not fit the AIR the reference panics in Air::new: CONTEXT here);
- independence of the proofs of a batch, mixed trace lengths, acceptable options, launches that do not grow with the batch,
  1024 proofs, and no device buffer left live after any return."""
import numpy as np
import pytest

import airs
import aux_builds as ab
import winterfell_b200 as wf

pytestmark = pytest.mark.gpu
P = wf.P
HASH_RATE_BYTE = 24


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


def fib_pair(n, a0, b0, last=True):
    """fib_small from (a0, b0); last=False drops the assertion at step n - 1 so that one description fits every length"""
    tr = np.zeros((2, n), dtype=np.uint64)
    a, b = a0, b0
    for i in range(n):
        tr[0, i], tr[1, i] = a, b
        a = (a + b) % P
        b = (b + a) % P
    A = airs.AirBuilder(2)
    A.pub = [int(tr[1, n - 1])] if last else []
    A.constraint(A.sub(A.nxt(0), A.add(A.cur(0), A.cur(1))), 1)
    A.constraint(A.sub(A.nxt(1), A.add(A.cur(1), A.nxt(0))), 1)
    A.assert_single(0, 0, a0)
    A.assert_single(1, 0, b0)
    if last:
        A.assert_single(1, n - 1, int(tr[1, n - 1]))
    return A.build(), tr


def _expected(oracle_code, desc, proof):
    """the oracle's verdict, except that a proof whose declared length the AIR does not fit is CONTEXT once it parses"""
    if oracle_code in (0, 2, 3, 4, 5, 6, 7, 8) and len(proof) > 16:
        rc, _ = wf.air_check(desc, proof[3], proof[16])
        if rc != 0:
            return wf.VERIFY_CONTEXT
    return oracle_code


# (air, log_n, options)
ACCEPT = [
    ("fib_small_x", 3, dict(ext=1, hash_id=0, folding=2, rem_max_deg=3, blowup=8, num_queries=16)),
    ("mulfib2", 6, dict(ext=2, hash_id=2, folding=4, rem_max_deg=7, blowup=2, batch_c=2)),
    ("periodic_mix", 7, dict(ext=3, hash_id=0, folding=2, rem_max_deg=7, blowup=16, batch_d=1)),
    ("sequence_mix", 8, dict(ext=2, hash_id=3, folding=8, rem_max_deg=7, blowup=8, grinding=5, batch_c=2)),
    ("rescue_like", 6, dict(ext=1, hash_id=1, folding=4, rem_max_deg=7, blowup=8, num_partitions=2, hash_rate=8)),
    ("fib_small_x", 13, dict(ext=3, hash_id=4, folding=16, rem_max_deg=15, blowup=4, grinding=3, batch_c=1, batch_d=2)),
    ("mulfib2", 10, dict(ext=1, hash_id=1, folding=8, rem_max_deg=31, blowup=4, batch_d=1)),
]


@pytest.mark.parametrize("air,log_n,kw", ACCEPT, ids=[f"{a}-n{l}-h{k['hash_id']}-e{k['ext']}" for a, l, k in ACCEPT])
def test_prove_air_proofs_are_accepted(ctx, oracle, air, log_n, kw):
    n = 1 << log_n
    kw = dict(kw)
    kw.setdefault("num_queries", 24)
    opts = oracle.make_opts(**kw)
    desc, trace = (airs.fib_small_x(2, n) if air == "fib_small_x" else getattr(airs, air)(n))[:2]
    proof = ctx.prove_air(desc, trace, opts)
    assert oracle.verify_air(desc, proof, kw["hash_id"]) == 0
    assert list(ctx.verify_air_batch([desc], [proof], kw["hash_id"])) == [0]
    assert ctx.mem_stats()[0] == 0


def test_prove_fib_and_batch_proofs_are_accepted(ctx, oracle):
    n = 1 << 9
    opts = oracle.make_opts(num_queries=20, ext=2, folding=4, rem_max_deg=7, blowup=8, grinding=4, hash_id=1)
    tr, res = oracle.build_fib_trace(3, n)
    proof = ctx.prove_fib(tr, res, opts)
    desc, _ = airs.fib_small_x(3, n)
    assert list(ctx.verify_air_batch([desc], [proof], 1)) == [oracle.verify_air(desc, proof, 1)] == [0]
    inputs = [fib_pair(64, 1 + 3 * j, 2 + 5 * j) for j in range(5)]
    descs, traces = [d for d, _ in inputs], [t for _, t in inputs]
    proofs = ctx.prove_air_batch(descs, traces, opts)
    assert list(ctx.verify_air_batch(descs, proofs, 1)) == [0] * 5


def test_aux_proofs_are_accepted(ctx, oracle):
    for log_n, kw in ((7, dict(ext=3, hash_id=0, folding=4, rem_max_deg=7, blowup=8, grinding=3, batch_c=1)),
                      (12, dict(ext=2, hash_id=1, folding=8, rem_max_deg=31, blowup=8, num_partitions=2, hash_rate=8))):
        n = 1 << log_n
        opts = oracle.make_opts(num_queries=20, **kw)
        desc, trace, builder = airs.perm_rap(n)
        p_host = ctx.prove_air_aux(desc, trace, opts, builder, airs.PERM_RAP_AUX_WIDTH, 2)
        p_built = ctx.prove_air_aux_built(desc, ab.perm_rap_build(), trace, opts)
        for p in (p_host, p_built):
            assert oracle.verify_air(desc, p, kw["hash_id"]) == 0
            assert list(ctx.verify_air_batch([desc], [p], kw["hash_id"])) == [0]
    # random-dependent aux assertion values (wf_prove_air_aux_dyn), the callback told which proof it serves
    n = 1 << 6
    opts = oracle.make_opts(num_queries=20, ext=3, folding=4, rem_max_deg=7, blowup=8)
    desc, trace, builder = airs.perm_rap(n, dyn_last_q=True)
    nv = builder.num_values
    proof = ctx.prove_air_aux_dyn(desc, trace, opts, builder, builder.values_fn, airs.PERM_RAP_AUX_WIDTH, 2, nv)
    assert oracle.verify_air_dyn(desc, proof, 0, builder.values_fn, 2, nv, 3) == 0
    seen = []

    def fn(j, rand, vals):
        seen.append(j)
        return builder.values_fn(rand, vals)
    bad = bytearray(proof)
    bad[40] ^= 1
    got = ctx.verify_air_batch([desc] * 3, [proof, bytes(bad), proof], 0, aux_values_fn=fn)
    assert list(got) == [0, oracle.verify_air_dyn(desc, bytes(bad), 0, builder.values_fn, 2, nv, 3), 0]
    assert 0 in seen and 2 in seen
    with pytest.raises(wf.WfError, match="proof 0: aux assertion callback failed"):
        ctx.verify_air_batch([desc], [proof], 0, aux_values_fn=lambda j, r, v: 1 // 0)
    assert ctx.mem_stats()[0] == 0


def test_deep_tree(ctx, oracle):
    n = 1 << 18
    opts = oracle.make_opts(num_queries=28, ext=2, folding=8, rem_max_deg=31, blowup=4, hash_id=0)
    desc, trace = airs.fib_small_x(1, n)
    proof = ctx.prove_air(desc, trace, opts)
    assert list(ctx.verify_air_batch([desc], [proof], 0)) == [oracle.verify_air(desc, proof, 0)] == [0]


@pytest.mark.parametrize("h,ext", [(0, 1), (1, 2), (3, 3), (2, 2), (4, 1)])
def test_refusals_equal_the_oracle(ctx, oracle, h, ext):
    n = 128
    desc, trace = airs.fib_small_x(1, n)
    opts = oracle.make_opts(num_queries=12, blowup=8, grinding=2, ext=ext, folding=4, rem_max_deg=7, hash_id=h)
    proof = ctx.prove_air(desc, trace, opts)
    rng = np.random.default_rng(h * 10 + ext)
    L = len(proof)
    muts = []
    for i in sorted(set(range(0, 160)) | set(range(L - 160, L)) | set(range(160, L - 160, 4))):
        b = bytearray(proof)
        b[i] ^= 1 << int(rng.integers(0, 8))
        muts.append(bytes(b))
    muts += [proof[:cut] for cut in (0, 1, 14, 15, 25, L // 2, L - 8, L - 1)] + [proof + b"\x00"]
    wrap = bytearray(proof)
    wrap[3] += 64
    zero_rate = bytearray(proof)
    zero_rate[HASH_RATE_BYTE] = 0
    muts += [bytes(wrap), bytes(zero_rate), proof]
    want = [_expected(oracle.verify_air(desc, m, h), desc, m) for m in muts]
    got = ctx.verify_air_batch([desc] * len(muts), muts, h)
    assert list(got) == want
    assert want[-1] == 0 and sum(w == 0 for w in want) >= 1
    # wrong public inputs
    d2, _ = fib_pair(n, 1, 1)
    d2 = d2.copy()
    d2[-2] = (int(d2[-2]) + 1) % P      # the public result (the last word before the exemptions)
    assert list(ctx.verify_air_batch([d2], [proof], h)) == [oracle.verify_air(d2, proof, h)] != [0]
    assert ctx.mem_stats()[0] == 0


def test_independence_and_mixed_lengths(ctx, oracle):
    opts = oracle.make_opts(num_queries=16, ext=2, folding=4, rem_max_deg=7, blowup=8)
    inputs = [fib_pair(64, 1 + j, 2 + j) for j in range(6)]
    descs = [d for d, _ in inputs]
    proofs = [ctx.prove_air(d, t, opts) for d, t in inputs]
    for j in (1, 4):
        b = bytearray(proofs[j])
        b[200 + 37 * j] ^= 4
        proofs[j] = bytes(b)
    alone = [int(ctx.verify_air_batch([d], [p], 0)[0]) for d, p in zip(descs, proofs)]
    assert alone == [oracle.verify_air(d, p, 0) for d, p in zip(descs, proofs)]
    assert alone[0] == 0 and alone[1] != 0 and alone[4] != 0
    assert list(ctx.verify_air_batch(descs, proofs, 0)) == alone
    assert list(ctx.verify_air_batch(descs[::-1], proofs[::-1], 0)) == alone[::-1]
    # one description that fits both lengths; proofs of 2^6 and 2^8 rows in one batch
    d64, t64 = fib_pair(64, 3, 4, last=False)
    d256, t256 = fib_pair(256, 3, 4, last=False)
    assert (d64 == d256).all()
    p64, p256 = ctx.prove_air(d64, t64, opts), ctx.prove_air(d256, t256, opts)
    bad = bytearray(p256)
    bad[-20] ^= 2
    mixed = [p64, p256, bytes(bad), p64]
    want = [oracle.verify_air(d64, p, 0) for p in mixed]
    assert want[:2] == [0, 0] and want[2] != 0
    assert list(ctx.verify_air_batch([d64] * 4, mixed, 0)) == want


def test_acceptable_options(ctx, oracle):
    kw = dict(num_queries=16, ext=2, folding=4, rem_max_deg=7, blowup=8, grinding=2, hash_id=1)
    opts = oracle.make_opts(**kw)
    desc, trace = airs.fib_small_x(1, 64)
    proof = ctx.prove_air(desc, trace, opts)
    other = oracle.make_opts(**dict(kw, num_queries=20))
    parts = oracle.make_opts(**dict(kw, num_partitions=2, hash_rate=4))
    assert list(ctx.verify_air_batch([desc], [proof], 1, acceptable=[opts])) == [0]
    assert list(ctx.verify_air_batch([desc], [proof], 1, acceptable=[other, opts])) == [0]
    assert list(ctx.verify_air_batch([desc], [proof], 1, acceptable=[other])) == [wf.VERIFY_UNACCEPTABLE_OPTIONS]
    assert list(ctx.verify_air_batch([desc], [proof], 1, acceptable=[parts])) == [wf.VERIFY_UNACCEPTABLE_OPTIONS]
    assert list(ctx.verify_air_batch([desc], [proof], 1)) == [oracle.verify_air(desc, proof, 1)] == [0]
    with pytest.raises(wf.WfError, match="acceptable option set 0 is for hash 0"):
        ctx.verify_air_batch([desc], [proof], 1, acceptable=[oracle.make_opts(**dict(kw, hash_id=0))])
    assert ctx.mem_stats()[0] == 0


def test_launches_do_not_grow_with_the_batch(ctx, oracle):
    opts = oracle.make_opts(num_queries=20, ext=2, folding=4, rem_max_deg=7, blowup=8, hash_id=1)
    inputs = [fib_pair(64, 1 + j, 2 + 3 * j) for j in range(16)]
    descs = [d for d, _ in inputs]
    proofs = ctx.prove_air_batch(descs, [t for _, t in inputs], opts)
    launches = {}
    for B in (1, 16, 256):
        ds = [descs[j % 16] for j in range(B)]
        ps = [proofs[j % 16] for j in range(B)]
        l0 = ctx.launches
        assert list(ctx.verify_air_batch(ds, ps, 1)) == [0] * B
        launches[B] = ctx.launches - l0
    assert launches[1] == launches[16] == launches[256], launches


def test_1024_proofs(ctx, oracle):
    opts = oracle.make_opts(num_queries=20, ext=2, folding=4, rem_max_deg=7, blowup=8, hash_id=0)
    inputs = [fib_pair(64, 1 + j, 2 + j) for j in range(1024)]
    descs = [d for d, _ in inputs]
    proofs = ctx.prove_air_batch(descs, [t for _, t in inputs], opts)
    assert list(ctx.verify_air_batch(descs, proofs, 0)) == [0] * 1024
    b = bytearray(proofs[512])
    b[len(b) // 2] ^= 8
    proofs[512] = bytes(b)
    got = ctx.verify_air_batch(descs, proofs, 0)
    want = oracle.verify_air(descs[512], proofs[512], 0)
    assert want != 0 and int(got[512]) == want and int((got != 0).sum()) == 1
    assert ctx.mem_stats()[0] == 0


def test_caller_errors_leave_nothing_behind(ctx, oracle):
    opts = oracle.make_opts(num_queries=16, ext=1, folding=4, rem_max_deg=7, blowup=8)
    d0, t0 = fib_pair(64, 1, 2)
    proof = ctx.prove_air(d0, t0, opts)
    dm, _ = airs.mulfib2(64)
    with pytest.raises(wf.WfError, match="proof 1 differs from proof 0"):
        ctx.verify_air_batch([d0, dm], [proof, proof], 0)
    assert ctx.mem_stats()[0] == 0
    with pytest.raises(wf.WfError, match="proof 1: malformed AIR description"):
        ctx.verify_air_batch([d0, d0[:5]], [proof, proof], 0)
    assert ctx.mem_stats()[0] == 0
    import ctypes as C
    u64p = C.POINTER(C.c_uint64)
    out = (C.c_uint32 * 1)()
    assert ctx.L.wf_verify_air_batch(ctx.h, 1, None, None, None, None, 0, None, 0, wf.AUX_ASSERTIONS_BATCH(), None, out) == -2
    dp = (u64p * 1)(d0.ctypes.data_as(u64p))
    dl = (C.c_size_t * 1)(d0.size)
    assert ctx.L.wf_verify_air_batch(ctx.h, 1, dp, dl, None, None, 0, None, 0, wf.AUX_ASSERTIONS_BATCH(), None, out) == -2
    assert ctx.mem_stats()[0] == 0
    assert list(ctx.verify_air_batch([d0], [proof], 0)) == [0]
    assert ctx.mem_stats()[0] == 0
