"""wf_verify_air_batch_min_security: verifier::verify under AcceptableOptions::MinConjecturedSecurity and MinProvenSecurity.
- proofs of wf_prove_air / wf_prove_air_aux over every hasher, ext 1 to 3 and every batching method, checked at a minimum one
  below, at and one above their estimate under each regime: ACCEPT or 11 / 12, with the bits of wf_proof_security and of the
  Python restatement;
- mixed batches: policy-refused proofs (some also dishonest) among honest and dishonest ones (tests/dishonest.py), malformed
  proofs and proofs whose context does not fit the AIR; every survivor gets wf_verify_air_batch's and the oracle's verdict;
- min_bits = 0 is wf_verify_air_batch(acceptable_opts = NULL), launches included; a batch refused whole; no device buffer
  left live after any return."""
import numpy as np
import pytest

import airs
import dishonest as D
import security_ref as sr
import winterfell_b200 as wf

pytestmark = pytest.mark.gpu
CONJ, PROVEN = wf.SECURITY_CONJECTURED, wf.SECURITY_PROVEN
REFUSED = {CONJ: wf.VERIFY_INSUFFICIENT_CONJECTURED_SECURITY, PROVEN: wf.VERIFY_INSUFFICIENT_PROVEN_SECURITY}
NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


def policy_bits(est, regime):
    """the bits AcceptableOptions::validate weighs: conjectured, or max(ldr, udr)"""
    return est[0] if regime == CONJ else max(est[1], est[2])


def context_estimate(proof, hash_id):
    """security_ref's estimate from the proof's Context bytes"""
    mw, aw, logn = proof[0], proof[1], proof[3]
    at = 6 + (proof[4] | proof[5] << 8)
    at += 1 + proof[at]
    o = list(proof[at:at + 8])
    ncons, _ = D._usize(proof, at + 10)
    return sr.estimate(o, 1 << logn, sr.COLLISION_RESISTANCE[hash_id], ncons, mw + aw + o[1])


# (air, log_n, hash, ext, options): every hasher, ext 1 to 3, each batching method for the constraints and the DEEP polynomial
SHAPES = [
    ("fib", 6, 0, 1, dict(num_queries=30, blowup=8, folding=4, rem_max_deg=7, batch_c=0, batch_d=0)),
    ("fib", 7, 1, 2, dict(num_queries=48, blowup=4, folding=2, rem_max_deg=3, grinding=4, batch_c=1, batch_d=2)),
    ("rap", 6, 2, 3, dict(num_queries=28, blowup=8, folding=8, rem_max_deg=7, grinding=2, batch_c=2, batch_d=1)),
    ("fib", 6, 3, 2, dict(num_queries=45, blowup=8, folding=4, rem_max_deg=7, grinding=6, batch_c=2, batch_d=0)),
    ("rap", 7, 4, 3, dict(num_queries=60, blowup=16, folding=16, rem_max_deg=15, grinding=8, batch_c=1, batch_d=1)),
    ("fib", 8, 4, 1, dict(num_queries=20, blowup=2, folding=2, rem_max_deg=1, batch_c=0, batch_d=2)),
    ("rap", 6, 0, 2, dict(num_queries=90, blowup=4, folding=4, rem_max_deg=7, grinding=10, batch_c=2, batch_d=2)),
]


def prove(ctx, oracle, air, log_n, hash_id, ext, kw):
    opts = oracle.make_opts(ext=ext, hash_id=hash_id, **kw)
    n = 1 << log_n
    if air == "fib":
        desc, trace = airs.fib_small_x(2, n)[:2]
        return desc, ctx.prove_air(desc, trace, opts)
    desc, trace, builder = airs.perm_rap(n)
    return desc, ctx.prove_air_aux(desc, trace, opts, builder, airs.PERM_RAP_AUX_WIDTH, 2)


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{a}-n{l}-h{h}-e{e}-b{k['batch_c']}{k['batch_d']}" for a, l, h, e, k in SHAPES])
def test_minimum_around_the_estimate(ctx, oracle, shape):
    air, log_n, h, ext, kw = shape
    desc, proof = prove(ctx, oracle, air, log_n, h, ext, kw)
    assert oracle.verify_air(desc, proof, h) == 0
    est = wf.proof_security(h, proof)
    assert est == context_estimate(proof, h)
    for regime in (CONJ, PROVEN):
        v = policy_bits(est, regime)
        assert v > 0
        for min_bits in (v - 1, v, v + 1):
            verdicts, bits = ctx.verify_air_batch_min_security([desc], [proof], h, regime, min_bits)
            assert list(bits) == [v]
            assert list(verdicts) == [0 if min_bits <= v else REFUSED[regime]], (regime, min_bits, v)
        assert ctx.mem_stats()[0] == 0


def test_blake3_192_caps_at_96_bits(ctx, oracle):
    desc, proof = prove(ctx, oracle, "fib", 6, wf.HASH_BLAKE3_192, 2, dict(num_queries=60, blowup=8, folding=4, rem_max_deg=7,
                                                                            grinding=16))
    # the same options under Blake3_256 estimate more than 100 conjectured bits
    assert wf.proof_security(wf.HASH_BLAKE3_256, proof)[0] > 100
    assert wf.proof_security(wf.HASH_BLAKE3_192, proof)[0] == 96
    verdicts, bits = ctx.verify_air_batch_min_security([desc], [proof], wf.HASH_BLAKE3_192, CONJ, 100)
    assert list(verdicts) == [wf.VERIFY_INSUFFICIENT_CONJECTURED_SECURITY] and list(bits) == [96]
    verdicts, bits = ctx.verify_air_batch_min_security([desc], [proof], wf.HASH_BLAKE3_192, CONJ, 96)
    assert list(verdicts) == [0] and list(bits) == [96]


def _mixed(oracle):
    """one AIR (FibSmall, 64 rows), interleaved: honest proofs at 20 queries, dishonest ones (tests/dishonest.py), weak
    proofs at 6 queries (honest and dishonest), a malformed proof and one whose context does not fit the AIR.
    Returns (description, proofs, kinds)."""
    fib = D.Prover("fib", 64)
    strong = oracle.make_opts(num_queries=20, blowup=8, ext=2, folding=2, rem_max_deg=3)
    weak = oracle.make_opts(num_queries=6, blowup=8, ext=2, folding=2, rem_max_deg=3)
    honest = fib.prove(strong)[0]
    wide = bytearray(honest)
    wide[0] += 1                                                 # one main column more than the AIR: CONTEXT at parse time
    items = [(honest, "honest")]
    items += [(c.proof, "dishonest") for c in D.precedence_cases(0) if c.key == ("fib", 64)]
    items += [(fib.prove(weak)[0], "weak"), (fib.prove(weak, [oracle.tamper(oracle.FRI_LAYER, 1, delta=(0, 5))])[0], "weak"),
              (fib.prove(weak, [oracle.tamper(oracle.MAIN_LDE, 0, delta=(4,))])[0], "weak"),
              (honest[:len(honest) // 2], "malformed"), (bytes(wide), "context"), (honest, "honest")]
    order = sorted(range(len(items)), key=lambda k: (5 * k) % len(items) if len(items) % 5 else k)
    return fib.desc, [items[k][0] for k in order], [items[k][1] for k in order]


@pytest.mark.parametrize("regime", [CONJ, PROVEN])
def test_mixed_batches(ctx, oracle, regime):
    desc, proofs, kinds = _mixed(oracle)
    h = 0
    descs = [desc] * len(proofs)
    weak_bits = policy_bits(wf.proof_security(h, proofs[kinds.index("weak")]), regime)
    strong_bits = policy_bits(wf.proof_security(h, proofs[kinds.index("honest")]), regime)
    assert weak_bits < strong_bits
    plain = [int(v) for v in ctx.verify_air_batch(descs, proofs, h)]
    verdicts, bits = ctx.verify_air_batch_min_security(descs, proofs, h, regime, strong_bits)
    assert {plain[j] for j, k in enumerate(kinds) if k == "dishonest"} - {0}   # the dishonest proofs fail a check
    for j, (p, kind) in enumerate(zip(proofs, kinds)):
        if kind in ("malformed", "context"):
            assert verdicts[j] == plain[j] == (wf.VERIFY_MALFORMED if kind == "malformed" else wf.VERIFY_CONTEXT), j
            assert bits[j] == NONE
            continue
        assert bits[j] == policy_bits(wf.proof_security(h, p), regime) == policy_bits(context_estimate(p, h), regime)
        if kind == "weak":
            assert verdicts[j] == REFUSED[regime], j                      # also when the proof is dishonest
        else:
            assert verdicts[j] == plain[j] == oracle.verify_air(desc, p, h), j
    assert ctx.mem_stats()[0] == 0


def test_zero_minimum_is_the_unrestricted_verifier(ctx, oracle):
    desc, proofs, _ = _mixed(oracle)
    descs = [desc] * len(proofs)
    l0 = ctx.launches
    plain = list(ctx.verify_air_batch(descs, proofs, 0))
    plain_launches = ctx.launches - l0
    for regime in (CONJ, PROVEN):
        l0 = ctx.launches
        verdicts, bits = ctx.verify_air_batch_min_security(descs, proofs, 0, regime, 0)
        assert list(verdicts) == plain
        assert ctx.launches - l0 == plain_launches
        assert all(b != NONE for b, v in zip(bits, verdicts) if v not in (wf.VERIFY_MALFORMED, wf.VERIFY_CONTEXT))
    assert ctx.mem_stats()[0] == 0


def test_batch_refused_whole(ctx, oracle):
    desc, proofs, kinds = _mixed(oracle)
    weak = [p for p, k in zip(proofs, kinds) if k == "weak"]
    for regime in (CONJ, PROVEN):
        verdicts, bits = ctx.verify_air_batch_min_security([desc] * len(weak), weak, 0, regime, 129)
        assert list(verdicts) == [REFUSED[regime]] * len(weak)
        assert all(b == policy_bits(wf.proof_security(0, p), regime) for b, p in zip(bits, weak))
    assert ctx.mem_stats()[0] == 0


def test_caller_errors_leave_nothing_live(ctx, oracle):
    desc, proofs, _ = _mixed(oracle)
    for regime in (0, 3, -1):
        with pytest.raises(wf.WfError):
            ctx.verify_air_batch_min_security([desc], [proofs[0]], 0, regime, 10)
        assert ctx.mem_stats()[0] == 0
    with pytest.raises(wf.WfError):
        ctx.verify_air_batch_min_security([desc], [proofs[0]], 9, CONJ, 10)           # unknown hash
    assert ctx.mem_stats()[0] == 0
    with pytest.raises(wf.WfError):
        ctx.verify_air_batch_min_security([np.array([0], dtype=np.uint64)], [proofs[0]], 0, PROVEN, 10)   # malformed description
    assert ctx.mem_stats()[0] == 0
    # the context still works
    verdicts, _ = ctx.verify_air_batch_min_security([desc], [proofs[0]], 0, CONJ, 1)
    assert list(verdicts) == [0]


def test_many_proofs_one_estimate(ctx, oracle):
    """1024 proofs of one shape: the estimate is memoised per distinct key; the verdicts equal the unrestricted verifier's"""
    opts = oracle.make_opts(num_queries=20, blowup=8, ext=2, folding=4, rem_max_deg=7)
    inputs = [D.fib_from(64, 100 + j, 2 + j) for j in range(1024)]
    ds = [d for d, _ in inputs]
    ps = ctx.prove_air_batch(ds, [t for _, t in inputs], opts)
    v = policy_bits(wf.proof_security(0, ps[0]), PROVEN)
    verdicts, bits = ctx.verify_air_batch_min_security(ds, ps, 0, PROVEN, v)
    assert list(verdicts) == [0] * 1024 and list(bits) == [v] * 1024
    verdicts, bits = ctx.verify_air_batch_min_security(ds, ps, 0, PROVEN, v + 1)
    assert list(verdicts) == [wf.VERIFY_INSUFFICIENT_PROVEN_SECURITY] * 1024
    assert ctx.mem_stats()[0] == 0
