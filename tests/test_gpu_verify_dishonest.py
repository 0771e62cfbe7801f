"""wf_verify_air_batch on dishonest proofs (tests/dishonest.py): proofs that open every commitment correctly and are still
wrong, so that they reach the device's FRI fold check (fold_one, every <ext, folding> instantiation), the DEEP composition
kernel and the remainder check. Every device verdict must equal the oracle verifier's and the verdict the case was built
for, on every hasher; mixed honest / dishonest batches, long FRI chains, host-decided against device-decided failures and the
aux-assertion callback path; no device memory is left live after any call."""
import numpy as np
import pytest

import dishonest as D
import winterfell_b200 as wf

pytestmark = pytest.mark.gpu
HASHERS = [0, 1, 2, 3, 4]   # Blake3_256, Rp64_256, RpJive64_256, Blake3_192, Sha3_256


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


def _verify(ctx, cases):
    """device verdicts of the cases, one call per AIR structure, in case order"""
    got = [None] * len(cases)
    groups = {}
    for i, c in enumerate(cases):
        groups.setdefault((c.key, c.hash_id, c.values_fn is not None), []).append(i)
    for (_, h, dyn), idx in groups.items():
        fn = None
        if dyn:
            vf = cases[idx[0]].values_fn
            fn = lambda j, rand, vals: vf(rand, vals)
        out = ctx.verify_air_batch([cases[i].desc for i in idx], [cases[i].proof for i in idx], h, aux_values_fn=fn)
        assert ctx.mem_stats()[0] == 0
        for i, v in zip(idx, out):
            got[i] = int(v)
    return got


def _oracle(cases):
    provers = {}
    return [provers.setdefault(c.key, D.Prover(*c.key)).oracle_verdict(c.proof, c.hash_id) for c in cases]


def _check(ctx, cases):
    got, want = _verify(ctx, cases), _oracle(cases)
    wrong = [(c.name, g, w, c.want) for c, g, w in zip(cases, got, want) if not g == w == c.want]
    assert not wrong, wrong
    return got


@pytest.mark.parametrize("h", HASHERS)
def test_dishonest_matrix(ctx, h):
    # all-rows tampers over ext 1 / 2 / 3 x folding 2 / 4 / 8 / 16 (all twelve fold_one instantiations) on a one- and a
    # two-segment AIR, batching methods and partitions rotating; the corner without FRI layers; single-row tampers, some
    # queried after another query of their FRI row; two failures in one proof; an honest prover on bad traces
    singles, kinds = D.single_row_cases(h, ext=1 + h % 3, folding=(4, 16, 2, 8, 4)[h])
    assert {"missed", "queried first", "queried later"} <= set(kinds)
    cases = D.matrix_cases(h) + D.no_layer_cases(h) + singles + D.precedence_cases(h, ext=1 + (h + 1) % 3) + D.bad_trace_cases(h)
    got = _check(ctx, cases)
    assert got.count(D.FRI_FOLD) >= 100 and D.FRI_REMAINDER in got and D.ACCEPT in got


def test_long_fri_chain(ctx, oracle):
    # 2^16 rows, blowup 2, folding 2, remainder degree 0: 16 FRI layers, fold checks up to the highest ranks
    n = 1 << 16
    opts = oracle.make_opts(num_queries=24, blowup=2, ext=2, folding=2, rem_max_deg=0, hash_id=0)
    nl = D.num_layers(n, opts)
    assert nl == 16
    pv = D.Prover("fib", n)
    cases = [pv.case("last layer", opts, [oracle.tamper(oracle.FRI_LAYER, nl - 1, delta=(0, 1))], D.FRI_FOLD),
             pv.case("remainder", opts, [oracle.tamper(oracle.REMAINDER, 0, delta=(0, 1))], D.FRI_REMAINDER),
             pv.case("layer 9 + layer 12 opening flipped", opts,
                     [oracle.tamper(oracle.FRI_LAYER, 9, delta=(2, 0)), oracle.tamper(oracle.FLIP_FRI, 12)], D.FRI_FOLD),
             pv.case("honest", opts, [], D.ACCEPT)]
    _check(ctx, cases)


def _mixed_cases(oracle):
    """16 proofs of fib_small from different starts (64 rows, folding 2: layers 0 .. 3), dishonest ones at every depth
    between honest ones"""
    opts = oracle.make_opts(num_queries=20, ext=2, folding=2, rem_max_deg=3, blowup=8, hash_id=0)
    T = oracle.tamper
    plan = [[], [T(oracle.FRI_LAYER, 0, delta=(0, 3))], [], [T(oracle.FRI_LAYER, 1, delta=(1, 0))], [T(oracle.MAIN_LDE, 1, delta=(7,))],
            [], [T(oracle.FRI_LAYER, 2, delta=(0, 1))], [T(oracle.REMAINDER, 1, delta=(0, 2))], [],
            [T(oracle.FRI_LAYER, 3, delta=(5, 5))], [T(oracle.REMAINDER_LONG, 1)], [T(oracle.CONSTRAINT_LDE, 0, delta=(0, 9))], [],
            [T(oracle.FRI_LAYER, 3, delta=(0, 1)), T(oracle.FLIP_FRI, 1)], [T(oracle.FLIP_TRACE, row=4)], []]
    want = [D.ACCEPT, D.FRI_FOLD, D.ACCEPT, D.FRI_FOLD, D.FRI_FOLD, D.ACCEPT, D.FRI_FOLD, D.FRI_REMAINDER, D.ACCEPT, D.FRI_FOLD,
            D.FRI_REMAINDER, D.FRI_FOLD, D.ACCEPT, D.FRI_LAYER, D.TRACE_QUERY, D.ACCEPT]
    descs, proofs = [], []
    for j, t in enumerate(plan):
        desc, trace = D.fib_from(64, 1 + j, 2 + 3 * j)
        proof, _ = oracle.prove_air(desc, trace, opts, tamper=t)
        descs.append(desc)
        proofs.append(proof)
    assert [oracle.verify_air(d, p, 0) for d, p in zip(descs, proofs)] == want
    return descs, proofs, want, opts


def test_mixed_batches(ctx, oracle):
    descs, proofs, want, _ = _mixed_cases(oracle)
    alone = [int(ctx.verify_air_batch([d], [p], 0)[0]) for d, p in zip(descs, proofs)]
    assert alone == want
    assert list(ctx.verify_air_batch(descs, proofs, 0)) == want
    assert list(ctx.verify_air_batch(descs[::-1], proofs[::-1], 0)) == want[::-1]
    idx = [(7 * j + 3) % 16 for j in range(256)]
    assert list(ctx.verify_air_batch([descs[i] for i in idx], [proofs[i] for i in idx], 0)) == [want[i] for i in idx]
    assert ctx.mem_stats()[0] == 0


def test_1024_proofs_with_dishonest_ones(ctx, oracle):
    descs, dishonest, want16, opts = _mixed_cases(oracle)
    inputs = [D.fib_from(64, 100 + j, 2 + j) for j in range(1024)]
    ds = [d for d, _ in inputs]
    ps = ctx.prove_air_batch(ds, [t for _, t in inputs], opts)
    want = [D.ACCEPT] * 1024
    for k, j in enumerate((0, 37, 300, 511, 512, 640, 777, 901, 1000, 1023, 5, 64, 128, 256, 700, 999)):
        ds[j], ps[j], want[j] = descs[k], dishonest[k], want16[k]
    assert list(ctx.verify_air_batch(ds, ps, 0)) == want
    assert ctx.mem_stats()[0] == 0


def _expected(oracle, oracle_code, desc, proof):
    """the oracle's verdict, except that a proof whose declared length the AIR does not fit is CONTEXT once it parses"""
    if oracle_code in (0, 2, 3, 4, 5, 6, 7, 8) and len(proof) > 16:
        rc, _ = wf.air_check(desc, proof[3], proof[16])
        if rc != 0:
            return wf.VERIFY_CONTEXT
    return oracle_code


@pytest.mark.parametrize("h,ext", [(0, 2), (3, 3)])   # ~14000 oracle verifications each: byte-oriented hashers only
def test_byte_flips_of_dishonest_proofs(ctx, oracle, h, ext):
    # every dishonest proof's failure is decided on the device; a flip that the host decides early (a malformed opening,
    # a bad option) must still lose to an earlier-ranked failure the device finds, and win over a later one
    n = 128
    opts = oracle.make_opts(num_queries=12, blowup=8, grinding=2, ext=ext, folding=4, rem_max_deg=7, hash_id=h)
    pv = D.Prover("fib", n)
    kinds = [[oracle.tamper(oracle.MAIN_LDE, 0, delta=(1,))], [oracle.tamper(oracle.CONSTRAINT_LDE, 0, delta=D.last_coord(ext))],
             [oracle.tamper(oracle.FRI_LAYER, 0, delta=D.last_coord(ext))], [oracle.tamper(oracle.FRI_LAYER, 1, delta=(1,))],
             [oracle.tamper(oracle.REMAINDER, 0, delta=D.last_coord(ext))], [oracle.tamper(oracle.REMAINDER_LONG, 1)]]
    muts = []
    for k, t in enumerate(kinds):
        proof, _ = pv.prove(opts, t)
        muts += D.flip_set(proof, 100 * h + 10 * ext + k)
    want = [_expected(oracle, oracle.verify_air(pv.desc, m, h), pv.desc, m) for m in muts]
    assert {D.FRI_FOLD, D.FRI_REMAINDER, D.FRI_LAYER, D.TRACE_QUERY, D.CONSTRAINT_QUERY} <= set(want)
    got = ctx.verify_air_batch([pv.desc] * len(muts), muts, h)
    bad = [(i, int(g), w) for i, (g, w) in enumerate(zip(got, want)) if int(g) != w]
    assert not bad, bad[:20]
    assert ctx.mem_stats()[0] == 0


def test_aux_dyn_callback_path(ctx, oracle):
    pv = D.Prover("perm_rap_dyn", 64)
    opts = oracle.make_opts(num_queries=16, blowup=8, ext=3, folding=4, rem_max_deg=7, hash_id=0)
    cases = [pv.case("honest", opts, [], D.ACCEPT),
             pv.case("aux col 1, last coordinate", opts, [oracle.tamper(oracle.AUX_LDE, 1, delta=(0, 0, 1))], D.FRI_FOLD),
             pv.case("aux col 0", opts, [oracle.tamper(oracle.AUX_LDE, 0, delta=(4, 5, 6))], D.FRI_FOLD),
             pv.case("FRI layer 1", opts, [oracle.tamper(oracle.FRI_LAYER, 1, delta=(0, 2, 0))], D.FRI_FOLD),
             pv.case("remainder", opts, [oracle.tamper(oracle.REMAINDER, 0, delta=(0, 0, 3))], D.FRI_REMAINDER)]
    _check(ctx, cases)
