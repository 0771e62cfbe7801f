"""The oracle verifier's verdicts on dishonest proofs (tests/dishonest.py): proofs that open every commitment correctly and
are still wrong. A byte flip in an honest proof fails at a Merkle root, the transcript, the OOD check or the remainder, and
never reaches the FRI layer-folding check (verdict 7); these proofs do, so they show that the folding, DEEP and remainder
checks still refuse. Every verdict is pinned to its exact code: a proof that gets 7 passed every opening, OOD and PoW."""
import pytest

import airs
import dishonest as D


def _check(cases):
    provers = {}
    got = [provers.setdefault(c.key, D.Prover(*c.key)).oracle_verdict(c.proof, c.hash_id) for c in cases]
    wrong = [(c.name, g, c.want) for c, g in zip(cases, got) if g != c.want]
    assert not wrong, wrong


@pytest.mark.parametrize("air", ["fib", "perm_rap"])
@pytest.mark.parametrize("ext", [1, 2, 3])
@pytest.mark.parametrize("folding", [2, 4, 8, 16])
def test_all_rows_tampers(oracle, air, ext, folding):
    opts = oracle.make_opts(num_queries=20, blowup=8, ext=ext, folding=folding, rem_max_deg=3)
    cases = D.all_rows_cases(air, 64, opts)
    assert sum(c.want == D.FRI_FOLD for c in cases) >= 3 + D.num_layers(64, opts)
    _check(cases)


def test_all_rows_tampers_with_partitions_and_batching(oracle):
    # the rotating options of the device matrix: batching methods 0 / 1 / 2, two partitions of hash rate 8
    _check(D.matrix_cases(oracle.BLAKE3_192))


def test_no_fri_layer(oracle):
    _check(D.no_layer_cases(oracle.BLAKE3))


@pytest.mark.parametrize("ext,folding", [(1, 4), (3, 2), (2, 16)])
def test_single_row_tamper_is_refused_exactly_when_queried(oracle, ext, folding):
    cases, kinds = D.single_row_cases(oracle.BLAKE3, ext, folding)
    assert {"missed", "queried first", "queried later"} <= set(kinds)
    _check(cases)


def test_bad_traces_fail_the_ood_check(oracle):
    _check(D.bad_trace_cases(oracle.BLAKE3))


def test_first_failed_check_wins(oracle):
    _check(D.precedence_cases(oracle.BLAKE3))


def test_tamper_hook(oracle):
    # no tamper: the honest proof, byte for byte, and the positions it opens; nothing carries over to the next proof
    n = 64
    desc, trace = airs.fib_small_x(1, n)
    opts = oracle.make_opts(num_queries=20, blowup=8, ext=2, folding=4, rem_max_deg=3, grinding=2)
    honest = oracle.prove_air(desc, trace, opts)
    same, pos = oracle.prove_air(desc, trace, opts, tamper=[])
    assert same == honest and oracle.verify_air(desc, honest) == 0
    assert list(pos) == sorted(set(int(p) for p in pos)) and 0 < len(pos) <= 20 and pos.max() < n * 8
    bad, _ = oracle.prove_air(desc, trace, opts, tamper=[oracle.tamper(oracle.FRI_LAYER, 1, delta=(0, 1))])
    assert bad != honest   # other commitments: other query positions
    assert oracle.prove_air(desc, trace, opts) == honest
    tr, res = oracle.build_fib_trace(1, n)
    fib_proof, fib_pos = oracle.prove_fib(tr, res, opts, tamper=[])
    assert fib_proof == honest and (fib_pos == pos).all()
    # a flip changes one bit of the named section and nothing else
    flipped, pos2 = oracle.prove_air(desc, trace, opts, tamper=[oracle.tamper(oracle.FLIP_CONSTRAINT, row=3, delta=(6,))])
    diff = [i for i in range(len(honest)) if honest[i] != flipped[i]]
    assert len(diff) == 1 and honest[diff[0]] ^ flipped[diff[0]] == 1 << 6 and (pos2 == pos).all()
    assert oracle.verify_air(desc, flipped) == D.CONSTRAINT_QUERY
    # a tamper that names nothing of the proof is an error, not an honest proof
    for t in (oracle.tamper(oracle.MAIN_LDE, 2), oracle.tamper(oracle.AUX_LDE, 0), oracle.tamper(oracle.CONSTRAINT_LDE, 1),
              oracle.tamper(oracle.FRI_LAYER, 3), oracle.tamper(oracle.FRI_LAYER, 0, row=n * 8), oracle.tamper(oracle.FLIP_FRI, 2),
              oracle.tamper(oracle.REMAINDER, 4), oracle.tamper(oracle.REMAINDER_LONG, 0), oracle.tamper(oracle.MAIN_LDE, delta=(D.P,)),
              oracle.tamper(oracle.FLIP_TRACE, row=10 ** 6), oracle.tamper(10)):
        with pytest.raises(RuntimeError, match=r"\(-4\)"):
            oracle.prove_air(desc, trace, opts, tamper=[t])
    assert oracle.prove_air(desc, trace, opts) == honest


def test_aux_dyn_tamper(oracle):
    pv = D.Prover("perm_rap_dyn", 64)
    opts = oracle.make_opts(num_queries=16, blowup=8, ext=3, folding=4, rem_max_deg=7)
    honest = pv.case("honest", opts, [], D.ACCEPT)
    _check([honest, pv.case("aux col 1", opts, [oracle.tamper(oracle.AUX_LDE, 1, delta=(0, 0, 1))], D.FRI_FOLD)])
    assert oracle.verify_air(pv.desc, honest.proof) != 0   # the placeholder value is not what the trace satisfies
