"""The CPU restatement of the standalone FRI verifier (tests/fri_ref.cpp wfr_fri_verify: FriVerifier::new + verify with
DefaultVerifierChannel, on top of the oracle) on the reference's FRI round trip, on dishonest proofs whose every opening
verifies, and on byte flips. CPU only."""
import numpy as np
import pytest

import fri_cases as F
from fri_cases import HASHES, SHAPES, Case, truncating_degree
from oracle import oracle as o

V = F.fri_verdict


@pytest.mark.parametrize("h", HASHES)
@pytest.mark.parametrize("nf,rem", SHAPES)
@pytest.mark.parametrize("d", [1, 2, 3])
def test_round_trip(h, nf, rem, d):
    # fri/src/prover/tests.rs fri_prove_verify: accepted at max_degree, refused at max_degree - 8
    c = Case(h, d, nf, rem)
    assert c.verify() == F.FRI_VERIFY_ACCEPT
    assert c.verify(max_deg=c.max_deg - 8) != F.FRI_VERIFY_ACCEPT


@pytest.mark.parametrize("d", [1, 3])
def test_round_trip_commitment_bytes(d):
    # the restatement's prover commits exactly what the oracle's wfo_fri_build_layers commits
    c = Case(o.BLAKE3, d, 4, 31, log_n=10)
    roots, rem, _ = o.fri_build_layers(o.BLAKE3, c.ev.reshape(-1), 4, 31, 8, d)
    assert (c.cm == roots).all()
    # FriProof: the layer count, then per layer the value and path lengths, the remainder, one partition
    assert c.proof[0] == c.nl and c.proof[-1] == 0
    assert c.proof[-1 - 2 - rem.size * 8: -1] == (rem.size * 8).to_bytes(2, "little") + rem.tobytes()


@pytest.mark.parametrize("h", [o.BLAKE3, o.RP64])
@pytest.mark.parametrize("nf,rem", [(2, 7), (4, 31)])
@pytest.mark.parametrize("d", [1, 3])
def test_dishonest_layer(h, nf, rem, d):
    # a changed value in layer `depth` > 0 at a queried row, its tree rebuilt and the rebuilt root committed: every opening
    # verifies, the fold of layer depth - 1 does not give it
    honest = Case(h, d, nf, rem)
    for depth in (1, honest.nl - 1):
        row = int(honest.pos[0]) % honest.layer_len(depth)
        delta = (5, 0, 0)[:d] if d == 1 else (0,) * (d - 1) + (9,)
        c = honest.tampered([o.tamper(o.FRI_LAYER, depth, row, delta)])
        assert not (c.cm[depth] == honest.cm[depth]).all()
        assert c.verify() == V(F.FRI_VERIFY_INVALID_LAYER_FOLDING, depth), depth


@pytest.mark.parametrize("d", [1, 2, 3])
def test_dishonest_remainder_long(d):
    # a remainder of twice the length max_degree_plus_1 allows after the last fold (its extra coefficients are zeros in
    # front: the values are right, the degree bound is not)
    honest = Case(o.BLAKE3, d, 4, 7)
    rn = honest.N // 4 ** honest.nl // honest.blowup
    c = honest.tampered([o.tamper(o.REMAINDER_LONG, rn)])
    assert c.verify() == F.FRI_VERIFY_REMAINDER_DEGREE_MISMATCH
    # a wrong remainder coefficient of the right length
    c = honest.tampered([o.tamper(o.REMAINDER, rn - 1, delta=(3,) * d)])
    assert c.verify() == F.FRI_VERIFY_INVALID_REMAINDER_FOLDING


@pytest.mark.parametrize("h", HASHES)
def test_remainder_commitment_is_not_compared(h):
    # read_remainder (fri/src/verifier/channel.rs:112-116) never looks at the last commitment: it only draws an alpha that
    # is never used, so an arbitrary digest in its place is accepted
    c = Case(h, 2, 4, 7)
    cm = c.cm.copy()
    cm[-1] = np.frombuffer(bytes(range(100, 132)), dtype=np.uint8)
    assert c.verify(cm=cm) == F.FRI_VERIFY_ACCEPT
    cm = c.cm.copy()
    cm[0, 3] ^= 1
    assert c.verify(cm=cm) != F.FRI_VERIFY_ACCEPT


@pytest.mark.parametrize("d", [1, 2, 3])
def test_wrong_evaluations(d):
    c = Case(o.RPJIVE, d, 8, 7)
    for k in range(d):   # only coordinate k of one evaluation differs, the last one included
        ev = c.evals.copy()
        ev[3, k] = (int(ev[3, k]) + 1) % o.P
        assert c.verify(evals=ev) == V(F.FRI_VERIFY_INVALID_LAYER_FOLDING, 0), k


@pytest.mark.parametrize("nf,rem", SHAPES)
def test_degree_truncation(nf, rem):
    c = Case(o.BLAKE3, 1, nf, rem)
    m, layer = truncating_degree(c.n, nf, c.nl)
    assert c.verify(max_deg=m) == V(F.FRI_VERIFY_DEGREE_TRUNCATION, layer)


def test_partition_byte():
    # num_partitions is honoured: 2^k partitions map the folded positions elsewhere in the commitment, which the single-
    # partition prover's openings do not open; indexes that repeat, and 2^64 partitions, are malformed
    c = Case(o.BLAKE3, 1, 4, 7, log_n=8, num_queries=8)
    for k, want in [(0, F.FRI_VERIFY_ACCEPT), (1, F.FRI_VERIFY_LAYER_COMMITMENT_MISMATCH), (2, F.FRI_VERIFY_LAYER_COMMITMENT_MISMATCH),
                    (40, F.FRI_VERIFY_MALFORMED), (64, F.FRI_VERIFY_MALFORMED), (255, F.FRI_VERIFY_MALFORMED)]:
        p = bytearray(c.proof)
        p[-1] = k
        assert c.verify(proof=bytes(p)) == want, k


def test_byte_flips_are_refused():
    # every single-byte flip of an honest proof changes the deserialized proof, and is refused
    c = Case(o.BLAKE3, 2, 4, 3, log_n=6, log_b=2, num_queries=6)
    assert c.verify() == F.FRI_VERIFY_ACCEPT
    for i in range(len(c.proof)):
        p = bytearray(c.proof)
        p[i] ^= 1 << (i % 8)
        assert c.verify(proof=bytes(p)) != F.FRI_VERIFY_ACCEPT, i
    for cut in (1, 9, len(c.proof) // 2):
        assert c.verify(proof=c.proof[:-cut]) == F.FRI_VERIFY_MALFORMED
    assert c.verify(proof=c.proof + b"\0") == F.FRI_VERIFY_MALFORMED


def test_caller_errors():
    c = Case(o.BLAKE3, 1, 4, 7, log_n=8, num_queries=4)
    with pytest.raises(ValueError):
        c.verify(cm=c.cm[:-1])
    ev = c.evals.copy()
    ev[0, 0] = o.P
    with pytest.raises(ValueError):
        c.verify(evals=ev)
    with pytest.raises(ValueError):
        F.fri_verify(c.h, 1, 4, 7, 8, c.max_deg, c.proof, c.cm, [c.N], c.evals[:1])
    with pytest.raises(ValueError):
        F.fri_verify(c.h, 1, 3, 7, 8, c.max_deg, c.proof, c.cm, c.pos, c.evals)
