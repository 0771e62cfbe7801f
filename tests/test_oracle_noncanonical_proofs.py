"""The oracle verifier's verdicts on proofs carrying words of p or more (dishonest.noncanonical_cases): any field element of
p or more is refused as malformed, as the reference's BaseElement::read_from refuses it; a Rescue digest word of p or more is
reduced, as ElementDigest::read_from reduces it, and then fails the check its digest meets."""
import pytest

import dishonest as D


@pytest.mark.parametrize("ext", [1, 2, 3])
@pytest.mark.parametrize("h", [0, 1, 2, 3, 4])
def test_oracle_verdicts_on_noncanonical_words(h, ext):
    pv = D.Prover("perm_rap", 64)
    for c in D.noncanonical_cases(h, ext):
        got = pv.oracle_verdict(c.proof, h)
        if c.want is None:
            assert got not in (D.ACCEPT, D.MALFORMED), (c.name, got)
        else:
            assert got == c.want, (c.name, got)



@pytest.mark.parametrize("h", [1, 2])
def test_path_node_word_plus_p_opens_the_same_root(oracle, h):
    # a Merkle path node word w < 2^32 - 1 written as w + p stands for w (ElementDigest::read_from reduces it): the opening
    # still gives the root; w + 1 does not. The first node of an opening of leaf 0 is leaf 1, so its words can be chosen
    import ctypes as C
    import numpy as np
    leaves = np.array([[7 * i + k for k in range(4)] for i in range(8)], dtype=np.uint64).view(np.uint8).reshape(8, 32)
    nodes = oracle.merkle_nodes(h, leaves)
    lv, pr = oracle.merkle_prove_batch(leaves, nodes, [0], h)
    at = 1 + 1 + 1                                   # depth byte, vint count of node vectors, vint length of the first
    assert pr[at:at + 32] == leaves[1].tobytes()
    u8p, u64p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint64)

    def verify(proof):
        idx = np.array([0], dtype=np.uint64)
        lvb, prb, rb = np.ascontiguousarray(lv), np.frombuffer(proof, dtype=np.uint8), nodes[1].copy()
        return oracle.lib().wfo_merkle_verify_batch(C.c_int(h), rb.ctypes.data_as(u8p), idx.ctypes.data_as(u64p), C.c_size_t(1),
                                                    lvb.ctypes.data_as(u8p), prb.ctypes.data_as(u8p), C.c_size_t(prb.size))
    w = int.from_bytes(pr[at:at + 8], "little")
    assert verify(pr) == 0
    assert verify(pr[:at] + (w + oracle.P).to_bytes(8, "little") + pr[at + 8:]) == 0
    assert verify(pr[:at] + (w + 1).to_bytes(8, "little") + pr[at + 8:]) != 0
