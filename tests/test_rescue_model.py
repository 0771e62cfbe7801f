"""The exact Rescue model (rescue_model.py) against the oracle, its backward targeting, and the edge classes the targeted
inputs reach: every (step kind, class) cell is reached or listed with the reason it is not."""
import numpy as np
import pytest

import rescue_model as M

P = M.P
HIDS = [M.RP64, M.RPJIVE]


def _d(words):
    return np.array(words, dtype=np.uint64).tobytes()


def _states(hid, seed=0):
    rng = np.random.default_rng(seed + hid)
    rand = [("random", [int(v) % P for v in rng.integers(0, 2**64, M.HASHERS[hid].w, dtype=np.uint64)]) for _ in range(8)]
    return rand + M.targeted_states(hid, rng)


@pytest.mark.parametrize("hid", HIDS)
def test_model_permutation_equals_oracle(oracle, hid):
    perm = oracle.rp64_permute if hid == M.RP64 else oracle.rpjive_permute
    for label, s in _states(hid):
        assert M.permute(hid, s) == [int(v) for v in perm(np.array(s, dtype=np.uint64))], label


@pytest.mark.parametrize("hid", HIDS)
def test_model_sponge_and_merges_equal_oracle(oracle, hid):
    rng = np.random.default_rng(hid)
    for n in list(range(0, 21)) + [63, 64, 65]:
        e = [int(v) for v in oracle.rand_elems(n, 7 * n + hid)]
        assert _d(M.hash_elements(hid, e)) == oracle.hash_elements(hid, np.array(e, dtype=np.uint64)), n
    for label, s in M.targeted_states(hid, rng)[::3]:
        s8 = s[:8]
        assert _d(M.merge(hid, s8)) == oracle.merge(hid, _d(s8[:4]), _d(s8[4:])), label
        for v in (0, 5, P - 1, P, P + 1, 2**64 - 1):
            assert _d(M.merge_with_int(hid, s8[:4], v)) == oracle.merge_with_int(hid, _d(s8[:4]), v), (label, v)


@pytest.mark.parametrize("hid", HIDS)
def test_backward_then_forward_reaches_the_requested_state(hid):
    rng = np.random.default_rng(5)
    w = M.HASHERS[hid].w
    for r in range(7):
        for b in M.BOUNDARIES:
            want = [int(v) for v in rng.integers(0, P, w, dtype=np.uint64)]
            want[r % w] = [0, 1, P - 1, 2**32][r % 4]
            tr = {}
            M.permute(hid, M.backward(hid, r, b, want), trace=tr)
            assert tr[(r, b)] == want, (r, b)


@pytest.mark.parametrize("hid", HIDS)
def test_round0_rows_reach_their_targets(hid):
    rng = np.random.default_rng(9)
    rate = 8 if hid == M.RP64 else 4
    for width in range(1, rate + 1):
        for row in M.round0_rows(hid, rng, width):
            cap = [width, 0, 0, 0] if hid == M.RP64 else [int(width % 4 != 0), 0, 0, 0]
            s = cap + list(row) + [0] * (rate - width)
            if hid == M.RPJIVE and width < 4:
                s[4 + width] = 1
            tr = {}
            M.permute(hid, s, trace=tr)
            if row[0] in M.SBOX_INPUTS:
                assert tr[(0, "sbox in")][4] == row[0]
    # the MDS-targeted rows of a full block put the catalogue values at the first `rate` MDS1 outputs
    rows = M.round0_rows(hid, rng, rate)
    n_mds = -(-len(M.SBOX_INPUTS) // rate)   # round0_rows appends the MDS-targeted rows last, `rate` targets per row
    mds_rows = rows[-n_mds:]
    hits = set()
    for row in mds_rows:
        s = ([rate, 0, 0, 0] if hid == M.RP64 else [0, 0, 0, 0]) + list(row)
        tr = {}
        M.permute(hid, s, trace=tr)
        hits |= set(tr[(0, "mds1 out")][:rate]) & set(M.SBOX_INPUTS)
    assert {0, 1, P - 1} <= hits


def test_slot_targets_reach_their_words():
    found, missing = M.slot_targets()
    for (slot, cls), xs in found.items():
        for x in xs:
            words = []
            (M.exp7 if slot.startswith("exp7") else M.inv7)(x, None, words)
            assert cls in M._word_classes(dict(words)[slot]), (slot, cls, x)
    # every slot's weak word reaches [p, 2^64) on some input
    assert all((s, "weak word >= p") in found for s in M.SLOT_EXPONENTS)
    assert set(found) | set(missing) == {(s, c) for s in M.SLOT_EXPONENTS for c in M.SLOT_CLASSES}


ADD_CLASSES = ["sum p - 1", "sum p", "sum p + 1", "sum in [p, 2^64)", "sum wraps 2^64"]
EXPECTED = {
    "mds1": ["l < lo carry", "canonicalised", "output 0", "output 1", "output p - 1", "output small"],
    "mds2": ["canonicalised", "output 0", "output 1", "output p - 1", "output small"],
    "ark1": ADD_CLASSES,
    "ark2": ADD_CLASSES,
    "ark2 last round": ADD_CLASSES,
    "absorb": ["sum p - 1", "sum p"],
    "jive inputs": ["sum p", "sum in [p, 2^64)", "sum wraps 2^64"],
    "jive outputs": ["sum p", "sum in [p, 2^64)", "sum wraps 2^64"],
    "jive last": ["sum in [p, 2^64)", "sum wraps 2^64"],
}
PRODUCT_CLASSES = ["borrow repaid", "carry folded", "weak word >= p", "operand low half 0", "operand high half 0"]
UNREACHED = {
    ("mds2", "l < lo carry"): "the MDS2 input is the x^(1/7) output: its low halves would have to sum above 2^64 - hi 2^32, "
                              "and the targeted inverse S-box inputs do not give such words",
    ("jive last", "sum p"): "x + y = p exactly makes the merge output word 0 from operands fixed by one permutation input: a "
                            "2^-64 event that no search reaches",
}
for _kind in ("ark1", "ark2", "ark2 last round"):
    UNREACHED[(_kind, "sum in [p, 2^64)")] = ("a canonical word plus a round constant below 2^64 - p lands in [p, 2^64) only when "
                                             "the constant is below 2^32 - 1; none of the 3 x 7 x 12 / 8 constants is")


def _product_reason(slot, cls):
    """why a product slot's class has no targeted input: its operands are powers of the S-box input, and only the first
    products take operands that are targets themselves"""
    e = M.SLOT_EXPONENTS[slot]
    if cls == "borrow repaid":
        return (f"the borrow needs the product's low 64 bits below its top 32 bits (~2^-32 per product); the operands of "
                f"{slot} are powers x^a, x^b with a + b = {e} and targets aim at operand values, not at this relation")
    found, missing = M.slot_targets()
    prev = {"operand low half 0": "word low half 0", "operand high half 0": "word high half 0"}[cls]
    return (f"no operand word of {slot} has a zero half: " + "; ".join(why for (s, c), why in missing.items() if c == prev
                                                                        and s in _operand_slots(slot)) + "; the S-box input x "
            "itself, when it is an operand, is a target only in round 0")


def _operand_slots(slot):
    order = list(M.SLOT_EXPONENTS)
    i = order.index(slot)
    return order[max(0, i - 3):i]


def test_coverage_matrix(capsys):
    log = M.Log()
    for hid in HIDS:
        rng = np.random.default_rng(hid)
        for _, s in M.targeted_states(hid, rng):
            M.permute(hid, s, log)
            M.merge(hid, s[:8], log)
        for row in M.two_block_rows(hid, rng):
            M.hash_elements(hid, row, log)
    for _, s in M.jive_edge_states(np.random.default_rng(3)):
        M.jive(s, log)
    # the MDS carry and the all-(2^64 - 1) input, on crafted words
    h = M.HASHERS[M.RP64]
    M.mds(h, [2**64 - 1] * 12, log, "mds1")
    c0 = h.mat[0][0]
    hi0 = (-(sum(h.mat[0][1:]) * (2**32 - 1)) - 1) * pow(c0, -1, 2**32) % 2**32
    M.mds(h, [(hi0 << 32) | (2**32 - 1)] + [2**64 - 1] * 11, log, "mds1")
    for x in M.SBOX_INPUTS:   # the catalogue through the product chains (the targeted states carry it at round 0)
        M.exp7(x, log)
        M.inv7(x, log)
    cells = [(k, c) for k, cs in EXPECTED.items() for c in cs]
    cells += [(slot, c) for slot in M.SLOT_EXPONENTS for c in PRODUCT_CLASSES]
    rows, missing = [], []
    for kind, c in cells:
        n = log.hits.get((kind, c), 0)
        if n:
            rows.append(f"{kind:18s} {c:22s} {n}")
            continue
        why = UNREACHED.get((kind, c)) or (_product_reason(kind, c) if kind in M.SLOT_EXPONENTS else None)
        if why is None:
            missing.append((kind, c))
        else:
            rows.append(f"{kind:18s} {c:22s} unreached: {why}")
    with capsys.disabled():
        print("\nRescue edge coverage (step kind, class, hits or why not):\n" + "\n".join(rows))
    assert not missing, missing
    # the classes the mutation tests rely on are reached, not excused
    for cell in [("jive inputs", "sum in [p, 2^64)"), ("jive outputs", "sum in [p, 2^64)"), ("jive last", "sum in [p, 2^64)"),
                 ("absorb", "sum p"), ("ark2 last round", "sum p"), ("mds1", "l < lo carry")]:
        assert log.hits.get(cell), cell
