"""wf_air_batch_check: the descriptions of one wf_prove_air_batch call may differ only in their public inputs and in the values of
their assertions; every other word (width, degrees, periodic columns, constants, programs, assertion columns / steps / strides /
value counts, exemptions, the aux section) must be identical, and each description must pass wf_air_check. Runs without a GPU;
the fuzz part mutates one description of a batch and checks that the answer follows from which word was changed."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import airs  # noqa: E402
import winterfell_b200 as wf  # noqa: E402

WF_OK, WF_ERR_INVALID = 0, -2
P = wf.P


def value_words(d, unused=None):
    """(indices of the words a batch may vary: assertion values and public inputs, index of the public-input count).
    unused: a set that receives the indices of the operand words CONST and OUT instructions do not read."""
    d = [int(x) for x in d]
    vary, p = [], 1
    unused = set() if unused is None else unused

    def program(p):
        for k in range(d[p]):
            if d[p + 1 + 4 * k] in (3, 4):
                unused.add(p + 4 + 4 * k)
        return p + 1 + 4 * d[p]
    nt = d[p]; p += 1
    for _ in range(nt):
        p += 2 + d[p + 1]
    npd = d[p]; p += 1
    for _ in range(npd):
        p += 1 + d[p]
    p += 1 + d[p]                      # constants
    p += 1                             # num_regs
    p = program(p)
    na = d[p]; p += 1
    for _ in range(na):
        nv = d[p + 3]; p += 4
        vary += range(p, p + nv); p += nv
    pub_at = p
    vary += range(p + 1, p + 1 + d[p]); p += 1 + d[p]
    p += 1                             # exemptions
    if p < len(d):
        nta = d[p + 2]; p += 3
        for _ in range(nta):
            p += 2 + d[p + 1]
        p += 1
        p = program(p)
        naa = d[p]; p += 1
        for _ in range(naa):
            nv = d[p + 3]; p += 4
            vary += range(p, p + 3 * nv); p += 3 * nv
    assert p == len(d)
    return sorted(vary), pub_at


def _all():
    return [("mulfib2", airs.mulfib2(64)[0], 6), ("periodic_mix", airs.periodic_mix(64)[0], 6), ("sequence_mix", airs.sequence_mix(64)[0], 6),
            ("rescue_like", airs.rescue_like(64)[0], 6), ("fib_small_x", airs.fib_small_x(4, 128)[0], 7), ("perm_rap", airs.perm_rap(128)[0], 7)]


def _revalue(d, rng):
    m = d.copy()
    idx, _ = value_words(d)
    m[idx] = rng.integers(0, P, size=len(idx), dtype=np.uint64)
    return m


@pytest.mark.parametrize("name,desc,log_n", _all(), ids=[a[0] for a in _all()])
def test_descriptions_differing_in_values_pass(name, desc, log_n):
    rng = np.random.default_rng(7)
    batch = [desc] + [_revalue(desc, rng) for _ in range(4)]
    assert not all(np.array_equal(batch[0], b) for b in batch[1:])
    assert wf.air_batch_check(batch, log_n, 8) == (WF_OK, "")
    assert wf.air_batch_check([desc], log_n, 8) == (WF_OK, "")


def _pair(n=64, width=2, degs=(1, 1), asserts=((0, 0, 0, [1]), (1, 0, 0, [1]), (1, 63, 0, [5])), exemptions=1, const=None, swap=False):
    A = airs.AirBuilder(width)
    A.pub = [5]
    A.exemptions = exemptions
    t0 = A.sub(A.nxt(0), A.add(A.cur(0), A.cur(1)))
    if const is not None:
        t0 = A.add(t0, A.const(const))
    A.constraint(t0, degs[0])
    A.constraint(A.sub(A.nxt(1), A.add(A.nxt(0), A.cur(1)) if swap else A.add(A.cur(1), A.nxt(0))), degs[1])
    for col, step, stride, vals in asserts:
        if len(vals) > 1:
            A.assert_sequence(col, step, stride, vals)
        elif stride:
            A.assert_periodic(col, step, stride, vals[0])
        else:
            A.assert_single(col, step, vals[0])
    return A.build()


def _without_aux(n):
    # perm_rap's main part alone: the same words up to the aux section
    d = airs.perm_rap(n)[0]
    _, pub_at = value_words(d)
    return d[: pub_at + 1 + int(d[pub_at]) + 1]


STRUCTURAL = {
    "trace width": lambda: (_pair(), _pair(width=3)),
    "transition constraint degrees": lambda: (_pair(), _pair(degs=(2, 1))),
    "constants": lambda: (_pair(const=0), _pair(const=1)),
    "transition program": lambda: (_pair(), _pair(swap=True)),
    "number of assertions": lambda: (_pair(), _pair(asserts=((0, 0, 0, [1]), (1, 0, 0, [1])))),
    "assertion columns": lambda: (_pair(), _pair(asserts=((0, 0, 0, [1]), (1, 0, 0, [1]), (0, 63, 0, [5])))),
    "assertion steps": lambda: (_pair(), _pair(asserts=((0, 0, 0, [1]), (1, 0, 0, [1]), (1, 62, 0, [5])))),
    "assertion strides": lambda: (_pair(asserts=((0, 1, 4, [1]),)), _pair(asserts=((0, 1, 8, [1]),))),
    "assertion value counts": lambda: (_pair(asserts=((0, 1, 16, [1]),)), _pair(asserts=((0, 1, 16, [1, 2, 3, 4]),))),
    "transition exemptions": lambda: (_pair(), _pair(exemptions=2)),
    "aux segment": lambda: (_without_aux(64), airs.perm_rap(64)[0]),
}


@pytest.mark.parametrize("reason", sorted(STRUCTURAL))
def test_each_structural_difference_is_refused_with_its_reason(reason):
    a, b = STRUCTURAL[reason]()
    assert wf.air_check(a, 6, 8) == (WF_OK, "") and wf.air_check(b, 6, 8) == (WF_OK, "")
    assert wf.air_batch_check([a, b], 6, 8) == (WF_ERR_INVALID, f"proof 1 differs from proof 0 in its {reason}")
    assert wf.air_batch_check([a, a, b], 6, 8) == (WF_ERR_INVALID, f"proof 2 differs from proof 0 in its {reason}")
    assert wf.air_batch_check([b, a], 6, 8)[0] == WF_ERR_INVALID


def _word_variant(desc, at, delta):
    m = desc.copy()
    m[at] = np.uint64((int(m[at]) + delta) % P)
    return m


def test_periodic_values_and_aux_words_are_structure():
    d = airs.periodic_mix(64)[0]
    at = 12                             # first value of the first periodic column: after [w, nT, {1, 1, 8}, {3, 1, 4}, {2, 0}, nP, len]
    assert int(d[at - 1]) == 8 and int(d[at - 2]) == 2
    assert wf.air_batch_check([d, _word_variant(d, at, 1)], 6, 8) == (WF_ERR_INVALID, "proof 1 differs from proof 0 in its periodic columns")
    a = airs.perm_rap(64)[0]
    _, pub_at = value_words(a)
    aux_at = pub_at + 1 + int(a[pub_at]) + 1            # [aw, nr, nTa, ...]
    for off, why in ((0, "aux width or random elements"), (1, "aux width or random elements")):
        rc, msg = wf.air_batch_check([a, _word_variant(a, aux_at + off, 1)], 6, 8)
        assert rc == WF_ERR_INVALID and msg.startswith("proof 1"), (off, msg)
    deg_at = aux_at + 3                                 # base degree of the first aux transition constraint
    b = _word_variant(a, deg_at, 1)
    assert wf.air_check(b, 6, 8)[0] == WF_OK
    assert wf.air_batch_check([a, b], 6, 8) == (WF_ERR_INVALID, "proof 1 differs from proof 0 in its aux transition constraint degrees")
    # an aux assertion value may differ, its step may not
    idx, _ = value_words(a)
    aux_vals = [i for i in idx if i > aux_at]
    assert wf.air_batch_check([a, _word_variant(a, aux_vals[0], 3)], 6, 8) == (WF_OK, "")
    step_at = aux_vals[0] - 3                           # {column, first_step, stride, nvals, values}
    rc, msg = wf.air_batch_check([a, _word_variant(a, step_at, 1)], 6, 8)
    assert rc == WF_ERR_INVALID and msg == "proof 1 differs from proof 0 in its aux assertion steps", msg


def test_each_description_is_checked_and_named():
    good = airs.sequence_mix(64)[0]
    assert wf.air_batch_check([good, good], 5, 8) == (WF_ERR_INVALID, "proof 0: invalid assertion")   # n / stride != number of values
    bad = good.copy()
    bad[0] = 0
    assert wf.air_batch_check([good, good, bad], 6, 8) == (WF_ERR_INVALID, "proof 2: malformed AIR description")
    assert wf.air_batch_check([good, airs.periodic_mix(64)[0]], 6, 2) == (WF_ERR_INVALID, "proof 1: blowup factor too small for the constraint degrees")
    assert wf.air_batch_check([], 6, 8) == (WF_ERR_INVALID, "bad arguments")
    assert wf.air_batch_check([good], 6, 12) == (WF_ERR_INVALID, "bad arguments")


@pytest.mark.parametrize("seed", range(4))
def test_fuzzed_batches_follow_the_changed_word(seed):
    rng = np.random.default_rng(2000 + seed)
    interesting = np.array([0, 1, 2, 3, 4, 7, 8, 16, 255, 256, 4096, 1 << 20, (1 << 32) - 1, 1 << 32, (1 << 63), P - 1, P, (1 << 64) - 1],
                           dtype=np.uint64)
    seen = {WF_OK: 0, WF_ERR_INVALID: 0}
    for name, d, log_n in _all():
        unused = set()
        vary, pub_at = value_words(d, unused)
        vary = set(vary)
        for _ in range(150):
            m = d.copy()
            kind = rng.integers(0, 4)
            if kind == 0:                                   # truncate or extend: a different parse
                m = m[: rng.integers(0, len(m))] if rng.integers(0, 2) else np.concatenate([m, rng.choice(interesting, size=rng.integers(1, 5))])
                at = None
            else:
                at = int(rng.choice(sorted(vary))) if kind == 1 else int(rng.integers(0, len(m)))
                v = rng.choice(interesting) if rng.integers(0, 2) else np.uint64((int(m[at]) + int(rng.integers(1, 3))) % (1 << 64))
                if v == m[at]:
                    continue
                m[at] = v
            j = int(rng.integers(1, 4))
            batch = [d] * j + [np.ascontiguousarray(m, dtype=np.uint64)]
            rc, msg = wf.air_batch_check(batch, log_n, 8)
            assert rc in (WF_OK, WF_ERR_INVALID), (name, rc, msg)
            assert (rc == WF_OK) == (msg == "")
            single = wf.air_check(m, log_n, 8)[0]
            if single != WF_OK:
                assert rc == WF_ERR_INVALID and msg.startswith(f"proof {j}"), (name, at, msg)
            elif at is not None and at in vary:
                assert rc == WF_OK, (name, at, msg)
            elif at is not None and at != pub_at and at not in unused:   # the parser keeps 32 bits of an unread operand
                assert rc == WF_ERR_INVALID and msg.startswith(f"proof {j} differs from proof 0"), (name, at, msg)
            seen[rc] += 1
    assert seen[WF_ERR_INVALID] > 200 and seen[WF_OK] > 100
