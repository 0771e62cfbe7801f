"""The security estimator without a device: wf_security_estimate (ConjecturedSecurity::compute / ProvenSecurity::compute,
air/src/proof/security.rs) and wf_proof_security (Proof::conjectured_security / proven_security, air/src/proof/mod.rs:96-126).
- every exact assertion of the reference's tests (tests/golden/security_kats.json) against the library and security_ref;
- a grid of a few thousand inputs, library == security_ref, including bounds that come out negative or infinite;
- the relations the reference's tests rely on, on that grid;
- wf_proof_security on the oracle prover's proofs equals the estimate of their context;
- malformed contexts and bad arguments."""
import ctypes as C
import itertools
import json
import os

import numpy as np
import pytest

import airs
import security_ref as sr
import winterfell_b200 as wf

HERE = os.path.dirname(os.path.abspath(__file__))
KATS = json.load(open(os.path.join(HERE, "golden", "security_kats.json")))
ERR_INVALID, ERR_UNSUPPORTED = -2, -3
HASHES = (wf.HASH_BLAKE3_256, wf.HASH_RP64_256, wf.HASH_RPJIVE64_256, wf.HASH_BLAKE3_192, wf.HASH_SHA3_256)


def raw_estimate(words, n, cr, ncons, ncom):
    """wf_security_estimate: (status, (conjectured, ldr, udr))"""
    w = np.zeros(9, dtype=np.uint32)
    w[:len(words)] = words
    out = [C.c_uint32() for _ in range(3)]
    rc = wf.lib().wf_security_estimate(w.ctypes.data_as(C.POINTER(C.c_uint32)), n, cr, ncons, ncom,
                                       C.byref(out[0]), C.byref(out[1]), C.byref(out[2]))
    return rc, tuple(v.value for v in out)


def raw_proof_security(hash_id, proof):
    p = np.frombuffer(bytes(proof), dtype=np.uint8) if len(proof) else np.zeros(1, dtype=np.uint8)
    out = [C.c_uint32() for _ in range(3)]
    rc = wf.lib().wf_proof_security(hash_id, p.ctypes.data_as(C.POINTER(C.c_uint8)), len(proof), C.byref(out[0]), C.byref(out[1]),
                                    C.byref(out[2]))
    return rc, tuple(v.value for v in out)


@pytest.mark.parametrize("i", range(len(KATS["kats"])), ids=[f"{k['test']}-{i}" for i, k in enumerate(KATS["kats"])])
def test_reference_kats(i):
    k = KATS["kats"][i]
    args = (k["opts"], k["trace_length"], k["collision_resistance"], k["num_constraints"], k["num_committed_polys"])
    got = wf.security_estimate(*args)
    assert got == sr.estimate(*args)
    _, ldr, udr = got
    if "udr" in k:
        assert udr == k["udr"]
    if "ldr" in k:
        assert ldr == k["ldr"]


@pytest.mark.parametrize("r", KATS["orderings"], ids=[r["test"] for r in KATS["orderings"]])
def test_reference_orderings(r):
    lo = wf.security_estimate(r["lower"][:8], r["lower"][8], 128, 100, 2)
    hi = wf.security_estimate(r["higher"][:8], r["higher"][8], 128, 100, 2)
    assert lo[1] < hi[1]


def grid():
    """(opts words 0-7, trace length, collision resistance, constraints, committed polynomials): a structured sweep of every
    axis, plus a seeded random sample over all of them at once"""
    cases = []
    counts = (1, 2, 3, 100, 1 << 20, (1 << 64) - 1)   # 1: a batching factor of 0; 2^64 - 1: bounds far below zero
    for ext, lb, bc, bd in itertools.product((1, 2, 3), range(1, 8), (0, 1, 2), (0, 1, 2)):
        cases.append(([40 + 7 * lb, 1 << lb, 20, ext, 4, 7, bc, bd], 1 << (3 + 3 * lb), 128, 100, 8))
    for q, g in itertools.product((1, 2, 13, 26, 27, 40, 79, 80, 81, 128, 200, 255), (0, 1, 16, 32)):   # around the floor of 80
        cases.append(([q, 2, g, 2, 8, 31, 0, 0], 1 << 10, 128, 10, 12))
        cases.append(([q, 8, g, 3, 4, 7, 1, 2], 1 << 16, 128, 3, 5))
    for f, r, logn in itertools.product((2, 4, 8, 16), (0, 1, 3, 7, 63, 255), (3, 4, 5, 6, 11, 12, 20, 32)):
        cases.append(([64, 4, 8, 3, f, r, 2, 1], 1 << logn, 128, 7, 9))
    for ncons, ncom, bc, bd in itertools.product(counts, counts, (0, 1, 2), (0, 1, 2)):
        cases.append(([100, 16, 10, 2, 8, 15, bc, bd], 1 << 14, 128, ncons, ncom))
    for cr in sorted(set(sr.COLLISION_RESISTANCE.values())) + [0, 1, 64, 200]:
        for ext in (1, 2, 3):
            cases.append(([120, 8, 20, ext, 8, 255, 0, 0], 1 << 22, cr, 100, 10))
    rng = np.random.default_rng(2026)
    for _ in range(1500):
        lb = int(rng.integers(1, 8))
        logn = int(rng.integers(3, 33))
        ext = int(rng.integers(1, 4))
        words = [int(rng.integers(1, 256)), 1 << lb, int(rng.integers(0, 33)), ext, 1 << int(rng.integers(1, 5)),
                 (1 << int(rng.integers(0, 9))) - 1, int(rng.integers(0, 3)), int(rng.integers(0, 3))]
        ncons = int(rng.choice([1, 2, int(rng.integers(1, 1 << 12)), int(rng.integers(1, 1 << 62))]))
        ncom = int(rng.choice([1, 2, int(rng.integers(1, 300)), int(rng.integers(1, 1 << 62))]))
        cr = int(rng.choice(list(sr.COLLISION_RESISTANCE.values())))
        cases.append((words, 1 << logn, cr, ncons, ncom))
    return cases


GRID = grid()


@pytest.fixture(scope="module")
def grid_results():
    return [(c, wf.security_estimate(*c)) for c in GRID]


def test_grid_size():
    assert len(GRID) > 2000


def test_grid_matches_restatement(grid_results):
    bad = []
    for c, got in grid_results:
        want = sr.estimate(*c)
        if got != want:
            bad.append((c, got, want))
    assert not bad, bad[:5]


def test_grid_reaches_saturation_and_infinities(grid_results):
    """the grid contains bounds below zero (saturated to 0) and batching factors of 0 (an epsilon of +inf)"""
    zeros = [c for c, (_, ldr, udr) in grid_results if ldr == 0 or udr == 0]
    assert zeros
    assert any(c[3] == 1 and c[0][6] != 0 for c in GRID) and any(c[4] == 1 and c[0][7] != 0 for c in GRID)


def test_more_queries_never_lower_security(grid_results):
    for c, (conj, ldr, udr) in grid_results[::3]:
        words = list(c[0])
        if words[0] >= 255:
            continue
        words[0] += 1 + words[0] // 4
        words[0] = min(words[0], 255)
        c2, l2, u2 = wf.security_estimate(words, *c[1:])
        assert u2 >= udr and l2 >= ldr and c2 >= conj, c


def test_algebraic_batching_never_raises_security_over_linear(grid_results):
    """Algebraic or Horner batching of C >= 2 items costs log2(C - 1) >= 0 bits; Linear costs none"""
    for c, _ in grid_results[::2]:
        words, n, cr, ncons, ncom = c
        if ncons < 2 or ncom < 2:
            continue
        lin = wf.security_estimate(words[:6] + [0, 0], n, cr, ncons, ncom)
        for bc, bd in itertools.product((0, 1, 2), repeat=2):
            got = wf.security_estimate(words[:6] + [bc, bd], n, cr, ncons, ncom)
            assert got[0] == lin[0] and got[1] <= lin[1] and got[2] <= lin[2], (c, bc, bd)
        # Horner and Algebraic cost the same
        assert wf.security_estimate(words[:6] + [1, 1], n, cr, ncons, ncom) == wf.security_estimate(words[:6] + [2, 2], n, cr, ncons, ncom)


def test_blake3_192_caps_at_96(grid_results):
    for c, _ in grid_results[::4]:
        got = wf.security_estimate(c[0], c[1], 96, c[3], c[4])
        assert max(got) <= 96
        full = wf.security_estimate(c[0], c[1], 128, c[3], c[4])
        assert got == tuple(min(v, 96) for v in full)


def test_grinding_counts_only_above_the_floor():
    for q in (26, 27, 39, 40, 79, 80):
        base = wf.security_estimate([q, 8, 0, 3, 8, 31, 0, 0], 1 << 12, 128, 10, 12)[0]
        ground = wf.security_estimate([q, 8, 16, 3, 8, 31, 0, 0], 1 << 12, 128, 10, 12)[0]
        assert base == min(3 * q - 1, 128)
        assert ground == (min(3 * q + 16 - 1, 128) if 3 * q >= 80 else base)


def _context(proof):
    """(opts words 0-7, trace length, constraints, committed polynomials) read from a proof's Context"""
    mw, aw, _nr, logn = proof[0], proof[1], proof[2], proof[3]
    at = 4 + 2 + (proof[4] | proof[5] << 8)
    ml = proof[at]
    at += 1 + ml
    o = list(proof[at:at + 8])
    at += 10
    ncons, _ = _usize(proof, at)
    return [o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7]], 1 << logn, ncons, mw + aw + o[1]


def _usize(b, pos):
    first = b[pos]
    if first == 0:
        return int.from_bytes(b[pos + 1:pos + 9], "little"), pos + 9
    ln = (first & -first).bit_length()
    return int.from_bytes(b[pos:pos + ln], "little") >> ln, pos + ln


@pytest.fixture(scope="module")
def oracle_proofs(oracle):
    out = []
    for h, ext, kw in ((0, 1, dict(folding=2, rem_max_deg=3, blowup=8, num_queries=16)),
                       (1, 2, dict(folding=4, rem_max_deg=7, blowup=4, num_queries=40, grinding=3, batch_c=1)),
                       (3, 3, dict(folding=8, rem_max_deg=7, blowup=16, num_queries=30, batch_d=2)),
                       (4, 2, dict(folding=2, rem_max_deg=1, blowup=2, num_queries=90, grinding=8, batch_c=2, batch_d=1))):
        opts = oracle.make_opts(ext=ext, hash_id=h, **kw)
        desc, trace = airs.fib_small_x(2, 1 << 6)[:2]
        out.append((h, oracle.prove_air(desc, trace, opts)))
    opts = oracle.make_opts(ext=3, hash_id=2, folding=4, rem_max_deg=7, blowup=8, num_queries=20, batch_c=2, batch_d=2)
    desc, trace, builder = airs.perm_rap(1 << 6)
    out.append((2, oracle.prove_air_aux(desc, trace, opts, builder, airs.PERM_RAP_AUX_WIDTH, 2)))
    return out


def test_proof_security_equals_estimate_of_its_context(oracle_proofs):
    for h, proof in oracle_proofs:
        words, n, ncons, ncom = _context(proof)
        want = wf.security_estimate(words, n, sr.COLLISION_RESISTANCE[h], ncons, ncom)
        assert wf.proof_security(h, proof) == want == sr.estimate(words, n, sr.COLLISION_RESISTANCE[h], ncons, ncom)
        # the rest of the proof is not read: the context alone gives the same answer
        assert wf.proof_security(h, proof[:len(proof) // 3]) == want
    # the perm_rap proof has an aux segment: its width counts
    words, n, ncons, ncom = _context(oracle_proofs[-1][1])
    assert ncom == 3 + airs.PERM_RAP_AUX_WIDTH + 8   # x0, x1, b; the aux columns; blowup 8
    # every hasher's collision resistance; Blake3_192 caps at 96
    h, proof = oracle_proofs[2]
    for hh in HASHES:
        assert wf.proof_security(hh, proof) == tuple(min(v, sr.COLLISION_RESISTANCE[hh]) for v in wf.proof_security(0, proof))


def test_proof_security_refusals(oracle_proofs):
    _, proof = oracle_proofs[0]
    at_mod = 6 + (proof[4] | proof[5] << 8)
    at_opts = at_mod + 1 + proof[at_mod]

    def with_byte(at, v):
        b = bytearray(proof)
        b[at] = v
        return bytes(b)
    assert raw_proof_security(0, proof)[0] == 0
    assert raw_proof_security(7, proof)[0] == ERR_UNSUPPORTED
    assert raw_proof_security(-1, proof)[0] == ERR_UNSUPPORTED
    bad = [
        proof[:0], proof[:3], proof[:at_opts + 5], proof[:at_opts + 10],   # ends inside the context
        with_byte(0, 0),                         # main width 0
        with_byte(1, 1),                         # an aux segment without random elements
        with_byte(2, 1),                         # random elements without an aux segment
        with_byte(3, 2),                         # 2^2 rows
        with_byte(3, 40),                        # 2^40 rows: beyond the field's two-adicity with the blowup
        with_byte(at_mod, 0),                    # no modulus
        with_byte(at_mod + 1, 3),                # another modulus
        with_byte(at_opts + 0, 0),               # no queries
        with_byte(at_opts + 1, 3),               # blowup 3
        with_byte(at_opts + 1, 1),               # blowup 1
        with_byte(at_opts + 2, 33),              # grinding 33
        with_byte(at_opts + 3, 0),               # extension degree 0
        with_byte(at_opts + 3, 4),               # extension degree 4
        with_byte(at_opts + 4, 32),              # folding 32
        with_byte(at_opts + 5, 6),               # remainder degree 6
        with_byte(at_opts + 6, 3),               # batching method 3
        with_byte(at_opts + 7, 3),
        with_byte(at_opts + 8, 0),               # no partitions
    ]
    for i, b in enumerate(bad):
        assert raw_proof_security(0, b)[0] == ERR_INVALID, i
    wide = bytearray(proof)
    wide[0], wide[1], wide[2] = 200, 55, 1       # 255 columns: TraceInfo::read_from refuses widths >= 255
    assert raw_proof_security(0, bytes(wide))[0] == ERR_INVALID
    wide[1] = 54
    assert raw_proof_security(0, bytes(wide))[0] == 0
    with pytest.raises(wf.WfError):
        wf.proof_security(0, proof[:5])
    out = [C.c_uint32() for _ in range(3)]
    p = np.frombuffer(proof, dtype=np.uint8)
    pp = p.ctypes.data_as(C.POINTER(C.c_uint8))
    L = wf.lib()
    assert L.wf_proof_security(0, None, len(proof), C.byref(out[0]), C.byref(out[1]), C.byref(out[2])) == ERR_INVALID
    assert L.wf_proof_security(0, pp, len(proof), None, C.byref(out[1]), C.byref(out[2])) == ERR_INVALID
    assert L.wf_proof_security(0, pp, len(proof), C.byref(out[0]), None, C.byref(out[2])) == ERR_INVALID
    assert L.wf_proof_security(0, pp, len(proof), C.byref(out[0]), C.byref(out[1]), None) == ERR_INVALID


def test_estimate_refusals():
    good = [40, 8, 10, 2, 4, 7, 0, 0]
    assert raw_estimate(good, 1 << 10, 128, 10, 10)[0] == 0
    for i, v in ((0, 0), (0, 256), (1, 1), (1, 3), (1, 256), (2, 33), (3, 0), (3, 4), (4, 1), (4, 3), (4, 32), (5, 2), (5, 256),
                 (6, 3), (7, 3)):
        w = list(good)
        w[i] = v
        assert raw_estimate(w, 1 << 10, 128, 10, 10)[0] == ERR_INVALID, (i, v)
    for n in (0, 1, 4, 7, 12, (1 << 32) + 1, 1 << 33, (1 << 64) - 1):
        assert raw_estimate(good, n, 128, 10, 10)[0] == ERR_INVALID, n
    assert raw_estimate(good, 1 << 32, 128, 10, 10)[0] == 0 and raw_estimate(good, 8, 128, 10, 10)[0] == 0
    assert raw_estimate(good, 1 << 10, 128, 0, 10)[0] == ERR_INVALID
    assert raw_estimate(good, 1 << 10, 128, 10, 0)[0] == ERR_INVALID
    # word 8 (hash and partitions) is not read
    w = np.array(good + [0xffffffff], dtype=np.uint32)
    out = [C.c_uint32() for _ in range(3)]
    L = wf.lib()
    assert L.wf_security_estimate(w.ctypes.data_as(C.POINTER(C.c_uint32)), 1 << 10, 128, 10, 10, C.byref(out[0]), C.byref(out[1]),
                                  C.byref(out[2])) == 0
    assert L.wf_security_estimate(None, 1 << 10, 128, 10, 10, C.byref(out[0]), C.byref(out[1]), C.byref(out[2])) == ERR_INVALID
    wp = w.ctypes.data_as(C.POINTER(C.c_uint32))
    assert L.wf_security_estimate(wp, 1 << 10, 128, 10, 10, None, C.byref(out[1]), C.byref(out[2])) == ERR_INVALID
    assert L.wf_security_estimate(wp, 1 << 10, 128, 10, 10, C.byref(out[0]), None, C.byref(out[2])) == ERR_INVALID
    assert L.wf_security_estimate(wp, 1 << 10, 128, 10, 10, C.byref(out[0]), C.byref(out[1]), None) == ERR_INVALID
    with pytest.raises(wf.WfError):
        wf.security_estimate(good, 12, 128, 10, 10)
