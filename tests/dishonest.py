"""Dishonest proofs for the verifier tests: proofs made by the oracle prover's tamper hook (oracle.oracle.tamper) that open
every commitment correctly and are still wrong, so that they reach the checks a byte flip never reaches: the FRI layer
folding (verdict 7), the DEEP composition at the queries and the remainder (verdict 8). Each case carries the verdict it must
get; the exact code shows that every earlier check (openings, OOD, proof of work) passed.

Shared by test_oracle_dishonest_proofs.py (the oracle's verdicts, on the CPU) and test_gpu_verify_dishonest.py (the
device's verdicts against the oracle's)."""
from collections import namedtuple

import numpy as np

import airs
from oracle import oracle as O

P = O.P
ACCEPT, OOD, TRACE_QUERY, CONSTRAINT_QUERY, FRI_LAYER, FRI_FOLD, FRI_REMAINDER = 0, 2, 4, 5, 6, 7, 8

# name: what was done; key: proofs with the same key share an AIR structure (one verifier batch); values_fn: the
# get_aux_assertions callback the verifier needs (None: none)
Case = namedtuple("Case", "name key desc proof want hash_id positions values_fn")


def last_coord(ext, v=5):
    """a delta that touches only the last extension coordinate: a check that compares word 0 alone misses it"""
    return tuple([0] * (ext - 1) + [v])


def every_coord(ext):
    return (3, 7, 11)[:ext]


def num_layers(n, opts):
    blowup, folding, rem = int(opts[1]), int(opts[4]), int(opts[5])
    return O.fri_num_layers(n * blowup, folding, rem, blowup)


def fib_from(n, a0, b0):
    """fib_small started at (a0, b0): description and trace (assertions at step 0 and n - 1)"""
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


class Prover:
    """Proves one AIR ('fib' = fib_small_x(1, n), 'perm_rap' = two segments, 'perm_rap_dyn' = two segments with an aux
    assertion value drawn from the random elements) at trace length n, honestly or with tampers."""

    def __init__(self, air, n, trace=None):
        self.air, self.n = air, n
        self.values_fn = None
        if air == "fib":
            self.desc, self.trace = airs.fib_small_x(1, n)
        else:
            self.desc, self.trace, self.builder = airs.perm_rap(n, dyn_last_q=air == "perm_rap_dyn")
            if air == "perm_rap_dyn":
                self.values_fn = self.builder.values_fn
        if trace is not None:
            self.trace = trace

    @property
    def aux_width(self):
        return 0 if self.air == "fib" else airs.PERM_RAP_AUX_WIDTH

    def prove(self, opts, tampers=()):
        """(proof, query positions)"""
        if self.air == "fib":
            return O.prove_air(self.desc, self.trace, opts, tamper=list(tampers))
        if self.air == "perm_rap":
            return O.prove_air_aux(self.desc, self.trace, opts, self.builder, airs.PERM_RAP_AUX_WIDTH, 2, tamper=list(tampers))
        nv = self.builder.num_values
        return O.prove_air_aux_dyn(self.desc, self.trace, opts, self.builder, self.values_fn, airs.PERM_RAP_AUX_WIDTH, 2, nv,
                                   tamper=list(tampers))

    def oracle_verdict(self, proof, hash_id):
        if self.values_fn is None:
            return O.verify_air(self.desc, proof, hash_id)
        return O.verify_air_dyn(self.desc, proof, hash_id, self.values_fn, 2, self.builder.num_values, int(proof[15 + 3]))

    def case(self, name, opts, tampers, want):
        proof, pos = self.prove(opts, tampers)
        return Case(name, (self.air, self.n), self.desc, proof, want, int(opts[8]) & 0xFF, pos, self.values_fn)


def all_rows_cases(air, n, opts):
    """Every all-rows tamper of one proof shape: the LDE targets and FRI layers 0 .. last give 7; with no FRI layer the DEEP
    codeword is the remainder's, so they give 8. REMAINDER and REMAINDER_LONG give 8."""
    pv = Prover(air, n)
    ext, nl = int(opts[3]), num_layers(n, opts)
    fold = FRI_FOLD if nl else FRI_REMAINDER
    spec = [("main col 0", [O.tamper(O.MAIN_LDE, 0, delta=(3,))], fold),
            ("main col 1", [O.tamper(O.MAIN_LDE, 1, delta=(P - 1,))], fold),
            ("constraint col 0, last coordinate", [O.tamper(O.CONSTRAINT_LDE, 0, delta=last_coord(ext))], fold)]
    if pv.aux_width:
        spec += [("aux col 0, last coordinate", [O.tamper(O.AUX_LDE, 0, delta=last_coord(ext))], fold),
                 ("aux col 2", [O.tamper(O.AUX_LDE, 2, delta=every_coord(ext))], fold),
                 ("constraint col 1", [O.tamper(O.CONSTRAINT_LDE, 1, delta=every_coord(ext))], fold)]
    for k in range(max(nl, 1)):
        delta = last_coord(ext) if k % 2 == 0 else every_coord(ext)
        spec.append((f"FRI layer {k}", [O.tamper(O.FRI_LAYER, k, delta=delta)], fold))
    spec += [("remainder coefficient 0, last coordinate", [O.tamper(O.REMAINDER, 0, delta=last_coord(ext))], FRI_REMAINDER),
             ("remainder one coefficient too long", [O.tamper(O.REMAINDER_LONG, 1)], FRI_REMAINDER)]
    if nl:
        spec.append((f"FRI layer {nl} (the remainder's codeword)", [O.tamper(O.FRI_LAYER, nl, delta=(1,))], FRI_REMAINDER))
    return [pv.case(f"{air} n={n} {name}", opts, t, want) for name, t, want in spec]


def shape_opts(i, **kw):
    """the i-th option set of a matrix: the batching methods and the partitions rotate with i"""
    kw.setdefault("batch_c", i % 3)
    kw.setdefault("batch_d", (i // 3) % 3)
    if i % 2:
        kw.setdefault("num_partitions", 2)
        kw.setdefault("hash_rate", 8)
    return O.make_opts(**kw)


def matrix_cases(hash_id, rotate=True):
    """All-rows tampers over ext 1, 2, 3, folding 2, 4, 8, 16 and a one- and a two-segment AIR (64 rows, blowup 8,
    remainder degree 3: 4, 2, 2 and 1 FRI layers)."""
    cases, i = [], 0
    for air in ("fib", "perm_rap"):
        for ext in (1, 2, 3):
            for folding in (2, 4, 8, 16):
                kw = dict(num_queries=20, blowup=8, ext=ext, folding=folding, rem_max_deg=3, hash_id=hash_id)
                opts = shape_opts(i, **kw) if rotate else O.make_opts(**kw)
                cases += all_rows_cases(air, 64, opts)
                i += 1
    return cases


def no_layer_cases(hash_id):
    """the corner with no FRI layer (N = (7 + 1) * 128): the remainder check is the DEEP check"""
    opts = O.make_opts(num_queries=5, blowup=128, grinding=0, ext=1, folding=16, rem_max_deg=7, hash_id=hash_id)
    assert num_layers(8, opts) == 0
    pv = Prover("fib", 8)
    return [pv.case("no layers: DEEP codeword", opts, [O.tamper(O.FRI_LAYER, 0, delta=(9,))], FRI_REMAINDER),
            pv.case("no layers: main col 1", opts, [O.tamper(O.MAIN_LDE, 1, delta=(2,))], FRI_REMAINDER),
            pv.case("no layers: remainder", opts, [O.tamper(O.REMAINDER, 3, delta=(1,))], FRI_REMAINDER),
            pv.case("no layers: remainder too long", opts, [O.tamper(O.REMAINDER_LONG, 2)], FRI_REMAINDER),
            pv.case("no layers: honest", opts, [], ACCEPT)]


def single_row_cases(hash_id, ext, folding=4):
    """One LDE row or one position of the DEEP codeword tampered (16 rows, blowup 4: 64 positions, 28 queries): 7 exactly
    when a query lands on it. Otherwise an LDE row is never read (0), while the DEEP codeword stops being of low degree,
    which the remainder check sees (8). Returns (cases, kinds): kinds[i] is 'missed', 'queried first' or 'queried later'
    (the position is queried after another one of its FRI row, so a fold check that stops at its row's first query
    misses it)."""
    n, blowup = 16, 4
    opts = O.make_opts(num_queries=28, blowup=blowup, ext=ext, folding=folding, rem_max_deg=3, hash_id=hash_id)
    N = n * blowup
    row_len = N // folding
    pv = Prover("fib", n)
    cases, kinds = [], []
    for target, col in ((O.MAIN_LDE, 1), (O.FRI_LAYER, 0)):
        for r in range(N):
            delta = (5,) if target == O.MAIN_LDE else last_coord(ext, 1 + r)
            proof, pos = pv.prove(opts, [O.tamper(target, col, row=r, delta=delta)])
            hit = r in set(int(p) for p in pos)
            want = FRI_FOLD if hit else ACCEPT if target == O.MAIN_LDE else FRI_REMAINDER
            earlier = any(int(p) < r and int(p) % row_len == r % row_len for p in pos)
            kinds.append("missed" if not hit else "queried later" if earlier else "queried first")
            name = f"single row {r} of {'main col 1' if target == O.MAIN_LDE else 'the DEEP codeword'}"
            cases.append(Case(name, ("fib", n), pv.desc, proof, want, hash_id, pos, None))
    return cases, kinds


def precedence_cases(hash_id, ext=2):
    """Two failures in one proof: the first check in the verifier's order decides (64 rows, folding 2: layers 0 .. 3)."""
    opts = O.make_opts(num_queries=20, blowup=8, ext=ext, folding=2, rem_max_deg=3, hash_id=hash_id)
    assert num_layers(64, opts) == 4
    d = last_coord(ext)
    fib, rap = Prover("fib", 64), Prover("perm_rap", 64)
    return [
        fib.case("layer 1 tampered + layer 3 opening flipped", opts, [O.tamper(O.FRI_LAYER, 1, delta=d), O.tamper(O.FLIP_FRI, 3, row=5)],
                 FRI_FOLD),
        fib.case("layer 3 tampered + layer 1 opening flipped", opts, [O.tamper(O.FRI_LAYER, 3, delta=d), O.tamper(O.FLIP_FRI, 1, row=2)],
                 FRI_LAYER),
        fib.case("main LDE tampered + constraint opening flipped", opts,
                 [O.tamper(O.MAIN_LDE, 0, delta=(4,)), O.tamper(O.FLIP_CONSTRAINT, row=9, delta=(3,))], CONSTRAINT_QUERY),
        fib.case("layer 2 tampered + remainder too long", opts, [O.tamper(O.FRI_LAYER, 2, delta=d), O.tamper(O.REMAINDER_LONG, 1)],
                 FRI_FOLD),
        fib.case("constraint LDE tampered + trace opening flipped", opts,
                 [O.tamper(O.CONSTRAINT_LDE, 0, delta=d), O.tamper(O.FLIP_TRACE, row=1)], TRACE_QUERY),
        fib.case("remainder tampered + layer 0 tampered", opts, [O.tamper(O.REMAINDER, 0, delta=d), O.tamper(O.FRI_LAYER, 0, delta=d)],
                 FRI_FOLD),
        rap.case("aux LDE tampered + aux opening flipped", opts, [O.tamper(O.AUX_LDE, 1, delta=d), O.tamper(O.FLIP_AUX, row=17)],
                 TRACE_QUERY),
        rap.case("aux LDE tampered + constraint opening flipped", opts,
                 [O.tamper(O.AUX_LDE, 1, delta=d), O.tamper(O.FLIP_CONSTRAINT, row=0)], CONSTRAINT_QUERY),
    ]


def bad_trace_cases(hash_id, ext=2):
    """An honest prover on a trace that breaks its AIR: the OOD check refuses it (2)."""
    opts = O.make_opts(num_queries=20, blowup=8, ext=ext, folding=4, rem_max_deg=7, hash_id=hash_id)
    n = 64
    fib = Prover("fib", n)
    t = fib.trace.copy()
    t[0, 17] = (int(t[0, 17]) + 1) % P
    transition = Prover("fib", n, trace=t)
    _, shifted = fib_from(n, 2, 1)            # every transition holds, the assertions at steps 0 and n - 1 do not
    assertion = Prover("fib", n, trace=shifted)
    rap = Prover("perm_rap", n)
    t = rap.trace.copy()
    t[2, 3] = (int(t[2, 3]) + 1) % P           # b is no longer a permutation of x0
    perm = Prover("perm_rap", n, trace=t)
    return [transition.case("broken transition", opts, [], OOD), assertion.case("broken assertions", opts, [], OOD),
            perm.case("broken permutation", opts, [], OOD)]


def flip_set(proof, seed):
    """the byte-flip set of the verifier's refusal tests: every byte of the first and last 160, every fourth in between,
    truncations, one byte more, a trace length that wraps, hash_rate 0, and the proof itself"""
    rng = np.random.default_rng(seed)
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
    zero_rate[24] = 0   # ProofOptions::hash_rate: the last of the ten option bytes after the 15-byte trace info + modulus
    return muts + [bytes(wrap), bytes(zero_rate), proof]


# ---- proofs carrying words of p or more ----
MALFORMED = 1


def _usize(b, pos):
    first = b[pos]
    ln = 9 if first == 0 else (first & -first).bit_length()
    if ln == 9:
        return int.from_bytes(b[pos + 1:pos + 9], "little"), pos + 9
    return int.from_bytes(b[pos:pos + ln], "little") >> ln, pos + ln


def proof_fields(proof, hash_id, two_segments):
    """byte offsets of the proof's parts (the layout parse_proof reads): {name: (offset, length)} for 'commitments',
    'trace values' / 'trace path', ['aux values' / 'aux path'], 'constraint values' / 'constraint path', 'ood trace',
    'ood quotient', 'fri values 0' / 'fri path 0' .., 'remainder'"""
    b = proof
    pos = 4
    meta = int.from_bytes(b[pos:pos + 2], "little")
    pos += 2 + meta
    pos += 1 + b[pos]                 # field modulus bytes
    pos += 10                         # options
    _, pos = _usize(b, pos)           # number of constraints
    pos += 1                          # unique queries
    out = {}
    clen = int.from_bytes(b[pos:pos + 2], "little")
    out["commitments"] = (pos + 2, clen)
    pos += 2 + clen
    for seg in ["trace"] + (["aux"] if two_segments else []) + ["constraint"]:
        for part in ("values", "path"):
            n, pos = _usize(b, pos)
            out[f"{seg} {part}"] = (pos, n)
            pos += n
    for name in ("ood trace", "ood quotient"):
        n = int.from_bytes(b[pos:pos + 2], "little")
        out[name] = (pos + 3, n - 1)  # after the frame-size byte
        pos += 2 + n
    nl = b[pos]
    pos += 1
    for i in range(nl):
        for part in ("values", "path"):
            n = int.from_bytes(b[pos:pos + 4], "little")
            out[f"fri {part} {i}"] = (pos + 4, n)
            pos += 4 + n
    n = int.from_bytes(b[pos:pos + 2], "little")
    out["remainder"] = (pos + 2, n)
    assert pos + 2 + n + 1 + 8 == len(b)
    return out


def _first_path_digest(proof, off, n):
    """offset of the first digest of a batch Merkle opening: depth byte, vint count, per node vector a vint length"""
    pos = off + 1
    nv, pos = _usize(proof, pos)
    for _ in range(nv):
        ln, pos = _usize(proof, pos)
        if ln:
            return pos
    return None


def _put(proof, at, word):
    b = bytearray(proof)
    b[at:at + 8] = int(word).to_bytes(8, "little")
    return bytes(b)


def noncanonical_cases(hash_id, ext):
    """An honest two-segment proof with one word replaced by a word of p or more. BaseElement::read_from refuses it in every
    field element the verifier reads (math/src/field/f64/mod.rs:673-681): an opened main, aux or constraint value, an OOD
    value, a FRI layer value, a remainder coefficient all give ProofDeserializationError (1). A Rescue digest word is read
    through BaseElement::new (rp64_256/digest.rs:61-69, rp64_256_jive/digest.rs:61-69), which reduces it: 2^64 - 1 stands for
    2^32 - 2, a different digest, so a commitment or path node changed so fails the check its digest meets (`want` None: the
    oracle decides). Words p + w for a digest word w < 2^32 - 1 would change nothing; honest digests almost never have one,
    so that is covered at the merge level. Byte digests (BLAKE3, SHA3) are bytes: the same replacement fails the same way."""
    opts = O.make_opts(num_queries=12, blowup=8, ext=ext, folding=4, rem_max_deg=3, hash_id=hash_id)
    pv = Prover("perm_rap", 64)
    proof, pos = pv.prove(opts)
    f = proof_fields(proof, hash_id, True)
    top = 2**64 - 1
    spec = [("honest", proof, ACCEPT)]
    for name, word_index, w in (("trace values", 0, top), ("trace values", -1, P), ("aux values", 1, top),
                                ("constraint values", -1, P + 5), ("ood trace", 0, top), ("ood trace", -1, P),
                                ("ood quotient", 2, top), ("fri values 0", 3, P), ("remainder", -1, top)):
        off, n = f[name]
        k = word_index % (n // 8)
        spec.append((f"{name} word {k} = {w:#x}", _put(proof, off + 8 * k, w), MALFORMED))
    if ext > 1:   # the last coordinate of the first extension element of the remainder
        off, _ = f["remainder"]
        spec.append((f"remainder coordinate {ext - 1} = p", _put(proof, off + 8 * (ext - 1), P), MALFORMED))
    if hash_id in (1, 2):
        off, _ = f["commitments"]
        spec.append(("trace commitment word 1 = 2^64 - 1", _put(proof, off + 8, top), None))
        spec.append(("constraint commitment word 0 = 2^64 - 1", _put(proof, off + 64, top), None))
        at = _first_path_digest(proof, *f["trace path"])
        spec.append(("trace path node word 0 = 2^64 - 1", _put(proof, at, top), None))
        at = _first_path_digest(proof, *f["fri path 0"])
        spec.append(("FRI path node word 3 = 2^64 - 1", _put(proof, at + 24, top), None))
    return [Case(f"h={hash_id} ext={ext} {name}", ("perm_rap", 64), pv.desc, p, want, hash_id, pos, None) for name, p, want in spec]
