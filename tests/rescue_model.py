"""An exact model of the device's Rescue permutations (winterfell_b200/csrc/rp64.cuh, rpjive.cuh, alg_hash.cuh) on Python
integers, and the inputs that drive its reduction edges.

The S-boxes run on weakly reduced words (gl_mul_weak: congruent to the product, below 2^64 but not always below p), so the
device's intermediate WORDS are not a function of the values alone. The model restates gl_mul_weak, gl_sqr_weak, gl_add and
the MDS with gl_reduce128 step by step as their PTX sequences compute them, and reports every product, MDS, round-constant,
absorb and Jive step with its operand and result words and the edge classes it reaches.

Backwards, it works on values: from a state chosen at any step boundary of any round it returns the permutation input that
reaches it (subtract the round constants, apply the inverse circulant mod p, and swap x^7 with x^(1/7): gcd(7, p - 1) = 1).
Product slots are aimed at through their exponent: slot value v = x^e is solved by a discrete logarithm to the generator 7
(p - 1 = 2^32 3 5 17 257 65537, so Pohlig-Hellman is cheap)."""
import functools
import os
import re

P = 0xFFFFFFFF00000001
EPS = 0xFFFFFFFF
M64 = (1 << 64) - 1
INV7 = 10540996611094048183          # 7 * INV7 = 1 mod p - 1
RP64, RPJIVE = 1, 2                 # winterfell_b200.HASH_RP64_256 / HASH_RPJIVE64_256

_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "winterfell_b200", "csrc")


def _tables(fname):
    text = open(os.path.join(_CSRC, fname)).read()
    out = {}
    for m in re.finditer(r"(\w+)(\[[^=]*)=\s*\{(.*?)\};", text, re.S):
        out[m.group(1)] = [int(v) for v in re.findall(r"(\d+)ULL", m.group(3))]
    return out


_T64, _TJ = _tables("rp64_constants.inc"), _tables("rpjive_constants.inc")


class Hasher:
    def __init__(self, hid):
        self.hid = hid
        t, pre = (_T64, "RP64") if hid == RP64 else (_TJ, "RPJ")
        self.w = 12 if hid == RP64 else 8
        self.row = t[pre + "_MDS_ROW0"]
        w = self.w
        self.ark1 = [t[pre + "_ARK1"][r * w:(r + 1) * w] for r in range(7)]
        self.ark2 = [t[pre + "_ARK2"][r * w:(r + 1) * w] for r in range(7)]
        self.mat = [[self.row[(j + w - i) % w] for j in range(w)] for i in range(w)]
        self.inv_mat = _inverse_mod_p(self.mat)


def _inverse_mod_p(m):
    n = len(m)
    a = [list(r) + [int(i == j) for j in range(n)] for i, r in enumerate(m)]
    for c in range(n):
        piv = next(r for r in range(c, n) if a[r][c] % P)
        a[c], a[piv] = a[piv], a[c]
        iv = pow(a[c][c], P - 2, P)
        a[c] = [x * iv % P for x in a[c]]
        for r in range(n):
            if r != c and a[r][c]:
                f = a[r][c]
                a[r] = [(x - f * y) % P for x, y in zip(a[r], a[c])]
    return [r[n:] for r in a]


def solve_mod_p(m, rhs):
    """x with m x = rhs (mod p), m square and invertible"""
    inv = _inverse_mod_p(m)
    return [sum(a * b for a, b in zip(r, rhs)) % P for r in inv]


HASHERS = {RP64: Hasher(RP64), RPJIVE: Hasher(RPJIVE)}


# ---- word-level arithmetic, as the PTX sequences of gl64.cuh compute it ----
class Log:
    """edge classes reached, keyed by (step kind, class); `None` records nothing"""

    def __init__(self):
        self.hits = {}

    def add(self, kind, cls):
        self.hits[(kind, cls)] = self.hits.get((kind, cls), 0) + 1


def _fold(lo, c2, c3, log=None, kind=None):
    """(lo - c3, a borrow repaid with -(2^32 - 1)) + c2 (2^32 - 1): (carry k, 64-bit word)"""
    t = (lo - c3) & M64
    if lo < c3:
        t = (t - EPS) & M64
        if log:
            log.add(kind, "borrow repaid")
    u = t + c2 * EPS
    return u >> 64, u & M64


def mul_weak(a, b, log=None, kind="mul"):
    """gl_mul_weak (and gl_sqr_weak, whose three partial products give the same 128-bit product) for any 64-bit words"""
    if log:
        for x in (a, b):
            if x & EPS == 0:
                log.add(kind, "operand low half 0")
            if x >> 32 == 0:
                log.add(kind, "operand high half 0")
    t = a * b
    k, r = _fold(t & M64, (t >> 64) & EPS, t >> 96, log, kind)
    if k and log:
        log.add(kind, "carry folded")
    r = (r + k * EPS) & M64
    if log and r >= P:
        log.add(kind, "weak word >= p")
    return r


def reduce128(lo, hi, log=None, kind="mds"):
    """gl_reduce128: canonical lo + 2^64 hi mod p"""
    k, r = _fold(lo, hi & EPS, hi >> 32, log, kind)
    k2 = (r + EPS) >> 64
    if k2 and log:
        log.add(kind, "canonicalised")
    return (r + (k + k2) * EPS) & M64


def add(a, b, log=None, kind="add"):
    """device gl_add: a - (p - b), a borrow repaid with -(2^32 - 1); canonical for canonical a, b"""
    if log:
        s = a + b
        for name, v in (("sum p - 1", P - 1), ("sum p", P), ("sum p + 1", P + 1)):
            if s == v:
                log.add(kind, name)
        if P <= s < 1 << 64:
            log.add(kind, "sum in [p, 2^64)")
        if s >= 1 << 64:
            log.add(kind, "sum wraps 2^64")
    nb = (P - b) & M64
    r = (a - nb) & M64
    if a < nb:
        r = (r - EPS) & M64
    return r


def mds(h, s, log=None, kind="mds"):
    out = []
    for i in range(h.w):
        lo = sum((s[j] & EPS) * h.mat[i][j] for j in range(h.w))
        hi = sum((s[j] >> 32) * h.mat[i][j] for j in range(h.w))
        l = (lo + (hi << 32)) & M64
        carry = l < lo
        if carry and log:
            log.add(kind, "l < lo carry")
        r = reduce128(l, (hi >> 32) + carry, log, kind)
        if log:
            for name, v in (("output 0", 0), ("output 1", 1), ("output p - 1", P - 1)):
                if r == v:
                    log.add(kind, name)
            if 1 < r < 1 << 32:
                log.add(kind, "output small")
        out.append(r)
    return out


# ---- the S-box chains, slot by slot ----
def exp7(x, log=None, slots=None):
    """rp64_exp7; slots (optional list) receives (slot name, word)"""
    x2 = mul_weak(x, x, log, "exp7 x2")
    x4 = mul_weak(x2, x2, log, "exp7 x4")
    x3 = mul_weak(x2, x, log, "exp7 x3")
    r = mul_weak(x3, x4, log, "exp7 x7")
    if slots is not None:
        slots += [("exp7 x2", x2), ("exp7 x4", x4), ("exp7 x3", x3), ("exp7 x7", r)]
    return r


def inv7(x, log=None, slots=None):
    """one element of rp64_inv7_group<G> (the G chains are independent): x^(1/7) by the chain of apply_inv_sbox"""
    def m(a, b, name):
        r = mul_weak(a, b, log, name)
        if slots is not None:
            slots.append((name, r))
        return r
    t1 = m(x, x, "inv t1")
    t2 = m(t1, t1, "inv t2")
    b = m(m(t1, t2, "inv t1t2"), x, "inv b")
    acc = t2
    for i in range(3):
        acc = m(acc, acc, f"inv sq3.{i}")
    acc = t3 = m(acc, t2, "inv t3")
    for i in range(6):
        acc = m(acc, acc, f"inv sq6a.{i}")
    acc = t4 = m(acc, t3, "inv t4")
    for i in range(12):
        acc = m(acc, acc, f"inv sq12.{i}")
    acc = m(acc, t4, "inv t5")
    for i in range(6):
        acc = m(acc, acc, f"inv sq6b.{i}")
    acc = t6 = m(acc, t3, "inv t6")
    for i in range(31):
        acc = m(acc, acc, f"inv sq31.{i}")
    a = m(acc, t6, "inv t7")
    a = m(m(a, a, "inv t7^2"), t6, "inv t7^2 t6")
    a = m(a, a, "inv last sq.0")
    a = m(a, a, "inv last sq.1")
    return m(a, b, "inv out")


def _slot_exponents():
    """exponent of x (mod p - 1) of every product slot of exp7 and inv7"""
    out = {}

    global mul_weak   # exponent arithmetic through the same chain code
    real = mul_weak
    try:
        mul_weak = lambda a, b, log=None, kind="": (a + b) % (P - 1)   # noqa: E731
        s1, s2 = [], []
        exp7(1, None, s1)
        inv7(1, None, s2)
    finally:
        mul_weak = real
    for name, e in s1 + s2:
        out[name] = e
    return out


SLOT_EXPONENTS = _slot_exponents()
assert SLOT_EXPONENTS["exp7 x7"] == 7 and SLOT_EXPONENTS["inv out"] == INV7


# ---- the permutations ----
BOUNDARIES = ("sbox in", "mds1 out", "inv in", "mds2 out", "round out")


def permute(hid, state, log=None, trace=None):
    """rp64_permute / rpj_permute on any words; trace (optional dict) receives the state at every (round, boundary)"""
    h = HASHERS[hid]
    s = list(state)
    for r in range(7):
        if trace is not None:
            trace[(r, "sbox in")] = list(s)
        s = [exp7(x, log) for x in s]
        s = mds(h, s, log, "mds1")
        if trace is not None:
            trace[(r, "mds1 out")] = list(s)
        s = [add(x, c, log, "ark1") for x, c in zip(s, h.ark1[r])]
        if trace is not None:
            trace[(r, "inv in")] = list(s)
        s = [inv7(x, log) for x in s]
        s = mds(h, s, log, "mds2")
        if trace is not None:
            trace[(r, "mds2 out")] = list(s)
        s = [add(x, c, log, "ark2 last round" if r == 6 else "ark2") for x, c in zip(s, h.ark2[r])]
        if trace is not None:
            trace[(r, "round out")] = list(s)
    return s


def backward(hid, r, boundary, values):
    """the permutation input whose state at (round r, boundary) has these (canonical) values"""
    h = HASHERS[hid]
    s = [v % P for v in values]
    inv_mds = lambda v: [sum(a * b for a, b in zip(row, v)) % P for row in h.inv_mat]   # noqa: E731
    k = BOUNDARIES.index(boundary)
    for rr in range(r, -1, -1):
        if k >= 4:
            s = [(x - c) % P for x, c in zip(s, h.ark2[rr])]
        if k >= 3:
            s = [pow(x, 7, P) for x in inv_mds(s)]             # undo MDS, then x^(1/7)
        if k >= 2:
            s = [(x - c) % P for x, c in zip(s, h.ark1[rr])]
        if k >= 1:
            s = [pow(x, INV7, P) for x in inv_mds(s)]          # undo MDS, then x^7
        k = 4
    return s


# ---- sponges and merges (alg_hash.cuh, rpjive.cuh) ----
def hash_elements(hid, elems, log=None):
    e = list(elems)
    if hid == RP64:    # state[0] = length, rate 8, no padding
        s = [0] * 12
        s[0] = len(e) % P
        i = 0
        for x in e:
            s[4 + i] = add(s[4 + i], x, log, "absorb")
            i += 1
            if i == 8:
                s, i = permute(hid, s, log), 0
        if i:
            s = permute(hid, s, log)
        return s[4:8]
    s = [0] * 8        # RpJive: capacity[0] = 1 for a partial last block, which is padded 1, 0, ...
    if len(e) % 4:
        s[0] = 1
    i = 0
    for x in e:
        s[4 + i] = add(s[4 + i], x, log, "absorb")
        i += 1
        if i == 4:
            s, i = permute(hid, s, log), 0
    if i:
        s[4 + i] = 1
        for q in range(i + 1, 4):
            s[4 + q] = 0
        s = permute(hid, s, log)
    return s[4:8]


def _canon(x):
    return x - P if x >= P else x


def jive(init, log=None):
    s = permute(RPJIVE, init, log)
    c = [_canon(x) for x in init]
    return [add(add(c[i], c[4 + i], log, "jive inputs"), add(s[i], s[4 + i], log, "jive outputs"), log, "jive last") for i in range(4)]


def merge(hid, words8, log=None):
    if hid == RP64:
        return permute(hid, [8, 0, 0, 0] + list(words8), log)[4:8]
    return jive(list(words8), log)


def merge_with_int(hid, seed4, value, log=None):
    if hid == RP64:
        s = [0] * 12
        s[4:8] = seed4
        if value < P:
            s[8], s[0] = value, 5
        else:
            s[8], s[9], s[0] = value - P, 1, 6
        return permute(hid, s, log)[4:8]
    s = list(seed4) + [0] * 4
    if value < P:
        s[4], s[7] = value, 5
    else:
        s[4], s[5], s[7] = value - P, 1, 6
    return jive(s, log)


# ---- edge catalogue and targeting ----
SBOX_INPUTS = [0, 1, 2, P - 1, P - 2, 2**32 - 1, 2**32, 2**32 + 1, P - 2**32, 2**63]


P_MINUS_1_FACTORS = ((2, 32), (3, 1), (5, 1), (17, 1), (257, 1), (65537, 1))


@functools.lru_cache(maxsize=None)
def _dlog_table(q):
    """the discrete logs of the order-q subgroup, to its generator 7^((p - 1) / q)"""
    gq = pow(7, (P - 1) // q, P)
    return {pow(gq, j, P): j for j in range(q)}


def dlog7(v):
    """L with 7^L = v (mod p), by Pohlig-Hellman over p - 1 = 2^32 3 5 17 257 65537 (7 generates the multiplicative group)"""
    rem, mod = 0, 1
    for q, k in P_MINUS_1_FACTORS:
        n = q ** k
        g = pow(7, (P - 1) // n, P)                    # order q^k
        h = pow(v, (P - 1) // n, P)
        table = _dlog_table(q)
        x = 0
        for i in range(k):                             # the base-q digits of L mod q^k
            t = pow(h * pow(g, (n - x) % n, P) % P, q ** (k - 1 - i), P)
            x += table[t] * q ** i
        # CRT: L = rem (mod mod), L = x (mod n)
        rem += mod * ((x - rem) * pow(mod, -1, n) % n)
        mod *= n
    assert pow(7, rem, P) == v % P
    return rem


def roots(e, v, limit=4):
    """up to `limit` x with x^e = v (mod p), by the discrete log to the generator 7"""
    from math import gcd
    if v % P == 0:
        return [0]
    L = dlog7(v % P)
    g = gcd(e, P - 1)
    if L % g:
        return []
    q = (P - 1) // g
    y0 = (L // g) * pow(e // g, -1, q) % q
    return [pow(7, y0 + k * q, P) for k in range(min(g, limit))]


SLOT_CLASSES = ("weak word >= p", "word low half 0", "word high half 0")


def _word_classes(w):
    return [c for c, hit in zip(SLOT_CLASSES, (w >= P, w & EPS == 0, w >> 32 == 0)) if hit]


def _why_not(slot, e, cls, cand):
    """what each candidate value gives at a slot whose value is x^e: no preimage, or preimages whose words miss the class"""
    from math import gcd
    g = gcd(e, P - 1)
    parts = []
    for v in cand:
        if cls == "word low half 0" and v & EPS:
            continue
        xs = roots(e, v)
        if not xs:
            parts.append(f"{v:#x} is not a {g}-th power")
        else:
            ws = []
            for x in xs:
                words = []
                (exp7 if slot.startswith("exp7") else inv7)(x, None, words)
                ws.append(dict(words)[slot])
            parts.append(f"{v:#x} comes out as " + "/".join(f"{w:#x}" for w in sorted(set(ws))))
    return f"{slot} = x^{e} (gcd with p - 1: {g}); " + "; ".join(parts)


@functools.lru_cache(maxsize=None)
def slot_targets(per_class=2):
    """S-box inputs x that put a product slot's word at an edge: a value below 2^32 - 1 whose weak word is v + p >= p, or a
    word with a zero low or high half (the next product's operand). Returns ({(slot, class): [x, ...]}, {(slot, class):
    reason}) for the classes reached and those no candidate reached."""
    found, missing = {}, {}
    cand = [1, 2, 3, 5, 7, 2**31, 2**32 - 2, 2**32, 3 * 2**32, 2**40]
    for slot, e in SLOT_EXPONENTS.items():
        for v in cand:
            for x in roots(e, v):
                words = []
                (exp7 if slot.startswith("exp7") else inv7)(x, None, words)
                for c in _word_classes(dict(words)[slot]):
                    if len(found.setdefault((slot, c), [])) < per_class:
                        found[(slot, c)].append(x)
        for c in SLOT_CLASSES:
            if not found.get((slot, c)):
                found.pop((slot, c), None)
                missing[(slot, c)] = _why_not(slot, e % (P - 1), c, cand)
    return found, missing


def _fill(rng, w, vals, at=0):
    s = [int(v) for v in rng.integers(0, P, w, dtype="uint64")]
    for k, v in enumerate(vals):
        s[(at + k) % w] = v
    return s


def targeted_states(hid, rng):
    """(label, permutation input) pairs that put catalogue values at every step boundary of every round: S-box inputs, the
    product slots' edge words (round 0), MDS outputs 0, 1, p - 1 and small, and round-constant sums p - 1, p, p + 1 (the
    last round's included: those sums become digest words)."""
    h = HASHERS[hid]
    w = h.w
    out = []
    small = [0, 1, P - 1, 2, 3, 2**32 - 1]
    found, _ = slot_targets()
    exp_x = sorted({x for (s, _), xs in found.items() if s.startswith("exp7") for x in xs})
    inv_x = sorted({x for (s, _), xs in found.items() if s.startswith("inv") for x in xs})
    for r in range(7):
        for k in range(0, len(SBOX_INPUTS), w):
            out.append((f"r{r} sbox in catalogue", backward(hid, r, "sbox in", _fill(rng, w, SBOX_INPUTS[k:k + w]))))
            out.append((f"r{r} inv in catalogue", backward(hid, r, "inv in", _fill(rng, w, SBOX_INPUTS[k:k + w]))))
        for b in ("mds1 out", "mds2 out"):
            out.append((f"r{r} {b} small", backward(hid, r, b, _fill(rng, w, small, r))))
        for name, off in (("p - 1", -1), ("p", 0), ("p + 1", 1)):
            out.append((f"r{r} ark1 sum {name}", backward(hid, r, "mds1 out", [(P + off - c) % P for c in h.ark1[r]])))
            out.append((f"r{r} ark2 sum {name}", backward(hid, r, "mds2 out", [(P + off - c) % P for c in h.ark2[r]])))
        out.append((f"r{r} ark2 sum wraps", backward(hid, r, "mds2 out", [P - 1] * w)))
    for xs, b in ((exp_x, "sbox in"), (inv_x, "inv in")):
        for k in range(0, len(xs), w):
            out.append((f"r0 {b} product slots", backward(hid, 0, b, _fill(rng, w, xs[k:k + w]))))
    return out


def round0_rows(hid, rng, width):
    """rows of `width` elements (one sponge block: width <= rate) whose permutation sees catalogue and product-slot edge values
    as round-0 S-box inputs, and catalogue values as eight round-0 MDS outputs (the 8 x 8 system in x^7, capacity fixed)"""
    h = HASHERS[hid]
    rate = 8 if hid == RP64 else 4
    assert width <= rate
    found, _ = slot_targets()
    vals = SBOX_INPUTS + sorted({x for (s, _), xs in found.items() if s.startswith("exp7") for x in xs})
    rows = [[vals[(k + j) % len(vals)] for j in range(width)] for k in range(0, len(vals), width)]
    if width == rate:   # MDS1 outputs: capacity (length or padding flag) fixed, rate words = solution of the 8 x 8 system
        cap = [width % P, 0, 0, 0] if hid == RP64 else [0, 0, 0, 0]
        free = list(range(4, h.w))
        rows_out = list(range(h.w))[:len(free)]
        for k in range(0, len(SBOX_INPUTS), len(free)):
            want = _fill(rng, len(free), SBOX_INPUTS[k:k + len(free)])
            c7 = [pow(c, 7, P) for c in cap]
            rhs = [(t - sum(h.mat[i][j] * c7[j] for j in range(4))) % P for i, t in zip(rows_out, want)]
            y = solve_mod_p([[h.mat[i][j] for j in free] for i in rows_out], rhs)
            rows.append([pow(v, INV7, P) for v in y])
    return rows


# An RpJive merge input whose last Jive add (x + y, x = in[i] + in[4 + i], y = out[i] + out[4 + i]) lands in [p, 2^64) at
# lane 2. Both operands come from this one input, so backward targeting cannot aim at it; tools/find_jive_edge.cu found it by
# searching word 0 on a GPU (about 2^29 tries).
JIVE_LAST_ADD_INPUT = [787694347, 4354685564936845354, 15755400384260043839, 8709371129873690708, 1663341875487337577,
                       13064056694810536062, 6018027440424182931, 17418742259747381416]


def jive_edge_states(rng):
    """RpJive merge inputs (8 words) that put each of the Jive sum's three adds at p and in [p, 2^64): the input pair through
    the input words, the output pair backward from the round-6 output, the last add through JIVE_LAST_ADD_INPUT"""
    out = []
    for a, b in ((P - 1, 1), (P - 1, 2**32 - 2), (P - 2**31, 2**31 + 1), (P - 1, P - 1)):
        s = _fill(rng, 8, [])
        s[0], s[4] = a, b
        s[3], s[7] = b, a
        out.append(("jive inputs", s))
        t = _fill(rng, 8, [])
        t[1], t[5] = a, b
        t[2], t[6] = b, a
        out.append(("jive outputs", backward(RPJIVE, 6, "round out", t)))
    out.append(("jive last", list(JIVE_LAST_ADD_INPUT)))
    return out


def two_block_rows(hid, rng, count=4):
    """rows of two sponge blocks whose second block's absorb sums are p - 1 and p: x = target - s after the first block"""
    rate = 8 if hid == RP64 else 4
    rows = []
    for k in range(count):
        first = [int(v) for v in rng.integers(0, P, rate, dtype="uint64")]
        s = permute(hid, ([2 * rate, 0, 0, 0] if hid == RP64 else [0, 0, 0, 0]) + first)
        rows.append(first + [((P - 1 if (k + i) % 2 else P) - s[4 + i]) % P for i in range(rate)])
    return rows
