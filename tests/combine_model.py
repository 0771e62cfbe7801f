"""An exact model of the delayed-reduction accumulator (GlAcc in gl64.cuh) and of the stages that combine committed values:
the out-of-domain evaluation (ood_partial_kernel), the DEEP sum and division (deep_sum_kernel, deep_div_kernel, syn_div_*)
and the FRI fold (fri_fold_kernel), with inputs aimed at the edges of their arithmetic.

  * `acc_mad` restates the PTX word by word: the odd column x0 y1 + x1 y0 with its carry m2, the even columns x0 y0 and
    x1 y1 added into w0..w3 with the carry into w4, then the odd column added at w1 with its carries into w4. It records
    m2 = 1, a carry out of w3 from either add, and a carry that ripples through w1..w3 when they are all ones.
  * `acc_reduce` restates `gl_reduce128` on (w1:w0, w3:w2) as its PTX runs, then `gl_sub(t, w4 << 32)`, and records the
    classes of REDUCE_CLASSES.
  * Aiming: a kernel's accumulator is a dot product with known multipliers, so a target 160-bit sum A can be reached.
    For free multipliers A = q (p-1)^2 + x (p-1) + r0 takes q terms (p-1, p-1), then (x, p-1) and (r0, 1) (`aim_terms`);
    for the OOD thread the multipliers are the powers z^r of its 64 rows: rows r >= 2 are filled greedily, then
    A - rest = c1 z + c0 (`ood_aim`). `reduce_targets` lists sums A aimed at every class that a kernel's largest sum allows.
  * The fold: `fold_inputs` puts `ntt_model.pair_edges` operands at the butterflies of a chosen layer of mini_dft<LOGNF>,
    running the earlier layers backwards (butterfly inverse and division by the power-of-two twiddle).
  * Reference arithmetic in Python integers for the extension fields (x^2 - x + 2, x^3 - x - 1) and the serial and
    vectorised synthetic division (polynom/mod.rs:498-505).
"""
import random

import numpy as np

import ntt_model as NM

P = NM.P
M32 = 2**32 - 1
M64 = 2**64 - 1
M128 = 2**128 - 1
EPS = M32

MAD_CLASSES = ("m2 = 1", "even carry out of w3", "odd carry out of w3", "odd carry ripples through all-ones w1..w3")
REDUCE_CLASSES = ("hh = 2^32 - 1", "lo < hh", "U carries out", "r + (2^32 - 1) carries", "result 0", "result p - 1", "w4 = 0",
                  "w4 at kernel max", "t < w4 << 32", "t = w4 << 32")
CLASSES = MAD_CLASSES + REDUCE_CLASSES


class Log:
    """classes reached, keyed by (kernel, class); `None` records nothing"""

    def __init__(self):
        self.hits = {}

    def add(self, kind, cls):
        self.hits[(kind, cls)] = self.hits.get((kind, cls), 0) + 1


def _hit(log, kind, cls):
    if log is not None:
        log.add(kind, cls)


# ---- the accumulator ----
def acc_mad(w, x, y, log=None, kind="dot"):
    """one acc_mad(w, x, y) on the words w = [w0..w4] (any 64-bit x, y), as the PTX adds them"""
    x0, x1, y0, y1 = x & M32, x >> 32, y & M32, y >> 32
    m = x0 * y1 + x1 * y0
    if m >> 64:
        _hit(log, kind, "m2 = 1")
    low = w[0] | w[1] << 32 | w[2] << 64 | w[3] << 96
    e = low + x0 * y0 + (x1 * y1 << 64)
    if e >> 128:
        _hit(log, kind, "even carry out of w3")
    w4 = (w[4] + (e >> 128)) & M32
    e &= M128
    if (e >> 32) & (2**96 - 1) == 2**96 - 1 and m:
        _hit(log, kind, "odd carry ripples through all-ones w1..w3")
    o = e + (m << 32)
    if o >> 128:
        _hit(log, kind, "odd carry out of w3")
    w4 = (w4 + (o >> 128)) & M32
    o &= M128
    return [o & M32, (o >> 32) & M32, (o >> 64) & M32, (o >> 96) & M32, w4]


def acc_words(A):
    return [(A >> (32 * i)) & M32 for i in range(5)]


def acc_value(w):
    return sum(v << (32 * i) for i, v in enumerate(w))


def dot(xs, ys, log=None, kind="dot"):
    w = [0] * 5
    for x, y in zip(xs, ys):
        w = acc_mad(w, x, y, log, kind)
    return w


def acc_reduce(w, w4_max=None, log=None, kind="dot"):
    """gl_reduce128((w1:w0), (w3:w2)) step by step, then gl_sub(t, w4 << 32); canonical result"""
    lo, hi, w4 = w[0] | w[1] << 32, w[2] | w[3] << 32, w[4]
    hh, hl = hi >> 32, hi & M32
    if hh == M32:
        _hit(log, kind, "hh = 2^32 - 1")
    t = (lo - hh) & M64
    if lo < hh:
        _hit(log, kind, "lo < hh")
        t = (t - EPS) & M64            # + p: cannot borrow again
    U = t + hl * EPS
    k1, r = U >> 64, U & M64
    k2 = (r + EPS) >> 64
    if k1:
        _hit(log, kind, "U carries out")
    if k2:
        _hit(log, kind, "r + (2^32 - 1) carries")
    assert not (k1 and k2)
    r = (r + (k1 + k2) * EPS) & M64
    assert r < P and r == (lo + (hi << 64)) % P
    s = w4 << 32
    if w4 == 0:
        _hit(log, kind, "w4 = 0")
    if w4_max is not None and w4 == w4_max:
        _hit(log, kind, "w4 at kernel max")
    if r < s:
        _hit(log, kind, "t < w4 << 32")
    elif w4 and r == s:
        _hit(log, kind, "t = w4 << 32")
    d = (r - s) & M64
    if r < s:
        d = (d - EPS) & M64
    if d == 0:
        _hit(log, kind, "result 0")
    if d == P - 1:
        _hit(log, kind, "result p - 1")
    return d


# ---- aiming ----
def aim_terms(A, k, rng=None):
    """k canonical terms (x_j, y_j) with sum x_j y_j = A exactly, in the order q x (p-1, p-1), (x, p-1), (r0, 1), then
    zero products; A < (k - 1) (p - 1)^2 (k >= 2)"""
    q, R = divmod(A, (P - 1) ** 2)
    x, r0 = divmod(R, P - 1)
    terms = [(P - 1, P - 1)] * q + [(x, P - 1), (r0, 1)]
    assert len(terms) <= k, (A, k)
    rng = rng or random.Random(0)
    while len(terms) < k:
        v = rng.randrange(P)
        terms.append((0, v) if len(terms) % 2 else (v, 0))
    return terms


def reduce_targets(amax, rng, w4_floor=0):
    """(class, A) with w4_floor 2^128 <= A <= amax aimed at each REDUCE_CLASSES class that such an A can reach"""
    out = []
    w4max = amax >> 128

    def add(cls, A):
        if w4_floor << 128 <= A <= amax:
            out.append((cls, A))

    lo_w4 = max(w4_floor, 0)
    for w4 in sorted({lo_w4, min(lo_w4 + 1, w4max), (lo_w4 + w4max) // 2, w4max}):
        base = w4 << 128
        add("hh = 2^32 - 1", base | M32 << 96 | rng.randrange(2**96))
        hh = rng.randrange(1, 2**32)
        add("lo < hh", base | hh << 96 | rng.randrange(2**32) << 64 | rng.randrange(hh))
        add("U carries out", base | M32 << 64 | (M64 - rng.randrange(2**32)))
        add("r + (2^32 - 1) carries", base | rng.randrange(P, 2**64))
        add("result 0", base + (-base) % P + P * rng.randrange(max(1, (2**128 - P) // P)))
        add("result p - 1", base + (P - 1 - base) % P + P * rng.randrange(max(1, (2**128 - 2 * P) // P)))
        if w4:
            j = rng.randrange(max(1, 2**128 // P - 1))
            add("t < w4 << 32", base | (P * j + rng.randrange(w4 << 32)))
            add("t = w4 << 32", base | (P * j + (w4 << 32)))
    add("w4 = 0", rng.randrange(min(amax, M128) + 1))
    add("w4 at kernel max", amax)
    add("w4 at kernel max", amax - rng.randrange(min(amax - (w4max << 128), 2**100) + 1))
    return out


def dot_rows(k, rng):
    """dot products of k canonical terms aimed at every class k terms can reach: (label, xs, ys)"""
    rows = [("all p - 1", [P - 1] * k, [P - 1] * k)]
    if k >= 2:
        amax = (k - 1) * (P - 1) ** 2 - 1
        for cls, A in reduce_targets(amax, rng):
            if cls == "w4 at kernel max":   # k - 1, reached by the all-(p-1) row; aimed sums stop at w4 = k - 2
                continue
            t = aim_terms(A, k, rng)
            rows.append((cls, [a for a, _ in t], [b for _, b in t]))
        if k >= 3:   # prefixes that leave w1..w3 all ones after the last term's even columns, or that carry out of w3 there
            last = (P - 2, P - 2)        # x0 y1 + x1 y0 >= 2^64: m2 = 1
            x0, x1 = last[0] & M32, last[0] >> 32
            even = x0 * x0 + (x1 * x1 << 64)
            for pre in (2**128 - 2**32 + rng.randrange(2**32) - even, 2**128 - 1):
                t = aim_terms(pre, k - 1, rng) + [last]
                rows.append(("ripple", [a for a, _ in t], [b for _, b in t]))
    # single products of words with zero or all-ones halves
    words = [0, 1, P - 1, P - 2, M32, M32 << 32 & M64, 2**63, rng.randrange(P)]
    for i in range(len(words)):
        xs = [words[(i + j) % len(words)] for j in range(k)]
        ys = [words[(3 * i + 5 * j + 1) % len(words)] for j in range(k)]
        rows.append(("words", xs, ys))
    return rows


def ood_aim(mult, A, rng):
    """coefficients c_0..c_63 (canonical) of one OOD thread with sum_r mult_r c_r = A exactly for the multipliers
    mult_r = component d of z^r (mult_0 = 1 for d = 0, 0 otherwise), or None when A is out of reach"""
    c = [0] * len(mult)
    rest = 0
    for r in range(len(mult) - 1, 1, -1):
        if mult[r]:
            c[r] = min(P - 1, (A - rest) // mult[r])
            rest += c[r] * mult[r]
    T = A - rest
    if mult[1]:
        c[1] = min(P - 1, T // mult[1])
        T -= c[1] * mult[1]
    if mult[0] == 1:   # z^0 = 1: component 0 only
        c[0], T = T, 0
    if T or c[0] >= P:
        return None
    return c


def ood_max(mult):
    return sum((P - 1) * m for m in mult)


def ood_thread_rows(mult, rng, w4_floor=0):
    """(class, 64 coefficients) aimed at the reduce classes for one OOD accumulator with multipliers mult"""
    out = [("all p - 1", [P - 1] * len(mult))]
    for cls, A in reduce_targets(ood_max(mult), rng, w4_floor):
        c = ood_aim(mult, A, rng)
        if c is not None:
            out.append((cls, c))
    return out


def deep_coeffs(c, d, comp):
    """DEEP coefficients of c main columns aiming component `comp`: p - 1 on columns < c - 1, 1 on the last; zero elsewhere"""
    dc = np.zeros((c, d), dtype=np.uint64)
    dc[:c - 1, comp] = P - 1
    dc[c - 1, comp] = 1
    return dc


def deep_rows(c, rng):
    """(class, row of c main-column values) whose dot product with deep_coeffs reaches the class"""
    assert c >= 2
    out = [("all p - 1", [P - 1] * c)]
    for cls, A in reduce_targets((c - 1) * (P - 1) ** 2 - 1, rng):
        q, R = divmod(A, (P - 1) ** 2)       # q (p-1)^2 + x (p-1) + r0 with q <= c - 2
        x, r0 = divmod(R, P - 1)
        out.append((cls, [P - 1] * q + [0] * (c - 2 - q) + [x, r0]))
    return out


def deep_max(c):
    return (c - 1) * (P - 1) ** 2 + (P - 1)


def structured_points(d):
    """out-of-domain points where the OOD, DEEP and scan kernels degenerate: (label, z as d canonical words)"""
    pad = [0] * (d - 1)
    pts = [("0", [0] + pad), ("1", [1] + pad), ("2^11-th root of unity", [NM.root(11)] + pad),
           ("8th root of unity", [NM.root(3)] + pad), ("p - 1", [P - 1] + pad), ("base field", [5] + pad)]
    if d > 1:
        pts += [("all components p - 1", [P - 1] * d), ("0 + u", [0, 1] + pad[1:]), ("extension", [3 + q for q in range(d)])]
    return pts


def ood_mults(z, comp):
    """the multipliers of one OOD thread's accumulator for component comp: component comp of z^r, r < 64"""
    out, zr = [], [1] + [0] * (len(z) - 1)
    for _ in range(64):
        out.append(zr[comp])
        zr = ext_mul(zr, z)
    return out


# ---- Goldilocks extensions on Python integers ----
def ext_mul(a, b):
    d = len(a)
    c = [0] * (2 * d - 1)
    for i in range(d):
        for j in range(d):
            c[i + j] += a[i] * b[j]
    if d == 2:     # x^2 = x - 2
        return [(c[0] - 2 * c[2]) % P, (c[1] + c[2]) % P]
    if d == 3:     # x^3 = x + 1, x^4 = x^2 + x
        return [(c[0] + c[3]) % P, (c[1] + c[3] + c[4]) % P, (c[2] + c[4]) % P]
    return [c[0] % P]


def ext_pow(a, e):
    r = [1] + [0] * (len(a) - 1)
    while e:
        if e & 1:
            r = ext_mul(r, a)
        a = ext_mul(a, a)
        e >>= 1
    return r


def ext_inv(a):
    return ext_pow(a, P ** len(a) - 2) if any(a) else list(a)


def ext_add(a, b):
    return [(u + v) % P for u, v in zip(a, b)]


def ext_sub(a, b):
    return [(u - v) % P for u, v in zip(a, b)]


def horner(coeffs, z):
    """sum_i coeffs_i z^i for base coefficients and an extension point z (Python ints)"""
    acc = [0] * len(z)
    for c in reversed(coeffs):
        acc = ext_mul(acc, z)
        acc[0] = (acc[0] + int(c)) % P
    return acc


# ---- numpy extension arithmetic (elementwise on [n, d] arrays) ----
def np_ext_mul(a, b):
    a, b = np.atleast_2d(a), np.atleast_2d(b)
    d = a.shape[-1]
    c = [None] * (2 * d - 1)
    for i in range(d):
        for j in range(d):
            t = NM.fmul(a[:, i], b[:, j])
            c[i + j] = t if c[i + j] is None else NM.fadd(c[i + j], t)
    if d == 1:
        return c[0][:, None]
    if d == 2:
        return np.stack([NM.fsub(c[0], NM.fadd(c[2], c[2])), NM.fadd(c[1], c[2])], axis=1)
    return np.stack([NM.fadd(c[0], c[3]), NM.fadd(NM.fadd(c[1], c[3]), c[4]), NM.fadd(c[2], c[4])], axis=1)


def host_syn_div(oracle, s, b, ext):
    """syn_div(p, 1, b) of polynom/mod.rs:498-505, serially: q_i = s_(i+1) + b q_(i+1), q_(n-1) = 0."""
    mul = (lambda x, y: oracle.ext_mul(x, y)) if ext > 1 else (lambda x, y: np.array([oracle.mul(int(x[0]), int(y[0]))], dtype=np.uint64))
    q = np.zeros_like(s)
    acc = np.zeros(ext, dtype=np.uint64)
    for i in range(len(s) - 1, 0, -1):
        acc = np.array([(int(u) + int(v)) % P for u, v in zip(s[i], mul(b, acc))], dtype=np.uint64)
        q[i - 1] = acc
    return q


def np_syn_div(s, b):
    """host_syn_div restated as a doubling suffix scan: a_i = sum_(k >= i) s_k b^(k-i) in log2(n) vector steps, q_i = a_(i+1)"""
    a = np.array(s, dtype=np.uint64, copy=True)
    n, d = a.shape
    bd = [int(v) for v in b]
    step = 1
    while step < n:   # window [i, i + step) -> [i, i + 2 step): a_i += b^step a_(i + step)
        t = np_ext_mul(a[step:], np.array([bd], dtype=np.uint64))
        a[:n - step] = np.stack([NM.fadd(a[:n - step, q], t[:, q]) for q in range(d)], axis=1)
        bd = ext_mul(bd, bd)
        step *= 2
    q = np.zeros_like(a)
    q[:-1] = a[1:]
    return q


# ---- the FRI fold's mini-DFT ----
def mini_dft_layers(lognf):
    """the layers of mini_dft<LOGNF>: (butterfly pairs, twiddles (index, K) applied after them)"""
    nf = 1 << lognf
    layers = []
    for lvl in range(lognf):
        B = nf >> lvl
        h = B // 2
        pairs = [(s + q, s + q + h) for s in range(0, nf, B) for q in range(h)]
        tws = [(s + h + q, q * (192 // B)) for s in range(0, nf, B) for q in range(1, h)]
        layers.append((pairs, tws))
    return layers


def mini_dft(x, lognf, observe=None):
    """DIF, in place, bit-reversed output, canonical words (Python ints)"""
    x = list(x)
    for lvl, (pairs, tws) in enumerate(mini_dft_layers(lognf)):
        if observe:
            observe(lvl, [x[i] for i, _ in pairs], [x[j] for _, j in pairs])
        for i, j in pairs:
            x[i], x[j] = (x[i] + x[j]) % P, (x[i] - x[j]) % P
        for i, k in tws:
            x[i] = x[i] * pow(2, k, P) % P
    return x


def mini_dft_input_for(state, lognf, layer):
    """the input that puts `state` at the input of layer `layer` of mini_dft<LOGNF>"""
    x = list(state)
    inv2 = (P + 1) // 2
    for pairs, tws in reversed(mini_dft_layers(lognf)[:layer]):
        for i, k in tws:
            x[i] = x[i] * pow(2, 192 - k, P) % P
        for i, j in pairs:
            x[i], x[j] = (x[i] + x[j]) * inv2 % P, (x[i] - x[j]) * inv2 % P
    return x


def fold_inputs(L, nf, d, rng_np):
    """a layer of L points x d components for wf_fri_fold_dev whose rows put pair_edges operands at the butterflies of
    mini_dft<LOGNF>: row i aims layer i mod LOGNF. Element (i + k m) of the layer is input k of row i (m = L / nf)."""
    lognf = nf.bit_length() - 1
    m = L // nf
    ev = np.zeros((L, d), dtype=np.uint64)
    layers = mini_dft_layers(lognf)
    for i in range(m):
        lvl = i % lognf
        pairs = layers[lvl][0]
        for c in range(d):
            a, b = NM.pair_edges((len(pairs),), rng_np)
            st = [0] * nf
            for (pi, pj), u, v in zip(pairs, a, b):
                st[pi], st[pj] = int(u), int(v)
            x = mini_dft_input_for(st, lognf, lvl)
            for k in range(nf):
                ev[i + k * m, c] = x[k]
    return ev


# ---- the FibSmall constraint kernel (fib_constraints_kernel) ----
def fib_mult(m):
    """the coefficients of one FibSmall accumulator in an aimed call: p - 1 on its first m - 1 terms, 1 on the last"""
    return [P - 1] * (m - 1) + [1]


def fib_k0(k):
    """K0 of an aimed B0 call, sum_j (b0a_j + b0b_j) (j + 1) mod p, for the coefficients fib_mult(2k)"""
    mult = fib_mult(2 * k)
    return sum((mult[2 * j] + mult[2 * j + 1]) * (j + 1) for j in range(k)) % P


def _row_for(m, A):
    q, R = divmod(A, (P - 1) ** 2)       # q (p-1)^2 + x (p-1) + r0 with q <= m - 2
    x, r0 = divmod(R, P - 1)
    return [P - 1] * q + [0] * (m - 2 - q) + [x, r0]


def fib_aims(k, rng):
    """(accumulator, class, term values) for the three accumulators of one FibSmall x k row: T over the 2k values t0_j, t1_j
    (interleaved), B0 over cur.x_j, cur.y_j (interleaved), B1 over the k values cur.y_j, each against fib_mult of its length.
    B0 also aims acc_reduce(a0) = K0 (B0 = 0) and acc_reduce(a0) < K0 (a borrow in gl_sub(., K0))."""
    out = []
    for acc, m in (("T", 2 * k), ("B0", 2 * k), ("B1", k)):
        if m < 2:
            continue
        out += [(acc, cls, row) for cls, row in deep_rows(m, rng)]
    if k >= 2:
        amax, K0 = (2 * k - 1) * (P - 1) ** 2 - 1, fib_k0(k)
        A = K0 + P * rng.randrange(max(1, (amax - K0) // P))
        out.append(("B0", "reduce(a0) = K0", _row_for(2 * k, A)))
        if K0:
            A = P * rng.randrange(max(1, amax // P - 1)) + rng.randrange(K0)
            out.append(("B0", "reduce(a0) < K0", _row_for(2 * k, A)))
    return out
