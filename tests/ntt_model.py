"""An exact model of the transform network the device runs for its NTT, iNTT and LDE, and inputs that drive it to the
reduction edges of its butterflies, shifts and products.

The model restates the schedule of `run_ntt` / `run_lde` (csrc/capi.cu: one pass up to 2^11 points, the four-step R x C
split up to 2^22, three passes above), the sub-transform plans (ntt2.cu `Plan<LOGS>` for 2^6 .. 2^11, ntt.cu's radix-8
`dif_round` chain below 2^6), every `mini_dft<r>` of minidft.cuh layer by layer (DIF `bf2` layers, the in-round
`gl_mul_2exp<K>` at the same positions, bit-reversed output), the inter-round twiddles of `ntt2_build_tw_kernel`, the coset
pre-scale, the post twiddle `w_M^(+-(j a_mul + (batch0 + b) b_mul) c) ctab[c] cconst`, the write-back scale and the
inverse's index map j -> (S - j) mod S. Every device operation returns canonical words, so the values inside the network
are field elements and the model computes them with numpy uint64 arithmetic mod p.

Two uses:
  * forward: `Network.forward(x, observe)` returns the output and hands every step's input state and operands to
    `observe(label, state, operands)`;
  * targeting: `Network.target(pass, steps, rng)` returns the transform input that puts catalogue edge operands
    (`pair_edges`, `shift_catalogue`, `product_edges`) at the chosen step of every chosen sub-transform, by running the
    earlier steps backwards exactly (butterfly inverse, division by the shift, twiddle, pre-scale or post factor, and the
    whole of every earlier pass).
"""
import functools

import numpy as np

P = 0xFFFFFFFF00000001
_P = np.uint64(P)
_M32 = np.uint64(0xFFFFFFFF)
_32 = np.uint64(32)
_INV2 = np.uint64((P + 1) // 2)
ROOT_2_32 = 7277203076849721926  # TWO_ADIC_ROOT_OF_UNITY
GENERATOR = 7
MAX_LOGS = 11


def root(log_n):
    return pow(ROOT_2_32, 1 << (32 - log_n), P)


# ---- field arithmetic on uint64 arrays (32-bit limbs) ----
def fmul(a, b):
    with np.errstate(over="ignore"):
        a = np.asarray(a, dtype=np.uint64)
        b = np.asarray(b, dtype=np.uint64)
        a0, a1, b0, b1 = a & _M32, a >> _32, b & _M32, b >> _32
        ll, lh, hl, hh = a0 * b0, a0 * b1, a1 * b0, a1 * b1
        t = (ll >> _32) + (lh & _M32) + (hl & _M32)
        lo = (ll & _M32) | (t << _32)
        t = (t >> _32) + (lh >> _32) + (hl >> _32) + (hh & _M32)
        c2, c3 = t & _M32, (t >> _32) + (hh >> _32)
        # lo + 2^64 c2 + 2^96 c3 = lo + (2^32 - 1) c2 - c3 (mod p)
        x = lo - c3
        x = np.where(lo < c3, x + _P, x)
        x = np.where(x >= _P, x - _P, x)
        y = c2 * _M32
        s = x + y
        return np.where((s < x) | (s >= _P), s - _P, s)


def fadd(a, b):
    with np.errstate(over="ignore"):
        s = a + b
        return np.where((s < a) | (s >= _P), s - _P, s)


def fsub(a, b):
    with np.errstate(over="ignore"):
        d = a - b
        return np.where(a < b, d + _P, d)


def powers(base, count):
    """base^i for i < count"""
    out = np.ones(1, dtype=np.uint64)
    while out.size < count:
        out = np.concatenate([out, fmul(out, np.uint64(pow(base, out.size, P)))])
    return out[:count]


@functools.lru_cache(maxsize=None)
def _root_tables(log_m):
    h = log_m // 2
    w = root(log_m) if log_m else 1
    return powers(pow(w, 1 << h, P), 1 << (log_m - h)), powers(w, 1 << h), h


def root_pow(e, log_m, negate=False):
    """w_M^(+-e) for an integer array e (any size, reduced mod M)"""
    e = np.asarray(e, dtype=np.uint64) & np.uint64((1 << log_m) - 1)
    if negate:
        e = (np.uint64(1 << log_m) - e) & np.uint64((1 << log_m) - 1)
    hi, lo, h = _root_tables(log_m)
    return fmul(hi[e >> np.uint64(h)], lo[e & np.uint64((1 << h) - 1)])


def brev(v, bits):
    v = np.asarray(v, dtype=np.int64)
    r = np.zeros_like(v)
    for i in range(bits):
        r |= ((v >> i) & 1) << (bits - 1 - i)
    return r


def radices(log_s):
    """round radices (log2) of a 2^log_s-point sub-transform: ntt2.cu Plan<LOGS> from 2^6, ntt.cu's radix-8 chain below"""
    if log_s >= 6:
        r0 = 4 if log_s == 8 else 3
        r1 = 4 if log_s in (11, 8, 7) else 3
        return [r0, r1] + ([log_s - r0 - r1] if log_s >= 9 else [])
    r = [3] * (log_s // 3)
    return r + ([log_s % 3] if log_s % 3 else [])


def split_log(log_n):
    if log_n <= MAX_LOGS:
        return 0, log_n
    r = min((log_n + 1) // 2, MAX_LOGS)
    return r, log_n - r


def split3(log_n):
    lr = (log_n + 2) // 3
    lr2, lc2 = split_log(log_n - lr)
    return lr, lr2, lc2


# ---- edge catalogues ----
PAIR_CLASSES = ("sum=p-1", "sum=p", "sum=p+1", "sum in (p+1,2^64)", "sum=2^64", "sum>2^64", "a=b", "a=b+1", "a=b-1",
                "a=0", "b=0", "a=p-1", "b=p-1", "b<=a<2^32")
SHIFT_RESULTS = (0, 1, 2**32 - 2, 2**32 - 1, 2**32, P - 2**32, P - 1)
SHIFT_CLASSES = tuple("x*2^K=%#x" % c for c in SHIFT_RESULTS) + ("low word 0", "y2=0", "y1=2^32-1")
PRODUCT_CLASSES = ("x*w=0", "0<x*w<2^32-1", "x*w=p-1")


def _rand(rng, shape, lo=0, hi=P):
    return rng.integers(lo, hi, size=shape, dtype=np.uint64, endpoint=False)


def pair_edges(shape, rng, d=None):
    """butterfly operands (a, b): each pair in one class of PAIR_CLASSES, or (one class in 15) with a - b = d"""
    cls = rng.integers(0, 15, size=shape)
    a, b = _rand(rng, shape), _rand(rng, shape)
    raw = _rand(rng, shape, 0, 2**64 - 1)
    with np.errstate(over="ignore"):
        forms = []
        x = _rand(rng, shape)
        forms.append((x, _P - np.uint64(1) - x))                                   # a + b = p - 1
        x = _rand(rng, shape, 1)
        forms.append((x, _P - x))                                                  # p
        x = _rand(rng, shape, 2)
        forms.append((x, _P - x + np.uint64(1)))                                   # p + 1
        x = _rand(rng, shape, 2**32 + 2)
        forms.append((x, _P - x + np.uint64(2) + (raw % np.uint64(2**32 - 3))))    # (p + 1, 2^64)
        x = _rand(rng, shape, 2**32)
        forms.append((x, np.uint64(0) - x))                                        # 2^64
        x = _rand(rng, shape, 2**32 + 1)
        forms.append((x, np.uint64(0) - x + np.uint64(1) + raw % (x - np.uint64(2**32))))  # (2^64, 2p)
        x = _rand(rng, shape)
        forms.append((x, x))                                                       # a = b
        x = _rand(rng, shape, 0, P - 1)
        forms.append((x + np.uint64(1), x))                                        # a = b + 1
        forms.append((x, x + np.uint64(1)))                                        # a = b - 1
        zero, top = np.zeros(shape, np.uint64), np.full(shape, P - 1, np.uint64)
        forms += [(zero, b), (a, zero), (top, b), (a, top)]
        x = _rand(rng, shape, 0, 2**32)
        forms.append((x, raw % (x + np.uint64(1))))                                # small a, b <= a: a - b needs no p
        forms.append((fadd(b, d if d is not None else a), b))                      # a - b = d
    for k, (fa, fb) in enumerate(forms):
        m = cls == k
        a[m], b[m] = fa[m], fb[m]
    return a, b


@functools.lru_cache(maxsize=None)
def shift_catalogue(k):
    """operands x of x * 2^K: results in SHIFT_RESULTS, a zero low word, y2 = 0 and y1 = 2^32 - 1 (gl_shl_dev's words
    y = x << (K mod 32))"""
    inv = pow(2, 192 - k, P)
    vals = [c * inv % P for c in SHIFT_RESULTS]
    rng = np.random.default_rng(1000 + k)
    r = k & 31
    vals += [int(h) << 32 for h in rng.integers(0, 2**32, 6)]
    vals += [int(v) for v in rng.integers(0, min(1 << (64 - r), P), 6, dtype=np.uint64)]
    for _ in range(6 if r else 0):          # r = 0: y1 = x1, and p - 1 (above) is the one such operand
        y2 = int(rng.integers(0, max((1 << r) - 1, 1)))
        y0 = int(rng.integers(0, 2**32)) & ~((1 << r) - 1)
        vals.append(((y2 << 64) | (0xFFFFFFFF << 32) | y0) >> r)
    assert all(v < P for v in vals)
    return np.array(vals, dtype=np.uint64)


def shift_edges(k, shape, rng):
    cat = shift_catalogue(k)
    return cat[rng.integers(0, cat.size, size=shape)]


def product_edges(shape, rng):
    """results c of a product x * w: 0, below 2^32 - 1 (the unreduced result is c + p), p - 1"""
    cls = rng.integers(0, 3, size=shape)
    c = _rand(rng, shape, 1, 2**32 - 1)
    c[cls == 0] = 0
    c[cls == 2] = P - 1
    return c


def classify_pairs(a, b):
    with np.errstate(over="ignore"):
        s = a + b
    carry = s < a
    tests = (~carry & (s == _P - np.uint64(1)), ~carry & (s == _P), ~carry & (s == _P + np.uint64(1)),
             ~carry & (s > _P + np.uint64(1)), carry & (s == 0), carry & (s > 0), a == b, a == b + np.uint64(1),
             a + np.uint64(1) == b, a == 0, b == 0, a == _P - np.uint64(1), b == _P - np.uint64(1),
             (a < np.uint64(2**32)) & (b <= a))
    return {c for c, t in zip(PAIR_CLASSES, tests) if t.any()}


def classify_shifts(x, k):
    x, k = np.broadcast_arrays(x, k)
    out = set()
    for kk in np.unique(k):
        xs = x[k == kk]
        c = fmul(xs, np.uint64(pow(2, int(kk), P)))
        r = int(kk) & 31
        x0, x1 = xs & _M32, xs >> _32
        y1 = ((x1 << np.uint64(r)) | (x0 >> np.uint64(32 - r))) & _M32 if r else x1
        y2 = x1 >> np.uint64(32 - r) if r else np.zeros_like(x1)
        tests = [c == np.uint64(v) for v in SHIFT_RESULTS] + [x0 == 0, y2 == 0, y1 == _M32]
        out |= {cl for cl, t in zip(SHIFT_CLASSES, tests) if t.any()}
    return out


def classify_products(x, w):
    c = fmul(x, w)
    tests = (c == 0, (c > 0) & (c < _M32), c == _P - np.uint64(1))
    return {cl for cl, t in zip(PRODUCT_CLASSES, tests) if t.any()}


def classify(kind, operands):
    return {"bf": classify_pairs, "shift": classify_shifts}.get(kind, classify_products)(*operands)


# ---- layouts: a pass reads its sub-transforms from, and writes them to, a (nb, ncols, n) array ----
def to_tiles(x, gdims, perm):
    lead = x.shape[:2]
    t = x.reshape(lead + tuple(gdims)).transpose((0, 1) + tuple(2 + p for p in perm))
    return t.reshape(lead + (-1, gdims[perm[-1]]))


def from_tiles(t, gdims, perm):
    lead = t.shape[:2]
    tdims = tuple(gdims[p] for p in perm)
    back = tuple(int(i) for i in np.argsort(perm))
    return t.reshape(lead + tdims).transpose((0, 1) + tuple(2 + p for p in back)).reshape(lead + (-1,))


class Pass:
    """One pass kernel launch: a batch of 2^log_s-point sub-transforms, tiles (nb, ncols, nsub, S).

    pre(ks) -> (len(ks), 1, 1, S) input scale or None; post(ks) -> (len(ks), 1, nsub, S) factor by output index, or None;
    scale: the write-back constant when there is no post twiddle."""

    def __init__(self, name, log_s, layout_in, layout_out, inverse=False, pre=None, post=None, scale=1):
        self.name, self.log_s, self.inverse = name, log_s, inverse
        self.layout_in, self.layout_out = layout_in, layout_out
        self.pre, self.post, self.scale = pre, post, scale
        S = 1 << log_s
        jf = (S - np.arange(S)) & (S - 1) if inverse else np.arange(S)
        self.src = brev(jf, log_s)                       # output j reads tile position brev(jf(j))
        self.rounds = []
        st = 0
        for r in radices(log_s):
            self.rounds.append((r, st, log_s - st - r))
            st += r
        steps = [("pre", None, None)] if pre is not None else []
        for ri, (r, _, _) in enumerate(self.rounds):
            for l in range(r):
                steps.append(("bf", ri, l))
                if l < r - 1:
                    steps.append(("shift", ri, l))
            if ri < len(self.rounds) - 1:
                steps.append(("tw", ri, None))
        steps.append(("post" if post is not None else ("scale" if scale != 1 else "out"), None, None))
        self.steps = steps

    def targets(self):
        """indices of the steps that carry an operation"""
        return [i for i, s in enumerate(self.steps) if s[0] != "out"]

    # ---- per-step helpers ----
    def _pairs_view(self, x, ri, l):
        r, st, ls = self.rounds[ri]
        return x.reshape(x.shape[:-1] + (1 << st, 1 << l, 2, 1 << (r - l - 1), 1 << ls))

    def _shift_k(self, ri, l):
        r = self.rounds[ri][0]
        half = 1 << (r - l - 1)
        return (np.arange(1, half) * 192 >> (r - l)).reshape(-1, 1)

    def _tw(self, ri, inv=False):
        r, st, ls = self.rounds[ri]
        S = 1 << self.log_s
        tab = powers(pow(root(self.log_s), S - 1, P) if inv else root(self.log_s), S)
        e = (np.arange(1 << ls)[None, :] * brev(np.arange(1 << r), r)[:, None]) << st
        return tab[e]

    def _factor(self, kind, ks):
        if kind == "pre":
            return self.pre(ks)
        if kind == "post":
            return self.post(ks)
        return np.uint64(self.scale if kind == "scale" else 1)

    def operands(self, i, x, ks):
        kind, ri, l = self.steps[i]
        if kind == "bf":
            v = self._pairs_view(x, ri, l)
            return v[..., 0, :, :], v[..., 1, :, :]
        if kind == "shift":
            return self._pairs_view(x, ri, l)[..., 1, 1:, :], self._shift_k(ri, l)
        if kind == "tw":
            r, st, ls = self.rounds[ri]
            return x.reshape(x.shape[:-1] + (1 << st, 1 << r, 1 << ls))[..., 1:, :], self._tw(ri)[1:]
        if kind == "pre":
            return x, self.pre(ks)
        return x[..., self.src], self._factor(kind, ks)

    def apply(self, i, x, ks, inv=False):
        kind, ri, l = self.steps[i]
        y = x.copy()
        if kind == "bf":
            v, w = self._pairs_view(x, ri, l), self._pairs_view(y, ri, l)
            a, b = v[..., 0, :, :], v[..., 1, :, :]
            s, d = fadd(a, b), fsub(a, b)
            if inv:
                s, d = fmul(s, _INV2), fmul(d, _INV2)
            w[..., 0, :, :], w[..., 1, :, :] = s, d
        elif kind == "shift":
            ks_ = self._shift_k(ri, l)
            f = np.array([[pow(2, int(192 - k if inv else k), P)] for k in ks_[:, 0]], dtype=np.uint64)
            w = self._pairs_view(y, ri, l)
            w[..., 1, 1:, :] = fmul(w[..., 1, 1:, :], f)
        elif kind == "tw":
            r, st, ls = self.rounds[ri]
            w = y.reshape(y.shape[:-1] + (1 << st, 1 << r, 1 << ls))
            w[..., 1:, :] = fmul(w[..., 1:, :], self._tw(ri, inv)[1:])
        elif kind == "pre":
            f = self.pre(ks)
            y = fmul(x, inverse_of(f) if inv else f)
        else:
            f = self._factor(kind, ks)
            if inv:
                y = np.empty_like(x)
                y[..., self.src] = fmul(x, inverse_of(f)) if kind != "out" else x
            else:
                y = fmul(x[..., self.src], f) if kind != "out" else x[..., self.src]
        return y

    def run(self, t, ks, observe=None, pass_index=0):
        for i, (kind, ri, l) in enumerate(self.steps):
            if observe is not None and kind != "out":
                observe((pass_index, i, kind, ri, l), t, self.operands(i, t, ks))
            t = self.apply(i, t, ks)
        return t

    def run_inverse(self, t, ks):
        for i in reversed(range(len(self.steps))):
            t = self.apply(i, t, ks, inv=True)
        return t

    def requested_state(self, i, count, subs, ks, rng):
        """tile states (1, count, S) of the sub-transforms `subs` before step i, whose operands at step i are catalogue
        edges everywhere the step operates"""
        kind, ri, l = self.steps[i]
        shape = (1, count, 1 << self.log_s)
        x = _rand(rng, shape)

        def factor(f):          # (nb, 1, nsub | 1, S) -> the rows of `subs`
            f = np.asarray(f)
            return f if f.ndim < 4 else (f[:, 0][:, subs] if f.shape[2] > 1 else f[:, 0])
        if kind == "bf":
            v = self._pairs_view(x, ri, l)
            d = None
            if l < self.rounds[ri][0] - 1:          # a shift of the difference follows: make its operand an edge too
                d = _rand(rng, v[..., 1, :, :].shape)
                kk = self._shift_k(ri, l)[:, 0]
                for q, k in enumerate(kk, start=1):
                    d[..., q, :] = shift_edges(int(k), d[..., q, :].shape, rng)
            v[..., 0, :, :], v[..., 1, :, :] = pair_edges(v[..., 0, :, :].shape, rng, d)
        elif kind == "shift":
            v = self._pairs_view(x, ri, l)
            for q, k in enumerate(self._shift_k(ri, l)[:, 0], start=1):
                v[..., 1, q, :] = shift_edges(int(k), v[..., 1, q, :].shape, rng)
        elif kind == "tw":
            r, st, ls = self.rounds[ri]
            v = x.reshape(x.shape[:-1] + (1 << st, 1 << r, 1 << ls))
            v[..., 1:, :] = fmul(product_edges(v[..., 1:, :].shape, rng), self._tw(ri, inv=True)[1:])
        elif kind == "pre":
            x = fmul(product_edges(shape, rng), inverse_of(factor(self.pre(ks))))
        elif kind in ("post", "scale"):
            x[..., self.src] = fmul(product_edges(shape, rng), inverse_of(factor(self._factor(kind, ks))))
        return x


def inverse_of(f):
    """elementwise field inverse of a factor array (or scalar) by Montgomery's batch trick"""
    f = np.asarray(f, dtype=np.uint64)
    if f.ndim == 0:
        return np.uint64(pow(int(f), P - 2, P))
    flat = f.reshape(-1)
    if flat.size <= 4096:
        return np.array([pow(int(v), P - 2, P) for v in flat], dtype=np.uint64).reshape(f.shape)
    # pairwise products tree: inv(x) = inv(x * y) * y
    n = flat.size
    half = n // 2
    a, b = flat[:half], flat[half:2 * half]
    ab = inverse_of(fmul(a, b))
    out = np.empty(n, dtype=np.uint64)
    out[:half], out[half:2 * half] = fmul(ab, b), fmul(ab, a)
    if n & 1:
        out[-1] = pow(int(flat[-1]), P - 2, P)
    return out.reshape(f.shape)


class Network:
    """The device's transform of 2^log_n points per column: NTT (evaluate), iNTT (interpolate, inverse=True), or the LDE
    over all 2^log_blowup cosets of 7 <w_N> (log_blowup given)."""

    def __init__(self, log_n, inverse=False, log_blowup=None):
        self.log_n, self.inverse, self.lde = log_n, inverse, log_blowup is not None
        lb = log_blowup or 0
        self.nb = 1 << lb
        n = 1 << log_n
        inv_n = pow(n, P - 2, P)
        g = root(log_n + lb) if self.lde else 1

        def coset_pre(count, exp_scale):       # pre[k][i] = (s_k^exp_scale)^i, s_k = 7 g^k
            def f(ks):
                return np.stack([powers(pow(GENERATOR * pow(g, int(k), P), exp_scale, P), count) for k in ks])[:, None, None, :]
            return f

        def four_step_post(log_s, log_c, log_m, a_mul, b_mul, ctab, cconst, negate, sub_c):
            # factor[k][sub][j] = w_M^(+-((j a_mul + k b_mul) c)) ctab[c] cconst, c = sub_c(sub)
            def f(ks):
                c = sub_c.astype(np.uint64)[None, :, None]
                j = np.arange(1 << log_s, dtype=np.uint64)[None, None, :]
                kk = np.asarray(ks, dtype=np.uint64)[:, None, None]
                with np.errstate(over="ignore"):
                    e = (j * np.uint64(a_mul) + kk * np.uint64(b_mul)) * c
                x = root_pow(e, log_m, negate)
                if ctab:
                    x = fmul(x, powers(GENERATOR, 1 << log_c)[sub_c][None, :, None])
                if cconst != 1:
                    x = fmul(x, np.uint64(cconst))
                return x[:, None]
            return f

        inv_flag = inverse and not self.lde
        log_m = log_n + lb
        logR, logC = split_log(log_n)
        if logR == 0:
            self.passes = [Pass("single", log_n, ((n,), (0,)), ((n,), (0,)), inv_flag,
                                pre=coset_pre(n, 1) if self.lde else None, scale=inv_n if inverse else 1)]
        elif logC <= MAX_LOGS:
            R, C = 1 << logR, 1 << logC
            self.passes = [
                Pass("strided", logR, ((R, C), (1, 0)), ((R, C), (1, 0)), inv_flag,
                     pre=coset_pre(R, C) if self.lde else None,
                     post=four_step_post(logR, logC, log_m, self.nb if self.lde else 1, 1 if self.lde else 0, self.lde,
                                         inv_n if inverse else 1, inv_flag, np.arange(C))),
                Pass("contig", logC, ((R, C), (0, 1)), ((C, R), (1, 0)), inv_flag),
            ]
        else:
            lr, lr2, lc2 = split3(log_n)
            lc = log_n - lr
            R, C, R2, C2 = 1 << lr, 1 << lc, 1 << lr2, 1 << lc2
            self.passes = [
                Pass("A", lr, ((R, C), (1, 0)), ((R, C), (1, 0)), inv_flag,
                     pre=coset_pre(R, C) if self.lde else None,
                     post=four_step_post(lr, lc, log_m, self.nb if self.lde else 1, 1 if self.lde else 0, self.lde,
                                         inv_n if inverse else 1, inv_flag, np.arange(C))),
                Pass("B", lr2, ((R, R2, C2), (0, 2, 1)), ((R, R2, C2), (0, 2, 1)), inv_flag,
                     post=four_step_post(lr2, lc2, lc, 1, 0, False, 1, inv_flag, np.tile(np.arange(C2), R))),
                Pass("C", lc2, ((R, R2, C2), (0, 1, 2)), ((C2, R2, R), (2, 1, 0)), inv_flag),
            ]

    def forward(self, x, observe=None):
        """x: (ncols, n) -> (ncols, n), or (ncols, n * blowup) for the LDE with row j * blowup + k = coset k, point j"""
        x = np.ascontiguousarray(x, dtype=np.uint64)
        ks = np.arange(self.nb)
        X = np.broadcast_to(x, (self.nb,) + x.shape).copy()
        for pi, ps in enumerate(self.passes):
            t = ps.run(to_tiles(X, *ps.layout_in), ks, observe, pi)
            X = from_tiles(t, *ps.layout_out)
        return X[0] if not self.lde else np.ascontiguousarray(X.transpose(1, 2, 0)).reshape(x.shape[0], -1)

    def nsub(self, pass_index):
        return (1 << self.log_n) >> self.passes[pass_index].log_s

    def target(self, pass_index, steps, rng, coset=0):
        """Input (ncols, n) that reaches step steps[c, s] of pass `pass_index` in sub-transform s of column c (of coset
        `coset` for the LDE) with catalogue edge operands; steps[c, s] = -1 leaves that sub-transform's input random.
        Returns (input, requested), requested[c, s] = the tile state before the targeted step."""
        ps = self.passes[pass_index]
        steps = np.asarray(steps)
        ncols, nsub = steps.shape
        assert nsub == self.nsub(pass_index)
        ks = np.array([coset])
        shape = (1, ncols, nsub, 1 << ps.log_s)
        t = _rand(rng, shape)
        for i in np.unique(steps[steps >= 0]):
            m = steps == i
            t[:, m] = ps.requested_state(int(i), int(m.sum()), np.nonzero(m)[1], ks, rng)
        requested = t.copy()
        for i in reversed(range(int(steps.max()))):
            m = (steps > i)[None, :, :, None]
            t = np.where(m, ps.apply(i, t, ks, inv=True), t)
        X = from_tiles(t, *ps.layout_in)
        for q in reversed(range(pass_index)):
            pq = self.passes[q]
            X = from_tiles(pq.run_inverse(to_tiles(X, *pq.layout_out), ks), *pq.layout_in)
        return X[0], requested[0]


def interpolate_with_offset(x, offset):
    """wf_mat_interpolate_with_offset: the iNTT, then coefficient i times offset^-i"""
    log_n = x.shape[-1].bit_length() - 1
    c = Network(log_n, inverse=True).forward(x)
    return fmul(c, powers(pow(offset, P - 2, P), 1 << log_n)[None, :])


def operands_at(ops, mask, coset=0):
    """the operands an `observe` call received, of the sub-transforms `mask` (ncols, nsub) of one coset"""
    return [np.broadcast_to(np.asarray(o), ops[0].shape)[coset][mask] for o in ops]


def columns_for(net, pass_index, per_step=400):
    """columns enough for every operation step of a pass to act on about `per_step` targeted elements"""
    ps = net.passes[pass_index]
    per_sub, nsub = max(1, (1 << ps.log_s) // 4), net.nsub(pass_index)
    return max(-(-per_step * len(ps.targets()) // (nsub * per_sub)), -(-len(ps.targets()) // nsub))


def spread_targets(net, pass_index, ncols, first=0):
    """steps (ncols, nsub): every operation step of the pass, cycled over the sub-transforms of the columns"""
    tg = net.passes[pass_index].targets()
    nsub = net.nsub(pass_index)
    idx = (np.arange(ncols)[:, None] * nsub + np.arange(nsub)[None, :] + first) % len(tg)
    return np.array(tg)[idx]
