"""ctypes front-end for the CPU oracle (oracle/_build/libwf_oracle.so).

TEST INFRASTRUCTURE: only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs may import this module. The product (winterfell_b200/) never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libwf_oracle.so")

P = 0xFFFFFFFF00000001
BLAKE3 = 0
RP64 = 1
RPJIVE = 2
BLAKE3_192 = 3
SHA3 = 4


def build(force=False):
    if force or not os.path.exists(_SO) or any(
        os.path.getmtime(os.path.join(_HERE, f)) > os.path.getmtime(_SO)
        for f in os.listdir(_HERE) if f.endswith((".cpp", ".h", ".inc"))
    ):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


_lib = None

u64p = C.POINTER(C.c_uint64)
u8p = C.POINTER(C.c_uint8)


class Coin(C.Structure):
    _fields_ = [("seed", C.c_uint8 * 32), ("counter", C.c_uint64), ("hash_id", C.c_int)]


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        for name in ("wfo_add", "wfo_sub", "wfo_mul", "wfo_exp"):
            getattr(L, name).restype = C.c_uint64
            getattr(L, name).argtypes = [C.c_uint64, C.c_uint64]
        for name in ("wfo_inv", "wfo_to_mont", "wfo_from_mont"):
            getattr(L, name).restype = C.c_uint64
            getattr(L, name).argtypes = [C.c_uint64]
        L.wfo_root_of_unity.restype = C.c_uint64
        L.wfo_root_of_unity.argtypes = [C.c_uint32]
        L.wfo_merkle_prove_batch.restype = C.c_long
        for name in ("wfo_fold_positions", "wfo_fri_num_layers", "wfo_fri_build_layers"):
            getattr(L, name).restype = C.c_size_t
        L.wfo_coin_leading_zeros.restype = C.c_uint32
        _lib = L
    return _lib


def _u64(a):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return a, a.ctypes.data_as(u64p)


def _u8(a):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    return a, a.ctypes.data_as(u8p)


def set_threads(n):
    lib().wfo_set_threads(C.c_int(n))


def get_threads():
    return lib().wfo_get_threads()


# ---- field ----
def add(a, b): return lib().wfo_add(a, b)
def sub(a, b): return lib().wfo_sub(a, b)
def mul(a, b): return lib().wfo_mul(a, b)
def inv(a): return lib().wfo_inv(a)
def exp(a, e): return lib().wfo_exp(a, e)
def to_mont(a): return lib().wfo_to_mont(a)
def from_mont(a): return lib().wfo_from_mont(a)
def root_of_unity(log_n): return lib().wfo_root_of_unity(log_n)


def ext_mul(a, b):
    d = len(a)
    a_, ap = _u64(a); b_, bp = _u64(b)
    o = np.zeros(d, dtype=np.uint64)
    lib().wfo_ext_mul(C.c_int(d), ap, bp, o.ctypes.data_as(u64p))
    return o


def ext_inv(a):
    d = len(a)
    a_, ap = _u64(a)
    o = np.zeros(d, dtype=np.uint64)
    lib().wfo_ext_inv(C.c_int(d), ap, o.ctypes.data_as(u64p))
    return o


# ---- fft ----
def get_twiddles(n):
    o = np.zeros(n // 2, dtype=np.uint64)
    lib().wfo_get_twiddles(C.c_size_t(n), o.ctypes.data_as(u64p))
    return o


def get_inv_twiddles(n):
    o = np.zeros(n // 2, dtype=np.uint64)
    lib().wfo_get_inv_twiddles(C.c_size_t(n), o.ctypes.data_as(u64p))
    return o


def fft_in_place(v, d=1, inverse=False, split_radix_threads=0):
    """fft_in_place (fft_inputs.rs:215-252; permuted output) or, with split_radix_threads > 0, the `concurrent`
    split_radix_fft (fft/concurrent.rs:131-171) on that many threads."""
    a, ap = _u64(np.array(v, dtype=np.uint64).copy())
    n = a.size // d
    if split_radix_threads:
        lib().wfo_split_radix_fft(ap, C.c_size_t(n), C.c_int(d), C.c_int(int(inverse)), C.c_int(split_radix_threads))
    else:
        lib().wfo_fft_in_place(ap, C.c_size_t(n), C.c_int(d), C.c_int(int(inverse)))
    return a


def evaluate_poly(p, d=1):
    v = np.array(p, dtype=np.uint64, copy=True).reshape(-1)
    lib().wfo_evaluate_poly(v.ctypes.data_as(u64p), C.c_size_t(v.size // d), C.c_int(d))
    return v


def interpolate_poly(e, d=1):
    v = np.array(e, dtype=np.uint64, copy=True).reshape(-1)
    lib().wfo_interpolate_poly(v.ctypes.data_as(u64p), C.c_size_t(v.size // d), C.c_int(d))
    return v


def evaluate_poly_with_offset(p, offset, blowup, d=1):
    p_, pp = _u64(np.asarray(p).reshape(-1))
    n = p_.size // d
    o = np.zeros(n * blowup * d, dtype=np.uint64)
    lib().wfo_evaluate_poly_with_offset(pp, C.c_size_t(n), C.c_int(d), C.c_uint64(offset),
                                        C.c_size_t(blowup), o.ctypes.data_as(u64p))
    return o


def interpolate_poly_with_offset(e, offset, d=1):
    v = np.array(e, dtype=np.uint64, copy=True).reshape(-1)
    lib().wfo_interpolate_poly_with_offset(v.ctypes.data_as(u64p), C.c_size_t(v.size // d), C.c_int(d),
                                           C.c_uint64(offset))
    return v


def eval_poly_at(p, x, dp=1):
    p_, pp = _u64(np.asarray(p).reshape(-1))
    x_, xp = _u64(x)
    dx = x_.size
    o = np.zeros(max(dp, dx), dtype=np.uint64)
    lib().wfo_eval_poly_at(pp, C.c_size_t(p_.size // dp), C.c_int(dp), xp, C.c_int(dx), o.ctypes.data_as(u64p))
    return o


# ---- matrices ----
def interpolate_columns(cols, d=1):
    """cols: [c, n*d] array (column-major trace). Returns polynomial coefficients, same shape."""
    v = np.array(cols, dtype=np.uint64, copy=True)
    c = v.shape[0]
    n = v.shape[1] // d
    lib().wfo_interpolate_columns(v.ctypes.data_as(u64p), C.c_size_t(c), C.c_size_t(n), C.c_int(d))
    return v


def lde_rows(polys, blowup, d=1):
    """polys: [c, n*d] -> row-major LDE [n*blowup, c*d]."""
    p_, pp = _u64(polys)
    c = p_.shape[0]
    n = p_.shape[1] // d
    o = np.zeros((n * blowup, c * d), dtype=np.uint64)
    lib().wfo_lde_rows(pp, C.c_size_t(c), C.c_size_t(n), C.c_int(d), C.c_size_t(blowup), o.ctypes.data_as(u64p))
    return o


# ---- hashing ----
def blake3(data: bytes) -> bytes:
    d_, dp = _u8(np.frombuffer(data, dtype=np.uint8) if len(data) else np.zeros(0, dtype=np.uint8))
    o = np.zeros(32, dtype=np.uint8)
    lib().wfo_blake3(dp, C.c_size_t(len(data)), o.ctypes.data_as(u8p))
    return o.tobytes()


def rp64_permute(state):
    s = np.array(state, dtype=np.uint64, copy=True)
    lib().wfo_rp64_permute(s.ctypes.data_as(u64p))
    return s


def rpjive_permute(state):
    s = np.array(state, dtype=np.uint64, copy=True)
    lib().wfo_rpjive_permute(s.ctypes.data_as(u64p))
    return s


def hash_elements(h, elems) -> bytes:
    e_, ep = _u64(np.asarray(elems).reshape(-1))
    o = np.zeros(32, dtype=np.uint8)
    lib().wfo_hash_elements(C.c_int(h), ep, C.c_size_t(e_.size), o.ctypes.data_as(u8p))
    return o.tobytes()


def merge(h, a: bytes, b: bytes) -> bytes:
    t_, tp = _u8(np.frombuffer(a + b, dtype=np.uint8))
    o = np.zeros(32, dtype=np.uint8)
    lib().wfo_merge(C.c_int(h), tp, o.ctypes.data_as(u8p))
    return o.tobytes()


def merge_many(h, digests: bytes) -> bytes:
    t_, tp = _u8(np.frombuffer(digests, dtype=np.uint8))
    o = np.zeros(32, dtype=np.uint8)
    lib().wfo_merge_many(C.c_int(h), tp, C.c_size_t(len(digests) // 32), o.ctypes.data_as(u8p))
    return o.tobytes()


def merge_with_int(h, seed: bytes, value: int) -> bytes:
    t_, tp = _u8(np.frombuffer(seed, dtype=np.uint8))
    o = np.zeros(32, dtype=np.uint8)
    lib().wfo_merge_with_int(C.c_int(h), tp, C.c_uint64(value), o.ctypes.data_as(u8p))
    return o.tobytes()


def hash_rows(h, rows, partition_size=0):
    r_, rp = _u64(rows)
    nrows, w = r_.shape
    o = np.zeros((nrows, 32), dtype=np.uint8)
    lib().wfo_hash_rows(C.c_int(h), rp, C.c_size_t(nrows), C.c_size_t(w),
                        C.c_size_t(partition_size or w), o.ctypes.data_as(u8p))
    return o


def merkle_nodes(h, leaves):
    l_, lp = _u8(leaves)
    n = l_.shape[0]
    o = np.zeros((n, 32), dtype=np.uint8)
    lib().wfo_merkle_nodes(C.c_int(h), lp, C.c_size_t(n), o.ctypes.data_as(u8p))
    return o


def merkle_prove_batch(leaves, nodes, indexes, hash_id=BLAKE3):
    """hash_id only matters for the digest length in the serialized proof (24 bytes for Blake3_192)."""
    l_, lp = _u8(leaves); n_, np_ = _u8(nodes); i_, ip = _u64(indexes)
    k = i_.size
    lo = np.zeros((k, 32), dtype=np.uint8)
    cap = 16 + k * (int(l_.shape[0]).bit_length() + 2) * 33
    out = np.zeros(cap, dtype=np.uint8)
    r = lib().wfo_merkle_prove_batch_h(C.c_int(hash_id), lp, np_, C.c_size_t(l_.shape[0]), ip, C.c_size_t(k),
                                       lo.ctypes.data_as(u8p), out.ctypes.data_as(u8p), C.c_size_t(cap))
    if r < 0:
        raise ValueError("prove_batch failed")
    return lo, out[:r].tobytes()


# ---- FRI ----
def transpose_slice(src, folding, d=1):
    s_, sp = _u64(np.asarray(src).reshape(-1))
    o = np.zeros_like(s_)
    lib().wfo_transpose_slice(sp, C.c_size_t(s_.size // d), C.c_int(d), C.c_size_t(folding), o.ctypes.data_as(u64p))
    return o


def apply_drp(transposed, folding, offset, alpha, d=1):
    t_, tp = _u64(np.asarray(transposed).reshape(-1))
    a_, ap = _u64(alpha)
    rows = t_.size // (d * folding)
    o = np.zeros(rows * d, dtype=np.uint64)
    lib().wfo_apply_drp(tp, C.c_size_t(rows), C.c_int(d), C.c_size_t(folding), C.c_uint64(offset), ap,
                        o.ctypes.data_as(u64p))
    return o


def fold_positions(pos, source_domain, folding):
    p_, pp = _u64(pos)
    o = np.zeros(p_.size, dtype=np.uint64)
    k = lib().wfo_fold_positions(pp, C.c_size_t(p_.size), C.c_size_t(source_domain), C.c_size_t(folding),
                                 o.ctypes.data_as(u64p))
    return o[:k]


def fri_num_layers(domain, folding, rem_max_deg, blowup):
    return lib().wfo_fri_num_layers(C.c_size_t(domain), C.c_size_t(folding), C.c_size_t(rem_max_deg),
                                    C.c_size_t(blowup))


def fri_build_layers(h, evals, folding, rem_max_deg, blowup, d=1):
    e_, ep = _u64(np.asarray(evals).reshape(-1))
    ln = e_.size // d
    roots = np.zeros((40, 32), dtype=np.uint8)
    rem = np.zeros(ln * d, dtype=np.uint64)
    alphas = np.zeros(40 * d, dtype=np.uint64)
    rl = C.c_size_t(0)
    nl = lib().wfo_fri_build_layers(C.c_int(h), ep, C.c_size_t(ln), C.c_int(d), C.c_size_t(folding),
                                    C.c_size_t(rem_max_deg), C.c_size_t(blowup), roots.ctypes.data_as(u8p),
                                    rem.ctypes.data_as(u64p), C.byref(rl), alphas.ctypes.data_as(u64p))
    return roots[: nl + 1].copy(), rem[: rl.value * d].copy(), alphas[: nl * d].copy()


# ---- coin ----
class RandomCoin:
    def __init__(self, h, seed_elems=()):
        self.c = Coin()
        s_, sp = _u64(np.asarray(seed_elems, dtype=np.uint64))
        lib().wfo_coin_new(C.byref(self.c), C.c_int(h), sp, C.c_size_t(s_.size))

    @property
    def seed(self):
        return bytes(self.c.seed)

    def reseed(self, data: bytes):
        t_, tp = _u8(np.frombuffer(data, dtype=np.uint8))
        lib().wfo_coin_reseed(C.byref(self.c), tp)

    def draw(self, d=1):
        o = np.zeros(d, dtype=np.uint64)
        if lib().wfo_coin_draw(C.byref(self.c), C.c_int(d), o.ctypes.data_as(u64p)) != 0:
            raise RuntimeError("failed to draw")
        return o

    def leading_zeros(self, value):
        return lib().wfo_coin_leading_zeros(C.byref(self.c), C.c_uint64(value))

    def draw_integers(self, num, domain, nonce):
        o = np.zeros(num, dtype=np.uint64)
        if lib().wfo_coin_draw_integers(C.byref(self.c), C.c_size_t(num), C.c_size_t(domain), C.c_uint64(nonce),
                                        o.ctypes.data_as(u64p)) != 0:
            raise RuntimeError("failed to draw integers")
        return o


# ---- full prover / verifier restatement (oracle/wf_prover.cpp) ----
def make_opts(num_queries=28, blowup=8, grinding=0, ext=1, folding=4, rem_max_deg=7, batch_c=0, batch_d=0, hash_id=BLAKE3,
              num_partitions=1, hash_rate=1):
    """ProofOptions::new(...).with_partitions(num_partitions, hash_rate) (air/src/options.rs:132-200) as the opts[9] array
    of the C ABI: the partition options ride in opts[8] above the hash id (0 = the default 1, 1)."""
    part = 0 if (num_partitions, hash_rate) == (1, 1) else (num_partitions << 8) | (hash_rate << 16)
    return np.array([num_queries, blowup, grinding, ext, folding, rem_max_deg, batch_c, batch_d, hash_id | part], dtype=np.uint32)


def build_fib_trace(k, n):
    tr = np.zeros((2 * k, n), dtype=np.uint64)
    res = np.zeros(k, dtype=np.uint64)
    lib().wfo_build_fib_trace(C.c_size_t(k), C.c_size_t(n), tr.ctypes.data_as(u64p), res.ctypes.data_as(u64p))
    return tr, res


# ---- dishonest proofs (oracle/wf_prover.cpp, "dishonest proofs") ----
# Targets of a Tamper. The LDE targets put the delta into the committed and opened rows of one column only; FRI_LAYER k
# adds it to layer k before it is committed (0 = the DEEP codeword; k = the number of layers: the remainder's codeword) and
# folds on from there; REMAINDER adds it to one serialized coefficient; REMAINDER_LONG puts `index` zero coefficients in
# front of the remainder; the FLIP_* targets flip bit (delta[0] mod 8) of byte `row` of a section's opened values after the
# proof is written (FLIP_FRI: of layer `index`).
MAIN_LDE, AUX_LDE, CONSTRAINT_LDE, FRI_LAYER, REMAINDER, REMAINDER_LONG, FLIP_TRACE, FLIP_AUX, FLIP_CONSTRAINT, FLIP_FRI = range(10)
ALL_ROWS = (1 << 64) - 1


def tamper(target, index=0, row=ALL_ROWS, delta=(1, 0, 0)):
    """One tamper: delta is an element of E as up to three canonical words (base-field targets use word 0)."""
    dl = [int(v) for v in delta] + [0] * (3 - len(delta))
    return (int(target), int(index), int(row), *dl)


def _prove(fn, args, tamper_list):
    """Calls a proving entry point with its trailing tamper arguments. Returns the proof bytes, or (proof, positions) when
    tamper_list is not None: the query positions the proof opens (sorted, distinct)."""
    cap = 1 << 23
    out = np.zeros(cap, dtype=np.uint8)
    fn.restype = C.c_long
    tl = [] if tamper_list is None else list(tamper_list)
    t_ = np.array(tl, dtype=np.uint64).reshape(-1, 6) if tl else np.zeros((1, 6), dtype=np.uint64)
    pos = np.zeros(256, dtype=np.uint64)
    npos = C.c_size_t(0)
    want_pos = tamper_list is not None
    ln = fn(*args, out.ctypes.data_as(u8p), C.c_size_t(cap), t_.ctypes.data_as(u64p), C.c_size_t(len(tl)),
            pos.ctypes.data_as(u64p) if want_pos else None, C.byref(npos) if want_pos else None)
    if ln < 0:
        raise RuntimeError(f"{fn.__name__} failed ({ln})")
    proof = out[:ln].tobytes()
    return (proof, pos[: npos.value].copy()) if want_pos else proof


def prove_fib(trace, results, opts, tamper=None):
    t_, tp = _u64(trace)
    r_, rp = _u64(results)
    k, n = t_.shape[0] // 2, t_.shape[1]
    return _prove(lib().wfo_prove_fib, (tp, C.c_size_t(k), C.c_size_t(n), rp, opts.ctypes.data_as(C.POINTER(C.c_uint32))), tamper)


def verify_fib(proof: bytes, k, results, hash_id=BLAKE3):
    p_, pp = _u8(np.frombuffer(proof, dtype=np.uint8))
    r_, rp = _u64(results)
    return lib().wfo_verify_fib(pp, C.c_size_t(len(proof)), C.c_size_t(k), rp, C.c_int(hash_id))


def prove_air(desc, trace, opts, tamper=None):
    d_, dp = _u64(desc)
    t_, tp = _u64(trace)
    return _prove(lib().wfo_prove_air, (dp, C.c_size_t(d_.size), tp, C.c_size_t(t_.shape[1]),
                                        opts.ctypes.data_as(C.POINTER(C.c_uint32))), tamper)


AUX_BUILDER = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64))


def aux_callback(builder, aw, nr, n, d):
    """Wraps `builder(rand [nr, d] uint64) -> aux columns [aw, n, d] uint64` as the C callback both
    provers take (prover/src/lib.rs:236-247 build_aux_trace)."""
    def cb(_user, rand_p, out_p):
        try:
            rand = np.ctypeslib.as_array(rand_p, shape=(nr, d)).copy() if nr else np.zeros((0, d), dtype=np.uint64)
            aux = np.ascontiguousarray(builder(rand), dtype=np.uint64).reshape(aw, n, d)
            np.ctypeslib.as_array(out_p, shape=(aw, n, d))[:] = aux
            return 0
        except Exception:  # an exception must not unwind through the C caller
            import traceback
            traceback.print_exc()
            return 1
    return AUX_BUILDER(cb)


def prove_air_aux(desc, trace, opts, builder, aw, nr, tamper=None):
    d_, dp = _u64(desc)
    t_, tp = _u64(trace)
    cb = aux_callback(builder, aw, nr, t_.shape[1], int(opts[3]))
    return _prove(lib().wfo_prove_air_aux, (dp, C.c_size_t(d_.size), tp, C.c_size_t(t_.shape[1]),
                                            opts.ctypes.data_as(C.POINTER(C.c_uint32)), cb, None), tamper)


def values_callback(values_fn, nr, nvals, d):
    """Wraps values_fn(rand [nr, d], values [nvals, d]) -> values as the get_aux_assertions callback of both provers / the verifier."""
    def cb(_user, rand_p, val_p):
        try:
            rand = np.ctypeslib.as_array(rand_p, shape=(nr, d)).copy()
            vals = np.ctypeslib.as_array(val_p, shape=(nvals, d))
            vals[:] = np.ascontiguousarray(values_fn(rand, vals.copy()), dtype=np.uint64).reshape(nvals, d)
            return 0
        except Exception:
            import traceback
            traceback.print_exc()
            return 1
    return AUX_BUILDER(cb)


def prove_air_aux_dyn(desc, trace, opts, builder, values_fn, aw, nr, nvals, tamper=None):
    d_, dp = _u64(desc)
    t_, tp = _u64(trace)
    d = int(opts[3])
    cb, cv = aux_callback(builder, aw, nr, t_.shape[1], d), values_callback(values_fn, nr, nvals, d)
    return _prove(lib().wfo_prove_air_aux_dyn, (dp, C.c_size_t(d_.size), tp, C.c_size_t(t_.shape[1]),
                                                opts.ctypes.data_as(C.POINTER(C.c_uint32)), cb, cv, None), tamper)


def verify_air_dyn(desc, proof: bytes, hash_id, values_fn, nr, nvals, d):
    d_, dp = _u64(desc)
    p_, pp = _u8(np.frombuffer(proof, dtype=np.uint8))
    cv = values_callback(values_fn, nr, nvals, d)
    return lib().wfo_verify_air_dyn(dp, C.c_size_t(d_.size), pp, C.c_size_t(len(proof)), C.c_int(hash_id), cv, None)


def perm_rap_aux(trace, rand):
    """Aux columns [3, n, d] of tests/airs.py perm_rap for the drawn random elements rand [2, d]."""
    t_, tp = _u64(trace)
    r_, rp = _u64(rand)
    n, d = t_.shape[1], r_.shape[1]
    out = np.zeros((3, n, d), dtype=np.uint64)
    lib().wfo_perm_rap_aux(tp, C.c_size_t(n), C.c_int(d), rp, out.ctypes.data_as(u64p))
    return out


def eval_constraint_rows(desc, n, blowup, ext, coeffs, rand, rows, cur, nxt, acur=None, anxt=None):
    """The prover's combined constraint evaluations on CE rows `rows` (wfo_eval_constraint_rows) from their frames:
    cur / nxt [k, w] main LDE rows, acur / anxt [k, aw * ext] aux LDE rows (None without an aux segment);
    coeffs [constraints + assertions, ext] in wf_eval_constraints' layout, rand [nr, ext]. Returns [k, ext]."""
    d_, dp = _u64(desc)
    c_, cp = _u64(coeffs)
    r_, rp = _u64(rand if rand is not None else np.zeros(1, dtype=np.uint64))
    w_, wp = _u64(rows)
    k = w_.size
    cu, cup = _u64(cur)
    nx, nxp = _u64(nxt)
    acp = anp = None
    if acur is not None:
        ac_, acp = _u64(acur)
        an_, anp = _u64(anxt)
    out = np.zeros((k, ext), dtype=np.uint64)
    L = lib()
    L.wfo_eval_constraint_rows.restype = C.c_long
    r = L.wfo_eval_constraint_rows(dp, C.c_size_t(d_.size), C.c_size_t(n), C.c_size_t(blowup), C.c_int(ext), cp, rp, wp, C.c_size_t(k),
                                   cup, nxp, acp, anp, out.ctypes.data_as(u64p))
    if r != 0:
        raise ValueError(f"wfo_eval_constraint_rows: {r}")
    return out


def verify_air(desc, proof: bytes, hash_id=BLAKE3):
    d_, dp = _u64(desc)
    p_, pp = _u8(np.frombuffer(proof, dtype=np.uint8))
    return lib().wfo_verify_air(dp, C.c_size_t(d_.size), pp, C.c_size_t(len(proof)), C.c_int(hash_id))


def rand_elems(shape, seed):
    """Uniform field elements in [0, p) from a seeded PRNG (rejection sampling)."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 2**64, size=shape, dtype=np.uint64)
    bad = a >= np.uint64(P)
    while bad.any():
        a[bad] = rng.integers(0, 2**64, size=int(bad.sum()), dtype=np.uint64)
        bad = a >= np.uint64(P)
    return a
