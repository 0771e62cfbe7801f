"""Standalone FRI proofs for the FRI verifier tests: the round trip of the reference's fri/src/prover/tests.rs (a polynomial of
degree < n evaluated over a domain of n * blowup points at offset 7, FriProver with DefaultProverChannel, positions from
draw_query_positions(0)), and the dishonest variants of the oracle's tamper list. Proofs and verdicts come from
tests/fri_ref.cpp (the CPU restatement of FriProver::build_proof and FriVerifier), compiled on first use into a temporary
directory on top of the oracle."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from oracle import oracle as o

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")

# verdicts of fri_verify: the fri::VerifierError variants FriVerifier returns (include/winterfell_b200.h WF_FRI_VERIFY_*); the
# layer of INVALID_LAYER_FOLDING and DEGREE_TRUNCATION is in bits 8 and up
FRI_VERIFY_ACCEPT, FRI_VERIFY_MALFORMED, FRI_VERIFY_LAYER_COMMITMENT_MISMATCH, FRI_VERIFY_INVALID_LAYER_FOLDING, \
    FRI_VERIFY_REMAINDER_DEGREE_MISMATCH, FRI_VERIFY_INVALID_REMAINDER_FOLDING, FRI_VERIFY_DEGREE_TRUNCATION, \
    FRI_VERIFY_RANDOM_COIN = range(8)

_ref = None


def _ref_lib():
    global _ref
    if _ref is None:
        o.lib()
        out = tempfile.mkdtemp(prefix="wf_fri_ref_")
        so = os.path.join(out, "libwf_fri_ref.so")
        try:
            subprocess.check_call(["/usr/bin/g++", "-O3", "-march=x86-64-v2", "-fopenmp", "-fPIC", "-std=c++17", "-shared",
                                   "-I", _ORACLE, "-o", so, os.path.join(_HERE, "fri_ref.cpp")])
            L = C.CDLL(so)
        finally:
            shutil.rmtree(out, ignore_errors=True)   # the loaded library stays mapped
        L.wfr_fri_build_proof.restype = C.c_long
        L.wfr_fri_verify.restype = C.c_int
        _ref = L
    return _ref


def fri_verdict(code, layer=0):
    return code | layer << 8


def fri_build_proof(h, evals, folding, rem_max_deg, blowup, positions, d=1, tamper=None):
    """FriProver::build_layers (DefaultProverChannel) + build_proof at `positions`, serialized as FriProof. tamper: a list of
    oracle.tamper(...) tuples with targets FRI_LAYER, REMAINDER, REMAINDER_LONG. Returns (proof bytes, commitments [nl + 1, 32])."""
    e_ = np.ascontiguousarray(np.asarray(evals, dtype=np.uint64).reshape(-1))
    p_ = np.ascontiguousarray(np.asarray(positions, dtype=np.uint64).reshape(-1))
    tl = list(tamper or [])
    t_ = np.array(tl, dtype=np.uint64).reshape(-1, 6) if tl else np.zeros((1, 6), dtype=np.uint64)
    cap = 1 << 24
    out = np.zeros(cap, dtype=np.uint8)
    cm = np.zeros((64, 32), dtype=np.uint8)
    u64p, u8p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint8)
    ln = _ref_lib().wfr_fri_build_proof(C.c_int(h), e_.ctypes.data_as(u64p), C.c_size_t(e_.size // d), C.c_int(d), C.c_size_t(folding),
                                        C.c_size_t(rem_max_deg), C.c_size_t(blowup), p_.ctypes.data_as(u64p), C.c_size_t(p_.size),
                                        t_.ctypes.data_as(u64p), C.c_size_t(len(tl)), cm.ctypes.data_as(u8p), out.ctypes.data_as(u8p),
                                        C.c_size_t(cap))
    if ln < 0:
        raise ValueError(f"wfr_fri_build_proof failed ({ln})")
    nl = o.fri_num_layers(e_.size // d, folding, rem_max_deg, blowup)
    return out[:ln].tobytes(), cm[: nl + 1].copy()


def fri_verify(h, d, folding, rem_max_deg, blowup, max_poly_degree, proof, commitments, positions, evaluations, coin_seed=None):
    """FriVerifier::new + verify (DefaultVerifierChannel) of one FriProof: the verdict (FRI_VERIFY_*, layer in bits 8+).
    coin_seed: the public coin's 32-byte seed (None: DefaultRandomCoin::new(&[])). Raises ValueError for arguments that
    describe no proof (the C function's negative returns)."""
    u64p, u8p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint8)
    pb = np.frombuffer(proof, dtype=np.uint8) if len(proof) else np.zeros(1, dtype=np.uint8)
    c_ = np.ascontiguousarray(np.asarray(commitments, dtype=np.uint8).reshape(-1, 32))
    p_ = np.ascontiguousarray(np.asarray(positions, dtype=np.uint64).reshape(-1))
    e_ = np.ascontiguousarray(np.asarray(evaluations, dtype=np.uint64).reshape(-1))
    s_ = None if coin_seed is None else np.frombuffer(bytes(coin_seed), dtype=np.uint8)
    r = _ref_lib().wfr_fri_verify(C.c_int(h), C.c_int(d), C.c_size_t(folding), C.c_size_t(rem_max_deg), C.c_size_t(blowup),
                                  C.c_size_t(max_poly_degree), pb.ctypes.data_as(u8p), C.c_size_t(len(proof)), c_.ctypes.data_as(u8p),
                                  C.c_size_t(c_.shape[0]), None if s_ is None else s_.ctypes.data_as(u8p), p_.ctypes.data_as(u64p),
                                  e_.ctypes.data_as(u64p), C.c_size_t(p_.size))
    if r < 0:
        raise ValueError(f"wfr_fri_verify: arguments describe no proof ({r})")
    return r


# fri_folding_2 and fri_folding_4 (2^12 trace, blowup 8; folding 2 / remainder 7 and folding 4 / remainder 255), then folding 8
# and 16: (folding, remainder max degree)
SHAPES = [(2, 7), (4, 255), (8, 7), (16, 7)]
HASHES = [o.BLAKE3, o.RP64, o.RPJIVE, o.BLAKE3_192, o.SHA3]


def codeword(log_n, log_b, d, seed):
    """[n * blowup, d] evaluations of a random polynomial of degree < n at 7 w^i."""
    n, N = 1 << log_n, 1 << (log_n + log_b)
    poly = np.concatenate([o.rand_elems(n * d, seed), np.zeros((N - n) * d, dtype=np.uint64)])
    return o.evaluate_poly_with_offset(poly, 7, 1, d).reshape(N, d)


def default_positions(h, commitments, d, domain, num_queries=32):
    """DefaultProverChannel::draw_query_positions(0) after the commit phase: every layer root reseeds the coin and draws its
    alpha, the remainder commitment only reseeds it (fri/src/prover/channel.rs). Unsorted, repeats kept."""
    coin = o.RandomCoin(h)
    for c in commitments[:-1]:
        coin.reseed(bytes(c))
        coin.draw(d)
    coin.reseed(bytes(commitments[-1]))
    return coin.draw_integers(num_queries, domain, 0)


class Case:
    """One FRI proof and everything its verifier takes: verify_args() are the arguments of oracle.fri_verify after the hash."""

    def __init__(self, h, d, nf, rem, log_n=12, log_b=3, num_queries=32, seed=1, tamper=None, positions=None):
        self.args = (h, d, nf, rem, log_n, log_b, num_queries, seed)
        self.h, self.d, self.nf, self.rem, self.blowup = h, d, nf, rem, 1 << log_b
        self.n, self.N = 1 << log_n, 1 << (log_n + log_b)
        self.max_deg = self.n - 1
        self.ev = codeword(log_n, log_b, d, seed)
        if positions is None:
            roots, _, _ = o.fri_build_layers(h, self.ev.reshape(-1), nf, rem, self.blowup, d)
            positions = default_positions(h, roots, d, self.N, num_queries)
        self.pos = np.asarray(positions, dtype=np.uint64)
        self.proof, self.cm = fri_build_proof(h, self.ev.reshape(-1), nf, rem, self.blowup, self.pos, d, tamper)
        self.evals = self.ev[self.pos.astype(np.int64)].copy()
        self.nl = self.cm.shape[0] - 1

    def tampered(self, tamper):
        """The dishonest proof of the same codeword at the same positions (oracle.tamper tuples): its own commitments."""
        return Case(*self.args, tamper=tamper, positions=self.pos)

    def layer_len(self, depth):
        return self.N // self.nf ** depth

    def verify(self, proof=None, cm=None, evals=None, max_deg=None, coin_seed=None):
        return fri_verify(self.h, self.d, self.nf, self.rem, self.blowup, self.max_deg if max_deg is None else max_deg,
                            self.proof if proof is None else proof, self.cm if cm is None else cm, self.pos,
                            self.evals if evals is None else evals, coin_seed)


def truncating_degree(n, nf, nl):
    """A max_poly_degree with the same domain as n - 1 whose max_poly_degree + 1 stops dividing by nf before the last layer,
    and the layer where FriVerifier::new finds it."""
    for m in range(n - 2, n // 2, -1):
        q = m + 1
        for i in range(nl):
            if q % nf:
                return m, i
            q //= nf
    raise AssertionError("no truncating degree")
