// verify.cu — verifier::verify (verifier/src/lib.rs:82-260) for a batch of proofs of one AIR (wf_verify_air_batch), and
// FriVerifier::new + verify (fri/src/verifier/mod.rs:107-331) for a batch of standalone FRI proofs of one shape
// (wf_fri_verify_batch). Both share the FRI part: the FriProof parser, the query-phase plan (plan_fri), the device records
// and kernels, and the batch runner (run_plan).
//
// Host, per proof in batch order: parse the proof bytes (the inverse of prove_air's writer), check the options against the
// acceptable set or the proof's security estimate against a minimum (security.hpp), check the AIR at the trace length the
// proof declares, replay the transcript (PublicCoin), check the OOD
// consistency (verifier/src/evaluator.rs) and turn every Merkle opening into a merge schedule without hashing anything.
// Device, once per batch (one upload, one download, one synchronisation): the leaf hashes of every opened row
// (commit_hash_rows), one merge launch per tree level for every tree of every proof (commit_merge_ops), the root compares,
// the DEEP composition at the queries, one FRI launch per depth, the remainder and the verdicts.
//
// A proof's verdict is its FIRST failed check in the reference's order. Every check that fails writes (rank << 4 | code) with
// atomicMin into the proof's word; ranks follow the order of the checks, codes are WF_VERIFY_* (WF_FRI_VERIFY_* for the
// standalone FRI verifier). A check the host can decide
// (a malformed opening, a position map that does not fit) seeds that word and ends the plan of the proof there: the device
// still runs the proof's earlier checks, which win when they fail.
#include <cstring>

#include "internal.hpp"
#include "air_host.hpp"
#include "minidft.cuh"
#include "security.hpp"

namespace {

constexpr u32 R_TRACE = 1, R_AUX = 2, R_CONS = 3, R_FRI = 4;  // FRI depth i: layer R_FRI + 2i, fold R_FRI + 2i + 1
constexpr u32 R_REMAINDER = R_FRI + 2 * 40;
constexpr u32 NO_FAIL = 0xffffffffu;
__host__ __device__ constexpr u32 fail_word(u32 rank, u32 code) { return rank << 4 | code; }
__host__ __device__ constexpr u32 fri_layer_rank(u32 depth) { return R_FRI + 2 * depth; }

// ---- device records (one upload) ----
struct ProofDev {
    u32 d, c, aw, kc;
    u32 log_N, rn;
    u32 a_off, r_off;   // alphas / remainder coefficients, words after `cst`
    u64 cst;            // word offset of: z, zg, deep coefficients [c + aw + kc], t_cur [c + aw], t_nxt, q_cur [kc], q_nxt
                        // (3 words per element), then the alphas and the remainder
    u32 slot, pad;      // batch index
};
struct DeepItem { u32 proof, out; u64 pos, t_off, a_off, c_off; u32 t_st, a_st, c_st, pad; };
struct FoldItem { u32 proof, depth, log_dom, out; u64 fpos, off; u32 stride, nf_log, chk0, nchk; };
struct CheckItem { u32 cur, col; };
struct RemItem { u32 proof, cur, log_dom, pad; u64 pos; };
struct CmpItem { u32 slot, fail, got, want; };

template <int D>
__device__ __forceinline__ GlExt<D> ld3(const u64* p) {
    GlExt<D> r;
#pragma unroll
    for (int k = 0; k < D; k++) r.v[k] = p[k];
    return r;
}
template <int D>
__device__ __forceinline__ void st3(u64* p, const GlExt<D>& v) {
#pragma unroll
    for (int k = 0; k < 3; k++) p[k] = k < D ? v.v[k] : 0;
}
template <int D>
__device__ __forceinline__ bool eq3(const GlExt<D>& a, const u64* b) {
    bool e = true;
#pragma unroll
    for (int k = 0; k < D; k++) e = e && a.v[k] == b[k];
    return e;
}

__global__ void verify_compare_kernel(const u64* __restrict__ arena, const CmpItem* __restrict__ items, u32 count, u32* fail) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const CmpItem it = items[i];
    bool e = true;
    for (int k = 0; k < 4; k++) e = e && arena[(size_t)it.got * 4 + k] == arena[(size_t)it.want * 4 + k];
    if (!e) atomicMin(fail + it.slot, it.fail);
}

// DEEP composition at one query (verifier/src/composer.rs): x = 7 g^pos,
// sum cc (v - T(z)) / (x - z) + sum cc (v - T(zg)) / (x - zg) over main, aux and composition columns
template <int D>
__device__ void deep_one(const ProofDev& pd, const u64* __restrict__ up, const DeepItem& it, u64* __restrict__ evals) {
    const u64* cs = up + pd.cst;
    const u32 ct = pd.c + pd.aw, kc = pd.kc;
    const GlExt<D> z = ld3<D>(cs), zg = ld3<D>(cs + 3);
    const u64* dc = cs + 6;
    const u64* tc = dc + 3 * (ct + kc);
    const u64* tn = tc + 3 * ct;
    const u64* qc = tn + 3 * ct;
    const u64* qn = qc + 3 * kc;
    GlExt<D> t1 = ext_zero<D>(), t2 = ext_zero<D>();
    for (u32 j = 0; j < pd.c; j++) {
        const GlExt<D> v = ext_from_base<D>(up[it.t_off + (size_t)j * it.t_st]), cc = ld3<D>(dc + 3 * j);
        t1 = ext_add(t1, ext_mul(ext_sub(v, ld3<D>(tc + 3 * j)), cc));
        t2 = ext_add(t2, ext_mul(ext_sub(v, ld3<D>(tn + 3 * j)), cc));
    }
    for (u32 j = 0; j < pd.aw; j++) {
        GlExt<D> v;
#pragma unroll
        for (int k = 0; k < D; k++) v.v[k] = up[it.a_off + (size_t)(j * D + k) * it.a_st];
        const u32 q = pd.c + j;
        const GlExt<D> cc = ld3<D>(dc + 3 * q);
        t1 = ext_add(t1, ext_mul(ext_sub(v, ld3<D>(tc + 3 * q)), cc));
        t2 = ext_add(t2, ext_mul(ext_sub(v, ld3<D>(tn + 3 * q)), cc));
    }
    for (u32 j = 0; j < kc; j++) {
        GlExt<D> v;
#pragma unroll
        for (int k = 0; k < D; k++) v.v[k] = up[it.c_off + (size_t)(j * D + k) * it.c_st];
        const GlExt<D> cc = ld3<D>(dc + 3 * (ct + j));
        t1 = ext_add(t1, ext_mul(ext_sub(v, ld3<D>(qc + 3 * j)), cc));
        t2 = ext_add(t2, ext_mul(ext_sub(v, ld3<D>(qn + 3 * j)), cc));
    }
    const u64 x = gl_mul(gl_pow(gl_root_of_unity(pd.log_N), it.pos), GL_GENERATOR);
    const GlExt<D> d1 = ext_sub(ext_from_base<D>(x), z), d2 = ext_sub(ext_from_base<D>(x), zg);
    st3<D>(evals + (size_t)it.out * 3, ext_mul(ext_add(ext_mul(t1, d2), ext_mul(t2, d1)), ext_inv(ext_mul(d1, d2))));
}
__global__ void __launch_bounds__(128) verify_deep_kernel(const ProofDev* __restrict__ pds, const u64* __restrict__ up,
                                                          const DeepItem* __restrict__ items, u32 count, u64* __restrict__ evals) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const DeepItem it = items[i];
    const ProofDev pd = pds[it.proof];
    switch (pd.d) {
        case 1: deep_one<1>(pd, up, it, evals); break;
        case 2: deep_one<2>(pd, up, it, evals); break;
        default: deep_one<3>(pd, up, it, evals); break;
    }
}

constexpr __device__ u32 cbrev_v(u32 v, int bits) {
    u32 r = 0;
    for (int i = 0; i < bits; i++) r |= ((v >> i) & 1u) << (bits - 1 - i);
    return r;
}
// One queried row of a FRI layer (fri/src/verifier/mod.rs:236-331): the queries that fall in it must carry the current
// evaluations at their slots; then the row is folded at alpha with the size-nf inverse mini-DFT of the prover's fold kernel
// (fri.cu fri_fold_kernel), x = 7 w_dom^fpos.
template <int D, int LOGNF>
__device__ void fold_one(const ProofDev& pd, const u64* __restrict__ up, const FoldItem& it, const CheckItem* __restrict__ chk,
                         u64* __restrict__ evals, u32* fail, u32 code) {
    constexpr int NF = 1 << LOGNF;
    u64 x[D][NF];
#pragma unroll
    for (int k = 0; k < NF; k++)
#pragma unroll
        for (int c = 0; c < D; c++) x[c][k] = up[it.off + (size_t)(k * D + c) * it.stride];
    for (u32 q = 0; q < it.nchk; q++) {
        const CheckItem ck = chk[it.chk0 + q];
        bool e = true;
        for (int c = 0; c < D; c++) e = e && up[it.off + (size_t)(ck.col * D + c) * it.stride] == evals[(size_t)ck.cur * 3 + c];
        if (!e) atomicMin(fail + pd.slot, fail_word(fri_layer_rank(it.depth) + 1, code));
    }
#pragma unroll
    for (int c = 0; c < D; c++) mini_dft<LOGNF>(x[c]);
    const u64 xinv = gl_inv(gl_mul(gl_pow(gl_root_of_unity(it.log_dom), it.fpos), GL_GENERATOR));
    const GlExt<D> beta = ext_mul_base(ld3<D>(up + pd.cst + pd.a_off + 3 * it.depth), xinv);
    GlExt<D> acc;
#pragma unroll
    for (int c = 0; c < D; c++) acc.v[c] = x[c][cbrev_v(1u, LOGNF)];
#pragma unroll
    for (int j = NF - 2; j >= 0; j--) {
        GlExt<D> cj;
#pragma unroll
        for (int c = 0; c < D; c++) cj.v[c] = x[c][cbrev_v((u32)((NF - j) % NF), LOGNF)];
        acc = ext_add(ext_mul(acc, beta), cj);
    }
    st3<D>(evals + (size_t)it.out * 3, ext_mul_base(acc, GL_P - ((GL_P - 1) >> LOGNF)));
}
template <int D>
__device__ void fold_d(const ProofDev& pd, const u64* up, const FoldItem& it, const CheckItem* chk, u64* evals, u32* fail, u32 code) {
    switch (it.nf_log) {
        case 1: fold_one<D, 1>(pd, up, it, chk, evals, fail, code); break;
        case 2: fold_one<D, 2>(pd, up, it, chk, evals, fail, code); break;
        case 3: fold_one<D, 3>(pd, up, it, chk, evals, fail, code); break;
        default: fold_one<D, 4>(pd, up, it, chk, evals, fail, code); break;
    }
}
// code: the verdict code of a row that does not carry the current evaluations (InvalidLayerFolding)
__global__ void __launch_bounds__(128) verify_fri_kernel(const ProofDev* __restrict__ pds, const u64* __restrict__ up,
                                                         const FoldItem* __restrict__ items, u32 count, const CheckItem* __restrict__ chk,
                                                         u64* __restrict__ evals, u32* fail, u32 code) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const FoldItem it = items[i];
    const ProofDev pd = pds[it.proof];
    switch (pd.d) {
        case 1: fold_d<1>(pd, up, it, chk, evals, fail, code); break;
        case 2: fold_d<2>(pd, up, it, chk, evals, fail, code); break;
        default: fold_d<3>(pd, up, it, chk, evals, fail, code); break;
    }
}

// the remainder polynomial (reversed coefficients, eval_horner_rev) at each final position
template <int D>
__device__ void rem_one(const ProofDev& pd, const u64* up, const RemItem& it, const u64* evals, u32* fail, u32 code) {
    const u64 x = gl_mul(gl_pow(gl_root_of_unity(it.log_dom), it.pos), GL_GENERATOR);
    const u64* r = up + pd.cst + pd.r_off;
    GlExt<D> acc = ext_zero<D>();
    for (u32 j = 0; j < pd.rn; j++) acc = ext_add(ext_mul_base(acc, x), ld3<D>(r + 3 * j));
    if (!eq3<D>(acc, evals + (size_t)it.cur * 3)) atomicMin(fail + pd.slot, fail_word(R_REMAINDER, code));
}
// code: the verdict code of a remainder that does not take the folded value (InvalidRemainderFolding)
__global__ void verify_remainder_kernel(const ProofDev* __restrict__ pds, const u64* __restrict__ up, const RemItem* __restrict__ items,
                                        u32 count, const u64* __restrict__ evals, u32* fail, u32 code) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const RemItem it = items[i];
    const ProofDev pd = pds[it.proof];
    switch (pd.d) {
        case 1: rem_one<1>(pd, up, it, evals, fail, code); break;
        case 2: rem_one<2>(pd, up, it, evals, fail, code); break;
        default: rem_one<3>(pd, up, it, evals, fail, code); break;
    }
}

__global__ void verify_verdict_kernel(const u32* __restrict__ fail, u32 batch, u32* __restrict__ verdicts) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < batch) verdicts[i] = fail[i] == NO_FAIL ? WF_VERIFY_ACCEPT : (fail[i] & 15u);
}

// ---- host: proof bytes ----
struct Reader {  // ByteReader (utils/core/src/serde/byte_reader.rs)
    const u8* p;
    size_t n, pos = 0;
    bool ok = true;
    u8 u8_() { if (pos + 1 > n) { ok = false; return 0; } return p[pos++]; }
    u64 le(int k) {
        if (pos + k > n) { ok = false; return 0; }
        u64 v = 0;
        for (int i = 0; i < k; i++) v |= (u64)p[pos + i] << (8 * i);
        pos += k;
        return v;
    }
    const u8* take(size_t k) { if (k > n - pos) { ok = false; return nullptr; } const u8* q = p + pos; pos += k; return q; }
    u64 usize() {  // vint64 (read_usize)
        if (pos >= n) { ok = false; return 0; }
        const u8 first = p[pos];
        const int len = first == 0 ? 9 : __builtin_ctz(first) + 1;
        if (pos + len > n) { ok = false; return 0; }
        if (len == 9) { pos += 1; return le(8); }
        u64 raw = 0;
        for (int i = 0; i < len; i++) raw |= (u64)p[pos + i] << (8 * i);
        pos += len;
        return raw >> len;
    }
};
struct Bytes { const u8* p = nullptr; size_t n = 0; };

// A digest of Rp64_256 / RpJive64_256 is read word by word through BaseElement::new, which reduces a word w >= p to w - p
// (ElementDigest::read_from, rp64_256/digest.rs:61-69, rp64_256_jive/digest.rs:61-69): such a commitment or Merkle path node
// stands for the reduced digest. The byte digests are taken as they are.
void read_digest(int hash_id, const u8* q, Digest& dg) {
    memcpy(dg.b, q, WF_DIGEST_BYTES(hash_id));
    if (hash_id != WF_HASH_RP64_256 && hash_id != WF_HASH_RPJIVE64_256) return;
    for (int k = 0; k < 4; k++) {
        u64 w;
        memcpy(&w, dg.b + 8 * k, 8);
        if (w >= GL_P) w -= GL_P;
        memcpy(dg.b + 8 * k, &w, 8);
    }
}
// Every field element of a proof is read through BaseElement::read_from, which refuses a word >= p (math/src/field/f64/
// mod.rs:673-681): the opened values (air/src/proof/table.rs:60-65), the OOD frames (ood_frame.rs:140,157), the FRI layer
// values and the remainder (fri/src/proof.rs:185,321). VerifierChannel::new reports each as ProofDeserializationError
// (verifier/src/channel.rs:92-118), after the acceptable options and the AIR (verifier/src/lib.rs:82-140).
bool all_canonical(const Bytes& b, size_t skip = 0) {
    for (size_t at = skip; at + 8 <= b.n; at += 8) {
        u64 w;
        memcpy(&w, b.p + at, 8);
        if (w >= GL_P) return false;
    }
    return true;
}
// FriProof (fri/src/proof.rs): per layer the queried rows and their batch opening, the remainder, num_partitions as a
// power of two (proof.rs:36,101-103)
struct FriBytes {
    std::vector<Bytes> fv, fp;
    Bytes rem;
    u8 log_parts = 0;
};
// FriProof::read_from (proof.rs:166-179, 295-310) without the value checks: false when the bytes end early
bool read_fri_proof(Reader& r, FriBytes& f) {
    const u8 fl = r.u8_();
    f.fv.resize(fl); f.fp.resize(fl);
    for (u32 i = 0; i < fl; i++) {
        f.fv[i].n = r.le(4); f.fv[i].p = r.take(f.fv[i].n);
        if (!r.ok) return false;
        f.fp[i].n = r.le(4); f.fp[i].p = r.take(f.fp[i].n);
        if (!r.ok) return false;
    }
    f.rem.n = r.le(2); f.rem.p = r.take(f.rem.n);
    f.log_parts = r.u8_();
    return r.ok;
}
struct Parsed {
    u32 logn = 0;
    Options o{};
    u32 nuq = 0, nl = 0;
    std::vector<Digest> cm;       // commitments in 32-byte slots (Blake3_192 zero-padded, as ByteDigest::as_bytes)
    Bytes tq_v, tq_p, aq_v, aq_p, cq_v, cq_p, ood_t, ood_q;
    FriBytes fri;
    u64 nonce = 0;
};

// The Context at the head of a proof (context.rs:159-184), the inverse of write_context (air_host.hpp), read without checks:
// head_ok when the bytes up to the modulus are there, ok when the options and the constraint count are too
struct ProofContext {
    u8 mw = 0, aw = 0, ar = 0, logn = 0, ml = 0;
    const u8* mod = nullptr;
    Options o{};
    u64 ncons = 0;
    bool head_ok = false, ok = false;
    bool goldilocks() const {
        const u64 p = GL_P;
        return ml == 8 && !memcmp(mod, &p, 8);
    }
    // the options' asserts, TraceInfo::read_from (2^logn >= 8) and the two-adicity of the field
    bool in_range() const { return options_in_range(o) && logn >= 3 && logn + log2_ceil(o.blowup) <= 32; }
};
void read_context(Reader& r, int hash_id, ProofContext& cx) {
    cx.mw = r.u8_(); cx.aw = r.u8_(); cx.ar = r.u8_(); cx.logn = r.u8_();
    const u64 meta = r.le(2);
    r.take(meta);
    cx.ml = r.u8_();
    cx.mod = r.take(cx.ml);
    cx.head_ok = r.ok;
    Options& o = cx.o;
    o.num_queries = r.u8_(); o.blowup = r.u8_(); o.grinding = r.u8_(); o.ext = r.u8_(); o.folding = r.u8_();
    o.rem_max_deg = r.u8_(); o.batch_c = r.u8_(); o.batch_d = r.u8_(); o.num_partitions = r.u8_(); o.hash_rate = r.u8_();
    o.hash_id = hash_id;
    cx.ncons = r.usize();
    cx.ok = r.ok;
}

// Proof::from_bytes with the oracle's order of checks: WF_VERIFY_ACCEPT when the bytes parse
u32 parse_proof(const AirHost& air, int hash_id, const u8* proof, size_t len, Parsed& pp) {
    Reader r{proof, len};
    ProofContext cx;
    read_context(r, hash_id, cx);
    const u8 mw = cx.mw, logn = cx.logn;
    if (!cx.head_ok || !cx.goldilocks() || cx.aw != air.aw || cx.ar != air.nr) return WF_VERIFY_CONTEXT;
    if (!cx.ok) return WF_VERIFY_MALFORMED;
    Options& o = pp.o;
    o = cx.o;
    const u64 ncons = cx.ncons;
    if (!cx.in_range()) return WF_VERIFY_MALFORMED;
    const u32 lb = log2_ceil(o.blowup);
    pp.logn = logn;
    const size_t n = (size_t)1 << logn, N = n << lb;
    if (mw != air.w || ncons != air.num_constraints() || o.ext < 1 || o.ext > 3) return WF_VERIFY_CONTEXT;
    const size_t d = o.ext, ct = air.w + air.aw, kc = air.num_comp_cols(n), nseg = air.aw ? 2 : 1;
    pp.nuq = r.u8_();
    const u64 clen = r.le(2);
    const u8* cm = r.take(clen);
    if (!r.ok) return WF_VERIFY_MALFORMED;
    {
        size_t dom = N, max_rem = (size_t)(o.rem_max_deg + 1) * o.blowup;
        while (dom > max_rem) { dom /= o.folding; pp.nl++; }
    }
    const size_t dl = WF_DIGEST_BYTES(hash_id), ncm = nseg + 1 + pp.nl + 1;
    if (clen != dl * ncm) return WF_VERIFY_MALFORMED;
    pp.cm.assign(ncm, Digest{});
    for (size_t i = 0; i < ncm; i++) read_digest(hash_id, cm + dl * i, pp.cm[i]);
    auto read_q = [&](Bytes& v, Bytes& pr) {
        v.n = r.usize(); v.p = r.take(v.n);
        if (!r.ok) return false;
        pr.n = r.usize(); pr.p = r.take(pr.n);
        return r.ok;
    };
    if (!read_q(pp.tq_v, pp.tq_p) || (air.aw && !read_q(pp.aq_v, pp.aq_p)) || !read_q(pp.cq_v, pp.cq_p)) return WF_VERIFY_MALFORMED;
    pp.ood_t.n = r.le(2); pp.ood_t.p = r.take(pp.ood_t.n);
    pp.ood_q.n = r.le(2); pp.ood_q.p = r.take(pp.ood_q.n);
    if (!r.ok || pp.ood_t.n != 1 + 2 * ct * d * 8 || pp.ood_q.n != 1 + 2 * kc * d * 8 || pp.ood_t.p[0] != 2 || pp.ood_q.p[0] != 2)
        return WF_VERIFY_MALFORMED;
    if (!read_fri_proof(r, pp.fri) || pp.fri.fv.size() != pp.nl) return WF_VERIFY_MALFORMED;
    pp.nonce = r.le(8);
    if (!r.ok || r.pos != len || pp.fri.rem.n % (8 * d)) return WF_VERIFY_MALFORMED;
    return WF_VERIFY_ACCEPT;
}
bool values_canonical(const Parsed& pp) {
    for (const Bytes* b : {&pp.tq_v, &pp.aq_v, &pp.cq_v, &pp.fri.rem})
        if (!all_canonical(*b)) return false;
    if (!all_canonical(pp.ood_t, 1) || !all_canonical(pp.ood_q, 1)) return false;   // after the frame-size byte
    for (const Bytes& b : pp.fri.fv)
        if (!all_canonical(b)) return false;
    return true;
}

// ---- host: the batch plan ----
// digest references before the arena is laid out: the region in the top two bits
constexpr u32 REF_UP = 0u << 30, REF_LEAF = 1u << 30, REF_NODE = 2u << 30, REF_MASK = (1u << 30) - 1;
struct RowGroup { u32 words, part; std::vector<const u8*> rows; };
struct Plan {
    std::vector<RowGroup> groups;
    std::map<std::pair<u32, u32>, u32> group_of;
    std::vector<std::pair<u32, u32>> leaves;   // leaf k: (group, row within the group)
    std::vector<Digest> up;                    // uploaded digests: proof nodes and commitments
    u32 nodes = 0;                             // computed digests
    std::vector<std::vector<uint3>> levels;    // merges per tree level
    std::vector<CmpItem> cmps;
    std::vector<ProofDev> pds;
    std::vector<u64> cst;
    struct Deep { u32 proof, out, t, a, c; u64 pos; };   // t / a / c: leaves of the opened rows
    std::vector<Deep> deep;
    struct Fold { FoldItem it; u32 leaf; };
    std::vector<std::vector<Fold>> folds;      // per depth
    std::vector<std::vector<CheckItem>> checks;  // per depth
    std::vector<RemItem> rems;
    u32 nevals = 0;
    std::vector<u64> ev0;                      // evaluations the caller gives, 3 words each: slots 0, 1, ... (standalone FRI)

    u32 add_row(u32 words, u32 part, const u8* row) {
        auto key = std::make_pair(words, part);
        auto it = group_of.find(key);
        if (it == group_of.end()) {
            it = group_of.insert({key, (u32)groups.size()}).first;
            groups.push_back({words, part, {}});
        }
        RowGroup& g = groups[it->second];
        leaves.push_back({it->second, (u32)g.rows.size()});
        g.rows.push_back(row);
        return (u32)leaves.size() - 1;
    }
    u32 upload(const Digest& d) { up.push_back(d); return REF_UP | (u32)(up.size() - 1); }

    // BatchMerkleProof::get_root (crypto/src/merkle/proofs.rs:110-205) as a merge schedule. false: the opening does not parse,
    // has the wrong depth or does not open the given indexes (what makes the oracle's check fail before any hash is compared)
    bool opening(const Bytes& path, int hash_id, size_t nleaves, const std::vector<u64>& idx, const std::vector<u32>& leaf_refs,
                 u32* root_ref) {
        Reader r{path.p, path.n};
        const u8 depth = r.u8_();
        const u64 nv = r.usize();
        if (!r.ok || nv > 100000 || depth < 1 || depth > 40) return false;
        const size_t dl = WF_DIGEST_BYTES(hash_id), up0 = up.size();
        auto undo = [&]() { up.resize(up0); return false; };
        std::vector<std::vector<u32>> nodes_of(nv);
        for (auto& v : nodes_of) {
            const u64 ln = r.usize();
            if (!r.ok || ln > 64) return undo();
            for (u64 i = 0; i < ln; i++) {
                const u8* q = r.take(dl);
                if (!q) return undo();
                Digest dg{};
                read_digest(hash_id, q, dg);
                v.push_back(upload(dg));
            }
        }
        if (!r.ok || r.pos != path.n || ((size_t)1 << depth) != nleaves) return undo();
        if (idx.empty() || idx.size() != leaf_refs.size()) return undo();
        const size_t nl = nleaves;
        std::map<u64, size_t> index_map;
        for (size_t i = 0; i < idx.size(); i++) { if (idx[i] >= nl) return undo(); index_map[idx[i]] = i; }
        if (index_map.size() != idx.size()) return undo();
        std::set<u64> norm;
        for (u64 i : idx) norm.insert(i & ~(u64)1);
        if (norm.size() != nodes_of.size()) return undo();
        std::vector<std::vector<uint3>> lv(depth);
        u32 made = 0;
        auto fresh = [&]() { return REF_NODE | (nodes + made++); };
        std::map<u64, u32> v;
        std::vector<u64> next;
        std::vector<size_t> ptr;
        size_t i = 0;
        for (u64 index : norm) {
            auto a = index_map.find(index), b = index_map.find(index + 1);
            u32 l, rr;
            if (a != index_map.end()) {
                l = leaf_refs[a->second];
                if (b != index_map.end()) { rr = leaf_refs[b->second]; ptr.push_back(0); }
                else { if (nodes_of[i].empty()) return undo(); rr = nodes_of[i][0]; ptr.push_back(1); }
            } else {
                if (nodes_of[i].empty() || b == index_map.end()) return undo();
                l = nodes_of[i][0]; rr = leaf_refs[b->second]; ptr.push_back(1);
            }
            const u32 out = fresh();
            lv[0].push_back(make_uint3(l, rr, out));
            const u64 pi = (nl + index) >> 1;
            v[pi] = out;
            next.push_back(pi);
            i++;
        }
        for (u32 level = 1; level < depth; level++) {
            const std::vector<u64> ids = next;
            next.clear();
            for (size_t q = 0; q < ids.size(); q++) {
                const u64 node = ids[q], sib_index = node ^ 1;
                const size_t slot = q;
                u32 sib;
                if (q + 1 < ids.size() && ids[q + 1] == sib_index) {
                    auto it = v.find(sib_index);
                    if (it == v.end()) return undo();
                    sib = it->second;
                    q++;
                } else {
                    if (nodes_of[slot].size() <= ptr[slot]) return undo();
                    sib = nodes_of[slot][ptr[slot]++];
                }
                auto nit = v.find(node);
                if (nit == v.end()) return undo();
                const u32 out = fresh();
                lv[level].push_back(node & 1 ? make_uint3(sib, nit->second, out) : make_uint3(nit->second, sib, out));
                v[node >> 1] = out;
                next.push_back(node >> 1);
            }
        }
        auto it = v.find(1);
        if (it == v.end()) return undo();
        *root_ref = it->second;
        nodes += made;
        if (levels.size() < lv.size()) levels.resize(lv.size());
        for (size_t l = 0; l < lv.size(); l++) levels[l].insert(levels[l].end(), lv[l].begin(), lv[l].end());
        return true;
    }
    // rows of one opening (queries.rs): leaf refs, or false when the values do not have the expected length
    bool rows(const Bytes& vals, size_t count, u32 words, u32 part, std::vector<u32>& refs) {
        if (vals.n != count * words * 8) return false;
        refs.clear();
        for (size_t i = 0; i < count; i++) refs.push_back(REF_LEAF | add_row(words, part, vals.p + i * words * 8));
        return true;
    }
};

template <int D>
GlExt<D> read_elem(const u8* p, size_t idx) {
    GlExt<D> e;
    memcpy(e.v, p + idx * D * 8, D * 8);
    return e;
}
template <int D>
void push_elem(std::vector<u64>& w, const GlExt<D>& e) {
    for (int k = 0; k < 3; k++) w.push_back(k < D ? e.v[k] : 0);
}
template <int D>
GlExt<D> horner(const std::vector<GlExt<D>>& p, const GlExt<D>& x) {
    GlExt<D> acc = ext_zero<D>();
    for (size_t i = p.size(); i-- > 0;) acc = ext_add(ext_mul(acc, x), p[i]);
    return acc;
}

// The verdict codes of the FRI checks: WF_VERIFY_* inside a full proof, WF_FRI_VERIFY_* for a standalone FRI proof
struct FriCodes { u32 malformed, layer, fold, rem_degree, rem_fold; };
constexpr FriCodes FULL_PROOF_CODES{WF_VERIFY_MALFORMED, WF_VERIFY_FRI_LAYER, WF_VERIFY_FRI_FOLD, WF_VERIFY_FRI_REMAINDER,
                                    WF_VERIFY_FRI_REMAINDER};
constexpr FriCodes FRI_CODES{WF_FRI_VERIFY_MALFORMED, WF_FRI_VERIFY_LAYER_COMMITMENT_MISMATCH, WF_FRI_VERIFY_INVALID_LAYER_FOLDING,
                             WF_FRI_VERIFY_REMAINDER_DEGREE_MISMATCH, WF_FRI_VERIFY_INVALID_REMAINDER_FOLDING};
// The commitment indexes a layer's folded positions are opened at (map_positions_to_indexes, fri/src/utils.rs:9-33): 0 with
// idx filled, or the code of a failure
using IndexMap = std::function<u32(const std::vector<u64>& fpos, size_t row_len, std::vector<u64>& idx)>;

// The query phase of FriVerifier::verify (fri/src/verifier/mod.rs:199-331) for one proof as device work. Per layer: the rows of
// the folded positions opened against the layer's root at the indexes `index_map` gives (read_layer_queries), the current
// evaluations compared with the rows (get_query_values) and every row folded at its alpha; then the remainder's length
// against max_degree_plus_1, and its value at the final positions. `cur`: the evaluation slots of `positions`; mdp1:
// max_poly_degree + 1. verify_generic's DegreeTruncation is not planned: FriVerifier::new already refused every degree it
// would. A failure the host decides seeds `fail` and ends the plan.
template <int D>
void plan_fri(Plan& pl, int h, u32 j, u32 pidx, const FriBytes& fb, const Digest* roots, size_t N, u32 nf, u32 nl, size_t mdp1,
              const FriCodes& codes, const IndexMap& index_map, std::vector<u64> positions, std::vector<u32> cur, u32& fail) {
    const u32 nf_log = log2_ceil(nf);
    size_t dom = N;
    u32 root;
    for (u32 depth = 0; depth < nl; depth++) {
        const size_t row_len = dom / nf;
        const std::vector<u64> fpos = fold_positions(positions, row_len);
        const u32 layer = fri_layer_rank(depth);
        if (depth >= fb.fv.size()) { fail = fail_word(layer, codes.malformed); return; }   // no layer left to read
        std::vector<u64> idx;
        if (const u32 bad = index_map(fpos, row_len, idx)) { fail = fail_word(layer, bad); return; }
        std::vector<u32> refs;
        if (!pl.rows(fb.fv[depth], fpos.size(), nf * D, 0, refs) || !pl.opening(fb.fp[depth], h, row_len, idx, refs, &root)) {
            fail = fail_word(layer, codes.layer);
            return;
        }
        pl.cmps.push_back({j, fail_word(layer, codes.layer), root, pl.upload(roots[depth])});
        if (pl.folds.size() <= depth) { pl.folds.resize(depth + 1); pl.checks.resize(depth + 1); }
        std::vector<std::vector<CheckItem>> per_row(fpos.size());
        for (size_t i = 0; i < positions.size(); i++) {
            const size_t row = std::find(fpos.begin(), fpos.end(), positions[i] % row_len) - fpos.begin();
            per_row[row].push_back({cur[i], (u32)(positions[i] / row_len)});
        }
        std::vector<u32> next(fpos.size());
        const u32 log_dom = log2_ceil(dom);
        for (size_t i = 0; i < fpos.size(); i++) {
            Plan::Fold f{};
            f.it.proof = pidx; f.it.depth = depth; f.it.log_dom = log_dom; f.it.out = next[i] = pl.nevals++;
            f.it.fpos = fpos[i]; f.it.nf_log = nf_log;
            f.it.chk0 = (u32)pl.checks[depth].size(); f.it.nchk = (u32)per_row[i].size();
            pl.checks[depth].insert(pl.checks[depth].end(), per_row[i].begin(), per_row[i].end());
            f.leaf = refs[i] & REF_MASK;
            pl.folds[depth].push_back(f);
        }
        cur = next;
        positions = fpos;
        dom = row_len;
    }
    const size_t rn = fb.rem.n / (8 * D);
    for (u32 i = 0; i < nl; i++) mdp1 /= nf;   // max_degree_plus_1 after folding (verifier/mod.rs:296-300)
    if (rn > mdp1) { fail = fail_word(R_REMAINDER, codes.rem_degree); return; }
    const u32 log_dom = log2_ceil(dom);
    for (size_t i = 0; i < positions.size(); i++) pl.rems.push_back({pidx, cur[i], log_dom, 0, positions[i]});
}

// the boundary terms of one segment (verifier/src/evaluator.rs:60-83): cc (T(z) - P(z x_offset)) / (z^a - b) per assertion,
// with P the value polynomial (one value, or the interpolant of a sequence over the size-a subgroup, x_offset = g^-first_step)
template <int D>
GlExt<D> boundary_sum(const std::vector<AirAssertion>& sorted, size_t words_per_value, const GlExt<D>* cc, const GlExt<D>* t_cur,
                      const GlExt<D>& z, size_t n, u64 g) {
    GlExt<D> res = ext_zero<D>();
    for (size_t i = 0; i < sorted.size(); i++) {
        const AirAssertion& as = sorted[i];
        const size_t L = as.values.size() / words_per_value;
        std::vector<u64> flat(L * D);
        for (size_t j = 0; j < L; j++)
            for (int k = 0; k < D; k++) flat[j * D + k] = (size_t)k < words_per_value ? as.values[j * words_per_value + k] : 0;
        u64 x_off = 1;
        if (L > 1) {
            wf_host_dft(flat, L, D, true, 1);
            if (as.first_step) x_off = gl_pow(gl_inv(g), as.first_step);
        }
        std::vector<GlExt<D>> poly(L);
        for (size_t j = 0; j < L; j++) for (int k = 0; k < D; k++) poly[j].v[k] = flat[j * D + k];
        const u64 a = as.stride == 0 ? 1 : n / as.stride, b = as.first_step == 0 ? 1 : gl_pow(g, a * as.first_step);
        const GlExt<D> num = ext_mul(ext_sub(t_cur[as.column], horner<D>(poly, ext_mul_base(z, x_off))), cc[i]);
        res = ext_add(res, ext_mul(num, ext_inv(ext_sub(ext_pow(z, a), ext_from_base<D>(b)))));
    }
    return res;
}

// Air::evaluate_transition / evaluate_aux_transition through the description's programs, over E
template <int D>
void run_program(const std::vector<u32>& prog, u32 nregs, std::vector<GlExt<D>>& r, const std::vector<u64>& consts, GlExt<D>* out) {
    r.resize(std::max<size_t>(r.size(), nregs), ext_zero<D>());
    for (size_t i = 0; i + 3 < prog.size(); i += 4) {
        const u32 op = prog[i], ds = prog[i + 1], a = prog[i + 2], b = prog[i + 3];
        switch (op) {
            case 0: r[ds] = ext_add(r[a], r[b]); break;
            case 1: r[ds] = ext_sub(r[a], r[b]); break;
            case 2: r[ds] = ext_mul(r[a], r[b]); break;
            case 3: r[ds] = ext_from_base<D>(consts[a]); break;
            default: out[ds] = r[a]; break;
        }
    }
}

struct Call {
    wf_ctx* ctx;
    int hash_id;
    wf_aux_assertions_batch_fn aux_assertions;
    void* aux_user;
};

// Everything of proof j the host decides: WF_OK with fail[j] seeded (NO_FAIL or the first host-side failure) and its device
// work appended to the plan; an error only for a failing callback.
template <int D>
int host_part(const Call& call, u32 j, const AirHost& air_in, const Parsed& pp, Plan& pl, u32& fail) {
    const Options& o = pp.o;
    const int h = call.hash_id;
    AirHost air_dyn;
    if (call.aux_assertions) air_dyn = air_in;
    const AirHost& air = call.aux_assertions ? air_dyn : air_in;
    const size_t n = (size_t)1 << pp.logn;
    const u32 lb = log2_ceil(o.blowup);
    const size_t N = n << lb;
    const u32 c = air.w, aw = air.aw, ct = c + aw, kc = air.num_comp_cols(n), nl = pp.nl;
    const u32 n_mtr = (u32)air.degrees.size(), n_tr = n_mtr + (u32)air.aux_degrees.size();
    const u32 n_mas = (u32)air.asserts.size();
    const u64 g = gl_root_of_unity(pp.logn);
    const size_t nseg = aw ? 2 : 1;
    // ---- transcript (lib.rs:149-260) ----
    const std::vector<u64> seed = context_seed(air, n, o);
    PublicCoin coin(h, seed.data(), seed.size());
    coin.reseed(pp.cm[0]);
    std::vector<GlExt<D>> rnd;
    if (aw) {  // lib.rs:170-184
        for (u32 i = 0; i < air.nr; i++) rnd.push_back(draw_ext<D>(coin));
        coin.reseed(pp.cm[1]);
        if (call.aux_assertions) {  // Air::get_aux_assertions(aux_rand_elements)
            std::vector<u64> rw, vals = get_aux_assertion_words(air_dyn, D, false);
            for (auto& e : rnd) for (int k = 0; k < D; k++) rw.push_back(e.v[k]);
            if (call.aux_assertions(call.aux_user, j, rw.data(), vals.data()) != 0)
                return wf_fail(call.ctx, WF_ERR_INVALID, "proof %u: aux assertion callback failed", j);
            if (!set_aux_assertion_words(air_dyn, vals.data(), D, false)) { fail = fail_word(0, WF_VERIFY_MALFORMED); return WF_OK; }
        }
    }
    const std::vector<GlExt<D>> cc = draw_coeffs<D>(coin, o.batch_c, air.num_constraints());
    coin.reseed(pp.cm[nseg]);
    const GlExt<D> z = draw_ext<D>(coin);
    std::vector<GlExt<D>> t_cur(ct), t_nxt(ct), q_cur(kc), q_nxt(kc);
    for (u32 i = 0; i < ct; i++) { t_cur[i] = read_elem<D>(pp.ood_t.p + 1, i); t_nxt[i] = read_elem<D>(pp.ood_t.p + 1, ct + i); }
    for (u32 i = 0; i < kc; i++) { q_cur[i] = read_elem<D>(pp.ood_q.p + 1, i); q_nxt[i] = read_elem<D>(pp.ood_q.p + 1, kc + i); }
    {   // OOD consistency (verifier/src/evaluator.rs:15-80)
        std::vector<GlExt<D>> per;
        for (auto& col : air.periodic) {   // periodic column polynomials at z^(n / L)
            std::vector<u64> poly = col;
            wf_host_dft(poly, col.size(), 1, true, 1);
            const GlExt<D> x = ext_pow(z, n / col.size());
            GlExt<D> acc = ext_zero<D>();
            for (size_t i = poly.size(); i-- > 0;) { acc = ext_mul(acc, x); acc.v[0] = gl_add(acc.v[0], poly[i]); }
            per.push_back(acc);
        }
        std::vector<GlExt<D>> tev(n_tr, ext_zero<D>()), r;
        r.assign(air.num_regs, ext_zero<D>());
        for (u32 i = 0; i < c; i++) { r[i] = t_cur[i]; r[c + i] = t_nxt[i]; }
        for (size_t i = 0; i < per.size(); i++) r[2 * c + i] = per[i];
        run_program<D>(air.prog, air.num_regs, r, air.consts, tev.data());
        if (aw) {
            r.assign(air.aux_num_regs, ext_zero<D>());
            for (u32 i = 0; i < c; i++) { r[i] = t_cur[i]; r[c + i] = t_nxt[i]; }
            for (u32 i = 0; i < aw; i++) { r[2 * c + i] = t_cur[c + i]; r[2 * c + aw + i] = t_nxt[c + i]; }
            const size_t pb = 2 * c + 2 * aw;
            for (size_t i = 0; i < per.size(); i++) r[pb + i] = per[i];
            for (u32 i = 0; i < air.nr; i++) r[pb + per.size() + i] = rnd[i];
            run_program<D>(air.aux_prog, air.aux_num_regs, r, air.consts, tev.data() + n_mtr);
        }
        GlExt<D> t = ext_zero<D>();
        for (u32 i = 0; i < n_tr; i++) t = ext_add(t, ext_mul(cc[i], tev[i]));
        GlExt<D> den = ext_from_base<D>(1);   // transition divisor (x^n - 1) / prod (x - g^k), k = n - exemptions .. n - 1
        for (size_t st = n - air.exemptions; st < n; st++) den = ext_mul(den, ext_sub(z, ext_from_base<D>(gl_pow(g, st))));
        GlExt<D> res = ext_mul(t, ext_mul(den, ext_inv(ext_sub(ext_pow(z, n), ext_from_base<D>(1)))));
        res = ext_add(res, boundary_sum<D>(air.sorted_assertions(), 1, cc.data() + n_tr, t_cur.data(), z, n, g));
        if (aw) res = ext_add(res, boundary_sum<D>(air.sorted_aux_assertions(), 3, cc.data() + n_tr + n_mas, t_cur.data() + c, z, n, g));
        GlExt<D> res2 = ext_zero<D>();
        for (u32 i = 0; i < kc; i++) res2 = ext_add(res2, ext_mul(ext_pow(z, (u64)i * n), q_cur[i]));
        if (memcmp(res.v, res2.v, sizeof(res.v))) { fail = fail_word(0, WF_VERIFY_OOD); return WF_OK; }
    }
    coin.reseed(ood_frames<D>(h, t_cur, t_nxt, q_cur, q_nxt));
    const std::vector<GlExt<D>> dc = draw_coeffs<D>(coin, o.batch_d, ct + kc);
    std::vector<GlExt<D>> alphas;   // FriVerifier::new (fri/src/verifier/mod.rs:48-90)
    for (u32 i = 0; i <= nl; i++) { coin.reseed(pp.cm[nseg + 1 + i]); alphas.push_back(draw_ext<D>(coin)); }
    if (coin.check_leading_zeros(pp.nonce) < o.grinding) { fail = fail_word(0, WF_VERIFY_POW); return WF_OK; }
    std::vector<u64> pos;
    if (!query_positions(coin, o.num_queries, N, pp.nonce, pos)) { fail = fail_word(0, WF_VERIFY_MALFORMED); return WF_OK; }
    if (pos.size() != pp.nuq) { fail = fail_word(0, WF_VERIFY_MALFORMED); return WF_OK; }

    // ---- device work ----
    const u32 rn = (u32)(pp.fri.rem.n / (8 * D));
    ProofDev pd{};
    pd.d = D; pd.c = c; pd.aw = aw; pd.kc = kc; pd.log_N = pp.logn + lb; pd.rn = rn; pd.slot = j;
    pd.cst = pl.cst.size();
    {
        std::vector<u64>& w = pl.cst;
        push_elem<D>(w, z);
        push_elem<D>(w, ext_mul_base(z, g));
        for (auto& e : dc) push_elem<D>(w, e);
        for (auto* v : {&t_cur, &t_nxt, &q_cur, &q_nxt}) for (auto& e : *v) push_elem<D>(w, e);
        pd.a_off = (u32)(w.size() - pd.cst);
        for (auto& e : alphas) push_elem<D>(w, e);
        pd.r_off = (u32)(w.size() - pd.cst);
        for (u32 i = 0; i < rn; i++) push_elem<D>(w, read_elem<D>(pp.fri.rem.p, i));
    }
    const u32 pidx = (u32)pl.pds.size();
    pl.pds.push_back(pd);
    // trace / constraint queries (verifier/src/channel.rs:206-260); rows hashed in partitions (channel.rs:431-453)
    std::vector<u32> t_refs, a_refs, c_refs;
    u32 root;
    auto open = [&](const Bytes& v, const Bytes& p, u32 words, u32 part, const Digest& want, u32 rank, u32 code, std::vector<u32>& refs) {
        if (!pl.rows(v, pos.size(), words, part, refs) || !pl.opening(p, h, N, pos, refs, &root)) { fail = fail_word(rank, code); return false; }
        pl.cmps.push_back({j, fail_word(rank, code), root, pl.upload(want)});
        return true;
    };
    if (!open(pp.tq_v, pp.tq_p, c, o.part_words(c, 1), pp.cm[0], R_TRACE, WF_VERIFY_TRACE_QUERY, t_refs)) return WF_OK;
    if (aw && !open(pp.aq_v, pp.aq_p, aw * D, o.part_words(aw, D), pp.cm[1], R_AUX, WF_VERIFY_TRACE_QUERY, a_refs)) return WF_OK;
    if (!open(pp.cq_v, pp.cq_p, kc * D, o.part_words(kc, D), pp.cm[nseg], R_CONS, WF_VERIFY_CONSTRAINT_QUERY, c_refs)) return WF_OK;
    std::vector<u32> cur(pos.size());
    for (size_t i = 0; i < pos.size(); i++) {
        cur[i] = pl.nevals++;
        pl.deep.push_back({pidx, cur[i], t_refs[i] & REF_MASK, aw ? a_refs[i] & REF_MASK : 0, c_refs[i] & REF_MASK, pos[i]});
    }
    // FRI (fri/src/verifier/mod.rs:210-331). The prover commits every layer in domain order (one partition): a proof whose
    // partition count maps a folded position anywhere else cannot open its layer
    const u8 lp = pp.fri.log_parts;
    auto index_map = [lp](const std::vector<u64>& fpos, size_t row_len, std::vector<u64>& idx) -> u32 {
        if (lp) {
            if (lp >= 32) return WF_VERIFY_MALFORMED;
            const u64 P_ = (u64)1 << lp, psize = row_len / P_;
            for (u64 p : fpos)
                if ((p % P_) * psize + (p - p % P_) / P_ != p) return WF_VERIFY_FRI_LAYER;
        }
        idx = fpos;
        return 0;
    };
    plan_fri<D>(pl, h, j, pidx, pp.fri, &pp.cm[nseg + 1], N, o.folding, nl, n, FULL_PROOF_CODES, index_map, pos, cur, fail);
    return WF_OK;
}

// AcceptableOptions::OptionSet (verifier/src/lib.rs:355-359): everything ProofOptions holds
bool options_match(const Options& o, const uint32_t* words) {
    const Options a = options_from_words(words);
    return o.num_queries == a.num_queries && o.blowup == a.blowup && o.grinding == a.grinding && o.ext == a.ext && o.folding == a.folding &&
           o.rem_max_deg == a.rem_max_deg && o.batch_c == a.batch_c && o.batch_d == a.batch_d && o.num_partitions == a.num_partitions &&
           o.hash_rate == a.hash_rate;
}

size_t align2(size_t words) { return (words + 1) & ~(size_t)1; }


// One batch on the device: one upload; the leaf hashes of every opened row (one launch per row shape); one merge launch per
// tree level; the root compares; the evaluations at the queries (DEEP composition for full proofs, the caller's copied in for
// standalone FRI proofs); one FRI launch per depth; the remainder. Then, in one download and one synchronisation, the proofs'
// fail words, or with verdict_kernel their WF_VERIFY_* verdicts. fail: the words the host seeded; out: batch words.
int run_plan(wf_ctx* ctx, int hash_id, Plan& pl, const std::vector<u32>& fail, u32 batch, const FriCodes& codes, bool verdict_kernel,
             u32* out) {
    // ---- layout: [pds | cst | fail | row groups | deep | folds | checks | rems | cmps | ops | caller evaluations | uploaded
    //      digests] is uploaded, then [leaf digests | merged digests | evaluations | verdicts] ----
    const u32 U = (u32)pl.up.size(), Lf = (u32)pl.leaves.size();
    std::vector<size_t> gbase(pl.groups.size()), goff(pl.groups.size());
    size_t w = 0;
    auto take = [&](size_t words) { size_t at = w; w += align2(words); return at; };
    const size_t o_pds = take(pl.pds.size() * sizeof(ProofDev) / 8), o_cst = take(pl.cst.size()), o_fail = take((batch + 1) / 2);
    {
        size_t lb = 0;
        for (size_t g = 0; g < pl.groups.size(); g++) {
            goff[g] = take((size_t)pl.groups[g].words * pl.groups[g].rows.size());
            gbase[g] = lb;
            lb += pl.groups[g].rows.size();
        }
    }
    std::vector<size_t> fold_at(pl.folds.size());
    size_t nfold = 0, nchk = 0;
    for (size_t d = 0; d < pl.folds.size(); d++) { fold_at[d] = nfold; nfold += pl.folds[d].size(); }
    std::vector<size_t> chk_at(pl.checks.size());
    for (size_t d = 0; d < pl.checks.size(); d++) { chk_at[d] = nchk; nchk += pl.checks[d].size(); }
    std::vector<size_t> lvl_at(pl.levels.size());
    size_t nops = 0;
    for (size_t l = 0; l < pl.levels.size(); l++) { lvl_at[l] = nops; nops += pl.levels[l].size(); }
    const size_t o_deep = take(pl.deep.size() * sizeof(DeepItem) / 8), o_fold = take(nfold * sizeof(FoldItem) / 8),
                 o_chk = take(nchk * sizeof(CheckItem) / 8), o_rem = take(pl.rems.size() * sizeof(RemItem) / 8),
                 o_cmp = take(pl.cmps.size() * sizeof(CmpItem) / 8), o_ops = take((nops * sizeof(uint3) + 7) / 8),
                 o_ev0 = take(pl.ev0.size()), o_arena = take((size_t)U * 4);
    const size_t up_words = w;
    take((size_t)Lf * 4);
    take((size_t)pl.nodes * 4);
    const size_t o_evals = take((size_t)pl.nevals * 3), o_verdict = take((batch + 1) / 2);
    const size_t total = w;
    auto slot = [&](u32 ref) -> u32 {
        const u32 k = ref & REF_MASK;
        if ((ref & ~REF_MASK) == REF_UP) return k;
        if ((ref & ~REF_MASK) == REF_LEAF) return U + (u32)gbase[pl.leaves[k].first] + pl.leaves[k].second;
        return U + Lf + k;
    };
    auto row_at = [&](u32 leaf, u64* off, u32* stride) {
        const auto& L = pl.leaves[leaf];
        *off = goff[L.first] + L.second;
        *stride = (u32)pl.groups[L.first].rows.size();
    };
    CKI(pinned_reserve(ctx, (up_words + (batch + 1) / 2 + 2) * 8));
    u64* hb = (u64*)ctx->pinned;
    for (ProofDev& pd : pl.pds) pd.cst += o_cst;   // offsets into the constants become offsets into the buffer
    memcpy(hb + o_pds, pl.pds.data(), pl.pds.size() * sizeof(ProofDev));
    memcpy(hb + o_cst, pl.cst.data(), pl.cst.size() * 8);
    memcpy(hb + o_fail, fail.data(), batch * 4);
    for (size_t g = 0; g < pl.groups.size(); g++) {   // column-major: word c of row i at c * rows + i (a SegMatrix with W = 1)
        const RowGroup& G = pl.groups[g];
        const size_t rows = G.rows.size();
        for (size_t i = 0; i < rows; i++)
            for (u32 c = 0; c < G.words; c++) memcpy(hb + goff[g] + (size_t)c * rows + i, G.rows[i] + (size_t)c * 8, 8);
    }
    {
        DeepItem* di = (DeepItem*)(hb + o_deep);
        for (size_t i = 0; i < pl.deep.size(); i++) {
            const auto& e = pl.deep[i];
            DeepItem it{};
            it.proof = e.proof; it.out = e.out; it.pos = e.pos;
            row_at(e.t, &it.t_off, &it.t_st);
            if (pl.pds[e.proof].aw) row_at(e.a, &it.a_off, &it.a_st);
            row_at(e.c, &it.c_off, &it.c_st);
            di[i] = it;
        }
        FoldItem* fi = (FoldItem*)(hb + o_fold);
        for (size_t d = 0; d < pl.folds.size(); d++)
            for (size_t i = 0; i < pl.folds[d].size(); i++) {
                FoldItem it = pl.folds[d][i].it;
                it.chk0 += (u32)chk_at[d];
                row_at(pl.folds[d][i].leaf, &it.off, &it.stride);
                fi[fold_at[d] + i] = it;
            }
        CheckItem* ci = (CheckItem*)(hb + o_chk);
        for (size_t d = 0; d < pl.checks.size(); d++) memcpy(ci + chk_at[d], pl.checks[d].data(), pl.checks[d].size() * sizeof(CheckItem));
        memcpy(hb + o_rem, pl.rems.data(), pl.rems.size() * sizeof(RemItem));
        CmpItem* mi = (CmpItem*)(hb + o_cmp);
        for (size_t i = 0; i < pl.cmps.size(); i++) mi[i] = {pl.cmps[i].slot, pl.cmps[i].fail, slot(pl.cmps[i].got), slot(pl.cmps[i].want)};
        uint3* oi = (uint3*)(hb + o_ops);
        for (size_t l = 0; l < pl.levels.size(); l++)
            for (size_t i = 0; i < pl.levels[l].size(); i++) {
                const uint3 op = pl.levels[l][i];
                oi[lvl_at[l] + i] = make_uint3(slot(op.x), slot(op.y), slot(op.z));
            }
        memcpy(hb + o_ev0, pl.ev0.data(), pl.ev0.size() * 8);
        for (u32 i = 0; i < U; i++) memcpy(hb + o_arena + (size_t)i * 4, pl.up[i].b, 32);
    }
    DevScratch tmp(ctx);
    void* dbuf;
    CKI(tmp.alloc(total * 8, &dbuf));
    u64* dv = (u64*)dbuf;
    CK(cudaMemcpyAsync(dv, hb, up_words * 8, cudaMemcpyHostToDevice, ctx->st));
    u64* arena = dv + o_arena;
    u32* dfail = (u32*)(dv + o_fail);
    for (size_t g = 0; g < pl.groups.size(); g++) {   // leaf hashes, one launch per row shape
        const RowGroup& G = pl.groups[g];
        SegMatrix m{dv + goff[g], G.rows.size(), G.words, 1, G.rows.size()};
        CK(commit_hash_rows(hash_id, m, arena + (size_t)(U + gbase[g]) * 4, ctx->st, G.part));
        ctx->launches++;
    }
    for (size_t l = 0; l < pl.levels.size(); l++) {   // Merkle roots, one launch per level of the deepest tree
        CK(commit_merge_ops(hash_id, arena, (const uint3*)(dv + o_ops) + lvl_at[l], (u32)pl.levels[l].size(), ctx->st));
        ctx->launches++;
    }
    auto blocks = [](size_t count, u32 t) { return (unsigned)((count + t - 1) / t); };
    if (!pl.cmps.empty()) {
        verify_compare_kernel<<<blocks(pl.cmps.size(), 128), 128, 0, ctx->st>>>(arena, (const CmpItem*)(dv + o_cmp), (u32)pl.cmps.size(), dfail);
        ctx->launches++;
    }
    const ProofDev* dpds = (const ProofDev*)(dv + o_pds);
    u64* evals = dv + o_evals;
    if (!pl.deep.empty()) {
        verify_deep_kernel<<<blocks(pl.deep.size(), 128), 128, 0, ctx->st>>>(dpds, dv, (const DeepItem*)(dv + o_deep), (u32)pl.deep.size(), evals);
        ctx->launches++;
    }
    if (!pl.ev0.empty()) CK(cudaMemcpyAsync(evals, dv + o_ev0, pl.ev0.size() * 8, cudaMemcpyDeviceToDevice, ctx->st));
    for (size_t d = 0; d < pl.folds.size(); d++) {
        if (pl.folds[d].empty()) continue;
        verify_fri_kernel<<<blocks(pl.folds[d].size(), 128), 128, 0, ctx->st>>>(dpds, dv, (const FoldItem*)(dv + o_fold) + fold_at[d],
                                                                               (u32)pl.folds[d].size(), (const CheckItem*)(dv + o_chk), evals, dfail,
                                                                               codes.fold);
        ctx->launches++;
    }
    if (!pl.rems.empty()) {
        verify_remainder_kernel<<<blocks(pl.rems.size(), 128), 128, 0, ctx->st>>>(dpds, dv, (const RemItem*)(dv + o_rem), (u32)pl.rems.size(),
                                                                                 evals, dfail, codes.rem_fold);
        ctx->launches++;
    }
    const u32* dout = dfail;
    if (verdict_kernel) {
        u32* dverdict = (u32*)(dv + o_verdict);
        verify_verdict_kernel<<<blocks(batch, 256), 256, 0, ctx->st>>>(dfail, batch, dverdict);
        ctx->launches++;
        dout = dverdict;
    }
    CK(cudaGetLastError());
    u32* hv = (u32*)(hb + up_words);
    CK(cudaMemcpyAsync(hv, dout, batch * 4, cudaMemcpyDeviceToHost, ctx->st));
    CK(cudaStreamSynchronize(ctx->st));
    memcpy(out, hv, batch * 4);
    return WF_OK;
}


// ---- standalone FRI proofs (wf_fri_verify_batch) ----
// BatchMerkleProof::read_from (crypto/src/merkle/proofs.rs:403-423) with the bounds Plan::opening keeps, every byte used: false
// when it does not parse
bool batch_proof_depth(const Bytes& path, int hash_id, u32* depth) {
    Reader r{path.p, path.n};
    const u8 dp = r.u8_();
    const u64 nv = r.usize();
    if (!r.ok || nv > 100000 || dp < 1 || dp > 40) return false;
    const size_t dl = WF_DIGEST_BYTES(hash_id);
    for (u64 i = 0; i < nv; i++) {
        const u64 ln = r.usize();
        if (!r.ok || ln > 64 || !r.take(ln * dl)) return false;
    }
    *depth = dp;
    return r.pos == path.n;
}

struct FriShape {
    int hash_id;
    u32 nf, nl;
    size_t domain, mdp1;   // max_poly_degree.next_power_of_two() * blowup; max_poly_degree + 1
};
// (domain, number of layers) of FriVerifier::new for these options; false when a layer would have fewer than two rows (no
// Merkle tree) or the remainder no element
bool fri_shape(u32 nf, u32 rem_max_deg, u32 blowup, u64 max_poly_degree, FriShape& s) {
    if (blowup == 0 || (blowup & (blowup - 1)) || max_poly_degree >= ((u64)1 << 32)) return false;
    u64 np2 = 1;
    while (np2 < max_poly_degree) np2 <<= 1;
    if (np2 * blowup > ((u64)1 << 32)) return false;
    size_t dom = np2 * blowup;
    const size_t max_rem = ((size_t)rem_max_deg + 1) * blowup;   // FriOptions::num_fri_layers (fri/src/options.rs:85-93)
    s.nl = 0;
    while (dom > max_rem) {
        if (dom / nf < 2) return false;
        dom /= nf;
        s.nl++;
    }
    if (dom / blowup == 0) return false;
    s.nf = nf;
    s.domain = np2 * blowup;
    s.mdp1 = max_poly_degree + 1;
    return true;
}

// Everything of proof j the host decides: DefaultVerifierChannel::new's deserialization (fri/src/verifier/channel.rs:146-170,
// fri/src/proof.rs:98-146), FriVerifier::new (reseed, draw, DegreeTruncation), then the query phase through plan_fri. Its
// positions' evaluations sit in slots ev_base ... A failure the host decides seeds `fail`; one of rank 0 (deserialization,
// FriVerifier::new) also writes its verdict to `verdict`.
template <int D>
void fri_host_part(const FriShape& s, u32 j, const u8* proof, size_t len, const u8* cms, const u8* seed, const u64* positions,
                   size_t k, u32 ev_base, Plan& pl, u32& fail, u32& verdict) {
    const int h = s.hash_id;
    const u32 nf = s.nf;
    auto refuse = [&](u32 code, u32 layer = 0) { fail = fail_word(0, code); verdict = code | layer << 8; };
    Reader r{proof, len};
    FriBytes fb;
    if (!read_fri_proof(r, fb) || r.pos != len || fb.log_parts >= 64) return refuse(WF_FRI_VERIFY_MALFORMED);   // 2^64 partitions
    const size_t rn = fb.rem.n / (8 * D);   // parse_remainder
    if (fb.rem.n % (8 * D) || rn == 0 || (rn & (rn - 1)) || !all_canonical(fb.rem)) return refuse(WF_FRI_VERIFY_MALFORMED);
    size_t ds = s.domain;   // parse_layers, FriProofLayer::read_from / parse
    for (size_t i = 0; i < fb.fv.size(); i++) {
        ds /= nf;
        u32 depth;
        if (fb.fv[i].n == 0 || fb.fv[i].n % (8 * D * nf) || !all_canonical(fb.fv[i]) || !batch_proof_depth(fb.fp[i], h, &depth) ||
            ((size_t)1 << depth) != ds)
            return refuse(WF_FRI_VERIFY_MALFORMED);
    }
    // FriVerifier::new (fri/src/verifier/mod.rs:107-152)
    PublicCoin coin(h, nullptr, 0);
    if (seed) memcpy(coin.seed.b, seed, 32);
    std::vector<Digest> cm(s.nl + 1);
    for (u32 i = 0; i <= s.nl; i++) { cm[i] = Digest{}; read_digest(h, cms + 32 * i, cm[i]); }
    std::vector<GlExt<D>> alphas;
    size_t mdp1 = s.mdp1;
    for (u32 i = 0; i <= s.nl; i++) {
        coin.reseed(cm[i]);
        GlExt<D> a = ext_zero<D>();
        if (!coin.draw(D, a.v)) return refuse(WF_FRI_VERIFY_RANDOM_COIN);
        alphas.push_back(a);
        if (i != s.nl && mdp1 % nf) return refuse(WF_FRI_VERIFY_DEGREE_TRUNCATION, i);
        mdp1 /= nf;
    }
    ProofDev pd{};
    pd.d = D; pd.log_N = log2_ceil(s.domain); pd.rn = (u32)rn; pd.slot = j;
    pd.cst = pl.cst.size();
    pd.a_off = 0;
    for (auto& e : alphas) push_elem<D>(pl.cst, e);
    pd.r_off = (u32)(pl.cst.size() - pd.cst);
    for (size_t i = 0; i < rn; i++) push_elem<D>(pl.cst, read_elem<D>(fb.rem.p, i));
    const u32 pidx = (u32)pl.pds.size();
    pl.pds.push_back(pd);
    std::vector<u32> cur(k);
    for (size_t i = 0; i < k; i++) cur[i] = ev_base + (u32)i;
    const u8 lp = fb.log_parts;
    auto index_map = [lp](const std::vector<u64>& fpos, size_t row_len, std::vector<u64>& idx) -> u32 {
        idx = fpos;
        if (!lp) return 0;
        const u64 P_ = (u64)1 << lp, psize = row_len / P_;
        for (u64& q : idx) q = (q % P_) * psize + (q - q % P_) / P_;
        const std::set<u64> seen(idx.begin(), idx.end());
        return seen.size() != idx.size() || (!seen.empty() && *seen.rbegin() >= row_len) ? WF_FRI_VERIFY_MALFORMED : 0;
    };
    plan_fri<D>(pl, h, j, pidx, fb, cm.data(), s.domain, nf, s.nl, s.mdp1, FRI_CODES, index_map,
                std::vector<u64>(positions, positions + k), cur, fail);
}

// The acceptance policy of verifier::verify (AcceptableOptions, verifier/src/lib.rs:324-358): an OptionSet (opts, NULL: any
// options), or a minimum security level in bits under one regime (regime 0: none). bits (may be NULL): per proof, the bits
// the policy weighed, ~0u where the proof was refused before the check.
struct Policy {
    const uint32_t* opts = nullptr;
    u32 num_opts = 0;
    int regime = 0;
    u32 min_bits = 0;
    uint32_t* bits = nullptr;
};

int verify_air_batch(wf_ctx* ctx, uint32_t batch, const uint64_t* const* air_descs, const size_t* air_desc_lens, const uint8_t* const* proofs,
                     const size_t* proof_lens, int hash_id, const Policy& pol, wf_aux_assertions_batch_fn aux_assertions, void* aux_user,
                     uint32_t* verdicts) {
    const uint32_t* acceptable_opts = pol.opts;
    const u32 num_acceptable = pol.num_opts;
    if (!ctx || batch == 0 || !air_descs || !air_desc_lens || !proofs || !proof_lens || !verdicts || (acceptable_opts && !num_acceptable))
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    if (!WF_HASH_IS_KNOWN(hash_id)) return wf_fail(ctx, WF_ERR_UNSUPPORTED, "unknown hash %d", hash_id);
    for (u32 i = 0; acceptable_opts && i < num_acceptable; i++)
        if ((int)(acceptable_opts[9 * i + 8] & 0xff) != hash_id)
            return wf_fail(ctx, WF_ERR_INVALID, "acceptable option set %u is for hash %u, not %d", i, acceptable_opts[9 * i + 8] & 0xff, hash_id);
    // the batch rule of wf_air_batch_check, without the trace length: it comes from each proof
    std::vector<AirHost> airs(batch);
    for (u32 j = 0; j < batch; j++) {
        if (!air_descs[j] || !parse_air_host(air_descs[j], air_desc_lens[j], airs[j]))
            return wf_fail(ctx, WF_ERR_INVALID, "proof %u: malformed AIR description", j);
        if (const char* why = j ? air_structure_mismatch(airs[0], airs[j]) : nullptr)
            return wf_fail(ctx, WF_ERR_INVALID, "proof %u differs from proof 0 in its %s", j, why);
        if (!proofs[j]) return wf_fail(ctx, WF_ERR_INVALID, "proof %u: no proof bytes", j);
    }
    wf_mark(ctx, "start");
    const Call call{ctx, hash_id, aux_assertions, aux_user};
    Plan pl;
    std::vector<u32> fail(batch, NO_FAIL);
    wf_security::EstimateCache estimates;
    for (u32 j = 0; j < batch; j++) {
        if (pol.bits) pol.bits[j] = ~0u;
        Parsed pp;
        u32 v = parse_proof(airs[j], hash_id, proofs[j], proof_lens[j], pp);
        if (v == WF_VERIFY_ACCEPT && acceptable_opts) {
            bool ok = false;
            for (u32 i = 0; i < num_acceptable && !ok; i++) ok = options_match(pp.o, acceptable_opts + 9 * i);
            if (!ok) v = WF_VERIFY_UNACCEPTABLE_OPTIONS;
        }
        if (v == WF_VERIFY_ACCEPT && pol.regime) {
            // Proof::conjectured_security / proven_security (air/src/proof/mod.rs:96-126). parse_proof has checked that the
            // context's widths and constraint count are the AIR's.
            const wf_security::Estimate e = estimates.get(pp.o, (u64)1 << pp.logn, wf_security::collision_resistance(hash_id),
                                                          airs[j].num_constraints(), (u64)airs[j].w + airs[j].aw + pp.o.blowup);
            const bool conj = pol.regime == WF_SECURITY_CONJECTURED;
            if (pol.bits) pol.bits[j] = conj ? e.conjectured : std::max(e.ldr, e.udr);
            if (conj && !wf_security::conjectured_at_least(e, pol.min_bits)) v = WF_VERIFY_INSUFFICIENT_CONJECTURED_SECURITY;
            if (!conj && !wf_security::proven_at_least(e, pol.min_bits)) v = WF_VERIFY_INSUFFICIENT_PROVEN_SECURITY;
        }
        if (v == WF_VERIFY_ACCEPT) {   // Air::new at the declared length: what the reference panics on
            wf_ctx note{};
            if (air_check_host(&note, airs[j], pp.logn, pp.o.blowup) != WF_OK) v = WF_VERIFY_CONTEXT;
        }
        if (v == WF_VERIFY_ACCEPT && !values_canonical(pp)) v = WF_VERIFY_MALFORMED;
        if (v != WF_VERIFY_ACCEPT) { fail[j] = fail_word(0, v); continue; }
        int r = pp.o.ext == 1 ? host_part<1>(call, j, airs[j], pp, pl, fail[j])
              : pp.o.ext == 2 ? host_part<2>(call, j, airs[j], pp, pl, fail[j]) : host_part<3>(call, j, airs[j], pp, pl, fail[j]);
        if (r != WF_OK) return r;
    }
    wf_mark(ctx, "verify_host");

    CKI(run_plan(ctx, hash_id, pl, fail, batch, FULL_PROOF_CODES, true, verdicts));
    wf_mark(ctx, "verify_device");
    return WF_OK;
}

}  // namespace

extern "C" int wf_verify_air_batch(wf_ctx* ctx, uint32_t batch, const uint64_t* const* air_descs, const size_t* air_desc_lens,
                                   const uint8_t* const* proofs, const size_t* proof_lens, int hash_id, const uint32_t* acceptable_opts,
                                   uint32_t num_acceptable, wf_aux_assertions_batch_fn aux_assertions, void* aux_user, uint32_t* verdicts) {
    Policy pol;
    pol.opts = acceptable_opts;
    pol.num_opts = num_acceptable;
    return verify_air_batch(ctx, batch, air_descs, air_desc_lens, proofs, proof_lens, hash_id, pol, aux_assertions, aux_user, verdicts);
}

extern "C" int wf_verify_air_batch_min_security(wf_ctx* ctx, uint32_t batch, const uint64_t* const* air_descs, const size_t* air_desc_lens,
                                                const uint8_t* const* proofs, const size_t* proof_lens, int hash_id, int regime,
                                                uint32_t min_bits, wf_aux_assertions_batch_fn aux_assertions, void* aux_user,
                                                uint32_t* verdicts, uint32_t* security_bits) {
    if (regime != WF_SECURITY_CONJECTURED && regime != WF_SECURITY_PROVEN)
        return wf_fail(ctx, WF_ERR_INVALID, "unknown security regime %d", regime);
    Policy pol;
    pol.regime = regime;
    pol.min_bits = min_bits;
    pol.bits = security_bits;
    return verify_air_batch(ctx, batch, air_descs, air_desc_lens, proofs, proof_lens, hash_id, pol, aux_assertions, aux_user, verdicts);
}

extern "C" int wf_security_estimate(const uint32_t* opts, uint64_t trace_length, uint32_t collision_resistance, uint64_t num_constraints,
                                    uint64_t num_committed_polys, uint32_t* conjectured, uint32_t* proven_ldr, uint32_t* proven_udr) {
    if (!opts || !conjectured || !proven_ldr || !proven_udr) return WF_ERR_INVALID;
    Options o = options_from_words(opts);
    o.num_partitions = 1; o.hash_rate = 1;   // word 8 is not read
    if (!options_in_range(o) || o.ext < 1 || o.ext > 3) return WF_ERR_INVALID;
    if (trace_length < 8 || trace_length > ((u64)1 << 32) || (trace_length & (trace_length - 1))) return WF_ERR_INVALID;
    if (num_constraints == 0 || num_committed_polys == 0) return WF_ERR_INVALID;
    const wf_security::Estimate e = wf_security::estimate(o, trace_length, collision_resistance, num_constraints, num_committed_polys);
    *conjectured = e.conjectured;
    *proven_ldr = e.ldr;
    *proven_udr = e.udr;
    return WF_OK;
}

extern "C" int wf_proof_security(int hash_id, const uint8_t* proof, size_t len, uint32_t* conjectured, uint32_t* proven_ldr,
                                 uint32_t* proven_udr) {
    if (!proof || !conjectured || !proven_ldr || !proven_udr) return WF_ERR_INVALID;
    const u32 cr = wf_security::collision_resistance(hash_id);
    if (!WF_HASH_IS_KNOWN(hash_id) || cr == 0) return WF_ERR_UNSUPPORTED;
    Reader r{proof, len};
    ProofContext cx;
    read_context(r, hash_id, cx);
    // what Context::read_from refuses or panics on (TraceInfo::read_from and new_multi_segment, trace_info.rs:84-130,266-330;
    // an empty modulus; ProofOptions::new's ranges), and a field other than Goldilocks. The rest of the proof is not read.
    if (!cx.ok || cx.mw == 0 || (u32)cx.mw + cx.aw >= 255 || (cx.aw != 0) != (cx.ar != 0) || !cx.in_range() || cx.o.ext < 1 ||
        cx.o.ext > 3 || !cx.goldilocks())
        return WF_ERR_INVALID;
    const wf_security::Estimate e =
        wf_security::estimate(cx.o, (u64)1 << cx.logn, cr, cx.ncons, (u64)cx.mw + cx.aw + cx.o.blowup);
    *conjectured = e.conjectured;
    *proven_ldr = e.ldr;
    *proven_udr = e.udr;
    return WF_OK;
}

extern "C" int wf_fri_verify_batch(wf_ctx* ctx, int hash_id, int ext_degree, uint32_t folding_factor, uint32_t remainder_max_degree,
                                   uint32_t blowup, uint64_t max_poly_degree, uint32_t batch, const uint8_t* const* proofs,
                                   const size_t* proof_lens, const uint8_t* const* commitments, const uint32_t* num_commitments,
                                   const uint8_t* const* coin_seeds, const uint64_t* const* positions,
                                   const uint64_t* const* evaluations, const size_t* num_queries, uint32_t* verdicts) {
    if (!ctx || batch == 0 || !proofs || !proof_lens || !commitments || !num_commitments || !positions || !evaluations || !num_queries ||
        !verdicts)
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    if (!WF_HASH_IS_KNOWN(hash_id)) return wf_fail(ctx, WF_ERR_UNSUPPORTED, "unknown hash %d", hash_id);
    if (folding_factor != 2 && folding_factor != 4 && folding_factor != 8 && folding_factor != 16)
        return wf_fail(ctx, WF_ERR_UNSUPPORTED, "folding factor %u is not supported", folding_factor);
    if (ext_degree < 1 || ext_degree > 3) return wf_fail(ctx, WF_ERR_INVALID, "extension degree %d", ext_degree);
    FriShape s{};
    s.hash_id = hash_id;
    if (!fri_shape(folding_factor, remainder_max_degree, blowup, max_poly_degree, s))
        return wf_fail(ctx, WF_ERR_INVALID, "no FRI proof has this shape (blowup %u, folding %u, remainder degree %u, max degree %llu)",
                       blowup, folding_factor, remainder_max_degree, (unsigned long long)max_poly_degree);
    const u32 D = (u32)ext_degree;
    size_t total = 0;
    for (u32 j = 0; j < batch; j++) {
        if (!proofs[j] || !commitments[j]) return wf_fail(ctx, WF_ERR_INVALID, "proof %u: no proof bytes or commitments", j);
        if (num_commitments[j] != s.nl + 1)
            return wf_fail(ctx, WF_ERR_INVALID, "proof %u: %u commitments, the shape has %u layers and a remainder", j, num_commitments[j], s.nl);
        const size_t k = num_queries[j];
        if (k && (!positions[j] || !evaluations[j])) return wf_fail(ctx, WF_ERR_INVALID, "proof %u: no positions or evaluations", j);
        for (size_t i = 0; i < k; i++) {
            if (positions[j][i] >= s.domain)
                return wf_fail(ctx, WF_ERR_INVALID, "proof %u: position %llu is outside the domain of %zu", j,
                               (unsigned long long)positions[j][i], s.domain);
            for (u32 c = 0; c < D; c++)
                if (evaluations[j][i * D + c] >= GL_P) return wf_fail(ctx, WF_ERR_INVALID, "proof %u: evaluation %zu is not canonical", j, i);
        }
        total += k;
    }
    if (total >= ((size_t)1 << 31)) return wf_fail(ctx, WF_ERR_INVALID, "too many queries in one batch");
    wf_mark(ctx, "start");
    // the caller's evaluations in slots 0 .. total - 1, proof by proof; the folds' evaluations follow
    Plan pl;
    pl.ev0.assign(total * 3, 0);
    std::vector<u32> ev_base(batch);
    {
        size_t at = 0;
        for (u32 j = 0; j < batch; j++) {
            ev_base[j] = (u32)at;
            for (size_t i = 0; i < num_queries[j]; i++, at++)
                for (u32 c = 0; c < D; c++) pl.ev0[at * 3 + c] = evaluations[j][i * D + c];
        }
        pl.nevals = (u32)total;
    }
    std::vector<u32> fail(batch, NO_FAIL), host(batch, WF_FRI_VERIFY_ACCEPT);
    for (u32 j = 0; j < batch; j++) {
        const u8* seed = coin_seeds ? coin_seeds[j] : nullptr;
        const size_t k = num_queries[j];
        if (D == 1) fri_host_part<1>(s, j, proofs[j], proof_lens[j], commitments[j], seed, positions[j], k, ev_base[j], pl, fail[j], host[j]);
        else if (D == 2) fri_host_part<2>(s, j, proofs[j], proof_lens[j], commitments[j], seed, positions[j], k, ev_base[j], pl, fail[j], host[j]);
        else fri_host_part<3>(s, j, proofs[j], proof_lens[j], commitments[j], seed, positions[j], k, ev_base[j], pl, fail[j], host[j]);
    }
    wf_mark(ctx, "verify_host");
    std::vector<u32> words(batch);
    CKI(run_plan(ctx, hash_id, pl, fail, batch, FRI_CODES, false, words.data()));
    // a rank-0 word is the deserialization's or FriVerifier::new's verdict, which may carry a layer; the later words carry their
    // code, and InvalidLayerFolding its depth in the rank
    for (u32 j = 0; j < batch; j++) {
        const u32 w = words[j];
        if (w == NO_FAIL) verdicts[j] = WF_FRI_VERIFY_ACCEPT;
        else if ((w >> 4) == 0) verdicts[j] = host[j];
        else if ((w & 15u) == WF_FRI_VERIFY_INVALID_LAYER_FOLDING) verdicts[j] = WF_FRI_VERIFY_INVALID_LAYER_FOLDING | ((w >> 4) - R_FRI - 1) / 2 << 8;
        else verdicts[j] = w & 15u;
    }
    wf_mark(ctx, "verify_device");
    return WF_OK;
}
