// fri.cu — FRI commit-phase kernels (K11 in SURVEY.md §2.1): leaf hashing of the transposed layer
// and the degree-respecting projection. See fri.cuh for the reference citations.
#include "fri.cuh"
#include "internal.hpp"

#include "blake3.cuh"
#include "commit.cuh"
#include "minidft.cuh"
#include "alg_hash.cuh"

__global__ void __launch_bounds__(256) fri_hash_blake3_kernel(const u64* __restrict__ ev, size_t m, int d, int ld, int nf,
                                                              uint4* __restrict__ digests, u32 dw) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const u32 ne = (u32)(nf * d);       // <= 48 elements: a single chunk
    const u32 nblk = (ne + 7) / 8;
    u32 cv[8];
    b3_iv(cv);
    for (u32 b = 0; b < nblk; b++) {
        u32 msg[16];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            u32 e = b * 8 + k;
            u64 v = 0;
            if (e < ne) {
                u32 kk = e / d, comp = e % d;
                v = ev[(i + (size_t)kk * m) * ld + comp];
            }
            msg[2 * k] = (u32)v;
            msg[2 * k + 1] = (u32)(v >> 32);
        }
        u32 bl = min(64u, (ne - b * 8) * 8);
        u32 fl = (b == 0 ? B3_CHUNK_START : 0) | (b == nblk - 1 ? (B3_CHUNK_END | B3_ROOT) : 0);
        b3_compress(cv, msg, 0, bl, fl, b3_runtime_one());
    }
    if (dw == 6) { cv[6] = 0; cv[7] = 0; }
    digests[2 * i] = make_uint4(cv[0], cv[1], cv[2], cv[3]);
    digests[2 * i + 1] = make_uint4(cv[4], cv[5], cv[6], cv[7]);
}

template <int HASH>
__global__ void __launch_bounds__(128) fri_hash_alg_kernel(const u64* __restrict__ ev, size_t m, int d, int ld, int nf,
                                                           u64* __restrict__ digests) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const u32 ne = (u32)(nf * d);
    AlgSponge<HASH> sp;
    sp.init(ne);
    for (u32 e = 0; e < ne; e++) {
        u32 kk = e / d, comp = e % d;
        sp.absorb(ev[(i + (size_t)kk * m) * ld + comp]);
    }
    u64 o[4];
    sp.finish(o);
#pragma unroll
    for (int k = 0; k < 4; k++) digests[i * 4 + k] = o[k];
}

__host__ __device__ constexpr u32 cbrev(u32 v, int bits) {
    u32 r = 0;
    for (int i = 0; i < bits; i++) r |= ((v >> i) & 1u) << (bits - 1 - i);
    return r;
}

template <int D, int LOGNF>
__global__ void __launch_bounds__(256) fri_fold_kernel(const u64* __restrict__ ev, size_t m, int ld, GlExt<D> alpha,
                                                       const u64* __restrict__ d_alpha, const u64* __restrict__ master,
                                                       u32 logL, u64* __restrict__ next, int next_ld, size_t i0) {
    // i0: index of this launch's first row in the (global) layer of 2^logL points; `ev` holds rows i0 .. i0 + m of each
    // of the NF strided pieces back to back (the whole layer when i0 = 0 and m = 2^logL / NF)
    constexpr int NF = 1 << LOGNF;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    if (d_alpha) {  // alpha drawn by the device coin (fri_coin_kernel) instead of passed by the host
#pragma unroll
        for (int c = 0; c < D; c++) alpha.v[c] = d_alpha[c];
    }
    u64 x[D][NF];
#pragma unroll
    for (int k = 0; k < NF; k++)
#pragma unroll
        for (int c = 0; c < D; c++) x[c][k] = ev[(i + (size_t)k * m) * ld + c];
#pragma unroll
    for (int c = 0; c < D; c++) mini_dft<LOGNF>(x[c]);
    // x[c][pos] = F[bitrev(pos)], F = forward size-NF DFT; inverse coefficient j = F[(NF - j) % NF] / NF
    const u32 L = 1u << logL;
    u32 e = (L - (u32)(i + i0)) & (L - 1);
    u64 winv = (e & (L >> 1)) ? gl_neg(master[e & ((L >> 1) - 1)]) : master[e & ((L >> 1) - 1)];
    u64 xinv = gl_mul(winv, 2635249152773512046ULL);  // 7^-1 mod p
    GlExt<D> beta = ext_mul_base(alpha, xinv);
    GlExt<D> acc;
    {
        constexpr u32 pos = cbrev(1u, LOGNF);  // j = NF-1 -> forward index 1
#pragma unroll
        for (int c = 0; c < D; c++) acc.v[c] = x[c][pos];
    }
#pragma unroll
    for (int j = NF - 2; j >= 0; j--) {
        const u32 pos = cbrev((u32)((NF - j) % NF), LOGNF);
        GlExt<D> cj;
#pragma unroll
        for (int c = 0; c < D; c++) cj.v[c] = x[c][pos];
        acc = ext_add(ext_mul(acc, beta), cj);
    }
    const u64 inv_nf = GL_P - ((GL_P - 1) >> LOGNF);  // (2^LOGNF)^-1 mod p
    acc = ext_mul_base(acc, inv_nf);
#pragma unroll
    for (int c = 0; c < D; c++) next[i * next_ld + c] = acc.v[c];
    for (int c = D; c < next_ld; c++) next[i * next_ld + c] = 0;   // pad lane (next_ld = 4 for D = 3)
}

cudaError_t fri_hash_layer(int hash_id, const u64* evals, size_t len, int d, int ld, int nf, u64* digests,
                           cudaStream_t st) {
    size_t m = len / nf;
    if (WF_HASH_IS_BLAKE3(hash_id))
        fri_hash_blake3_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(evals, m, d, ld, nf,
                                                                            reinterpret_cast<uint4*>(digests), WF_DIGEST_WORDS32(hash_id));
    else if (hash_id == WF_HASH_RP64_256)
        fri_hash_alg_kernel<WF_HASH_RP64_256><<<(unsigned)((m + 127) / 128), 128, 0, st>>>(evals, m, d, ld, nf, digests);
    else if (hash_id == WF_HASH_SHA3_256)
        fri_hash_alg_kernel<WF_HASH_SHA3_256><<<(unsigned)((m + 127) / 128), 128, 0, st>>>(evals, m, d, ld, nf, digests);
    else
        fri_hash_alg_kernel<WF_HASH_RPJIVE64_256><<<(unsigned)((m + 127) / 128), 128, 0, st>>>(evals, m, d, ld, nf, digests);
    return cudaGetLastError();
}

template <int D>
static cudaError_t fold_dispatch(const u64* evals, size_t len, int ld, int nf, const u64* alpha, const u64* d_alpha,
                                 const u64* master, u64* next, int next_ld, cudaStream_t st, size_t i0, u32 logL_global) {
    size_t m = len / nf;
    const u32 logL = logL_global ? logL_global : log2_ceil(len);
    GlExt<D> a;
    for (int c = 0; c < D; c++) a.v[c] = alpha ? alpha[c] : 0;
    unsigned blocks = (unsigned)((m + 255) / 256);
    switch (nf) {
        case 2: fri_fold_kernel<D, 1><<<blocks, 256, 0, st>>>(evals, m, ld, a, d_alpha, master, logL, next, next_ld, i0); break;
        case 4: fri_fold_kernel<D, 2><<<blocks, 256, 0, st>>>(evals, m, ld, a, d_alpha, master, logL, next, next_ld, i0); break;
        case 8: fri_fold_kernel<D, 3><<<blocks, 256, 0, st>>>(evals, m, ld, a, d_alpha, master, logL, next, next_ld, i0); break;
        case 16: fri_fold_kernel<D, 4><<<blocks, 256, 0, st>>>(evals, m, ld, a, d_alpha, master, logL, next, next_ld, i0); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

cudaError_t fri_fold_layer(const u64* evals, size_t len, int d, int ld, int nf, const u64* alpha, const u64* master,
                           u64* next, int next_ld, cudaStream_t st, const u64* d_alpha, size_t i0, u32 logL_global) {
    switch (d) {
        case 1: return fold_dispatch<1>(evals, len, ld, nf, alpha, d_alpha, master, next, next_ld, st, i0, logL_global);
        case 2: return fold_dispatch<2>(evals, len, ld, nf, alpha, d_alpha, master, next, next_ld, st, i0, logL_global);
        case 3: return fold_dispatch<3>(evals, len, ld, nf, alpha, d_alpha, master, next, next_ld, st, i0, logL_global);
        default: return cudaErrorInvalidValue;
    }
}

// ---- device copy of the public coin for the FRI commit phase -----------------------------------------
// ProverChannel::commit_fri_layer + draw_fri_alpha (prover/src/channel.rs:215-234) = DefaultRandomCoin::
// reseed (crypto/src/random/default.rs:131-134: seed = merge(seed, root), counter = 0) followed by draw
// (:156-170: counter += 1, merge_with_int(seed, counter), rejection of words >= p). One thread; it lets the
// whole layer loop be enqueued without a host round trip per layer. The host replays the same steps on
// its own coin afterwards and checks that it drew the same alphas.
template <int HASH>
__device__ __forceinline__ void coin_merge(const u64 a[4], const u64 b[4], u64 out[4]) {
    if (WF_HASH_IS_BLAKE3(HASH)) {
        u32 wa[8], wb[8], cv[8];
#pragma unroll
        for (int i = 0; i < 4; i++) { wa[2 * i] = (u32)a[i]; wa[2 * i + 1] = (u32)(a[i] >> 32); wb[2 * i] = (u32)b[i]; wb[2 * i + 1] = (u32)(b[i] >> 32); }
        b3_merge_words<WF_DIGEST_WORDS32(HASH)>(wa, wb, cv);
#pragma unroll
        for (int i = 0; i < 4; i++) out[i] = (u64)cv[2 * i] | ((u64)cv[2 * i + 1] << 32);
    } else {
        u64 in[8];
#pragma unroll
        for (int i = 0; i < 4; i++) { in[i] = a[i]; in[4 + i] = b[i]; }
        alg_merge<HASH>(in, out);
    }
}
template <int HASH>
__device__ __forceinline__ void coin_merge_with_int(const u64 seed[4], u64 value, u64 out[4]) {
    if (WF_HASH_IS_BLAKE3(HASH)) {  // blake/mod.rs:41-46, :95-102
        u32 ws[8], cv[8];
#pragma unroll
        for (int i = 0; i < 4; i++) { ws[2 * i] = (u32)seed[i]; ws[2 * i + 1] = (u32)(seed[i] >> 32); }
        b3_merge_with_int_words<WF_DIGEST_WORDS32(HASH)>(ws, value, cv);
#pragma unroll
        for (int i = 0; i < 4; i++) out[i] = (u64)cv[2 * i] | ((u64)cv[2 * i + 1] << 32);
    } else {  // rp64_256/mod.rs:198-218, rp64_256_jive/mod.rs:206-229
        alg_merge_with_int<HASH>(seed, value, out);
    }
}
// state: seed[4]; log: per layer root[4] then alpha[3]
template <int HASH>  // one instantiation per hasher: the Blake3 coin does not carry the Rp64 permutation's registers
__global__ void fri_coin_kernel(u64* state, const u64* root, int d, u64* alpha_out, u64* log_entry) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    u64 seed[4], r[4], v[4];
    for (int i = 0; i < 4; i++) { seed[i] = state[i]; r[i] = root[i]; }
    coin_merge<HASH>(seed, r, seed);  // reseed
    u64 counter = 0;
    bool ok = false;
    for (int t = 0; t < 1000 && !ok; t++) {
        counter += 1;
        coin_merge_with_int<HASH>(seed, counter, v);
        ok = true;
        for (int k = 0; k < d; k++) ok = ok && v[k] < GL_P;
    }
    for (int i = 0; i < 4; i++) { state[i] = seed[i]; log_entry[i] = r[i]; }
    state[4] = counter;
    for (int k = 0; k < 3; k++) { u64 a = (ok && k < d) ? v[k] : 0; alpha_out[k] = a; log_entry[4 + k] = a; }
    log_entry[7] = ok ? 1 : 0;
}
cudaError_t fri_coin_step(int hash_id, u64* state, const u64* root, int d, u64* alpha_out, u64* log_entry, cudaStream_t st) {
    if (hash_id == WF_HASH_BLAKE3_256) fri_coin_kernel<WF_HASH_BLAKE3_256><<<1, 32, 0, st>>>(state, root, d, alpha_out, log_entry);
    else if (hash_id == WF_HASH_BLAKE3_192) fri_coin_kernel<WF_HASH_BLAKE3_192><<<1, 32, 0, st>>>(state, root, d, alpha_out, log_entry);
    else if (hash_id == WF_HASH_RP64_256) fri_coin_kernel<WF_HASH_RP64_256><<<1, 32, 0, st>>>(state, root, d, alpha_out, log_entry);
    else if (hash_id == WF_HASH_SHA3_256) fri_coin_kernel<WF_HASH_SHA3_256><<<1, 32, 0, st>>>(state, root, d, alpha_out, log_entry);
    else fri_coin_kernel<WF_HASH_RPJIVE64_256><<<1, 32, 0, st>>>(state, root, d, alpha_out, log_entry);
    return cudaGetLastError();
}
