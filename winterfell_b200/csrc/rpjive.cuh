// rpjive.cuh — Rescue Prime with the Jive compression mode, RpJive64_256, for device kernels and the host
// transcript. Follows crypto/src/hash/rescue/rp64_256_jive/mod.rs: state width 8, capacity = elements 0..4,
// rate = digest = 4..8, 7 rounds of (x^7, MDS, +ARK1, x^(1/7), MDS, +ARK2) (apply_round :321-333); the sponge
// hash_elements :240-282 (capacity[0] = 1 when the length is not a multiple of the rate, the last partial block is padded by
// OVERWRITING the next rate element with 1 and the rest with 0); merge :186-196 and merge_with_int :206-229 are NOT sponge
// calls: the 8-element input is permuted once and the digest is input[i] + input[4+i] + output[i] + output[4+i]
// (apply_jive_summation :337-350, Jive mode of eprint 2022/840); merge_many = hash_elements of the digests' elements :198-200.
// The MDS is the circulant with first row [23, 8, 13, 10, 7, 6, 21, 8] (:417; the reference multiplies through a real FFT,
// mds_f64_8x8.rs) — entries < 32, so the product is accumulated from 32-bit halves without reduction, as in rp64.cuh.
#pragma once
#include "rp64.cuh"  // rp64_exp7 / rp64_inv7_group: the S-boxes are the same maps x^7 and x^(1/7) (mod.rs:366-412)

#ifdef __CUDACC__
#define RPJ_CONST_QUAL static __device__ __constant__ const
#include "rpjive_constants.inc"
#undef RPJ_CONST_QUAL
#endif
namespace rpj_host {
#define RPJ_CONST_QUAL static const
#include "rpjive_constants.inc"
#undef RPJ_CONST_QUAL
}  // namespace rpj_host

#ifdef __CUDA_ARCH__
#define RPJ_TAB(name) name
#else
#define RPJ_TAB(name) rpj_host::name
#endif

GL_HD void rpj_mds(u64 s[8]) {
    u64 r[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        u64 lo = 0, hi = 0;  // sums of 32-bit halves times coefficients < 32: each < 2^40
#pragma unroll
        for (int j = 0; j < 8; j++) {
            u64 c = RPJ_TAB(RPJ_MDS_ROW0)[(j + 8 - i) % 8];
            lo += (s[j] & GL_EPS) * c;
            hi += (s[j] >> 32) * c;
        }
        u64 l = lo + (hi << 32);
        u64 h = (hi >> 32) + (l < lo ? 1 : 0);
        r[i] = gl_reduce128(l, h);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) s[i] = r[i];
}

GL_HD void rpj_permute(u64 s[8]) {
#pragma unroll 1
    for (int r = 0; r < 7; r++) {
#pragma unroll
        for (int i = 0; i < 8; i++) s[i] = rp64_exp7(s[i]);
        rpj_mds(s);
#pragma unroll
        for (int i = 0; i < 8; i++) s[i] = gl_add(s[i], RPJ_TAB(RPJ_ARK1)[r][i]);
#pragma unroll 1
        for (int g = 0; g < 8; g += 4) rp64_inv7_group<4>(s + g);
        rpj_mds(s);
#pragma unroll
        for (int i = 0; i < 8; i++) s[i] = gl_add(s[i], RPJ_TAB(RPJ_ARK2)[r][i]);
    }
}

// Jive compression of an 8-element state (apply_jive_summation :337-350). The input may hold any 64-bit words: the reference
// reads a digest word w >= p as w - p (ElementDigest::read_from, rp64_256_jive/digest.rs:61-69), and gl_add needs canonical
// operands, so the sum reduces its inputs first (the permutation takes any word).
GL_HD void rpj_compress(const u64 in[8], u64 out[4]) {
    u64 s[8], c[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { s[i] = in[i]; c[i] = in[i] >= GL_P ? in[i] - GL_P : in[i]; }
    rpj_permute(s);
#pragma unroll
    for (int i = 0; i < 4; i++) out[i] = gl_add(gl_add(c[i], c[4 + i]), gl_add(s[i], s[4 + i]));
}
// merge of two digests given as 8 canonical elements (:186-196)
GL_HD void rpj_merge(const u64 in[8], u64 out[4]) { rpj_compress(in, out); }
// merge_with_int (:206-229): seed in elements 0..4, value (split if >= p) in 4 / 5, the element count in 7
GL_HD void rpj_merge_with_int(const u64 seed[4], u64 value, u64 out[4]) {
    u64 s[8] = {seed[0], seed[1], seed[2], seed[3], 0, 0, 0, 0};
    if (value < GL_P) { s[4] = value; s[7] = 5; }
    else { s[4] = value - GL_P; s[5] = value / GL_P; s[7] = 6; }   // BaseElement::new(value) reduces; value / MODULUS = 1
    rpj_compress(s, out);
}

// Sponge (hash_elements :240-282) as an absorb-one-element-at-a-time state machine for kernels and the host alike
struct RpjSponge {
    u64 s[8];
    u32 i;
    GL_HD void init(size_t n) {
#pragma unroll
        for (int k = 0; k < 8; k++) s[k] = 0;
        if (n % 4 != 0) s[0] = 1;
        i = 0;
    }
    GL_HD void absorb(u64 x) {
        s[4 + i] = gl_add(s[4 + i], x);
        if (++i == 4) { rpj_permute(s); i = 0; }
    }
    GL_HD void finish(u64 out[4]) {
        if (i > 0) {
            s[4 + i] = 1;                                   // overwritten, not added (:270-277)
            for (u32 q = i + 1; q < 4; q++) s[4 + q] = 0;
            rpj_permute(s);
        }
#pragma unroll
        for (int k = 0; k < 4; k++) out[k] = s[4 + k];
    }
};
static inline void rpj_host_hash_elements(const u64* e, size_t n, u64 out[4]) {
    RpjSponge sp;
    sp.init(n);
    for (size_t k = 0; k < n; k++) sp.absorb(e[k]);
    sp.finish(out);
}
