// gl64.cuh — Goldilocks field p = 2^64 - 2^32 + 1 and its quadratic / cubic extensions, for
// sm_90a device code and for the host-side transcript code of the product.
//
// Semantics follow winter-math (reference math/src/field/f64/mod.rs): add :319, sub :339, mul :357,
// inv :157, GENERATOR = 7 :251, TWO_ADIC_ROOT_OF_UNITY :267, ext2 (x^2 - x + 2) :401-435,
// ext3 (x^3 - x - 1) :443-499. The reference stores Montgomery words (x * 2^64 mod p); the device
// works on CANONICAL words in [0, p) because the Goldilocks reduction 2^64 = 2^32 - 1, 2^96 = -1
// needs no Montgomery factor and every hash input must be canonical anyway (blake/mod.rs:52-65).
// Conversion helpers for Montgomery-form buffers crossing the C ABI are gl_from_mont / gl_to_mont.
#pragma once
#ifdef __CUDACC_RTC__  // runtime compilation of constraint kernels (jit.cu): NVRTC ships no <stdint.h>
typedef unsigned long long uint64_t;
typedef unsigned int uint32_t;
typedef unsigned char uint8_t;
#else
#include <stdint.h>
#endif

#ifdef __CUDACC__
#define GL_HD __host__ __device__ __forceinline__
#else
#define GL_HD inline
#endif

typedef uint64_t u64;
typedef uint32_t u32;
typedef uint8_t u8;

#define GL_P 0xffffffff00000001ULL
#define GL_EPS 0xffffffffULL
#define GL_GENERATOR 7ULL
#define GL_TWO_ADIC_ROOT 7277203076849721926ULL

// ---- host reference forms (also what the device forms compute) -------------------------------
static inline u64 gl_add_host(u64 a, u64 b) {
    u64 r = a + b;
    // a, b < p: a + b < 2p; wrapped (carry) or >= p  =>  subtract p (== add 2^32 - 1 mod 2^64)
    if (r < a || r >= GL_P) r += GL_EPS;
    return r;
}
static inline u64 gl_sub_host(u64 a, u64 b) {
    u64 r = a - b;
    if (a < b) r -= GL_EPS;  // + p == - (2^32 - 1) mod 2^64
    return r;
}
// lo + 2^64 * hi  mod p, canonical result
static inline u64 gl_reduce128_host(u64 lo, u64 hi) {
    u64 hh = hi >> 32, hl = hi & GL_EPS;
    u64 t = lo - hh;
    if (lo < hh) t -= GL_EPS;
    u64 m = (hl << 32) - hl;  // hl * (2^32 - 1)
    u64 r = t + m;
    if (r < m) r += GL_EPS;
    if (r >= GL_P) r -= GL_P;
    return r;
}

#if defined(__CUDACC__) && !defined(GL_LITERAL_EPS)
// 2^32 - 1 as a constant-bank operand ptxas cannot fold: with the literal, "x * 0xffffffff + y" is strength-reduced to
// IMAD.IADD + IMAD.HI.U32 (the latter a half-rate instruction of the FMA pipe); with an opaque multiplier the
// mad.lo.cc / madc.hi.cc pair becomes ONE IMAD.WIDE.U32 with a carry-out predicate.
static __constant__ u32 GL_EPS_CONST = 0xffffffffu;
#define GL_EPS_OPERAND , "r"(GL_EPS_CONST)
#define GL_EPSM(n) "%" #n
#else
#define GL_EPS_OPERAND
#define GL_EPSM(n) "0xffffffff"
#endif
#ifdef __CUDA_ARCH__
// ---- device forms: explicit carry chains (ncu on the first version showed 35% of all issued
// instructions were ISETP/SEL pairs from the C conditionals above, on the saturated ALU pipe) ----
// a - b for a < p, b <= p: canonical result. 5 ALU instructions.
__device__ __forceinline__ u64 gl_sub(u64 a, u64 b) {
    u64 r;
    asm("{\n\t"
        ".reg .u32 a0, a1, b0, b1, m;\n\t"
        "mov.b64 {a0, a1}, %1;\n\t"
        "mov.b64 {b0, b1}, %2;\n\t"
        "sub.cc.u32 a0, a0, b0;\n\t"
        "subc.cc.u32 a1, a1, b1;\n\t"
        "subc.u32 m, 0, 0;\n\t"          // m = -borrow
        "sub.cc.u32 a0, a0, m;\n\t"      // borrow: r -= 2^32 - 1  (lo += 1, hi -= 1 - carry)
        "subc.u32 a1, a1, 0;\n\t"
        "mov.b64 %0, {a0, a1};\n\t"
        "}"
        : "=l"(r)
        : "l"(a), "l"(b));
    return r;
}
// a + b = a - (p - b): 7 ALU instructions, canonical for a, b < p.
__device__ __forceinline__ u64 gl_add(u64 a, u64 b) {
    u64 r;
    asm("{\n\t"
        ".reg .u32 a0, a1, b0, b1, m;\n\t"
        "mov.b64 {a0, a1}, %1;\n\t"
        "mov.b64 {b0, b1}, %2;\n\t"
        "sub.cc.u32 b0, 1, b0;\n\t"             // p - b, p = 0xffffffff_00000001
        "subc.u32 b1, 0xffffffff, b1;\n\t"
        "sub.cc.u32 a0, a0, b0;\n\t"
        "subc.cc.u32 a1, a1, b1;\n\t"
        "subc.u32 m, 0, 0;\n\t"
        "sub.cc.u32 a0, a0, m;\n\t"
        "subc.u32 a1, a1, 0;\n\t"
        "mov.b64 %0, {a0, a1};\n\t"
        "}"
        : "=l"(r)
        : "l"(a), "l"(b));
    return r;
}
// (a, b) -> (a + b, a - b), sharing the operand unpacking. The sum is folded as in gl_reduce128: U = a + b = carry 2^64 + r
// (U < 2p), U >= p exactly when carry or r + (2^32 - 1) carries (never both), and then U - p = r + (2^32 - 1) mod 2^64, applied
// by one IMAD.WIDE. The NTT rounds are bound by the integer ALU pipe, and this form moves the sum's work to the FMA pipe: the
// sum is 5 ALU + 2 FMA-pipe instructions (the gl_add form, a - (p - b), was 7 + 1), the difference 4 + 1 as in gl_sub.
__device__ __forceinline__ void gl_butterfly(u64& a, u64& b) {
    u64 s, d;
    asm("{\n\t"
        ".reg .u32 a0, a1, b0, b1, s0, s1, t0, t1, k, m;\n\t"
        "mov.b64 {a0, a1}, %2;\n\t"
        "mov.b64 {b0, b1}, %3;\n\t"
        "add.cc.u32 s0, a0, b0;\n\t"
        "addc.cc.u32 s1, a1, b1;\n\t"
        "addc.u32 k, 0, 0;\n\t"
        "add.cc.u32 t0, s0, 0xffffffff;\n\t"
        "addc.cc.u32 t1, s1, 0;\n\t"
        "addc.u32 k, k, 0;\n\t"
        "mad.lo.cc.u32 s0, k, " GL_EPSM(4) ", s0;\n\t"
        "madc.hi.u32 s1, k, " GL_EPSM(4) ", s1;\n\t"
        "mov.b64 %0, {s0, s1};\n\t"
        "sub.cc.u32 a0, a0, b0;\n\t"
        "subc.cc.u32 a1, a1, b1;\n\t"
        "subc.u32 m, 0, 0;\n\t"
        "sub.cc.u32 a0, a0, m;\n\t"
        "subc.u32 a1, a1, 0;\n\t"
        "mov.b64 %1, {a0, a1};\n\t"
        "}"
        : "=l"(s), "=l"(d)
        : "l"(a), "l"(b) GL_EPS_OPERAND);
    a = s;
    b = d;
}
// r in [0, 2^64) -> [0, p): r >= p exactly when hi = 2^32 - 1 and lo >= 1, i.e. when r + (2^32 - 1)
// carries out of 64 bits; then r - p = (lo - 1, 0) = (lo - carry, hi + carry). Two carry-only adds, the
// carry bit (IMAD.X) and two 32-bit adds. (One add chain only: PTX's CC.CF after add.cc must not be fed
// to subc — ptxas implements sub chains with the inverted flag.) The compare/branch form of this step
// was if-converted by ptxas into 6-7 ALU instructions, a large share of all instructions the NTT issued.
__device__ __forceinline__ u64 gl_canon(u64 r) {
    u64 o;
    asm("{\n\t"
        ".reg .u32 r0, r1, t0, t1, k;\n\t"
        "mov.b64 {r0, r1}, %1;\n\t"
        "add.cc.u32 t0, r0, 0xffffffff;\n\t"
        "addc.cc.u32 t1, r1, 0;\n\t"
        "addc.u32 k, 0, 0;\n\t"
        "sub.u32 r0, r0, k;\n\t"
        "add.u32 r1, r1, k;\n\t"
        "mov.b64 %0, {r0, r1};\n\t"
        "}"
        : "=l"(o)
        : "l"(r));
    return o;
}
// lo + 2^64 hi mod p, canonical: V = x0 + 2^32 x1 + (2^32 - 1) x2 - x3 in two one-sided steps (the order of
// reduce128 in math/src/field/f64/mod.rs:714-730 mont_red_cst's Goldilocks analogue):
//   t = (x1:x0) - x3; a borrow is repaid with - (2^32 - 1) (t + p: cannot borrow twice, t_wrapped >= 2^64 - 2^32 + 1);
//   U = t + x2 * (2^32 - 1) < 2p as carry * 2^64 + r; U >= p exactly when carry or r + (2^32 - 1) carries (never
//   both), and then U - p = r + (2^32 - 1) mod 2^64. One add chain decides, one IMAD.WIDE applies it.
// 12 SASS instructions; the first version (carry - borrow as a signed adjustment, then a separate canonicalisation)
// compiled to 17.
__device__ __forceinline__ u64 gl_reduce128(u64 lo, u64 hi) {
    u64 r;
    asm("{\n\t"
        ".reg .u32 c0, c1, c2, c3, k, m, t0, t1;\n\t"
        "mov.b64 {c0, c1}, %1;\n\t"
        "mov.b64 {c2, c3}, %2;\n\t"
        "sub.cc.u32 c0, c0, c3;\n\t"
        "subc.cc.u32 c1, c1, 0;\n\t"
        "subc.u32 m, 0, 0;\n\t"
        "sub.cc.u32 c0, c0, m;\n\t"
        "subc.u32 c1, c1, 0;\n\t"
        "mad.lo.cc.u32 c0, c2, " GL_EPSM(3) ", c0;\n\t"
        "madc.hi.cc.u32 c1, c2, " GL_EPSM(3) ", c1;\n\t"
        "addc.u32 k, 0, 0;\n\t"
        "add.cc.u32 t0, c0, 0xffffffff;\n\t"
        "addc.cc.u32 t1, c1, 0;\n\t"
        "addc.u32 k, k, 0;\n\t"
        "mad.lo.cc.u32 c0, k, " GL_EPSM(3) ", c0;\n\t"
        "madc.hi.u32 c1, k, " GL_EPSM(3) ", c1;\n\t"
        "mov.b64 %0, {c0, c1};\n\t"
        "}"
        : "=l"(r)
        : "l"(lo), "l"(hi) GL_EPS_OPERAND);
    return r;
}
// 64 x 64 -> 128 as even columns (a0 b0 | a1 b1) plus the odd column a0 b1 + a1 b0 shifted by 32 (ptxas turns the
// mul.lo / mul.hi pairs into IMAD.WIDE.U32 with carry predicates), fused with the reduction above: ~20 SASS
// instructions, canonical result.
__device__ __forceinline__ u64 gl_mul(u64 a, u64 b) {
    u64 r;
    asm("{\n\t"
        ".reg .u32 a0, a1, b0, b1, c0, c1, c2, c3, o0, o1, o2, k, m, t0, t1;\n\t"
        "mov.b64 {a0, a1}, %1;\n\t"
        "mov.b64 {b0, b1}, %2;\n\t"
        "mul.lo.u32 c0, a0, b0;\n\t"
        "mul.hi.u32 c1, a0, b0;\n\t"
        "mul.lo.u32 c2, a1, b1;\n\t"
        "mul.hi.u32 c3, a1, b1;\n\t"
        "mul.lo.u32 o0, a0, b1;\n\t"
        "mul.hi.u32 o1, a0, b1;\n\t"
        "mad.lo.cc.u32 o0, a1, b0, o0;\n\t"
        "madc.hi.cc.u32 o1, a1, b0, o1;\n\t"
        "addc.u32 o2, 0, 0;\n\t"
        "add.cc.u32 c1, c1, o0;\n\t"
        "addc.cc.u32 c2, c2, o1;\n\t"
        "addc.u32 c3, c3, o2;\n\t"
        "sub.cc.u32 c0, c0, c3;\n\t"
        "subc.cc.u32 c1, c1, 0;\n\t"
        "subc.u32 m, 0, 0;\n\t"
        "sub.cc.u32 c0, c0, m;\n\t"
        "subc.u32 c1, c1, 0;\n\t"
        "mad.lo.cc.u32 c0, c2, " GL_EPSM(3) ", c0;\n\t"
        "madc.hi.cc.u32 c1, c2, " GL_EPSM(3) ", c1;\n\t"
        "addc.u32 k, 0, 0;\n\t"
        "add.cc.u32 t0, c0, 0xffffffff;\n\t"
        "addc.cc.u32 t1, c1, 0;\n\t"
        "addc.u32 k, k, 0;\n\t"
        "mad.lo.cc.u32 c0, k, " GL_EPSM(3) ", c0;\n\t"
        "madc.hi.u32 c1, k, " GL_EPSM(3) ", c1;\n\t"
        "mov.b64 %0, {c0, c1};\n\t"
        "}"
        : "=l"(r)
        : "l"(a), "l"(b) GL_EPS_OPERAND);
    return r;
}
// a * b for ANY 64-bit words a, b (canonical or not), result congruent to the product but only below 2^64, not below p:
// gl_mul without its last step. U = t + c2 (2^32 - 1) = carry 2^64 + r with r < 2^64 - 2^33 + 1 when carry is set, so
// r + carry (2^32 - 1) cannot carry again. For chains of multiplications (the Rescue S-boxes: 76 per element and round)
// whose end is canonicalised by whatever consumes it; 3 instructions fewer than gl_mul.
__device__ __forceinline__ u64 gl_mul_weak(u64 a, u64 b) {
    u64 r;
    asm("{\n\t"
        ".reg .u32 a0, a1, b0, b1, c0, c1, c2, c3, o0, o1, o2, k, m;\n\t"
        "mov.b64 {a0, a1}, %1;\n\t"
        "mov.b64 {b0, b1}, %2;\n\t"
        "mul.lo.u32 c0, a0, b0;\n\t"
        "mul.hi.u32 c1, a0, b0;\n\t"
        "mul.lo.u32 c2, a1, b1;\n\t"
        "mul.hi.u32 c3, a1, b1;\n\t"
        "mul.lo.u32 o0, a0, b1;\n\t"
        "mul.hi.u32 o1, a0, b1;\n\t"
        "mad.lo.cc.u32 o0, a1, b0, o0;\n\t"
        "madc.hi.cc.u32 o1, a1, b0, o1;\n\t"
        "addc.u32 o2, 0, 0;\n\t"
        "add.cc.u32 c1, c1, o0;\n\t"
        "addc.cc.u32 c2, c2, o1;\n\t"
        "addc.u32 c3, c3, o2;\n\t"
        "sub.cc.u32 c0, c0, c3;\n\t"
        "subc.cc.u32 c1, c1, 0;\n\t"
        "subc.u32 m, 0, 0;\n\t"
        "sub.cc.u32 c0, c0, m;\n\t"
        "subc.u32 c1, c1, 0;\n\t"
        "mad.lo.cc.u32 c0, c2, " GL_EPSM(3) ", c0;\n\t"
        "madc.hi.cc.u32 c1, c2, " GL_EPSM(3) ", c1;\n\t"
        "addc.u32 k, 0, 0;\n\t"
        "mad.lo.cc.u32 c0, k, " GL_EPSM(3) ", c0;\n\t"
        "madc.hi.u32 c1, k, " GL_EPSM(3) ", c1;\n\t"
        "mov.b64 %0, {c0, c1};\n\t"
        "}"
        : "=l"(r)
        : "l"(a), "l"(b) GL_EPS_OPERAND);
    return r;
}
// a * a for any 64-bit word, weakly reduced like gl_mul_weak. Written with mul.wide so that the three partial products are
// three IMAD.WIDE: from the mul.lo / mul.hi form ptxas builds a square out of IMAD + IMAD.HI pairs, and IMAD.HI occupies the
// FMA-heavy pipe more than twice as long as IMAD.WIDE. The cross product is doubled on the ALU pipe. On the earlier build the
// bound only moved to the ALU pipe and this form was not faster, so it is an option (RP64_SQR_WIDE), not the default.
__device__ __forceinline__ u64 gl_sqr_weak(u64 a) {
    u64 r;
    asm("{\n\t"
        ".reg .u32 a0, a1, c0, c1, c2, c3, o0, o1, o2, k, m;\n\t"
        ".reg .u64 w;\n\t"
        "mov.b64 {a0, a1}, %1;\n\t"
        "mul.wide.u32 w, a0, a0;\n\t"
        "mov.b64 {c0, c1}, w;\n\t"
        "mul.wide.u32 w, a1, a1;\n\t"
        "mov.b64 {c2, c3}, w;\n\t"
        "mul.wide.u32 w, a0, a1;\n\t"
        "mov.b64 {o0, o1}, w;\n\t"
        "add.cc.u32 o0, o0, o0;\n\t"          // 2 a0 a1 < 2^65
        "addc.cc.u32 o1, o1, o1;\n\t"
        "addc.u32 o2, 0, 0;\n\t"
        "add.cc.u32 c1, c1, o0;\n\t"
        "addc.cc.u32 c2, c2, o1;\n\t"
        "addc.u32 c3, c3, o2;\n\t"
        "sub.cc.u32 c0, c0, c3;\n\t"
        "subc.cc.u32 c1, c1, 0;\n\t"
        "subc.u32 m, 0, 0;\n\t"
        "sub.cc.u32 c0, c0, m;\n\t"
        "subc.u32 c1, c1, 0;\n\t"
        "mad.lo.cc.u32 c0, c2, " GL_EPSM(2) ", c0;\n\t"
        "madc.hi.cc.u32 c1, c2, " GL_EPSM(2) ", c1;\n\t"
        "addc.u32 k, 0, 0;\n\t"
        "mad.lo.cc.u32 c0, k, " GL_EPSM(2) ", c0;\n\t"
        "madc.hi.u32 c1, k, " GL_EPSM(2) ", c1;\n\t"
        "mov.b64 %0, {c0, c1};\n\t"
        "}"
        : "=l"(r)
        : "l"(a) GL_EPS_OPERAND);
    return r;
}
// x * 2^K for a compile-time K < 96 and canonical x, written on the three words y = x << (K mod 32) (y2 < 2^(K mod 32)):
//   K < 32      : (y1:y0) + (2^32 - 1) y2                      -> carry * 2^64 + r < 2p, folded as in gl_reduce128 (11 instr.)
//   32 <= K < 64: 2^32 y0 + (2^32 - 1) y1 - y2 = ((y0:0) - y2, a borrow repaid with -(2^32 - 1)) + (2^32 - 1) y1 -> fold
//   64 <= K < 96: (2^32 - 1) y0 - (y2:y1) (2^96 = -1, 2^128 = -2^32): below p already, a borrow repaid with -(2^32 - 1):
//                 canonical without a fold (9 instr. with (2^32 - 1) y0 as one IMAD.WIDE; the first version went through two
//                 128-bit reductions: 45)
template <int K>
__device__ __forceinline__ u64 gl_shl_dev(u64 x) {
    constexpr int R = K & 31;
    const u32 x0 = (u32)x, x1 = (u32)(x >> 32);
    const u32 y0 = x0 << R, y1 = R ? __funnelshift_l(x0, x1, R) : x1, y2 = R ? (x1 >> ((32 - R) & 31)) : 0;
    u64 o;
    if (K < 32) {
        asm("{\n\t"
            ".reg .u32 r0, r1, k, t0, t1;\n\t"
            "mad.lo.cc.u32 r0, %3, " GL_EPSM(4) ", %1;\n\t"
            "madc.hi.cc.u32 r1, %3, " GL_EPSM(4) ", %2;\n\t"
            "addc.u32 k, 0, 0;\n\t"
            "add.cc.u32 t0, r0, 0xffffffff;\n\t"
            "addc.cc.u32 t1, r1, 0;\n\t"
            "addc.u32 k, k, 0;\n\t"
            "mad.lo.cc.u32 r0, k, " GL_EPSM(4) ", r0;\n\t"
            "madc.hi.u32 r1, k, " GL_EPSM(4) ", r1;\n\t"
            "mov.b64 %0, {r0, r1};\n\t"
            "}" : "=l"(o) : "r"(y0), "r"(y1), "r"(y2) GL_EPS_OPERAND);
    } else if (K < 64) {
        asm("{\n\t"
            ".reg .u32 r0, r1, k, m, t0, t1;\n\t"
            "sub.cc.u32 r0, 0, %3;\n\t"                 // (y0 : 0) - y2
            "subc.cc.u32 r1, %1, 0;\n\t"
            "subc.u32 m, 0, 0;\n\t"
            "sub.cc.u32 r0, r0, m;\n\t"
            "subc.u32 r1, r1, 0;\n\t"
            "mad.lo.cc.u32 r0, %2, " GL_EPSM(4) ", r0;\n\t"  // + y1 * (2^32 - 1)
            "madc.hi.cc.u32 r1, %2, " GL_EPSM(4) ", r1;\n\t"
            "addc.u32 k, 0, 0;\n\t"
            "add.cc.u32 t0, r0, 0xffffffff;\n\t"
            "addc.cc.u32 t1, r1, 0;\n\t"
            "addc.u32 k, k, 0;\n\t"
            "mad.lo.cc.u32 r0, k, " GL_EPSM(4) ", r0;\n\t"
            "madc.hi.u32 r1, k, " GL_EPSM(4) ", r1;\n\t"
            "mov.b64 %0, {r0, r1};\n\t"
            "}" : "=l"(o) : "r"(y0), "r"(y1), "r"(y2) GL_EPS_OPERAND);
    } else {
        asm("{\n\t"
            ".reg .u32 m0, m1, b;\n\t"
            ".reg .u64 w;\n\t"
            "mul.wide.u32 w, %1, " GL_EPSM(4) ";\n\t"    // one IMAD.WIDE (mul.lo / mul.hi: IMAD + IMAD.HI)
            "mov.b64 {m0, m1}, w;\n\t"
            "sub.cc.u32 m0, m0, %2;\n\t"
            "subc.cc.u32 m1, m1, %3;\n\t"
            "subc.u32 b, 0, 0;\n\t"
            "sub.cc.u32 m0, m0, b;\n\t"
            "subc.u32 m1, m1, 0;\n\t"
            "mov.b64 %0, {m0, m1};\n\t"
            "}" : "=l"(o) : "r"(y0), "r"(y1), "r"(y2) GL_EPS_OPERAND);
    }
    return o;
}
#else
GL_HD u64 gl_add(u64 a, u64 b) { return gl_add_host(a, b); }
GL_HD u64 gl_sub(u64 a, u64 b) { return gl_sub_host(a, b); }
GL_HD u64 gl_reduce128(u64 lo, u64 hi) { return gl_reduce128_host(lo, hi); }
GL_HD u64 gl_mul(u64 a, u64 b) {
    unsigned __int128 x = (unsigned __int128)a * b;
    return gl_reduce128((u64)x, (u64)(x >> 64));
}
GL_HD u64 gl_mul_weak(u64 a, u64 b) { return gl_mul(a, b); }   // the host form is canonical anyway
GL_HD u64 gl_sqr_weak(u64 a) { return gl_mul(a, a); }
static inline void gl_butterfly(u64& a, u64& b) {
    u64 s = gl_add(a, b);
    b = gl_sub(a, b);
    a = s;
}
#endif
#ifdef __CUDACC__
// Delayed-reduction dot products: a 160-bit unsigned accumulator of full 64x64-bit products (room for 2^32 of them),
// reduced once. One multiply-accumulate is ~9 SASS instructions (4 IMAD.WIDE + the carry chain) against ~33 for
// gl_mul + gl_add; used wherever a row of base-field values meets a row of coefficients (constraint combination,
// DEEP composition, out-of-domain evaluation).
struct GlAcc {
    u32 w0, w1, w2, w3, w4;
};
__device__ __forceinline__ GlAcc acc_zero() { return GlAcc{0, 0, 0, 0, 0}; }
__device__ __forceinline__ void acc_mad(GlAcc& a, u64 x, u64 y) {
    asm("{\n\t"
        ".reg .u32 x0, x1, y0, y1, m0, m1, m2;\n\t"
        "mov.b64 {x0, x1}, %5;\n\t"
        "mov.b64 {y0, y1}, %6;\n\t"
        "mul.lo.u32 m0, x0, y1;\n\t"
        "mul.hi.u32 m1, x0, y1;\n\t"
        "mad.lo.cc.u32 m0, x1, y0, m0;\n\t"
        "madc.hi.cc.u32 m1, x1, y0, m1;\n\t"
        "addc.u32 m2, 0, 0;\n\t"
        "mad.lo.cc.u32 %0, x0, y0, %0;\n\t"
        "madc.hi.cc.u32 %1, x0, y0, %1;\n\t"
        "madc.lo.cc.u32 %2, x1, y1, %2;\n\t"
        "madc.hi.cc.u32 %3, x1, y1, %3;\n\t"
        "addc.u32 %4, %4, 0;\n\t"
        "add.cc.u32 %1, %1, m0;\n\t"
        "addc.cc.u32 %2, %2, m1;\n\t"
        "addc.cc.u32 %3, %3, m2;\n\t"
        "addc.u32 %4, %4, 0;\n\t"
        "}"
        : "+r"(a.w0), "+r"(a.w1), "+r"(a.w2), "+r"(a.w3), "+r"(a.w4)
        : "l"(x), "l"(y));
}
// w0 + 2^32 w1 + 2^64 w2 + 2^96 w3 + 2^128 w4 mod p, canonical; 2^128 = -2^32 (mod p). w4 < 2^32 - 1 (fewer than
// 2^31 accumulated products), so (w4 << 32) is a canonical word.
__device__ __forceinline__ u64 acc_reduce(const GlAcc& a) {
    const u64 t = gl_reduce128((u64)a.w0 | ((u64)a.w1 << 32), (u64)a.w2 | ((u64)a.w3 << 32));
    return gl_sub(t, (u64)a.w4 << 32);
}
#endif
GL_HD u64 gl_neg(u64 a) { return a ? GL_P - a : 0; }
GL_HD u64 gl_dbl(u64 a) { return gl_add(a, a); }
GL_HD u64 gl_sqr(u64 a) { return gl_mul(a, a); }

// x * 2^k mod p for a compile-time k in [0, 96]: the twiddles of DFTs of size <= 64 are powers
// of two (w_64 = 8, w_32 = 64, w_16 = 2^12, w_8 = 2^24, w_4 = 2^48, w_2 = 2^96 = -1), so the inner
// butterflies of the radix-8/16 NTT rounds need no 64x64 multiplier.
template <int K>
GL_HD u64 gl_mul_2exp(u64 x) {
    if (K == 0) return x;
    if (K == 96) return gl_neg(x);
#ifdef __CUDA_ARCH__
    return gl_shl_dev<K>(x);
#else
    if (K < 64) return gl_reduce128(x << (K & 63), x >> ((64 - K) & 63));
    // 64 <= K < 96: x * 2^K = (x << (K - 64)) * 2^64; let y = x << (K-64) = yl + 2^64 yh (yh < 2^32)
    // => yl * 2^64 + yh * 2^128, and 2^128 = -2^32 (mod p).
    u64 yl = x << ((K - 64) & 63), yh = (K == 64) ? 0 : (x >> ((128 - K) & 63));
    u64 r = gl_reduce128(0, yl);
    return gl_sub(r, gl_reduce128(yh << 32, 0));
#endif
}

GL_HD u64 gl_pow(u64 a, u64 e) {
    u64 r = 1;
    while (e) {
        if (e & 1) r = gl_mul(r, a);
        a = gl_mul(a, a);
        e >>= 1;
    }
    return r;
}
// a^(p-2) with p - 2 = (2^32 - 2) * 2^32 + (2^32 - 1): 63 squarings + 10 multiplications
// (instead of 125 for square-and-multiply). inv(0) = 0 as in f64/mod.rs:157.
GL_HD u64 gl_sqr_n(u64 a, int n) {
    for (int i = 0; i < n; i++) a = gl_sqr(a);
    return a;
}
GL_HD u64 gl_inv(u64 x) {
    u64 e2 = gl_mul(gl_sqr(x), x);              // x^(2^2 - 1)
    u64 e4 = gl_mul(gl_sqr_n(e2, 2), e2);       // x^(2^4 - 1)
    u64 e8 = gl_mul(gl_sqr_n(e4, 4), e4);       // x^(2^8 - 1)
    u64 e16 = gl_mul(gl_sqr_n(e8, 8), e8);      // x^(2^16 - 1)
    u64 e24 = gl_mul(gl_sqr_n(e16, 8), e8);     // x^(2^24 - 1)
    u64 e28 = gl_mul(gl_sqr_n(e24, 4), e4);     // x^(2^28 - 1)
    u64 e30 = gl_mul(gl_sqr_n(e28, 2), e2);     // x^(2^30 - 1)
    u64 e31 = gl_mul(gl_sqr(e30), x);           // x^(2^31 - 1)
    u64 a2 = gl_sqr(e31);                       // x^(2^32 - 2)
    u64 b = gl_mul(a2, x);                      // x^(2^32 - 1)
    return gl_mul(gl_sqr_n(a2, 32), b);         // x^((2^32 - 2) 2^32 + 2^32 - 1) = x^(p - 2); 0 -> 0
}
GL_HD u64 gl_root_of_unity(u32 log_n) { return gl_pow(GL_TWO_ADIC_ROOT, 1ULL << (32 - log_n)); }
// Montgomery words (x * 2^64 mod p, f64/mod.rs:57-83) <-> canonical: (2^64)^-1 = 18446744065119617025,
// 2^64 = 2^32 - 1 (mod p).
GL_HD u64 gl_from_mont(u64 m) { return gl_mul(m, 18446744065119617025ULL); }
GL_HD u64 gl_to_mont(u64 x) { return gl_mul(x, GL_EPS); }

// ---------------------------------------------------------------------------------------------
// Extension elements: D consecutive base elements (extensions/cubic.rs:117-121).
// ---------------------------------------------------------------------------------------------
template <int D>
struct GlExt {
    u64 v[D];
};

template <int D>
GL_HD GlExt<D> ext_zero() {
    GlExt<D> r;
#pragma unroll
    for (int i = 0; i < D; i++) r.v[i] = 0;
    return r;
}
template <int D>
GL_HD GlExt<D> ext_from_base(u64 b) {
    GlExt<D> r = ext_zero<D>();
    r.v[0] = b;
    return r;
}
template <int D>
GL_HD GlExt<D> ext_add(const GlExt<D>& a, const GlExt<D>& b) {
    GlExt<D> r;
#pragma unroll
    for (int i = 0; i < D; i++) r.v[i] = gl_add(a.v[i], b.v[i]);
    return r;
}
template <int D>
GL_HD GlExt<D> ext_sub(const GlExt<D>& a, const GlExt<D>& b) {
    GlExt<D> r;
#pragma unroll
    for (int i = 0; i < D; i++) r.v[i] = gl_sub(a.v[i], b.v[i]);
    return r;
}
template <int D>
GL_HD GlExt<D> ext_mul_base(const GlExt<D>& a, u64 b) {
    GlExt<D> r;
#pragma unroll
    for (int i = 0; i < D; i++) r.v[i] = gl_mul(a.v[i], b);
    return r;
}
GL_HD GlExt<1> ext_mul(const GlExt<1>& a, const GlExt<1>& b) {
    GlExt<1> r;
    r.v[0] = gl_mul(a.v[0], b.v[0]);
    return r;
}
GL_HD GlExt<2> ext_mul(const GlExt<2>& a, const GlExt<2>& b) {  // f64/mod.rs:403-409
    GlExt<2> r;
    u64 a0b0 = gl_mul(a.v[0], b.v[0]);
    r.v[0] = gl_sub(a0b0, gl_dbl(gl_mul(a.v[1], b.v[1])));
    r.v[1] = gl_sub(gl_mul(gl_add(a.v[0], a.v[1]), gl_add(b.v[0], b.v[1])), a0b0);
    return r;
}
GL_HD GlExt<3> ext_mul(const GlExt<3>& a, const GlExt<3>& b) {  // f64/mod.rs:445-466
    GlExt<3> r;
    u64 a0b0 = gl_mul(a.v[0], b.v[0]), a1b1 = gl_mul(a.v[1], b.v[1]), a2b2 = gl_mul(a.v[2], b.v[2]);
    u64 s01 = gl_mul(gl_add(a.v[0], a.v[1]), gl_add(b.v[0], b.v[1]));
    u64 s02 = gl_mul(gl_add(a.v[0], a.v[2]), gl_add(b.v[0], b.v[2]));
    u64 s12 = gl_mul(gl_add(a.v[1], a.v[2]), gl_add(b.v[1], b.v[2]));
    u64 m = gl_sub(a0b0, a1b1);
    r.v[0] = gl_sub(gl_add(s12, m), a2b2);
    r.v[1] = gl_sub(gl_sub(gl_add(s01, s12), gl_dbl(a1b1)), a0b0);
    r.v[2] = gl_sub(s02, m);
    return r;
}
GL_HD GlExt<1> ext_frobenius(const GlExt<1>& x) { return x; }
GL_HD GlExt<2> ext_frobenius(const GlExt<2>& x) {  // f64/mod.rs:431
    GlExt<2> r;
    r.v[0] = gl_add(x.v[0], x.v[1]);
    r.v[1] = gl_neg(x.v[1]);
    return r;
}
GL_HD GlExt<3> ext_frobenius(const GlExt<3>& x) {  // f64/mod.rs:490-498
    GlExt<3> r;
    r.v[0] = gl_add(x.v[0], gl_add(gl_mul(10615703402128488253ULL, x.v[1]), gl_mul(6700183068485440220ULL, x.v[2])));
    r.v[1] = gl_add(gl_mul(10050274602728160328ULL, x.v[1]), gl_mul(14531223735771536287ULL, x.v[2]));
    r.v[2] = gl_add(gl_mul(11746561000929144102ULL, x.v[1]), gl_mul(8396469466686423992ULL, x.v[2]));
    return r;
}
GL_HD GlExt<1> ext_inv(const GlExt<1>& a) {
    GlExt<1> r;
    r.v[0] = gl_inv(a.v[0]);
    return r;
}
GL_HD GlExt<2> ext_inv(const GlExt<2>& a) {  // extensions/quadratic.rs:81-94
    if ((a.v[0] | a.v[1]) == 0) return a;
    GlExt<2> num = ext_frobenius(a);
    GlExt<2> norm = ext_mul(a, num);
    return ext_mul_base(num, gl_inv(norm.v[0]));
}
GL_HD GlExt<3> ext_inv(const GlExt<3>& a) {  // extensions/cubic.rs:81-97
    if ((a.v[0] | a.v[1] | a.v[2]) == 0) return a;
    GlExt<3> c1 = ext_frobenius(a);
    GlExt<3> c2 = ext_frobenius(c1);
    GlExt<3> num = ext_mul(c1, c2);
    GlExt<3> norm = ext_mul(a, num);
    return ext_mul_base(num, gl_inv(norm.v[0]));
}
template <int D>
GL_HD GlExt<D> ext_pow(GlExt<D> a, u64 e) {
    GlExt<D> r = ext_from_base<D>(1);
    while (e) {
        if (e & 1) r = ext_mul(r, a);
        a = ext_mul(a, a);
        e >>= 1;
    }
    return r;
}
