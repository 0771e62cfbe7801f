// ntt2.cu — the sm_90a NTT pass kernel for sub-transforms of 2^6 .. 2^11 points (ntt.cuh describes the layout,
// the four-step schedule and the parameters; ntt.cu keeps the small-size kernel for sub-transforms below 2^6).
//
// What changed against the round-1 kernel (many issued instructions per element per pass that were not arithmetic,
// and shared-memory bank conflicts):
//  * every block owns a tile of 8192 elements (64 KB): S rows x LANES words with LANES = 8 for S <= 2^10 and
//    LANES = 4 (half a segment row) for S = 2^11, so two blocks are resident per SM at every size and the
//    global load / store phases of one overlap the butterflies of the other;
//  * sixteen values per thread per round: a radix-16 butterfly on one lane (64-bit shared-memory accesses) or a
//    radix-8 butterfly on two adjacent lanes (128-bit accesses, one twiddle load for both columns). Round radices
//    per size: 2^11 = 8.16.16, 2^10 = 8.8.16, 2^9 = 8.8.8, 2^8 = 16.16, 2^7 = 8.16, 2^6 = 8.8 — two shared-memory
//    exchanges and two rounds of 64x64-bit twiddle products for 2^10 / 2^11 instead of three / three;
//  * the sub-transform size is a template parameter: all index arithmetic of the rounds is resolved at compile time;
//  * global accesses are 128-bit (two adjacent words of a segment row);
//  * rows are placed in shared memory at (row ^ hash(row)), hash = XOR-fold of the row index above the bits that
//    select the 128-byte bank window, so that rows 2^k apart — what every butterfly stage and the bit-reversed
//    write-back touch together — never share a bank;
//  * inter-round twiddles come from per-round tables [lo][position] (positions of one butterfly contiguous, read as
//    128-bit pairs, conflict-free across the warp) staged by TMA bulk copies; the strided four-step twiddle is
//    w^(e_hi * 2^h) * w^(e_lo) from two small tables instead of a gather over a table of N/2 entries.
#include "minidft.cuh"
#include "ntt.cuh"

#ifndef NTT2_THREADS
#define NTT2_THREADS 256
#endif
#ifndef NTT2_MINB
#define NTT2_MINB 2
#endif
#define NTT2_TILE_ELEMS 8192

// ---- compile-time plan of a sub-transform of 2^LOGS points ----------------------------------------
template <int LOGS>
struct Plan {
    static constexpr int rounds = LOGS >= 9 ? 3 : 2;
    // radix-8 rounds first: the last round carries no twiddles, so the widest butterflies go where they save most
    static constexpr int r0 = (LOGS == 8) ? 4 : 3;
    static constexpr int r1 = (LOGS == 11 || LOGS == 8 || LOGS == 7) ? 4 : 3;
    static constexpr int r2 = LOGS >= 9 ? LOGS - r0 - r1 : 0;
    static_assert(LOGS >= 6 && LOGS <= 11, "plan covers 2^6 .. 2^11");
    static_assert(r0 + r1 + r2 == LOGS && (rounds == 2 || (r2 == 3 || r2 == 4)), "radices must add up");
    static constexpr int lanes = LOGS == 11 ? 4 : 8;
    // twiddle table of round k (k < rounds - 1): [span_k][2^r_k] entries
    static constexpr int tw0_entries = 1 << LOGS;                  // span0 * 2^r0 = S
    static constexpr int tw1_entries = rounds == 3 ? (1 << (LOGS - r0)) : 0;
    static constexpr int tw_entries = tw0_entries + tw1_entries;
};
template <int LOGS> __host__ __device__ constexpr int plan_radix(int k) { return k == 0 ? Plan<LOGS>::r0 : (k == 1 ? Plan<LOGS>::r1 : Plan<LOGS>::r2); }
template <int LOGS> __host__ __device__ constexpr int plan_stage(int k) { return k == 0 ? 0 : (k == 1 ? Plan<LOGS>::r0 : Plan<LOGS>::r0 + Plan<LOGS>::r1); }

// ---- shared-memory row placement --------------------------------------------------------------------
// LK = log2(rows per 128-byte bank window) = 1 for 64-byte rows (LANES = 8), 2 for 32-byte rows (LANES = 4).
template <int LK>
__host__ __device__ constexpr u32 swz_const(u32 r) {
    u32 x = r >> LK, h = 0;
    while (x) { h ^= x & ((1u << LK) - 1); x >>= LK; }
    return h;
}
// A round reads rows base + Q (Q = q << LOGSPAN, base zero on Q's bits) at (base + Q) ^ hash(base) ^ swz_const(Q). The XOR
// only reaches the low LK bits, so that row is ((base ^ hash(base)) ^ swz_lo(Q)) + swz_hi(Q): a task holds 2^LK row pointers
// and every access is one of them plus a compile-time offset (the per-access form cost four integer instructions).
template <int LK>
__host__ __device__ constexpr u32 swz_lo(u32 Q) { return swz_const<LK>(Q) ^ (Q & ((1u << LK) - 1)); }
template <int LK>
__host__ __device__ constexpr u32 swz_hi(u32 Q) { return Q & ~((1u << LK) - 1); }
__host__ __device__ constexpr u32 brev_const(u32 v, int bits) {
    u32 r = 0;
    for (int i = 0; i < bits; i++) r |= ((v >> i) & 1u) << (bits - 1 - i);
    return r;
}
// Calls f(it, lo, hi) for it = IT .. N - 1, where tile row brev(it STEP) (LOGS bits) sits at row pointer lo plus hi rows: the
// offsets are compile-time constants in every call.
template <int LOGS, int LK, u32 STEP, u32 N, u32 IT = 0, class F>
__device__ __forceinline__ void for_brev_rows(F&& f) {
    if constexpr (IT < N) {
        constexpr u32 c = brev_const(IT * STEP, LOGS);
        f(IT, swz_lo<LK>(c), swz_hi<LK>(c));
        for_brev_rows<LOGS, LK, STEP, N, IT + 1>(f);
    }
}
template <int LK>
__device__ __forceinline__ u32 swz_hash(u32 r) {  // r < 2^11
    if (LK == 1) return __popc(r >> 1) & 1;
    u32 x = r >> 2;           // 9 bits
    x ^= x >> 4;              // bits 0-3 fold 4-7; bit 8 folds into bit 4 -> handled below
    x ^= x >> 8;
    x ^= x >> 2;
    return x & 3;
}
template <int LK>
__device__ __forceinline__ u32 prow(u32 r) { return r ^ swz_hash<LK>(r); }

// ---- TMA bulk copy (global -> shared) -----------------------------------------------------------------
__device__ __forceinline__ void bulk_init(u64* mbar, int tid) {
    if (tid == 0) {
        u32 mb = (u32)__cvta_generic_to_shared(mbar);
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mb));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
}
__device__ __forceinline__ void bulk_expect(u64* mbar, u32 bytes) {
    u32 mb = (u32)__cvta_generic_to_shared(mbar);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy(void* smem_dst, const void* gsrc, u32 bytes, u64* mbar) {
    u32 mb = (u32)__cvta_generic_to_shared(mbar), dst = (u32)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(gsrc), "r"(bytes),
                 "r"(mb)
                 : "memory");
}
__device__ __forceinline__ void bulk_wait(u64* mbar) {
    u32 mb = (u32)__cvta_generic_to_shared(mbar), done = 0;
    while (!done)
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(mb) : "memory");
}

// ---- cp.async tile loads (global -> shared, no register staging) ---------------------------------------
// src_size 0 fills the destination with zeros without reading `gsrc`, which must still be a valid address
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool ok) {
    const u32 dst = (u32)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(gsrc), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gsrc, bool ok) {
    const u32 dst = (u32)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(gsrc), "r"(ok ? 8 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// ---- one round ----------------------------------------------------------------------------------------
// Round K of the plan on the tile `s` (S rows x LANES words, swizzled rows). tw: this round's table
// [span][2^R] (null for the last round). pre: null, or the input scale pre[row] applied as the round reads the tile
// (round 0 only). Each task = 16 values.
template <int LOGS, int K>
__device__ __forceinline__ void tile_round(u64* __restrict__ s, const u64* __restrict__ tw, const u64* __restrict__ pre, int tid) {
    constexpr int LANES = Plan<LOGS>::lanes, LK = LANES == 8 ? 1 : 2;
    constexpr int R = plan_radix<LOGS>(K), ST = plan_stage<LOGS>(K);
    constexpr int LOGSPAN = LOGS - ST - R;
    constexpr u32 SPAN = 1u << LOGSPAN;
    constexpr bool LAST = LOGSPAN == 0;
    constexpr u32 TASKS = (1u << LOGS) * LANES / 16;
    if (R == 4) {
        // radix-16 on one lane (the task loops stay rolled: unrolled, the 2^11 pass was slower and the 2^8 one much slower)
#pragma unroll 1
        for (u32 task = tid; task < TASKS; task += NTT2_THREADS) {
            const u32 lane = task % LANES, bf = task / LANES;
            const u32 lo = bf & (SPAN - 1), base = ((bf >> LOGSPAN) << (LOGSPAN + 4)) + lo;
            const u32 bh = base ^ swz_hash<LK>(base);
            u64* pr[1 << LK];
#pragma unroll
            for (int v = 0; v < (1 << LK); v++) pr[v] = s + ((bh ^ v) * LANES + lane);
            u64 x[16];
#pragma unroll
            for (int q = 0; q < 16; q++) x[q] = pr[swz_lo<LK>((u32)q << LOGSPAN)][swz_hi<LK>((u32)q << LOGSPAN) * LANES];
            if (K == 0 && pre) {
#pragma unroll
                for (int q = 0; q < 16; q++) x[q] = gl_mul(x[q], __ldg(pre + base + ((u32)q << LOGSPAN)));
            }
            mini_dft<4>(x);
            if (!LAST) {
                const ulonglong2* t2 = reinterpret_cast<const ulonglong2*>(tw + (size_t)lo * 16);
#pragma unroll
                for (int h = 0; h < 8; h++) {
                    const ulonglong2 w = t2[h];
                    if (h > 0) x[2 * h] = gl_mul(x[2 * h], w.x);
                    x[2 * h + 1] = gl_mul(x[2 * h + 1], w.y);
                }
            }
#pragma unroll
            for (int q = 0; q < 16; q++) pr[swz_lo<LK>((u32)q << LOGSPAN)][swz_hi<LK>((u32)q << LOGSPAN) * LANES] = x[q];
        }
    } else {
        // radix-8 on two adjacent lanes
        constexpr int LP = LANES / 2;
#pragma unroll 1
        for (u32 task = tid; task < TASKS; task += NTT2_THREADS) {
            const u32 lp = task % LP, bf = task / LP;
            const u32 lo = bf & (SPAN - 1), base = ((bf >> LOGSPAN) << (LOGSPAN + 3)) + lo;
            const u32 bh = base ^ swz_hash<LK>(base);
            ulonglong2* pr[1 << LK];
#pragma unroll
            for (int v = 0; v < (1 << LK); v++) pr[v] = reinterpret_cast<ulonglong2*>(s + ((bh ^ v) * LANES + 2 * lp));
            u64 xa[8], xb[8];
#pragma unroll
            for (int q = 0; q < 8; q++) {
                const ulonglong2 v = pr[swz_lo<LK>((u32)q << LOGSPAN)][swz_hi<LK>((u32)q << LOGSPAN) * (LANES / 2)];
                xa[q] = v.x;
                xb[q] = v.y;
            }
            if (K == 0 && pre) {
#pragma unroll
                for (int q = 0; q < 8; q++) {
                    const u64 f = __ldg(pre + base + ((u32)q << LOGSPAN));
                    xa[q] = gl_mul(xa[q], f);
                    xb[q] = gl_mul(xb[q], f);
                }
            }
            mini_dft<3>(xa);
            mini_dft<3>(xb);
            if (!LAST) {
                const ulonglong2* t2 = reinterpret_cast<const ulonglong2*>(tw + (size_t)lo * 8);
#pragma unroll
                for (int h = 0; h < 4; h++) {
                    const ulonglong2 w = t2[h];
                    if (h > 0) { xa[2 * h] = gl_mul(xa[2 * h], w.x); xb[2 * h] = gl_mul(xb[2 * h], w.x); }
                    xa[2 * h + 1] = gl_mul(xa[2 * h + 1], w.y);
                    xb[2 * h + 1] = gl_mul(xb[2 * h + 1], w.y);
                }
            }
#pragma unroll
            for (int q = 0; q < 8; q++) pr[swz_lo<LK>((u32)q << LOGSPAN)][swz_hi<LK>((u32)q << LOGSPAN) * (LANES / 2)] = make_ulonglong2(xa[q], xb[q]);
        }
    }
}

// ---- the pass kernel ------------------------------------------------------------------------------------
// grid = (tile columns x chunks per row, segments, batch), or (batch, tile columns x chunks per row, segments) with
// y_in_out. Shared memory:
//   tile [S][LANES] | round twiddles [tw_entries] | post twiddles [S][T] (STRIDED with has_post) | mbarrier
template <int MODE, int LOGS>
__global__ void __launch_bounds__(NTT2_THREADS, NTT2_MINB) ntt2_pass_kernel(const NttPassParams p) {
    extern __shared__ __align__(16) u64 smem[];
    constexpr int LANES = Plan<LOGS>::lanes, LK = LANES == 8 ? 1 : 2, LP = LANES / 2;
    constexpr u32 S = 1u << LOGS;
    const int tid = threadIdx.x;
    const int W = p.W, logW = 31 - __clz(W);
    const int T = W >= LANES ? 1 : (LANES >> logW);         // tile columns per tile
    const int chunks = W >= LANES ? W / LANES : 1;           // tiles across one segment row
    u64* s = smem;
    u64* rtw = s + (size_t)S * LANES;
    u64* ctw = rtw + Plan<LOGS>::tw_entries;
    u64* mbar = ctw + (p.has_post ? (size_t)S * T : 0);

    const bool ymap = p.y_in_out;
    const u32 tc = ymap ? blockIdx.y : blockIdx.x;
    const u32 tile = tc / chunks, q0 = (tc % chunks) * LANES;
    const u32 g = ymap ? blockIdx.z : blockIdx.y, b = ymap ? blockIdx.x : blockIdx.z;
    const u32 R = 1u << p.logR, C = 1u << p.logC;
    const u32 ncols = MODE == NTT_STRIDED ? C : R;

    // ---- load, issued first: thread -> (row i, lane pair), every 16-byte (W = 1: 8-byte) piece of the tile in flight at once
    // as a cp.async copy, so that the post twiddles below are computed while the tile arrives. The coset pre-scale is applied
    // by round 0 as it first reads each element.
    {
        const u64* in = p.in + (size_t)g * p.in_seg_stride + (size_t)b * p.in_batch_stride;
        const u32 lp = tid % LP;
        const u32 l0 = 2 * lp;                                     // first lane of the pair
        const u32 t0 = W >= LANES ? 0 : (l0 >> logW), t1 = W >= LANES ? 0 : ((l0 + 1) >> logW);
        const u32 w0 = W >= LANES ? q0 + l0 : (l0 & (W - 1)), w1 = W >= LANES ? q0 + l0 + 1 : ((l0 + 1) & (W - 1));
        const u32 c0 = tile * T + t0, c1 = tile * T + t1;
        const bool ok0 = c0 < ncols, ok1 = c1 < ncols;
        // element (i, col c, word w): STRIDED row C*i + c; CONTIG row c*C + i, or with y_in_out the row it is written back
        // to, (c + R*i)*mul + b*add of the output geometry. A lane past the last column is zero-filled from a valid address.
        const bool yin = MODE == NTT_CONTIG && ymap;
        const u64 istride = MODE == NTT_STRIDED ? ((u64)W << p.logC) : (yin ? ((u64)p.out_row_mul << p.logR) * p.out_W : (u64)W);
        const u64* a0 = MODE == NTT_STRIDED ? in + (size_t)c0 * W + w0
                        : yin ? in + ((size_t)c0 * p.out_row_mul + (size_t)b * p.out_row_add) * p.out_W + p.out_col0 + w0
                              : in + (((size_t)c0 << p.logC) * W + w0);
        const u64* a1 = MODE == NTT_STRIDED ? in + (size_t)c1 * W + w1
                        : yin ? in + ((size_t)c1 * p.out_row_mul + (size_t)b * p.out_row_add) * p.out_W + p.out_col0 + w1
                              : in + (((size_t)c1 << p.logC) * W + w1);
        if (!ok0) a0 = p.in;
        if (!ok1) a1 = p.in;
        const u64 s0 = ok0 ? istride : 0, s1 = ok1 ? istride : 0;
        const bool vec = p.vec_in;
        constexpr u32 ROWS_PER_IT = NTT2_THREADS / LP;
#pragma unroll 4
        for (u32 i = tid / LP; i < S; i += ROWS_PER_IT) {
            u64* dst = s + prow<LK>(i) * LANES + l0;
            if (vec) {
                cp_async16(dst, a0 + i * s0, ok0);
            } else {
                cp_async8(dst, a0 + i * s0, ok0);
                cp_async8(dst + 1, a1 + i * s1, ok1);
            }
        }
        cp_async_commit();
    }

    // round twiddles: one TMA bulk copy
    bulk_init(mbar, tid);
    __syncthreads();
    if (tid == 0) {
        bulk_expect(mbar, Plan<LOGS>::tw_entries * 8);
        bulk_copy(rtw, p.sub_tw, Plan<LOGS>::tw_entries * 8, mbar);
    }

    // post twiddles of this tile: ctw[j][t] = w_M^(+-(j a_mul + (batch0 + b) b_mul) c) * ctab[c] * cconst, c = tile*T + t,
    // with w_M^e = hi_tab[e >> split] * lo_tab[e & (2^split - 1)]
    if (p.has_post && T == 1) {
        // one tile column c: ctw[j] = K g^j with g = w_M^(+-a_mul c), K = w_M^(+-(batch0 + b) b_mul c) ctab[c] cconst — a geometric
        // progression in j: every thread starts at j = tid (one table product) and steps by g^NTT2_THREADS, one multiplication
        // per entry instead of the two or three of the direct form below
        const u32 M = 1u << p.logM, lo_mask = (1u << p.tw_split) - 1, c = tile;
        auto wpow = [&](u64 e64) {
            u32 e = (u32)(e64 & (M - 1));
            if (p.inverse && e) e = M - e;
            return gl_mul(p.tw_hi[e >> p.tw_split], p.tw_lo[e & lo_mask]);
        };
        u64 K = wpow((u64)(p.batch0 + b) * p.b_mul * c);
        if (p.ctab) K = gl_mul(K, p.ctab[c < ncols ? c : 0]);
        if (p.cconst != 1) K = gl_mul(K, p.cconst);
        const u64 step = wpow((u64)NTT2_THREADS * p.a_mul * c);
        u64 x = gl_mul(K, wpow((u64)tid * p.a_mul * c));
        for (u32 j = tid; j < S; j += NTT2_THREADS) {
            ctw[j] = x;
            x = gl_mul(x, step);
        }
    } else if (p.has_post) {
        const u32 M = 1u << p.logM, lo_mask = (1u << p.tw_split) - 1;
        for (u32 idx = tid; idx < S * (u32)T; idx += NTT2_THREADS) {
            const u32 j = idx / T, tt = idx % T, c = tile * T + tt;
            u64 e64 = ((u64)j * p.a_mul + (u64)(p.batch0 + b) * p.b_mul) * c;
            u32 e = (u32)(e64 & (M - 1));
            if (p.inverse && e) e = M - e;
            u64 x = gl_mul(p.tw_hi[e >> p.tw_split], p.tw_lo[e & lo_mask]);
            if (p.ctab) x = gl_mul(x, p.ctab[c < ncols ? c : 0]);
            if (p.cconst != 1) x = gl_mul(x, p.cconst);
            ctw[idx] = x;
        }
    }

    cp_async_wait_all();
    bulk_wait(mbar);
    __syncthreads();

    // ---- the sub-transform: forward DIF network, output position pos holds X[bitrev(pos)] ----
    tile_round<LOGS, 0>(s, rtw, p.pre_tab ? p.pre_tab + (size_t)b * p.pre_batch_stride : nullptr, tid);
    __syncthreads();
    if (Plan<LOGS>::rounds == 3) {
        tile_round<LOGS, 1>(s, rtw + Plan<LOGS>::tw0_entries, nullptr, tid);
        __syncthreads();
        tile_round<LOGS, 2>(s, nullptr, nullptr, tid);
    } else {
        tile_round<LOGS, 1>(s, nullptr, nullptr, tid);
    }
    __syncthreads();

    // ---- write back ----
    u64* out = p.out + (size_t)g * p.out_seg_stride + (size_t)b * p.out_batch_stride;
    {
        const u32 lp = tid % LP, l0 = 2 * lp;
        const u32 t0 = W >= LANES ? 0 : (l0 >> logW), t1 = W >= LANES ? 0 : ((l0 + 1) >> logW);
        const u32 w0 = W >= LANES ? q0 + l0 : (l0 & (W - 1)), w1 = W >= LANES ? q0 + l0 + 1 : ((l0 + 1) & (W - 1));
        const u32 c0 = tile * T + t0, c1 = tile * T + t1;
        const bool ok0 = c0 < ncols, ok1 = c1 < ncols;
        u64 *o0, *o1, jstride;
        if (MODE == NTT_STRIDED && ymap) {  // Y[j][m2] -> out row (j + R*col)*mul + b*add, where X[j + R*col] goes
            o0 = out + (((size_t)c0 << p.logR) * p.out_row_mul + (size_t)b * p.out_row_add) * p.out_W + p.out_col0 + w0;
            o1 = out + (((size_t)c1 << p.logR) * p.out_row_mul + (size_t)b * p.out_row_add) * p.out_W + p.out_col0 + w1;
            jstride = (u64)p.out_row_mul * p.out_W;
        } else if (MODE == NTT_STRIDED) {  // Y[j][m2] = row j*C + col
            o0 = out + (size_t)c0 * W + w0;
            o1 = out + (size_t)c1 * W + w1;
            jstride = (u64)W << p.logC;
        } else {                     // X[j1 + R*j] -> out row (col + R*j)*mul + b*add
            o0 = out + ((size_t)c0 * p.out_row_mul + (size_t)b * p.out_row_add) * p.out_W + p.out_col0 + w0;
            o1 = out + ((size_t)c1 * p.out_row_mul + (size_t)b * p.out_row_add) * p.out_W + p.out_col0 + w1;
            jstride = ((u64)p.out_row_mul << p.logR) * p.out_W;
        }
        const bool post = p.has_post, scale = !p.has_post && p.cconst != 1, vec = p.vec_out;
        const u32 inv_mask = p.inverse ? (S - 1) : 0;  // jf = inverse ? (S - j) mod S : j
        constexpr u32 ROWS_PER_IT = NTT2_THREADS / LP;
        if (!p.inverse && vec && T == 1) {
            // Forward transform, 128-bit stores, one tile column (every LDE): output row j = j0 + it ROWS_PER_IT is tile row
            // brev(j0) | brev(it ROWS_PER_IT), two bit fields apart, so with the linear row hash it sits at
            // prow(brev(j0)) ^ prow(brev(it ROWS_PER_IT)), the second a compile-time constant. As in the rounds, 2^LK row pointers and
            // compile-time offsets replace the per-row bit reversal and hash, and the output and twiddle rows advance by constants.
            const u32 j0 = tid / LP, r0 = __brev(j0) >> (32 - LOGS), rh = r0 ^ swz_hash<LK>(r0);
            const ulonglong2* pr[1 << LK];
#pragma unroll
            for (int v = 0; v < (1 << LK); v++) pr[v] = reinterpret_cast<const ulonglong2*>(s + ((rh ^ v) * LANES + l0));
            const u64* cj = ctw + j0;
            u64* oj = o0 + (u64)j0 * jstride;
            const u64 ostep = (u64)ROWS_PER_IT * jstride;
            for_brev_rows<LOGS, LK, ROWS_PER_IT, S / ROWS_PER_IT>([&](u32 it, u32 lo, u32 hi) {
                ulonglong2 v = pr[lo][hi * (LANES / 2)];
                if (post) {
                    const u64 f = cj[it * ROWS_PER_IT];
                    v.x = gl_mul(v.x, f);
                    v.y = gl_mul(v.y, f);
                } else if (scale) {
                    v.x = gl_mul(v.x, p.cconst);
                    v.y = gl_mul(v.y, p.cconst);
                }
                if (ok0) *reinterpret_cast<ulonglong2*>(oj + it * ostep) = v;
            });
            return;
        }
#pragma unroll 4
        for (u32 j = tid / LP; j < S; j += ROWS_PER_IT) {
            const u32 jf = inv_mask ? ((S - j) & inv_mask) : j;
            const u32 r = __brev(jf) >> (32 - LOGS);
            ulonglong2 v = *reinterpret_cast<const ulonglong2*>(s + prow<LK>(r) * LANES + l0);
            if (post) {
                const u64 f0 = ctw[j * T + t0];
                v.x = gl_mul(v.x, f0);
                v.y = gl_mul(v.y, t1 == t0 ? f0 : ctw[j * T + t1]);
            } else if (scale) {
                v.x = gl_mul(v.x, p.cconst);
                v.y = gl_mul(v.y, p.cconst);
            }
            if (vec) {
                if (ok0) *reinterpret_cast<ulonglong2*>(o0 + (u64)j * jstride) = v;
            } else {
                if (ok0) o0[(u64)j * jstride] = v.x;
                if (ok1) o1[(u64)j * jstride] = v.y;
            }
        }
    }
}

// ---- round-twiddle tables -----------------------------------------------------------------------------
// table of a 2^LOGS-point plan: round k < rounds-1: [lo < span_k][qo < 2^r_k] = w_S^((lo * bitrev_r(qo)) << stage_k)
template <int LOGS>
__global__ void ntt2_build_tw_kernel(u64* out, u64 w_s) {
    const u32 idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (u32)Plan<LOGS>::tw_entries) return;
    int k = idx < (u32)Plan<LOGS>::tw0_entries ? 0 : 1;
    const u32 li = k == 0 ? idx : idx - Plan<LOGS>::tw0_entries;
    const int r = plan_radix<LOGS>(k), st = plan_stage<LOGS>(k);
    const u32 lo = li >> r, qo = li & ((1u << r) - 1);
    const u32 e = (lo * (__brev(qo) >> (32 - r))) << st;
    out[idx] = gl_pow(w_s, e);
}

template <int LOGS>
static size_t smem_bytes_t(const NttPassParams& p) {
    const int lanes = Plan<LOGS>::lanes;
    const size_t S = (size_t)1 << LOGS, T = p.W >= lanes ? 1 : lanes / p.W;
    return (S * lanes + Plan<LOGS>::tw_entries + (p.has_post ? S * T : 0) + 2) * 8;
}
template <int MODE, int LOGS>
static cudaError_t launch_t(const NttPassParams& p, u32 n_segments, u32 n_batch, cudaStream_t st) {
    const int lanes = Plan<LOGS>::lanes;
    const u32 T = p.W >= lanes ? 1 : lanes / p.W, chunks = p.W >= lanes ? p.W / lanes : 1;
    const u32 ncols = MODE == NTT_STRIDED ? (1u << p.logC) : (1u << p.logR);
    const size_t smem = smem_bytes_t<LOGS>(p);
    const u32 tiles = ((ncols + T - 1) / T) * chunks;
    const dim3 grid = p.y_in_out ? dim3(n_batch, tiles, n_segments) : dim3(tiles, n_segments, n_batch);
    cudaError_t e = cudaFuncSetAttribute(ntt2_pass_kernel<MODE, LOGS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    ntt2_pass_kernel<MODE, LOGS><<<grid, NTT2_THREADS, smem, st>>>(p);
    return cudaGetLastError();
}
template <int MODE>
static cudaError_t launch_m(const NttPassParams& p, u32 n_segments, u32 n_batch, cudaStream_t st) {
    switch (p.logS) {
        case 6: return launch_t<MODE, 6>(p, n_segments, n_batch, st);
        case 7: return launch_t<MODE, 7>(p, n_segments, n_batch, st);
        case 8: return launch_t<MODE, 8>(p, n_segments, n_batch, st);
        case 9: return launch_t<MODE, 9>(p, n_segments, n_batch, st);
        case 10: return launch_t<MODE, 10>(p, n_segments, n_batch, st);
        case 11: return launch_t<MODE, 11>(p, n_segments, n_batch, st);
    }
    return cudaErrorInvalidValue;
}
cudaError_t ntt2_launch_pass(int mode, const NttPassParams& p, u32 n_segments, u32 n_batch, cudaStream_t st) {
    return mode == NTT_STRIDED ? launch_m<NTT_STRIDED>(p, n_segments, n_batch, st) : launch_m<NTT_CONTIG>(p, n_segments, n_batch, st);
}
size_t ntt2_tw_entries(int logS) {
    switch (logS) {
        case 6: return Plan<6>::tw_entries; case 7: return Plan<7>::tw_entries; case 8: return Plan<8>::tw_entries;
        case 9: return Plan<9>::tw_entries; case 10: return Plan<10>::tw_entries; case 11: return Plan<11>::tw_entries;
    }
    return 0;
}
cudaError_t ntt2_build_tw(int logS, u64* d_out, cudaStream_t st) {
    const u64 w = gl_root_of_unity((u32)logS);
    const unsigned nb = (unsigned)((ntt2_tw_entries(logS) + 255) / 256);
    switch (logS) {
        case 6: ntt2_build_tw_kernel<6><<<nb, 256, 0, st>>>(d_out, w); break;
        case 7: ntt2_build_tw_kernel<7><<<nb, 256, 0, st>>>(d_out, w); break;
        case 8: ntt2_build_tw_kernel<8><<<nb, 256, 0, st>>>(d_out, w); break;
        case 9: ntt2_build_tw_kernel<9><<<nb, 256, 0, st>>>(d_out, w); break;
        case 10: ntt2_build_tw_kernel<10><<<nb, 256, 0, st>>>(d_out, w); break;
        case 11: ntt2_build_tw_kernel<11><<<nb, 256, 0, st>>>(d_out, w); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}
