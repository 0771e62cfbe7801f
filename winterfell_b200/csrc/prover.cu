// prover.cu — the full proving pipeline on device behind one C-ABI call (wf_prove_fib / wf_prove_air /
// wf_prove_air_aux), i.e. the body of winterfell's Prover::generate_proof (prover/src/lib.rs:282-492) with
// every hot loop on the GPU, and the same steps as separate exports (wf_eval_constraints, ...):
//   K1-K4  trace commitment          (ntt.cu, commit.cu)          DefaultTraceLde::new, set_aux_trace
//   K5     constraint evaluation     (fib_ / generic_constraints) DefaultConstraintEvaluator::evaluate
//   K6/K7  composition poly + commit (ntt.cu, commit.cu)          DefaultConstraintCommitment::new
//   K8     out-of-domain frames      (ood_partial_kernel)         TracePolyTable/CompositionPoly::get_ood_frame
//   K9/K10 DEEP composition          (deep_sum_kernel, syn_div_*) DeepCompositionPoly::{add_trace_polys, evaluate}
//   K11    FRI commit phase          (fri.cu, device coin)        FriProver::build_layers
//   K13    proof-of-work grinding    (grind_kernel)               ProverChannel::grind_query_seed, smallest nonce
// The Fiat-Shamir transcript (ProverChannel, prover/src/channel.rs) and the proof wire format
// (air/src/proof/*.rs) are host code here, bit-exact with the reference; during the FRI commit phase the
// coin is mirrored on the device and the host replays it afterwards.
//
// The DEEP composition D = (S - S(z)) / (X - z) + (S - S(zg)) / (X - zg),  S = sum_j cc_j T_j + sum_j cc'_j H_j, is built as the
// reference builds it (composer/mod.rs:67-210): S over the coefficients, two synthetic divisions (a parallel suffix scan
// here), one LDE (:171). The stepwise wf_deep_compose and the row-sharded prover, which hold LDE rows and not coefficients,
// compute the same values in EVALUATION form row by row over the LDE domain: exact field arithmetic, identical values
// (SURVEY.md A.4).
//
// Constraint evaluation needs the AIR on the device (Air::evaluate_transition is user Rust code,
// air/src/air/mod.rs:210): generic AIRs arrive as a flat description (transition programs for both
// segments, periodic columns, single / periodic / sequence assertions, exemptions; format in
// include/winterfell_b200.h) and run on a bytecode evaluator; the "FibSmall x k" family = k copies of
// examples/src/fibonacci/fib_small/air.rs:16-69 side by side (k = 1 is the reference example, k = 4 / 32
// the 8- / 64-column configurations of BASELINE.json) has a specialised kernel.
#include <algorithm>
#include <chrono>

#include "internal.hpp"
#include "air_host.hpp"
#include "blake3.cuh"
#include "alg_hash.cuh"

// =================================================================================================
// kernels
// =================================================================================================
#include "constraints_generic.cuh"  // ld_ext / seg_at, GenEvalParams, generic_constraints_kernel (also the source NVRTC compiles per AIR)

#ifndef FIB_ROWS_D3
#define FIB_ROWS_D3 2   // CE rows per thread sharing one inversion, cubic extension (register budget)
#endif
struct FibEvalParams {
    SegMatrix lde;      // N x 2k trace LDE
    SegMatrix out;      // ce x D combined constraint evaluations
    u32 k, log_n, log_blowup, log_ce_blowup;
    const u64* coef;    // [k][5][D]: per pair j the coefficients of t0, t1 (transition), of column 2j and 2j+1 in the
                        // step-0 boundary group, and of column 2j+1 in the last-step group
    u64 K0[3], K1[3];   // constants of the two boundary groups: sum_q bcoef0_q * value_q, sum_j bcoef1_j * result_j
    const u64* tw_ce;   // w_ce^i, i < ce/2
    u64 zt[8];          // 1 / (x^n - 1) at CE step i mod ce_blowup
    u64 last;           // g_trace^(n-1): transition exemption point and divisor offset of group 1
    // row-sharded evaluation (multi-GPU): this launch covers CE rows [row0, row0 + ce_rows); `lde` then holds the LDE
    // rows of that range followed by `blowup` halo rows (the first rows of the next shard), so the next-state row is
    // local row + blowup without wrap-around. ce_rows = 0: the whole domain.
    size_t row0, ce_rows;
    // sub-coset evaluation (ce_rows = 0 only): launch row il is CE row il << log_step, ce >> log_step rows in all
    u32 log_step;
};

// CE-domain rows, FIB_ROWS per thread sharing one field inversion (evaluator/default.rs:165-214
// evaluate_fragment_main + evaluation_table.rs:317-367 acc_column, fused). The three linear forms of a row
// (transition combination, the two boundary groups) are dot products of base-field frame values with extension
// coefficients: they run on delayed-reduction accumulators (GlAcc), one reduction per row and form instead of one per
// term — the first version spent 22 k instructions per row of the 64-column cubic configuration in gl_mul / gl_add.
template <int D>
__global__ void __launch_bounds__(256) fib_constraints_kernel(FibEvalParams p) {
    extern __shared__ __align__(16) u64 fsm[];
    constexpr int ROWS = D == 3 ? FIB_ROWS_D3 : 4;
    for (u32 i = threadIdx.x; i < p.k * 5 * D; i += blockDim.x) fsm[i] = p.coef[i];
    __syncthreads();
    const size_t ce_all = (size_t)1 << (p.log_n + p.log_ce_blowup);
    const size_t ce = p.ce_rows ? p.ce_rows : ce_all >> p.log_step;   // rows of this launch
    const size_t N = (size_t)1 << (p.log_n + p.log_blowup);
    const u32 lde_shift = p.log_blowup - p.log_ce_blowup;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const u32 half = (u32)(ce_all >> 1);
    const int W = p.lde.W;
    GlExt<D> T[ROWS], B0[ROWS], B1[ROWS];
    u64 d0[ROWS], d1[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
        const size_t il = tid + r * stride;   // row of this launch
        const size_t ic = il << p.log_step;   // its CE row, local to the shard
        const size_t i = ic + p.row0;         // row of the CE domain
        T[r] = ext_zero<D>(); B0[r] = ext_zero<D>(); B1[r] = ext_zero<D>();
        d0[r] = 1; d1[r] = 1;
        if (il >= ce) continue;
        const size_t ls = ic << lde_shift;
        const size_t nx = p.ce_rows ? ls + ((size_t)1 << p.log_blowup)
                                    : ((ls + ((size_t)1 << p.log_blowup)) & (N - 1));  // trace_lde/default/mod.rs:169-180
        GlAcc aT[D], a0[D], a1[D];
#pragma unroll
        for (int q = 0; q < D; q++) { aT[q] = acc_zero(); a0[q] = acc_zero(); a1[q] = acc_zero(); }
#pragma unroll 2
        for (u32 j = 0; j < p.k; j++) {
            // columns 2j, 2j+1 are adjacent words of one segment row: one 16-byte load per frame row
            const size_t off = (size_t)((2 * j) / W) * p.lde.seg_stride + (2 * j) % W;
            const ulonglong2 cur = __ldg(reinterpret_cast<const ulonglong2*>(p.lde.base + off + ls * W));
            const ulonglong2 nxt = __ldg(reinterpret_cast<const ulonglong2*>(p.lde.base + off + nx * W));
            const u64 t0 = gl_sub(nxt.x, gl_add(cur.x, cur.y));  // fib_small/air.rs:58
            const u64 t1 = gl_sub(nxt.y, gl_add(cur.y, nxt.x));  // :59
            const u64* cf = fsm + (size_t)j * 5 * D;
#pragma unroll
            for (int q = 0; q < D; q++) {
                acc_mad(aT[q], cf[q], t0);
                acc_mad(aT[q], cf[D + q], t1);
                acc_mad(a0[q], cf[2 * D + q], cur.x);
                acc_mad(a0[q], cf[3 * D + q], cur.y);
                acc_mad(a1[q], cf[4 * D + q], cur.y);
            }
        }
#pragma unroll
        for (int q = 0; q < D; q++) {
            T[r].v[q] = acc_reduce(aT[q]);
            B0[r].v[q] = gl_sub(acc_reduce(a0[q]), p.K0[q]);
            B1[r].v[q] = gl_sub(acc_reduce(a1[q]), p.K1[q]);
        }
        u64 w = p.tw_ce[i & (half - 1)];
        if (i & half) w = gl_neg(w);
        u64 x = gl_mul(w, GL_GENERATOR);  // domain.rs:123 get_ce_x_at
        d0[r] = gl_sub(x, 1);             // boundary divisor of the step-0 group
        d1[r] = gl_sub(x, p.last);        // boundary divisor of the last-step group = transition exemption
    }
    // batch inversion of the products d0*d1 (never zero: x lies on the coset 7<w>, 1 and g^(n-1) do not)
    u64 prod[ROWS], pre[ROWS], run = 1;
#pragma unroll
    for (int r = 0; r < ROWS; r++) { prod[r] = gl_mul(d0[r], d1[r]); pre[r] = run; run = gl_mul(run, prod[r]); }
    run = gl_inv(run);
#pragma unroll
    for (int r = ROWS - 1; r >= 0; r--) { u64 inv = gl_mul(run, pre[r]); run = gl_mul(run, prod[r]); prod[r] = inv; }
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
        const size_t il = tid + r * stride, i = (il << p.log_step) + p.row0;
        if (il >= ce) continue;
        u64 z0 = gl_mul(prod[r], d1[r]), z1 = gl_mul(prod[r], d0[r]);                   // 1/(x - 1), 1/(x - g^(n-1))
        u64 zt = gl_mul(p.zt[i & (((size_t)1 << p.log_ce_blowup) - 1)], d1[r]);         // e(x) / (x^n - 1)
        GlExt<D> acc = ext_add(ext_add(ext_mul_base(T[r], zt), ext_mul_base(B0[r], z0)), ext_mul_base(B1[r], z1));
        u64* o = p.out.base + il * p.out.W;
#pragma unroll
        for (int q = 0; q < D; q++) o[q] = acc.v[q];
    }
}

// composition_poly.rs:128-140 segment(): column j = coefficients [j*n, (j+1)*n) of the interpolated
// CE-domain polynomial; each is an extension column of D base columns.
__global__ void comp_split_kernel(SegMatrix coefs, size_t n, u32 kc, int D, SegMatrix out) {
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = n * kc * D;
    if (idx >= total) return;
    size_t i = idx / (kc * D);
    u32 col = (u32)(idx % (kc * D));
    u32 j = col / D, comp = col % D;
    u64 v = coefs.base[(j * n + i) * coefs.W + comp];
    out.base[(size_t)(col / out.W) * out.seg_stride + i * out.W + (col % out.W)] = v;
}

// row i of the n x W segment `src` -> row i * b of `dst` (coset 0 of an LDE in natural order), pad lanes included
__global__ void coset0_rows_kernel(const u64* src, size_t n, int W, u32 b, u64* dst) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * W) return;
    const size_t row = idx / W;
    dst[(row * b) * W + idx % W] = src[idx];
}

// Evaluation of every base-coefficient column at TWO extension points (z and z*g), as per-block partial sums
// (polynom::eval, math/src/polynom/mod.rs:55-62; ColMatrix::evaluate_columns_at :245; TracePolyTable::get_ood_frame
// poly_table.rs:68-76). Block = 32 row groups x 8 lanes (lane = column of the segment); a thread owns OOD_RPT
// consecutive coefficients of ONE column and accumulates sum_r a_r z^r for both points on delayed-reduction
// accumulators against a shared table of z^r (one base-by-extension product per coefficient and point, no reduction
// inside the loop); the row-group power (z^OOD_RPT)^rg and the block power z^(first row of the block) are applied once
// per thread / once per block. All three power tables are filled once per call by ood_pow_kernel: built per block, their
// ext_pow chains cost about as many instructions as the block's coefficient loop and held its loads back behind a
// barrier. partial[col][chunk][point] = sum_{m in chunk} a_m z^m.
#define OOD_RPT 64
#define OOD_ROWS_PER_BLOCK (32 * OOD_RPT)
#define OOD_TAB (OOD_RPT + 32)   // per point: z^r (r < OOD_RPT), then z^(OOD_RPT * rg) (rg < 32)
template <int D>
__global__ void ood_pow_kernel(GlExt<D> z0, GlExt<D> z1, u32 chunks, u64* zb /*[2][chunks][D]*/, u64* zt /*[2][OOD_TAB][D]*/) {
    const u32 idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < 2 * chunks) {
        const u32 pt = idx / chunks, c = idx % chunks;
        const GlExt<D> v = ext_pow(pt ? z1 : z0, (u64)c * OOD_ROWS_PER_BLOCK);
#pragma unroll
        for (int d = 0; d < D; d++) zb[(size_t)idx * D + d] = v.v[d];
    } else if (idx < 2 * chunks + 2 * OOD_TAB) {
        const u32 u = idx - 2 * chunks, pt = u / OOD_TAB, r = u % OOD_TAB;
        const GlExt<D> v = ext_pow(pt ? z1 : z0, r < OOD_RPT ? r : (u64)(r - OOD_RPT) * OOD_RPT);
#pragma unroll
        for (int d = 0; d < D; d++) zt[(size_t)u * D + d] = v.v[d];
    }
}
template <int D>
__global__ void __launch_bounds__(256) ood_partial_kernel(SegMatrix polys, const u64* zt, const u64* zb,
                                                          u64* partial /*[cols][chunks][2][D]*/, u32 chunks) {
    const u32 g = blockIdx.y, chunk = blockIdx.x, t = threadIdx.x;
    const int W = polys.W;
    const size_t n = polys.rows;
    const u64* base = polys.base + (size_t)g * polys.seg_stride;
    __shared__ u64 tab[2][OOD_TAB][D];
    __shared__ u64 red[2][32][8][D];
    auto zpow = [&](u32 pt, u32 r) -> const u64* { return tab[pt][r]; };                // z^r
    auto zrg = [&](u32 pt, u32 rg) -> const u64* { return tab[pt][OOD_RPT + rg]; };    // z^(OOD_RPT * rg)
    for (u32 i = t; i < 2 * OOD_TAB * D; i += 256) (&tab[0][0][0])[i] = zt[i];
    __syncthreads();
    const u32 rg = t >> 3, lane = t & 7;
    const size_t start = (size_t)chunk * OOD_ROWS_PER_BLOCK + (size_t)rg * OOD_RPT;
    GlAcc acc[2][D];
#pragma unroll
    for (int pt = 0; pt < 2; pt++)
#pragma unroll
        for (int d = 0; d < D; d++) acc[pt][d] = acc_zero();
    if (lane < (u32)W) {
        const u64* src = base + start * W + lane;
        // the next 8 coefficients are requested before this 8's products: loaded in the step that consumes them, each load
        // was issued right before its first product and the warp waited out a full memory latency per coefficient
        u64 nx[8];
#pragma unroll
        for (int k = 0; k < 8; k++) nx[k] = (start + k < n) ? __ldg(src + (size_t)k * W) : 0;
#pragma unroll 1
        for (int r0 = 0; r0 < OOD_RPT; r0 += 8) {
            u64 cf[8];
#pragma unroll
            for (int k = 0; k < 8; k++) cf[k] = nx[k];
            if (r0 + 8 < OOD_RPT) {
#pragma unroll
                for (int k = 0; k < 8; k++) nx[k] = (start + r0 + 8 + k < n) ? __ldg(src + (size_t)(r0 + 8 + k) * W) : 0;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
#pragma unroll
                for (int d = 0; d < D; d++) {
                    acc_mad(acc[0][d], zpow(0, r0 + k)[d], cf[k]);
                    acc_mad(acc[1][d], zpow(1, r0 + k)[d], cf[k]);
                }
            }
        }
    }
#pragma unroll
    for (int pt = 0; pt < 2; pt++) {
        GlExt<D> v;
#pragma unroll
        for (int d = 0; d < D; d++) v.v[d] = acc_reduce(acc[pt][d]);
        v = ext_mul(v, ld_ext<D>(zrg(pt, rg)));
#pragma unroll
        for (int d = 0; d < D; d++) red[pt][rg][lane][d] = v.v[d];
    }
    __syncthreads();
    if (t < 16) {
        const u32 pt = t >> 3, q = t & 7, col = g * W + q;
        if (q < (u32)W && col < polys.cols) {
            GlExt<D> sacc = ext_zero<D>();
            for (int k = 0; k < 32; k++) sacc = ext_add(sacc, ld_ext<D>(&red[pt][k][q][0]));
            sacc = ext_mul(sacc, ld_ext<D>(zb + ((size_t)pt * chunks + chunk) * D));
            u64* o = partial + (((size_t)col * chunks + chunk) * 2 + pt) * D;
#pragma unroll
            for (int d = 0; d < D; d++) o[d] = sacc.v[d];
        }
    }
}
// one warp per (column, point): lanes stride over the chunks (2048 of them for a 2^22-row column — a single thread
// walking them serially took 0.5 ms per call), then a shuffle tree over the extension components
template <int D>
__global__ void __launch_bounds__(256) ood_reduce_kernel(const u64* partial, u32 cols, u32 chunks, u64* out /*[cols][2][D]*/) {
    const u32 idx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (idx >= cols * 2) return;   // warp-uniform
    const u32 col = idx >> 1, pt = idx & 1;
    GlExt<D> s = ext_zero<D>();
    for (u32 c = lane; c < chunks; c += 32) s = ext_add(s, ld_ext<D>(partial + (((size_t)col * chunks + c) * 2 + pt) * D));
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        GlExt<D> o;
#pragma unroll
        for (int c = 0; c < D; c++) o.v[c] = __shfl_down_sync(0xffffffffu, s.v[c], off);
        s = ext_add(s, o);
    }
    if (lane == 0)
        for (int c = 0; c < D; c++) out[(size_t)idx * D + c] = s.v[c];
}

struct DeepParams {
    SegMatrix trace;   // N x c
    SegMatrix cons;    // N x kc*D
    SegMatrix out;     // N x D
    SegMatrix aux;     // N x aw*D (aux segment LDE; aw == 0 when single-segment)
    u32 c, kc, log_N, aw;
    const u64* acc;    // [aw][D] DEEP coefficients for aux columns (composer/mod.rs:100-125)
    const u64* tcc;    // [c][D]  DEEP coefficients for trace columns
    const u64* ccc;    // [kc][D] DEEP coefficients for composition columns
    const u64* tw_N;   // w_N^i, i < N/2
    size_t row0, nrows;  // row-sharded launch: rows [row0, row0 + nrows) of the LDE domain (nrows = 0: all N rows)
};
// DeepCompositionPoly in evaluation form, two kernels:
//   deep_sum_kernel: S(x) = sum_j cc_j T_j(x) + sum_j cc'_j A_j(x) + sum_j cc''_j H_j(x) for every LDE row — the
//     pass that reads the whole LDE (the coefficient form runs it over the coefficient rows, see syn_div_* below);
//     one row per thread, coefficients in shared memory, ~40 registers, so
//     the SMs stay full (the earlier single kernel needed 242 registers per thread with cubic elements:
//     12 % occupancy, 28 % issue utilisation, 2.0 ms for 2^21 rows x 64 columns);
//   deep_div_kernel: D(x) = (S(x) - S(z)) / (x - z) + (S(x) - S(zg)) / (x - zg) in place, DEEP_ROWS rows per
//     thread sharing one batch inversion (math/src/utils/mod.rs:169).
// (Tried and dropped: chains of rows i, i + b, ... that reuse 1 / (x_{i-b} - z) = g / (x_i - z g) to halve
// the inversions — the strided row pattern cost more than the arithmetic saved.)
#ifndef DEEP_SUM_THREADS
#define DEEP_SUM_THREADS 256
#endif
template <int D>
__global__ void __launch_bounds__(DEEP_SUM_THREADS) deep_sum_kernel(DeepParams p) {
    extern __shared__ __align__(16) u64 dsm[];
    u64* s_t = dsm;                                  // [c][D]
    u64* s_a = s_t + (size_t)p.c * D;                // [aw][D]
    u64* s_c = s_a + (size_t)p.aw * D;               // [kc][D]
    for (u32 i = threadIdx.x; i < p.c * D; i += DEEP_SUM_THREADS) s_t[i] = p.tcc[i];
    for (u32 i = threadIdx.x; i < p.aw * D; i += DEEP_SUM_THREADS) s_a[i] = p.acc[i];
    for (u32 i = threadIdx.x; i < p.kc * D; i += DEEP_SUM_THREADS) s_c[i] = p.ccc[i];
    __syncthreads();
    const size_t N = p.nrows ? p.nrows : ((size_t)1 << p.log_N);   // rows of this launch
    const size_t row = (size_t)blockIdx.x * DEEP_SUM_THREADS + threadIdx.x;
    if (row >= N) return;
    // S over the base-field trace columns = D dot products of the row with the coefficient components: delayed-reduction
    // accumulators, one reduction per component per row
    GlAcc acc[D];
#pragma unroll
    for (int d = 0; d < D; d++) acc[d] = acc_zero();
    if (p.trace.W == 8) {
        // one 64-byte segment row = four 16-byte loads; the next segment's row is requested before this one is consumed
        // (the kernel was latency-bound on these loads)
        const u32 nseg = (p.c + 7) / 8;
        ulonglong2 nx[4];
        {
            const ulonglong2* rp = reinterpret_cast<const ulonglong2*>(p.trace.base + row * 8);
#pragma unroll
            for (int k = 0; k < 4; k++) nx[k] = __ldg(rp + k);
        }
        for (u32 g = 0; g < nseg; g++) {
            u64 v[8];
#pragma unroll
            for (int k = 0; k < 4; k++) { v[2 * k] = nx[k].x; v[2 * k + 1] = nx[k].y; }
            if (g + 1 < nseg) {
                const ulonglong2* rp = reinterpret_cast<const ulonglong2*>(p.trace.base + (size_t)(g + 1) * p.trace.seg_stride + row * 8);
#pragma unroll
                for (int k = 0; k < 4; k++) nx[k] = __ldg(rp + k);
            }
#pragma unroll
            for (int q = 0; q < 8; q++) {
                u32 j = g * 8 + q;
                if (j < p.c) {
#pragma unroll
                    for (int d = 0; d < D; d++) acc_mad(acc[d], s_t[(size_t)j * D + d], v[q]);
                }
            }
        }
    } else {
        for (u32 j = 0; j < p.c; j++) {
            const u64 v = seg_at(p.trace, row, j);
#pragma unroll
            for (int d = 0; d < D; d++) acc_mad(acc[d], s_t[(size_t)j * D + d], v);
        }
    }
    GlExt<D> S;
#pragma unroll
    for (int d = 0; d < D; d++) S.v[d] = acc_reduce(acc[d]);
    for (u32 j = 0; j < p.aw; j++) {
        GlExt<D> av;
#pragma unroll
        for (int q = 0; q < D; q++) av.v[q] = seg_at(p.aux, row, j * D + q);
        S = ext_add(S, ext_mul(ld_ext<D>(s_a + (size_t)j * D), av));
    }
    for (u32 j = 0; j < p.kc; j++) {
        GlExt<D> hv;
#pragma unroll
        for (int q = 0; q < D; q++) hv.v[q] = seg_at(p.cons, row, j * D + q);
        S = ext_add(S, ext_mul(ld_ext<D>(s_c + (size_t)j * D), hv));
    }
    u64* o = p.out.base + row * p.out.W;
#pragma unroll
    for (int q = 0; q < D; q++) o[q] = S.v[q];
    for (int q = D; q < p.out.W; q++) o[q] = 0;  // pad lane (W = 4 for D = 3): the LDE of the coefficient form transforms it too
}

// rows per thread sharing one batch inversion
#ifndef DEEP_ROWS1
#define DEEP_ROWS1 8
#endif
#ifndef DEEP_ROWS2
#define DEEP_ROWS2 8
#endif
#ifndef DEEP_ROWS3
#define DEEP_ROWS3 8
#endif
#ifndef DEEP_DIV_MINB
#define DEEP_DIV_MINB 2
#endif
#define DEEP_ROWS (D == 1 ? DEEP_ROWS1 : (D == 2 ? DEEP_ROWS2 : DEEP_ROWS3))
// 1 / (x - z) for x in the BASE field and z in the extension, without an extension-field inversion: with m_z the minimal
// polynomial of z over the base field (degree D, base-field coefficients) and Q_z(X) = m_z(X) / (X - z) (degree D - 1, extension
// coefficients, monic),   1 / (x - z) = Q_z(x) / m_z(x),   m_z(x) = N(x - z) in the base field.
// So the per-row inversion is a BASE-field one (3 multiplications per denominator in a batch inversion instead of 3
// extension products = 18 for the cubic extension) and Q_z(x) costs D - 1 base-by-extension products. The host supplies
//   D = 3: m = X^3 - t X^2 + s X - n (t = trace, n = norm), Q = X^2 - q1 X + q0, q1 = z' + z'', q0 = z' z'' (Frobenius conjugates)
//   D = 2: m = X^2 - t X + n,                                Q = X - q0,          q0 = z'
//   D = 1: m = X - z,                                        Q = 1.
template <int D>
struct DeepPoint {
    u64 t, s, n;        // base-field coefficients of m_z
    GlExt<D> q1, q0;    // extension coefficients of Q_z
};
template <int D>
__device__ __forceinline__ u64 deep_m(const DeepPoint<D>& pt, u64 x, u64 x2) {
    if (D == 1) return gl_sub(x, pt.n);                                          // x - z
    if (D == 2) return gl_add(gl_sub(x2, gl_mul(pt.t, x)), pt.n);               // x^2 - t x + n
    return gl_sub(gl_add(gl_mul(x2, gl_sub(x, pt.t)), gl_mul(pt.s, x)), pt.n);  // x^2 (x - t) + s x - n
}
template <int D>
__device__ __forceinline__ GlExt<D> deep_q(const DeepPoint<D>& pt, u64 x, u64 x2) {
    GlExt<D> q;
    if (D == 1) { q.v[0] = 1; return q; }
    if (D == 2) { q = ext_sub(ext_from_base<D>(x), pt.q0); return q; }
    q = ext_sub(pt.q0, ext_mul_base(pt.q1, x));
    q.v[0] = gl_add(q.v[0], x2);
    return q;
}
template <int D>
__global__ void __launch_bounds__(256, DEEP_DIV_MINB) deep_div_kernel(DeepParams p, DeepPoint<D> pz, DeepPoint<D> pzg, GlExt<D> Sz, GlExt<D> Szg) {
    const size_t N = p.nrows ? p.nrows : ((size_t)1 << p.log_N);   // rows of this launch
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    constexpr int ROWS = DEEP_ROWS;
    u64 xs[D == 1 ? 1 : ROWS], den[2 * ROWS];   // x is only needed again by Q_z for D > 1
    const u32 half = (u32)(((size_t)1 << p.log_N) >> 1);
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
        size_t row = tid + r * stride;
        if (D > 1) xs[r] = 0;
        den[2 * r] = 1; den[2 * r + 1] = 1;
        if (row >= N) continue;
        const size_t grow = row + p.row0;   // row of the LDE domain
        u64 w = p.tw_N[grow & (half - 1)];
        if (grow & half) w = gl_neg(w);
        const u64 x = gl_mul(w, GL_GENERATOR), x2 = gl_sqr(x);
        if (D > 1) xs[r] = x;
        den[2 * r] = deep_m<D>(pz, x, x2);
        den[2 * r + 1] = deep_m<D>(pzg, x, x2);
    }
    // batch inversion in the base field; the norms are never zero (deep_compose refuses a z or z*g on the LDE domain)
    u64 pre[2 * ROWS], run = 1;
#pragma unroll
    for (int q = 0; q < 2 * ROWS; q++) { pre[q] = run; run = gl_mul(run, den[q]); }
    run = gl_inv(run);
#pragma unroll
    for (int q = 2 * ROWS - 1; q >= 0; q--) { const u64 inv = gl_mul(run, pre[q]); run = gl_mul(run, den[q]); den[q] = inv; }
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
        size_t row = tid + r * stride;
        if (row >= N) continue;
        u64* o = p.out.base + row * p.out.W;
        const GlExt<D> S = ld_ext<D>(o);
        const u64 x = D > 1 ? xs[r] : 0, x2 = D > 1 ? gl_sqr(x) : 0;
        const GlExt<D> a = ext_mul_base(ext_mul(ext_sub(S, Sz), deep_q<D>(pz, x, x2)), den[2 * r]);
        const GlExt<D> b = ext_mul_base(ext_mul(ext_sub(S, Szg), deep_q<D>(pzg, x, x2)), den[2 * r + 1]);
        const GlExt<D> v = ext_add(a, b);
#pragma unroll
        for (int q = 0; q < D; q++) o[q] = v.v[q];
    }
}
// host side of DeepPoint: the conjugates of z under the Frobenius map (math/src/field/f64/mod.rs:431, :490-498)
template <int D>
static bool deep_point(const GlExt<D>& z, DeepPoint<D>& pt) {
    pt.t = pt.s = pt.n = 0;
    pt.q1 = ext_zero<D>(); pt.q0 = ext_zero<D>();
    if (D == 1) { pt.n = z.v[0]; return true; }
    const GlExt<D> z1 = ext_frobenius(z);
    if (D == 2) {
        const GlExt<D> tr = ext_add(z, z1), nm = ext_mul(z, z1);
        pt.t = tr.v[0]; pt.n = nm.v[0]; pt.q0 = z1;
        return tr.v[1] == 0 && nm.v[1] == 0;
    }
    const GlExt<D> z2 = ext_frobenius(z1);
    const GlExt<D> tr = ext_add(z, ext_add(z1, z2));
    const GlExt<D> z12 = ext_mul(z1, z2);
    const GlExt<D> sm = ext_add(ext_mul(z, ext_add(z1, z2)), z12), nm = ext_mul(z, z12);
    pt.t = tr.v[0]; pt.s = sm.v[0]; pt.n = nm.v[0];
    pt.q1 = ext_add(z1, z2); pt.q0 = z12;
    bool ok = true;
    for (int k = 1; k < D; k++) ok = ok && tr.v[k] == 0 && sm.v[k] == 0 && nm.v[k] == 0;
    return ok;
}

// DeepCompositionPoly in coefficient form (prove_air, wf_deep_compose_polys), as the reference builds it: S = sum_j dc_j p_j over
// the n coefficients (deep_sum_kernel run on the coefficient matrices), the synthetic divisions by X - z and X - zg
// (polynom/mod.rs:498-505), q_i = sum_{k > i} s_k b^(k-i-1), q_(n-1) = 0, i.e. the recurrence q_(i-1) = s_i + b q_i run downwards,
// then one LDE of q_z + q_zg. The constant term s_0 only reaches the remainder, so S(z) and S(zg) need not be subtracted first (the
// reference subtracts them, composer/mod.rs:202-210, and the remainder it then drops is zero).
// The rows [u, v) map q_(v-1) to q_(u-1) = a + p q_(v-1), a = sum_{k in [u, v)} s_k b^(k-u), p = b^(v-u); adjacent runs L = [u, v)
// and R = [v, w) compose to (a_L + p_L a_R, p_L p_R). The recurrence is a suffix scan of these runs, in the three-launch shape of
// auxbuild.cu's prefix scans, both points in the same launches. Inside a tile every run has a known length, so its p is a known
// power of b and only the a's are scanned: combining two runs is one extension product by a power that is constant per scan level.
//   syn_div_reduce  per tile of SYN_TILE rows: each thread's run a over its SYN_ITEMS rows (Horner), a warp suffix scan of those
//                   (level k multiplies by b^(8·2^k)), a suffix scan of the 8 warp totals; it keeps, per thread, the a of the
//                   rest of its warp above it and, per warp, the a of the warps above it, and writes the tile's a (p = b^SYN_TILE);
//   syn_div_carry   one block: exclusive suffix scan of the tile runs = q at the top row of every tile; it also fills the table
//                   b^(8k), k < 32, and b^(256 j), j < 8, that apply reads;
//   syn_div_apply   per tile: q at the top row of each warp from the kept warp suffix and the carry (one lane, then shuffled to
//                   the warp), q at each thread's top row from the kept in-warp suffix, then the recurrence down the thread's
//                   SYN_ITEMS rows, q_z + q_zg written in place. No run is computed twice.
// Rows >= n read as zero, which changes no q (q_(n-1) = 0 either way). Field arithmetic is exact, so the association order of the
// scan changes no bit, and the LDE of the quotient equals deep_div_kernel's rows.
#define SYN_THREADS 256
#define SYN_ITEMS 8
#define SYN_TILE (SYN_THREADS * SYN_ITEMS)
#define SYN_WARPS (SYN_THREADS / 32)
#define SYN_PW (32 + SYN_WARPS)   // table per point: b^(SYN_ITEMS k), k < 32, then b^(32 SYN_ITEMS j), j < SYN_WARPS
template <int D>
struct SynDivParams {
    GlExt<D> b[2];        // z, zg
    GlExt<D> b_items[2];  // b^SYN_ITEMS
    GlExt<D> b_tile[2];   // b^SYN_TILE
    GlExt<D> lvl[2][8];   // b^(SYN_ITEMS 2^k): k < 5 for the warp scan levels, 5..7 for the scan over the warps
};
// scratch of one division, in one allocation of (tiles (1 + SYN_WARPS + SYN_THREADS) + SYN_PW) 2 D words
struct SynDivBufs {
    u64* agg;   // [tiles][2][D]: tile run a, then (after syn_div_carry) q at the tile's top row
    u64* wsuf;  // [tiles][SYN_WARPS][2][D]: a of the warps above this one in its tile
    u64* tsuf;  // [tiles][SYN_THREADS][2][D]: a of the threads above this one in its warp
    u64* pw;    // [2][SYN_PW][D]
};
template <int D>
struct SynRun {  // x -> a + p x for each point
    GlExt<D> a[2], p[2];
};
template <int D>
__device__ __forceinline__ SynRun<D> syn_ident() {
    SynRun<D> r;
#pragma unroll
    for (int pt = 0; pt < 2; pt++) { r.a[pt] = ext_zero<D>(); r.p[pt] = ext_from_base<D>(1); }
    return r;
}
// lo: the lower rows, hi: the rows right above them
template <int D>
__device__ __forceinline__ SynRun<D> syn_cat(const SynRun<D>& lo, const SynRun<D>& hi) {
    SynRun<D> r;
#pragma unroll
    for (int pt = 0; pt < 2; pt++) { r.a[pt] = ext_add(lo.a[pt], ext_mul(lo.p[pt], hi.a[pt])); r.p[pt] = ext_mul(lo.p[pt], hi.p[pt]); }
    return r;
}
template <int D>
__device__ __forceinline__ SynRun<D> syn_shfl_down(const SynRun<D>& v, u32 off) {
    SynRun<D> r;
#pragma unroll
    for (int pt = 0; pt < 2; pt++)
#pragma unroll
        for (int q = 0; q < D; q++) {
            r.a[pt].v[q] = __shfl_down_sync(0xffffffffu, v.a[pt].v[q], off);
            r.p[pt].v[q] = __shfl_down_sync(0xffffffffu, v.p[pt].v[q], off);
        }
    return r;
}
// exclusive suffix scan over the block (SYN_THREADS threads, thread order = row order): the run of the threads above this one;
// `total` = the whole block's run
template <int D>
__device__ __forceinline__ SynRun<D> syn_block_suffix(const SynRun<D>& v, SynRun<D>& total) {
    constexpr u32 NW = SYN_THREADS / 32;
    __shared__ SynRun<D> wrun[NW];
    const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    SynRun<D> x = v;
#pragma unroll
    for (u32 off = 1; off < 32; off <<= 1) {
        const SynRun<D> y = syn_shfl_down(x, off);
        if (lane + off < 32) x = syn_cat(x, y);
    }
    if (lane == 0) wrun[wid] = x;
    __syncthreads();
    if (wid == 0) {
        SynRun<D> s = lane < NW ? wrun[lane] : syn_ident<D>();
#pragma unroll
        for (u32 off = 1; off < NW; off <<= 1) {
            const SynRun<D> y = syn_shfl_down(s, off);
            if (lane + off < NW) s = syn_cat(s, y);
        }
        if (lane < NW) wrun[lane] = s;
    }
    __syncthreads();
    total = wrun[0];
    SynRun<D> ex = syn_shfl_down(x, 1);
    if (lane == 31) ex = syn_ident<D>();
    if (wid + 1 < NW) ex = syn_cat(ex, wrun[wid + 1]);
    __syncthreads();  // wrun is free for the next call
    return ex;
}
// rows of the n x D quotient matrix (one segment of width 1, 2 or 4; the pad lane stays zero)
template <int D>
__device__ __forceinline__ GlExt<D> syn_ld(const u64* m, size_t i) {
    GlExt<D> r;
    if constexpr (D == 1) {
        r.v[0] = m[i];
    } else {
        const ulonglong2 lo = *reinterpret_cast<const ulonglong2*>(m + i * (D == 3 ? 4 : 2));
        r.v[0] = lo.x; r.v[1] = lo.y;
        if constexpr (D == 3) r.v[2] = m[i * 4 + 2];
    }
    return r;
}
template <int D>
__device__ __forceinline__ void syn_st(u64* m, size_t i, const GlExt<D>& v) {
    if constexpr (D == 1) {
        m[i] = v.v[0];
    } else if constexpr (D == 2) {
        *reinterpret_cast<ulonglong2*>(m + i * 2) = make_ulonglong2(v.v[0], v.v[1]);
    } else {
        ulonglong2* o = reinterpret_cast<ulonglong2*>(m + i * 4);
        o[0] = make_ulonglong2(v.v[0], v.v[1]);
        o[1] = make_ulonglong2(v.v[2], 0);
    }
}
// this thread's run a over its rows [r0, r0 + SYN_ITEMS), both points, by Horner from the top row down (its p is b^SYN_ITEMS)
template <int D>
__device__ __forceinline__ void syn_thread_run(const u64* m, size_t n, size_t r0, const SynDivParams<D>& sp, GlExt<D> a[2]) {
#pragma unroll
    for (int pt = 0; pt < 2; pt++) a[pt] = ext_zero<D>();
#pragma unroll
    for (int k = SYN_ITEMS - 1; k >= 0; k--) {
        const GlExt<D> s = r0 + k < n ? syn_ld<D>(m, r0 + k) : ext_zero<D>();
#pragma unroll
        for (int pt = 0; pt < 2; pt++) a[pt] = ext_add(s, ext_mul(sp.b[pt], a[pt]));
    }
}
template <int D>
__device__ __forceinline__ GlExt<D> syn_shfl_ext(const GlExt<D>& v, u32 off) {
    GlExt<D> r;
#pragma unroll
    for (int q = 0; q < D; q++) r.v[q] = __shfl_down_sync(0xffffffffu, v.v[q], off);
    return r;
}
template <int D>
__device__ __forceinline__ void syn_st_ext(u64* p, const GlExt<D>& v) {
#pragma unroll
    for (int q = 0; q < D; q++) p[q] = v.v[q];
}
template <int D>
__global__ void __launch_bounds__(SYN_THREADS) syn_div_reduce(const u64* s, size_t n, SynDivParams<D> sp, SynDivBufs bufs) {
    __shared__ GlExt<D> wtot[2][SYN_WARPS];
    const u32 t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const size_t tile = blockIdx.x, r0 = tile * SYN_TILE + (size_t)t * SYN_ITEMS;
    GlExt<D> x[2];
    syn_thread_run<D>(s, n, r0, sp, x);
    // inclusive suffix over the warp: x = a of the rows of lanes lane..31. Where level k combines, x covers exactly 2^k lanes.
#pragma unroll
    for (int k = 0; k < 5; k++) {
#pragma unroll
        for (int pt = 0; pt < 2; pt++) {
            const GlExt<D> y = syn_shfl_ext(x[pt], 1u << k);
            if (lane + (1u << k) < 32) x[pt] = ext_add(x[pt], ext_mul(sp.lvl[pt][k], y));
        }
    }
    u64* ts = bufs.tsuf + (tile * SYN_THREADS + t) * 2 * D;
#pragma unroll
    for (int pt = 0; pt < 2; pt++) {
        GlExt<D> ex = syn_shfl_ext(x[pt], 1);   // the lanes above this one
        if (lane == 31) ex = ext_zero<D>();
        syn_st_ext(ts + pt * D, ex);
        if (lane == 0) wtot[pt][wid] = x[pt];
    }
    __syncthreads();
    if (wid == 0) {   // the same over the warp totals
#pragma unroll
        for (int pt = 0; pt < 2; pt++) {
            GlExt<D> w = lane < SYN_WARPS ? wtot[pt][lane] : ext_zero<D>();
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const GlExt<D> y = syn_shfl_ext(w, 1u << k);
                if (lane + (1u << k) < SYN_WARPS) w = ext_add(w, ext_mul(sp.lvl[pt][5 + k], y));
            }
            GlExt<D> ex = syn_shfl_ext(w, 1);   // the warps above
            if (lane + 1 >= SYN_WARPS) ex = ext_zero<D>();
            if (lane < SYN_WARPS) syn_st_ext(bufs.wsuf + ((tile * SYN_WARPS + lane) * 2 + pt) * D, ex);
            if (lane == 0) syn_st_ext(bufs.agg + (tile * 2 + pt) * D, w);
        }
    }
}
// one block; tile runs -> carry-in of every tile (q at its top row), in place. Thread t owns a run of consecutive tiles.
template <int D>
__global__ void __launch_bounds__(SYN_THREADS) syn_div_carry(u64* agg, size_t ntiles, SynDivParams<D> sp, u64* pw) {
    if (threadIdx.x < 2 * SYN_PW) {   // apply's power table
        const u32 pt = threadIdx.x / SYN_PW, j = threadIdx.x % SYN_PW;
        syn_st_ext(pw + (size_t)threadIdx.x * D, ext_pow(pt ? sp.b_items[1] : sp.b_items[0], j < 32 ? j : 32 * (j - 32)));
    }
    const size_t per = (ntiles + SYN_THREADS - 1) / SYN_THREADS;
    const size_t b = threadIdx.x * per < ntiles ? threadIdx.x * per : ntiles, e = b + per < ntiles ? b + per : ntiles;
    SynRun<D> mine;
#pragma unroll
    for (int pt = 0; pt < 2; pt++) { mine.a[pt] = ext_zero<D>(); mine.p[pt] = ext_from_base<D>(1); }
    for (size_t i = e; i-- > b;) {
#pragma unroll
        for (int pt = 0; pt < 2; pt++) {
            mine.a[pt] = ext_add(ld_ext<D>(agg + (i * 2 + pt) * D), ext_mul(sp.b_tile[pt], mine.a[pt]));
            mine.p[pt] = ext_mul(sp.b_tile[pt], mine.p[pt]);
        }
    }
    SynRun<D> total;
    const SynRun<D> above = syn_block_suffix<D>(mine, total);
    GlExt<D> run[2] = {above.a[0], above.a[1]};  // nothing lies above the last tile: q there is the run's a
    for (size_t i = e; i-- > b;) {
#pragma unroll
        for (int pt = 0; pt < 2; pt++) {
            u64* g = agg + (i * 2 + pt) * D;
            const GlExt<D> a = ld_ext<D>(g);
#pragma unroll
            for (int q = 0; q < D; q++) g[q] = run[pt].v[q];
            run[pt] = ext_add(a, ext_mul(sp.b_tile[pt], run[pt]));
        }
    }
}
template <int D>
__global__ void __launch_bounds__(SYN_THREADS) syn_div_apply(u64* s, size_t n, SynDivParams<D> sp, SynDivBufs bufs) {
    const u32 t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const size_t tile = blockIdx.x, r0 = tile * SYN_TILE + (size_t)t * SYN_ITEMS;
    GlExt<D> q[2];  // q at row r0 + SYN_ITEMS - 1
#pragma unroll
    for (int pt = 0; pt < 2; pt++) {
        const u64* pw = bufs.pw + (size_t)pt * SYN_PW * D;
        // q at the top row of this warp's rows: the warps above it in the tile, then the tile's carry-in (one lane computes it)
        GlExt<D> zw = ext_zero<D>();
        if (lane == 0)
            zw = ext_add(ld_ext<D>(bufs.wsuf + ((tile * SYN_WARPS + wid) * 2 + pt) * D),
                         ext_mul(ld_ext<D>(pw + (32 + SYN_WARPS - 1 - wid) * D), ld_ext<D>(bufs.agg + (tile * 2 + pt) * D)));
#pragma unroll
        for (int c = 0; c < D; c++) zw.v[c] = __shfl_sync(0xffffffffu, zw.v[c], 0);
        q[pt] = ext_add(ld_ext<D>(bufs.tsuf + ((tile * SYN_THREADS + t) * 2 + pt) * D), ext_mul(ld_ext<D>(pw + (31 - lane) * D), zw));
    }
#pragma unroll
    for (int k = SYN_ITEMS - 1; k >= 0; k--) {
        const size_t i = r0 + k;
        if (i >= n) continue;
        const GlExt<D> si = syn_ld<D>(s, i);
        syn_st<D>(s, i, ext_add(q[0], q[1]));
#pragma unroll
        for (int pt = 0; pt < 2; pt++) q[pt] = ext_add(si, ext_mul(sp.b[pt], q[pt]));
    }
}

// Proof-of-work grinding (K13; prover/src/channel.rs:169-184, crypto/src/random/default.rs:141-146):
// thread idx tests nonce = start + idx: trailing_zeros(LE u64 of merge_with_int(seed, nonce)[..8]) >=
// grinding. atomicMin keeps the SMALLEST qualifying nonce of the batch, and batches are scanned in
// increasing order, so the result is the serial-semantics nonce (the reference's `concurrent`
// find_any is nondeterministic; byte-identity is defined against the serial branch).
__global__ void __launch_bounds__(256) grind_kernel(int hash_id, const u64* seed /*4 words*/, u64 start, u64 count, u32 grinding,
                                                    unsigned long long* result) {
    u64 idx = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    u64 nonce = start + idx;
    u64 head;
    if (WF_HASH_IS_BLAKE3(hash_id)) {
        u32 ws[8], cv[8];
#pragma unroll
        for (int i = 0; i < 4; i++) { ws[2 * i] = (u32)seed[i]; ws[2 * i + 1] = (u32)(seed[i] >> 32); }
        if (hash_id == WF_HASH_BLAKE3_256) b3_merge_with_int_words<8>(ws, nonce, cv, b3_runtime_one());  // blake/mod.rs:41-46
        else b3_merge_with_int_words<6>(ws, nonce, cv, b3_runtime_one());                                 // :95-102
        head = (u64)cv[0] | ((u64)cv[1] << 32);
    } else {
        u64 sd[4], o[4];
#pragma unroll
        for (int i = 0; i < 4; i++) sd[i] = seed[i];
        if (hash_id == WF_HASH_RP64_256) alg_merge_with_int<WF_HASH_RP64_256>(sd, nonce, o);       // rp64_256/mod.rs:198-218
        else if (hash_id == WF_HASH_SHA3_256) alg_merge_with_int<WF_HASH_SHA3_256>(sd, nonce, o);  // sha/mod.rs:38-43
        else alg_merge_with_int<WF_HASH_RPJIVE64_256>(sd, nonce, o);                                // rp64_256_jive/mod.rs:206-229
        head = o[0];
    }
    u64 mask = grinding >= 64 ? ~0ULL : ((1ULL << grinding) - 1);
    if ((head & mask) == 0) atomicMin(result, (unsigned long long)nonce);
}

// =================================================================================================
// host orchestration
// =================================================================================================
static int grind_on_device(wf_ctx* ctx, int hash_id, const Digest& seed, u32 grinding, u64* nonce_out) {
    if (grinding == 0) { *nonce_out = 1; return WF_OK; }
    void *d_seed, *d_res;
    CKI(wf_dev_alloc(ctx, 32, &d_seed));
    CKI(wf_dev_alloc(ctx, 8, &d_res));
    CK(cudaMemcpyAsync(d_seed, seed.b, 32, cudaMemcpyHostToDevice, ctx->st));
    CK(cudaMemsetAsync(d_res, 0xff, 8, ctx->st));
    const u64 batch = WF_HASH_IS_BLAKE3(hash_id) ? (1ULL << 20) : (1ULL << 16);
    u64 start = 1, found = ~0ULL;
    while (found == ~0ULL) {
        grind_kernel<<<(unsigned)((batch + 255) / 256), 256, 0, ctx->st>>>(hash_id, (const u64*)d_seed, start, batch, grinding,
                                                                         (unsigned long long*)d_res);
        ctx->launches++;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(&found, d_res, 8, cudaMemcpyDeviceToHost, ctx->st));
        CK(cudaStreamSynchronize(ctx->st));
        start += batch;
    }
    wf_dev_free(ctx, d_seed);
    wf_dev_free(ctx, d_res);
    *nonce_out = found;
    return WF_OK;
}

namespace {

static AirHost fib_air_host(u32 k, size_t n, const u64* results) {
    AirHost a;
    a.w = 2 * k;
    a.pub_inputs.assign(results, results + k);
    a.is_fib = true; a.fib_k = k; a.fib_results.assign(results, results + k);
    for (u32 j = 0; j < k; j++) {
        a.degrees.push_back({1, {}});
        a.degrees.push_back({1, {}});
        a.asserts.push_back({2 * j, 0, 0, {(u64)(j + 1)}});
        a.asserts.push_back({2 * j + 1, 0, 0, {(u64)(j + 1)}});
        a.asserts.push_back({2 * j + 1, n - 1, 0, {results[j]}});
    }
    return a;
}

struct Channel {  // ProverChannel (prover/src/channel.rs)
    PublicCoin coin;
    ByteVec commitments;
    explicit Channel(int h, const std::vector<u64>& seed) : coin(h, seed.data(), seed.size()) {}
    void commit(const u8 root[32]) {  // commit_trace / commit_constraints / commit_fri_layer
        commitments.bytes(root, WF_DIGEST_BYTES(coin.hash_id));   // ByteDigest<N>::write_into: N bytes
        Digest d;
        memcpy(d.b, root, 32);
        coin.reseed(d);
    }
};

template <int D>
int upload_ext(wf_ctx* ctx, const std::vector<GlExt<D>>& v, size_t first, size_t count, u64** out) {
    void* p;
    CKI(wf_dev_alloc(ctx, std::max(count, (size_t)1) * D * 8, &p));
    std::vector<u64> flat(count * D);
    for (size_t i = 0; i < count; i++) for (int q = 0; q < D; q++) flat[i * D + q] = v[first + i].v[q];
    CK(cudaMemcpyAsync(p, flat.data(), flat.size() * 8, cudaMemcpyHostToDevice, ctx->st));
    CK(cudaStreamSynchronize(ctx->st));  // `flat` is a stack object
    *out = (u64*)p;
    return WF_OK;
}

// evaluate all columns of the coefficient matrices at z0 and z1 -> host vectors [cols][D]
// (out[2m] = mats[m] @ z0, out[2m+1] = mats[m] @ z1); one synchronisation for all matrices
template <int D>
int ood_eval(wf_ctx* ctx, const std::vector<const wf_mat*>& mats, const GlExt<D>& z0, const GlExt<D>& z1,
             std::vector<std::vector<GlExt<D>>>& out) {
    const int nm = (int)mats.size();
    DevScratch tmp(ctx);               // every buffer below returns to the pool on any exit
    std::vector<void*> part(nm);
    void* res;
    size_t total_cols = 0;
    for (auto* m : mats) total_cols += m->m.cols;
    out.assign(2 * nm, {});
    CKI(tmp.alloc(total_cols * 2 * D * 8, &res));
    size_t off = 0;
    std::vector<void*> zbs(nm, nullptr);
    for (int m = 0; m < nm; m++) {
        const size_t n = mats[m]->m.rows;
        const u32 chunks = (u32)((n + OOD_ROWS_PER_BLOCK - 1) / OOD_ROWS_PER_BLOCK);
        const u32 cols = mats[m]->m.cols;
        CKI(tmp.alloc((size_t)cols * chunks * 2 * D * 8, &part[m]));
        CKI(tmp.alloc((size_t)2 * (chunks + OOD_TAB) * D * 8, &zbs[m]));
        u64* zt = (u64*)zbs[m] + (size_t)2 * chunks * D;
        ood_pow_kernel<D><<<(2 * (chunks + OOD_TAB) + 127) / 128, 128, 0, ctx->st>>>(z0, z1, chunks, (u64*)zbs[m], zt);
        ood_partial_kernel<D><<<dim3(chunks, mats[m]->m.nseg()), 256, 0, ctx->st>>>(mats[m]->m, zt, (const u64*)zbs[m], (u64*)part[m], chunks);
        ood_reduce_kernel<D><<<(2 * cols * 32 + 255) / 256, 256, 0, ctx->st>>>((const u64*)part[m], cols, chunks, (u64*)res + off);
        ctx->launches += 3;
        CK(cudaGetLastError());
        off += (size_t)cols * 2 * D;
    }
    std::vector<u64> host(total_cols * 2 * D);
    CK(cudaMemcpyAsync(host.data(), res, host.size() * 8, cudaMemcpyDeviceToHost, ctx->st));
    CK(cudaStreamSynchronize(ctx->st));
    off = 0;
    for (int m = 0; m < nm; m++) {
        const u32 cols = mats[m]->m.cols;
        out[2 * m].resize(cols);
        out[2 * m + 1].resize(cols);
        for (u32 j = 0; j < cols; j++)
            for (int pt = 0; pt < 2; pt++)
                for (int q = 0; q < D; q++) out[2 * m + pt][j].v[q] = host[off + ((size_t)j * 2 + pt) * D + q];
        off += (size_t)cols * 2 * D;
    }
    return WF_OK;
}

// Queries::new (air/src/proof/queries.rs:51-78) + Serializable (:138-146), from batched gathers
void write_queries(const GatherBatch& gb, size_t row_id, size_t dig_id, size_t nvals, ByteVec& w) {
    ByteVec proof;
    wf_open_finish(gb.digs[dig_id].plan, gb.digest_result(dig_id), nullptr, proof);
    w.usize(nvals * 8);
    w.bytes(gb.row_result(row_id), nvals * 8);
    w.usize(proof.v.size());
    w.bytes(proof.v.data(), proof.v.size());
}

// Value table of a sequence assertion over the CE domain (LargePolyConstraint::new,
// prover/src/constraints/evaluator/boundary.rs:400-425): interpolate the L values over the size-L
// subgroup (air/src/air/boundary/constraint.rs:58-68), then evaluate that polynomial at 7 * w_ce^i for
// all i (coefficient k scaled by 7^k, zero-padded, one plain NTT of size ce). The reference's
// SmallPolyConstraint (Horner at x * g^(-first_step), :340-375) yields the same values, so one path
// serves both; the x offset becomes the row shift (i - first_step * ce_blowup) mod ce (:428-445).
static int sequence_table(wf_ctx* ctx, const u64* values, size_t L, u32 words_per_value, u32 dcols, size_t ce, wf_mat** out) {
    std::vector<u64> cols((size_t)dcols * L);
    std::vector<const u64*> ptr(dcols);
    for (u32 q = 0; q < dcols; q++) {
        for (size_t k = 0; k < L; k++) cols[q * L + k] = values[k * words_per_value + q];
        ptr[q] = &cols[q * L];
    }
    wf_mat *vals, *poly, *padded;
    CKI(wf_mat_from_host_columns(ctx, ptr.data(), dcols, L, 1, 0, &vals));  // synchronous w.r.t. `cols`
    CKI(wf_mat_interpolate(ctx, vals, &poly));
    wf_mat_free(ctx, vals);
    CKI(wf_mat_alloc(ctx, ce, dcols, &padded));
    CK(cudaMemsetAsync(padded->m.base, 0, padded->m.words() * 8, ctx->st));
    // dcols <= 3 -> one segment: the first L rows of `padded` are the L rows of `poly`
    CK(cudaMemcpyAsync(padded->m.base, poly->m.base, poly->m.words() * 8, cudaMemcpyDeviceToDevice, ctx->st));
    wf_mat_free(ctx, poly);
    CK(layout_scale_rows_by_powers(padded->m, GL_GENERATOR, ctx->st));
    ctx->launches++;
    int r = wf_mat_evaluate(ctx, padded, out);
    wf_mat_free(ctx, padded);
    return r;
}

// OUT j, v sets constraint j's value (result[dst] = r[a], include/winterfell_b200.h), as the verifiers evaluate it: of several
// OUTs of one constraint only the last one counts. The combining kernels add every OUT they run into the combination, so they
// get the program without the earlier ones (an OUT writes no register; dropping it changes nothing else).
static std::vector<u32> last_outs_only(const std::vector<u32>& prog) {
    std::vector<u32> out;
    std::vector<bool> seen;
    for (size_t k = prog.size() / 4; k-- > 0;) {
        const u32* in = &prog[4 * k];
        if (in[0] == 4) {
            if (in[1] >= seen.size()) seen.resize(in[1] + 1, false);
            if (seen[in[1]]) continue;
            seen[in[1]] = true;
        }
        out.insert(out.begin(), in, in + 4);
    }
    return out;
}

// DefaultConstraintEvaluator::evaluate (prover/src/constraints/evaluator/default.rs:60-118) fused with
// ConstraintEvaluationTable::combine (evaluation_table.rs:163-407): the combined, divisor-normalised
// constraint evaluations over the CE domain = CompositionPolyTrace, as a (n * ce_blowup) x D matrix.
// cc: main transition, aux transition, main assertions, aux assertions (sorted order).
template <int D>
int eval_constraints(wf_ctx* ctx, const AirHost& air, const wf_mat* lde, const wf_mat* alde, const std::vector<GlExt<D>>& cc,
                     const std::vector<u64>& rnd_flat, u32 log_n, u32 log_b, wf_mat** out, size_t row0 = 0, size_t ce_rows = 0,
                     u32 log_step = 0) {
    // ce_rows != 0: row-sharded call — CE rows [row0, row0 + ce_rows) only; `lde` (and `alde`) then hold the LDE rows of that
    // range followed by `blowup` halo rows (FibEvalParams::row0, GenEvalParams::row0)
    // log_step != 0: the sub-coset 7 <w_ce^(2^log_step)> only, row j of *out = CE row j << log_step (the rows the composition
    // polynomial is interpolated from, composition_polys)
    const size_t n = (size_t)1 << log_n;
    const u32 c = air.w, aw = air.aw, log_ceb = air.log_ce_blowup();
    const u32 n_atr = (u32)air.aux_degrees.size(), n_mtr = (u32)air.degrees.size(), n_mas = (u32)air.asserts.size();
    const u32 n_tr = n_mtr + n_atr;
    const size_t ce = n << log_ceb;
    if (log_step && (ce_rows || log_step > log_n + log_ceb)) return wf_fail(ctx, WF_ERR_INVALID, "CE row step with a row window, or past the domain");
    const size_t rows = ce_rows ? ce_rows : ce >> log_step;   // rows of *out
    wf_mat* comp;
    CKI(wf_mat_alloc(ctx, rows, D, &comp));
    if (comp->m.W > D) CK(cudaMemsetAsync(comp->m.base, 0, comp->m.words() * 8, ctx->st));
    const u64 g_tr = gl_root_of_unity(log_n);
    std::vector<u64> zt((size_t)1 << log_ceb);  // ce_blowup <= blowup <= 128 entries
    {   // x^n over the CE domain takes ce_blowup values: (7 w_ce^i)^n = 7^n * w_ceb^i
        u64 o_n = gl_pow(GL_GENERATOR, n), w_ceb = gl_root_of_unity(log_ceb);
        for (u32 i = 0; i < (1u << log_ceb); i++) zt[i] = gl_inv(gl_sub(gl_mul(o_n, gl_pow(w_ceb, i)), 1));
    }
    // device buffers of this stage; `comp` too until it is handed to the caller (returned to the pool on every error path)
    struct StageBufs {
        DevScratch dev;
        wf_mat* comp;
        std::vector<wf_mat*> mats;
        StageBufs(wf_ctx* c, wf_mat* m) : dev(c), comp(m) {}
        ~StageBufs() { if (comp) wf_mat_free(dev.ctx, comp); for (wf_mat* t : mats) wf_mat_free(dev.ctx, t); }
    } stage(ctx, comp);
    auto upload = [&](const void* src, size_t bytes, void** out) -> int {
        void* p;
        CKI(stage.dev.alloc(std::max(bytes, (size_t)8), &p));
        // stream-ordered copy; the (pageable) source vectors stay alive until the synchronisation below
        if (bytes) CK(cudaMemcpyAsync(p, src, bytes, cudaMemcpyHostToDevice, ctx->st));
        *out = p;
        return WF_OK;
    };
    auto flat = [&](size_t first, size_t count) {
        std::vector<u64> f(count * D);
        for (size_t i = 0; i < count; i++) for (int q = 0; q < D; q++) f[i * D + q] = cc[first + i].v[q];
        return f;
    };
    if (air.is_fib) {
        // boundary coefficients follow the assertions sorted by (stride, first_step, column)
        // (air/src/air/assertions/mod.rs:301-315): 2k assertions at step 0, then k at step n-1
        const u32 k = air.fib_k;
        void* d_cf = nullptr;
        std::vector<u64> cf((size_t)k * 5 * D);
        GlExt<D> K0 = ext_zero<D>(), K1 = ext_zero<D>();
        for (u32 j = 0; j < k; j++) {
            const GlExt<D>&tc0 = cc[2 * j], &tc1 = cc[2 * j + 1], &b0a = cc[n_tr + 2 * j], &b0b = cc[n_tr + 2 * j + 1], &b1 = cc[n_tr + 2 * k + j];
            for (int q = 0; q < D; q++) {
                u64* o = &cf[(size_t)j * 5 * D];
                o[q] = tc0.v[q]; o[D + q] = tc1.v[q]; o[2 * D + q] = b0a.v[q]; o[3 * D + q] = b0b.v[q]; o[4 * D + q] = b1.v[q];
            }
            // asserted values: columns 2j and 2j+1 start at j + 1, column 2j+1 ends at results[j] (fib_air_host)
            K0 = ext_add(K0, ext_mul_base(ext_add(b0a, b0b), (u64)(j + 1)));
            K1 = ext_add(K1, ext_mul_base(b1, air.fib_results[j]));
        }
        CKI(upload(cf.data(), cf.size() * 8, &d_cf));
        FibEvalParams p;
        memset(&p, 0, sizeof(p));
        p.lde = lde->m; p.out = comp->m; p.k = k; p.log_n = log_n; p.log_blowup = log_b; p.log_ce_blowup = log_ceb;
        p.coef = (const u64*)d_cf;
        for (int q = 0; q < D; q++) { p.K0[q] = K0.v[q]; p.K1[q] = K1.v[q]; }
        CKI(wf_get_twiddles(ctx, log_n + log_ceb, &p.tw_ce));
        p.last = gl_pow(g_tr, n - 1);
        if (log_ceb > 3) return wf_fail(ctx, WF_ERR_STATE, "FibSmall has degree-1 constraints");  // FibEvalParams::zt[8]
        for (u32 i = 0; i < (1u << log_ceb); i++) p.zt[i] = zt[i];
        p.row0 = row0; p.ce_rows = ce_rows; p.log_step = log_step;
        const size_t rows_per_thread = D == 3 ? FIB_ROWS_D3 : 4;
        size_t threads = (rows + rows_per_thread - 1) / rows_per_thread;
        fib_constraints_kernel<D><<<(unsigned)((threads + 255) / 256), 256, cf.size() * 8, ctx->st>>>(p);
        ctx->launches++;
        CK(cudaGetLastError());
    } else {
        GenEvalParams p;
        memset(&p, 0, sizeof(p));
        p.lde = lde->m; p.out = comp->m; p.w = c; p.log_n = log_n; p.log_blowup = log_b; p.log_ce_blowup = log_ceb;
        const std::vector<u32> prog = last_outs_only(air.prog), aprog = last_outs_only(air.aux_prog);
        p.prog_len = (u32)(prog.size() / 4); p.num_regs = air.num_regs; p.num_periodic = (u32)air.periodic.size(); p.num_tc = n_mtr;
        void* dp = nullptr;
        CKI(upload(prog.data(), prog.size() * 4, &dp)); p.prog = (u32*)dp;
        CKI(upload(air.consts.data(), air.consts.size() * 8, &dp)); p.consts = (u64*)dp;
        // periodic value tables (evaluator/periodic_table.rs:24-76): poly_j over offset^(n/L) <w_(L*ceb)>
        std::vector<u64> ptab;
        std::vector<u32> poff, plen;
        air.periodic_ce_tables(n, log_ceb, ptab, poff, plen);
        CKI(upload(ptab.data(), ptab.size() * 8, &dp)); p.ptab = (u64*)dp;
        CKI(upload(poff.data(), poff.size() * 4, &dp)); p.ptab_off = (u32*)dp;
        CKI(upload(plen.data(), plen.size() * 4, &dp)); p.ptab_len = (u32*)dp;
        auto f0 = flat(0, n_mtr);
        CKI(upload(f0.data(), f0.size() * 8, &dp)); p.tcoef = (u64*)dp;
        // boundary groups: BTreeMap keyed by (stride, first_step) (air/src/air/boundary/mod.rs:154),
        // coefficients assigned in sorted-assertion order; divisor x^a - g^(a*first_step) (divisor.rs:44-56)
        auto as = air.sorted_assertions();
        std::map<std::pair<u64, u64>, std::vector<size_t>> groups;
        for (size_t i = 0; i < as.size(); i++) groups[{as[i].stride, as[i].first_step}].push_back(i);
        std::vector<u32> goff = {0}, ecol, etstride, eshift;
        std::vector<u64> ga, gb, goa, eval, ecc;
        std::vector<const u64*> etab;
        std::vector<wf_mat*>& seq_tables = stage.mats;  // returned to the pool when the stage ends (stream-ordered: after the kernel)
        for (auto& kv : groups) {
            u64 a = kv.first.first == 0 ? 1 : n / kv.first.first;
            ga.push_back(a);
            gb.push_back(kv.first.second == 0 ? 1 : gl_pow(g_tr, a * kv.first.second));
            goa.push_back(gl_pow(GL_GENERATOR, a));
            for (size_t i : kv.second) {
                ecol.push_back((u32)as[i].column); eval.push_back(as[i].values[0]);
                for (int q = 0; q < D; q++) ecc.push_back(cc[n_tr + i].v[q]);
                if (as[i].values.size() > 1) {
                    wf_mat* t;
                    CKI(sequence_table(ctx, as[i].values.data(), as[i].values.size(), 1, 1, ce, &t));
                    seq_tables.push_back(t);
                    etab.push_back(t->m.base); etstride.push_back((u32)t->m.W);
                    eshift.push_back((u32)(((u64)as[i].first_step << log_ceb) & (ce - 1)));
                } else { etab.push_back(nullptr); etstride.push_back(0); eshift.push_back(0); }
            }
            goff.push_back((u32)ecol.size());
        }
        p.num_groups = (u32)ga.size();
        CKI(upload(goff.data(), goff.size() * 4, &dp)); p.g_off = (u32*)dp;
        CKI(upload(ga.data(), ga.size() * 8, &dp)); p.g_a = (u64*)dp;
        CKI(upload(gb.data(), gb.size() * 8, &dp)); p.g_b = (u64*)dp;
        CKI(upload(goa.data(), goa.size() * 8, &dp)); p.g_oa = (u64*)dp;
        CKI(upload(ecol.data(), ecol.size() * 4, &dp)); p.e_col = (u32*)dp;
        CKI(upload(eval.data(), eval.size() * 8, &dp)); p.e_val = (u64*)dp;
        CKI(upload(ecc.data(), ecc.size() * 8, &dp)); p.e_cc = (u64*)dp;
        CKI(upload(etab.data(), etab.size() * 8, &dp)); p.e_tab = (const u64* const*)dp;
        CKI(upload(etstride.data(), etstride.size() * 4, &dp)); p.e_tstride = (u32*)dp;
        CKI(upload(eshift.data(), eshift.size() * 4, &dp)); p.e_shift = (u32*)dp;
        CKI(wf_get_twiddles(ctx, log_n + log_ceb, &p.tw_ce));
        CKI(upload(zt.data(), zt.size() * 8, &dp)); p.zt = (const u64*)dp;
        p.row0 = row0; p.ce_rows = ce_rows; p.log_step = log_step;
        p.num_exempt = air.exemptions;
        for (u32 e = 0; e < air.exemptions; e++) p.exempt[e] = gl_pow(g_tr, n - air.exemptions + e);  // divisor.rs:31-41
        std::vector<u32> agoff = {0}, aecol, aetstride, aeshift;
        std::vector<u64> aga, agb, agoa, aeval, aecc, fa;
        std::vector<const u64*> aetab;
        if (aw) {
            p.alde = alde->m; p.aw = aw; p.nr = air.nr; p.aprog_len = (u32)(aprog.size() / 4);
            CKI(upload(aprog.data(), aprog.size() * 4, &dp)); p.aprog = (u32*)dp;
            CKI(upload(rnd_flat.data(), rnd_flat.size() * 8, &dp)); p.rnd = (u64*)dp;
            fa = flat(n_mtr, n_atr);
            CKI(upload(fa.data(), fa.size() * 8, &dp)); p.atcoef = (u64*)dp;
            auto aas = air.sorted_aux_assertions();
            std::map<std::pair<u64, u64>, std::vector<size_t>> agroups;
            for (size_t i = 0; i < aas.size(); i++) agroups[{aas[i].stride, aas[i].first_step}].push_back(i);
            for (auto& kv : agroups) {
                u64 a = kv.first.first == 0 ? 1 : n / kv.first.first;
                aga.push_back(a);
                agb.push_back(kv.first.second == 0 ? 1 : gl_pow(g_tr, a * kv.first.second));
                agoa.push_back(gl_pow(GL_GENERATOR, a));
                for (size_t i : kv.second) {
                    aecol.push_back((u32)aas[i].column);
                    for (int q = 0; q < D; q++) { aeval.push_back(aas[i].values[q]); aecc.push_back(cc[n_tr + n_mas + i].v[q]); }
                    if (aas[i].values.size() > 3) {
                        wf_mat* t;
                        CKI(sequence_table(ctx, aas[i].values.data(), aas[i].values.size() / 3, 3, D, ce, &t));
                        seq_tables.push_back(t);
                        aetab.push_back(t->m.base); aetstride.push_back((u32)t->m.W);
                        aeshift.push_back((u32)(((u64)aas[i].first_step << log_ceb) & (ce - 1)));
                    } else { aetab.push_back(nullptr); aetstride.push_back(0); aeshift.push_back(0); }
                }
                agoff.push_back((u32)aecol.size());
            }
            p.num_agroups = (u32)aga.size();
            CKI(upload(agoff.data(), agoff.size() * 4, &dp)); p.ag_off = (u32*)dp;
            CKI(upload(aga.data(), aga.size() * 8, &dp)); p.ag_a = (u64*)dp;
            CKI(upload(agb.data(), agb.size() * 8, &dp)); p.ag_b = (u64*)dp;
            CKI(upload(agoa.data(), agoa.size() * 8, &dp)); p.ag_oa = (u64*)dp;
            CKI(upload(aecol.data(), aecol.size() * 4, &dp)); p.ae_col = (u32*)dp;
            CKI(upload(aeval.data(), aeval.size() * 8, &dp)); p.ae_val = (u64*)dp;
            CKI(upload(aecc.data(), aecc.size() * 8, &dp)); p.ae_cc = (u64*)dp;
            CKI(upload(aetab.data(), aetab.size() * 8, &dp)); p.ae_tab = (const u64* const*)dp;
            CKI(upload(aetstride.data(), aetstride.size() * 4, &dp)); p.ae_tstride = (u32*)dp;
            CKI(upload(aeshift.data(), aeshift.size() * 4, &dp)); p.ae_shift = (u32*)dp;
        }
        // the kernel compiled for this AIR (NVRTC, jit.cu) when there is one, else the interpreter
        cudaKernel_t jk = nullptr;
        const bool jit = ctx->jit_enabled &&
                         wf_jit_get_kernel(ctx, wf_jit_source(D, air.w, (u32)air.periodic.size(), air.num_regs, prog, air.consts, aw, air.nr,
                                                              air.aux_num_regs, aprog), &jk) == WF_OK;
        const unsigned blocks = (unsigned)((rows + 127) / 128);
        if (jit) {
            void* args[] = {&p};
            CK(cudaLaunchKernel((const void*)jk, dim3(blocks), dim3(128), args, 0, ctx->st));
        } else if (aw) {
            generic_constraints_kernel<D, true><<<blocks, 128, 0, ctx->st>>>(p);
        } else {
            generic_constraints_kernel<D, false><<<blocks, 128, 0, ctx->st>>>(p);
        }
        ctx->launches++;
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(ctx->st));
    stage.comp = nullptr;   // the caller's now
    *out = comp;
    return WF_OK;
}

// DefaultConstraintCommitment::new (prover/src/constraints/commitment/default.rs:44-150): composition
// trace (CE-domain evaluations, ce x D) -> CompositionPoly columns (n x kc*D coefficient matrix,
// composition_poly.rs:58-78,128-140), their LDE (N x kc*D) and the row commitment.
// The composition polynomial has degree < kc * n by the AIR's declared degrees (that is what kc is computed from), so the
// evaluations on the sub-coset 7 <w_m>, m = the power of two >= kc * n — every (ce / m)-th row of the CE domain — already
// determine it: the size-m inverse transform returns exactly the coefficients the reference reads out of its size-ce one
// (whose upper ce - kc * n coefficients are zero, composition_poly.rs:64-70). For FibSmall m = n = ce / 2.
static size_t comp_subcoset_rows(size_t n, u32 kc) {
    size_t m = n;
    while (m < n * kc) m <<= 1;
    return m;
}
// CompositionPoly::new (composition_poly.rs:58-78): CE-domain evaluations -> kc column polynomials of degree < n. `comp` holds
// either the whole CE domain or only the comp_subcoset_rows(n, kc) rows of the sub-coset.
int composition_polys(wf_ctx* ctx, const wf_mat* comp, u32 log_n, int D, u32 kc, wf_mat** polys_out) {
    const size_t n = (size_t)1 << log_n;
    if (comp->m.rows < n * kc || (int)comp->m.cols != D) return wf_fail(ctx, WF_ERR_INVALID, "composition trace shape");
    wf_mat *ccoefs, *cpolys;
    const size_t m = comp_subcoset_rows(n, kc);
    if (m < comp->m.rows && comp->m.nseg() == 1) {
        wf_mat* sub;
        CKI(wf_mat_alloc_w(ctx, m, comp->m.cols, comp->m.W, &sub));
        const size_t rb = (size_t)comp->m.W * 8, stride = comp->m.rows / m;
        cudaError_t e = cudaMemcpy2DAsync(sub->m.base, rb, comp->m.base, stride * rb, rb, m, cudaMemcpyDeviceToDevice, ctx->st);
        int rc = e == cudaSuccess ? wf_mat_interpolate_with_offset(ctx, sub, GL_GENERATOR, &ccoefs)
                                  : wf_fail(ctx, WF_ERR_CUDA, "composition sub-coset copy: %s", cudaGetErrorString(e));
        wf_mat_free(ctx, sub);
        if (rc != WF_OK) return rc;
    } else {
        CKI(wf_mat_interpolate_with_offset(ctx, comp, GL_GENERATOR, &ccoefs));
    }
    if (kc == 1 && ccoefs->m.rows == n) {   // one column: the coefficients as they are, in the layout of an n x D matrix
        wf_mark(ctx, "composition_interpolate");
        *polys_out = ccoefs;
        return WF_OK;
    }
    CKI(wf_mat_alloc(ctx, n, kc * D, &cpolys));
    if (cpolys->m.W > (int)(kc * D)) CK(cudaMemsetAsync(cpolys->m.base, 0, cpolys->m.words() * 8, ctx->st));
    comp_split_kernel<<<(unsigned)((n * kc * D + 255) / 256), 256, 0, ctx->st>>>(ccoefs->m, n, kc, D, cpolys->m);
    ctx->launches++;
    CK(cudaGetLastError());
    wf_mat_free(ctx, ccoefs);
    wf_mark(ctx, "composition_interpolate");
    *polys_out = cpolys;
    return WF_OK;
}
// The LDE of the composition columns. With one column interpolated from n rows, those rows are the column's values at 7 w_n^j:
// coset 0 of the LDE (rows b*j), which the interpolant reproduces exactly. They are copied there, and only cosets 1..b-1 are
// transformed.
static int composition_lde(wf_ctx* ctx, const wf_mat* comp, const wf_mat* cpolys, u32 log_n, u32 log_b, u32 kc, wf_mat** lde_out) {
    const size_t n = (size_t)1 << log_n;
    if (kc != 1 || comp->m.rows != n || comp->m.nseg() != 1 || comp->m.W != cpolys->m.W || cpolys->m.nseg() != 1)
        return wf_mat_lde(ctx, cpolys, log_b, lde_out);
    if (log_b > 7 || log_n + log_b > 32) return wf_fail(ctx, WF_ERR_INVALID, "bad blowup");
    const u32 b = 1u << log_b;
    wf_mat* clde;
    CKI(wf_mat_alloc(ctx, n << log_b, cpolys->m.cols, &clde));
    // a kernel rather than cudaMemcpy2DAsync, which is slow on rows this narrow (32 bytes for the cubic extension)
    coset0_rows_kernel<<<(unsigned)((n * comp->m.W + 255) / 256), 256, 0, ctx->st>>>(comp->m.base, n, comp->m.W, b, clde->m.base);
    ctx->launches++;
    const cudaError_t e = cudaGetLastError();
    int r = e == cudaSuccess ? wf_mat_lde_from_coset(ctx, cpolys, log_b, 1, clde)
                             : wf_fail(ctx, WF_ERR_CUDA, "composition coset 0 copy: %s", cudaGetErrorString(e));
    if (r != WF_OK) { wf_mat_free(ctx, clde); return r; }
    *lde_out = clde;
    return WF_OK;
}
int composition_commit(wf_ctx* ctx, int h, const wf_mat* comp, u32 log_n, u32 log_b, int D, u32 kc, wf_mat** polys_out,
                       wf_mat** lde_out, wf_tree** tree_out, u32 partition_words = 0) {
    wf_mat *cpolys = nullptr, *clde = nullptr;
    CKI(composition_polys(ctx, comp, log_n, D, kc, &cpolys));
    int r = composition_lde(ctx, comp, cpolys, log_n, log_b, kc, &clde);
    if (r == WF_OK) {
        wf_mark(ctx, "composition_lde");
        if (tree_out) r = wf_commit_rows_partitioned(ctx, h, clde, partition_words, tree_out);  // sharded proofs commit their own row range
    }
    if (r != WF_OK) { wf_mat_free(ctx, cpolys); wf_mat_free(ctx, clde); return r; }
    *polys_out = cpolys;
    *lde_out = clde;
    return WF_OK;
}

// DeepCompositionPoly::{add_trace_polys, add_composition_poly, evaluate} (prover/src/composer/mod.rs:67-210)
// in evaluation form over the LDE domain (see the header of this file). dc: c + aw + kc coefficients.
template <int D>
int deep_compose(wf_ctx* ctx, const wf_mat* lde, const wf_mat* alde, const wf_mat* clde, u32 kc, u32 log_N,
                 const std::vector<GlExt<D>>& dc, const GlExt<D>& z, const GlExt<D>& zg, const GlExt<D>& Sz, const GlExt<D>& Szg,
                 wf_mat** out, size_t row0 = 0, size_t nrows = 0) {
    // nrows != 0: row-sharded call — the matrices hold LDE rows [row0, row0 + nrows) only
    const u32 c = lde->m.cols, aw = alde ? alde->m.cols / D : 0, ct = c + aw;
    const size_t N = nrows ? nrows : ((size_t)1 << log_N);
    // x - z vanishes at a row x = 7 w_N^i only for z in the base field with (z / 7)^N = 1 (outside the base field the norm of x - z
    // is nonzero); the batch inversion would then zero the inverses of a whole thread's rows, so such a point is refused
    for (const GlExt<D>* w : {&z, &zg}) {
        bool base = true;
        for (int q = 1; q < D; q++) base = base && w->v[q] == 0;
        if (base && gl_sqr_n(gl_mul(w->v[0], 2635249152773512046ULL), (int)log_N) == 1)  // 7^-1 mod p
            return wf_fail(ctx, WF_ERR_INVALID, "DEEP point %s lies on the LDE domain: its denominators vanish", w == &z ? "z" : "z*g");
    }
    DeepPoint<D> pz, pzg;
    if (!deep_point<D>(z, pz) || !deep_point<D>(zg, pzg)) return wf_fail(ctx, WF_ERR_STATE, "conjugates of the out-of-domain point are inconsistent");
    u64 *d_dt, *d_dq, *d_da;
    CKI(upload_ext<D>(ctx, dc, 0, ct + kc, &d_dt));  // one upload (one synchronisation) for all coefficients
    d_da = d_dt + (size_t)c * D;
    d_dq = d_dt + (size_t)ct * D;
    wf_mat* deep;
    CKI(wf_mat_alloc(ctx, N, D, &deep));
    DeepParams p;
    p.trace = lde->m; p.cons = clde->m; p.out = deep->m; p.c = c; p.kc = kc; p.log_N = log_N;
    p.row0 = row0; p.nrows = nrows;
    p.tcc = d_dt; p.ccc = d_dq; p.acc = d_da; p.aw = aw;
    p.aux = aw ? alde->m : lde->m;
    CKI(wf_get_twiddles(ctx, log_N, &p.tw_N));
    const size_t coef_bytes = (size_t)(c + aw + kc) * D * 8;
    deep_sum_kernel<D><<<(unsigned)((N + DEEP_SUM_THREADS - 1) / DEEP_SUM_THREADS), DEEP_SUM_THREADS, coef_bytes, ctx->st>>>(p);
    const size_t rows_per_thread = DEEP_ROWS;
    size_t threads = (N + rows_per_thread - 1) / rows_per_thread;
    deep_div_kernel<D><<<(unsigned)((threads + 255) / 256), 256, 0, ctx->st>>>(p, pz, pzg, Sz, Szg);
    ctx->launches += 2;
    CK(cudaGetLastError());
    // the coefficient buffers are pool allocations on the same stream: safe to release after the launch
    wf_dev_free(ctx, d_dt);
    *out = deep;
    return WF_OK;
}

// The same DEEP composition in coefficient form (see syn_div_*): polys n x c, apolys n x aw*D (nullptr: single segment), cpolys
// n x kc*D coefficient matrices -> the N x D LDE of the quotient, N = n << log_b, the matrix deep_compose returns. It reads the
// coefficients (8(c + a·d + k·d) B per coefficient row) instead of the LDE rows.
template <int D>
int deep_compose_polys(wf_ctx* ctx, const wf_mat* polys, const wf_mat* apolys, const wf_mat* cpolys, u32 kc, u32 log_b,
                       const std::vector<GlExt<D>>& dc, const GlExt<D>& z, const GlExt<D>& zg, wf_mat** out) {
    const u32 c = polys->m.cols, aw = apolys ? apolys->m.cols / D : 0, ct = c + aw;
    const size_t n = polys->m.rows, ntiles = (n + SYN_TILE - 1) / SYN_TILE;
    const u32 log_n = log2_ceil(n);
    DevScratch tmp(ctx);
    u64* d_dt;
    CKI(upload_ext<D>(ctx, dc, 0, ct + kc, &d_dt));
    tmp.bufs.push_back(d_dt);
    void* d_agg;
    CKI(tmp.alloc((ntiles * (1 + SYN_WARPS + SYN_THREADS) + SYN_PW) * 2 * D * 8, &d_agg));
    SynDivBufs sb;
    sb.agg = (u64*)d_agg;
    sb.wsuf = sb.agg + ntiles * 2 * D;
    sb.tsuf = sb.wsuf + ntiles * SYN_WARPS * 2 * D;
    sb.pw = sb.tsuf + ntiles * SYN_THREADS * 2 * D;
    wf_mat* quot;
    CKI(wf_mat_alloc(ctx, n, D, &quot));
    DeepParams p{};
    p.trace = polys->m; p.cons = cpolys->m; p.out = quot->m; p.c = c; p.kc = kc; p.log_N = log_n;
    p.tcc = d_dt; p.acc = d_dt + (size_t)c * D; p.ccc = d_dt + (size_t)ct * D; p.aw = aw;
    p.aux = aw ? apolys->m : polys->m;
    deep_sum_kernel<D><<<(unsigned)((n + DEEP_SUM_THREADS - 1) / DEEP_SUM_THREADS), DEEP_SUM_THREADS, (size_t)(ct + kc) * D * 8, ctx->st>>>(p);
    SynDivParams<D> sp;
    sp.b[0] = z; sp.b[1] = zg;
    for (int pt = 0; pt < 2; pt++) {
        sp.b_items[pt] = ext_pow(sp.b[pt], SYN_ITEMS);
        sp.b_tile[pt] = ext_pow(sp.b[pt], SYN_TILE);
        sp.lvl[pt][0] = sp.b_items[pt];
        for (int k = 1; k < 8; k++) sp.lvl[pt][k] = ext_mul(sp.lvl[pt][k - 1], sp.lvl[pt][k - 1]);
    }
    syn_div_reduce<D><<<(unsigned)ntiles, SYN_THREADS, 0, ctx->st>>>(quot->m.base, n, sp, sb);
    syn_div_carry<D><<<1, SYN_THREADS, 0, ctx->st>>>(sb.agg, ntiles, sp, sb.pw);
    syn_div_apply<D><<<(unsigned)ntiles, SYN_THREADS, 0, ctx->st>>>(quot->m.base, n, sp, sb);
    ctx->launches += 4;
    const cudaError_t e = cudaGetLastError();
    // the quotient and the scratch go back to the pool in stream order, behind the LDE that reads them
    const int r = e == cudaSuccess ? wf_mat_lde(ctx, quot, log_b, out) : wf_fail(ctx, WF_ERR_CUDA, "DEEP quotient launch: %s", cudaGetErrorString(e));
    wf_mat_free(ctx, quot);
    return r;
}

// wf_ctx_set_validation: a violation found by a check stops the call with the reference's panic message
static int validation_result(wf_ctx* ctx, int r, const TraceReport& rep) {
    if (r != WF_OK) return r;
    return rep.kind == WF_VALID ? WF_OK : wf_fail(ctx, WF_ERR_INVALID, "%s", rep.msg.c_str());
}

// Device objects of one proof: whatever is still registered when prove_air leaves (normally or through
// an error return) goes back to the context's pool. `held` trees and `bufs` buffers are owned by value.
struct ProofScope {
    wf_ctx* ctx;
    std::vector<wf_mat**> mats;
    std::vector<wf_tree**> trees;
    std::vector<wf_tree*> held;
    DevScratch bufs;
    wf_fri** fri = nullptr;
    explicit ProofScope(wf_ctx* c) : ctx(c), bufs(c) {}
    void own(std::initializer_list<wf_mat**> l) { mats.insert(mats.end(), l); }
    void own(std::initializer_list<wf_tree**> l) { trees.insert(trees.end(), l); }
    void drop(wf_mat*& m) { wf_mat_free(ctx, m); m = nullptr; }
    ~ProofScope() {
        for (wf_tree* t : held) wf_tree_free(ctx, t);
        if (fri && *fri) wf_fri_free(ctx, *fri);
        for (wf_mat** m : mats) if (*m) wf_mat_free(ctx, *m);
        for (wf_tree** t : trees) if (*t) wf_tree_free(ctx, *t);
    }
};

// ---- the steps both provers (prove_air, prove_sharded) take in the same way ----

// Air::get_aux_rand_elements (air/src/air/mod.rs:292-306): rnd <- nr elements drawn from the coin, [nr][D] canonical;
// rnd_user <- the same as the user's callbacks see them (x * R, R = 2^64 mod p, when `mont`)
template <int D>
static void draw_aux_rand(PublicCoin& coin, u32 nr, int mont, std::vector<u64>& rnd, std::vector<u64>& rnd_user) {
    for (u32 i = 0; i < nr; i++) { GlExt<D> e = draw_ext<D>(coin); for (int q = 0; q < D; q++) rnd.push_back(e.v[q]); }
    rnd_user = rnd;
    if (mont) for (u64& v : rnd_user) v = gl_mul(v, 0xFFFFFFFFULL);
}
// Air::get_aux_assertions(aux_rand_elements) (air/src/air/mod.rs:279): the callback (none: nothing to do) rewrites the
// aux assertion values of `air`
static int apply_aux_assertions(wf_ctx* ctx, AirHost& air, wf_aux_assertions_fn aux_assertions, void* aux_user,
                                const std::vector<u64>& rnd_user, int D, int mont) {
    if (!aux_assertions) return WF_OK;
    std::vector<u64> vals = get_aux_assertion_words(air, D, mont);
    if (aux_assertions(aux_user, rnd_user.data(), vals.data()) != 0) return wf_fail(ctx, WF_ERR_INVALID, "aux assertion callback failed");
    if (!set_aux_assertion_words(air, vals.data(), D, mont))
        return wf_fail(ctx, WF_ERR_INVALID, "aux assertion value is not a canonical field element");
    return WF_OK;
}

// The out-of-domain frames (lib.rs:392-401) and their serialisation
template <int D>
struct OodFrame { std::vector<GlExt<D>> t_cur, t_nxt, q_cur, q_nxt; ByteVec t, q; };
// f.t_cur / f.t_nxt: the main columns at z / zg; q[0..1] (a[0..1]: the aux segment's, or none): the composition columns'
// base components at z / zg. Trace frame rows = main then aux columns (ood_frame.rs:40-72); the coin is reseeded with the
// frames' hash, which is not added to the commitments.
template <int D>
static void ood_frame(Channel& ch, OodFrame<D>& f, const std::vector<GlExt<D>>* q, const std::vector<GlExt<D>>* a) {
    if (a) {
        auto a_cur = ext_from_components<D>(a[0]), a_nxt = ext_from_components<D>(a[1]);
        f.t_cur.insert(f.t_cur.end(), a_cur.begin(), a_cur.end());
        f.t_nxt.insert(f.t_nxt.end(), a_nxt.begin(), a_nxt.end());
    }
    f.q_cur = ext_from_components<D>(q[0]);
    f.q_nxt = ext_from_components<D>(q[1]);
    ch.coin.reseed(ood_frames<D>(ch.coin.hash_id, f.t_cur, f.t_nxt, f.q_cur, f.q_nxt, &f.t, &f.q));
}

// grinding + query positions (channel.rs:151-184; serial semantics: smallest nonce) over an LDE domain of N points
static int grind_and_query(wf_ctx* ctx, Channel& ch, const Options& o, size_t N, u64* nonce, std::vector<u64>& pos) {
    CKI(grind_on_device(ctx, ch.coin.hash_id, ch.coin.seed, o.grinding, nonce));
    if (ch.coin.check_leading_zeros(*nonce) < o.grinding) return wf_fail(ctx, WF_ERR_STATE, "grinding self-check failed");
    if (!query_positions(ch.coin, o.num_queries, N, *nonce, pos)) return wf_fail(ctx, WF_ERR_STATE, "failed to draw query positions");
    return WF_OK;
}

// The ids in a GatherBatch of the opened rows and their Merkle openings: trace, constraint, aux (with an aux segment). The
// rows at positions `p` are queued here, the openings by the caller.
struct QueryIds {
    size_t tr_rows, cr_rows, ar_rows, tr_dig = 0, cr_dig = 0, ar_dig = 0;
    QueryIds(GatherBatch& gb, const SegMatrix& t, const SegMatrix& c, const SegMatrix* a, const std::vector<u64>& p)
        : tr_rows(gb.add_rows(t, p)), cr_rows(gb.add_rows(c, p)), ar_rows(a ? gb.add_rows(*a, p) : 0) {}
};
// The proof object (lib.rs:464-489; air/src/proof/mod.rs:189-200) once every gather of `gb` has run. `before`: the sharded
// prover's FRI layers folded on its shards, which come ahead of the layers of `fri`.
template <int D>
static void write_proof(const AirHost& air, u32 log_n, const Options& o, const Channel& ch, const std::vector<u64>& pos,
                        const GatherBatch& gb, const QueryIds& id, const OodFrame<D>& ood, const wf_fri* fri,
                        const FriProofPlan& fplan, const FriProofPlan* before, u64 nonce, std::vector<u8>& proof_out) {
    ByteVec w;
    write_context(w, air, log_n, o);
    w.u8_((u8)pos.size());
    w.u16_((uint16_t)ch.commitments.v.size());
    w.bytes(ch.commitments.v.data(), ch.commitments.v.size());
    write_queries(gb, id.tr_rows, id.tr_dig, pos.size() * air.w, w);
    if (air.aw) write_queries(gb, id.ar_rows, id.ar_dig, pos.size() * air.aw * D, w);  // trace_lde/default/mod.rs:199-218
    write_queries(gb, id.cr_rows, id.cr_dig, pos.size() * air.num_comp_cols((size_t)1 << log_n) * D, w);
    w.u16_((uint16_t)ood.t.v.size()); w.bytes(ood.t.v.data(), ood.t.v.size());
    w.u16_((uint16_t)ood.q.v.size()); w.bytes(ood.q.v.data(), ood.q.v.size());
    wf_fri_finish_proof(fri, gb, fplan, w, before);
    w.u64_(nonce);
    proof_out.swap(w.v);
}

template <int D>
int prove_air(wf_ctx* ctx, const AirHost& air_in, const uint64_t* const* trace_cols, const uint64_t* d_trace, int mont, u32 log_n,
              const Options& o, wf_aux_builder_fn aux_builder, void* aux_user, std::vector<u8>& proof_out,
              wf_aux_assertions_fn aux_assertions = nullptr, const AuxBuildHost* aux_build = nullptr) {
    AirHost air_dyn;                       // copy whose aux assertion values are rewritten from the random elements
    if (aux_assertions) air_dyn = air_in;  // (Air::get_aux_assertions(aux_rand_elements), air/src/air/mod.rs:279)
    const AirHost& air = aux_assertions ? air_dyn : air_in;
    const int h = o.hash_id;
    const size_t n = (size_t)1 << log_n;
    const u32 log_b = log2_ceil(o.blowup);
    const size_t N = n << log_b;
    const u32 c = air.w, kc = air.num_comp_cols(n), log_ceb = air.log_ce_blowup();
    const u32 aw = air.aw;
    if (aw && !aux_builder && !aux_build) return wf_fail(ctx, WF_ERR_INVALID, "multi-segment AIR needs an aux trace builder");
    const bool validate = ctx->validate && !air.is_fib;   // wf_ctx_set_validation; the FibSmall path is not checked
    if (log_ceb > log_b) return wf_fail(ctx, WF_ERR_INVALID, "blowup factor too small for the constraint degrees");
    for (auto& col : air.periodic) if (col.size() > n) return wf_fail(ctx, WF_ERR_INVALID, "periodic column longer than the trace");
    CKI(validate_degrees(ctx, air.all_degrees(), n));
    CKI(validate_assertions(ctx, air.aux_asserts, n, 3, "aux assertion"));
    CKI(validate_assertions(ctx, air.asserts, n, 1, "assertion"));
    Channel ch(h, context_seed(air, n, o));

    // ---- 1. trace commitment (lib.rs:497-522) ----
    wf_mat *trace = nullptr, *polys = nullptr, *lde = nullptr, *atrace = nullptr, *apolys = nullptr, *alde = nullptr, *comp = nullptr,
           *cpolys = nullptr, *clde = nullptr, *deep = nullptr;
    wf_tree *ttree = nullptr, *atree = nullptr, *ctree = nullptr;
    wf_fri* fri = nullptr;
    ProofScope scope(ctx);
    scope.own({&trace, &polys, &lde, &atrace, &apolys, &alde, &comp, &cpolys, &clde, &deep});
    scope.own({&ttree, &atree, &ctree});
    scope.fri = &fri;
    wf_mark(ctx, "start");
    if (d_trace) {
        CKI(wf_mat_from_device_columns(ctx, d_trace, c, n, &trace));
        wf_mark(ctx, "trace_upload_layout");
        CKI(wf_mat_interpolate(ctx, trace, &polys));
        if (!aux_build && !validate) scope.drop(trace);   // else: the evaluations the aux build or the trace check reads
        wf_mark(ctx, "trace_interpolate");
        CKI(wf_mat_lde(ctx, polys, log_b, &lde));
    } else {
        // host trace: upload, layout, iNTT and LDE pipelined per column chunk (capi.cu)
        CKI(wf_trace_lde_from_host(ctx, trace_cols, c, n, mont, log_b, &polys, &lde));
    }
    wf_mark(ctx, "trace_lde");
    CKI(wf_commit_rows_partitioned(ctx, h, lde, o.part_words(c, 1), &ttree));
    u8 root[32];
    CKI(wf_tree_root(ctx, ttree, root));
    wf_mark(ctx, "trace_commit");
    ch.commit(root);

    // ---- 1b. auxiliary segment (lib.rs:309-349; Air::get_aux_rand_elements air/src/air/mod.rs:292-306;
    //          DefaultTraceLde::set_aux_trace trace_lde/default/mod.rs:140-166) ----
    std::vector<u64> rnd_flat, rnd_user;  // [nr][D], canonical / as the callbacks see them
    if (aw) {
        draw_aux_rand<D>(ch.coin, air.nr, mont, rnd_flat, rnd_user);
        std::vector<u64> aux_host;  // [aw][n][D]: ColMatrix<E>, one Vec<E> per column
        if (aux_build) {
            // the described build reads the main trace's evaluations: kept from the device trace, or one forward NTT of the
            // polynomials for a host trace (its pipelined upload + LDE never materialises the layouted trace)
            if (!trace) CKI(wf_mat_evaluate(ctx, polys, &trace));
            CKI(wf_aux_build_run(ctx, *aux_build, trace, c, air.periodic, rnd_flat.data(), air.nr, D, &atrace));
            if (!validate) scope.drop(trace);
            wf_mark(ctx, "aux_build");
        } else {
            aux_host.resize((size_t)aw * n * D);
            if (aux_builder(aux_user, rnd_user.data(), aux_host.data()) != 0) return wf_fail(ctx, WF_ERR_INVALID, "aux trace builder failed");
        }
        CKI(apply_aux_assertions(ctx, air_dyn, aux_assertions, aux_user, rnd_user, D, mont));
        if (!aux_build) {
            // E column j -> D base columns j*D + q (rows of the LDE then serialise exactly like [E] rows)
            std::vector<const u64*> cols(aw);
            for (u32 j = 0; j < aw; j++) cols[j] = &aux_host[(size_t)j * n * D];
            CKI(wf_mat_from_host_columns(ctx, cols.data(), aw, n, D, mont, &atrace));
        }
        CKI(wf_mat_interpolate(ctx, atrace, &apolys));
        if (!validate) scope.drop(atrace);
        CKI(wf_mat_lde(ctx, apolys, log_b, &alde));
        CKI(wf_commit_rows_partitioned(ctx, h, alde, o.part_words(aw, D), &atree));
        CKI(wf_tree_root(ctx, atree, root));
        wf_mark(ctx, "aux_commit");
        ch.commit(root);
    }
    if (validate) {   // Trace::validate (lib.rs:355-356): the aux segment and its assertion values are final
        if (!trace) CKI(wf_mat_evaluate(ctx, polys, &trace));
        TraceReport rep;
        CKI(validation_result(ctx, wf_check_trace(ctx, air, trace, atrace, rnd_flat.data(), log_n, D, rep), rep));
        scope.drop(trace);
        scope.drop(atrace);
    }

    // ---- 2. constraint evaluation (lib.rs:373-378) ----
    // coefficient order: main transition, aux transition (transition/mod.rs:63-72), main assertions,
    // aux assertions (boundary/mod.rs:108-110)
    std::vector<GlExt<D>> cc = draw_coeffs<D>(ch.coin, o.batch_c, air.num_constraints());
    // only the rows of the sub-coset the composition polynomial is interpolated from (composition_polys)
    const size_t m = comp_subcoset_rows(n, kc);
    const u32 log_step = m < (n << log_ceb) ? log_n + log_ceb - log2_ceil(m) : 0;
    CKI(eval_constraints<D>(ctx, air, lde, alde, cc, rnd_flat, log_n, log_b, &comp, 0, 0, log_step));
    if (validate) {   // validate_transition_degrees (evaluator/default.rs:114) on the prover's own LDEs
        TraceReport rep;
        CKI(validation_result(ctx, wf_check_degrees(ctx, air, lde, alde, rnd_flat.data(), log_n, log_b, D, rep), rep));
    }
    wf_mark(ctx, "constraint_eval");
    // ---- 3. composition polynomial + commitment (lib.rs:527-552) ----
    CKI(composition_commit(ctx, h, comp, log_n, log_b, D, kc, &cpolys, &clde, &ctree, o.part_words(kc, D)));
    scope.drop(comp);
    CKI(wf_tree_root(ctx, ctree, root));
    wf_mark(ctx, "composition_commit");
    ch.commit(root);

    // ---- 4. out-of-domain frames (lib.rs:392-401) ----
    GlExt<D> z = draw_ext<D>(ch.coin);
    GlExt<D> zg = ext_mul_base(z, gl_root_of_unity(log_n));
    std::vector<std::vector<GlExt<D>>> ood;
    {
        std::vector<const wf_mat*> mats = {polys, cpolys};
        if (aw) mats.push_back(apolys);
        CKI(ood_eval<D>(ctx, mats, z, zg, ood));
    }
    OodFrame<D> of{std::move(ood[0]), std::move(ood[1])};
    ood_frame<D>(ch, of, &ood[2], aw ? &ood[4] : nullptr);
    const u32 ct = c + aw;
    wf_mark(ctx, "ood_frames");
    // ---- 5. DEEP composition (lib.rs:403-440), coefficient form ----
    std::vector<GlExt<D>> dc = draw_coeffs<D>(ch.coin, o.batch_d, ct + kc);
    CKI(deep_compose_polys<D>(ctx, polys, apolys, cpolys, kc, log_b, dc, z, zg, &deep));
    wf_mark(ctx, "deep_composition");
    // ---- 6. FRI (lib.rs:442-448) ----
    {   // transcript replicated on the device: one synchronisation for the whole commit phase (capi.cu)
        std::vector<Digest> fri_roots;
        CKI(wf_fri_build_layers_coin(ctx, h, deep, D, o.folding, o.rem_max_deg, o.blowup, ch.coin, fri_roots, &fri, deep));
        for (auto& r : fri_roots) ch.commitments.bytes(r.b, WF_DIGEST_BYTES(h));
    }
    scope.drop(deep);
    wf_mark(ctx, "fri_layers");
    // ---- 7. grinding + query positions ----
    u64 nonce;
    std::vector<u64> pos;
    CKI(grind_and_query(ctx, ch, o, N, &nonce, pos));
    wf_mark(ctx, "grinding");
    // ---- 8. proof object: every gather of the proof (trace rows, constraint rows, all FRI layers + their Merkle paths)
    //         goes through one batch: one index upload, one download, one synchronisation ----
    GatherBatch gb;
    FriProofPlan fplan;
    QueryIds id(gb, lde->m, clde->m, aw ? &alde->m : nullptr, pos);
    CKI(gb.add_opening(ctx, ttree, pos, &id.tr_dig));
    CKI(gb.add_opening(ctx, ctree, pos, &id.cr_dig));
    if (aw) CKI(gb.add_opening(ctx, atree, pos, &id.ar_dig));
    CKI(wf_fri_queue_proof(ctx, fri, pos, gb, fplan));
    CKI(gb.run(ctx));
    write_proof<D>(air, log_n, o, ch, pos, gb, id, of, fri, fplan, nullptr, nonce, proof_out);
    wf_mark(ctx, "queries_and_proof");
    // `scope` returns every device object of this proof to the pool
    return WF_OK;
}

// =================================================================================================
// One proof sharded over several GPUs (include/winterfell_b200.h: wf_comm, wf_prove_fib_sharded, wf_prove_air_sharded)
// =================================================================================================
// staging: [b cosets][rows_j][W] (per segment) -> natural order row j * b + k of the row shard
__global__ void __launch_bounds__(256) coset_interleave_kernel(SegMatrix src, SegMatrix dst, size_t rows_j, u32 b) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;   // (row of dst, word)
    const int W = dst.W;
    if (idx >= dst.rows * (size_t)W) return;
    const size_t row = idx / W;
    const u32 w = (u32)(idx % W), g = blockIdx.y;
    const size_t j = row / b, k = row % b;
    dst.base[(size_t)g * dst.seg_stride + idx] = src.base[(size_t)g * src.seg_stride + (k * rows_j + j) * W + w];
}

struct ShardCtx {
    wf_ctx* ctx;
    const wf_comm* cm;
    int G, r;
    double bytes_sent = 0, bytes_overlapped = 0, ncoll = 0, ms_small = 0;
    bool forked = false;
    bool peer_push = false;   // shard_trace_lde pushed its blocks with peer copies
    // exchanges issued between fork() and join() run on the communicator's stream, behind the ctx stream's tail at fork time
    // (wf_comm::fork / join; without the callbacks they simply stay on the ctx stream)
    int fork() {
        if (cm->fork) { if (cm->fork(cm->user) != 0) return wf_fail(ctx, WF_ERR_STATE, "fork callback failed"); forked = true; }
        return WF_OK;
    }
    int join() {
        if (forked) { forked = false; if (cm->join(cm->user) != 0) return wf_fail(ctx, WF_ERR_STATE, "join callback failed"); }
        return WF_OK;
    }
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev;  // around every exchange on the ctx stream (not the overlapped ones)
    ~ShardCtx() { for (auto& e : ev) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); } }
    // send[i] -> rank sp[i], recv[i] <- rank rp[i], all `bytes` long; entries naming this rank are not allowed
    int exchange(const std::vector<int>& sp, const std::vector<const void*>& sv, const std::vector<int>& rp, const std::vector<void*>& rv,
                 size_t bytes) {
        cudaEvent_t a = nullptr, b = nullptr;
        if (!forked) {
            CK(cudaEventCreate(&a));
            CK(cudaEventCreate(&b));
            ev.push_back({a, b});
            CK(cudaEventRecord(a, ctx->st));
        }
        if (cm->exchange(cm->user, sp.size(), sp.data(), sv.data(), rp.size(), rp.data(), rv.data(), bytes) != 0)
            return wf_fail(ctx, WF_ERR_STATE, "exchange callback failed");
        if (!forked) CK(cudaEventRecord(b, ctx->st));
        (forked ? bytes_overlapped : bytes_sent) += (double)bytes * (double)sp.size();
        ncoll += 1;
        return WF_OK;
    }
    // every rank contributes `bytes` device bytes at `mine`; all[q * bytes ..] receives rank q's (all-gather over exchange)
    int all_gather_dev(const void* mine, void* all, size_t bytes) {
        std::vector<int> sp, rp;
        std::vector<const void*> sv;
        std::vector<void*> rv;
        for (int q = 0; q < G; q++) {
            if (q == r) continue;
            sp.push_back(q); sv.push_back(mine);
            rp.push_back(q); rv.push_back((u8*)all + (size_t)q * bytes);
        }
        if ((const u8*)mine != (u8*)all + (size_t)r * bytes)
            CK(cudaMemcpyAsync((u8*)all + (size_t)r * bytes, mine, bytes, cudaMemcpyDeviceToDevice, ctx->st));
        return exchange(sp, sv, rp, rv, bytes);
    }
    int gather_host(const void* send, void* recv, size_t bytes) {
        cudaEvent_t a, b;  // host-side wall time is what this costs (the stream is already drained by the caller)
        (void)a; (void)b;
        const auto t0 = std::chrono::steady_clock::now();
        if (cm->all_gather_host(cm->user, send, recv, bytes) != 0) return wf_fail(ctx, WF_ERR_STATE, "all_gather_host callback failed");
        ms_small += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        ncoll += 1;
        return WF_OK;
    }
    // Maps the buffer at `local_base` (a cudaMalloc allocation of the same size on every rank) of every other rank into this
    // process (cudaIpcGetMemHandle -> all-gather of the handles -> cudaIpcOpenMemHandle, cached in the context). Returns
    // WF_ERR_UNSUPPORTED when the driver refuses (ranks on different nodes, IPC disabled): the caller then falls back to the
    // communicator's exchange.
    int map_peers(void* local_base, std::vector<void*>& out) {
        out.assign(G, nullptr);
        if (const char* e = getenv("WF_PEER_PUSH")) if (atoi(e) == 0) return WF_ERR_UNSUPPORTED;
        cudaIpcMemHandle_t h;
        memset(&h, 0, sizeof(h));
        int ok = cudaIpcGetMemHandle(&h, local_base) == cudaSuccess ? 1 : 0;
        if (!ok) cudaGetLastError();
        struct Msg { cudaIpcMemHandle_t h; int ok; int pad; } mine{h, ok, 0};
        std::vector<Msg> all(G);
        CKI(gather_host(&mine, all.data(), sizeof(Msg)));
        for (int q = 0; q < G; q++) ok &= all[q].ok;
        if (!ok) return WF_ERR_UNSUPPORTED;
        int opened = 1;
        for (int q = 0; q < G; q++) {
            if (q == r) { out[q] = local_base; continue; }
            std::string key((const char*)&all[q].h, sizeof(cudaIpcMemHandle_t));
            auto it = ctx->ipc_opened.find(key);
            if (it != ctx->ipc_opened.end()) { out[q] = it->second; continue; }
            void* pp = nullptr;
            if (cudaIpcOpenMemHandle(&pp, all[q].h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); opened = 0; continue; }
            ctx->ipc_opened[key] = pp;
            out[q] = pp;
        }
        // every rank must take the same path: agree on the outcome
        std::vector<int> flags(G);
        CKI(gather_host(&opened, flags.data(), sizeof(int)));
        for (int q = 0; q < G; q++) if (!flags[q]) return WF_ERR_UNSUPPORTED;
        return WF_OK;
    }
    int host_barrier() {
        int one = 1;
        std::vector<int> all(G);
        return gather_host(&one, all.data(), sizeof(int));
    }
    double exchange_ms() {
        double t = 0;
        for (auto& e : ev) { float ms = 0; if (cudaEventElapsedTime(&ms, e.first, e.second) == cudaSuccess) t += ms; }
        return t;
    }
};

// A Merkle tree of n_global leaves held as one subtree per rank (this rank's: `local`) plus the top log2(G) levels,
// recomputed on every rank from the all-gathered subtree roots: exactly the reference's heap (crypto/src/merkle/mod.rs:
// 344-368) because rank r's leaves [r n/G, (r+1) n/G) are the leaves of node G + r.
struct ShardTree {
    wf_tree* local = nullptr;
    size_t n_global = 0;
    std::vector<Digest> top;  // [1, G): internal nodes; [G, 2G): subtree roots
};
static int shard_tree_finish(ShardCtx& sc, int h, ShardTree& t, Digest* root) {
    wf_ctx* ctx = sc.ctx;
    Digest mine;
    CKI(wf_tree_root(ctx, t.local, mine.b));
    std::vector<Digest> all(sc.G);
    CKI(sc.gather_host(mine.b, all.data(), 32));
    t.top.assign(2 * sc.G, Digest{});
    for (int q = 0; q < sc.G; q++) t.top[sc.G + q] = all[q];
    for (int i = sc.G - 1; i >= 1; i--) t.top[i] = hh_merge(h, t.top[2 * i], t.top[2 * i + 1]);
    *root = t.top[1];
    return WF_OK;
}

// Columns [first, first + count) of a `w`-column trace that rank r of G owns (wf_shard_columns): contiguous runs of whole
// 8-column segments, the first (segments mod G) ranks one segment more than the others; the last segment may be partly filled
// and trailing ranks may own none. With a segment count divisible by G every rank owns the same number of whole segments.
static void shard_segments(u32 w, u32 G, u32 r, u32& seg0, u32& nseg) {
    const u32 S = (w + 7) / 8, base = S / G, extra = S % G;
    seg0 = r * base + std::min(r, extra);
    nseg = base + (r < extra ? 1u : 0u);
}
static void shard_columns(u32 w, u32 G, u32 r, u32& first, u32& count) {
    u32 s0, ns;
    shard_segments(w, G, r, s0, ns);
    first = std::min(w, s0 * 8);
    count = std::min(w, (s0 + ns) * 8) - first;
}

// rows [m.rows, m.rows + b) of every segment of `m` (allocated with b rows more than m.rows) <- the first b rows of every
// segment of rank (r + 1) mod G: the next-state rows of the last rows of a row shard
static int exchange_halo(ShardCtx& sc, const SegMatrix& m, size_t b) {
    wf_ctx* ctx = sc.ctx;
    DevScratch tmp(ctx);
    void *pk, *pk2;
    const size_t hb = b * m.W * 8;
    const u32 nsg = m.nseg();
    CKI(tmp.alloc(hb * nsg, &pk));
    CKI(tmp.alloc(hb * nsg, &pk2));
    CK(cudaMemcpy2DAsync(pk, hb, m.base, m.seg_stride * 8, hb, nsg, cudaMemcpyDeviceToDevice, ctx->st));
    CKI(sc.exchange({(sc.r + sc.G - 1) % sc.G}, {pk}, {(sc.r + 1) % sc.G}, {pk2}, hb * nsg));
    CK(cudaMemcpy2DAsync(m.base + m.rows * m.W, m.seg_stride * 8, pk2, hb, hb, nsg, cudaMemcpyDeviceToDevice, ctx->st));
    return WF_OK;
}

// *out (rows + halo rows allocated, m.rows = rows) <- rows [row0, row0 + rows) of every segment of `full`, then its rows
// [h0, h0 + halo): a row shard with its halo, cut from a matrix this rank holds whole
static int copy_row_window(wf_ctx* ctx, const wf_mat* full, size_t row0, size_t rows, size_t h0, size_t halo, wf_mat** out) {
    wf_mat* win = nullptr;
    CKI(wf_mat_alloc_w(ctx, rows + halo, full->m.cols, full->m.W, &win));
    win->m.rows = rows;
    const size_t rb = (size_t)full->m.W * 8, sp = full->m.seg_stride * 8, dp = win->m.seg_stride * 8;
    const u32 nsg = full->m.nseg();
    cudaError_t e = cudaMemcpy2DAsync(win->m.base, dp, full->m.base + row0 * full->m.W, sp, rows * rb, nsg, cudaMemcpyDeviceToDevice, ctx->st);
    if (e == cudaSuccess)
        e = cudaMemcpy2DAsync(win->m.base + rows * full->m.W, dp, full->m.base + h0 * full->m.W, sp, halo * rb, nsg, cudaMemcpyDeviceToDevice, ctx->st);
    if (e != cudaSuccess) { wf_mat_free(ctx, win); return wf_fail(ctx, WF_ERR_CUDA, "row shard copy: %s", cudaGetErrorString(e)); }
    *out = win;
    return WF_OK;
}

// This rank's LDE rows [r N/G, (r+1) N/G) of polynomials every rank holds, too few columns to shard by column (the composition
// polynomial, the aux segment). With blowup % G == 0 the LDE is sharded by COSET: rank r extends cosets [r b/G, (r+1) b/G)
// (coset-major), one exchange hands every rank the rows of its range from every coset's owner, one kernel interleaves them into
// natural order (row = b j + k). Otherwise every rank extends the whole polynomial and keeps its range. `halo`: the result also
// holds the first `blowup` rows of rank (r + 1) mod G's range after its own (rows stays N/G), as the trace's row shard does.
// *out: the matrix to free; `view`: the row range (without halo it may point into a replicated whole LDE held by *out).
static int shard_lde_rows(ShardCtx& sc, const wf_mat* polys, u32 log_b, bool halo, wf_mat** out, wf_mat& view) {
    wf_ctx* ctx = sc.ctx;
    const int G = sc.G, r = sc.r;
    const size_t n = polys->m.rows, b = (size_t)1 << log_b, rows_per = (n << log_b) / (size_t)G;
    const int W = polys->m.W;
    const u32 cols = polys->m.cols;
    if (b % (size_t)G != 0) {
        wf_mat *full = nullptr, *rows = nullptr;
        CKI(wf_mat_lde(ctx, polys, log_b, &full));
        if (!halo) {
            *out = full;
            view.m = full->m;
            view.m.base += (size_t)r * rows_per * full->m.W;
            view.m.rows = rows_per;
            return WF_OK;
        }
        const int rc = copy_row_window(ctx, full, (size_t)r * rows_per, rows_per, (size_t)((r + 1) % G) * rows_per, b, &rows);
        wf_mat_free(ctx, full);
        if (rc != WF_OK) return rc;
        *out = rows;
        view.m = rows->m;
        return WF_OK;
    }
    const u32 kpr = (u32)(b / (size_t)G);
    const size_t nj = n / (size_t)G;     // points of every coset that fall into one rank's row range
    wf_mat *ccos = nullptr, *stage = nullptr, *lde = nullptr;
    int rc = wf_mat_alloc_w(ctx, (size_t)kpr * n, cols, W, &ccos);
    if (rc == WF_OK) rc = wf_mat_lde_cosets(ctx, polys, log_b, (u32)r * kpr, (u32)(r + 1) * kpr, ccos);
    if (rc == WF_OK) rc = wf_mat_alloc_w(ctx, rows_per, cols, W, &stage);
    if (rc == WF_OK) rc = wf_mat_alloc_w(ctx, rows_per + (halo ? b : 0), cols, W, &lde);
    if (rc == WF_OK) {
        lde->m.rows = rows_per;
        const size_t blk = nj * W;       // words of one (coset, destination) block of one segment
        std::vector<int> sp, rp;
        std::vector<const void*> sv;
        std::vector<void*> rv;
        for (u32 sg = 0; sg < ccos->m.nseg(); sg++) {
            const u64* cb = ccos->m.base + (size_t)sg * ccos->m.seg_stride;
            u64* sb = stage->m.base + (size_t)sg * stage->m.seg_stride;
            for (u32 kl = 0; kl < kpr; kl++)
                for (int q = 0; q < G; q++) {
                    const u64* src = cb + ((size_t)kl * n + (size_t)q * nj) * W;
                    if (q == r) CK(cudaMemcpyAsync(sb + ((size_t)r * kpr + kl) * blk, src, blk * 8, cudaMemcpyDeviceToDevice, ctx->st));
                    else { sp.push_back(q); sv.push_back(src); }
                }
            for (u32 k = 0; k < (u32)b; k++) {
                const int owner = (int)(k / kpr);
                if (owner != r) { rp.push_back(owner); rv.push_back(sb + (size_t)k * blk); }
            }
        }
        // pairwise order: sender r -> q lists (segment, local coset) ascending; receiver q <- s lists (segment, coset) ascending
        rc = sc.exchange(sp, sv, rp, rv, blk * 8);
        if (rc == WF_OK) {
            dim3 grid((unsigned)((rows_per * W + 255) / 256), lde->m.nseg());
            coset_interleave_kernel<<<grid, 256, 0, ctx->st>>>(stage->m, lde->m, nj, (u32)b);
            ctx->launches++;
            if (cudaGetLastError() != cudaSuccess) rc = wf_fail(ctx, WF_ERR_CUDA, "coset_interleave_kernel launch failed");
        }
    }
    wf_mat_free(ctx, ccos);
    wf_mat_free(ctx, stage);
    if (rc == WF_OK && halo) rc = exchange_halo(sc, lde->m, b);
    if (rc != WF_OK) { wf_mat_free(ctx, lde); return rc; }
    *out = lde;
    view.m = lde->m;
    return WF_OK;
}

// The column -> row turn of a c-column trace LDE at blowup 2^log_b, the first phase of a sharded proof (and of the sharded
// degree check, at the constraint evaluation blowup). Rank r owns columns shard_columns(c, G, r) (local_cols / d_local, as
// wf_prove_air_sharded takes them; none: both may be NULL): it interpolates them (*polys, n rows) and extends them coset by
// coset with no communication. Coset k is written coset-major, so that the rows of rank q's range (n / G points of the
// coset) are one contiguous block per segment: its exchange runs while coset k + 1 is being extended. A rank that owns no
// columns only receives. *shard: LDE rows [r N/G, (r+1) N/G) of every column, in natural order, followed by the first 2^log_b
// rows of rank (r + 1) mod G's range (the halo the constraint frames read). polys / shard are the caller's to free.
static int shard_trace_lde(ShardCtx& sc, const uint64_t* const* local_cols, const uint64_t* d_local, int mont, u32 log_n, u32 c, u32 log_b,
                           const std::vector<u32>& seg0, const std::vector<u32>& segs, wf_mat*& polys, wf_mat*& shard) {
    wf_ctx* ctx = sc.ctx;
    const int G = sc.G, r = sc.r;
    const size_t n = (size_t)1 << log_n, b = (size_t)1 << log_b, N = n << log_b, rows_per = N / (size_t)G;
    const u32 nsg = (c + 7) / 8, fs = seg0[r], nsl = segs[r];
    u32 first, cl;
    shard_columns(c, (u32)G, (u32)r, first, cl);
    const size_t nj = n / (size_t)G;   // points of one coset inside one rank's row range
    wf_mat *lde = nullptr, *stage = nullptr;
    ProofScope scope(ctx);
    scope.own({&lde, &stage});
    // the row shard and the staging matrix hold all c columns in 8-column segments, a partly filled last one included
    CKI(wf_mat_alloc_w(ctx, rows_per + b, c, 8, &shard));
    shard->m.rows = rows_per;  // seg_stride stays (rows_per + b) * 8: rows [rows_per, rows_per + b) are the halo
    // what arrives: [global segment][coset][nj][8]
    if (cl) CKI(wf_mat_alloc_w(ctx, N, cl, 8, &lde));  // mine, coset-major: [local segment][coset][n][8]
    CKI(wf_mat_alloc_w(ctx, rows_per, c, 8, &stage));
    // Preferred transport: every rank maps the others' `stage` buffers (CUDA IPC) and PUSHES its blocks there with peer copies
    // on side streams — copy engines over NVLink, no SM taken from the NTT kernels they overlap (NCCL send/recv kernels on a
    // side stream were measured: they slow the LDE down by as much as they hide). Fallback: the communicator's exchange.
    std::vector<void*> peer_stage;
    const bool push = sc.map_peers(stage->m.base, peer_stage) == WF_OK;
    sc.peer_push = push;
    if (push) {
        for (int i = 0; i < 4; i++) if (!ctx->push_st[i]) CK(cudaStreamCreateWithFlags(&ctx->push_st[i], cudaStreamNonBlocking));
        for (int i = 0; i < 16; i++) if (!ctx->push_ev[i]) CK(cudaEventCreateWithFlags(&ctx->push_ev[i], cudaEventDisableTiming));
    }
    auto lde_block = [&](u32 sg, u32 k, int q) {   // my segment sg, coset k, the points of rank q's row range
        return lde->m.base + (size_t)sg * lde->m.seg_stride + ((size_t)k * n + (size_t)q * nj) * 8;
    };
    const std::function<int(u32)> after_coset = [&](u32 k) -> int {   // coset k of every local column is enqueued: ship it
        if (push) {
            cudaEvent_t ev = ctx->push_ev[k % 16];
            CK(cudaEventRecord(ev, ctx->st));
            for (int dq = 1; dq < G; dq++) {             // start with the next rank: no two ranks hit the same peer first
                const int q = (r + dq) % G;
                cudaStream_t ps = ctx->push_st[dq % 4];
                CK(cudaStreamWaitEvent(ps, ev, 0));
                for (u32 sg = 0; sg < nsl; sg++) {
                    u64* dst = (u64*)peer_stage[q] + (size_t)(fs + sg) * stage->m.seg_stride + (size_t)k * nj * 8;
                    CK(cudaMemcpyAsync(dst, lde_block(sg, k, q), nj * 64, cudaMemcpyDeviceToDevice, ps));
                }
            }
            for (u32 sg = 0; sg < nsl; sg++)
                CK(cudaMemcpyAsync(stage->m.base + (size_t)(fs + sg) * stage->m.seg_stride + (size_t)k * nj * 8, lde_block(sg, k, r), nj * 64,
                                   cudaMemcpyDeviceToDevice, ctx->st));
            sc.bytes_overlapped += (double)(G - 1) * nsl * nj * 64;
            return WF_OK;
        }
        std::vector<int> sp, rp;
        std::vector<const void*> sv;
        std::vector<void*> rv;
        for (u32 sg = 0; sg < nsl; sg++)    // to rank q: my segments ascending
            for (int q = 0; q < G; q++) {
                u64* dst = stage->m.base + (size_t)(fs + sg) * stage->m.seg_stride + (size_t)k * nj * 8;
                if (q == r) CK(cudaMemcpyAsync(dst, lde_block(sg, k, q), nj * 64, cudaMemcpyDeviceToDevice, ctx->st));
                else { sp.push_back(q); sv.push_back(lde_block(sg, k, q)); }
            }
        for (int q = 0; q < G; q++)         // from rank q: its segments ascending
            for (u32 sg = 0; q != r && sg < segs[q]; sg++) {
                rp.push_back(q);
                rv.push_back(stage->m.base + (size_t)(seg0[q] + sg) * stage->m.seg_stride + (size_t)k * nj * 8);
            }
        CKI(sc.fork());
        return sc.exchange(sp, sv, rp, rv, nj * 64);
    };
    // (upload ->) layout -> interpolate -> extend, pipelined per column chunk for host columns; the cosets of the last chunk
    // are extended one by one and after_coset(k) ships coset k while coset k + 1 is computed
    if (cl) CKI(wf_trace_lde_cosetwise(ctx, local_cols, d_local, cl, n, mont, log_b, &polys, &lde, true, &after_coset));
    else for (u32 k = 0; k < (u32)b; k++) CKI(after_coset(k));
    wf_mark(ctx, "trace_lde");
    if (push) {
        // my pushes have landed when my side streams drain; everybody's have when every rank says so
        for (int i = 0; i < 4; i++) CK(cudaStreamSynchronize(ctx->push_st[i]));
        CKI(sc.host_barrier());
        sc.ncoll += 1;
    } else {
        CKI(sc.join());
    }
    {   // coset-major -> natural order (row = b j + k) of my row range, every segment
        SegMatrix dstv = shard->m;
        dim3 grid((unsigned)((rows_per * 8 + 255) / 256), nsg);
        coset_interleave_kernel<<<grid, 256, 0, ctx->st>>>(stage->m, dstv, nj, (u32)b);
        ctx->launches++;
        CK(cudaGetLastError());
    }
    scope.drop(lde);
    scope.drop(stage);
    CKI(exchange_halo(sc, shard->m, b));   // the first `blowup` rows of every segment of rank (r + 1) mod G
    wf_mark(ctx, "trace_exchange");
    return WF_OK;
}

// dst (this rank's columns in 8-column segments) <- the evaluations of this rank's column polynomials on the trace domain
static int evaluate_own_columns(wf_ctx* ctx, const wf_mat* polys, const SegMatrix& dst) {
    wf_mat* ev;
    CKI(wf_mat_evaluate(ctx, polys, &ev));
    const cudaError_t e = layout_select_cols(ev->m, 0, dst, ctx->st);
    ctx->launches++;
    wf_mat_free(ctx, ev);
    CK(e);
    return WF_OK;
}

// *mtrace <- the whole n x c main trace on every rank (the aux build reads main rows i and i + 1 of every column): rank r
// evaluates its columns (`polys`, none: NULL) on the trace domain and one all-gather by segment fills in everyone else's.
static int gather_main_trace(ShardCtx& sc, const wf_mat* polys, u32 log_n, u32 c, const std::vector<u32>& seg0, const std::vector<u32>& segs,
                             wf_mat*& mtrace) {
    wf_ctx* ctx = sc.ctx;
    const int G = sc.G, r = sc.r;
    const size_t n = (size_t)1 << log_n;
    const u32 fs = seg0[r], nsl = segs[r];
    u32 first, cl;
    shard_columns(c, (u32)G, (u32)r, first, cl);
    CKI(wf_mat_alloc_w(ctx, n, c, 8, &mtrace));
    if (cl) {
        SegMatrix dv = mtrace->m;
        dv.base += (size_t)fs * dv.seg_stride;
        dv.cols = cl;
        CKI(evaluate_own_columns(ctx, polys, dv));
    }
    std::vector<int> sp, rp;
    std::vector<const void*> sv;
    std::vector<void*> rv;
    for (int q = 0; q < G; q++) {
        if (q == r) continue;
        for (u32 sg = 0; sg < nsl; sg++) { sp.push_back(q); sv.push_back(mtrace->m.base + (size_t)(fs + sg) * mtrace->m.seg_stride); }
        for (u32 sg = 0; sg < segs[q]; sg++) { rp.push_back(q); rv.push_back(mtrace->m.base + (size_t)(seg0[q] + sg) * mtrace->m.seg_stride); }
    }
    return sc.exchange(sp, sv, rp, rv, n * 64);
}

// ---- wf_ctx_set_validation in the sharded prover: the one-GPU prover's two checks (validate.cu), each rank doing its share
//      of the work. One all_gather_host hands every rank everyone's raw results and every rank reduces them with the same host
//      code, so all ranks reach the same verdict, return at the same point and stay in step for the next collective ----

// Trace::validate into `rep` (fresh; the same on every rank). Rank r checks the main assertions on its own columns, every aux
// assertion (the aux segment is replicated) and transition steps [r n/G, (r+1) n/G) of [0, n - exemptions). With mtrace, the
// whole main trace (the aux build gathered it), own columns included. Without: rank r evaluates its columns (`polys`) on the
// trace domain, and one exchange gives every rank its n/G rows of every column plus the next row (n c 8 / G bytes per rank);
// a replicated aux segment (atrace, whole) gives its rows of the same window by a device copy.
// The raw results combine by their minimum: for the assertions (assertion << 40 | cell), the reference's order.
template <int D>
static int sharded_check_trace(ShardCtx& sc, const AirHost& air, const wf_mat* polys, const wf_mat* mtrace, const wf_mat* atrace,
                               const std::vector<u64>& rnd, u32 log_n, const std::vector<u32>& seg0, const std::vector<u32>& segs,
                               TraceReport& rep) {
    wf_ctx* ctx = sc.ctx;
    const int G = sc.G, r = sc.r;
    const size_t n = (size_t)1 << log_n, nt = n / (size_t)G;
    const u32 fs = seg0[r], nsl = segs[r];
    const u32 col0 = std::min(air.w, fs * 8), cl = std::min(air.w, (fs + nsl) * 8) - col0;
    wf_mat *own = nullptr, *rows = nullptr, *arows = nullptr;
    ProofScope scope(ctx);
    scope.own({&own, &rows, &arows});
    TraceCheckPart part;
    part.acol0 = col0;
    part.s0 = (size_t)r * nt;
    part.s1 = std::min((size_t)(r + 1) * nt, n - air.exemptions);
    if (mtrace) {
        part.amain = mtrace->m;
        part.amain.base += (size_t)fs * mtrace->m.seg_stride;
        part.amain.cols = cl;
        part.main = mtrace;
        part.aux = atrace;
    } else {
        CKI(wf_mat_alloc_w(ctx, n, cl, 8, &own));
        if (cl) CKI(evaluate_own_columns(ctx, polys, own->m));
        part.amain = own->m;
        CKI(wf_mat_alloc_w(ctx, nt + 1, air.w, 8, &rows));
        rows->m.rows = nt;   // row nt: the halo row
        std::vector<int> sp, rp;
        std::vector<const void*> sv;
        std::vector<void*> rv;
        for (int q = 0; q < G; q++) {   // my segments' rows of rank q's range, ascending; from rank q its segments, ascending
            for (u32 sg = 0; sg < nsl; sg++) {
                const u64* src = own->m.base + (size_t)sg * own->m.seg_stride + (size_t)q * nt * 8;
                if (q == r) CK(cudaMemcpyAsync(rows->m.base + (size_t)(fs + sg) * rows->m.seg_stride, src, nt * 64, cudaMemcpyDeviceToDevice, ctx->st));
                else { sp.push_back(q); sv.push_back(src); }
            }
            for (u32 sg = 0; q != r && sg < segs[q]; sg++) { rp.push_back(q); rv.push_back(rows->m.base + (size_t)(seg0[q] + sg) * rows->m.seg_stride); }
        }
        CKI(sc.exchange(sp, sv, rp, rv, nt * 64));
        CKI(exchange_halo(sc, rows->m, 1));
        part.main = rows;
        part.row0 = (size_t)r * nt;
        part.rows = nt;
        if (atrace) {
            CKI(copy_row_window(ctx, atrace, (size_t)r * nt, nt, (size_t)((r + 1) % G) * nt, 1, &arows));
            part.aux = arows;
            part.aasrt = atrace->m;
        }
    }
    std::vector<u64> raw;
    CKI(wf_check_trace_part(ctx, air, part, rnd.data(), log_n, D, raw));
    std::vector<u64> all(raw.size() * (size_t)G);
    CKI(sc.gather_host(raw.data(), all.data(), raw.size() * 8));
    for (int q = 0; q < G; q++)
        for (size_t j = 0; j < raw.size(); j++) raw[j] = std::min(raw[j], all[(size_t)q * raw.size() + j]);
    wf_trace_verdict(air, atrace != nullptr, D, raw, rep);
    return WF_OK;
}

// validate_transition_degrees into `rep` (its trace check's verdict, which a degree violation does not override; expected and
// actual filled either way) on row shards of the trace LDE at blowup 2^log_b (`lde`, `alde`: LDE rows [r N/G, (r+1) N/G) and
// the blowup halo rows; the prover's own, or the validator's at the CE blowup). Rank r evaluates every transition constraint over its divisor on CE rows [r ce/G, (r+1) ce/G); one exchange
// moves that ce/G x ncols matrix into column blocks (rank q: shard_segments(ncols, G, q)'s 8-column segments over all ce
// rows); every rank interpolates its block and finds its columns' degrees; one all_gather_host of the blocks' degrees (padded
// to the largest block) gives every rank all of them. An aux constraint's D columns may lie in two blocks: the verdict takes
// the maximum over its columns either way. With ncols <= 8 rank 0 alone transforms.
template <int D>
static int sharded_check_degrees(ShardCtx& sc, const AirHost& air, const wf_mat* lde, const wf_mat* alde, const std::vector<u64>& rnd,
                                 u32 log_n, u32 log_b, TraceReport& rep) {
    wf_ctx* ctx = sc.ctx;
    const int G = sc.G, r = sc.r;
    const u32 ncols = (u32)air.degrees.size() + (alde ? (u32)air.aux_degrees.size() * D : 0);
    const size_t ce = (size_t)1 << (log_n + air.log_ce_blowup()), ce_per = ce / (size_t)G;
    std::vector<u32> cs0(G), cns(G);
    u32 blk = 0;
    for (int q = 0; q < G; q++) { shard_segments(ncols, (u32)G, (u32)q, cs0[q], cns[q]); blk = std::max(blk, cns[q] * 8); }
    u32 first, cnt;
    shard_columns(ncols, (u32)G, (u32)r, first, cnt);
    wf_mat *loc = nullptr, *mine = nullptr;
    ProofScope scope(ctx);
    scope.own({&loc, &mine});
    CKI(wf_mat_alloc_w(ctx, ce_per, ncols, 8, &loc));
    CKI(wf_transition_columns(ctx, air, lde, alde, rnd.data(), log_n, log_b, D, (size_t)r * ce_per, ce_per, loc->m));
    if (cnt) CKI(wf_mat_alloc_w(ctx, ce, cnt, 8, &mine));
    {
        std::vector<int> sp, rp;
        std::vector<const void*> sv;
        std::vector<void*> rv;
        for (int q = 0; q < G; q++) {   // to rank q: its segments ascending; from rank q: my segments ascending
            for (u32 sg = 0; sg < cns[q]; sg++) {
                const u64* src = loc->m.base + (size_t)(cs0[q] + sg) * loc->m.seg_stride;
                if (q == r) CK(cudaMemcpyAsync(mine->m.base + (size_t)sg * mine->m.seg_stride + (size_t)r * ce_per * 8, src, ce_per * 64,
                                               cudaMemcpyDeviceToDevice, ctx->st));
                else { sp.push_back(q); sv.push_back(src); }
            }
            for (u32 sg = 0; q != r && sg < cns[r]; sg++) { rp.push_back(q); rv.push_back(mine->m.base + (size_t)sg * mine->m.seg_stride + (size_t)q * ce_per * 8); }
        }
        CKI(sc.exchange(sp, sv, rp, rv, ce_per * 64));
    }
    scope.drop(loc);
    std::vector<u64> d1;
    if (cnt) CKI(wf_column_degrees(ctx, mine, d1));
    d1.resize(blk, 0);
    std::vector<u64> all((size_t)blk * G), deg1(ncols);
    CKI(sc.gather_host(d1.data(), all.data(), (size_t)blk * 8));
    for (int q = 0; q < G; q++)
        for (u32 j = cs0[q] * 8; j < std::min(ncols, (cs0[q] + cns[q]) * 8); j++) deg1[j] = all[(size_t)q * blk + j - cs0[q] * 8];
    wf_degree_verdict(air, alde != nullptr, D, log_n, deg1, rep);
    return WF_OK;
}

// One proof of `air_in` sharded over the ranks of `cm` (wf_prove_air_sharded, wf_prove_fib_sharded). Rank r owns the main-trace
// columns shard_columns() gives it: local_cols / d_local hold exactly those (none: both may be NULL). aux_build: the described
// build of a two-segment AIR's aux segment (replicated on every rank from the all-gathered main trace).
template <int D>
int prove_sharded(wf_ctx* ctx, const wf_comm* cm, const AirHost& air_in, const AuxBuildHost* aux_build, wf_aux_assertions_fn aux_assertions,
                  void* aux_user, const uint64_t* const* local_cols, const uint64_t* d_local, int mont, u32 log_n, const Options& o,
                  std::vector<u8>& proof_out, double* stats) {
    AirHost air_dyn;                       // copy whose aux assertion values are rewritten from the random elements (as prove_air)
    if (aux_assertions) air_dyn = air_in;
    const AirHost& air = aux_assertions ? air_dyn : air_in;
    ShardCtx sc{ctx, cm, cm->world, cm->rank};
    const int G = sc.G, r = sc.r;
    const int h = o.hash_id;
    const size_t n = (size_t)1 << log_n;
    const u32 log_b = log2_ceil(o.blowup);
    const size_t N = n << log_b, b = o.blowup;
    const u32 c = air.w, aw = air.aw;
    const size_t rows_per = N / (size_t)G;
    if (G < 2 || (G & (G - 1)) || r < 0 || r >= G) return wf_fail(ctx, WF_ERR_INVALID, "world size must be a power of two >= 2");
    if (aw && !aux_build) return wf_fail(ctx, WF_ERR_INVALID, "multi-segment AIR needs an aux build description");
    std::vector<u32> seg0(G), segs(G), col0(G), ncol(G);   // every rank's block: first segment, segments, first column, columns
    for (int q = 0; q < G; q++) {
        shard_segments(c, (u32)G, (u32)q, seg0[q], segs[q]);
        shard_columns(c, (u32)G, (u32)q, col0[q], ncol[q]);
    }
    const u32 cl = ncol[r];
    const u32 maxcl = *std::max_element(ncol.begin(), ncol.end());
    const u32 kc = air.num_comp_cols(n), log_ceb = air.log_ce_blowup();
    const size_t ce = n << log_ceb, ce_per = ce / (size_t)G;
    if (rows_per < 64 * b || ce_per < 64) return wf_fail(ctx, WF_ERR_UNSUPPORTED, "trace too short to shard over %d ranks", G);
    const bool validate = ctx->validate && !air.is_fib;   // wf_ctx_set_validation, as prove_air; wf_prove_fib_sharded is not checked
    Channel ch(h, context_seed(air, n, o));  // every rank replays the whole transcript

    wf_mat *polys = nullptr, *shard = nullptr, *mtrace = nullptr, *atrace = nullptr, *apolys = nullptr, *arows = nullptr,
           *comp_l = nullptr, *comp = nullptr, *cpolys = nullptr, *clde = nullptr, *deep = nullptr, *fri_in = nullptr;
    ShardTree ttree, atree, ctree;
    wf_fri* fri = nullptr;
    ProofScope scope(ctx);   // holds the ADDRESSES of these pointers: every owned pointer lives as long as the scope
    scope.own({&polys, &shard, &mtrace, &atrace, &apolys, &arows, &comp_l, &comp, &cpolys, &clde, &deep, &fri_in});
    scope.own({&ttree.local, &atree.local, &ctree.local});
    scope.fri = &fri;
    struct SLayer { u64* vals; size_t m_l, m_g; ShardTree tree; };
    std::vector<SLayer> slayers;   // FRI layers folded on row shards (their buffers and trees: `scope`'s)

    // ---- 1. interpolate the local columns, extend them coset by coset (no communication: columns are independent) and turn
    //         them into my row shard with its halo (shard_trace_lde) ----
    wf_mark(ctx, "start");
    CKI(shard_trace_lde(sc, local_cols, d_local, mont, log_n, c, log_b, seg0, segs, polys, shard));
    // ---- 2. leaves + subtree over my rows, all-gather of the subtree roots ----
    Digest root;
    CKI(wf_commit_rows_partitioned(ctx, h, shard, o.part_words(c, 1), &ttree.local));
    ttree.n_global = N;
    CKI(shard_tree_finish(sc, h, ttree, &root));
    wf_mark(ctx, "trace_commit");
    ch.commit(root.b);

    // ---- 2b. auxiliary segment (as prove_air). The build reads main rows i and i + 1 of every column: every rank evaluates its
    //          columns on the trace domain, one all-gather by segment gives every rank the whole n x c main trace, and every
    //          rank builds and interpolates the aux segment (replicated, deterministic); its LDE is sharded as the composition
    //          polynomial's, with the halo the constraint evaluation reads ----
    std::vector<u64> rnd_flat, rnd_user;  // [nr][D], canonical / as the callback sees them
    wf_mat aview;                         // my aux rows
    if (aw) {
        draw_aux_rand<D>(ch.coin, air.nr, mont, rnd_flat, rnd_user);
        CKI(gather_main_trace(sc, polys, log_n, c, seg0, segs, mtrace));
        wf_mark(ctx, "main_trace_gather");
        CKI(wf_aux_build_run(ctx, *aux_build, mtrace, c, air.periodic, rnd_flat.data(), air.nr, D, &atrace));
        if (!validate) scope.drop(mtrace);   // else: the whole main trace the trace check reads
        wf_mark(ctx, "aux_build");
        CKI(apply_aux_assertions(ctx, air_dyn, aux_assertions, aux_user, rnd_user, D, mont));
        CKI(wf_mat_interpolate(ctx, atrace, &apolys));
        if (!validate) scope.drop(atrace);
        CKI(shard_lde_rows(sc, apolys, log_b, true, &arows, aview));
        wf_mark(ctx, "aux_lde");
        CKI(wf_commit_rows_partitioned(ctx, h, &aview, o.part_words(aw, D), &atree.local));
        atree.n_global = N;
        CKI(shard_tree_finish(sc, h, atree, &root));
        wf_mark(ctx, "aux_commit");
        ch.commit(root.b);
    }
    if (validate) {   // Trace::validate (lib.rs:355-356): the aux segment and its assertion values are final
        TraceReport rep;
        CKI(sharded_check_trace<D>(sc, air, polys, mtrace, atrace, rnd_flat, log_n, seg0, segs, rep));
        CKI(validation_result(ctx, WF_OK, rep));
        scope.drop(mtrace);
        scope.drop(atrace);
    }
    // ---- 3. constraint evaluation over my CE rows ----
    std::vector<GlExt<D>> cc = draw_coeffs<D>(ch.coin, o.batch_c, air.num_constraints());
    CKI(eval_constraints<D>(ctx, air, shard, aw ? arows : nullptr, cc, rnd_flat, log_n, log_b, &comp_l, (size_t)r * ce_per, ce_per));
    if (validate) {   // evaluator/default.rs:114
        TraceReport rep;
        CKI(sharded_check_degrees<D>(sc, air, shard, aw ? arows : nullptr, rnd_flat, log_n, log_b, rep));
        CKI(validation_result(ctx, WF_OK, rep));
    }
    wf_mark(ctx, "constraint_eval");
    // ---- 4. composition polynomial: all-gather the CE evaluations (a few hundred MiB at most), interpolate on every rank (the
    //         transform is over the row index), extend and commit my row range ----
    CKI(wf_mat_alloc(ctx, ce, D, &comp));
    CKI(sc.all_gather_dev(comp_l->m.base, comp->m.base, ce_per * comp->m.W * 8));
    scope.drop(comp_l);
    CKI(composition_polys(ctx, comp, log_n, D, kc, &cpolys));
    scope.drop(comp);
    wf_mat cview;  // my rows of the composition LDE
    CKI(shard_lde_rows(sc, cpolys, log_b, false, &clde, cview));
    wf_mark(ctx, "composition_lde");
    CKI(wf_commit_rows_partitioned(ctx, h, &cview, o.part_words(kc, D), &ctree.local));
    ctree.n_global = N;
    CKI(shard_tree_finish(sc, h, ctree, &root));
    wf_mark(ctx, "composition_commit");
    ch.commit(root.b);
    // ---- 5. out-of-domain frames: my columns' polynomials, all-gathered (blocks padded to the largest); composition and aux
    //         columns are replicated ----
    GlExt<D> z = draw_ext<D>(ch.coin);
    GlExt<D> zg = ext_mul_base(z, gl_root_of_unity(log_n));
    std::vector<std::vector<GlExt<D>>> ood;
    {
        std::vector<const wf_mat*> mats = {cpolys};
        if (aw) mats.push_back(apolys);
        if (cl) mats.push_back(polys);
        CKI(ood_eval<D>(ctx, mats, z, zg, ood));
    }
    const u32 ct = c + aw;
    OodFrame<D> of{std::vector<GlExt<D>>(c), std::vector<GlExt<D>>(c)};
    {
        std::vector<u64> mine((size_t)maxcl * 2 * D, 0), all((size_t)G * maxcl * 2 * D);
        const size_t mi = aw ? 4 : 2;   // my columns' values in `ood`
        for (u32 j = 0; j < cl; j++)
            for (int q = 0; q < D; q++) { mine[((size_t)j * 2) * D + q] = ood[mi][j].v[q]; mine[((size_t)j * 2 + 1) * D + q] = ood[mi + 1][j].v[q]; }
        CKI(sc.gather_host(mine.data(), all.data(), mine.size() * 8));
        for (int s = 0; s < G; s++)
            for (u32 jl = 0; jl < ncol[s]; jl++) {
                const u32 j = col0[s] + jl;
                const u64* v = &all[((size_t)s * maxcl + jl) * 2 * D];
                for (int q = 0; q < D; q++) { of.t_cur[j].v[q] = v[q]; of.t_nxt[j].v[q] = v[D + q]; }
            }
    }
    ood_frame<D>(ch, of, &ood[0], aw ? &ood[2] : nullptr);
    wf_mark(ctx, "ood_frames");
    // ---- 6. DEEP composition over my LDE rows (evaluation form is row-local) ----
    std::vector<GlExt<D>> dc = draw_coeffs<D>(ch.coin, o.batch_d, ct + kc);
    GlExt<D> Sz = ext_zero<D>(), Szg = ext_zero<D>();
    for (u32 j = 0; j < ct; j++) { Sz = ext_add(Sz, ext_mul(dc[j], of.t_cur[j])); Szg = ext_add(Szg, ext_mul(dc[j], of.t_nxt[j])); }
    for (u32 j = 0; j < kc; j++) { Sz = ext_add(Sz, ext_mul(dc[ct + j], of.q_cur[j])); Szg = ext_add(Szg, ext_mul(dc[ct + j], of.q_nxt[j])); }
    CKI(deep_compose<D>(ctx, shard, aw ? &aview : nullptr, &cview, kc, log_n + log_b, dc, z, zg, Sz, Szg, &deep, (size_t)r * rows_per, rows_per));
    wf_mark(ctx, "deep_composition");
    // ---- 7. FRI: layers folded on shards while they are large. A layer of L points is held as contiguous position
    //         ranges; leaf i joins positions i, i + L/nf, ...: one exchange gives the owner of leaf range o (L/nf/G leaves)
    //         its nf pieces, which then look like a complete layer of nf * L/nf/G points to the hash and fold kernels ----
    const u32 nf = o.folding;
    const int ld = deep->m.W;
    const size_t max_rem = (size_t)(o.rem_max_deg + 1) * o.blowup;
    u64* cur = deep->m.base;  // my range of the current layer: L / G elements, ld words each
    size_t L = N;
    // a layer stays sharded while a rank's range has >= 2^17 elements (below that one exchange + two host round trips per
    // layer cost more than folding the whole layer everywhere); WF_SHARD_FRI_MIN_LOG lowers the bound for small tests
    u32 min_log = 17;
    if (const char* e = getenv("WF_SHARD_FRI_MIN_LOG")) min_log = (u32)atoi(e);
    while (L > max_rem && L / (size_t)G >= ((size_t)1 << min_log) && (L / nf) % (size_t)G == 0 && L / nf / (size_t)G >= 2) {
        SLayer sl;
        sl.m_g = L / nf;
        sl.m_l = sl.m_g / (size_t)G;
        void* vp;
        CKI(scope.bufs.alloc((size_t)nf * sl.m_l * ld * 8, &vp));
        sl.vals = (u64*)vp;
        std::vector<int> sp, rp;
        std::vector<const void*> sv;
        std::vector<void*> rv;
        for (u32 t = 0; t < nf; t++) {  // my range = pieces nf*r .. nf*r + nf - 1 of the layer; piece P belongs to leaf range P % G, slot P / G
            const size_t P = (size_t)nf * r + t;
            const int owner = (int)(P % (size_t)G);
            const size_t q = P / (size_t)G;
            const u64* src = cur + (size_t)t * sl.m_l * ld;
            if (owner == r) CK(cudaMemcpyAsync(sl.vals + q * sl.m_l * ld, src, sl.m_l * ld * 8, cudaMemcpyDeviceToDevice, ctx->st));
            else { sp.push_back(owner); sv.push_back(src); }
        }
        for (u32 q = 0; q < nf; q++) {
            const size_t P = (size_t)q * G + r;
            const int src_rank = (int)(P / nf);
            if (src_rank != r) { rp.push_back(src_rank); rv.push_back(sl.vals + (size_t)q * sl.m_l * ld); }
        }
        CKI(sc.exchange(sp, sv, rp, rv, sl.m_l * ld * 8));
        CKI(wf_fri_layer_tree(ctx, h, sl.vals, (size_t)nf * sl.m_l, D, ld, (int)nf, &sl.tree.local));
        scope.held.push_back(sl.tree.local);
        sl.tree.n_global = sl.m_g;
        slayers.push_back(sl);
        CKI(shard_tree_finish(sc, h, slayers.back().tree, &root));
        ch.commit(root.b);              // commit_fri_layer, then draw_fri_alpha (prover/src/channel.rs:215-234)
        GlExt<D> alpha = draw_ext<D>(ch.coin);
        const u32 logL = log2_ceil(L);
        const u64* master;
        CKI(wf_get_twiddles(ctx, logL, &master));
        void* nx;
        CKI(scope.bufs.alloc(sl.m_l * ld * 8, &nx));
        if (ld > D) CK(cudaMemsetAsync(nx, 0, sl.m_l * ld * 8, ctx->st));
        u64 av[3] = {0, 0, 0};
        for (int q = 0; q < D; q++) av[q] = alpha.v[q];
        CK(fri_fold_layer(sl.vals, (size_t)nf * sl.m_l, D, ld, (int)nf, av, master, (u64*)nx, ld, ctx->st, nullptr, (size_t)r * sl.m_l, logL));
        ctx->launches++;
        cur = (u64*)nx;
        L = sl.m_g;
    }
    // the rest of the commit phase on every rank: all-gather the current layer (small by now)
    CKI(wf_mat_alloc(ctx, L, D, &fri_in));
    CKI(sc.all_gather_dev(cur, fri_in->m.base, (L / (size_t)G) * ld * 8));
    scope.drop(deep);
    {
        std::vector<Digest> fri_roots;
        CKI(wf_fri_build_layers_coin(ctx, h, fri_in, D, o.folding, o.rem_max_deg, o.blowup, ch.coin, fri_roots, &fri));
        for (auto& rt : fri_roots) ch.commitments.bytes(rt.b, WF_DIGEST_BYTES(h));
    }
    scope.drop(fri_in);
    wf_mark(ctx, "fri_layers");
    // ---- 8. grinding + query positions (every rank; deterministic) ----
    u64 nonce;
    std::vector<u64> pos;
    CKI(grind_and_query(ctx, ch, o, N, &nonce, pos));
    wf_mark(ctx, "grinding");
    // ---- 9. proof object: every rank queues the same gathers, contributes what it holds, the words are summed ----
    GatherBatch gb;
    gb.comm = cm;
    const u64 NONE = ~(u64)0;
    auto owned_rows = [&](const std::vector<u64>& p, size_t per) {  // global row -> my local row, or NONE
        std::vector<u64> l(p.size(), NONE);
        for (size_t i = 0; i < p.size(); i++) if ((int)(p[i] / per) == r) l[i] = p[i] % per;
        return l;
    };
    std::vector<std::pair<size_t, u64>> top_t, top_a, top_c;
    const std::vector<u64> mine = owned_rows(pos, rows_per);
    QueryIds id(gb, shard->m, cview.m, aw ? &aview.m : nullptr, mine);
    CKI(gb.add_opening_sharded(ctx, ttree.local, N, G, r, pos, &id.tr_dig, &top_t));
    CKI(gb.add_opening_sharded(ctx, ctree.local, N, G, r, pos, &id.cr_dig, &top_c));
    if (aw) CKI(gb.add_opening_sharded(ctx, atree.local, N, G, r, pos, &id.ar_dig, &top_a));
    FriProofPlan splan;   // the sharded layers' gathers, and per layer the slots of the nodes above the subtree roots
    std::vector<std::vector<std::pair<size_t, u64>>> top_f(slayers.size());
    std::vector<u64> fpos = pos;
    for (size_t l = 0; l < slayers.size(); l++) {  // FriProver::build_proof (fri/src/prover/mod.rs:254-319) on the sharded layers
        const SLayer& sl = slayers[l];
        fpos = fold_positions(fpos, sl.m_g);
        std::vector<u64> gpos(fpos.size() * nf, NONE);
        for (size_t i = 0; i < fpos.size(); i++)
            if ((int)(fpos[i] / sl.m_l) == r)
                for (u32 j = 0; j < nf; j++) gpos[i * nf + j] = (u64)j * sl.m_l + fpos[i] % sl.m_l;
        SegMatrix lm;
        lm.base = sl.vals; lm.rows = (size_t)nf * sl.m_l; lm.cols = (u32)D; lm.W = ld; lm.seg_stride = lm.rows * ld;
        size_t dig_id;
        splan.row_ids.push_back(gb.add_rows(lm, gpos));
        CKI(gb.add_opening_sharded(ctx, sl.tree.local, sl.m_g, G, r, fpos, &dig_id, &top_f[l]));
        splan.dig_ids.push_back(dig_id);
        splan.nq.push_back(fpos.size());
    }
    FriProofPlan fplan;
    {
        const size_t r0 = gb.rows.size(), d0 = gb.digs.size();
        CKI(wf_fri_queue_proof(ctx, fri, fpos, gb, fplan));
        if (r != 0) {  // replicated layers: rank 0 contributes
            for (size_t i = r0; i < gb.rows.size(); i++) std::fill(gb.rows[i].pos.begin(), gb.rows[i].pos.end(), NONE);
            for (size_t i = d0; i < gb.digs.size(); i++) std::fill(gb.digs[i].idx.begin(), gb.digs[i].idx.end(), NONE);
        }
    }
    CKI(gb.run(ctx));
    auto patch = [&](size_t dig_id, const std::vector<std::pair<size_t, u64>>& slots, const ShardTree& t) {
        for (auto& se : slots) memcpy(gb.digest_words(dig_id) + se.first * 4, t.top[se.second].b, 32);
    };
    patch(id.tr_dig, top_t, ttree);
    patch(id.cr_dig, top_c, ctree);
    if (aw) patch(id.ar_dig, top_a, atree);
    for (size_t l = 0; l < slayers.size(); l++) patch(splan.dig_ids[l], top_f[l], slayers[l].tree);
    write_proof<D>(air, log_n, o, ch, pos, gb, id, of, fri, fplan, &splan, nonce, proof_out);
    wf_mark(ctx, "queries_and_proof");
    if (stats) {
        CK(cudaStreamSynchronize(ctx->st));
        stats[0] = sc.bytes_sent; stats[1] = sc.exchange_ms(); stats[2] = sc.ncoll + 1; stats[3] = sc.ms_small;
        for (int i = 4; i < 8; i++) stats[i] = 0;
        stats[4] = (double)slayers.size();
        stats[5] = sc.bytes_overlapped;
        stats[6] = sc.peer_push ? 1.0 : 0.0;
    }
    return WF_OK;
}

}  // namespace

extern "C" int wf_grind(wf_ctx* ctx, int hash_id, const uint8_t seed[32], uint32_t grinding, uint64_t* nonce) {
    if (!ctx || !seed || !nonce || grinding > 40) return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    Digest d;
    memcpy(d.b, seed, 32);
    return grind_on_device(ctx, hash_id, d, grinding, nonce);
}

static int parse_options(wf_ctx* ctx, const uint32_t* opts, Options& o) {
    o = options_from_words(opts);
    if (o.num_partitions > 16) return wf_fail(ctx, WF_ERR_INVALID, "at most 16 partitions (air/src/options.rs:413-414)");
    if (!options_in_range(o) || o.ext < 1 || o.ext > 3) return wf_fail(ctx, WF_ERR_INVALID, "bad proof options");
    if (!WF_HASH_IS_KNOWN(o.hash_id)) return wf_fail(ctx, WF_ERR_UNSUPPORTED, "unknown hash %d", o.hash_id);
    return WF_OK;
}
// the proof bytes of one proof, prove_air<D> for the extension degree of the options
static int prove_bytes(wf_ctx* ctx, const AirHost& air, const uint64_t* const* trace_cols, const uint64_t* d_trace, int mont,
                       uint32_t log_n, const Options& o, std::vector<u8>& out, wf_aux_builder_fn aux_builder, void* aux_user,
                       wf_aux_assertions_fn aux_assertions, const AuxBuildHost* aux_build) {
    switch (o.ext) {
        case 1: return prove_air<1>(ctx, air, trace_cols, d_trace, mont, log_n, o, aux_builder, aux_user, out, aux_assertions, aux_build);
        case 2: return prove_air<2>(ctx, air, trace_cols, d_trace, mont, log_n, o, aux_builder, aux_user, out, aux_assertions, aux_build);
        case 3: return prove_air<3>(ctx, air, trace_cols, d_trace, mont, log_n, o, aux_builder, aux_user, out, aux_assertions, aux_build);
    }
    return wf_fail(ctx, WF_ERR_UNSUPPORTED, "field extension %u", o.ext);
}
// the caller's proof buffer <- the proof bytes
static int copy_proof_out(wf_ctx* ctx, const std::vector<u8>& out, uint8_t* proof, size_t* proof_len) {
    if (out.size() > *proof_len) return wf_fail(ctx, WF_ERR_INVALID, "proof buffer too small (%zu needed)", out.size());
    memcpy(proof, out.data(), out.size());
    *proof_len = out.size();
    return WF_OK;
}
static int prove_dispatch(wf_ctx* ctx, const AirHost& air, const uint64_t* const* trace_cols, const uint64_t* d_trace, int mont,
                          uint32_t log_n, const Options& o, uint8_t* proof, size_t* proof_len, wf_aux_builder_fn aux_builder = nullptr,
                          void* aux_user = nullptr, wf_aux_assertions_fn aux_assertions = nullptr, const AuxBuildHost* aux_build = nullptr) {
    std::vector<u8> out;
    CKI(prove_bytes(ctx, air, trace_cols, d_trace, mont, log_n, o, out, aux_builder, aux_user, aux_assertions, aux_build));
    return copy_proof_out(ctx, out, proof, proof_len);
}
static int prove_fib_entry(wf_ctx* ctx, const uint64_t* const* trace_cols, const uint64_t* d_trace, int mont, uint32_t k,
                           uint32_t log_n, const uint64_t* results, const uint32_t* opts, uint8_t* proof, size_t* proof_len) {
    if (!ctx || (!trace_cols && !d_trace) || !results || !opts || !proof || !proof_len || k == 0 || 2 * k > 255 || log_n < 3)
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    Options o;
    CKI(parse_options(ctx, opts, o));
    AirHost air = fib_air_host(k, (size_t)1 << log_n, results);
    return prove_dispatch(ctx, air, trace_cols, d_trace, mont, log_n, o, proof, proof_len);
}
extern "C" int wf_prove_air(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* const* trace_cols, int mont,
                            uint32_t log_n, const uint32_t* opts, uint8_t* proof, size_t* proof_len) {
    if (!ctx || !air_desc || !trace_cols || !opts || !proof || !proof_len || log_n < 3)
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    Options o;
    CKI(parse_options(ctx, opts, o));
    AirHost air;
    if (!parse_air_host(air_desc, air_desc_len, air)) return wf_fail(ctx, WF_ERR_INVALID, "malformed AIR description");
    if (air.aw) return wf_fail(ctx, WF_ERR_INVALID, "multi-segment AIR: use wf_prove_air_aux");
    return prove_dispatch(ctx, air, trace_cols, nullptr, mont, log_n, o, proof, proof_len);
}
extern "C" int wf_prove_air_aux(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* const* trace_cols, int mont,
                                uint32_t log_n, const uint32_t* opts, wf_aux_builder_fn aux_builder, void* aux_user, uint8_t* proof,
                                size_t* proof_len) {
    if (!ctx || !air_desc || !trace_cols || !opts || !proof || !proof_len || log_n < 3)
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    Options o;
    CKI(parse_options(ctx, opts, o));
    AirHost air;
    if (!parse_air_host(air_desc, air_desc_len, air)) return wf_fail(ctx, WF_ERR_INVALID, "malformed AIR description");
    return prove_dispatch(ctx, air, trace_cols, nullptr, mont, log_n, o, proof, proof_len, aux_builder, aux_user);
}
extern "C" int wf_prove_air_aux_dyn(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* const* trace_cols, int mont,
                                    uint32_t log_n, const uint32_t* opts, wf_aux_builder_fn aux_builder,
                                    wf_aux_assertions_fn aux_assertions, void* aux_user, uint8_t* proof, size_t* proof_len) {
    if (!ctx || !air_desc || !trace_cols || !opts || !proof || !proof_len || log_n < 3 || !aux_assertions)
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    Options o;
    CKI(parse_options(ctx, opts, o));
    AirHost air;
    if (!parse_air_host(air_desc, air_desc_len, air)) return wf_fail(ctx, WF_ERR_INVALID, "malformed AIR description");
    return prove_dispatch(ctx, air, trace_cols, nullptr, mont, log_n, o, proof, proof_len, aux_builder, aux_user, aux_assertions);
}

// msg <- t, cut to msg_cap - 1 bytes (nothing without a buffer)
static void copy_msg(char* msg, size_t msg_cap, const char* t) {
    if (msg && msg_cap) { strncpy(msg, t, msg_cap - 1); msg[msg_cap - 1] = 0; }
}

// ---- aux segment from a described build (auxbuild.cu): the device analogue of Prover::build_aux_trace ----
// Refuses init words beyond extension degree `ext` (3: any degree)
static int parse_aux_build(wf_ctx* ctx, const AirHost& air, const uint64_t* aux_build, size_t aux_build_len, u32 ext, AuxBuildHost& b) {
    if (!air.aw) return wf_fail(ctx, WF_ERR_INVALID, "single-segment AIR: it has no aux segment to build");
    if (const char* why = wf_aux_build_parse(aux_build, aux_build_len, air.w, air.aw, (u32)air.periodic.size(), air.nr, b))
        return wf_fail(ctx, WF_ERR_INVALID, "%s", why);
    for (auto& col : b.cols)
        for (u32 q = ext; q < 3; q++) if (col.init[q]) return wf_fail(ctx, WF_ERR_INVALID, "aux column init has non-zero words beyond the extension degree");
    return WF_OK;
}
extern "C" int wf_aux_build_check(const uint64_t* air_desc, size_t air_desc_len, const uint64_t* aux_build, size_t aux_build_len,
                                  uint32_t log_n, char* msg, size_t msg_cap) {
    copy_msg(msg, msg_cap, "");
    if (!air_desc || !aux_build || log_n < 3 || log_n > 32) { copy_msg(msg, msg_cap, "bad arguments"); return WF_ERR_INVALID; }
    AirHost air;
    if (!parse_air_host(air_desc, air_desc_len, air)) { copy_msg(msg, msg_cap, "malformed AIR description"); return WF_ERR_INVALID; }
    wf_ctx note{};   // carries the message, nothing else
    AuxBuildHost b;
    int r = parse_aux_build(&note, air, aux_build, aux_build_len, 3, b);
    for (auto& col : air.periodic)
        if (r == WF_OK && col.size() > ((size_t)1 << log_n)) r = wf_fail(&note, WF_ERR_INVALID, "periodic column longer than the trace");
    copy_msg(msg, msg_cap, note.err.c_str());
    return r;
}
extern "C" int wf_aux_build(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* aux_build, size_t aux_build_len,
                            const wf_mat* main_evals, const uint64_t* rand, uint32_t ext, wf_mat** aux) {
    if (!ctx || !air_desc || !aux_build || !main_evals || !aux || ext < 1 || ext > 3) return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    AirHost air;
    if (!parse_air_host(air_desc, air_desc_len, air)) return wf_fail(ctx, WF_ERR_INVALID, "malformed AIR description");
    AuxBuildHost b;
    CKI(parse_aux_build(ctx, air, aux_build, aux_build_len, 3, b));   // wf_aux_build_run refuses init words beyond `ext`
    if (air.nr && !rand) return wf_fail(ctx, WF_ERR_INVALID, "random elements missing");
    return wf_aux_build_run(ctx, b, main_evals, air.w, air.periodic, rand, air.nr, (int)ext, aux);
}
extern "C" int wf_prove_air_aux_built(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* aux_build,
                                      size_t aux_build_len, const uint64_t* const* trace_cols, const uint64_t* d_trace, int mont,
                                      uint32_t log_n, const uint32_t* opts, wf_aux_assertions_fn aux_assertions, void* aux_user,
                                      uint8_t* proof, size_t* proof_len) {
    if (!ctx || !air_desc || !aux_build || !opts || !proof || !proof_len || log_n < 3) return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    if (!trace_cols == !d_trace) return wf_fail(ctx, WF_ERR_INVALID, "pass exactly one of trace_cols (host) and d_trace (device)");
    Options o;
    CKI(parse_options(ctx, opts, o));
    AirHost air;
    if (!parse_air_host(air_desc, air_desc_len, air)) return wf_fail(ctx, WF_ERR_INVALID, "malformed AIR description");
    AuxBuildHost b;
    CKI(parse_aux_build(ctx, air, aux_build, aux_build_len, o.ext, b));
    return prove_dispatch(ctx, air, trace_cols, d_trace, mont, log_n, o, proof, proof_len, nullptr, aux_user, aux_assertions, &b);
}

// Compiles the constraint kernel of an AIR description; needs no device (a build-time / CI check of the JIT path and of the
// generated code). *cubin_bytes = size of the sm_90a cubin; `log` receives the compiler log (warnings or errors).
extern "C" int wf_jit_compile_air(const uint64_t* air_desc, size_t air_desc_len, uint32_t ext, size_t* cubin_bytes, char* log, size_t log_cap) {
    if (!air_desc || ext < 1 || ext > 3) return WF_ERR_INVALID;
    AirHost air;
    if (!parse_air_host(air_desc, air_desc_len, air)) return WF_ERR_INVALID;
    std::vector<char> cubin;
    std::string lg;
    const int rc = wf_jit_compile(wf_jit_source((int)ext, air.w, (u32)air.periodic.size(), air.num_regs, air.prog, air.consts, air.aw, air.nr,
                                                air.aux_num_regs, air.aux_prog), cubin, lg);
    copy_msg(log, log_cap, lg.c_str());
    if (cubin_bytes) *cubin_bytes = cubin.size();
    if (const char* dump = getenv("WF_JIT_DUMP")) if (rc == 0) { FILE* f = fopen(dump, "wb"); if (f) { fwrite(cubin.data(), 1, cubin.size(), f); fclose(f); } }
    return rc == 0 ? WF_OK : WF_ERR_UNSUPPORTED;
}

extern "C" int wf_air_check(const uint64_t* air_desc, size_t air_desc_len, uint32_t log_n, uint32_t blowup, char* msg, size_t msg_cap) {
    copy_msg(msg, msg_cap, "");
    if (!air_desc || log_n < 3 || log_n > 32 || blowup < 2 || blowup > 128 || (blowup & (blowup - 1))) { copy_msg(msg, msg_cap, "bad arguments"); return WF_ERR_INVALID; }
    AirHost air;
    if (!parse_air_host(air_desc, air_desc_len, air)) { copy_msg(msg, msg_cap, "malformed AIR description"); return WF_ERR_INVALID; }
    wf_ctx note{};   // carries the message of the shared validators, nothing else
    const int r = air_check_host(&note, air, log_n, blowup);
    copy_msg(msg, msg_cap, note.err.c_str());
    return r;
}

// ---- batches of proofs of one AIR (wf_prove_air_batch) ----
// Parses the descriptions of a batch and runs every check of wf_air_check on each, and the structure check against proof 0
static int air_batch_parse(wf_ctx* ctx, uint32_t batch, const uint64_t* const* air_descs, const size_t* air_desc_lens, uint32_t log_n,
                           uint32_t blowup, std::vector<AirHost>& airs) {
    if (batch == 0 || !air_descs || !air_desc_lens || log_n < 3 || log_n > 32 || blowup < 2 || blowup > 128 || (blowup & (blowup - 1)))
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    airs.assign(batch, AirHost());
    for (u32 j = 0; j < batch; j++) {
        if (!air_descs[j] || !parse_air_host(air_descs[j], air_desc_lens[j], airs[j]))
            return wf_fail(ctx, WF_ERR_INVALID, "proof %u: malformed AIR description", j);
        if (air_check_host(ctx, airs[j], log_n, blowup) != WF_OK) return wf_fail(ctx, WF_ERR_INVALID, "proof %u: %s", j, std::string(ctx->err).c_str());
        if (const char* why = j ? air_structure_mismatch(airs[0], airs[j]) : nullptr)
            return wf_fail(ctx, WF_ERR_INVALID, "proof %u differs from proof 0 in its %s", j, why);
    }
    return WF_OK;
}
extern "C" int wf_air_batch_check(uint32_t batch, const uint64_t* const* air_descs, const size_t* air_desc_lens, uint32_t log_n,
                                  uint32_t blowup, char* msg, size_t msg_cap) {
    wf_ctx note{};
    std::vector<AirHost> airs;
    const int r = air_batch_parse(&note, batch, air_descs, air_desc_lens, log_n, blowup, airs);
    copy_msg(msg, msg_cap, note.err.c_str());
    return r;
}
extern "C" int wf_prove_air_batch(wf_ctx* ctx, uint32_t batch, const uint64_t* const* air_descs, const size_t* air_desc_lens,
                                  const uint64_t* aux_build, size_t aux_build_len, const uint64_t* const* trace_cols, const uint64_t* d_traces,
                                  int mont, uint32_t log_n, const uint32_t* opts, uint8_t* const* proofs, size_t* proof_lens) {
    if (!ctx || !opts || !proofs || !proof_lens) return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    if (!trace_cols == !d_traces) return wf_fail(ctx, WF_ERR_INVALID, "pass exactly one of trace_cols (host) and d_traces (device)");
    Options o;
    CKI(parse_options(ctx, opts, o));
    std::vector<AirHost> airs;
    CKI(air_batch_parse(ctx, batch, air_descs, air_desc_lens, log_n, o.blowup, airs));
    for (u32 j = 0; j < batch; j++) if (!proofs[j]) return wf_fail(ctx, WF_ERR_INVALID, "proof %u: no output buffer", j);
    AuxBuildHost b;
    if (aux_build) {
        CKI(parse_aux_build(ctx, airs[0], aux_build, aux_build_len, o.ext, b));
    } else if (airs[0].aw) {
        return wf_fail(ctx, WF_ERR_INVALID, "multi-segment AIR: a batch builds its aux segments from aux_build");
    }
    const u32 w = airs[0].w;
    const size_t n = (size_t)1 << log_n;
    // The proofs run one after another through the single-proof sequence: launches and synchronisations grow with the batch.
    // They are kept on the host until all of them exist: nothing is written when one fails.
    std::vector<std::vector<u8>> out(batch);
    for (u32 j = 0; j < batch; j++) {
        const uint64_t* const* cols = trace_cols ? trace_cols + (size_t)j * w : nullptr;
        const uint64_t* dev = d_traces ? d_traces + (size_t)j * w * n : nullptr;
        const int r = prove_bytes(ctx, airs[j], cols, dev, mont, log_n, o, out[j], nullptr, nullptr, nullptr, aux_build ? &b : nullptr);
        if (r != WF_OK) return wf_fail(ctx, r, "proof %u: %s", j, std::string(ctx->err).c_str());
    }
    for (u32 j = 0; j < batch; j++)
        if (out[j].size() > proof_lens[j]) return wf_fail(ctx, WF_ERR_INVALID, "proof %u: proof buffer too small (%zu needed)", j, out[j].size());
    for (u32 j = 0; j < batch; j++) {
        memcpy(proofs[j], out[j].data(), out[j].size());
        proof_lens[j] = out[j].size();
    }
    return WF_OK;
}

// ---- the reference's debug-build checks of a trace (validate.cu), standalone ----
// the report of wf_trace_validate / wf_trace_validate_sharded
static void write_validation(const TraceReport& rep, const AirHost& air, int check_degrees, wf_validation* report, uint64_t* first_failing_step,
                             uint64_t* expected_degrees, uint64_t* actual_degrees, char* msg, size_t msg_cap) {
    report->kind = rep.kind; report->index = rep.index; report->step = rep.step; report->column = rep.column;
    report->num_transition_constraints = (u32)(air.degrees.size() + (air.aw ? air.aux_degrees.size() : 0));
    if (first_failing_step) std::copy(rep.first_fail.begin(), rep.first_fail.end(), first_failing_step);
    if (check_degrees && expected_degrees) std::copy(rep.expected.begin(), rep.expected.end(), expected_degrees);
    if (check_degrees && actual_degrees) std::copy(rep.actual.begin(), rep.actual.end(), actual_degrees);
    copy_msg(msg, msg_cap, rep.msg.c_str());
}
// The checks of wf_trace_validate / wf_trace_validate_sharded on the description and the aux segment's source, in this order
static int trace_validate_args(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* aux_build, size_t aux_build_len,
                               const uint64_t* const* aux_cols, const uint64_t* rand, uint32_t log_n, uint32_t ext, AirHost& air,
                               AuxBuildHost& b) {
    if (!parse_air_host(air_desc, air_desc_len, air)) return wf_fail(ctx, WF_ERR_INVALID, "malformed AIR description");
    CKI(air_check_host(ctx, air, log_n, 1u << air.log_ce_blowup()));
    if (air.aw) {
        if (!aux_build == !aux_cols) return wf_fail(ctx, WF_ERR_INVALID, "two-segment AIR: pass exactly one of aux_build and aux_cols");
        if (air.nr && !rand) return wf_fail(ctx, WF_ERR_INVALID, "random elements missing");
        if (aux_build) CKI(parse_aux_build(ctx, air, aux_build, aux_build_len, ext, b));
    } else if (aux_build || aux_cols) {
        return wf_fail(ctx, WF_ERR_INVALID, "single-segment AIR: it has no aux segment");
    }
    return WF_OK;
}
extern "C" int wf_trace_validate(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* aux_build, size_t aux_build_len,
                                 const uint64_t* const* aux_cols, const uint64_t* const* trace_cols, const uint64_t* d_trace, int mont,
                                 const uint64_t* rand, uint32_t log_n, uint32_t ext, int check_degrees, wf_validation* report,
                                 uint64_t* first_failing_step, uint64_t* expected_degrees, uint64_t* actual_degrees, char* msg, size_t msg_cap) {
    if (msg && msg_cap) msg[0] = 0;
    if (!ctx || !air_desc || !report || log_n < 3 || log_n > 30 || ext < 1 || ext > 3) return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    if (!trace_cols == !d_trace) return wf_fail(ctx, WF_ERR_INVALID, "pass exactly one of trace_cols (host) and d_trace (device)");
    AirHost air;
    AuxBuildHost b;
    CKI(trace_validate_args(ctx, air_desc, air_desc_len, aux_build, aux_build_len, aux_cols, rand, log_n, ext, air, b));
    const u32 log_ceb = air.log_ce_blowup();
    const size_t n = (size_t)1 << log_n;
    const u32 c = air.w;
    const std::vector<u64> rnd(rand, rand + (air.aw ? (size_t)air.nr * ext : 0));
    wf_mat *trace = nullptr, *atrace = nullptr, *polys = nullptr, *apolys = nullptr, *lde = nullptr, *alde = nullptr;
    ProofScope scope(ctx);
    scope.own({&trace, &atrace, &polys, &apolys, &lde, &alde});
    if (d_trace) CKI(wf_mat_from_device_columns(ctx, d_trace, c, n, &trace));
    else CKI(wf_mat_from_host_columns(ctx, trace_cols, c, n, 1, mont, &trace));
    if (air.aw) {
        if (aux_build) CKI(wf_aux_build_run(ctx, b, trace, c, air.periodic, rnd.data(), air.nr, (int)ext, &atrace));
        else CKI(wf_mat_from_host_columns(ctx, aux_cols, air.aw, n, (int)ext, mont, &atrace));
    }
    TraceReport rep;
    CKI(wf_check_trace(ctx, air, trace, atrace, rnd.data(), log_n, (int)ext, rep));
    if (check_degrees) {
        // the CE domain's frames from LDEs at the constraint evaluation blowup: the frame stride is 1 * ce_blowup
        CKI(wf_mat_interpolate(ctx, trace, &polys));
        scope.drop(trace);
        CKI(wf_mat_lde(ctx, polys, log_ceb, &lde));
        scope.drop(polys);
        if (atrace) {
            CKI(wf_mat_interpolate(ctx, atrace, &apolys));
            scope.drop(atrace);
            CKI(wf_mat_lde(ctx, apolys, log_ceb, &alde));
            scope.drop(apolys);
        }
        CKI(wf_check_degrees(ctx, air, lde, alde, rnd.data(), log_n, log_ceb, (int)ext, rep));
    }
    write_validation(rep, air, check_degrees, report, first_failing_step, expected_degrees, actual_degrees, msg, msg_cap);
    return WF_OK;
}

// A sharded call's checks on this rank's own arguments: its block of main columns and, for the prover, its output buffer
// (out_ok; nullptr: the call has none). Every rank learns every rank's verdict in the call's first collective, and all of them
// return when one refuses.
static int agree_on_columns(wf_ctx* ctx, const wf_comm* comm, u32 w, u32 local_count, const uint64_t* const* local_cols,
                            const uint64_t* d_local, const bool* out_ok) {
    const int G = comm->world;
    u32 first, count;
    shard_columns(w, (u32)G, (u32)comm->rank, first, count);
    int mine = WF_OK;
    if (local_count != count)
        mine = wf_fail(ctx, WF_ERR_INVALID, "rank %d owns %u columns of %u (wf_shard_columns), not %u", comm->rank, count, w, local_count);
    else if ((count && !local_cols == !d_local) || (out_ok && !*out_ok))
        mine = wf_fail(ctx, WF_ERR_INVALID, "bad arguments: pass exactly one of local_cols and d_local%s", out_ok ? ", and an output buffer" : "");
    std::vector<int> verdicts(G);
    if (comm->all_gather_host(comm->user, &mine, verdicts.data(), sizeof(int)) != 0) return wf_fail(ctx, WF_ERR_STATE, "all_gather_host callback failed");
    if (mine != WF_OK) return mine;
    for (int q = 0; q < G; q++)
        if (verdicts[q] != WF_OK) return wf_fail(ctx, WF_ERR_INVALID, "rank %d refused its column block%s", q, out_ok ? " or output buffer" : "");
    return WF_OK;
}

// wf_trace_validate over the ranks of `cm`, each rank with its block of main columns (as prove_sharded takes them): the
// sharded prover's two checks without the proof. The degree check reads LDE row shards at the CE blowup, as the one-GPU
// validator reads its whole LDE at that blowup; the aux segment is built (aux_build, from the gathered main trace) or
// uploaded (aux_cols) whole on every rank, and its LDE sharded as the prover's.
template <int D>
static int validate_sharded(wf_ctx* ctx, const wf_comm* cm, const AirHost& air, const AuxBuildHost* aux_build, const uint64_t* const* aux_cols,
                            const uint64_t* const* local_cols, const uint64_t* d_local, int mont, const std::vector<u64>& rnd, u32 log_n,
                            bool check_degrees, TraceReport& rep) {
    ShardCtx sc{ctx, cm, cm->world, cm->rank};
    const int G = sc.G, r = sc.r;
    const size_t n = (size_t)1 << log_n;
    const u32 c = air.w, log_ceb = air.log_ce_blowup();
    std::vector<u32> seg0(G), segs(G);
    for (int q = 0; q < G; q++) shard_segments(c, (u32)G, (u32)q, seg0[q], segs[q]);
    u32 first, cl;
    shard_columns(c, (u32)G, (u32)r, first, cl);
    wf_mat *trace = nullptr, *polys = nullptr, *shard = nullptr, *mtrace = nullptr, *atrace = nullptr, *apolys = nullptr, *arows = nullptr;
    ProofScope scope(ctx);
    scope.own({&trace, &polys, &shard, &mtrace, &atrace, &apolys, &arows});
    if (check_degrees) {
        CKI(shard_trace_lde(sc, local_cols, d_local, mont, log_n, c, log_ceb, seg0, segs, polys, shard));
    } else if (cl) {
        if (d_local) CKI(wf_mat_from_device_columns(ctx, d_local, cl, n, &trace));
        else CKI(wf_mat_from_host_columns(ctx, local_cols, cl, n, 1, mont, &trace));
        CKI(wf_mat_interpolate(ctx, trace, &polys));
        scope.drop(trace);
    }
    if (aux_build) {
        CKI(gather_main_trace(sc, polys, log_n, c, seg0, segs, mtrace));
        CKI(wf_aux_build_run(ctx, *aux_build, mtrace, c, air.periodic, rnd.data(), air.nr, D, &atrace));
    } else if (aux_cols) {
        CKI(wf_mat_from_host_columns(ctx, aux_cols, air.aw, n, D, mont, &atrace));
    }
    CKI(sharded_check_trace<D>(sc, air, polys, mtrace, atrace, rnd, log_n, seg0, segs, rep));
    scope.drop(mtrace);
    scope.drop(polys);
    if (!check_degrees) return WF_OK;
    if (atrace) {
        wf_mat aview;
        CKI(wf_mat_interpolate(ctx, atrace, &apolys));
        scope.drop(atrace);
        CKI(shard_lde_rows(sc, apolys, log_ceb, true, &arows, aview));
        scope.drop(apolys);
    }
    return sharded_check_degrees<D>(sc, air, shard, arows, rnd, log_n, log_ceb, rep);
}

extern "C" int wf_trace_validate_sharded(wf_ctx* ctx, const wf_comm* comm, const uint64_t* air_desc, size_t air_desc_len,
                                         const uint64_t* aux_build, size_t aux_build_len, const uint64_t* const* aux_cols,
                                         const uint64_t* const* local_cols, const uint64_t* d_local, uint32_t local_count, int mont,
                                         const uint64_t* rand, uint32_t log_n, uint32_t ext, int check_degrees, wf_validation* report,
                                         uint64_t* first_failing_step, uint64_t* expected_degrees, uint64_t* actual_degrees, char* msg,
                                         size_t msg_cap) {
    if (msg && msg_cap) msg[0] = 0;
    if (!ctx) return WF_ERR_INVALID;
    if (!comm || !comm->exchange || !comm->all_gather_host) return wf_fail(ctx, WF_ERR_INVALID, "bad communicator");
    // Checks on what every rank shares (description, aux segment, random elements, log_n, world size): the same verdict
    // everywhere, before any collective, so a refusal leaves no rank waiting.
    const int G = comm->world;
    if (G < 2 || (G & (G - 1)) || comm->rank < 0 || comm->rank >= G) return wf_fail(ctx, WF_ERR_INVALID, "world size must be a power of two >= 2");
    if (!air_desc || !report || log_n < 3 || log_n > 30 || ext < 1 || ext > 3) return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    AirHost air;
    AuxBuildHost b;
    CKI(trace_validate_args(ctx, air_desc, air_desc_len, aux_build, aux_build_len, aux_cols, rand, log_n, ext, air, b));
    const u32 log_ceb = air.log_ce_blowup();
    // the row shard of the prover (rows_per >= 64 blowup, ce_per >= 64) with the CE blowup in place of the proof's: n >= 64 G
    const size_t rows_per = ((size_t)1 << (log_n + log_ceb)) / (size_t)G;
    if (log_n + log_ceb > 32 || rows_per < ((size_t)64 << log_ceb))
        return wf_fail(ctx, WF_ERR_UNSUPPORTED, "trace too short to shard over %d ranks", G);
    CKI(agree_on_columns(ctx, comm, air.w, local_count, local_cols, d_local, nullptr));
    const std::vector<u64> rnd(rand, rand + (air.aw ? (size_t)air.nr * ext : 0));
    const AuxBuildHost* bp = air.aw && aux_build ? &b : nullptr;
    TraceReport rep;
    int r;
    switch (ext) {
        case 1: r = validate_sharded<1>(ctx, comm, air, bp, aux_cols, local_cols, d_local, mont, rnd, log_n, check_degrees != 0, rep); break;
        case 2: r = validate_sharded<2>(ctx, comm, air, bp, aux_cols, local_cols, d_local, mont, rnd, log_n, check_degrees != 0, rep); break;
        default: r = validate_sharded<3>(ctx, comm, air, bp, aux_cols, local_cols, d_local, mont, rnd, log_n, check_degrees != 0, rep); break;
    }
    CKI(r);
    write_validation(rep, air, check_degrees, report, first_failing_step, expected_degrees, actual_degrees, msg, msg_cap);
    return WF_OK;
}

// ---- stepwise exports: the seams of prover/src/lib.rs:125-223 (ConstraintEvaluator, ConstraintCommitment)
//      and the concrete steps between them, for a host that keeps the transcript itself ----------------
template <int D>
static int eval_constraints_entry(wf_ctx* ctx, const AirHost& air, u32 log_n, u32 log_b, const wf_mat* lde, const wf_mat* alde,
                                  const uint64_t* coeffs, const uint64_t* aux_rand, wf_mat** out, size_t row0, size_t ce_rows, u32 log_step) {
    const size_t ncc = air.degrees.size() + air.aux_degrees.size() + air.asserts.size() + air.aux_asserts.size();
    std::vector<GlExt<D>> cc(ncc);
    for (size_t i = 0; i < ncc; i++) for (int q = 0; q < D; q++) cc[i].v[q] = coeffs[i * D + q];
    std::vector<u64> rnd;
    if (air.aw) rnd.assign(aux_rand, aux_rand + (size_t)air.nr * D);
    CKI(eval_constraints<D>(ctx, air, lde, alde, cc, rnd, log_n, log_b, out, row0, ce_rows, log_step));
    if (ctx->validate && !ce_rows) {   // validate_transition_degrees, as evaluator/default.rs:114 runs it after the evaluation
        TraceReport rep;
        const int r = validation_result(ctx, wf_check_degrees(ctx, air, lde, alde, rnd.data(), log_n, log_b, D, rep), rep);
        if (r != WF_OK) { wf_mat_free(ctx, *out); *out = nullptr; return r; }
    }
    return WF_OK;
}
// The LDE rows a call over CE rows [row0, row0 + ce_rows) reads (ce_rows = 0: the whole domain, row0 = 0): the whole LDE, or the
// window's rows followed by `blowup` halo rows (the layout shard_lde_rows gives the row-sharded prover). Refuses a window outside
// the domain or of fewer than 64 rows.
static int check_window(wf_ctx* ctx, u32 log_n, u32 log_b, u32 log_ceb, size_t row0, size_t ce_rows, size_t* lde_rows) {
    const size_t ce = (size_t)1 << (log_n + log_ceb);
    if (!ce_rows) {
        if (row0) return wf_fail(ctx, WF_ERR_INVALID, "row0 without a window");
        *lde_rows = (size_t)1 << (log_n + log_b);
        return WF_OK;
    }
    if (ce_rows < 64 || row0 >= ce || ce_rows > ce - row0) return wf_fail(ctx, WF_ERR_INVALID, "CE row window outside the domain or under 64 rows");
    *lde_rows = (ce_rows << (log_b - log_ceb)) + ((size_t)1 << log_b);
    return WF_OK;
}
// The row step of a call over `rows` rows of the CE domain's sub-coset (rows = 0: the whole domain or a window, step 1). Refuses
// a row count that is not a power of two at most the domain's size.
static int subcoset_step(wf_ctx* ctx, u32 log_n, u32 log_ceb, size_t rows, u32* log_step) {
    *log_step = 0;
    if (!rows) return WF_OK;
    const u32 lr = log2_ceil(rows);
    if (rows != ((size_t)1 << lr) || lr > log_n + log_ceb) return wf_fail(ctx, WF_ERR_INVALID, "sub-coset rows must be a power of two at most the CE domain's size");
    *log_step = log_n + log_ceb - lr;
    return WF_OK;
}
static int eval_constraints_desc(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, uint32_t log_n, uint32_t blowup, uint32_t ext,
                                 const wf_mat* main_lde, const wf_mat* aux_lde, const uint64_t* coeffs, const uint64_t* aux_rand,
                                 size_t row0, size_t ce_rows, size_t sub_rows, wf_mat** out) {
    if (!ctx || !air_desc || !main_lde || !coeffs || !out || log_n < 3 || blowup < 2 || (blowup & (blowup - 1)))
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    AirHost air;
    if (!parse_air_host(air_desc, air_desc_len, air)) return wf_fail(ctx, WF_ERR_INVALID, "malformed AIR description");
    const u32 log_b = log2_ceil(blowup);
    if (air.log_ce_blowup() > log_b) return wf_fail(ctx, WF_ERR_INVALID, "blowup factor too small for the constraint degrees");
    size_t N = 0;
    u32 log_step;
    CKI(check_window(ctx, log_n, log_b, air.log_ce_blowup(), row0, ce_rows, &N));
    CKI(subcoset_step(ctx, log_n, air.log_ce_blowup(), sub_rows, &log_step));
    if (main_lde->m.rows != N || main_lde->m.cols != air.w) return wf_fail(ctx, WF_ERR_INVALID, "main LDE shape does not match the AIR");
    if (air.aw && (!aux_lde || !aux_rand || aux_lde->m.rows != N || aux_lde->m.cols != air.aw * ext))
        return wf_fail(ctx, WF_ERR_INVALID, "aux LDE / random elements missing or of the wrong shape");
    for (auto& col : air.periodic) if (col.size() > ((size_t)1 << log_n)) return wf_fail(ctx, WF_ERR_INVALID, "periodic column longer than the trace");
    CKI(validate_degrees(ctx, air.all_degrees(), (size_t)1 << log_n));
    CKI(validate_assertions(ctx, air.aux_asserts, (size_t)1 << log_n, 3, "aux assertion"));
    CKI(validate_assertions(ctx, air.asserts, (size_t)1 << log_n, 1, "assertion"));
    const wf_mat* al = air.aw ? aux_lde : nullptr;
    switch (ext) {
        case 1: return eval_constraints_entry<1>(ctx, air, log_n, log_b, main_lde, al, coeffs, aux_rand, out, row0, ce_rows, log_step);
        case 2: return eval_constraints_entry<2>(ctx, air, log_n, log_b, main_lde, al, coeffs, aux_rand, out, row0, ce_rows, log_step);
        case 3: return eval_constraints_entry<3>(ctx, air, log_n, log_b, main_lde, al, coeffs, aux_rand, out, row0, ce_rows, log_step);
    }
    return wf_fail(ctx, WF_ERR_UNSUPPORTED, "field extension %u", ext);
}
extern "C" int wf_eval_constraints(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, uint32_t log_n, uint32_t blowup,
                                   uint32_t ext, const wf_mat* main_lde, const wf_mat* aux_lde, const uint64_t* coeffs,
                                   const uint64_t* aux_rand, wf_mat** out) {
    return eval_constraints_desc(ctx, air_desc, air_desc_len, log_n, blowup, ext, main_lde, aux_lde, coeffs, aux_rand, 0, 0, 0, out);
}
extern "C" int wf_eval_constraints_window(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, uint32_t log_n, uint32_t blowup,
                                          uint32_t ext, const wf_mat* main_lde, const wf_mat* aux_lde, const uint64_t* coeffs,
                                          const uint64_t* aux_rand, size_t row0, size_t ce_rows, wf_mat** out) {
    if (!ce_rows) return wf_fail(ctx, WF_ERR_INVALID, "empty CE row window");
    return eval_constraints_desc(ctx, air_desc, air_desc_len, log_n, blowup, ext, main_lde, aux_lde, coeffs, aux_rand, row0, ce_rows, 0, out);
}
extern "C" int wf_eval_constraints_subcoset(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, uint32_t log_n, uint32_t blowup,
                                            uint32_t ext, const wf_mat* main_lde, const wf_mat* aux_lde, const uint64_t* coeffs,
                                            const uint64_t* aux_rand, size_t rows, wf_mat** out) {
    if (!rows) return wf_fail(ctx, WF_ERR_INVALID, "empty sub-coset");
    return eval_constraints_desc(ctx, air_desc, air_desc_len, log_n, blowup, ext, main_lde, aux_lde, coeffs, aux_rand, 0, 0, rows, out);
}
static int eval_constraints_fib(wf_ctx* ctx, uint32_t k, const uint64_t* results, uint32_t log_n, uint32_t blowup, uint32_t ext,
                                const wf_mat* lde, const uint64_t* coeffs, size_t row0, size_t ce_rows, size_t sub_rows, wf_mat** out) {
    if (!ctx || !results || !lde || !coeffs || !out || k == 0 || 2 * k > 255 || log_n < 3 || blowup < 2 ||
        (blowup & (blowup - 1)) || blowup > 128)
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    const u32 log_b = log2_ceil(blowup);
    const AirHost air = fib_air_host(k, (size_t)1 << log_n, results);
    size_t N = 0;
    u32 log_step;
    CKI(check_window(ctx, log_n, log_b, air.log_ce_blowup(), row0, ce_rows, &N));
    CKI(subcoset_step(ctx, log_n, air.log_ce_blowup(), sub_rows, &log_step));
    if (lde->m.rows != N || lde->m.cols != 2 * k) return wf_fail(ctx, WF_ERR_INVALID, "LDE shape does not match FibSmall x %u", k);
    switch (ext) {
        case 1: return eval_constraints_entry<1>(ctx, air, log_n, log_b, lde, nullptr, coeffs, nullptr, out, row0, ce_rows, log_step);
        case 2: return eval_constraints_entry<2>(ctx, air, log_n, log_b, lde, nullptr, coeffs, nullptr, out, row0, ce_rows, log_step);
        case 3: return eval_constraints_entry<3>(ctx, air, log_n, log_b, lde, nullptr, coeffs, nullptr, out, row0, ce_rows, log_step);
    }
    return wf_fail(ctx, WF_ERR_INVALID, "field extension %u", ext);
}
extern "C" int wf_eval_constraints_fib(wf_ctx* ctx, uint32_t k, const uint64_t* results, uint32_t log_n, uint32_t blowup, uint32_t ext,
                                       const wf_mat* lde, const uint64_t* coeffs, size_t row0, size_t ce_rows, wf_mat** out) {
    return eval_constraints_fib(ctx, k, results, log_n, blowup, ext, lde, coeffs, row0, ce_rows, 0, out);
}
extern "C" int wf_eval_constraints_fib_subcoset(wf_ctx* ctx, uint32_t k, const uint64_t* results, uint32_t log_n, uint32_t blowup,
                                                uint32_t ext, const wf_mat* lde, const uint64_t* coeffs, size_t rows, wf_mat** out) {
    if (!rows) return wf_fail(ctx, WF_ERR_INVALID, "empty sub-coset");
    return eval_constraints_fib(ctx, k, results, log_n, blowup, ext, lde, coeffs, 0, 0, rows, out);
}

extern "C" int wf_composition_commit(wf_ctx* ctx, int hash_id, const wf_mat* comp_trace, uint32_t log_n, uint32_t blowup, uint32_t ext,
                                     uint32_t num_cols, wf_mat** polys, wf_mat** lde, wf_tree** tree) {
    if (!ctx || !comp_trace || !polys || !lde || !tree || ext < 1 || ext > 3 || num_cols == 0 || blowup < 2 || (blowup & (blowup - 1)))
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    return composition_commit(ctx, hash_id, comp_trace, log_n, log2_ceil(blowup), (int)ext, num_cols, polys, lde, tree);
}
extern "C" int wf_composition_commit_partitioned(wf_ctx* ctx, int hash_id, const wf_mat* comp_trace, uint32_t log_n, uint32_t blowup,
                                                 uint32_t ext, uint32_t num_cols, uint32_t partition_size, wf_mat** polys, wf_mat** lde,
                                                 wf_tree** tree) {
    if (!ctx || !comp_trace || !polys || !lde || !tree || ext < 1 || ext > 3 || num_cols == 0 || blowup < 2 || (blowup & (blowup - 1)))
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    return composition_commit(ctx, hash_id, comp_trace, log_n, log2_ceil(blowup), (int)ext, num_cols, polys, lde, tree, partition_size);
}

template <int D>
static int evaluate_at_entry(wf_ctx* ctx, const wf_mat* polys, u32 col_ext, const uint64_t* z0, const uint64_t* z1, uint64_t* o0,
                             uint64_t* o1) {
    GlExt<D> a = ext_zero<D>(), b = ext_zero<D>();
    for (int q = 0; q < D; q++) { a.v[q] = z0[q]; b.v[q] = z1[q]; }
    std::vector<std::vector<GlExt<D>>> ev;
    CKI(ood_eval<D>(ctx, {polys}, a, b, ev));
    for (int pt = 0; pt < 2; pt++) {
        uint64_t* o = pt ? o1 : o0;
        const std::vector<GlExt<D>> cols = ext_from_components<D>(ev[pt], col_ext);
        for (size_t j = 0; j < cols.size(); j++) for (int q = 0; q < D; q++) o[j * D + q] = cols[j].v[q];
    }
    return WF_OK;
}
extern "C" int wf_mat_evaluate_at(wf_ctx* ctx, const wf_mat* polys, uint32_t ext, uint32_t col_ext, const uint64_t* z0, const uint64_t* z1,
                                  uint64_t* out0, uint64_t* out1) {
    if (!ctx || !polys || !z0 || !z1 || !out0 || !out1 || (col_ext != 1 && col_ext != ext) || polys->m.cols % col_ext)
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    switch (ext) {
        case 1: return evaluate_at_entry<1>(ctx, polys, col_ext, z0, z1, out0, out1);
        case 2: return evaluate_at_entry<2>(ctx, polys, col_ext, z0, z1, out0, out1);
        case 3: return evaluate_at_entry<3>(ctx, polys, col_ext, z0, z1, out0, out1);
    }
    return wf_fail(ctx, WF_ERR_UNSUPPORTED, "field extension %u", ext);
}

template <int D>
static int deep_entry(wf_ctx* ctx, const wf_mat* lde, const wf_mat* alde, const wf_mat* clde, u32 log_n, const uint64_t* zw,
                      const uint64_t* coeffs, const uint64_t* ood_cur, const uint64_t* ood_next, wf_mat** out) {
    const u32 c = lde->m.cols, aw = alde ? alde->m.cols / D : 0, kc = clde->m.cols / D, tot = c + aw + kc;
    const u32 log_N = log2_ceil(lde->m.rows);
    if (log_n > log_N) return wf_fail(ctx, WF_ERR_INVALID, "trace length exceeds the LDE domain");
    std::vector<GlExt<D>> dc(tot);
    GlExt<D> z = ext_zero<D>(), Sz = ext_zero<D>(), Szg = ext_zero<D>();
    for (int q = 0; q < D; q++) z.v[q] = zw[q];
    for (u32 i = 0; i < tot; i++) {
        GlExt<D> a = ext_zero<D>(), b = ext_zero<D>();
        for (int q = 0; q < D; q++) { dc[i].v[q] = coeffs[i * D + q]; a.v[q] = ood_cur[i * D + q]; b.v[q] = ood_next[i * D + q]; }
        Sz = ext_add(Sz, ext_mul(dc[i], a));
        Szg = ext_add(Szg, ext_mul(dc[i], b));
    }
    GlExt<D> zg = ext_mul_base(z, gl_root_of_unity(log_n));
    return deep_compose<D>(ctx, lde, alde, clde, kc, log_N, dc, z, zg, Sz, Szg, out);
}
extern "C" int wf_deep_compose(wf_ctx* ctx, uint32_t ext, const wf_mat* main_lde, const wf_mat* aux_lde, const wf_mat* cons_lde,
                               uint32_t log_n, const uint64_t* z, const uint64_t* coeffs, const uint64_t* ood_cur,
                               const uint64_t* ood_next, wf_mat** out) {
    if (!ctx || !main_lde || !cons_lde || !z || !coeffs || !ood_cur || !ood_next || !out || ext < 1 || ext > 3 ||
        cons_lde->m.cols % ext || cons_lde->m.rows != main_lde->m.rows || (aux_lde && (aux_lde->m.cols % ext || aux_lde->m.rows != main_lde->m.rows)))
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    switch (ext) {
        case 1: return deep_entry<1>(ctx, main_lde, aux_lde, cons_lde, log_n, z, coeffs, ood_cur, ood_next, out);
        case 2: return deep_entry<2>(ctx, main_lde, aux_lde, cons_lde, log_n, z, coeffs, ood_cur, ood_next, out);
        default: return deep_entry<3>(ctx, main_lde, aux_lde, cons_lde, log_n, z, coeffs, ood_cur, ood_next, out);
    }
}

template <int D>
static int deep_polys_entry(wf_ctx* ctx, const wf_mat* polys, const wf_mat* apolys, const wf_mat* cpolys, u32 log_n, u32 log_b,
                            const uint64_t* zw, const uint64_t* coeffs, wf_mat** out) {
    const u32 kc = cpolys->m.cols / D, tot = polys->m.cols + (apolys ? apolys->m.cols / D : 0) + kc;
    std::vector<GlExt<D>> dc(tot);
    GlExt<D> z = ext_zero<D>();
    for (int q = 0; q < D; q++) z.v[q] = zw[q];
    for (u32 i = 0; i < tot; i++) for (int q = 0; q < D; q++) dc[i].v[q] = coeffs[i * D + q];
    return deep_compose_polys<D>(ctx, polys, apolys, cpolys, kc, log_b, dc, z, ext_mul_base(z, gl_root_of_unity(log_n)), out);
}
extern "C" int wf_deep_compose_polys(wf_ctx* ctx, uint32_t ext, const wf_mat* main_polys, const wf_mat* aux_polys, const wf_mat* cons_polys,
                                     uint32_t log_blowup, const uint64_t* z, const uint64_t* coeffs, wf_mat** out) {
    if (!ctx || !main_polys || !cons_polys || !z || !coeffs || !out || ext < 1 || ext > 3 || cons_polys->m.cols % ext ||
        cons_polys->m.rows != main_polys->m.rows || (aux_polys && (aux_polys->m.cols % ext || aux_polys->m.rows != main_polys->m.rows)))
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    const size_t n = main_polys->m.rows;
    const u32 log_n = log2_ceil(n);
    if (n < 8 || (n & (n - 1))) return wf_fail(ctx, WF_ERR_INVALID, "rows must be a power of two >= 8");
    if (log_blowup < 1 || log_blowup > 7 || log_n + log_blowup > 32) return wf_fail(ctx, WF_ERR_INVALID, "bad blowup");
    switch (ext) {
        case 1: return deep_polys_entry<1>(ctx, main_polys, aux_polys, cons_polys, log_n, log_blowup, z, coeffs, out);
        case 2: return deep_polys_entry<2>(ctx, main_polys, aux_polys, cons_polys, log_n, log_blowup, z, coeffs, out);
        default: return deep_polys_entry<3>(ctx, main_polys, aux_polys, cons_polys, log_n, log_blowup, z, coeffs, out);
    }
}

// the proof bytes of one sharded proof, prove_sharded<D> for the extension degree of the options
static int prove_sharded_bytes(wf_ctx* ctx, const wf_comm* comm, const AirHost& air, const AuxBuildHost* aux_build,
                               wf_aux_assertions_fn aux_assertions, void* aux_user, const uint64_t* const* local_cols, const uint64_t* d_local,
                               int mont, uint32_t log_n, const Options& o, std::vector<u8>& out, double* stats) {
    switch (o.ext) {
        case 1: return prove_sharded<1>(ctx, comm, air, aux_build, aux_assertions, aux_user, local_cols, d_local, mont, log_n, o, out, stats);
        case 2: return prove_sharded<2>(ctx, comm, air, aux_build, aux_assertions, aux_user, local_cols, d_local, mont, log_n, o, out, stats);
        default: return prove_sharded<3>(ctx, comm, air, aux_build, aux_assertions, aux_user, local_cols, d_local, mont, log_n, o, out, stats);
    }
}
extern "C" int wf_prove_fib_sharded(wf_ctx* ctx, const wf_comm* comm, const uint64_t* const* local_cols, const uint64_t* d_local, int mont,
                                    uint32_t k, uint32_t log_n, const uint64_t* results, const uint32_t* opts, uint8_t* proof,
                                    size_t* proof_len, double* stats) {
    if (!ctx || !comm || !comm->exchange || !comm->all_gather_host || !comm->all_reduce_sum || (!local_cols && !d_local) || !results ||
        !opts || !proof || !proof_len || k == 0 || 2 * k > 255 || log_n < 3)
        return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    Options o;
    CKI(parse_options(ctx, opts, o));
    const AirHost air = fib_air_host(k, (size_t)1 << log_n, results);
    std::vector<u8> out;
    CKI(prove_sharded_bytes(ctx, comm, air, nullptr, nullptr, nullptr, local_cols, d_local, mont, log_n, o, out, stats));
    return copy_proof_out(ctx, out, proof, proof_len);
}
extern "C" int wf_shard_columns(uint32_t width, uint32_t world, uint32_t rank, uint32_t* first, uint32_t* count) {
    if (!first || !count || width == 0 || width > 255 || world == 0 || (world & (world - 1)) || rank >= world) return WF_ERR_INVALID;
    shard_columns(width, world, rank, *first, *count);
    return WF_OK;
}
extern "C" int wf_prove_air_sharded(wf_ctx* ctx, const wf_comm* comm, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* aux_build,
                                    size_t aux_build_len, wf_aux_assertions_fn aux_assertions, void* aux_user, const uint64_t* const* local_cols,
                                    const uint64_t* d_local, uint32_t local_count, int mont, uint32_t log_n, const uint32_t* opts,
                                    uint8_t* proof, size_t* proof_len, double* stats) {
    if (!ctx) return WF_ERR_INVALID;
    if (!comm || !comm->exchange || !comm->all_gather_host || !comm->all_reduce_sum) return wf_fail(ctx, WF_ERR_INVALID, "bad communicator");
    // Checks on what every rank shares (description, options, log_n, world size): the same verdict everywhere, before any
    // collective, so a refusal leaves no rank waiting.
    const int G = comm->world;
    if (G < 2 || (G & (G - 1)) || comm->rank < 0 || comm->rank >= G) return wf_fail(ctx, WF_ERR_INVALID, "world size must be a power of two >= 2");
    if (!air_desc || !opts || log_n < 3 || log_n > 32) return wf_fail(ctx, WF_ERR_INVALID, "bad arguments");
    Options o;
    CKI(parse_options(ctx, opts, o));
    AirHost air;
    if (!parse_air_host(air_desc, air_desc_len, air)) return wf_fail(ctx, WF_ERR_INVALID, "malformed AIR description");
    CKI(air_check_host(ctx, air, log_n, o.blowup));
    AuxBuildHost b;
    if (air.aw) {
        if (!aux_build) return wf_fail(ctx, WF_ERR_INVALID, "two-segment AIR: the sharded prover builds its aux segment from aux_build");
        CKI(parse_aux_build(ctx, air, aux_build, aux_build_len, o.ext, b));
    } else if (aux_build || aux_assertions) {
        return wf_fail(ctx, WF_ERR_INVALID, "single-segment AIR: it has no aux segment");
    }
    const size_t rows_per = ((size_t)1 << (log_n + log2_ceil(o.blowup))) / (size_t)G, ce_per = ((size_t)1 << (log_n + air.log_ce_blowup())) / (size_t)G;
    if (log_n + log2_ceil(o.blowup) > 32 || rows_per < 64 * (size_t)o.blowup || ce_per < 64)
        return wf_fail(ctx, WF_ERR_UNSUPPORTED, "trace too short to shard over %d ranks", G);
    const bool out_ok = proof && proof_len;
    CKI(agree_on_columns(ctx, comm, air.w, local_count, local_cols, d_local, &out_ok));
    std::vector<u8> out;
    CKI(prove_sharded_bytes(ctx, comm, air, air.aw ? &b : nullptr, aux_assertions, aux_user, local_cols, d_local, mont, log_n, o, out, stats));
    return copy_proof_out(ctx, out, proof, proof_len);
}
extern "C" int wf_prove_fib(wf_ctx* ctx, const uint64_t* const* trace_cols, int mont, uint32_t k, uint32_t log_n,
                            const uint64_t* results, const uint32_t* opts, uint8_t* proof, size_t* proof_len) {
    return prove_fib_entry(ctx, trace_cols, nullptr, mont, k, log_n, results, opts, proof, proof_len);
}
extern "C" int wf_prove_fib_dev(wf_ctx* ctx, const uint64_t* d_trace, uint32_t k, uint32_t log_n, const uint64_t* results,
                                const uint32_t* opts, uint8_t* proof, size_t* proof_len) {
    return prove_fib_entry(ctx, nullptr, d_trace, 0, k, log_n, results, opts, proof, proof_len);
}
