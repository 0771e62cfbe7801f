// auxbuild.cu — the auxiliary trace segment built on the device from a column-program description (the described
// alternative to Prover::build_aux_trace, prover/src/lib.rs:236-247; format and semantics at wf_aux_build in
// include/winterfell_b200.h). Every column is "a per-row term from a straight-line program, then a prefix scan":
//   aux_term_kernel    interprets the column's program for a run of AUX_TERM_ROWS consecutive rows per thread, registers in a
//                      local array as in the interpreted generic_constraints_kernel; the run's denominators share one extension
//                      field inversion (Montgomery's trick). POINTWISE columns are written straight into the aux matrix, the
//                      running kinds into a term buffer [n][D], LINEAR_RECURRENCE columns the pair (m_i, t_i) into [n][2D].
//   aux_scan_reduce    per tile of AUX_SCAN_TILE rows: the product / sum of its terms;
//   aux_scan_carry     one block: exclusive scan of the tile aggregates, seeded with the column's init;
//   aux_scan_apply     per tile: block-wide exclusive scan with the tile's carry-in, written into the aux matrix.
//   aux_affine_reduce / _carry / _apply   the same three steps for LINEAR_RECURRENCE columns, over the affine maps
//                      x -> m_i x + t_i: a tile's aggregate is the composition of its rows' maps, the carry is the column's value
//                      at each tile start (the composed prefix applied to init). Composition does not commute, so every step
//                      keeps the rows in order: a thread combines consecutive rows, and the warp and block steps keep the
//                      earlier operand on the left.
//   aux_moebius_term_kernel   RATIONAL_RECURRENCE columns: the program's four outputs, the map a -> (m_i a + n_i) / (c_i a + d_i)
//                      as the matrix (m_i, n_i, c_i, d_i), into [n][4D]; nothing is inverted there.
//   aux_moebius_reduce / _carry / _apply   the three scan steps over those 2x2 matrices, acting on projective pairs (x, y) ~ x / y:
//                      a tile's aggregate is the product of its rows' matrices (later rows on the left), the carry is the pair at
//                      each tile start (the composed prefix applied to (init, 1)), and apply writes a[i] = x_i inv(y_i) with one
//                      inversion per thread run (Montgomery's trick). Where y_z = 0 first, the serial value is a[z] = 0 (inv(0) = 0)
//                      and the pairs after z no longer follow it, so the host scans rows z .. again from (0, 1) (aux_moebius).
//   aux_coupled_term_kernel   COUPLED_RECURRENCE groups of k columns: the leader's program gives row i's affine map on E^k,
//                      the augmented matrix [M_i | t_i] row by row into [n][k (k + 1) D]; nothing is inverted there.
//   aux_coupled_reduce / _carry / _apply   the three scan steps over those maps, one map per group of k lanes (padded to 2 or
//                      4): a tile's aggregate is the composition of its rows' maps (later rows on the left), the carry is the
//                      state vector at each tile start (the composed prefix applied to the inits), and apply writes the k
//                      columns. Nothing is inverted, so no row is ever scanned again.
// Field arithmetic is exact, so the association order of the scan does not change a bit of the result.
#include "internal.hpp"
#include "constraints_generic.cuh"  // ld_ext, seg_at, AUX_MAX_REGS

#define AUX_TERM_ROWS 4
#define AUX_TERM_THREADS 128
#define AUX_SCAN_THREADS 256
#define AUX_SCAN_ITEMS 8
#define AUX_SCAN_TILE (AUX_SCAN_THREADS * AUX_SCAN_ITEMS)

struct AuxTermParams {
    SegMatrix main;        // n x w evaluations of the main segment
    SegMatrix aux;         // n x aw*D, columns < col already built
    u32 w, aw, np, nr, col, log_n;
    const u32* prog;       // [len][4] op, dst, a, b
    u32 prog_len;
    const u64* consts;
    const u64* ptab;       // periodic columns over the trace domain, concatenated
    const u32* ptab_off;
    const u32* ptab_len;   // powers of two
    const u64* rnd;        // [nr][D]
    u64* terms;            // [n][D] running kinds, [n][2D] (m_i, t_i) LINEAR_RECURRENCE, [n][4D] (m_i, n_i, c_i, d_i)
                           // RATIONAL_RECURRENCE, [n][k (k + 1) D] [M_i | t_i] COUPLED_RECURRENCE; nullptr: POINTWISE, written
                           // into aux column `col`
};

template <int D>
__device__ __forceinline__ void st_aux(const SegMatrix& m, size_t row, u32 col, const GlExt<D>& v) {
#pragma unroll
    for (int q = 0; q < D; q++) {
        const u32 c = col * D + q;
        m.base[(size_t)(c / m.W) * m.seg_stride + row * m.W + (c % m.W)] = v.v[q];
    }
}

// the registers a program may read at row i (wf_aux_build_check): main rows, aux columns < col, periodic values, random elements
template <int D>
__device__ __forceinline__ void aux_load_regs(const AuxTermParams& p, size_t i, size_t nx, u32 ab, u32 pb, GlExt<D>* ra) {
    for (u32 c = 0; c < p.w; c++) { ra[c] = ext_from_base<D>(seg_at(p.main, i, c)); ra[p.w + c] = ext_from_base<D>(seg_at(p.main, nx, c)); }
    for (u32 j = 0; j < p.col; j++) {
#pragma unroll
        for (int q = 0; q < D; q++) {
            ra[ab + j].v[q] = seg_at(p.aux, i, j * D + q);
            ra[ab + p.aw + j].v[q] = seg_at(p.aux, nx, j * D + q);
        }
    }
    for (u32 j = 0; j < p.np; j++) ra[pb + j] = ext_from_base<D>(p.ptab[p.ptab_off[j] + (u32)(i & (p.ptab_len[j] - 1))]);
    for (u32 j = 0; j < p.nr; j++) ra[pb + p.np + j] = ld_ext<D>(p.rnd + (size_t)j * D);
}

template <int D>
__device__ __forceinline__ GlExt<D> ld_aux(const SegMatrix& m, size_t row, u32 col) {
    GlExt<D> v;
#pragma unroll
    for (int q = 0; q < D; q++) {
        const u32 c = col * D + q;
        v.v[q] = m.base[(size_t)(c / m.W) * m.seg_stride + row * m.W + (c % m.W)];
    }
    return v;
}

// AFFINE: a LINEAR_RECURRENCE column, whose program also gives the multiplier m_i (OUT 2)
template <int D, bool AFFINE>
__global__ void __launch_bounds__(AUX_TERM_THREADS) aux_term_kernel(AuxTermParams p) {
    const size_t n = (size_t)1 << p.log_n;
    const size_t row0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * AUX_TERM_ROWS;
    if (row0 >= n) return;
    GlExt<D> num[AUX_TERM_ROWS], den[AUX_TERM_ROWS], pre[AUX_TERM_ROWS], mlt[AUX_TERM_ROWS];
    bool zero[AUX_TERM_ROWS];
    GlExt<D> run = ext_from_base<D>(1);
    GlExt<D> ra[AUX_MAX_REGS];
    const u32 ab = 2 * p.w, pb = 2 * p.w + 2 * p.aw;
#pragma unroll
    for (int r = 0; r < AUX_TERM_ROWS; r++) {
        const size_t i = row0 + r, nx = (i + 1) & (n - 1);
        aux_load_regs<D>(p, i, nx, ab, pb, ra);
        num[r] = ext_zero<D>();
        den[r] = ext_from_base<D>(1);
        for (u32 k = 0; k < p.prog_len; k++) {
            const u32 op = p.prog[4 * k], dst = p.prog[4 * k + 1], a = p.prog[4 * k + 2], b = p.prog[4 * k + 3];
            switch (op) {
                case 0: ra[dst] = ext_add(ra[a], ra[b]); break;
                case 1: ra[dst] = ext_sub(ra[a], ra[b]); break;
                case 2: ra[dst] = ext_mul(ra[a], ra[b]); break;
                case 3: ra[dst] = ext_from_base<D>(p.consts[a]); break;
                default:  // OUT 0 numerator, OUT 1 denominator, OUT 2 multiplier
                    if (dst == 0) num[r] = ra[a];
                    else if (AFFINE && dst == 2) mlt[r] = ra[a];
                    else den[r] = ra[a];
                    break;
            }
        }
        // Montgomery's trick; a zero denominator becomes 1 inside the batch and its term 0 (inv(0) = 0)
        zero[r] = true;
#pragma unroll
        for (int q = 0; q < D; q++) zero[r] = zero[r] && den[r].v[q] == 0;
        if (zero[r]) den[r] = ext_from_base<D>(1);
        pre[r] = run;
        run = ext_mul(run, den[r]);
    }
    run = ext_inv(run);
#pragma unroll
    for (int r = AUX_TERM_ROWS - 1; r >= 0; r--) {
        const GlExt<D> inv = ext_mul(run, pre[r]);
        run = ext_mul(run, den[r]);
        const GlExt<D> t = zero[r] ? ext_zero<D>() : ext_mul(num[r], inv);
        const size_t i = row0 + r;
        if (AFFINE) {
#pragma unroll
            for (int q = 0; q < D; q++) { p.terms[i * 2 * D + q] = mlt[r].v[q]; p.terms[i * 2 * D + D + q] = t.v[q]; }
        } else if (p.terms) {
#pragma unroll
            for (int q = 0; q < D; q++) p.terms[i * D + q] = t.v[q];
        } else {
            st_aux<D>(p.aux, i, p.col, t);
        }
    }
}

template <int D, bool MUL>
__device__ __forceinline__ GlExt<D> scan_op(const GlExt<D>& a, const GlExt<D>& b) { return MUL ? ext_mul(a, b) : ext_add(a, b); }
template <int D, bool MUL>
__device__ __forceinline__ GlExt<D> scan_id() { return MUL ? ext_from_base<D>(1) : ext_zero<D>(); }
template <int D>
__device__ __forceinline__ GlExt<D> shfl_up_ext(const GlExt<D>& v, u32 off) {
    GlExt<D> r;
#pragma unroll
    for (int q = 0; q < D; q++) r.v[q] = __shfl_up_sync(0xffffffffu, v.v[q], off);
    return r;
}
// The combine of a block scan as a type: T its state, W its u64 words, id() the identity, op(a, b) = a then b (the earlier
// operand on the left), and T's warp shuffle and memory forms.
template <int D, bool MUL>
struct RunOp {   // RUNNING_PRODUCT / RUNNING_SUM: one extension element
    using T = GlExt<D>;
    static constexpr int W = D;
    static __device__ __forceinline__ T id() { return scan_id<D, MUL>(); }
    static __device__ __forceinline__ T op(const T& a, const T& b) { return scan_op<D, MUL>(a, b); }
    static __device__ __forceinline__ T shfl_up(const T& v, u32 off) { return shfl_up_ext(v, off); }
    static __device__ __forceinline__ T ld(const u64* p) { return ld_ext<D>(p); }
    static __device__ __forceinline__ void st(u64* p, const T& v) {
#pragma unroll
        for (int q = 0; q < D; q++) p[q] = v.v[q];
    }
};
template <int D>
struct Affine { GlExt<D> m, t; };   // the map x -> m x + t; in memory m then t, 2D words
template <int D>
__device__ __forceinline__ GlExt<D> aff_apply(const Affine<D>& a, const GlExt<D>& x) { return ext_add(ext_mul(a.m, x), a.t); }
template <int D>
struct AffOp {   // LINEAR_RECURRENCE: composition of affine maps; a then b = (a.m b.m, b.m a.t + b.t)
    using T = Affine<D>;
    static constexpr int W = 2 * D;
    static __device__ __forceinline__ T id() { return {ext_from_base<D>(1), ext_zero<D>()}; }
    static __device__ __forceinline__ T op(const T& a, const T& b) { return {ext_mul(a.m, b.m), aff_apply(b, a.t)}; }
    static __device__ __forceinline__ T shfl_up(const T& v, u32 off) { return {shfl_up_ext(v.m, off), shfl_up_ext(v.t, off)}; }
    static __device__ __forceinline__ T ld(const u64* p) { return {ld_ext<D>(p), ld_ext<D>(p + D)}; }
    static __device__ __forceinline__ void st(u64* p, const T& v) {
#pragma unroll
        for (int q = 0; q < D; q++) { p[q] = v.m.v[q]; p[D + q] = v.t.v[q]; }
    }
};
template <int D>
struct Moebius { GlExt<D> m, n, c, d; };   // the matrix [[m, n], [c, d]]: a -> (m a + n) / (c a + d); in memory m, n, c, d, 4D words
template <int D>
__device__ __forceinline__ void mob_apply(const Moebius<D>& a, GlExt<D>& x, GlExt<D>& y) {   // (x, y) <- A (x, y)
    const GlExt<D> x2 = ext_add(ext_mul(a.m, x), ext_mul(a.n, y));
    y = ext_add(ext_mul(a.c, x), ext_mul(a.d, y));
    x = x2;
}
template <int D>
struct MobOp {   // RATIONAL_RECURRENCE: composition of Moebius maps as 2x2 matrices up to scale; a then b = B A
    using T = Moebius<D>;
    static constexpr int W = 4 * D;
    static __device__ __forceinline__ T id() { return {ext_from_base<D>(1), ext_zero<D>(), ext_zero<D>(), ext_from_base<D>(1)}; }
    static __device__ __forceinline__ T op(const T& a, const T& b) {
        return {ext_add(ext_mul(b.m, a.m), ext_mul(b.n, a.c)), ext_add(ext_mul(b.m, a.n), ext_mul(b.n, a.d)),
                ext_add(ext_mul(b.c, a.m), ext_mul(b.d, a.c)), ext_add(ext_mul(b.c, a.n), ext_mul(b.d, a.d))};
    }
    static __device__ __forceinline__ T shfl_up(const T& v, u32 off) {
        return {shfl_up_ext(v.m, off), shfl_up_ext(v.n, off), shfl_up_ext(v.c, off), shfl_up_ext(v.d, off)};
    }
    static __device__ __forceinline__ T ld(const u64* p) { return {ld_ext<D>(p), ld_ext<D>(p + D), ld_ext<D>(p + 2 * D), ld_ext<D>(p + 3 * D)}; }
    static __device__ __forceinline__ void st(u64* p, const T& v) {
#pragma unroll
        for (int q = 0; q < D; q++) { p[q] = v.m.v[q]; p[D + q] = v.n.v[q]; p[2 * D + q] = v.c.v[q]; p[3 * D + q] = v.d.v[q]; }
    }
};

// RATIONAL_RECURRENCE: row i's map (m_i, n_i, c_i, d_i) = (OUT 2, OUT 0, OUT 3, OUT 1) into terms [n][4D]; one row per thread
template <int D>
__global__ void __launch_bounds__(AUX_TERM_THREADS) aux_moebius_term_kernel(AuxTermParams p) {
    const size_t n = (size_t)1 << p.log_n;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    GlExt<D> ra[AUX_MAX_REGS];
    aux_load_regs<D>(p, i, (i + 1) & (n - 1), 2 * p.w, 2 * p.w + 2 * p.aw, ra);
    Moebius<D> o = MobOp<D>::id();   // d_i defaults to 1; the program writes the other three exactly once
    for (u32 k = 0; k < p.prog_len; k++) {
        const u32 op = p.prog[4 * k], dst = p.prog[4 * k + 1], a = p.prog[4 * k + 2], b = p.prog[4 * k + 3];
        switch (op) {
            case 0: ra[dst] = ext_add(ra[a], ra[b]); break;
            case 1: ra[dst] = ext_sub(ra[a], ra[b]); break;
            case 2: ra[dst] = ext_mul(ra[a], ra[b]); break;
            case 3: ra[dst] = ext_from_base<D>(p.consts[a]); break;
            default:  // OUT 0 numerator n_i, OUT 1 denominator d_i, OUT 2 multiplier m_i, OUT 3 denominator multiplier c_i
                if (dst == 0) o.n = ra[a];
                else if (dst == 1) o.d = ra[a];
                else if (dst == 2) o.m = ra[a];
                else o.c = ra[a];
                break;
        }
    }
    MobOp<D>::st(p.terms + i * 4 * D, o);
}

// exclusive scan of one value per thread over the block (AUX_SCAN_THREADS threads), in thread order; `total` = the whole
// block's result
template <class Op>
__device__ __forceinline__ typename Op::T block_exclusive_scan(const typename Op::T& v, typename Op::T& total) {
    using T = typename Op::T;
    __shared__ u64 wsum[AUX_SCAN_THREADS / 32][Op::W];
    const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    constexpr u32 NW = AUX_SCAN_THREADS / 32;
    T x = v;
#pragma unroll
    for (u32 off = 1; off < 32; off <<= 1) {
        const T y = Op::shfl_up(x, off);
        if (lane >= off) x = Op::op(y, x);
    }
    if (lane == 31) Op::st(&wsum[wid][0], x);
    __syncthreads();
    if (wid == 0) {
        T s = lane < NW ? Op::ld(&wsum[lane][0]) : Op::id();
#pragma unroll
        for (u32 off = 1; off < NW; off <<= 1) {
            const T y = Op::shfl_up(s, off);
            if (lane >= off) s = Op::op(y, s);
        }
        if (lane < NW) Op::st(&wsum[lane][0], s);
    }
    __syncthreads();
    total = Op::ld(&wsum[NW - 1][0]);
    const T wpre = wid ? Op::ld(&wsum[wid - 1][0]) : Op::id();
    T ex = Op::shfl_up(x, 1);
    if (lane == 0) ex = Op::id();
    __syncthreads();  // wsum is free for the next call
    return Op::op(wpre, ex);
}

template <int D, bool MUL>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_scan_reduce(const u64* terms, size_t n, u64* agg) {
    const size_t t0 = (size_t)blockIdx.x * AUX_SCAN_TILE;
    GlExt<D> v = scan_id<D, MUL>();
#pragma unroll
    for (int k = 0; k < AUX_SCAN_ITEMS; k++) {   // coalesced: the order inside a tile does not matter for its aggregate
        const size_t i = t0 + (size_t)k * AUX_SCAN_THREADS + threadIdx.x;
        if (i < n) v = scan_op<D, MUL>(v, ld_ext<D>(terms + i * D));
    }
    GlExt<D> total;
    block_exclusive_scan<RunOp<D, MUL>>(v, total);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int q = 0; q < D; q++) agg[(size_t)blockIdx.x * D + q] = total.v[q];
    }
}

// one block; tile aggregates -> exclusive prefixes seeded with init, in place. Thread t owns a run of consecutive tiles.
template <int D, bool MUL>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_scan_carry(u64* agg, size_t ntiles, GlExt<D> init) {
    const size_t per = (ntiles + AUX_SCAN_THREADS - 1) / AUX_SCAN_THREADS;
    const size_t b = threadIdx.x * per, e = b + per < ntiles ? b + per : ntiles;
    GlExt<D> v = scan_id<D, MUL>();
    for (size_t i = b; i < e; i++) v = scan_op<D, MUL>(v, ld_ext<D>(agg + i * D));
    GlExt<D> total;
    GlExt<D> run = scan_op<D, MUL>(init, block_exclusive_scan<RunOp<D, MUL>>(v, total));
    for (size_t i = b; i < e; i++) {
        const GlExt<D> a = ld_ext<D>(agg + i * D);
#pragma unroll
        for (int q = 0; q < D; q++) agg[i * D + q] = run.v[q];
        run = scan_op<D, MUL>(run, a);
    }
}

// a[i] = carry(tile) * (terms of the tile's rows before i), written as aux column `col`; thread t owns AUX_SCAN_ITEMS
// consecutive rows (the second pass re-reads them from L1)
template <int D, bool MUL>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_scan_apply(const u64* terms, size_t n, const u64* carry, SegMatrix out, u32 col) {
    const size_t r0 = (size_t)blockIdx.x * AUX_SCAN_TILE + (size_t)threadIdx.x * AUX_SCAN_ITEMS;
    GlExt<D> v = scan_id<D, MUL>();
#pragma unroll
    for (int k = 0; k < AUX_SCAN_ITEMS; k++)
        if (r0 + k < n) v = scan_op<D, MUL>(v, ld_ext<D>(terms + (r0 + k) * D));
    GlExt<D> total;
    GlExt<D> run = scan_op<D, MUL>(ld_ext<D>(carry + (size_t)blockIdx.x * D), block_exclusive_scan<RunOp<D, MUL>>(v, total));
#pragma unroll
    for (int k = 0; k < AUX_SCAN_ITEMS; k++) {
        const size_t i = r0 + k;
        if (i < n) {
            st_aux<D>(out, i, col, run);
            run = scan_op<D, MUL>(run, ld_ext<D>(terms + i * D));
        }
    }
}

// The composition of the maps of rows r0 .. r0 + AUX_SCAN_ITEMS - 1 (those < n), in row order; the identity when r0 >= n.
template <int D>
__device__ __forceinline__ Affine<D> affine_run(const u64* terms, size_t n, size_t r0) {
    Affine<D> v = r0 < n ? AffOp<D>::ld(terms + r0 * 2 * D) : AffOp<D>::id();
#pragma unroll
    for (int k = 1; k < AUX_SCAN_ITEMS; k++)
        if (r0 + k < n) v = AffOp<D>::op(v, AffOp<D>::ld(terms + (r0 + k) * 2 * D));
    return v;
}

// per tile: the composition of its rows' maps into agg [ntiles][2D]; thread t owns AUX_SCAN_ITEMS consecutive rows
template <int D>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_affine_reduce(const u64* terms, size_t n, u64* agg) {
    const Affine<D> v = affine_run<D>(terms, n, (size_t)blockIdx.x * AUX_SCAN_TILE + (size_t)threadIdx.x * AUX_SCAN_ITEMS);
    Affine<D> total;
    block_exclusive_scan<AffOp<D>>(v, total);
    if (threadIdx.x == 0) AffOp<D>::st(agg + (size_t)blockIdx.x * 2 * D, total);
}

// one block; tile maps -> the column's value at each tile start (the maps of the tiles before it applied to init), written
// over the first D words of the tile's slot. Thread t owns a run of consecutive tiles.
template <int D>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_affine_carry(u64* agg, size_t ntiles, GlExt<D> init) {
    const size_t per = (ntiles + AUX_SCAN_THREADS - 1) / AUX_SCAN_THREADS;
    const size_t b = threadIdx.x * per, e = b + per < ntiles ? b + per : ntiles;
    Affine<D> v = AffOp<D>::id();
    for (size_t i = b; i < e; i++) v = AffOp<D>::op(v, AffOp<D>::ld(agg + i * 2 * D));
    Affine<D> total;
    GlExt<D> x = aff_apply(block_exclusive_scan<AffOp<D>>(v, total), init);
    for (size_t i = b; i < e; i++) {
        const Affine<D> a = AffOp<D>::ld(agg + i * 2 * D);
#pragma unroll
        for (int q = 0; q < D; q++) agg[i * 2 * D + q] = x.v[q];
        x = aff_apply(a, x);
    }
}

// a[i] = the maps of the tile's rows before i applied to the tile's carry-in, written as aux column `col`; thread t owns
// AUX_SCAN_ITEMS consecutive rows (the second pass re-reads them from L1)
template <int D>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_affine_apply(const u64* terms, size_t n, const u64* carry, SegMatrix out, u32 col) {
    const size_t r0 = (size_t)blockIdx.x * AUX_SCAN_TILE + (size_t)threadIdx.x * AUX_SCAN_ITEMS;
    const Affine<D> v = affine_run<D>(terms, n, r0);
    Affine<D> total;
    GlExt<D> x = aff_apply(block_exclusive_scan<AffOp<D>>(v, total), ld_ext<D>(carry + (size_t)blockIdx.x * 2 * D));
#pragma unroll 1   // unrolled, the D = 3 kernel spills to local memory
    for (int k = 0; k < AUX_SCAN_ITEMS; k++) {
        const size_t i = r0 + k;
        if (i < n) {
            st_aux<D>(out, i, col, x);
            x = aff_apply(AffOp<D>::ld(terms + i * 2 * D), x);
        }
    }
}

// The product of the matrices of rows r0 .. r0 + AUX_SCAN_ITEMS - 1 (those < n), later rows on the left; the identity when r0 >= n.
template <int D>
__device__ __forceinline__ Moebius<D> moebius_run(const u64* terms, size_t n, size_t r0) {
    Moebius<D> v = r0 < n ? MobOp<D>::ld(terms + r0 * 4 * D) : MobOp<D>::id();
#pragma unroll
    for (int k = 1; k < AUX_SCAN_ITEMS; k++)
        if (r0 + k < n) v = MobOp<D>::op(v, MobOp<D>::ld(terms + (r0 + k) * 4 * D));
    return v;
}

// per tile: the product of its rows' matrices into agg [ntiles][4D]; thread t owns AUX_SCAN_ITEMS consecutive rows
template <int D>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_moebius_reduce(const u64* terms, size_t n, u64* agg) {
    const Moebius<D> v = moebius_run<D>(terms, n, (size_t)blockIdx.x * AUX_SCAN_TILE + (size_t)threadIdx.x * AUX_SCAN_ITEMS);
    Moebius<D> total;
    block_exclusive_scan<MobOp<D>>(v, total);
    if (threadIdx.x == 0) MobOp<D>::st(agg + (size_t)blockIdx.x * 4 * D, total);
}

// one block; tile matrices -> the pair (x, y) at each tile start (the matrices of the tiles before it applied to (init, 1)),
// written over the first 2D words of the tile's slot. Thread t owns a run of consecutive tiles.
template <int D>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_moebius_carry(u64* agg, size_t ntiles, GlExt<D> init) {
    const size_t per = (ntiles + AUX_SCAN_THREADS - 1) / AUX_SCAN_THREADS;
    const size_t b = threadIdx.x * per, e = b + per < ntiles ? b + per : ntiles;
    Moebius<D> v = MobOp<D>::id();
    for (size_t i = b; i < e; i++) v = MobOp<D>::op(v, MobOp<D>::ld(agg + i * 4 * D));
    Moebius<D> total;
    GlExt<D> x = init, y = ext_from_base<D>(1);
    mob_apply(block_exclusive_scan<MobOp<D>>(v, total), x, y);
    for (size_t i = b; i < e; i++) {
        const Moebius<D> a = MobOp<D>::ld(agg + i * 4 * D);
#pragma unroll
        for (int q = 0; q < D; q++) { agg[i * 4 * D + q] = x.v[q]; agg[i * 4 * D + D + q] = y.v[q]; }
        mob_apply(a, x, y);
    }
}

// rows base + r of aux column `col`, r < n: (x_r, y_r) = the matrices of the tile's rows before r applied to the tile's carry-in,
// a = x_r inv(y_r), the run's y_r inverted together (Montgomery's trick). A row with y_r = 0 counts as 1 in that batch and lowers
// *zmin to base + r; it and the rows after it are scanned again. Thread t owns AUX_SCAN_ITEMS consecutive rows.
template <int D>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_moebius_apply(const u64* terms, size_t n, const u64* carry, SegMatrix out, u32 col,
                                                                      size_t base, unsigned long long* zmin) {
    const size_t r0 = (size_t)blockIdx.x * AUX_SCAN_TILE + (size_t)threadIdx.x * AUX_SCAN_ITEMS;
    const Moebius<D> v = moebius_run<D>(terms, n, r0);
    Moebius<D> total;
    const Moebius<D> pre = block_exclusive_scan<MobOp<D>>(v, total);
    GlExt<D> x = ld_ext<D>(carry + (size_t)blockIdx.x * 4 * D), y = ld_ext<D>(carry + (size_t)blockIdx.x * 4 * D + D);
    mob_apply(pre, x, y);
    // forward: w_k = x_k * (y of the run's rows before k), parked in the output; backward: a_k = w_k * (y of the rows after k) /
    // (product of all y)
    GlExt<D> ys[AUX_SCAN_ITEMS];
    GlExt<D> run = ext_from_base<D>(1);
    unsigned long long z = ~0ull;
#pragma unroll
    for (int k = 0; k < AUX_SCAN_ITEMS; k++) {
        const size_t r = r0 + k;
        if (r < n) {
            bool zero = true;
#pragma unroll
            for (int q = 0; q < D; q++) zero = zero && y.v[q] == 0;
            if (zero && z == ~0ull) z = base + r;
            ys[k] = zero ? ext_from_base<D>(1) : y;
            st_aux<D>(out, base + r, col, ext_mul(x, run));
            run = ext_mul(run, ys[k]);
            mob_apply(MobOp<D>::ld(terms + r * 4 * D), x, y);
        }
    }
    run = ext_inv(run);
#pragma unroll
    for (int k = AUX_SCAN_ITEMS - 1; k >= 0; k--) {
        const size_t r = r0 + k;
        if (r < n) {
            st_aux<D>(out, base + r, col, ext_mul(ld_aux<D>(out, base + r, col), run));
            run = ext_mul(run, ys[k]);
        }
    }
    if (z != ~0ull) atomicMin(zmin, z);
}

// ---- COUPLED_RECURRENCE groups: a[i+1] = M_i a[i] + t_i over k = 2..4 columns --------------------------------------------
// A map (M, t) on E^k is k rows of the augmented matrix [M | t], k + 1 elements each; in the term buffer row r of row i's map is
// at words i S + r (k + 1) D, S = k (k + 1) D. In the scan kernels a map lives on a group of K lanes (k padded to 2 or 4): lane
// r < k holds row r, the padding lane holds zeros and is never read. Composition takes the other rows from the group by
// shuffles; applying a map to a state vector (lane r holds a_r) takes k shuffles of one element.
template <int k>
__host__ __device__ constexpr int cp_lanes() { return k == 2 ? 2 : 4; }
template <int k, int D>
struct CRow { GlExt<D> e[k + 1]; };   // row r of [M | t]: M[r][0 .. k-1], then t_r

// the rows of one scan tile that a lane group owns: AUX_SCAN_TILE rows over AUX_SCAN_THREADS / K groups
template <int k>
__host__ __device__ constexpr int cp_items() { return AUX_SCAN_TILE / (AUX_SCAN_THREADS / cp_lanes<k>()); }

template <int D>
__device__ __forceinline__ GlExt<D> shfl_grp(u32 mask, const GlExt<D>& v, int src, int width) {
    GlExt<D> r;
#pragma unroll
    for (int q = 0; q < D; q++) r.v[q] = __shfl_sync(mask, v.v[q], src, width);
    return r;
}
template <int k, int D>
__device__ __forceinline__ CRow<k, D> crow_id(u32 r) {
    CRow<k, D> v;
#pragma unroll
    for (int c = 0; c <= k; c++) v.e[c] = (u32)c == r ? ext_from_base<D>(1) : ext_zero<D>();
    return v;
}
template <int k, int D>
__device__ __forceinline__ CRow<k, D> crow_ld(const u64* p, u32 r) {   // p: one map (S words); zeros on the padding lane
    CRow<k, D> v;
#pragma unroll
    for (int c = 0; c <= k; c++) v.e[c] = r < (u32)k ? ld_ext<D>(p + (r * (k + 1) + c) * D) : ext_zero<D>();
    return v;
}
template <int k, int D>
__device__ __forceinline__ void crow_st(u64* p, u32 r, const CRow<k, D>& v) {
    if (r >= (u32)k) return;
#pragma unroll
    for (int c = 0; c <= k; c++)
#pragma unroll
        for (int q = 0; q < D; q++) p[(r * (k + 1) + c) * D + q] = v.e[c].v[q];
}
// "a then b" = B o A, row r: M'[r][c] = sum_s B[r][s] A[s][c], t'_r = sum_s B[r][s] A_t[s] + B_t[r]; lane r holds row r of a and
// b, the rows of a come from its group (gmask, width K)
template <int k, int D>
__device__ __forceinline__ CRow<k, D> crow_op(u32 gmask, const CRow<k, D>& a, const CRow<k, D>& b) {
    CRow<k, D> o;
#pragma unroll
    for (int c = 0; c < k; c++) o.e[c] = ext_zero<D>();
    o.e[k] = b.e[k];
#pragma unroll
    for (int s = 0; s < k; s++)
#pragma unroll
        for (int c = 0; c <= k; c++) o.e[c] = ext_add(o.e[c], ext_mul(b.e[s], shfl_grp(gmask, a.e[c], s, cp_lanes<k>())));
    return o;
}
// the state vector after the map: lane r gets sum_s M[r][s] x_s + t_r
template <int k, int D>
__device__ __forceinline__ GlExt<D> crow_apply(u32 gmask, const CRow<k, D>& m, const GlExt<D>& x) {
    GlExt<D> y = m.e[k];
#pragma unroll
    for (int s = 0; s < k; s++) y = ext_add(y, ext_mul(m.e[s], shfl_grp(gmask, x, s, cp_lanes<k>())));
    return y;
}
template <int k, int D>
__device__ __forceinline__ CRow<k, D> crow_shfl_up(const CRow<k, D>& v, u32 off) {
    CRow<k, D> r;
#pragma unroll
    for (int c = 0; c <= k; c++) r.e[c] = shfl_up_ext(v.e[c], off);
    return r;
}
__device__ __forceinline__ u32 cp_gmask(u32 K) { return ((1u << K) - 1) << ((threadIdx.x & 31) & ~(K - 1)); }

// exclusive scan of one map per lane group over the block, in group order; `total` = the whole block's composition
template <int k, int D>
__device__ __forceinline__ CRow<k, D> coupled_block_exclusive_scan(const CRow<k, D>& v, CRow<k, D>& total) {
    constexpr u32 K = cp_lanes<k>(), G = 32 / K, NW = AUX_SCAN_THREADS / 32;
    __shared__ u64 wsum[NW][K][(k + 1) * D];
    const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5, r = lane & (K - 1), g = lane / K, gm = cp_gmask(K);
    auto ld = [&](u32 w) { CRow<k, D> x; for (int c = 0; c <= k; c++) x.e[c] = ld_ext<D>(&wsum[w][r][c * D]); return x; };
    auto st = [&](u32 w, const CRow<k, D>& x) {
        for (int c = 0; c <= k; c++)
            for (int q = 0; q < D; q++) wsum[w][r][c * D + q] = x.e[c].v[q];
    };
    CRow<k, D> x = v;
#pragma unroll
    for (u32 off = 1; off < G; off <<= 1) {
        const CRow<k, D> y = crow_op(gm, crow_shfl_up(x, off * K), x);
        if (g >= off) x = y;
    }
    if (g == G - 1) st(wid, x);
    __syncthreads();
    if (wid == 0) {
        CRow<k, D> s = g < NW ? ld(g) : crow_id<k, D>(r);
#pragma unroll
        for (u32 off = 1; off < NW; off <<= 1) {
            const CRow<k, D> y = crow_op(gm, crow_shfl_up(s, off * K), s);
            if (g >= off) s = y;
        }
        if (g < NW) st(g, s);
    }
    __syncthreads();
    total = ld(NW - 1);
    const CRow<k, D> wpre = wid ? ld(wid - 1) : crow_id<k, D>(r);
    CRow<k, D> ex = crow_shfl_up(x, K);
    if (g == 0) ex = crow_id<k, D>(r);
    __syncthreads();  // wsum is free for the next call
    return crow_op(gm, wpre, ex);
}

// COUPLED_RECURRENCE: row i's map from the leader's program into terms [n][S]: OUT r = t_r, OUT 4 + 4r + c = M[r][c]; the slots
// the program never writes (bit set in `unwritten`, slot r (k + 1) + c) are 0. One row per thread.
template <int D>
__global__ void __launch_bounds__(AUX_TERM_THREADS) aux_coupled_term_kernel(AuxTermParams p, u32 k, u32 unwritten) {
    const size_t n = (size_t)1 << p.log_n;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    GlExt<D> ra[AUX_MAX_REGS];
    aux_load_regs<D>(p, i, (i + 1) & (n - 1), 2 * p.w, 2 * p.w + 2 * p.aw, ra);
    u64* t = p.terms + i * k * (k + 1) * D;
    for (u32 s = 0; s < k * (k + 1); s++)
        if (unwritten >> s & 1)
#pragma unroll
            for (int q = 0; q < D; q++) t[s * D + q] = 0;
    for (u32 j = 0; j < p.prog_len; j++) {
        const u32 op = p.prog[4 * j], dst = p.prog[4 * j + 1], a = p.prog[4 * j + 2], b = p.prog[4 * j + 3];
        switch (op) {
            case 0: ra[dst] = ext_add(ra[a], ra[b]); break;
            case 1: ra[dst] = ext_sub(ra[a], ra[b]); break;
            case 2: ra[dst] = ext_mul(ra[a], ra[b]); break;
            case 3: ra[dst] = ext_from_base<D>(p.consts[a]); break;
            default: {
                const u32 s = dst < 4 ? dst * (k + 1) + k : (dst - 4) / 4 * (k + 1) + (dst - 4) % 4;
#pragma unroll
                for (int q = 0; q < D; q++) t[s * D + q] = ra[a].v[q];
                break;
            }
        }
    }
}

// The composition of the maps of rows r0 .. r0 + cp_items - 1 (those < n), in row order; the identity when r0 >= n.
template <int k, int D>
__device__ __forceinline__ CRow<k, D> coupled_run(const u64* terms, size_t n, size_t r0, u32 r, u32 gm) {
    constexpr size_t S = k * (k + 1) * D;
    CRow<k, D> v = r0 < n ? crow_ld<k, D>(terms + r0 * S, r) : crow_id<k, D>(r);
#pragma unroll 1
    for (int j = 1; j < cp_items<k>(); j++)
        if (r0 + j < n) v = crow_op(gm, v, crow_ld<k, D>(terms + (r0 + j) * S, r));
    return v;
}

// per tile: the composition of its rows' maps into agg [ntiles][S]
template <int k, int D>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_coupled_reduce(const u64* terms, size_t n, u64* agg) {
    constexpr u32 K = cp_lanes<k>();
    const u32 r = threadIdx.x & (K - 1);
    const CRow<k, D> v = coupled_run<k, D>(terms, n, (size_t)blockIdx.x * AUX_SCAN_TILE + (size_t)(threadIdx.x / K) * cp_items<k>(), r,
                                           cp_gmask(K));
    CRow<k, D> total;
    coupled_block_exclusive_scan<k, D>(v, total);
    if (threadIdx.x < K) crow_st<k, D>(agg + (size_t)blockIdx.x * k * (k + 1) * D, r, total);
}

template <int k, int D>
struct CVec { GlExt<D> a[k]; };   // a state vector of the group: a_r = the value of column j + r

// one block; tile maps -> the state vector at each tile start (the maps of the tiles before it applied to init); a_r is written
// over the first D words of row r of the tile's slot. Each lane group owns a run of consecutive tiles.
template <int k, int D>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_coupled_carry(u64* agg, size_t ntiles, CVec<k, D> init) {
    constexpr u32 K = cp_lanes<k>();
    constexpr size_t S = k * (k + 1) * D;
    const u32 r = threadIdx.x & (K - 1), gm = cp_gmask(K);
    const size_t per = (ntiles + AUX_SCAN_THREADS / K - 1) / (AUX_SCAN_THREADS / K);
    const size_t b = (threadIdx.x / K) * per, e = b + per < ntiles ? b + per : ntiles;
    CRow<k, D> v = crow_id<k, D>(r);
#pragma unroll 1
    for (size_t i = b; i < e; i++) v = crow_op(gm, v, crow_ld<k, D>(agg + i * S, r));
    GlExt<D> x = ext_zero<D>();
#pragma unroll
    for (int s = 0; s < k; s++) if ((u32)s == r) x = init.a[s];
    CRow<k, D> total;
    x = crow_apply(gm, coupled_block_exclusive_scan<k, D>(v, total), x);
#pragma unroll 1
    for (size_t i = b; i < e; i++) {
        const CRow<k, D> a = crow_ld<k, D>(agg + i * S, r);
        if (r < (u32)k)
#pragma unroll
            for (int q = 0; q < D; q++) agg[i * S + r * (k + 1) * D + q] = x.v[q];
        x = crow_apply(gm, a, x);
    }
}

// a[i] = the maps of the tile's rows before i applied to the tile's carry-in; lane r writes aux column col + r
template <int k, int D>
__global__ void __launch_bounds__(AUX_SCAN_THREADS) aux_coupled_apply(const u64* terms, size_t n, const u64* carry, SegMatrix out, u32 col) {
    constexpr u32 K = cp_lanes<k>();
    constexpr size_t S = k * (k + 1) * D;
    const u32 r = threadIdx.x & (K - 1), gm = cp_gmask(K);
    const size_t r0 = (size_t)blockIdx.x * AUX_SCAN_TILE + (size_t)(threadIdx.x / K) * cp_items<k>();
    const CRow<k, D> v = coupled_run<k, D>(terms, n, r0, r, gm);
    CRow<k, D> total;
    const CRow<k, D> pre = coupled_block_exclusive_scan<k, D>(v, total);
    GlExt<D> x = r < (u32)k ? ld_ext<D>(carry + (size_t)blockIdx.x * S + r * (k + 1) * D) : ext_zero<D>();
    x = crow_apply(gm, pre, x);
#pragma unroll 1
    for (int j = 0; j < cp_items<k>(); j++) {
        const size_t i = r0 + j;
        if (i < n) {
            if (r < (u32)k) st_aux<D>(out, i, col + r, x);
            x = crow_apply(gm, crow_ld<k, D>(terms + i * S, r), x);
        }
    }
}

// ---- host ---------------------------------------------------------------------------------------------------------------
// Parses and checks an aux build description against the AIR's shape (w main columns, aw aux columns, np periodic columns,
// nr random elements). Returns nullptr, or the reason it is rejected.
const char* wf_aux_build_parse(const u64* d, size_t len, u32 w, u32 aw, u32 np, u32 nr, AuxBuildHost& b) {
    size_t p = 0;
    auto rd = [&](u64& v) { if (p >= len) return false; v = d[p++]; return true; };
    u64 v, cnt;
    if (!d || !rd(v)) return "malformed aux build description";
    if (v != aw) return "aux build width does not match the AIR's aux width";
    b.aw = aw;
    if (!rd(cnt) || cnt > len) return "malformed aux build description";
    for (u64 i = 0; i < cnt; i++) {
        if (!rd(v)) return "malformed aux build description";
        if (v >= GL_P) return "aux build constant is not a canonical field element";
        b.consts.push_back(v);
    }
    const u32 ab = 2 * w, pb = 2 * w + 2 * aw, first_tmp = pb + np + nr;
    // the open COUPLED_RECURRENCE group: its leader's index and the OUT slots its program writes (bit = OUT index); the group
    // size k, and with it the slots allowed, is known when the next column is not a member
    u32 lead = ~0u, lead_slots = 0;
    auto close_group = [&]() -> const char* {
        if (lead == ~0u) return nullptr;
        const u32 k = (u32)b.cols.size() - lead;
        lead = ~0u;
        if (k < 2 || k > 4) return "aux build COUPLED_RECURRENCE group has fewer than 2 or more than 4 columns";
        for (u32 s = 0; s < 20; s++)
            if ((lead_slots >> s & 1) && (s < 4 ? s >= k : (s - 4) / 4 >= k || (s - 4) % 4 >= k))
                return "aux build COUPLED_RECURRENCE OUT selects a slot outside the group's t (0 .. k-1) and M (4 + 4r + c, r, c < k)";
        return nullptr;
    };
    for (u32 j = 0; j < aw; j++) {
        AuxBuildCol c;
        if (!rd(v)) return "malformed aux build description";
        if (v > 2 && v != 4 && v != 6 && v != 8 && v != 9) return "unknown aux column kind";
        c.kind = (u32)v;
        if (c.kind != 9) {
            if (const char* why = close_group()) return why;
        } else if (lead == ~0u) {
            return "aux build COUPLED_MEMBER column does not follow a COUPLED_RECURRENCE column or another member";
        }
        for (int q = 0; q < 3; q++) {
            if (!rd(c.init[q])) return "malformed aux build description";
            if (c.init[q] >= GL_P) return "aux column init is not a canonical field element";
        }
        if (!rd(v)) return "malformed aux build description";
        if (c.kind == 9) {   // {9, init, 0, 0}: the leader's program gives the whole group's step
            if (!rd(cnt)) return "malformed aux build description";
            if (v != 0 || cnt != 0) return "aux build COUPLED_MEMBER column has registers or instructions";
            b.cols.push_back(c);
            continue;
        }
        if (v > AUX_MAX_REGS || v < first_tmp) return "aux build register count out of range";
        c.num_regs = (u32)v;
        if (!rd(cnt) || cnt > (1u << 20)) return "malformed aux build description";
        std::vector<bool> written(c.num_regs, false);
        for (u32 r = 0; r < first_tmp; r++) written[r] = !(r >= ab && r < pb) || ((r - ab) % aw) < j;
        const bool affine = c.kind == 4, moebius = c.kind == 6, coupled = c.kind == 8;
        u32 outs[4] = {0, 0, 0, 0}, slots = 0;
        for (u64 k = 0; k < cnt; k++) {
            u64 op, ds, x, y;
            if (!rd(op) || !rd(ds) || !rd(x) || !rd(y)) return "malformed aux build description";
            if (op > 4) return "unknown aux build opcode";
            auto readable = [&](u64 r) { return r < c.num_regs && written[r]; };
            if (op == 4) {
                if (coupled && ds > 19)
                    return "aux build COUPLED_RECURRENCE OUT selects a slot outside the group's t (0 .. k-1) and M (4 + 4r + c, r, c < k)";
                if (coupled && (slots >> ds & 1)) return "aux build COUPLED_RECURRENCE program writes an OUT slot more than once";
                if (moebius && ds > 3)
                    return "aux build OUT selects neither numerator (0), denominator (1), multiplier (2) nor denominator multiplier (3)";
                if (affine && ds > 2) return "aux build OUT selects neither numerator (0), denominator (1) nor multiplier (2)";
                if (!affine && !moebius && !coupled && ds > 1) return "aux build OUT selects neither numerator (0) nor denominator (1)";
                if (!readable(x)) return "aux build program reads a register out of range, an aux column >= its own, or an unwritten temporary";
                if (coupled) slots |= 1u << ds;
                else outs[ds]++;
            } else {
                if (ds >= c.num_regs || ds < first_tmp) return "aux build program writes a register outside its temporaries";
                if (op == 3) { if (x >= b.consts.size()) return "aux build constant index out of range"; }
                else if (!readable(x) || !readable(y))
                    return "aux build program reads a register out of range, an aux column >= its own, or an unwritten temporary";
                written[ds] = true;
            }
            c.prog.insert(c.prog.end(), {(u32)op, (u32)ds, (u32)x, (u32)y});
        }
        if (coupled) { lead = j; lead_slots = slots; }
        if (!coupled && outs[0] != 1) return "aux build column needs exactly one numerator (OUT 0)";
        if (outs[1] > 1) return "aux build column has more than one denominator (OUT 1)";
        if (affine && outs[2] == 0) return "aux build LINEAR_RECURRENCE column has no multiplier (OUT 2)";
        if (affine && outs[2] > 1) return "aux build LINEAR_RECURRENCE column has more than one multiplier (OUT 2)";
        if (moebius && outs[2] == 0) return "aux build RATIONAL_RECURRENCE column has no multiplier (OUT 2)";
        if (moebius && outs[2] > 1) return "aux build RATIONAL_RECURRENCE column has more than one multiplier (OUT 2)";
        if (moebius && outs[3] == 0) return "aux build RATIONAL_RECURRENCE column has no denominator multiplier (OUT 3)";
        if (moebius && outs[3] > 1) return "aux build RATIONAL_RECURRENCE column has more than one denominator multiplier (OUT 3)";
        b.cols.push_back(c);
    }
    if (const char* why = close_group()) return why;
    if (p != len) return "malformed aux build description";
    return nullptr;
}

template <int D, bool MUL>
static int aux_scan(wf_ctx* ctx, const u64* terms, size_t n, u64* agg, const u64* init, SegMatrix out, u32 col) {
    const size_t ntiles = (n + AUX_SCAN_TILE - 1) / AUX_SCAN_TILE;
    GlExt<D> in;
    for (int q = 0; q < D; q++) in.v[q] = init[q];
    aux_scan_reduce<D, MUL><<<(unsigned)ntiles, AUX_SCAN_THREADS, 0, ctx->st>>>(terms, n, agg);
    aux_scan_carry<D, MUL><<<1, AUX_SCAN_THREADS, 0, ctx->st>>>(agg, ntiles, in);
    aux_scan_apply<D, MUL><<<(unsigned)ntiles, AUX_SCAN_THREADS, 0, ctx->st>>>(terms, n, agg, out, col);
    ctx->launches += 3;
    CK(cudaGetLastError());
    return WF_OK;
}

// terms: [n][2D] (m_i, t_i); agg: [ntiles][2D]
template <int D>
static int aux_affine(wf_ctx* ctx, const u64* terms, size_t n, u64* agg, const u64* init, SegMatrix out, u32 col) {
    const size_t ntiles = (n + AUX_SCAN_TILE - 1) / AUX_SCAN_TILE;
    GlExt<D> in;
    for (int q = 0; q < D; q++) in.v[q] = init[q];
    aux_affine_reduce<D><<<(unsigned)ntiles, AUX_SCAN_THREADS, 0, ctx->st>>>(terms, n, agg);
    aux_affine_carry<D><<<1, AUX_SCAN_THREADS, 0, ctx->st>>>(agg, ntiles, in);
    aux_affine_apply<D><<<(unsigned)ntiles, AUX_SCAN_THREADS, 0, ctx->st>>>(terms, n, agg, out, col);
    ctx->launches += 3;
    CK(cudaGetLastError());
    return WF_OK;
}

// terms: [n][4D] (m_i, n_i, c_i, d_i); agg: [ntiles][4D]; zmin: one device word. The projective scan equals the serial
// definition before the first row z with y_z = 0, where the serial value is 0: rows z .. are scanned again from (0, 1) until no
// zero is left, so k such rows cost k further scans, O(k n). One host synchronisation per scan.
template <int D>
static int aux_moebius(wf_ctx* ctx, const u64* terms, size_t n, u64* agg, unsigned long long* zmin, const u64* init, SegMatrix out, u32 col) {
    GlExt<D> in;
    for (int q = 0; q < D; q++) in.v[q] = init[q];
    for (size_t base = 0;;) {
        const size_t m = n - base, ntiles = (m + AUX_SCAN_TILE - 1) / AUX_SCAN_TILE;
        const u64* t = terms + base * 4 * D;
        CK(cudaMemsetAsync(zmin, 0xff, sizeof(*zmin), ctx->st));
        aux_moebius_reduce<D><<<(unsigned)ntiles, AUX_SCAN_THREADS, 0, ctx->st>>>(t, m, agg);
        aux_moebius_carry<D><<<1, AUX_SCAN_THREADS, 0, ctx->st>>>(agg, ntiles, in);
        aux_moebius_apply<D><<<(unsigned)ntiles, AUX_SCAN_THREADS, 0, ctx->st>>>(t, m, agg, out, col, base, zmin);
        ctx->launches += 3;
        CK(cudaGetLastError());
        unsigned long long z;
        CK(cudaMemcpyAsync(&z, zmin, sizeof(z), cudaMemcpyDeviceToHost, ctx->st));
        CK(cudaStreamSynchronize(ctx->st));
        if (z >= n) return WF_OK;
        base = (size_t)z;
        in = ext_zero<D>();
    }
}

// the group of columns col .. col + k - 1; terms: [n][S] (M_i, t_i) row by row, S = k (k + 1) D; agg: [ntiles][S]
template <int k, int D>
static int aux_coupled(wf_ctx* ctx, const u64* terms, size_t n, u64* agg, const AuxBuildCol* cols, SegMatrix out, u32 col) {
    const size_t ntiles = (n + AUX_SCAN_TILE - 1) / AUX_SCAN_TILE;
    CVec<k, D> in;
    for (int r = 0; r < k; r++)
        for (int q = 0; q < D; q++) in.a[r].v[q] = cols[r].init[q];
    aux_coupled_reduce<k, D><<<(unsigned)ntiles, AUX_SCAN_THREADS, 0, ctx->st>>>(terms, n, agg);
    aux_coupled_carry<k, D><<<1, AUX_SCAN_THREADS, 0, ctx->st>>>(agg, ntiles, in);
    aux_coupled_apply<k, D><<<(unsigned)ntiles, AUX_SCAN_THREADS, 0, ctx->st>>>(terms, n, agg, out, col);
    ctx->launches += 3;
    CK(cudaGetLastError());
    return WF_OK;
}

// the size of the COUPLED_RECURRENCE group led by column j: 1 + the COUPLED_MEMBER columns after it
static u32 coupled_size(const AuxBuildHost& b, u32 j) {
    u32 k = 1;
    while (j + k < b.cols.size() && b.cols[j + k].kind == 9) k++;
    return k;
}

template <int D>
static int aux_build_d(wf_ctx* ctx, const AuxBuildHost& b, const wf_mat* main, u32 w, const std::vector<std::vector<u64>>& periodic,
                       const u64* rnd, u32 nr, wf_mat** out) {
    const size_t n = main->m.rows;
    const u32 log_n = log2_ceil(n);
    const u32 np = (u32)periodic.size();
    // one upload: constants | random elements | periodic tables | programs (u32 pairs) -- pageable, staged before return
    std::vector<u64> up(b.consts);
    const size_t o_rnd = up.size();
    up.insert(up.end(), rnd, rnd + (size_t)nr * D);
    const size_t o_per = up.size();
    std::vector<u32> poff, plen;
    for (auto& c : periodic) { poff.push_back((u32)(up.size() - o_per)); plen.push_back((u32)c.size()); up.insert(up.end(), c.begin(), c.end()); }
    std::vector<u32> u32s(poff);
    u32s.insert(u32s.end(), plen.begin(), plen.end());
    std::vector<size_t> prog_off;
    for (auto& c : b.cols) { prog_off.push_back(u32s.size()); u32s.insert(u32s.end(), c.prog.begin(), c.prog.end()); }
    if (u32s.size() & 1) u32s.push_back(0);
    const size_t o_u32 = up.size();
    for (size_t i = 0; i < u32s.size(); i += 2) up.push_back((u64)u32s[i] | ((u64)u32s[i + 1] << 32));
    bool running = false, affine = false, moebius = false;
    u32 kmax = 0;
    for (u32 j = 0; j < b.aw; j++) {
        const u32 kind = b.cols[j].kind;
        running = running || kind != 0; affine = affine || kind == 4; moebius = moebius || kind == 6;
        if (kind == 8) kmax = std::max(kmax, coupled_size(b, j));
    }
    // words per row of the term buffer: (m_i, n_i, c_i, d_i) or (m_i, t_i) when a column needs them, the largest group's
    // (M_i, t_i) when there is a group
    const size_t tw = std::max((size_t)kmax * (kmax + 1) * D, (size_t)(moebius ? 4 * D : affine ? 2 * D : D));
    DevScratch tmp(ctx);
    void *d_up, *d_terms = nullptr, *d_agg = nullptr, *d_zmin = nullptr;
    CKI(tmp.alloc(std::max(up.size(), (size_t)1) * 8, &d_up));
    if (running) {
        CKI(tmp.alloc(n * tw * 8, &d_terms));
        CKI(tmp.alloc((n + AUX_SCAN_TILE - 1) / AUX_SCAN_TILE * tw * 8, &d_agg));
    }
    if (moebius) CKI(tmp.alloc(8, &d_zmin));
    CK(cudaMemcpyAsync(d_up, up.data(), up.size() * 8, cudaMemcpyHostToDevice, ctx->st));
    wf_mat* a;
    CKI(wf_mat_alloc(ctx, n, b.aw * D, &a));
    const u64* dev = (const u64*)d_up;
    const u32* dev32 = (const u32*)(dev + o_u32);
    AuxTermParams p{};
    p.main = main->m; p.aux = a->m;
    p.w = w; p.aw = b.aw; p.np = np; p.nr = nr; p.log_n = log_n;
    p.consts = dev; p.rnd = dev + o_rnd; p.ptab = dev + o_per; p.ptab_off = dev32; p.ptab_len = dev32 + np;
    const unsigned grid = (unsigned)((n / AUX_TERM_ROWS + AUX_TERM_THREADS - 1) / AUX_TERM_THREADS);
    int r = WF_OK;
    for (u32 j = 0; j < b.aw && r == WF_OK; j++) {
        const AuxBuildCol& c = b.cols[j];
        if (c.kind == 9) continue;   // built with its group's leader
        p.col = j;
        p.prog = dev32 + prog_off[j];
        p.prog_len = (u32)(c.prog.size() / 4);
        p.terms = c.kind ? (u64*)d_terms : nullptr;
        const u32 k = c.kind == 8 ? coupled_size(b, j) : 0;
        if (c.kind == 8) {
            u32 written = 0;
            for (size_t q = 0; q < c.prog.size(); q += 4)
                if (c.prog[q] == 4) {
                    const u32 ds = c.prog[q + 1];
                    written |= 1u << (ds < 4 ? ds * (k + 1) + k : (ds - 4) / 4 * (k + 1) + (ds - 4) % 4);
                }
            aux_coupled_term_kernel<D><<<(unsigned)((n + AUX_TERM_THREADS - 1) / AUX_TERM_THREADS), AUX_TERM_THREADS, 0, ctx->st>>>(
                p, k, ((1u << k * (k + 1)) - 1) & ~written);
        } else if (c.kind == 6) aux_moebius_term_kernel<D><<<(unsigned)((n + AUX_TERM_THREADS - 1) / AUX_TERM_THREADS), AUX_TERM_THREADS, 0, ctx->st>>>(p);
        else if (c.kind == 4) aux_term_kernel<D, true><<<grid, AUX_TERM_THREADS, 0, ctx->st>>>(p);
        else aux_term_kernel<D, false><<<grid, AUX_TERM_THREADS, 0, ctx->st>>>(p);
        ctx->launches++;
        if (cudaGetLastError() != cudaSuccess) { r = wf_fail(ctx, WF_ERR_CUDA, "aux_term_kernel launch failed"); break; }
        if (c.kind == 1) r = aux_scan<D, true>(ctx, (const u64*)d_terms, n, (u64*)d_agg, c.init, a->m, j);
        else if (c.kind == 2) r = aux_scan<D, false>(ctx, (const u64*)d_terms, n, (u64*)d_agg, c.init, a->m, j);
        else if (c.kind == 4) r = aux_affine<D>(ctx, (const u64*)d_terms, n, (u64*)d_agg, c.init, a->m, j);
        else if (c.kind == 6) r = aux_moebius<D>(ctx, (const u64*)d_terms, n, (u64*)d_agg, (unsigned long long*)d_zmin, c.init, a->m, j);
        else if (c.kind == 8) {
            const u64* t = (const u64*)d_terms;
            u64* g = (u64*)d_agg;
            r = k == 2 ? aux_coupled<2, D>(ctx, t, n, g, &c, a->m, j)
              : k == 3 ? aux_coupled<3, D>(ctx, t, n, g, &c, a->m, j)
                       : aux_coupled<4, D>(ctx, t, n, g, &c, a->m, j);
        }
    }
    if (r != WF_OK) { wf_mat_free(ctx, a); return r; }
    *out = a;
    return WF_OK;
}

int wf_aux_build_run(wf_ctx* ctx, const AuxBuildHost& b, const wf_mat* main, u32 w, const std::vector<std::vector<u64>>& periodic,
                     const u64* rnd, u32 nr, int D, wf_mat** out) {
    const size_t n = main->m.rows;
    if (n < 8 || (n & (n - 1)) || main->m.cols != w) return wf_fail(ctx, WF_ERR_INVALID, "main trace shape does not match the AIR (n x width, n a power of two >= 8)");
    for (auto& c : periodic) if (c.size() > n) return wf_fail(ctx, WF_ERR_INVALID, "periodic column longer than the trace");
    for (auto& c : b.cols)
        for (int q = D; q < 3; q++) if (c.init[q]) return wf_fail(ctx, WF_ERR_INVALID, "aux column init has non-zero words beyond the extension degree");
    for (size_t i = 0; i < (size_t)nr * D; i++) if (rnd[i] >= GL_P) return wf_fail(ctx, WF_ERR_INVALID, "random element is not a canonical field element");
    switch (D) {
        case 1: return aux_build_d<1>(ctx, b, main, w, periodic, rnd, nr, out);
        case 2: return aux_build_d<2>(ctx, b, main, w, periodic, rnd, nr, out);
        case 3: return aux_build_d<3>(ctx, b, main, w, periodic, rnd, nr, out);
    }
    return wf_fail(ctx, WF_ERR_INVALID, "field extension %d", D);
}
