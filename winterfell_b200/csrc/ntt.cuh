// ntt.cuh — batched Goldilocks NTT / iNTT / coset-LDE passes for sm_90a.
//
// Replaces the reference's CPU loops K1/K2/K6/K7/K10 (SURVEY.md §2.1): fft_in_place
// (math/src/fft/fft_inputs.rs:215-252), interpolate_poly / evaluate_poly_with_offset
// (math/src/fft/serial.rs:29-101), ColMatrix::interpolate_columns (prover/src/matrix/col_matrix.rs:192)
// and RowMatrix::evaluate_polys_over + Segment::new_with_buffer (row_matrix.rs:84, segments.rs:96-158).
// Exact arithmetic mod p: any schedule computing the same DFT gives identical canonical words
// (SURVEY.md A.4), so the schedule here is GPU-shaped, not the reference's radix-2 recursion.
//
// DATA LAYOUT ("segment layout", cf. the reference's own 8-column Segment): a matrix of `rows` x
// `cols` base-field columns is stored as G = ceil(cols/W) segments, segment g holding columns
// [gW, gW+W) row-major: elem(row, col) = base[g * seg_stride + row * W + (col % W)], W in {1,2,4,8}.
// A row of a segment is W*8 <= 64 contiguous bytes, so every pass below moves 64-byte pieces
// (8 lanes x u64) and a warp always touches whole 32-byte sectors.
//
// SCHEDULE: a transform of n = R*C points is two passes (four-step, natural order in and out):
//   pass 1 (STRIDED): for each tile column m2: Y[j1][m2] = tw(j1, m2) * sum_m1 x[C m1 + m2] w_R^(j1 m1)
//   pass 2 (CONTIG) : for each j1:            X[j1 + R j2] = sum_m2 Y[j1][m2] w_C^(j2 m2)
// n <= 2^11 runs as one CONTIG pass with R = 1. Each block owns a tile of S x 8 words in shared
// memory (S = sub-transform size, 8 lanes = T tile columns x W segment columns, T = 8/W) and runs
// the S-point DFT as radix-8 rounds held in registers: inside a round the twiddles are powers of
// two (w_8 = 2^24, w_4 = 2^48 in this field), so only the 7 inter-round twiddles per 8 points need
// the 64x64 multiplier. The sub-transform twiddle table (w_S^i, i < S/2) is staged into shared
// memory by one TMA bulk copy (cp.async.bulk ... mbarrier::complete_tx).
// Inverse transforms reuse the forward network: iDFT[j] = DFT[(S - j) mod S], applied as an index
// map when the tile is written back.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gl64.cuh"

#define NTT_LANES 8
#ifndef NTT_THREADS
#define NTT_THREADS 512
#endif
#ifndef NTT_LD_BATCH
#define NTT_LD_BATCH 8
#endif
#ifndef NTT_MIN_BLOCKS
#define NTT_MIN_BLOCKS 2
#endif
#define NTT_MAX_LOGS 11

struct NttPassParams {
    const u64* in;
    u64* out;
    size_t in_seg_stride, out_seg_stride;      // words between consecutive segments
    size_t in_batch_stride, out_batch_stride;  // words between batch items (cosets); 0 = shared
    int W;                                     // segment width (1, 2, 4 or 8)
    int logS;                                  // sub-transform size of this pass
    u32 logR, logC;                            // n = R * C
    int inverse;                               // 1: inverse sub-transform (index-reversed output)
    // CONTIG output row mapping: out_row = row * out_row_mul + batch * out_row_add
    u32 out_row_mul, out_row_add;
    // y_in_out = 1 (two-pass LDE): the intermediate Y[j1][m2] of the four-step schedule lives in the output matrix, in the
    // row that X[j1 + R m2] will occupy, (j1 + R m2) * out_row_mul + batch * out_row_add at out_col0 of the out_W-wide rows.
    // The STRIDED pass writes it there and the CONTIG pass reads it from there (in == out: in place; every block reads
    // exactly the rows and lanes it writes). The batch index is then blockIdx.x, so that the cosets of one tile run side
    // by side: the STRIDED pass reads each input tile from HBM once and every 512-byte group of output rows is written
    // while it is in L2. ntt2 kernels only.
    int y_in_out;
    // CONTIG output segment geometry: the output matrix may be wider than the input segment (a column
    // chunk of W columns lands at column offset out_col0 of an out_W-wide segment row)
    u32 out_W, out_col0;
    const u64* sub_tw;                         // w_S^i, i < S/2 (forward root)
    const u64* pre_tab;                        // optional [batch][S] input scale, indexed by sub-transform input index
    size_t pre_batch_stride;
    // optional post twiddle (STRIDED): tw(j, col) = w_M^(+-(j*a_mul*col + (batch0+batch)*b_mul*col)) * ctab[col] * cconst
    int has_post;
    const u64* master;                         // w_M^i, i < M/2
    u32 logM;
    u32 a_mul, b_mul;
    u32 batch0;                                // added to the batch index in the twiddle exponent
    // ntt2 kernels (logS >= 6) read w_M^e as tw_hi[e >> tw_split] * tw_lo[e & (2^tw_split - 1)]: two tables of
    // 2^(logM - tw_split) and 2^tw_split entries instead of a gather over M/2 entries
    const u64 *tw_hi, *tw_lo;
    u32 tw_split;
    int vec_in, vec_out;                       // lane pairs are contiguous (16-byte aligned) in the input / output
    const u64* ctab;                           // optional per-column constant table
    u64 cconst;                                // constant factor (e.g. 1/n) folded into the post twiddle, or applied
                                               // alone at write-back when has_post == 0; 1 if unused
};

enum { NTT_STRIDED = 0, NTT_CONTIG = 1 };

size_t ntt_pass_smem_bytes(const NttPassParams& p);
// small sub-transforms (logS < NTT2_MIN_LOGS): generic kernel of ntt.cu; sub_tw = half table w_S^i, master = half table w_M^i
cudaError_t ntt_launch_pass(int mode, const NttPassParams& p, u32 n_segments, u32 n_batch, cudaStream_t st);
// sub-transforms of 2^6 .. 2^11 points (ntt2.cu): sub_tw = the plan's round-twiddle table (ntt2_build_tw), post
// twiddles through tw_hi / tw_lo
#define NTT2_MIN_LOGS 6
cudaError_t ntt2_launch_pass(int mode, const NttPassParams& p, u32 n_segments, u32 n_batch, cudaStream_t st);
size_t ntt2_tw_entries(int logS);
cudaError_t ntt2_build_tw(int logS, u64* d_out, cudaStream_t st);
