// commit.cuh — segment-layout matrix descriptor + row hashing / Merkle entry points (commit.cu).
#pragma once
#ifndef __CUDACC_RTC__
#include <cuda_runtime.h>
#endif

#include "gl64.cuh"

#define WF_HASH_BLAKE3_256 0
#define WF_HASH_RP64_256 1
#define WF_HASH_RPJIVE64_256 2
#define WF_HASH_BLAKE3_192 3
#define WF_HASH_SHA3_256 4
#define WF_HASH_IS_KNOWN(h) ((h) >= 0 && (h) <= 4)
#define WF_HASH_IS_BLAKE3(h) ((h) == WF_HASH_BLAKE3_256 || (h) == WF_HASH_BLAKE3_192)
// digests occupy 32-byte slots everywhere; Blake3_192 (crypto/src/hash/blake/mod.rs:73-123) keeps and serializes the first 24
// bytes (the rest of the slot is zero, as ByteDigest::as_bytes pads it)
#define WF_DIGEST_BYTES(h) ((h) == WF_HASH_BLAKE3_192 ? 24 : 32)
#define WF_DIGEST_WORDS32(h) ((h) == WF_HASH_BLAKE3_192 ? 6 : 8)

// rows x cols base-field matrix in segment layout (see ntt.cuh):
// elem(row, col) = base[(col / W) * seg_stride + row * W + col % W]
struct SegMatrix {
    u64* base;
    size_t rows;
    u32 cols;
    int W;
    size_t seg_stride;  // words; >= rows * W
    u32 nseg() const { return (cols + W - 1) / W; }
    size_t words() const { return (size_t)nseg() * seg_stride; }
};

#ifndef __CUDACC_RTC__
static inline int seg_width_for(u32 cols) { return cols >= 8 ? 8 : cols > 2 ? 4 : cols == 2 ? 2 : 1; }

// digests: rows x 4 words (32 bytes each)
// partition_size (base columns) = 0 or >= cols: whole-row hashing; else row digest = merge_many of chunk digests
cudaError_t commit_hash_rows(int hash_id, const SegMatrix& m, u64* digests, cudaStream_t st, u32 partition_size = 0);
// nodes: nleaves x 4 words; nodes[0] = 0, nodes[1] = root
cudaError_t commit_merkle_nodes(int hash_id, const u64* leaves, size_t nleaves, u64* nodes, cudaStream_t st);
// one level of merges over a digest arena (4 words per slot): arena[z] = merge(arena[x], arena[y]) for each op (x, y, z)
cudaError_t commit_merge_ops(int hash_id, u64* arena, const uint3* ops, u32 count, cudaStream_t st);
#endif  // !__CUDACC_RTC__
