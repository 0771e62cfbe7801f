// commit.cu — row hashing and Merkle tree construction on device (K3 / K4 in SURVEY.md §2.1).
//
// Replaces RowMatrix::commit_to_rows (prover/src/matrix/row_matrix.rs:184-228): digest_i =
// H::hash_elements(row_i) over the first `cols` base elements of row i, as canonical LE bytes for
// Blake3_256 (crypto/src/hash/blake/mod.rs:52-65) or as a sponge for Rp64_256
// (crypto/src/hash/rescue/rp64_256/mod.rs:224-257); and MerkleTree::new / build_merkle_nodes
// (crypto/src/merkle/mod.rs:116-135, :344-368): nodes[n/2 + i] = merge(leaf 2i, leaf 2i+1),
// nodes[i] = merge(nodes[2i], nodes[2i+1]), nodes[1] = root, nodes[0] = zeros.
//
// One hash per thread: BLAKE3's 7 rounds run entirely in registers (blake3.cuh); a warp of 32 rows
// reads 32 consecutive 64-byte segment rows = 2 KB contiguous per segment.
#include "commit.cuh"

#include "blake3.cuh"
#include "alg_hash.cuh"

// ---- row access in segment layout -----------------------------------------------------------
struct RowSrc {
    const u64* base;
    size_t seg_stride;
    int W, logW;
    u32 cols;
};
__device__ __forceinline__ u64 row_elem(const RowSrc& m, size_t row, u32 e) {
    return m.base[(size_t)(e >> m.logW) * m.seg_stride + row * m.W + (e & (m.W - 1))];
}

// BLAKE3 of `cols` elements (cols*8 bytes) of one row. Handles any length: chunks of 1024 bytes
// (128 elements) merged through a small chaining-value stack.
__device__ void blake3_row(const RowSrc& m, size_t row, u32 out[8], u32 first = 0, u32 count = 0xffffffffu) {
    const u32 cols = min(count, m.cols - first);
    const u32 nchunks = cols <= 128 ? 1 : (cols + 127) / 128;
    u32 stack[5][8];
    int sp = 0;
    u32 cv[8];
    for (u32 c = 0; c < nchunks; c++) {
        u32 e0 = c * 128, e1 = min(cols, e0 + 128);
        u32 nblk = e1 == e0 ? 1 : (e1 - e0 + 7) / 8;
        b3_iv(cv);
        for (u32 b = 0; b < nblk; b++) {
            u32 msg[16];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                u32 e = e0 + b * 8 + k;
                u64 v = e < e1 ? row_elem(m, row, first + e) : 0;
                msg[2 * k] = (u32)v;
                msg[2 * k + 1] = (u32)(v >> 32);
            }
            u32 bl = min(64u, (e1 - e0 - b * 8) * 8);
            u32 fl = (b == 0 ? B3_CHUNK_START : 0) |
                     (b == nblk - 1 ? (B3_CHUNK_END | (nchunks == 1 ? B3_ROOT : 0)) : 0);
            b3_compress(cv, msg, c, bl, fl, b3_runtime_one());
        }
        if (c == nchunks - 1) break;
        u32 total = c + 1;
        while ((total & 1) == 0) {
            u32 msg[16];
            --sp;
#pragma unroll
            for (int k = 0; k < 8; k++) { msg[k] = stack[sp][k]; msg[8 + k] = cv[k]; }
            b3_iv(cv);
            b3_compress(cv, msg, 0, 64, B3_PARENT);
            total >>= 1;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) stack[sp][k] = cv[k];
        sp++;
    }
    while (sp > 0) {
        u32 msg[16];
        --sp;
#pragma unroll
        for (int k = 0; k < 8; k++) { msg[k] = stack[sp][k]; msg[8 + k] = cv[k]; }
        b3_iv(cv);
        b3_compress(cv, msg, 0, 64, B3_PARENT | (sp == 0 ? B3_ROOT : 0));
    }
#pragma unroll
    for (int k = 0; k < 8; k++) out[k] = cv[k];
}

// fast path: one 8-column segment row == exactly one 64-byte BLAKE3 block
__global__ void __launch_bounds__(256) hash_rows_blake3_w8c8_kernel(const u64* __restrict__ base, size_t nrows,
                                                                    uint4* __restrict__ digests, u32 dw /*digest words kept: 8 | 6*/) {
    size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    const uint4* src = reinterpret_cast<const uint4*>(base + row * 8);
    u32 msg[16];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        uint4 v = __ldg(src + k);
        msg[4 * k] = v.x; msg[4 * k + 1] = v.y; msg[4 * k + 2] = v.z; msg[4 * k + 3] = v.w;
    }
    u32 cv[8];
    b3_hash64(msg, cv, b3_runtime_one());
    if (dw == 6) { cv[6] = 0; cv[7] = 0; }   // Blake3_192: ByteDigest<24>
    digests[2 * row] = make_uint4(cv[0], cv[1], cv[2], cv[3]);
    digests[2 * row + 1] = make_uint4(cv[4], cv[5], cv[6], cv[7]);
}

// rows of whole 8-column segments, at most one BLAKE3 chunk (<= 128 columns): segment g of the row IS message block g (64 bytes,
// four 16-byte loads), chained through the chaining value; the next block's loads are issued before the current compression
__global__ void __launch_bounds__(256) hash_rows_blake3_w8_kernel(const u64* __restrict__ base, size_t seg_stride, u32 nseg, size_t nrows,
                                                                  uint4* __restrict__ digests, u32 dw) {
    size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    const u32 one = b3_runtime_one();
    u32 cv[8];
    b3_iv(cv);
    uint4 nx[4];
    {
        const uint4* src = reinterpret_cast<const uint4*>(base + row * 8);
#pragma unroll
        for (int k = 0; k < 4; k++) nx[k] = __ldg(src + k);
    }
    for (u32 g = 0; g < nseg; g++) {
        u32 msg[16];
#pragma unroll
        for (int k = 0; k < 4; k++) { msg[4 * k] = nx[k].x; msg[4 * k + 1] = nx[k].y; msg[4 * k + 2] = nx[k].z; msg[4 * k + 3] = nx[k].w; }
        if (g + 1 < nseg) {
            const uint4* src = reinterpret_cast<const uint4*>(base + (size_t)(g + 1) * seg_stride + row * 8);
#pragma unroll
            for (int k = 0; k < 4; k++) nx[k] = __ldg(src + k);
        }
        const u32 fl = (g == 0 ? B3_CHUNK_START : 0) | (g == nseg - 1 ? (B3_CHUNK_END | B3_ROOT) : 0);
        b3_compress(cv, msg, 0, 64, fl, one);
    }
    if (dw == 6) { cv[6] = 0; cv[7] = 0; }
    digests[2 * row] = make_uint4(cv[0], cv[1], cv[2], cv[3]);
    digests[2 * row + 1] = make_uint4(cv[4], cv[5], cv[6], cv[7]);
}

__global__ void __launch_bounds__(256) hash_rows_blake3_kernel(RowSrc m, size_t nrows, uint4* __restrict__ digests, u32 dw) {
    size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    u32 cv[8];
    blake3_row(m, row, cv);
    if (dw == 6) { cv[6] = 0; cv[7] = 0; }
    digests[2 * row] = make_uint4(cv[0], cv[1], cv[2], cv[3]);
    digests[2 * row + 1] = make_uint4(cv[4], cv[5], cv[6], cv[7]);
}

template <int HASH>
__global__ void __launch_bounds__(128) hash_rows_alg_kernel(RowSrc m, size_t nrows, u64* __restrict__ digests) {
    size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    AlgSponge<HASH> sp;  // rp64_256/mod.rs:237-246, rp64_256_jive/mod.rs:240-282
    sp.init(m.cols);
    for (u32 e = 0; e < m.cols; e++) sp.absorb(row_elem(m, row, e));
    u64 o[4];
    sp.finish(o);
#pragma unroll
    for (int k = 0; k < 4; k++) digests[row * 4 + k] = o[k];
}

// Partitioned row hashing (row_matrix.rs:204-223, PartitionOptions air/src/options.rs:405-445):
// digest = merge_many(hash_elements(chunk_0), hash_elements(chunk_1), ...), chunks of `psize` base
// columns. merge_many = BLAKE3 of the concatenated digests (blake/mod.rs:37) or the Rp64 sponge over
// their elements (rp64_256/mod.rs:194).
template <int HASH>
__device__ __forceinline__ void partitioned_alg_row(const RowSrc& m, size_t row, u32 psize, u32 np, u64* __restrict__ digests) {
    AlgSponge<HASH> outer;  // merge_many = hash_elements over the np * 4 digest elements
    outer.init((size_t)np * 4);
    for (u32 j = 0; j < np; j++) {
        const u32 e0 = j * psize, e1 = min(m.cols, e0 + psize);
        AlgSponge<HASH> sp;
        sp.init(e1 - e0);
        for (u32 e = e0; e < e1; e++) sp.absorb(row_elem(m, row, e));
        u64 d[4];
        sp.finish(d);
#pragma unroll
        for (int k = 0; k < 4; k++) outer.absorb(d[k]);
    }
    u64 o[4];
    outer.finish(o);
#pragma unroll
    for (int k = 0; k < 4; k++) digests[row * 4 + k] = o[k];
}
__global__ void __launch_bounds__(128) hash_rows_partitioned_kernel(int hash_id, RowSrc m, size_t nrows, u32 psize,
                                                                    u64* __restrict__ digests) {
    size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    const u32 np = (m.cols + psize - 1) / psize;  // <= 16
    if (WF_HASH_IS_BLAKE3(hash_id)) {
        const u32 dw = WF_DIGEST_WORDS32(hash_id);
        u32 parts[16][8];
        for (u32 j = 0; j < np; j++) blake3_row(m, row, parts[j], j * psize, psize);
        // merge_many = BLAKE3 of the np digests back to back, dw words each (<= 512 bytes: one chunk)
        u32 cv[8];
        b3_iv(cv);
        const u32 total = np * dw, nblk = (total + 15) / 16;
        for (u32 b = 0; b < nblk; b++) {
            u32 msg[16];
#pragma unroll
            for (int k = 0; k < 16; k++) {
                const u32 t = b * 16 + k;
                msg[k] = t < total ? parts[t / dw][t % dw] : 0;
            }
            u32 bl = min(64u, (total - b * 16) * 4);
            u32 fl = (b == 0 ? B3_CHUNK_START : 0) | (b == nblk - 1 ? (B3_CHUNK_END | B3_ROOT) : 0);
            b3_compress(cv, msg, 0, bl, fl, b3_runtime_one());
        }
        if (dw == 6) { cv[6] = 0; cv[7] = 0; }
#pragma unroll
        for (int k = 0; k < 4; k++) digests[row * 4 + k] = (u64)cv[2 * k] | ((u64)cv[2 * k + 1] << 32);
    } else if (hash_id == WF_HASH_RP64_256) {
        partitioned_alg_row<WF_HASH_RP64_256>(m, row, psize, np, digests);
    } else if (hash_id == WF_HASH_SHA3_256) {
        partitioned_alg_row<WF_HASH_SHA3_256>(m, row, psize, np, digests);
    } else {
        partitioned_alg_row<WF_HASH_RPJIVE64_256>(m, row, psize, np, digests);
    }
}

// ---- Merkle levels ----------------------------------------------------------------------------
template <int DW>
__global__ void __launch_bounds__(256) merkle_level_blake3_kernel(const uint4* __restrict__ in, uint4* __restrict__ out,
                                                                  size_t count) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    u32 w[16];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        uint4 v = __ldg(in + 4 * i + k);
        w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
    }
    u32 cv[8];
    if (DW == 8) b3_hash64(w, cv, b3_runtime_one());
    else b3_merge_words<DW>(w, w + 8, cv, b3_runtime_one());
    out[2 * i] = make_uint4(cv[0], cv[1], cv[2], cv[3]);
    out[2 * i + 1] = make_uint4(cv[4], cv[5], cv[6], cv[7]);
}
template <int HASH>
__global__ void __launch_bounds__(128) merkle_level_alg_kernel(const u64* __restrict__ in, u64* __restrict__ out, size_t count) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    u64 v[8], o[4];
#pragma unroll
    for (int k = 0; k < 8; k++) v[k] = in[8 * i + k];
    alg_merge<HASH>(v, o);
#pragma unroll
    for (int k = 0; k < 4; k++) out[4 * i + k] = o[k];
}

// Up to 9 tree levels per launch: block b turns 512 consecutive child digests into their 256 parents
// and keeps reducing in shared memory down to the single ancestor of the block; every level is written
// to its heap position (nodes[m + ...], crypto/src/merkle/mod.rs:344-368). `m` = number of nodes on
// the first level computed (children = `src`, 2m digests); levels stop at `m_stop` (inclusive).
template <int HASH>
__device__ __forceinline__ void merge_digests(const u64* a /*8 words: two digests*/, u64* out /*4 words*/) {
    if (WF_HASH_IS_BLAKE3(HASH)) {
        u32 msg[16], cv[8];
#pragma unroll
        for (int k = 0; k < 8; k++) { msg[2 * k] = (u32)a[k]; msg[2 * k + 1] = (u32)(a[k] >> 32); }
        if (HASH == WF_HASH_BLAKE3_256) b3_hash64(msg, cv, b3_runtime_one());
        else b3_merge_words<6>(msg, msg + 8, cv, b3_runtime_one());
#pragma unroll
        for (int k = 0; k < 4; k++) out[k] = (u64)cv[2 * k] | ((u64)cv[2 * k + 1] << 32);
    } else {
        alg_merge<HASH>(a, out);
    }
}
template <int HASH>
__global__ void __launch_bounds__(256) merkle_subtree_kernel(const u64* __restrict__ src, u64* __restrict__ nodes, size_t m) {
    __shared__ u64 lvl[256][4];
    const u32 t = threadIdx.x;
    const size_t b = blockIdx.x;
    size_t i = b * 256 + t;  // parent index within the level
    if (i < m) {
        u64 in[8], o[4];
        const ulonglong2* p = reinterpret_cast<const ulonglong2*>(src + i * 8);
#pragma unroll
        for (int k = 0; k < 4; k++) { ulonglong2 v = __ldg(p + k); in[2 * k] = v.x; in[2 * k + 1] = v.y; }
        merge_digests<HASH>(in, o);
#pragma unroll
        for (int k = 0; k < 4; k++) { lvl[t][k] = o[k]; nodes[(m + i) * 4 + k] = o[k]; }
    }
    // further levels inside the block: level size (per block) 128, 64, ..., 1
    size_t level_m = m;
    for (u32 width = 128; width >= 1; width >>= 1) {
        level_m >>= 1;
        if (level_m == 0) break;
        __syncthreads();
        u64 in[8], o[4];
        const bool active = t < width && (b * width + t) < level_m;
        if (active) {
#pragma unroll
            for (int k = 0; k < 4; k++) { in[k] = lvl[2 * t][k]; in[4 + k] = lvl[2 * t + 1][k]; }
            merge_digests<HASH>(in, o);
        }
        __syncthreads();
        if (active) {
#pragma unroll
            for (int k = 0; k < 4; k++) { lvl[t][k] = o[k]; nodes[(level_m + b * width + t) * 4 + k] = o[k]; }
        }
    }
    if (m <= 256 && b == 0 && t < 4) nodes[t] = 0;  // nodes[0] = default digest (merkle/mod.rs:349); set by the last launch
}

// One level of many batch Merkle openings (BatchMerkleProof::get_root, crypto/src/merkle/proofs.rs:110-205) over one digest
// arena: op i merges arena[ops[i].x] and arena[ops[i].y] into arena[ops[i].z]
template <int HASH>
__global__ void __launch_bounds__(128) merkle_merge_ops_kernel(u64* __restrict__ arena, const uint3* __restrict__ ops, u32 count) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint3 op = ops[i];
    u64 in[8], o[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { in[k] = arena[(size_t)op.x * 4 + k]; in[4 + k] = arena[(size_t)op.y * 4 + k]; }
    merge_digests<HASH>(in, o);
#pragma unroll
    for (int k = 0; k < 4; k++) arena[(size_t)op.z * 4 + k] = o[k];
}

cudaError_t commit_merge_ops(int hash_id, u64* arena, const uint3* ops, u32 count, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    const unsigned blocks = (count + 127) / 128;
    if (hash_id == WF_HASH_BLAKE3_256) merkle_merge_ops_kernel<WF_HASH_BLAKE3_256><<<blocks, 128, 0, st>>>(arena, ops, count);
    else if (hash_id == WF_HASH_BLAKE3_192) merkle_merge_ops_kernel<WF_HASH_BLAKE3_192><<<blocks, 128, 0, st>>>(arena, ops, count);
    else if (hash_id == WF_HASH_RP64_256) merkle_merge_ops_kernel<WF_HASH_RP64_256><<<blocks, 128, 0, st>>>(arena, ops, count);
    else if (hash_id == WF_HASH_SHA3_256) merkle_merge_ops_kernel<WF_HASH_SHA3_256><<<blocks, 128, 0, st>>>(arena, ops, count);
    else merkle_merge_ops_kernel<WF_HASH_RPJIVE64_256><<<blocks, 128, 0, st>>>(arena, ops, count);
    return cudaGetLastError();
}

cudaError_t commit_hash_rows(int hash_id, const SegMatrix& m, u64* digests, cudaStream_t st, u32 partition_size) {
    if (m.rows == 0) return cudaSuccess;
    RowSrc src;
    src.base = m.base; src.seg_stride = m.seg_stride; src.W = m.W; src.cols = m.cols;
    src.logW = m.W == 8 ? 3 : m.W == 4 ? 2 : m.W == 2 ? 1 : 0;
    if (partition_size != 0 && partition_size != m.cols) {  // > cols: one partition, still merge_many (row_matrix.rs:204-223)
        if ((m.cols + partition_size - 1) / partition_size > 16) return cudaErrorInvalidValue;
        hash_rows_partitioned_kernel<<<(unsigned)((m.rows + 127) / 128), 128, 0, st>>>(hash_id, src, m.rows, partition_size, digests);
        return cudaGetLastError();
    }
    if (WF_HASH_IS_BLAKE3(hash_id)) {
        unsigned blocks = (unsigned)((m.rows + 255) / 256);
        const u32 dw = WF_DIGEST_WORDS32(hash_id);
        if (m.W == 8 && m.cols == 8)
            hash_rows_blake3_w8c8_kernel<<<blocks, 256, 0, st>>>(m.base, m.rows, reinterpret_cast<uint4*>(digests), dw);
        else if (m.W == 8 && m.cols % 8 == 0 && m.cols <= 128)
            hash_rows_blake3_w8_kernel<<<blocks, 256, 0, st>>>(m.base, m.seg_stride, m.cols / 8, m.rows, reinterpret_cast<uint4*>(digests), dw);
        else
            hash_rows_blake3_kernel<<<blocks, 256, 0, st>>>(src, m.rows, reinterpret_cast<uint4*>(digests), dw);
    } else {
        unsigned blocks = (unsigned)((m.rows + 127) / 128);
        if (hash_id == WF_HASH_RP64_256) hash_rows_alg_kernel<WF_HASH_RP64_256><<<blocks, 128, 0, st>>>(src, m.rows, digests);
        else if (hash_id == WF_HASH_SHA3_256) hash_rows_alg_kernel<WF_HASH_SHA3_256><<<blocks, 128, 0, st>>>(src, m.rows, digests);
        else hash_rows_alg_kernel<WF_HASH_RPJIVE64_256><<<blocks, 128, 0, st>>>(src, m.rows, digests);
    }
    return cudaGetLastError();
}

cudaError_t commit_merkle_nodes(int hash_id, const u64* leaves, size_t nleaves, u64* nodes, cudaStream_t st) {
    // nodes: nleaves digests (4 words each). Each launch covers up to 9 levels.
    if (nleaves < 2) return cudaErrorInvalidValue;
    size_t m = nleaves / 2;  // parents of leaf pairs live at nodes[m .. 2m)
    const u64* src = leaves;
    // wide levels: one full-occupancy launch per level (the in-block tail of the fused kernel would
    // idle 7/8 of every block); narrow levels (launch-latency-bound): fused, 9 levels per launch
    while (m > (1u << 13)) {
        u64* dst = nodes + m * 4;
        if (hash_id == WF_HASH_BLAKE3_256)
            merkle_level_blake3_kernel<8><<<(unsigned)((m + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uint4*>(src),
                                                                                      reinterpret_cast<uint4*>(dst), m);
        else if (hash_id == WF_HASH_BLAKE3_192)
            merkle_level_blake3_kernel<6><<<(unsigned)((m + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uint4*>(src),
                                                                                      reinterpret_cast<uint4*>(dst), m);
        else if (hash_id == WF_HASH_RP64_256)
            merkle_level_alg_kernel<WF_HASH_RP64_256><<<(unsigned)((m + 127) / 128), 128, 0, st>>>(src, dst, m);
        else if (hash_id == WF_HASH_SHA3_256)
            merkle_level_alg_kernel<WF_HASH_SHA3_256><<<(unsigned)((m + 127) / 128), 128, 0, st>>>(src, dst, m);
        else
            merkle_level_alg_kernel<WF_HASH_RPJIVE64_256><<<(unsigned)((m + 127) / 128), 128, 0, st>>>(src, dst, m);
        src = dst;
        m >>= 1;
    }
    for (;;) {
        unsigned blocks = (unsigned)((m + 255) / 256);
        if (hash_id == WF_HASH_BLAKE3_256) merkle_subtree_kernel<WF_HASH_BLAKE3_256><<<blocks, 256, 0, st>>>(src, nodes, m);
        else if (hash_id == WF_HASH_BLAKE3_192) merkle_subtree_kernel<WF_HASH_BLAKE3_192><<<blocks, 256, 0, st>>>(src, nodes, m);
        else if (hash_id == WF_HASH_RP64_256) merkle_subtree_kernel<WF_HASH_RP64_256><<<blocks, 256, 0, st>>>(src, nodes, m);
        else if (hash_id == WF_HASH_SHA3_256) merkle_subtree_kernel<WF_HASH_SHA3_256><<<blocks, 256, 0, st>>>(src, nodes, m);
        else merkle_subtree_kernel<WF_HASH_RPJIVE64_256><<<blocks, 256, 0, st>>>(src, nodes, m);
        if (m <= 256) break;           // this launch reached the root
        // the launch produced levels m, m/2, ..., m/256 (one node per block); continue above them
        size_t top = m >> 8;
        src = nodes + 2 * (top >> 1) * 4;  // children of the next level = nodes[top .. 2*top)
        m = top >> 1;
        if (m == 0) break;
    }
    return cudaGetLastError();
}
