/* winterfell_b200.h — C ABI of the H100-native STARK proving hot path.
 *
 * Drop-in boundary for facebook/winterfell v0.13.1 (reference paths relative to /root/reference):
 * the library sits behind the four plug-in traits the reference's `Prover` selects through
 * associated types (prover/src/lib.rs:125-158): `TraceLde` (prover/src/trace/trace_lde/mod.rs:26-76),
 * `ConstraintEvaluator` (prover/src/constraints/evaluator/mod.rs:28-42), `ConstraintCommitment`
 * (prover/src/constraints/commitment/mod.rs:24-37) and `VectorCommitment`
 * (crypto/src/commitment.rs:28-86), plus the concrete FriProver (fri/src/prover/mod.rs:100-300)
 * that a GPU prover replaces by overriding `Prover::generate_proof` (prover/src/lib.rs:282).
 * INTEGRATION.md shows the Rust shim (`impl TraceLde for GpuTraceLde` ...) binding every entry
 * point below.
 *
 * Conventions
 *  - plain pointers and sizes only; every function returns WF_OK (0) or a negative error code and
 *    records a message retrievable with wf_last_error(). The Rust traits are infallible
 *    (they panic on misuse, e.g. trace_lde/default/mod.rs:150-158): the shim turns non-zero into panic!.
 *  - field elements are 64-bit words. `mont` flags say whether a HOST buffer holds the reference's
 *    in-memory Montgomery words (x * 2^64 mod p — what a Rust `&[BaseElement]` reinterpreted as
 *    `*const u64` exposes, math/src/field/f64/mod.rs:57-64,212-217) or canonical values in [0, p).
 *    Device buffers are always canonical. Digests are 32 bytes (Blake3_256 bytes, or the four
 *    canonical LE words of an Rp64_256 digest, rescue/rp64_256/digest.rs:36-45).
 *  - one wf_ctx per prover object / per GPU; calls on one ctx are issued on its CUDA stream in
 *    program order and are not re-entrant (the reference calls the factories sequentially from
 *    the proving thread, prover/src/lib.rs:282-492).
 *  - there is NO CPU fallback: every entry point fails with WF_ERR_CUDA when no sm_90 (Hopper) device is
 *    usable.
 */
#ifndef WINTERFELL_B200_H
#define WINTERFELL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WF_OK 0
#define WF_ERR_CUDA (-1)
#define WF_ERR_INVALID (-2)
#define WF_ERR_UNSUPPORTED (-3)
#define WF_ERR_STATE (-4)

#define WF_HASH_BLAKE3_256 0 /* crypto/src/hash/blake/mod.rs:21 */
#define WF_HASH_RP64_256 1   /* crypto/src/hash/rescue/rp64_256/mod.rs:118 */
#define WF_HASH_RPJIVE64_256 2 /* crypto/src/hash/rescue/rp64_256_jive/mod.rs:112 (Jive compression for merges) */
#define WF_HASH_SHA3_256 4     /* crypto/src/hash/sha/mod.rs:19 */
#define WF_HASH_BLAKE3_192 3   /* crypto/src/hash/blake/mod.rs:73: 24-byte digests. Digests cross this ABI in 32-byte slots (the last
                                * 8 bytes zero, as ByteDigest::as_bytes pads them); proofs carry 24 bytes per digest */

typedef struct wf_ctx wf_ctx;
typedef struct wf_mat wf_mat;   /* device matrix of base-field columns (segment layout, see DESIGN.md) */
typedef struct wf_tree wf_tree; /* device Merkle tree: leaves + nodes (crypto/src/merkle/mod.rs:86-98) */
typedef struct wf_fri wf_fri;   /* FRI prover state (fri/src/prover/mod.rs:100-116) */

/* ---- context ---------------------------------------------------------------------------------- */
/* `stream` is a cudaStream_t (NULL = legacy default stream). */
int wf_ctx_create(wf_ctx** out, int device, void* stream);
void wf_ctx_destroy(wf_ctx* ctx);
const char* wf_last_error(const wf_ctx* ctx);
/* One wf_ctx belongs to one device and one calling thread at a time; the library makes ctx's device current on the calling thread
 * wherever work for it starts (allocation, transform launch, gather, sync), so a process may hold contexts for several GPUs. */
int wf_ctx_sync(wf_ctx* ctx);
/* number of kernels this ctx has launched since creation (bench.py's gpu_launches) */
uint64_t wf_ctx_launch_count(const wf_ctx* ctx);
/* device memory this ctx holds: buffers handed out and not yet freed (count and bytes: the matrices, trees, FRI layers the
 * caller still owns) and bytes parked in the ctx's pool for reuse. After every handle is freed, live_buffers is 0 — also
 * after a call that returned an error. Any of the pointers may be NULL. */
int wf_ctx_mem_stats(const wf_ctx* ctx, uint64_t* live_buffers, uint64_t* live_bytes, uint64_t* pooled_bytes);
const char* wf_version(void);
/* stage tracing (the reference's `tracing` spans, prover/src/lib.rs:312-466): when on, the proving
 * entry points record a CUDA event at every stage boundary; wf_ctx_stage_times returns the stage
 * names (comma separated) and their durations in ms since the previous boundary, and resets. */
int wf_ctx_set_profiling(wf_ctx* ctx, int on);
int wf_ctx_stage_times(wf_ctx* ctx, char* names, size_t names_cap, float* ms, size_t* count);

/* ---- matrices --------------------------------------------------------------------------------- */
/* ColMatrix<E> (prover/src/matrix/col_matrix.rs:33): `ncols` host columns of `nrows` elements of
 * extension degree `ext_degree`; becomes ncols*ext_degree base columns on the device. The copies are enqueued on the ctx
 * stream: with PINNED host memory they are asynchronous, and the columns must stay valid and unmodified until the next call that
 * synchronises the context (wf_ctx_sync, any wf_*_root / *_to_host / wf_prove_*); pageable memory is staged before return. */
int wf_mat_from_host_columns(wf_ctx* ctx, const uint64_t* const* cols, uint32_t ncols, size_t nrows,
                             int ext_degree, int mont, wf_mat** out);
/* same, from a DEVICE buffer laid out column-major [ncols][nrows] (base columns, canonical) */
int wf_mat_from_device_columns(wf_ctx* ctx, const uint64_t* d_cols, uint32_t ncols, size_t nrows, wf_mat** out);
/* new matrix holding base columns [first, first + count) of m */
int wf_mat_select_columns(wf_ctx* ctx, const wf_mat* m, uint32_t first, uint32_t count, wf_mat** out);
int wf_mat_free(wf_ctx* ctx, wf_mat* m);
size_t wf_mat_rows(const wf_mat* m);
uint32_t wf_mat_cols(const wf_mat* m);
/* copy out as column-major [cols][rows] or row-major [rows][cols]; dst is host (to_host=1) or device */
int wf_mat_to_columns(wf_ctx* ctx, const wf_mat* m, uint64_t* dst, int to_host, int mont);
int wf_mat_to_rows(wf_ctx* ctx, const wf_mat* m, uint64_t* dst, int to_host, int mont);
/* rows at `positions` (k x cols words, canonical unless mont) -> host; TraceLde::query values
 * (trace_lde/default/mod.rs:199-230, build_segment_queries :284-297) */
int wf_mat_read_rows(wf_ctx* ctx, const wf_mat* m, const uint64_t* positions, size_t k, uint64_t* dst, int mont);

/* ColMatrix::interpolate_columns (col_matrix.rs:192-202): evaluations over the size-n subgroup
 * -> coefficients. n = rows must be a power of two >= 2. */
int wf_mat_interpolate(wf_ctx* ctx, const wf_mat* evals, wf_mat** polys);
/* fft::evaluate_poly per column (math/src/fft/mod.rs:85): coefficients -> evaluations, natural order */
int wf_mat_evaluate(wf_ctx* ctx, const wf_mat* polys, wf_mat** evals);
/* RowMatrix::evaluate_polys_over::<8> (row_matrix.rs:84-100): LDE over the coset 7 * <w_N>,
 * N = n << log_blowup, row i <-> point 7 * w_N^i (natural order). */
int wf_mat_lde(wf_ctx* ctx, const wf_mat* polys, uint32_t log_blowup, wf_mat** lde);
/* same, into a matrix the caller provides (e.g. a wf_mat_wrap_device view of a collective's send buffer) */
int wf_mat_lde_into(wf_ctx* ctx, const wf_mat* polys, uint32_t log_blowup, wf_mat* lde);
/* non-owning handle over device memory that already holds a rows x cols matrix in segment layout
 * (ceil(cols / W) segments of rows x W words, W = 8 for cols >= 8, else the next power of two >= cols);
 * wf_mat_free releases the handle, not the memory */
int wf_mat_wrap_device(wf_ctx* ctx, uint64_t* d_segments, size_t rows, uint32_t cols, wf_mat** out);
/* DefaultTraceLde::new up to the commitment (prover/src/trace/trace_lde/default/mod.rs:63-100,
 * build_trace_commitment :245-265) straight from HOST columns: equivalent to wf_mat_from_host_columns ->
 * wf_mat_interpolate -> wf_mat_lde, but the upload of column chunk k+1 overlaps the layout / iNTT / LDE of
 * chunk k (pass pinned host memory to get the overlap). Returns the coefficient matrix (TracePolyTable)
 * and the LDE. */
int wf_trace_lde_from_host(wf_ctx* ctx, const uint64_t* const* cols, uint32_t ncols, size_t nrows, int mont, uint32_t log_blowup,
                           wf_mat** polys, wf_mat** lde);
/* fft::interpolate_poly_with_offset per column (math/src/fft/mod.rs:351) */
int wf_mat_interpolate_with_offset(wf_ctx* ctx, const wf_mat* evals, uint64_t domain_offset, wf_mat** polys);

/* ---- commitments ------------------------------------------------------------------------------ */
/* RowMatrix::commit_to_rows (row_matrix.rs:184-228) with partition_size == num_cols, then
 * MerkleTree::new (crypto/src/merkle/mod.rs:116-135). */
int wf_commit_rows(wf_ctx* ctx, int hash_id, const wf_mat* m, wf_tree** out);
/* same with column partitions (row_matrix.rs:204-223): the row digest is H::merge_many of the digests of
 * chunks of `partition_size` BASE columns — partition_size = PartitionOptions::partition_size::<E>(cols)
 * * E::EXTENSION_DEGREE (air/src/options.rs:428-444); at most 16 partitions. 0 = whole rows. */
int wf_commit_rows_partitioned(wf_ctx* ctx, int hash_id, const wf_mat* m, uint32_t partition_size, wf_tree** out);
/* MerkleTree::new from host/device leaf digests (VectorCommitment::new, crypto/src/commitment.rs:41) */
int wf_tree_from_leaves(wf_ctx* ctx, int hash_id, const uint8_t* leaves, size_t nleaves, int leaves_on_device,
                        wf_tree** out);
int wf_tree_free(wf_ctx* ctx, wf_tree* t);
int wf_tree_root(wf_ctx* ctx, const wf_tree* t, uint8_t root[32]); /* VectorCommitment::commitment */
size_t wf_tree_num_leaves(const wf_tree* t);
/* copies leaves (nleaves*32 B) and nodes (nleaves*32 B) to host: MerkleTree::from_raw_parts inputs
 * (crypto/src/merkle/mod.rs:148) */
int wf_tree_to_host(wf_ctx* ctx, const wf_tree* t, uint8_t* leaves, uint8_t* nodes);
/* VectorCommitment::open_many = MerkleTree::prove_batch (merkle/mod.rs:217-272): writes the k leaf
 * digests (in the order of `positions`) and the serialized BatchMerkleProof (proofs.rs:390-401).
 * *proof_len: in = capacity, out = bytes written. */
int wf_tree_open_many(wf_ctx* ctx, const wf_tree* t, const uint64_t* positions, size_t k, uint8_t* leaves_out,
                      uint8_t* proof, size_t* proof_len);

/* ---- FRI (fri/src/prover/mod.rs) --------------------------------------------------------------- */
/* FriProver::new + build_layers (:179-239) over `len` evaluations of extension degree d held in
 * device matrix `evals` (d base columns, len rows), domain offset 7.
 * The transcript is the caller's: after each layer the library calls `commit(user, root32)` and
 * then `draw_alpha(user, alpha_out[d])` (ProverChannel::commit_fri_layer / draw_fri_alpha,
 * fri/src/prover/channel.rs:20-27); after the remainder it calls commit(user, remainder_hash). */
typedef void (*wf_fri_commit_fn)(void* user, const uint8_t root[32]);
typedef void (*wf_fri_draw_fn)(void* user, uint64_t* alpha_out);
int wf_fri_build_layers(wf_ctx* ctx, int hash_id, const wf_mat* evals, int ext_degree, uint32_t folding_factor,
                        uint32_t remainder_max_degree, uint32_t blowup, wf_fri_commit_fn commit,
                        wf_fri_draw_fn draw_alpha, void* user, wf_fri** out);
/* same, with the library's own DefaultProverChannel-style coin seeded with hash_elements([])
 * (fri/src/prover/channel.rs:60-72); roots_out receives (num_layers + 1) x 32 bytes. */
int wf_fri_build_layers_default_channel(wf_ctx* ctx, int hash_id, const wf_mat* evals, int ext_degree,
                                        uint32_t folding_factor, uint32_t remainder_max_degree, uint32_t blowup,
                                        uint8_t* roots_out, size_t roots_cap, wf_fri** out);
uint32_t wf_fri_num_layers(const wf_fri* f);
/* remainder polynomial, reversed coefficients (fri/src/prover/mod.rs:230-239); returns element count */
size_t wf_fri_remainder(const wf_fri* f, uint64_t* coeffs, size_t cap_words);
/* FriProver::build_proof (:254-296) serialized as FriProof (fri/src/proof.rs): *len in=cap, out=bytes */
int wf_fri_build_proof(wf_ctx* ctx, wf_fri* f, const uint64_t* positions, size_t k, uint8_t* out, size_t* len);
int wf_fri_free(wf_ctx* ctx, wf_fri* f);

/* ---- verifying standalone FRI proofs (FriVerifier, fri/src/verifier/mod.rs:107-331) ------------------------------------
 * verdicts[j] is the FIRST error FriVerifier::new and then verify return for proof j, in the reference's order: the
 * deserialization of DefaultVerifierChannel::new, new()'s draws and DegreeTruncation checks, then per layer the opening
 * (LayerCommitmentMismatch) and InvalidLayerFolding, then RemainderDegreeMismatch and InvalidRemainderFolding. The codes
 * are the fri::VerifierError variants the verifier returns; INVALID_LAYER_FOLDING and DEGREE_TRUNCATION carry their layer
 * in bits 8 and up (WF_FRI_VERIFY_LAYER). The remainder commitment is never compared with the remainder (read_remainder,
 * fri/src/verifier/channel.rs:112-116): it only reseeds the coin. */
#define WF_FRI_VERIFY_ACCEPT                     0
#define WF_FRI_VERIFY_MALFORMED                  1   /* DeserializationError, a layer missing from the proof, or layer indexes
                                                        (map_positions_to_indexes) that repeat or leave the layer's tree */
#define WF_FRI_VERIFY_LAYER_COMMITMENT_MISMATCH  2   /* LayerCommitmentMismatch */
#define WF_FRI_VERIFY_INVALID_LAYER_FOLDING      3   /* InvalidLayerFolding(layer); layer 0: the caller's evaluations */
#define WF_FRI_VERIFY_REMAINDER_DEGREE_MISMATCH  4   /* RemainderDegreeMismatch */
#define WF_FRI_VERIFY_INVALID_REMAINDER_FOLDING  5   /* InvalidRemainderFolding */
#define WF_FRI_VERIFY_DEGREE_TRUNCATION          6   /* DegreeTruncation(.., folding, layer) */
#define WF_FRI_VERIFY_RANDOM_COIN                7   /* RandomCoinError: no alpha in 1000 draws */
#define WF_FRI_VERIFY_CODE(v)  ((v) & 0xffu)
#define WF_FRI_VERIFY_LAYER(v) ((v) >> 8)
/* FriVerifier::new + verify with DefaultVerifierChannel (fri/src/verifier/channel.rs) for `batch` proofs of one shape:
 * hasher, extension degree (1, 2, 3), FriOptions(blowup, folding_factor, remainder_max_degree) and max_poly_degree; the
 * domain is max_poly_degree.next_power_of_two() * blowup (at most 2^32), offset 7. Per proof j: proofs[j] (proof_lens[j]
 * bytes) holds the serialized FriProof and nothing after it; commitments[j] holds num_commitments[j] x 32 bytes, the layer
 * roots then the remainder commitment as wf_fri_build_layers_default_channel writes them (num_layers + 1 of them);
 * coin_seeds[j] is the 32-byte seed of the public coin when FriVerifier::new starts reseeding it (coin_seeds NULL, or a NULL
 * entry: DefaultRandomCoin::new(&[])); positions[j] and evaluations[j] hold the num_queries[j] query positions and the
 * values at them, [k][ext] canonical words. The proof's num_partitions is honoured (map_positions_to_indexes,
 * fri/src/utils.rs:9-33). WF_ERR_INVALID for caller errors (NULL pointers, a shape with a layer of fewer than two rows or
 * no remainder, a commitment count other than num_layers + 1, a non-canonical evaluation, a position outside the domain),
 * naming the proof; WF_ERR_UNSUPPORTED for a folding factor other than 2, 4, 8 or 16 or an unknown hash. A refused proof
 * is a result: the call returns WF_OK whenever verdicts were written. No device buffer stays live after any return. The
 * host parses and plans without hashing; the device checks the whole batch together, and the number of kernel launches
 * does not depend on `batch` for proofs of one shape. */
int wf_fri_verify_batch(wf_ctx* ctx, int hash_id, int ext_degree, uint32_t folding_factor, uint32_t remainder_max_degree,
                        uint32_t blowup, uint64_t max_poly_degree, uint32_t batch, const uint8_t* const* proofs,
                        const size_t* proof_lens, const uint8_t* const* commitments, const uint32_t* num_commitments,
                        const uint8_t* const* coin_seeds, const uint64_t* const* positions,
                        const uint64_t* const* evaluations, const size_t* num_queries, uint32_t* verdicts);

/* ---- full proof (Prover::prove / generate_proof, prover/src/lib.rs:250-492) --------------------- */
/* Proves the built-in AIR family "FibSmall x k" (k copies of examples/src/fibonacci/fib_small/air.rs
 * side by side, trace width 2k; k = 1 is the reference's fib_small example) and writes the
 * serialized Proof (air/src/proof/mod.rs:189-200). trace_cols: 2k host columns of 2^log_n words;
 * results: the k public inputs (last value of column 2j+1).
 * opts[9] = { num_queries, blowup, grinding, field_extension (1|2|3), fri_folding, fri_remainder_max_degree,
 *             constraint batching (0 Linear | 1 Algebraic | 2 Horner), DEEP batching,
 *             hash_id | num_partitions << 8 | hash_rate << 16 }
 * (ProofOptions::new, air/src/options.rs:132; the two upper fields of opts[8] are ProofOptions::with_partitions,
 * options.rs:193-200 — 0 means the default PartitionOptions::new(1, 1); with more than one partition the main, auxiliary
 * and constraint commitments hash every row as merge_many of the digests of its column partitions, row_matrix.rs:204-223,
 * and the two bytes are written into the proof's serialized options). *proof_len: in = capacity, out = bytes written. */
int wf_prove_fib(wf_ctx* ctx, const uint64_t* const* trace_cols, int mont, uint32_t k, uint32_t log_n,
                 const uint64_t* results, const uint32_t* opts, uint8_t* proof, size_t* proof_len);

/* Generic single-segment AIR: Air::evaluate_transition (air/src/air/mod.rs:210) described as a
 * straight-line program, so that user AIRs beyond the built-in family run on the device evaluator.
 * air_desc (u64 words):
 *   [width, nT, {base_degree, ncycles, cycle...} x nT        TransitionConstraintDegree (transition/degree.rs)
 *    nP, {len, values...} x nP                               get_periodic_column_values (air/mod.rs:300)
 *    nC, constants...,  num_regs,  nI, {op, dst, a, b} x nI   registers: [0,w) current row, [w,2w) next row,
 *                                                             [2w,2w+nP) periodic values, then temporaries;
 *                                                             op 0 ADD, 1 SUB, 2 MUL (dst = r[a] op r[b]),
 *                                                             3 CONST (dst = constants[a]), 4 OUT (result[dst] = r[a])
 *    nA, {column, first_step, stride, nvals, values...} x nA  Assertion::single (stride 0, 1 value) / ::periodic
 *                                                             (stride > 0, 1 value) / ::sequence (stride > 0,
 *                                                             nvals = n / stride values) (assertions/mod.rs:62-120)
 *    nPub, public input elements...,  num_transition_exemptions]
 * Multi-segment descriptions go through wf_prove_air_aux. */
int wf_prove_air(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* const* trace_cols, int mont,
                 uint32_t log_n, const uint32_t* opts, uint8_t* proof, size_t* proof_len);

/* Multi-segment AIR (one auxiliary segment, as in the reference: air/src/air/trace_info.rs:24-40).
 * The description above is followed by the aux section
 *   [aux_width, num_rand_elements,
 *    nTa, {base_degree, ncycles, cycle...} x nTa            aux_transition_constraint_degrees (context.rs:93)
 *    aux_num_regs, nIa, {op, dst, a, b} x nIa                Air::evaluate_aux_transition (air/mod.rs:248-260):
 *                                                            registers over E: [0,w) main current, [w,2w) main next,
 *                                                            [2w,2w+aw) aux current, [2w+aw,2w+2aw) aux next, then
 *                                                            nP periodic values, then the random elements, then
 *                                                            temporaries; same opcodes
 *    nAa, {column, first_step, stride, nvals, {v0, v1, v2} x nvals} x nAa]   Air::get_aux_assertions (:279),
 *                                                            values in E (first ext words used)
 * After the main commitment the prover draws num_rand_elements E elements from the public coin
 * (Air::get_aux_rand_elements, air/mod.rs:292-306) and calls `aux_builder` (Prover::build_aux_trace,
 * prover/src/lib.rs:236-247) on the HOST: rand_elements = [num_rand][d] words, aux_out = [aux_width][n][d]
 * words (one Vec<E> per column, as ColMatrix<E>), both in the representation selected by `mont`.
 * The builder returns 0 on success. d = opts.field_extension. */
typedef int (*wf_aux_builder_fn)(void* user, const uint64_t* rand_elements, uint64_t* aux_out);
int wf_prove_air_aux(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* const* trace_cols, int mont,
                     uint32_t log_n, const uint32_t* opts, wf_aux_builder_fn aux_builder, void* aux_user, uint8_t* proof,
                     size_t* proof_len);

/* Same, for AIRs whose auxiliary assertions depend on the random elements (Air::get_aux_assertions(&self, aux_rand_elements),
 * air/src/air/mod.rs:279): after the random elements are drawn — and after aux_builder has run — `aux_assertions` is called
 * on the HOST with the same rand_elements and with `values` = [sum of nvals over the aux assertions][d] words in description
 * order, preloaded with the description's values; what it leaves there is asserted (positions, strides and counts stay the
 * description's). Representation selected by `mont`; returns 0 on success. A verifier must apply the same function. */
typedef int (*wf_aux_assertions_fn)(void* user, const uint64_t* rand_elements, uint64_t* values);
int wf_prove_air_aux_dyn(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* const* trace_cols, int mont,
                         uint32_t log_n, const uint32_t* opts, wf_aux_builder_fn aux_builder, wf_aux_assertions_fn aux_assertions,
                         void* aux_user, uint8_t* proof, size_t* proof_len);

/* same, trace already on the device: column-major [2k][2^log_n], canonical words */
int wf_prove_fib_dev(wf_ctx* ctx, const uint64_t* d_trace, uint32_t k, uint32_t log_n, const uint64_t* results,
                     const uint32_t* opts, uint8_t* proof, size_t* proof_len);

/* ---- aux segment built on the device from a description (the described alternative to the aux_builder callback) ----
 * Prover::build_aux_trace (prover/src/lib.rs:236-247) as data: each aux column is a per-row term computed by a straight-line
 * program, then (for the running kinds and the recurrences) an exclusive prefix scan. The verifier never sees how aux
 * columns were built, so the AIR description and verification are unchanged. aux_build (u64 words):
 *   [aw, nC, constants...,                                         aw = the AIR's aux width; constants canonical
 *    {kind, init0, init1, init2, num_regs, nI, {op, dst, a, b} x nI} x aw]
 *   kind: 0 POINTWISE, 1 RUNNING_PRODUCT, 2 RUNNING_SUM, 4 LINEAR_RECURRENCE, 6 RATIONAL_RECURRENCE, 8 COUPLED_RECURRENCE,
 *   9 COUPLED_MEMBER (3, 5 and 7 are not kinds).
 *   init: element of E (words >= ext must be 0).
 *   Registers over E, the layout of the aux constraint program: [0,w) main row i, [w,2w) main row (i+1) mod n,
 *   [2w,2w+aw) aux row i, [2w+aw,2w+2aw) aux row (i+1) mod n, nP periodic values col[i mod len], nr random elements,
 *   temporaries; num_regs <= 96. The program of column j reads aux registers of columns < j only, and no temporary before
 *   writing it. Ops as in the constraint programs: 0 ADD, 1 SUB, 2 MUL, 3 CONST (constants of this description), 4 OUT:
 *   OUT 0, r = numerator (exactly once), OUT 1, r = denominator (at most once, default 1), and in LINEAR_RECURRENCE
 *   and RATIONAL_RECURRENCE columns only OUT 2, r = multiplier m_i (exactly once; a polynomial in the registers, never
 *   inverted), in RATIONAL_RECURRENCE columns only OUT 3, r = denominator multiplier c_i (exactly once).
 * For each column j in order, and each row i: t_i = num_i * inv(den_i), inv(0) = 0 (E::inv);
 *   POINTWISE a[i] = t_i;  RUNNING_PRODUCT a[0] = init, a[i+1] = a[i] * t_i;  RUNNING_SUM a[0] = init, a[i+1] = a[i] + t_i;
 *   LINEAR_RECURRENCE a[0] = init, a[i+1] = m_i * a[i] + t_i (i < n - 1): a Horner fingerprint (m = gamma), an accumulator
 *   that restarts where a selector f is 1 (m = 1 - f), the numerator of a fraction sum kept as N / D (m = d_i, t = n_i D[i]);
 *   RATIONAL_RECURRENCE a[0] = init, a[i+1] = (m_i * a[i] + n_i) * inv(c_i * a[i] + d_i) (i < n - 1), with n_i = num_i and
 *   d_i = den_i (not divided first): a Moebius map per row, e.g. continued-fraction convergents (r' = a_i + 1/r: m = a_i, n = 1,
 *   c = 1, d = 0), Riccati-type recurrences, a fractional fingerprint in one column (a' = (alpha a + v_i) / (a + beta), one
 *   constraint a' (c a + d) = m a + n). With c = 0 and d = 1 it is LINEAR_RECURRENCE with t = n_i. The device scans the
 *   maps as 2x2 matrices on projective pairs; where a denominator c_i a[i] + d_i vanishes (a[i+1] = 0) it scans the rows after
 *   it again, so k such rows cost k further scans of the rest of the column, O(k n): negligible for honest traces with random
 *   challenges, where a zero is improbable, and at most one host synchronisation per such column when there is none.
 *   COUPLED_RECURRENCE groups: a kind-8 column j and the k - 1 kind-9 entries right after it, each {9, init0, init1, init2,
 *   0, 0} (no registers, no program), are one group of k = 2..4 columns whose state is a vector: a[i] = (a_0[i], ..,
 *   a_{k-1}[i]) with a_r the column j + r, a_r[0] = the init of column j + r, and a[i+1] = M_i a[i] + t_i over E (i < n - 1).
 *   The leader's program gives the whole step: OUT r, reg = t_r (r < k) and OUT 4 + 4r + c, reg = M[r][c] (r, c < k), each
 *   slot at most once, an unwritten slot 0 (a sparse M needs no zero constants); there is no denominator (a divided term goes
 *   into an earlier POINTWISE column, which the program reads). The leader reads aux columns < j under the rule above; a column
 *   after the group reads all of it. E.g. a second-order recurrence u[i+2] = p_i u[i+1] + q_i u[i] + v_i as the pair
 *   (u[i+1], u[i]) (M = [[p, q], [1, 0]], t = (v, 0)), ordered products of 2x2 to 4x4 matrices of trace values as fingerprints,
 *   linear state machines or filters driven by the trace and the random elements; state that passes through 0 too. A diagonal
 *   M gives k LINEAR_RECURRENCE columns; a 2-group with t = 0 and init (a0, 1) is the projective pair (x, y) of the
 *   RATIONAL_RECURRENCE column of the same matrix (x = y a while no denominator vanishes). The device scans the affine maps
 *   on E^k: one term launch and three scan launches per group, no host synchronisation.
 * wf_aux_build_check: the checks of the description against the AIR (structure, width, register ranges and the columns < j
 * rule, one numerator, one multiplier in a LINEAR_RECURRENCE or RATIONAL_RECURRENCE column, one denominator multiplier in a
 * RATIONAL_RECURRENCE column, a group's members right after its leader, 2 <= k <= 4, members without registers or
 * instructions, a leader's OUT slots inside its group's t and M and none written twice, kinds, canonical constants and
 * inits), without a device. WF_OK, or WF_ERR_INVALID with the reason. */
int wf_aux_build_check(const uint64_t* air_desc, size_t air_desc_len, const uint64_t* aux_build, size_t aux_build_len, uint32_t log_n,
                       char* msg, size_t msg_cap);
/* The build as a step: main_evals = the main trace's evaluations (n x width, as from wf_mat_from_host_columns), rand =
 * [num_rand][ext] canonical words (host). *aux = n x aw*ext base columns in the layout wf_mat_from_host_columns(..., ext)
 * produces, ready for wf_mat_interpolate. */
int wf_aux_build(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* aux_build, size_t aux_build_len,
                 const wf_mat* main_evals, const uint64_t* rand, uint32_t ext, wf_mat** aux);
/* wf_prove_air_aux[_dyn] with the aux segment built on the device from aux_build. Exactly one of trace_cols (host columns, in
 * the representation selected by `mont`) and d_trace (device, column-major [width][2^log_n], canonical). aux_assertions may be
 * NULL; otherwise it is called as in wf_prove_air_aux_dyn, with the random elements only. Same proof bytes as
 * wf_prove_air_aux with a host builder that computes the same columns. */
int wf_prove_air_aux_built(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* aux_build, size_t aux_build_len,
                           const uint64_t* const* trace_cols, const uint64_t* d_trace, int mont, uint32_t log_n, const uint32_t* opts,
                           wf_aux_assertions_fn aux_assertions, void* aux_user, uint8_t* proof, size_t* proof_len);

/* ---- batches: `batch` proofs of ONE AIR structure in one call ----------------------------------------------------------
 * Proof j is byte-identical to wf_prove_air (aux_build == NULL) or to wf_prove_air_aux_built (aux_build given, no aux
 * assertion callback) on air_descs[j] and trace j, with the same opts and log_n. air_descs[j] may differ from air_descs[0]
 * only in the public inputs and in the VALUES of the assertions (sequence assertions included); everything else the prover
 * reads from a description must be identical (wf_air_batch_check). Exactly one of trace_cols ([batch * width] host column pointers,
 * proof-major, representation by `mont`) and d_traces (device, [batch][width][2^log_n], canonical). proofs[j] /
 * proof_lens[j]: in = capacity, out = bytes. All or nothing: on any error no proof is written, the error names the proof
 * it concerns, and no device buffer stays live. The proofs are currently computed one after the other inside the call: a
 * batch issues as many kernel launches as a loop over wf_prove_air. */
int wf_prove_air_batch(wf_ctx* ctx, uint32_t batch, const uint64_t* const* air_descs, const size_t* air_desc_lens,
                       const uint64_t* aux_build, size_t aux_build_len, const uint64_t* const* trace_cols, const uint64_t* d_traces,
                       int mont, uint32_t log_n, const uint32_t* opts, uint8_t* const* proofs, size_t* proof_lens);
/* The checks wf_prove_air_batch runs on its descriptions, without a device: every description passes wf_air_check, and all
 * share the structure of air_descs[0]. WF_OK, or WF_ERR_INVALID with the reason (and the proof it concerns) in msg. */
int wf_air_batch_check(uint32_t batch, const uint64_t* const* air_descs, const size_t* air_desc_lens, uint32_t log_n, uint32_t blowup,
                       char* msg, size_t msg_cap);

/* ---- verifying a batch of proofs of one AIR (verifier::verify, verifier/src/lib.rs:82-147) ---------------------------------
 * verdicts[j] is the FIRST check proof j fails, in the reference's order (the code numbers are not that order: CONTEXT comes
 * first). A refused proof is a result: the call returns WF_OK whenever verdicts were written. */
#define WF_VERIFY_ACCEPT               0
#define WF_VERIFY_MALFORMED            1   /* ProofDeserializationError; the ranges ProofOptions::new / TraceInfo::read_from assert */
#define WF_VERIFY_OOD                  2   /* InconsistentOodConstraintEvaluations */
#define WF_VERIFY_POW                  3   /* QuerySeedProofOfWorkVerificationFailed */
#define WF_VERIFY_TRACE_QUERY          4   /* TraceQueryDoesNotMatchCommitment (main or aux) */
#define WF_VERIFY_CONSTRAINT_QUERY     5   /* ConstraintQueryDoesNotMatchCommitment */
#define WF_VERIFY_FRI_LAYER            6   /* FriVerificationFailed(LayerCommitmentMismatch) */
#define WF_VERIFY_FRI_FOLD             7   /* FriVerificationFailed(InvalidLayerFolding) */
#define WF_VERIFY_FRI_REMAINDER        8   /* FriVerificationFailed(InvalidRemainderFolding / RemainderDegreeMismatch) */
#define WF_VERIFY_CONTEXT              9   /* the proof's context does not fit the AIR (InconsistentBaseField, widths, constraint count) */
#define WF_VERIFY_UNACCEPTABLE_OPTIONS 10  /* AcceptableOptions::OptionSet refused the proof's options */
#define WF_VERIFY_INSUFFICIENT_CONJECTURED_SECURITY 11  /* AcceptableOptions::MinConjecturedSecurity refused the proof */
#define WF_VERIFY_INSUFFICIENT_PROVEN_SECURITY      12  /* AcceptableOptions::MinProvenSecurity refused the proof */
/* Air::get_aux_assertions(aux_rand_elements) of proof `proof` (its index in the batch): rand_elements [nr][ext], values
 * [number of aux assertion values][ext], in: the description's values, out: the values to assert. Non-zero = failure. */
typedef int (*wf_aux_assertions_batch_fn)(void* user, uint32_t proof, const uint64_t* rand_elements, uint64_t* values);
/* air_descs[j]: the flat description of wf_prove_air / wf_prove_air_aux with proof j's public inputs and assertion values; all
 * must share the structure of air_descs[0] (the rule of wf_air_batch_check). The trace length is not part of that structure: it
 * is read from each proof, and a proof whose declared length the AIR does not fit (wf_air_check, the n / stride values of a
 * sequence assertion) gets WF_VERIFY_CONTEXT. hash_id selects the hasher. acceptable_opts: NULL accepts the options the proof
 * carries; else num_acceptable opts[9] vectors of the proving entry points (AcceptableOptions::OptionSet, compared on words
 * 0-7 and the partition bytes of word 8; the hash byte must be hash_id), checked before anything else. aux_assertions
 * (may be NULL): called on the host once per proof that reaches Air::get_aux_assertions, with its index. WF_ERR_INVALID for
 * caller errors (NULL pointers, a description that does not parse or breaks the batch rule, a failing callback), naming the
 * proof; no device buffer stays live after any return. The surviving proofs are checked on the device together: the number
 * of kernel launches does not depend on `batch` for proofs of one shape. For the other two AcceptableOptions variants,
 * MinConjecturedSecurity and MinProvenSecurity, see wf_verify_air_batch_min_security. */
int wf_verify_air_batch(wf_ctx* ctx, uint32_t batch, const uint64_t* const* air_descs, const size_t* air_desc_lens,
                        const uint8_t* const* proofs, const size_t* proof_lens, int hash_id,
                        const uint32_t* acceptable_opts, uint32_t num_acceptable,
                        wf_aux_assertions_batch_fn aux_assertions, void* aux_user, uint32_t* verdicts);
/* wf_verify_air_batch with AcceptableOptions::MinConjecturedSecurity(min_bits) (regime WF_SECURITY_CONJECTURED) or
 * MinProvenSecurity(min_bits) (WF_SECURITY_PROVEN) in place of an option set (verifier/src/lib.rs:333-354). The estimate is
 * Proof::conjectured_security / proven_security of hash_id (wf_proof_security), checked where wf_verify_air_batch checks its
 * option set: after the proof parses (MALFORMED and the parse-time CONTEXT verdicts come first), before the AIR is built at
 * the proof's length. A proof below min_bits gets WF_VERIFY_INSUFFICIENT_CONJECTURED_SECURITY / _PROVEN_SECURITY and never
 * reaches the device; the others are verified exactly as wf_verify_air_batch verifies them. The proven rule accepts when
 * either the list-decoding or the unique-decoding bound reaches min_bits. security_bits (may be NULL): per proof, the bits
 * the reference's error carries (the conjectured bits, or max(ldr, udr)), also for an accepted proof; ~0u for a proof refused
 * before the check. min_bits = 0 gives wf_verify_air_batch(acceptable_opts = NULL)'s verdicts and launches. WF_ERR_INVALID
 * for another regime; every other error is wf_verify_air_batch's. The estimate is memoised per distinct (options, trace
 * length) within a call. */
#define WF_SECURITY_CONJECTURED 1
#define WF_SECURITY_PROVEN      2
int wf_verify_air_batch_min_security(wf_ctx* ctx, uint32_t batch, const uint64_t* const* air_descs, const size_t* air_desc_lens,
                                     const uint8_t* const* proofs, const size_t* proof_lens, int hash_id, int regime, uint32_t min_bits,
                                     wf_aux_assertions_batch_fn aux_assertions, void* aux_user, uint32_t* verdicts,
                                     uint32_t* security_bits);
/* The reference's security estimate (air/src/proof/security.rs) for the Goldilocks field, without a device:
 * ConjecturedSecurity::compute(options, 64, collision_resistance) and ProvenSecurity::compute(options, 64, trace_length,
 * collision_resistance, num_constraints, num_committed_polys), with their own arguments. opts: the opts[9] vector of the
 * proving entry points; words 0-7 are read. collision_resistance: Hasher::COLLISION_RESISTANCE (128 for Blake3_256, Sha3_256,
 * Rp64_256 and RpJive64_256, 96 for Blake3_192). WF_OK, or WF_ERR_INVALID for options outside ProofOptions::new's ranges,
 * a trace length that is not a power of two in [8, 2^32], zero constraints or committed polynomials, or a NULL pointer. */
int wf_security_estimate(const uint32_t* opts, uint64_t trace_length, uint32_t collision_resistance, uint64_t num_constraints,
                         uint64_t num_committed_polys, uint32_t* conjectured, uint32_t* proven_ldr, uint32_t* proven_udr);
/* Proof::conjectured_security::<H>() and proven_security::<H>() (air/src/proof/mod.rs:96-126) of a serialized proof, without
 * a device: the Context at the head of the proof (trace info, modulus, options, constraint count) gives the estimate's
 * inputs; num_committed_polys is the trace width (main + aux) plus the blowup factor. The rest of the proof is not read.
 * WF_ERR_INVALID for a context Context::read_from refuses or a field other than Goldilocks (or a NULL pointer);
 * WF_ERR_UNSUPPORTED for an unknown hash. */
int wf_proof_security(int hash_id, const uint8_t* proof, size_t len, uint32_t* conjectured, uint32_t* proven_ldr, uint32_t* proven_udr);

/* ---- checking a trace against its AIR: the reference's debug builds (Trace::validate, prover/src/trace/mod.rs:86-201;
 *      ConstraintEvaluationTable::validate_transition_degrees, prover/src/constraints/evaluation_table.rs:181-230) ----------
 * Trace check: every main assertion (description order, each one's steps increasing), then every aux assertion (values in E:
 * the first `ext` words of each value), then every transition constraint on steps 0 .. n - exemptions over the trace rows
 * (step, step + 1); periodic value j at step i is column j's value i mod its length. A constraint's value is the sum of all
 * its OUT instructions. Degree check (check_degrees != 0): each transition constraint's evaluations over the constraint
 * evaluation domain 7 <w_ce>, divided by the transition divisor, interpolated; the index of the highest non-zero coefficient
 * must equal the declared degree base (n-1) + sum (n/c)(c-1) - (n - exemptions), and max(max actual, n + 1) rounded up to a
 * power of two must equal ce. */
#define WF_VALID 0
#define WF_VIOLATION_MAIN_ASSERTION 1
#define WF_VIOLATION_AUX_ASSERTION 2
#define WF_VIOLATION_MAIN_TRANSITION 3
#define WF_VIOLATION_AUX_TRANSITION 4
#define WF_VIOLATION_DEGREES 5
#define WF_VIOLATION_CE_DOMAIN 6
typedef struct wf_validation {
    uint32_t kind;    /* the FIRST violation in the reference's order (assertions, transitions by step with main before aux,
                         degrees, domain size), or WF_VALID */
    uint32_t index;   /* assertion index in description order, or constraint index within its segment */
    uint64_t step;    /* failing step (assertions, transitions) */
    uint32_t column;  /* assertion column */
    uint32_t num_transition_constraints;  /* main + aux: length of the arrays below */
} wf_validation;
/* Exactly one of trace_cols (host columns, representation by `mont`) and d_trace (device, column-major [width][2^log_n],
 * canonical). A two-segment AIR takes exactly one of aux_build (the aux segment built on the device from rand, as
 * wf_aux_build) and aux_cols ([aw] host columns of [2^log_n][ext] words, representation by `mont`). rand: [nr][ext] canonical.
 * WF_OK when the check ran (report->kind says whether the trace is valid; msg gets the reference's panic message);
 * WF_ERR_INVALID for a bad description or arguments, with the reason of wf_air_check / wf_aux_build_check.
 * first_failing_step (or NULL): per transition constraint, main then aux, the smallest failing step, ~0 when it never fails.
 * expected_degrees / actual_degrees (or NULL): filled when check_degrees is set, even when the trace check failed. No device
 * buffer stays live after any return. Device scratch of the degree check: ce * (n_main + n_aux * ext) * 8 bytes, twice. */
int wf_trace_validate(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* aux_build, size_t aux_build_len,
                      const uint64_t* const* aux_cols, const uint64_t* const* trace_cols, const uint64_t* d_trace, int mont,
                      const uint64_t* rand, uint32_t log_n, uint32_t ext, int check_degrees, wf_validation* report,
                      uint64_t* first_failing_step, uint64_t* expected_degrees, uint64_t* actual_degrees, char* msg, size_t msg_cap);
/* The analogue of a debug build (default off). On: wf_prove_air, wf_prove_air_aux, wf_prove_air_aux_dyn, wf_prove_air_aux_built
 * and wf_prove_air_batch run the trace check after the aux segment is built and its assertion values are final (with the
 * transcript's random elements), and the degree check on their own LDEs right after constraint evaluation;
 * wf_eval_constraints runs the degree check. A violation returns WF_ERR_INVALID with the reference's message, writes no proof
 * and leaves no buffer live. Off: these paths are unchanged. wf_prove_air_sharded runs the same checks at the same points,
 * each rank on its share (see there). wf_prove_fib and wf_prove_fib_sharded are not checked. */
int wf_ctx_set_validation(wf_ctx* ctx, int on);

/* ---- the same pipeline as separate steps, for a host that owns the transcript (the Rust shim of
 *      INTEGRATION.md: impl ConstraintEvaluator / ConstraintCommitment, prover/src/lib.rs:195-223) ---- */
/* ConstraintEvaluator::evaluate (prover/src/constraints/evaluator/mod.rs:28-42, default.rs:60-118) +
 * ConstraintEvaluationTable::combine (evaluation_table.rs:163): CompositionPolyTrace over the CE domain
 * as a (n * ce_blowup) x ext matrix. air_desc as for wf_prove_air[_aux]; main_lde N x width, aux_lde
 * N x aux_width*ext (NULL for single-segment AIRs). coeffs: ConstraintCompositionCoefficients
 * (air/src/air/coefficients.rs:72) flattened [transition: main, aux | boundary: main, aux][ext] with
 * boundary coefficients in the sorted-assertion order; aux_rand [num_rand][ext]. Canonical words. */
int wf_eval_constraints(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, uint32_t log_n, uint32_t blowup, uint32_t ext,
                        const wf_mat* main_lde, const wf_mat* aux_lde, const uint64_t* coeffs, const uint64_t* aux_rand,
                        wf_mat** out);
/* Prover::build_constraint_commitment (prover/src/lib.rs:215-223; DefaultConstraintCommitment::new,
 * constraints/commitment/default.rs:44-150): composition trace -> num_cols column polynomials of
 * degree < n (CompositionPoly, n x num_cols*ext), their LDE (N x num_cols*ext) and its row commitment */
int wf_composition_commit(wf_ctx* ctx, int hash_id, const wf_mat* comp_trace, uint32_t log_n, uint32_t blowup, uint32_t ext,
                          uint32_t num_cols, wf_mat** polys, wf_mat** lde, wf_tree** tree);
/* same with the PartitionOptions argument of build_constraint_commitment (lib.rs:220): partition_size in BASE columns =
 * PartitionOptions::partition_size::<E>(num_cols) * ext (0 or num_cols * ext = whole rows), as wf_commit_rows_partitioned */
int wf_composition_commit_partitioned(wf_ctx* ctx, int hash_id, const wf_mat* comp_trace, uint32_t log_n, uint32_t blowup,
                                      uint32_t ext, uint32_t num_cols, uint32_t partition_size, wf_mat** polys, wf_mat** lde,
                                      wf_tree** tree);
/* ColMatrix::evaluate_columns_at (prover/src/matrix/col_matrix.rs:245) at two points of E (z and z*g for
 * TracePolyTable::get_ood_frame, trace/poly_table.rs:68-76; CompositionPoly::get_ood_frame,
 * composition_poly.rs:101-108). col_ext = 1: base columns; col_ext = ext: the matrix holds columns of E
 * (ext consecutive base columns each). out0/out1: [cols / col_ext][ext] host words. */
int wf_mat_evaluate_at(wf_ctx* ctx, const wf_mat* polys, uint32_t ext, uint32_t col_ext, const uint64_t* z0, const uint64_t* z1,
                       uint64_t* out0, uint64_t* out1);
/* DeepCompositionPoly::{add_trace_polys, add_composition_poly, evaluate} (prover/src/composer/mod.rs:67-210):
 * DEEP composition evaluated over the LDE domain, N x ext. coeffs / ood_cur / ood_next: [width + aux_width +
 * composition columns][ext] in that order (DeepCompositionCoefficients, TraceOodFrame + QuotientOodFrame rows).
 * WF_ERR_INVALID when z or z*g lies on the LDE domain 7 <w_N> (a base-field point with (point / 7)^N = 1): some row's
 * denominator x - z vanishes there. wf_deep_compose_polys is exact at such a point. */
int wf_deep_compose(wf_ctx* ctx, uint32_t ext, const wf_mat* main_lde, const wf_mat* aux_lde, const wf_mat* cons_lde, uint32_t log_n,
                    const uint64_t* z, const uint64_t* coeffs, const uint64_t* ood_cur, const uint64_t* ood_next, wf_mat** out);
/* The same DEEP composition from the COEFFICIENT matrices, as the reference builds it: S = sum_j coeffs_j p_j over the n
 * coefficients, the synthetic divisions by (X - z) and (X - z*g), and one LDE of the quotient (blowup 2^log_blowup) — the
 * N x ext matrix wf_deep_compose returns for the LDEs of the same polynomials, bit for bit. main_polys n x width,
 * aux_polys n x aux_width*ext (NULL for single-segment AIRs), cons_polys n x composition columns*ext (wf_composition_commit's
 * polys); n a power of two >= 8. No OOD values are taken: the quotient of a synthetic division does not depend on the constant
 * term, which is all that subtracting S(z) and S(z*g) changes. Reads the n coefficient rows instead of the N LDE rows. */
int wf_deep_compose_polys(wf_ctx* ctx, uint32_t ext, const wf_mat* main_polys, const wf_mat* aux_polys, const wf_mat* cons_polys,
                          uint32_t log_blowup, const uint64_t* z, const uint64_t* coeffs, wf_mat** out);

/* ProverChannel::grind_query_seed (prover/src/channel.rs:169-184), serial semantics: the SMALLEST
 * nonce >= 1 with trailing_zeros(first 8 LE bytes of H::merge_with_int(seed, nonce)) >= grinding. */
int wf_grind(wf_ctx* ctx, int hash_id, const uint8_t seed[32], uint32_t grinding, uint64_t* nonce);

/* ---- one proof sharded over several GPUs (SURVEY.md 8e; one process and one wf_ctx per GPU) ------------------
 * The reference has no distributed prover; its unit of distribution is the column (ColMatrix columns are independent,
 * prover/src/matrix/col_matrix.rs:192-202) and PartitionOptions (air/src/options.rs:405-445). Here rank r of `world`
 * owns trace columns [r*w/world, (r+1)*w/world): it interpolates and extends them locally, the LDE is exchanged into
 * row shards (rank r holds LDE rows [r*N/world, (r+1)*N/world) of ALL columns plus `blowup` halo rows), and leaf
 * hashing, constraint evaluation, DEEP composition and the first FRI layers run on row shards; every Merkle tree is a
 * local subtree per rank plus log2(world) top levels built from an all-gather of the subtree roots; query openings are
 * gathered from their owners. The proof is byte-identical to wf_prove_fib's on one GPU.
 * The host program supplies the collectives (NCCL point-to-point in bench.py; any MPI-like layer works): */
typedef struct wf_comm {
    void* user;
    int rank, world; /* world: a power of two */
    /* Point-to-point exchange of DEVICE buffers of `bytes` bytes each: send[i] goes to rank send_peer[i], recv[i] is
     * filled by rank recv_peer[i]; transfers between one pair of ranks match in list order; no entry names the caller's
     * own rank. Must be ordered after the work already enqueued on the ctx stream and be complete, or ordered on that
     * stream, when it returns. */
    int (*exchange)(void* user, size_t nsend, const int* send_peer, const void* const* send, size_t nrecv,
                    const int* recv_peer, void* const* recv, size_t bytes);
    /* all-gather of `bytes` bytes per rank between HOST buffers: recv = world x bytes in rank order */
    int (*all_gather_host)(void* user, const void* send, void* recv, size_t bytes);
    /* element-wise wrapping sum over the ranks of `words` 64-bit words of a DEVICE buffer, in place (merges gathers
     * whose entries are non-zero on exactly one rank); same ordering rule as exchange */
    int (*all_reduce_sum)(void* user, void* d_buf, size_t words);
    /* Optional (may be NULL: every exchange is then ordered on the ctx stream). fork: exchanges issued from now on run on the
     * communicator's own stream, ordered after everything enqueued on the ctx stream so far — the library keeps enqueuing
     * kernels on the ctx stream meanwhile (the LDE of the next coset overlaps the exchange of the previous one). fork may
     * be called repeatedly; each call adds "wait for the ctx stream's current tail" to the communicator stream. join: the
     * ctx stream waits for every exchange issued since the first fork; later exchanges are on the ctx stream again. */
    int (*fork)(void* user);
    int (*join)(void* user);
} wf_comm;
/* The main-trace columns [*first, *first + *count) that `rank` of `world` (a power of two) owns in a sharded proof of a trace
 * of `width` (1..255) columns: contiguous runs of whole 8-column segments in rank order, the first (segments mod world) ranks
 * one segment more than the others; the last segment may be partly filled and trailing ranks may own no column. Needs no
 * device. WF_ERR_INVALID for a world that is not a power of two, a rank outside it or a width outside 1..255. */
int wf_shard_columns(uint32_t width, uint32_t world, uint32_t rank, uint32_t* first, uint32_t* count);
/* FibSmall x k (as wf_prove_fib) sharded over comm->world GPUs: this rank passes ITS columns, wf_shard_columns(2k, world,
 * rank) (host columns, or d_local = device column-major [count][2^log_n]).
 * `results` and `opts` are the full proof's; every rank returns the same proof bytes.
 * stats (optional, 8 doubles): [0] bytes this rank sent through exchanges ordered on the ctx stream, [1] ms inside those,
 * [2] number of collectives, [3] ms inside all_gather_host + all_reduce_sum, [4] FRI layers folded on shards, [5] bytes sent
 * overlapped with compute (the trace LDE's cosets), [6] how those travelled: 1 = peer copies (copy engines) into the owners'
 * staging buffers mapped through CUDA IPC (the default when the driver allows it), 0 = comm->exchange between fork and join
 * (the driver refused the mapping, or WF_PEER_PUSH=0). */
int wf_prove_fib_sharded(wf_ctx* ctx, const wf_comm* comm, const uint64_t* const* local_cols, const uint64_t* d_local, int mont,
                         uint32_t k, uint32_t log_n, const uint64_t* results, const uint32_t* opts, uint8_t* proof,
                         size_t* proof_len, double* stats);
/* A user-described AIR (the description of wf_prove_air / wf_prove_air_aux_built) sharded over comm->world GPUs. Every rank
 * passes the same description, options, log_n and aux build, plus its own block of main-trace columns: local_count =
 * wf_shard_columns(width, world, rank)'s count, as host columns (local_cols, representation by `mont`) or device memory
 * (d_local, column-major [local_count][2^log_n], canonical); a rank that owns no column passes local_count = 0 and may pass
 * NULL for both. Single-segment AIR: aux_build = NULL, aux_assertions = NULL; every rank returns the bytes wf_prove_air gives
 * for the whole trace. Two-segment AIR: aux_build is required (host-callback builders are not supported here); every rank
 * gathers the whole main trace (n * width * 8 bytes of device memory per rank), builds the aux segment on the device with the
 * transcript's random elements and returns the bytes wf_prove_air_aux_built gives; aux_assertions (may be NULL) is called on
 * every rank with the same random elements, as there. stats as wf_prove_fib_sharded. With wf_ctx_set_validation on, the trace
 * check runs once the aux segment and its assertion values are final and the degree check right after constraint
 * evaluation, as in the one-GPU prover, each rank on its share: the main assertions on its own columns, every aux assertion,
 * transition steps [r n/G, (r+1) n/G) (a single-segment AIR's rows come by one exchange of n * width * 8 / G bytes per rank),
 * and the degrees of its block of the CE x (n_main + n_aux * ext) transition matrix (its CE rows from its own LDE rows, one
 * exchange into column blocks). One all_gather_host of the raw results gives every rank the same verdict: a violation returns
 * WF_ERR_INVALID on every rank with the message the one-GPU prover gives for the same inputs, writes no proof and leaves no
 * buffer live. Off: this path is unchanged. Refusals (WF_ERR_INVALID / WF_ERR_UNSUPPORTED: a world that is not a power of two >= 2, a trace too short for the
 * world, a description that fails wf_air_check, a bad aux build, a local_count that is not this rank's) happen before any
 * device buffer is allocated, and every rank returns an error: the checks on shared values need no communication, and every
 * rank's verdict on its own block is all-gathered before the first exchange. */
int wf_prove_air_sharded(wf_ctx* ctx, const wf_comm* comm, const uint64_t* air_desc, size_t air_desc_len, const uint64_t* aux_build,
                         size_t aux_build_len, wf_aux_assertions_fn aux_assertions, void* aux_user, const uint64_t* const* local_cols,
                         const uint64_t* d_local, uint32_t local_count, int mont, uint32_t log_n, const uint32_t* opts, uint8_t* proof,
                         size_t* proof_len, double* stats);
/* wf_trace_validate over comm->world GPUs, without a proof: the checks wf_prove_air_sharded runs with validation on, with the
 * report wf_trace_validate gives. Every rank passes the same description, log_n, ext, check_degrees and random elements
 * (rand: [nr][ext] canonical), plus its own block of main-trace columns as wf_prove_air_sharded takes it: local_count =
 * wf_shard_columns(width, world, rank)'s count, host columns (local_cols, representation by `mont`) or device memory (d_local,
 * column-major [local_count][2^log_n], canonical); a rank that owns no column passes local_count = 0 and may pass NULL for
 * both. A two-segment AIR takes exactly one of aux_build (built on the device on every rank from the gathered main trace, as
 * the sharded prover builds it) and aux_cols (the whole aux segment, [aw] host columns of [2^log_n][ext] words, representation
 * by `mont`, the same on every rank). On every rank the return value, report, first_failing_step, expected_degrees,
 * actual_degrees and msg are exactly what wf_trace_validate returns for the whole trace with the same arguments: WF_OK when the
 * checks ran, a violation being a result; the degree check runs even when the trace check failed.
 * Work per rank r: the main assertions on its own columns, every aux assertion, transition steps [r n/G, (r+1) n/G); the
 * degree check on CE rows [r ce/G, (r+1) ce/G) from LDE row shards at the CE blowup (its columns extended locally and turned
 * into row shards with ce_blowup halo rows; the aux segment extended on every rank and sharded as the prover's), then the
 * degrees of its 8-column block of the CE x (n_main + n_aux * ext) transition matrix.
 * Device memory per rank, with c main columns of which cl are its own and k = n_main + n_aux * ext:
 *   trace check: n * cl * 8 * 2 (its columns' coefficients and evaluations) and (n/G + 1) * c * 8 (its rows: one exchange of
 *     n * c * 8 / G bytes) -- except with aux_build, which gathers the whole main trace, n * c * 8, as the sharded prover does;
 *     the aux segment n * aw * ext * 8 is held whole (it is replicated, not sharded);
 *   degree check: n * ce_blowup * cl * 8 (its columns' LDE) and 2 * (ce/G + ce_blowup) * c * 8 (staging and row shard), then
 *     (ce/G) * k * 8 (its CE rows) and, twice, ce * 8 * (8 x its share of the k/8 column segments) (its block and its
 *     coefficients); about 1/G of wf_trace_validate's ce * k * 8, twice.
 * Refusals (WF_ERR_INVALID / WF_ERR_UNSUPPORTED: a world that is not a power of two >= 2, a trace shorter than 64 * world rows
 * -- the prover's row-shard condition, N/G >= 64 * blowup, with the CE blowup in place of the proof's --, what
 * wf_trace_validate refuses, a local_count that is not this rank's) happen before any device buffer is allocated, and every
 * rank returns an error: the checks on shared values need no communication, and every rank's verdict on its own block is
 * all-gathered before the first exchange. No device buffer stays live after any return. */
int wf_trace_validate_sharded(wf_ctx* ctx, const wf_comm* comm, const uint64_t* air_desc, size_t air_desc_len,
                              const uint64_t* aux_build, size_t aux_build_len, const uint64_t* const* aux_cols,
                              const uint64_t* const* local_cols, const uint64_t* d_local, uint32_t local_count, int mont,
                              const uint64_t* rand, uint32_t log_n, uint32_t ext, int check_degrees, wf_validation* report,
                              uint64_t* first_failing_step, uint64_t* expected_degrees, uint64_t* actual_degrees,
                              char* msg, size_t msg_cap);

/* ---- constraint kernels compiled per AIR ---------------------------------------------------------------------------
 * wf_eval_constraints / wf_prove_air[_aux] evaluate the AIR's transition programs with a kernel compiled at run time for that
 * AIR (NVRTC: the programs become straight-line code, registers and constants are literals), cached in the context; without
 * NVRTC on the machine, or with wf_ctx_set_jit(ctx, 0), the same programs are interpreted by the built-in kernel (same
 * results bit for bit). wf_ctx_jit_stats: kernels compiled, launches served from the cache, compilations that failed and
 * fell back. wf_jit_compile_air compiles the kernel of a description without a device (log: compiler output). */
int wf_ctx_set_jit(wf_ctx* ctx, int on);
int wf_ctx_jit_stats(wf_ctx* ctx, uint64_t* compiled, uint64_t* cache_hits, uint64_t* fallbacks);
int wf_jit_compile_air(const uint64_t* air_desc, size_t air_desc_len, uint32_t ext, size_t* cubin_bytes, char* log, size_t log_cap);
/* Everything wf_prove_air / wf_eval_constraints check about a description before they touch the device, without a device:
 * structure, degrees against the blowup factor, periodic columns, assertion validity and overlaps (the conditions
 * Air::new, BoundaryConstraints::new and prepare_assertions panic on, air/src/air/boundary/mod.rs:190-215). WF_OK, or
 * WF_ERR_INVALID with the reason in msg. */
int wf_air_check(const uint64_t* air_desc, size_t air_desc_len, uint32_t log_n, uint32_t blowup, char* msg, size_t msg_cap);

/* ---- plain kernels on caller-owned DEVICE buffers (unit parity + bench legs) ------------------- */
/* in-place NTT (inverse=0) / iNTT (inverse=1) of `cols` columns, column-major [cols][n], n = 1 << log_n */
int wf_ntt_dev(wf_ctx* ctx, uint64_t* d_data, uint32_t log_n, uint32_t cols, int inverse);
/* leaf digests of a row-major [nrows][cols] device matrix */
int wf_hash_rows_dev(wf_ctx* ctx, int hash_id, const uint64_t* d_rows, size_t nrows, uint32_t cols, uint8_t* d_digests);
/* Merkle nodes (nleaves x 32 B, nodes[0] = 0, nodes[1] = root) from device leaf digests */
int wf_merkle_dev(wf_ctx* ctx, int hash_id, const uint8_t* d_leaves, size_t nleaves, uint8_t* d_nodes);
/* one FRI fold: d_evals [len][d] -> d_next [len/folding][d]; alpha = d host words */
int wf_fri_fold_dev(wf_ctx* ctx, const uint64_t* d_evals, size_t len, int ext_degree, uint32_t folding_factor,
                    const uint64_t* alpha, uint64_t* d_next);

/* field arithmetic of the device code on caller-chosen operands (a, b: n canonical words each, device):
 * d_out[0..n) = a*b (math/src/field/f64/mod.rs:357), [n..2n) = a+b (:319), [2n..3n) = a-b (:339),
 * [3n..4n) = 1/a (:157; 0 for a = 0), then 18 blocks a * 2^s for s in WF_FIELD_TEST_SHIFTS.
 * d_out holds 22 n words. */
#define WF_FIELD_TEST_SHIFTS {1, 3, 6, 12, 24, 31, 32, 33, 48, 63, 64, 65, 72, 80, 84, 90, 95, 96}
int wf_field_ops_dev(wf_ctx* ctx, const uint64_t* d_a, const uint64_t* d_b, size_t n, uint64_t* d_out);
/* the device's power-of-two multiply for every compile-time shift: d_out[k*n + i] = a[i] * 2^k for k = 0..96
 * (a: n canonical words, device). d_out holds 97 n words. */
int wf_field_shifts_dev(wf_ctx* ctx, const uint64_t* d_a, size_t n, uint64_t* d_out);
/* the Rescue arithmetic of the Rp64_256 / RpJive64_256 kernels (rp64.cuh, rpjive.cuh) on ANY 64-bit words a, b (n of each,
 * device, n a multiple of 24), through the same device functions the kernels call. d_out holds 10 blocks of n words:
 * gl_mul_weak(a, b), gl_sqr_weak(a), rp64_exp7(a) (congruent to the exact results, below 2^64 only), then x^(1/7) by
 * rp64_inv7_group<G> on consecutive groups of G words of a for each G in WF_RESCUE_TEST_GROUPS (weak as well), then rp64_mds on
 * consecutive groups of 12 words of a and rpj_mds on groups of 8 (canonical). */
#define WF_RESCUE_TEST_GROUPS {1, 2, 3, 4, 6}
int wf_rescue_ops_dev(wf_ctx* ctx, const uint64_t* d_a, const uint64_t* d_b, size_t n, uint64_t* d_out);
/* the device's permutation, merge and merge_with_int of hash_id (WF_HASH_RP64_256: states of W = 12 words,
 * WF_HASH_RPJIVE64_256: W = 8) on n states of any words (device) and n values: d_out = [n][W] permuted states, then [n][4]
 * merge of words 0..8 of each state as two digests, then [n][4] merge_with_int(words 0..4, values[i]). */
int wf_rescue_permute_dev(wf_ctx* ctx, int hash_id, const uint64_t* d_states, const uint64_t* d_values, size_t n, uint64_t* d_out);
/* extension-field arithmetic of the device code (ExtensibleField<2> / <3> for BaseElement, math/src/field/f64/mod.rs:401-499;
 * inverses extensions/quadratic.rs:81-94, cubic.rs:81-97): a, b = n elements of `ext` (2 | 3) canonical words each (device);
 * d_out = 6 blocks of n elements: a*b, 1/a (0 for 0), frobenius(a), a.mul_base(b[0]), a+b, a-b. */
int wf_ext_ops_dev(wf_ctx* ctx, uint32_t ext, const uint64_t* d_a, const uint64_t* d_b, size_t n, uint64_t* d_out);
/* the delayed-reduction dot product of the OOD, DEEP-sum and constraint kernels (GlAcc: acc_zero / acc_mad / acc_reduce,
 * gl64.cuh) on n rows of k terms (1 <= k < 2^31): d_x, d_y = [n][k] ANY 64-bit words (device). d_out = [n][6] words: the raw
 * 160-bit accumulator sum_j x_j y_j as w0..w4 (32-bit words, w0 lowest, one per output word), then its reduction mod p. */
int wf_acc_ops_dev(wf_ctx* ctx, const uint64_t* d_x, const uint64_t* d_y, uint32_t k, size_t n, uint64_t* d_out);
/* the constraint evaluation of wf_eval_constraints over CE rows [row0, row0 + ce_rows) only (ce_rows >= 64, inside the domain),
 * as the row-sharded prover runs it: main_lde / aux_lde hold the window's LDE rows (ce_rows << log2(blowup / ce_blowup) of them,
 * from row row0 << log2(blowup / ce_blowup)) followed by `blowup` halo rows (the LDE rows after the window, wrapping to row 0).
 * *out = ce_rows x ext, row j = CE row row0 + j of wf_eval_constraints. */
int wf_eval_constraints_window(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, uint32_t log_n, uint32_t blowup,
                               uint32_t ext, const wf_mat* main_lde, const wf_mat* aux_lde, const uint64_t* coeffs,
                               const uint64_t* aux_rand, size_t row0, size_t ce_rows, wf_mat** out);
/* the specialised FibSmall x k constraint kernel of wf_prove_fib with caller-chosen coefficients: the same values as
 * wf_eval_constraints on the description of FibSmall x k (pair j starting at (j+1, j+1), results[j] the last value of column
 * 2j+1), with the same coefficient layout. ce_rows = 0 (and row0 = 0): the whole CE domain, lde = the (n * blowup) x 2k trace
 * LDE; otherwise the window of wf_eval_constraints_window. */
int wf_eval_constraints_fib(wf_ctx* ctx, uint32_t k, const uint64_t* results, uint32_t log_n, uint32_t blowup, uint32_t ext,
                            const wf_mat* lde, const uint64_t* coeffs, size_t row0, size_t ce_rows, wf_mat** out);
/* the constraint evaluation of wf_eval_constraints (resp. wf_eval_constraints_fib) on the sub-coset of `rows` points of the CE
 * domain only (rows a power of two, at most n * ce_blowup), as wf_prove_air / wf_prove_fib run it: the composition polynomial is
 * interpolated from those rows. Takes the whole LDEs; *out = rows x ext, row j = CE row j * (n * ce_blowup / rows). */
int wf_eval_constraints_subcoset(wf_ctx* ctx, const uint64_t* air_desc, size_t air_desc_len, uint32_t log_n, uint32_t blowup,
                                 uint32_t ext, const wf_mat* main_lde, const wf_mat* aux_lde, const uint64_t* coeffs,
                                 const uint64_t* aux_rand, size_t rows, wf_mat** out);
int wf_eval_constraints_fib_subcoset(wf_ctx* ctx, uint32_t k, const uint64_t* results, uint32_t log_n, uint32_t blowup, uint32_t ext,
                                     const wf_mat* lde, const uint64_t* coeffs, size_t rows, wf_mat** out);

/* ---- host-side helpers of the product (transcript arithmetic; no GPU needed) ------------------- */
/* H::hash_elements / merge / merge_with_int on the host (crypto/src/hash/mod.rs:31-64) */
int wf_host_hash_elements(int hash_id, const uint64_t* elems, size_t n, uint8_t out[32]);
int wf_host_merge(int hash_id, const uint8_t two[64], uint8_t out[32]);
int wf_host_merge_with_int(int hash_id, const uint8_t seed[32], uint64_t value, uint8_t out[32]);
uint64_t wf_host_mul(uint64_t a, uint64_t b);           /* canonical Goldilocks product */
uint64_t wf_host_mul_2exp(uint64_t x, uint32_t k);      /* x * 2^k mod p, k <= 96 (kernel twiddle path) */
uint64_t wf_host_mont_to_canonical(uint64_t m);
uint64_t wf_host_canonical_to_mont(uint64_t x);
/* ByteWriter::write_usize (utils/core/src/serde/byte_writer.rs:77-92), the vint64 of the proof format;
 * returns the number of bytes written (1..9) */
size_t wf_host_write_usize(uint64_t value, uint8_t out[9]);
/* DefaultRandomCoin::new(seed elements) [+ reseed(digest)] + draw x count (crypto/src/random/default.rs:95-170):
 * the transcript arithmetic the proof path runs on the host. out[count][d]; 0 on success */
int wf_host_coin_draw(int hash_id, const uint64_t* seed_elems, size_t n_seed, const uint8_t* reseed32, int d, size_t count,
                      uint64_t* out);

/* index arithmetic of an opening in a tree stored as one subtree per rank (wf_prove_fib_sharded): want[i] = heap node
 * (< n_global) or n_global + leaf that MerkleTree::prove_batch (crypto/src/merkle/mod.rs:217-272) reads for `positions`;
 * idx[i] = its index in rank `rank`'s subtree (node < n_local, else n_local + leaf), ~0 when another rank holds it,
 * ~0 - 1 for a node of the top log2(world) levels. Returns the number of entries or -1. Host code. */
long wf_host_sharded_opening_plan(size_t n_global, int world, int rank, const uint64_t* positions, size_t k, uint64_t* want,
                                  uint64_t* idx, size_t cap);
/* FibSmallProver::build_trace (examples/src/fibonacci/fib_small/prover.rs:37-53) for the built-in "FibSmall x k"
 * family: cols = [2k][n] canonical words, pair j starting at (j+1, j+1); results[j] = its public input. Host code. */
int wf_host_build_fib_trace(uint32_t k, size_t n, uint64_t* cols, uint64_t* results);

#ifdef __cplusplus
}
#endif
#endif /* WINTERFELL_B200_H */
