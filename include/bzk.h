/* libbzk — H100-native prover kernels for Bazuka's MPN Groth16 path.  C ABI (drop-in boundary).
 *
 * Everything here is plain C: opaque handles, raw pointers and sizes, int32 status codes.  No
 * exception, abort or global mutable state crosses this boundary.  One `bzk_ctx` per GPU; calls
 * on one ctx are serialised by the caller, distinct ctxs may be used from different threads.
 *
 * Data images are the reference's own in-memory images, so a Rust caller passes `&[T]` pointers
 * without conversion (see INTEGRATION.md):
 *   bzk_fr        = `ZkScalar([u64;4])`                      /root/reference/src/zk/mod.rs:202-206
 *                   = bls12_381::Scalar (transmute)          /root/reference/src/zk/groth16/mod.rs:7-17
 *                   4 little-endian u64 limbs, Montgomery form (R = 2^256), fully reduced.
 *   bzk_g1_affine = `(Fp, Fp, bool)` = bls12_381::G1Affine   /root/reference/src/zk/groth16/mod.rs:21-23,44-60
 *                   x, y: 6 LE u64 limbs each, Montgomery (R = 2^384); `infinity` byte; 7 pad bytes.
 *   bzk_g2_affine = `((Fp,Fp),(Fp,Fp),bool)` = G2Affine      /root/reference/src/zk/groth16/mod.rs:25-27
 *
 * Which reference interface each entry point replaces is stated on the entry point.  The
 * arithmetic the reference calls lives in un-vendored crates (bellman 0.14.0, bls12_381 0.8.0,
 * ff 0.13 — /root/reference/Cargo.toml:19,27-28); "replaces" therefore names the crate function
 * and the reference call site that reaches it.
 */
#ifndef BZK_H
#define BZK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ types */
typedef struct { uint64_t l[4]; } bzk_fr;                                          /* 32 B */
typedef struct { uint64_t x[6]; uint64_t y[6]; uint8_t infinity; uint8_t pad[7]; } bzk_g1_affine; /* 104 B */
typedef struct { uint64_t x[12]; uint64_t y[12]; uint8_t infinity; uint8_t pad[7]; } bzk_g2_affine; /* 200 B */

typedef struct bzk_ctx bzk_ctx;            /* one per GPU */
typedef struct bzk_g1_bases bzk_g1_bases;  /* device-resident, packed base vector (a proving-key column) */
typedef struct bzk_g2_bases bzk_g2_bases;

/* ------------------------------------------------------------------ status */
#define BZK_OK 0
#define BZK_ERR_BAD_ARG (-1)       /* null pointer, size out of range, unknown op */
#define BZK_ERR_CUDA (-2)          /* a CUDA call failed; bzk_last_error(ctx) has the text */
#define BZK_ERR_OOM (-3)           /* device or host allocation failed */
#define BZK_ERR_NOT_ON_CURVE (-4)  /* a base failed the curve equation (only when checking is requested) */
#define BZK_ERR_NO_PARAMS (-5)     /* Poseidon parameter table not loaded */
#define BZK_ERR_NO_DEVICE (-6)     /* no CUDA device: the library never falls back to the CPU */
#define BZK_ERR_UNSAT (-7)         /* witness does not satisfy the constraint system */
#define BZK_ERR_BAD_ENCODING (-8)  /* a key file image is truncated or holds a bad flag, a non-canonical coordinate or a point at infinity */
#define BZK_ERR_NOT_IN_SUBGROUP (-9) /* a point is on the curve but not in the prime-order subgroup */
#define BZK_ERR_REJECTED (-10)     /* a proof the prover made failed its own verification (bzk_mpn_worker_prove_response) */

const char *bzk_strerror(int32_t status);
const char *bzk_last_error(const bzk_ctx *ctx);
/* ABI version of this header: (major << 16) | minor */
uint32_t bzk_abi_version(void);

/* ------------------------------------------------------------------ context */
/* Binds to CUDA device `device`, creates the ctx-owned stream and workspace.
 * Fails with BZK_ERR_NO_DEVICE when no GPU is present — there is no CPU path. */
int32_t bzk_ctx_create(int32_t device, bzk_ctx **out);
int32_t bzk_ctx_destroy(bzk_ctx *ctx);
/* Run subsequent work on a caller-owned CUDA stream (a `cudaStream_t` cast to void*, e.g. torch's
 * current stream); NULL restores the ctx-owned stream — to name CUDA's default stream pass
 * cudaStreamLegacy ((cudaStream_t)0x1) or cudaStreamPerThread ((cudaStream_t)0x2). */
int32_t bzk_ctx_set_stream(bzk_ctx *ctx, void *cuda_stream);
int32_t bzk_ctx_synchronize(bzk_ctx *ctx);
/* Per-stage device timing: when on, the MSM driver records CUDA events on the launching stream
 * between its kernels (stage order: 0 digits+histogram, 1 scan, 2 scatter, 3 accumulate, 4 fixup,
 * 5 bucket slices, 6 window sums).  bzk_ctx_stage_ms copies the last call's per-stage milliseconds
 * (up to `cap` floats) and returns how many calls have been timed since timing was switched on. */
int32_t bzk_ctx_set_timing(bzk_ctx *ctx, int32_t on);
uint64_t bzk_ctx_stage_ms(const bzk_ctx *ctx, float *last_ms, double *sum_ms, uint32_t cap);
/* Batched-affine rounds in front of the XYZZ bucket accumulation of G1 / G2 sums (csrc/msm_affine.cuh): each round
 * replaces the entries of every bucket by their pairwise affine sums with one shared inversion.  Results are the same
 * group elements for any value; it is a speed knob (0..6; negative = the library default, currently 0 for both groups —
 * see DESIGN.md for the measurements). */
int32_t bzk_ctx_set_msm_affine_rounds(bzk_ctx *ctx, int32_t g1_rounds, int32_t g2_rounds);
/* Window c of the fixed-base tables that bzk_g*_bases_precompute / bzk_groth16_params_precompute build from now on on this
 * context: 0 lets the planner choose (or the BZK_TABLE_C environment value, read once per process), 8..23 forces it;
 * anything else is BZK_ERR_BAD_ARG.  Results are the same group elements for any window. */
int32_t bzk_ctx_set_msm_table_window(bzk_ctx *ctx, uint32_t c);
/* The plan of the last single MSM run on this context (bzk_msm_g*, bzk_msm_g*_resident[_dev]; not the Groth16 driver's
 * concurrent sums): out = { c, W, T, G, NB, slice, nbits, long_len } — window bits, windows, table levels in use, bucket
 * groups, buckets per group, buckets per reduction slice, bits of the slice index, and the number of bucket runs queued
 * for the CTA-wide fold (read back only while bzk_ctx_set_timing is on, else 0).  W = 0: empty sum or no MSM yet. */
int32_t bzk_ctx_last_msm_plan(const bzk_ctx *ctx, uint32_t out[8]);
/* Points per device chunk buffer of the sums over host-resident vectors (bzk_g*_bases_move) on this context: 0 = the
 * library default (2^22 G1 / 2^21 G2 points, 384 MB per buffer, two buffers per sum), otherwise 256 <= points < 2^31;
 * anything else is BZK_ERR_BAD_ARG.  Results are the same group elements for any chunk. */
int32_t bzk_ctx_set_msm_stream_chunk(bzk_ctx *ctx, uint64_t points);
/* How the last single MSM on this context (as bzk_ctx_last_msm_plan) used its bases: out = { chunks, points per chunk,
 * bytes copied host->device, 1 if it streamed a host-resident vector }; all 0 for a device vector.  A streamed sum records
 * no stage marks (bzk_ctx_stage_ms) and runs no batched-affine rounds whatever bzk_ctx_set_msm_affine_rounds says. */
int32_t bzk_ctx_last_msm_stream(const bzk_ctx *ctx, uint64_t out[4]);
/* kernels launched through this ctx since creation (bench.py's `gpu_launches`) */
uint64_t bzk_ctx_launch_count(const bzk_ctx *ctx);

/* ------------------------------------------------------------------ Poseidon
 * Replaces `poseidon::poseidon(vals)` / `PoseidonHasher::hash`
 *   /root/reference/src/zk/poseidon/mod.rs:81-84 , /root/reference/src/zk/mod.rs:496-511
 * arity 1..16 (state width arity+1, zero capacity lane 0, digest = lane 1). */
/* `blob` = the BZKPOSv1 constant table (bazuka_b200/data/poseidon_params.bin). */
int32_t bzk_poseidon_load_params(bzk_ctx *ctx, const uint8_t *blob, size_t len);
/* host buffers: in[n][arity] -> out[n] */
int32_t bzk_poseidon_hash(bzk_ctx *ctx, uint32_t arity, const bzk_fr *in, size_t n, bzk_fr *out);
/* device buffers (same layout), asynchronous on the ctx stream */
int32_t bzk_poseidon_hash_dev(bzk_ctx *ctx, uint32_t arity, const void *d_in, size_t n, void *d_out);

/* The same hash on the HOST, for the one-at-a-time calls of `impl ZkHasher for PoseidonHasher`
 * (/root/reference/src/zk/mod.rs:491-511: every state-manager read path, transaction hash and calldata check makes single
 * hashes behind a global mutex-guarded LRU): a kernel launch per hash would be slower than the CPU it replaces.
 * `blob` = the same BZKPOSv1 table; the handle is immutable and thread-safe; in/out are Montgomery `ZkScalar` images. */
typedef struct bzk_poseidon_host bzk_poseidon_host;
int32_t bzk_poseidon_host_create(const uint8_t *blob, size_t len, bzk_poseidon_host **out);
int32_t bzk_poseidon_host_free(bzk_poseidon_host *hasher);
int32_t bzk_poseidon_host_hash(const bzk_poseidon_host *hasher, uint32_t arity, const bzk_fr *in, size_t n, bzk_fr *out);

/* 4-ary Poseidon Merkle trees (dense) — the hash structure behind `KvStoreStateManager::{prove,
 * set_data}` (/root/reference/src/zk/state/mod.rs:218-264,310-420) and the merkle gadget
 * (/root/reference/src/zk/groth16/gadgets/merkle/mod.rs:21-65): node = Poseidon-4(children); a proof is,
 * per level from the leaves up, the 3 siblings in ascending child order with self skipped.
 * d_nodes holds level 0 (4^k leaves) | level 1 | ... | root = (4^(k+1)-1)/3 elements.
 *   build : leaves pre-filled, fills every upper level (k batched Poseidon-4 launches)
 *   prove : d_proofs[m][k][3] for m leaf indices (u64)
 *   root  : recompute the root of m (index, leaf, proof) triples (what the witness builder and the
 *           circuit's calc_root do), one thread per path */
int32_t bzk_merkle4_build_dev(bzk_ctx *ctx, void *d_nodes, uint32_t log4_size);
int32_t bzk_merkle4_prove_dev(bzk_ctx *ctx, const void *d_nodes, uint32_t log4_size, const void *d_indices, size_t m, void *d_proofs);
int32_t bzk_merkle4_root_dev(bzk_ctx *ctx, uint32_t log4_size, const void *d_indices, const void *d_leaves, const void *d_proofs, size_t m, void *d_roots);
/* Batch of `n` ordered leaf writes to a forest of sparse 4-ary Poseidon trees, one pass per level instead of
 * one root path per write.  Replaces the transition builders' loop of `KvStoreStateManager::set_data` /
 * `prove` calls (/root/reference/src/zk/state/mod.rs:218-264,310-420; /root/reference/src/mpn/update.rs:40-258).
 *   d_tree_id u32[n], d_indices u64[n]: write e goes to leaf d_indices[e] of tree d_tree_id[e];
 *   d_vals Fr[(depth+1)*n]: in: d_vals[e] = the leaf value written; out: d_vals[l*n + e] = the level-l node on
 *     write e's path after the write (level 0 = leaf, level depth = the tree's root after write e);
 *   d_init_proofs Fr[n][depth][3]: the Merkle proof of each written leaf in the tree BEFORE the batch
 *     (leaf level first, siblings in ascending child order — `prove()`'s layout; read from the store, no hashing);
 *   d_out_proofs Fr[n][depth][3]: the proof of each written leaf just before ITS write, i.e. with every earlier
 *     write of the batch applied — what the sequential loop's `prove` calls would have returned. */
int32_t bzk_tree4_versioned_update_dev(bzk_ctx *ctx, uint32_t depth, const void *d_tree_id, const void *d_indices, size_t n, void *d_vals,
                                       const void *d_init_proofs, void *d_out_proofs);

/* ------------------------------------------------------------------ NTT over Fr
 * Replaces bellman 0.14.0 `domain::EvaluationDomain::{fft, ifft, coset_fft, icoset_fft,
 * divide_by_z_on_coset}` reached from `create_proof` (reference call sites
 * /root/reference/src/mpn/circuits/test.rs:135,175,215).  Natural order in, natural order out,
 * in place; n = 2^log_n, log_n <= 28. */
#define BZK_NTT_FFT 0
#define BZK_NTT_IFFT 1
#define BZK_NTT_COSET_FFT 2
#define BZK_NTT_ICOSET_FFT 3
int32_t bzk_ntt(bzk_ctx *ctx, bzk_fr *data, uint32_t log_n, int32_t op);         /* host buffer */
int32_t bzk_ntt_dev(bzk_ctx *ctx, void *d_data, uint32_t log_n, int32_t op);      /* device buffer, async */
/* d[i] *= (7^n - 1)^-1 */
int32_t bzk_divide_by_z_on_coset_dev(bzk_ctx *ctx, void *d_data, uint32_t log_n);
/* Groth16 quotient: given the A, B, C evaluation vectors (each n = 2^log_n, overwritten), leaves
 * the coefficients of H = (A*B - C)/Z in d_a (bellman prover.rs: 3x ifft, 3x coset_fft, pointwise
 * a*b-c, divide_by_z_on_coset, icoset_fft). */
int32_t bzk_groth16_h_dev(bzk_ctx *ctx, void *d_a, void *d_b, void *d_c, uint32_t log_n);

/* ------------------------------------------------------------------ MSM
 * Replaces bellman 0.14.0 `multiexp::multiexp(pool, (bases, 0), FullDensity, exponents)`
 * (the h / l / a / b_g1 / b_g2 sums of `create_proof`; reference call sites as above).
 * Scalars are Montgomery `bzk_fr` images (the prover's assignment vectors as they sit in memory);
 * the result is the affine sum  sum_i [s_i] P_i  as a wire image. */
int32_t bzk_msm_g1(bzk_ctx *ctx, const bzk_g1_affine *bases, const bzk_fr *scalars, size_t n, bzk_g1_affine *out);
int32_t bzk_msm_g2(bzk_ctx *ctx, const bzk_g2_affine *bases, const bzk_fr *scalars, size_t n, bzk_g2_affine *out);

/* Resident bases (`Parameters<Bls12>` columns stay on the GPU between proofs, as `Arc<Vec<_>>`
 * stays in RAM in the reference).  `check_on_curve` != 0 validates every base. */
int32_t bzk_g1_bases_upload(bzk_ctx *ctx, const bzk_g1_affine *bases, size_t n, int32_t check_on_curve, bzk_g1_bases **out);
int32_t bzk_g2_bases_upload(bzk_ctx *ctx, const bzk_g2_affine *bases, size_t n, int32_t check_on_curve, bzk_g2_bases **out);
/* adopt n wire images already in device memory (104 / 200 B each) */
int32_t bzk_g1_bases_from_dev(bzk_ctx *ctx, const void *d_images, size_t n, bzk_g1_bases **out);
int32_t bzk_g2_bases_from_dev(bzk_ctx *ctx, const void *d_images, size_t n, bzk_g2_bases **out);
int32_t bzk_g1_bases_free(bzk_ctx *ctx, bzk_g1_bases *b);
int32_t bzk_g2_bases_free(bzk_ctx *ctx, bzk_g2_bases *b);
/* Fixed-base table for a resident vector (bases of a proving key never change): grows the vector to up to `max_levels`
 * levels, level t = [2^(c*G*t)] P_i, so that every MSM over it needs only G = ceil(W/levels) bucket groups.  Results are
 * the same group elements; memory grows to levels x n points.  No-op for max_levels <= 1 or an already tabled vector. */
int32_t bzk_g1_bases_precompute(bzk_ctx *ctx, bzk_g1_bases *bases, uint32_t max_levels);
int32_t bzk_g2_bases_precompute(bzk_ctx *ctx, bzk_g2_bases *bases, uint32_t max_levels);
uint32_t bzk_g1_bases_levels(const bzk_g1_bases *bases);
uint32_t bzk_g2_bases_levels(const bzk_g2_bases *bases);
size_t bzk_g1_bases_len(const bzk_g1_bases *b);
size_t bzk_g2_bases_len(const bzk_g2_bases *b);
/* Host-resident vectors, for keys that need not fit in device memory.  move(to_host != 0) puts the vector's points
 * (level 0, packed Montgomery, 96 / 192 B each) in pinned host memory and frees its device storage, tables included;
 * move(0) brings them back as an untabled device vector.  The context's streams, side streams included, are synchronised
 * first; the vector is never held twice on the device.  A failed pinned allocation is BZK_ERR_OOM (the size in
 * bzk_last_error; there is no pageable fallback) and leaves the vector where it was.  Every MSM and prover entry point
 * takes a host vector and streams its points to the device in chunks (bzk_ctx_set_msm_stream_chunk), overlapped with the
 * accumulation, with the same results.  precompute on a host vector is BZK_ERR_BAD_ARG; _len, _levels (1) and _free
 * work in both places.  on_host: 1 when the vector is in host memory, else 0. */
int32_t bzk_g1_bases_move(bzk_ctx *ctx, bzk_g1_bases *b, int32_t to_host);
int32_t bzk_g2_bases_move(bzk_ctx *ctx, bzk_g2_bases *b, int32_t to_host);
int32_t bzk_g1_bases_on_host(const bzk_g1_bases *b);
int32_t bzk_g2_bases_on_host(const bzk_g2_bases *b);
/* sum over bases[offset .. offset+n) with host scalars (copied in) or device scalars */
int32_t bzk_msm_g1_resident(bzk_ctx *ctx, const bzk_g1_bases *b, size_t offset, const bzk_fr *scalars, size_t n, bzk_g1_affine *out);
int32_t bzk_msm_g2_resident(bzk_ctx *ctx, const bzk_g2_bases *b, size_t offset, const bzk_fr *scalars, size_t n, bzk_g2_affine *out);
int32_t bzk_msm_g1_resident_dev(bzk_ctx *ctx, const bzk_g1_bases *b, size_t offset, const void *d_scalars, size_t n, bzk_g1_affine *out);
int32_t bzk_msm_g2_resident_dev(bzk_ctx *ctx, const bzk_g2_bases *b, size_t offset, const void *d_scalars, size_t n, bzk_g2_affine *out);

/* Group helpers on wire images (host arithmetic, used to fold per-GPU partial sums after the
 * all-gather and by tests): out = a + b ; out = [k] a. */
int32_t bzk_g1_add(const bzk_g1_affine *a, const bzk_g1_affine *b, bzk_g1_affine *out);
int32_t bzk_g2_add(const bzk_g2_affine *a, const bzk_g2_affine *b, bzk_g2_affine *out);

/* Synthetic inputs generated on the GPU (bench / tests): P_i = [k_i] G with k_i the SplitMix64(seed)
 * Fr stream of SURVEY.md §8(d); writes n wire images to device memory `d_out`. */
int32_t bzk_g1_random_bases_dev(bzk_ctx *ctx, uint64_t seed, size_t n, void *d_out);
int32_t bzk_g2_random_bases_dev(bzk_ctx *ctx, uint64_t seed, size_t n, void *d_out);
/* n uniform Fr (Montgomery) from SplitMix64(seed), same stream rule */
int32_t bzk_fr_random_dev(bzk_ctx *ctx, uint64_t seed, size_t n, void *d_out);

/* ------------------------------------------------------------------ Groth16 prover
 * Replaces bellman 0.14.0 `groth16::create_proof(circuit, &params, r, s)` — reference call sites
 * /root/reference/src/mpn/circuits/test.rs:135,175,215 (`create_random_proof`), gadget tests, and in
 * production the external prover behind `MpnWork` (/root/reference/src/mpn/mod.rs:264-295).
 *
 * The circuit arrives as its R1CS in CSR form (what `Circuit::synthesize` emits into bellman's
 * `ProvingAssignment`), one matrix per side: rowptr[num_constraints+1], col[nnz] = index into
 * z = inputs ++ aux (z[0] = ONE), val[nnz] = Montgomery coefficients.  Like bellman, the library
 * appends the `Input(i) * 0 = 0` rows itself and derives the A/B density lists from the non-zero
 * coefficients.  Parameters are bellman's `Parameters<Bls12>` vectors: h (m-1), l (num_aux),
 * a (num_inputs + |A aux density|), b_g1 / b_g2 (|B input density| + |B aux density|), in
 * bellman's order (inputs first), identity entries already filtered out.
 * A term counts as present when its coefficient image is not all-zero limbs, so every coefficient must be canonical
 * (< r, as bellman's Fr holds it): an image >= r is BZK_ERR_BAD_ARG before anything is allocated.  Otherwise r itself
 * would be a present zero, and its variable would get an identity column that a key file may not hold. */
typedef struct bzk_r1cs bzk_r1cs;
typedef struct bzk_groth16_params bzk_groth16_params;
int32_t bzk_r1cs_upload(bzk_ctx *ctx, uint64_t num_inputs, uint64_t num_aux, uint64_t num_constraints,
                        const uint64_t *a_rowptr, const uint32_t *a_col, const bzk_fr *a_val,
                        const uint64_t *b_rowptr, const uint32_t *b_col, const bzk_fr *b_val,
                        const uint64_t *c_rowptr, const uint32_t *c_col, const bzk_fr *c_val, bzk_r1cs **out);
int32_t bzk_r1cs_free(bzk_ctx *ctx, bzk_r1cs *r1cs);
/* out = { log2 m, |h| = m-1, |l|, |a|, |b_g1| = |b_g2| } the parameter vectors must have */
int32_t bzk_r1cs_shape(const bzk_r1cs *r1cs, uint64_t out[5]);
/* A blocked R1CS: a circuit whose middle is one block of rows repeated `reps` times, held once.  Logical rows, in order:
 * head_rows explicit rows, reps copies of the tmpl_rows template rows, tail_rows explicit rows; each side's CSR
 * (rowptr[head_rows + tmpl_rows + tail_rows + 1], col, val) stores head | template | tail.  Head and tail columns are z
 * indices.  A template column c >= var_lo names c + k * var_stride in copy k (0-based); a template column c < var_lo
 * names c in every copy.  An MPN update batch is head = prologue + slot 0, template = slot 1, reps = n - 1, var_lo =
 * num_inputs + the prologue's aux count, var_stride = one slot's variables, tail = epilogue (bzk_mpn_circuit_blocks).
 * The handle is an ordinary bzk_r1cs for bzk_r1cs_shape / _free and every prover entry point, with the density lists
 * bzk_r1cs_upload would derive from the expanded matrices.  BZK_ERR_BAD_ARG, before anything is allocated: a rowptr
 * that does not start at 0 or decreases, a missing array, an expanded column (the last copy's included) >= num_inputs +
 * num_aux, num_inputs + num_aux > 2^32, var_stride = 0 with reps > 0, or a coefficient image >= r (as bzk_r1cs_upload). */
int32_t bzk_r1cs_upload_blocked(bzk_ctx *ctx, uint64_t num_inputs, uint64_t num_aux, uint64_t head_rows, uint64_t tmpl_rows, uint64_t reps,
                                uint64_t tail_rows, uint64_t var_lo, uint64_t var_stride, const uint64_t *const rowptr[3], const uint32_t *const col[3],
                                const bzk_fr *const val[3], bzk_r1cs **out);
/* The transposed product the trusted setup needs: d_out[j] = sum_row M_side[row][j] * d_lag[row] for every variable j
 * (side 0, 1, 2 = A, B, C; d_lag has one entry per logical row, d_out num_inputs + num_aux), on the context's stream,
 * without atomics.  Blocked handles only: BZK_ERR_BAD_ARG for an explicit one. */
int32_t bzk_r1cs_columns_dev(bzk_ctx *ctx, const bzk_r1cs *r1cs, uint32_t side, const void *d_lag, void *d_out);
/* adopts the five resident base vectors (freed with the handle) plus the vk points the tail needs */
int32_t bzk_groth16_params_create(bzk_ctx *ctx, const bzk_g1_affine *alpha_g1, const bzk_g1_affine *beta_g1, const bzk_g2_affine *beta_g2,
                                  const bzk_g1_affine *delta_g1, const bzk_g2_affine *delta_g2,
                                  bzk_g1_bases *h, bzk_g1_bases *l, bzk_g1_bases *a, bzk_g1_bases *b_g1, bzk_g2_bases *b_g2,
                                  bzk_groth16_params **out);
int32_t bzk_groth16_params_free(bzk_ctx *ctx, bzk_groth16_params *params);
/* What a key handle holds, each output optional: lens = the lengths of its five vectors {h, l, a, b_g1, b_g2} (a shard's: its
 * slices), and the verifying-key points the proof tail uses, as wire images.  Host only, no device access. */
int32_t bzk_groth16_params_info(const bzk_groth16_params *params, uint64_t lens[5], bzk_g1_affine *alpha_g1, bzk_g1_affine *beta_g1,
                                bzk_g2_affine *beta_g2, bzk_g1_affine *delta_g1, bzk_g2_affine *delta_g2);
/* inputs[num_inputs] (inputs[0] = ONE), aux[num_aux], r, s: host Montgomery images.  With
 * check_satisfied != 0 returns BZK_ERR_UNSAT when a*b != c on some constraint (bellman proves
 * garbage silently).  Outputs are the wire images of Proof {a, b, c}. */
int32_t bzk_groth16_prove(bzk_ctx *ctx, const bzk_groth16_params *params, const bzk_r1cs *r1cs,
                          const bzk_fr *inputs, const bzk_fr *aux, const bzk_fr *r, const bzk_fr *s, int32_t check_satisfied,
                          bzk_g1_affine *proof_a, bzk_g2_affine *proof_b, bzk_g1_affine *proof_c);
/* Same prover with the witness already in device memory (Montgomery images; written e.g. by
 * bzk_witness_run_dev): d_inputs[num_inputs], d_aux[num_aux].  Work queued on the context's stream before
 * the call (the witness kernels) is ordered before the prover's reads. */
int32_t bzk_groth16_prove_dev(bzk_ctx *ctx, const bzk_groth16_params *params, const bzk_r1cs *r1cs,
                              const void *d_inputs, const void *d_aux, const bzk_fr *r, const bzk_fr *s, int32_t check_satisfied,
                              bzk_g1_affine *proof_a, bzk_g2_affine *proof_b, bzk_g1_affine *proof_c);

/* Fixed-base tables for the five base vectors of a key; max_levels = 0: as many levels (<= 16) as fit in
 * mem_fraction_percent % (0 = 50) of the free device memory.  See bzk_g1_bases_precompute.  Host-resident vectors are
 * left untabled. */
int32_t bzk_groth16_params_precompute(bzk_ctx *ctx, bzk_groth16_params *params, uint32_t max_levels, uint32_t mem_fraction_percent);
/* Places each of the key's five vectors: bit v of host_mask (order h, l, a, b_g1, b_g2) set = pinned host memory, clear =
 * device memory (bzk_g1_bases_move; the moves to the host run first).  host_mask > 31 is BZK_ERR_BAD_ARG.  A key may mix
 * both; every prover entry point gives the same proofs for any placement. */
int32_t bzk_groth16_params_move(bzk_ctx *ctx, bzk_groth16_params *params, uint32_t host_mask);

/* Proving keys as bellman 0.14 keeps them on disk: the image `Parameters::write` makes and `Parameters::read` takes
 * (layout in csrc/params_io.cu).  Points stream through two fixed staging chunks into the key's resident vectors, so
 * device memory beyond the key is two chunks; every point is decoded and, when checked, tested on the GPU.
 *   file_info  host only, no context: the lengths the image states and the byte count they imply (`bytes` may be less
 *              than len: nothing after b_g2 is read); BZK_ERR_BAD_ENCODING when the image is shorter than that.
 *   read       checked != 0: `Parameters::read(.., true)` (curve equation and prime-order subgroup for every point),
 *              0: `read(.., false)`; the verifying key is checked either way.  The vk points come out as wire images
 *              (ic[ic_cap], ic_cap >= n_ic) and the key as a handle like bzk_groth16_params_create makes (tables:
 *              bzk_groth16_params_precompute afterwards).  On a refusal bzk_last_error names the first bad point in file
 *              order ("l[65536]: not in the prime-order subgroup"): BZK_ERR_BAD_ENCODING (also |b_g1| != |b_g2|),
 *              BZK_ERR_NOT_ON_CURVE or BZK_ERR_NOT_IN_SUBGROUP; nothing stays allocated.
 *   write      the key's file image, level 0 of each vector whatever its table levels; out == NULL: *len = size only.
 *              gamma_g2 and ic are not held by the handle.  A shard (set_shard, world > 1) is BZK_ERR_BAD_ARG. */
typedef struct { uint64_t n_ic, n_h, n_l, n_a, n_b_g1, n_b_g2, bytes; } bzk_params_file_info;
int32_t bzk_groth16_params_file_info(const uint8_t *bytes, size_t len, bzk_params_file_info *out);
int32_t bzk_groth16_params_read(bzk_ctx *ctx, const uint8_t *bytes, size_t len, int32_t checked,
                                bzk_g1_affine *alpha_g1, bzk_g1_affine *beta_g1, bzk_g2_affine *beta_g2, bzk_g2_affine *gamma_g2,
                                bzk_g1_affine *delta_g1, bzk_g2_affine *delta_g2, bzk_g1_affine *ic, size_t ic_cap,
                                bzk_groth16_params **out);
/*   read_placed  read with each vector placed where host_mask says: bit v (order h, l, a, b_g1, b_g2) set = the vector
 *              goes to pinned host memory (bzk_g1_bases_move) through a device landing chunk, so a key larger than the
 *              device can be read, checked; device memory is then the staging chunks and the device-placed vectors.
 *              host_mask > 31 is BZK_ERR_BAD_ARG.  Refusals as for read; nothing stays allocated, pinned memory
 *              included.  read is read_placed with host_mask = 0.  write takes host vectors too. */
int32_t bzk_groth16_params_read_placed(bzk_ctx *ctx, const uint8_t *bytes, size_t len, int32_t checked,
                                       bzk_g1_affine *alpha_g1, bzk_g1_affine *beta_g1, bzk_g2_affine *beta_g2, bzk_g2_affine *gamma_g2,
                                       bzk_g1_affine *delta_g1, bzk_g2_affine *delta_g2, bzk_g1_affine *ic, size_t ic_cap,
                                       uint32_t host_mask, bzk_groth16_params **out);
int32_t bzk_groth16_params_write(bzk_ctx *ctx, const bzk_groth16_params *params, const bzk_g2_affine *gamma_g2,
                                 const bzk_g1_affine *ic, size_t n_ic, uint8_t *out, size_t cap, size_t *len);

/* Stage times of the last prove call made while bzk_ctx_set_timing was on (CUDA events): milliseconds after the start
 * of the call at which [1] z upload + the three SpMVs finished, [2] the quotient pipeline (7 NTTs), [3] the h sum (main
 * stream), [4..7] the l / a / b_g1 / b_g2 sums (side streams, concurrent with the main one).  Returns 1 when valid. */
int32_t bzk_groth16_stage_ms(const bzk_ctx *ctx, float out[8]);

/* Base-sharded proving over several GPUs (one process / context per GPU): every MSM of bellman's
 * `create_proof` is a sum over terms, so rank k of `world` keeps only the contiguous range
 * [len*k/world, len*(k+1)/world) of each of the five base vectors (pass those slices to
 * bzk_groth16_params_create, then set_shard), computes the witness-side pipeline on its own GPU, and
 * returns its four partial sums (a; b_g1; b_g2; h + l).  The caller exchanges world x 512 B (one
 * all-gather), adds the partials (bzk_g1_add / bzk_g2_add) and calls bzk_groth16_finalize — host arithmetic,
 * no context — which is the tail of `create_proof` (g_a, g_b, g_c from r, s and the verifying-key points). */
int32_t bzk_groth16_params_set_shard(bzk_groth16_params *params, uint32_t rank, uint32_t world);
int32_t bzk_groth16_prove_partial(bzk_ctx *ctx, const bzk_groth16_params *params, const bzk_r1cs *r1cs, const void *inputs, const void *aux,
                                  int32_t witness_on_device, int32_t check_satisfied,
                                  bzk_g1_affine *a_sum, bzk_g1_affine *b1_sum, bzk_g2_affine *b2_sum, bzk_g1_affine *hl_sum);
/* The same schedule with the quotient pipeline split over the ranks as well (every rank would otherwise repeat the three
 * SpMVs and seven NTTs, the part of a proof that does not shrink with `world`): evaluation vector s (0 = a, 1 = b, 2 = c) is
 * owned by rank s mod world, which computes it from z and takes it to the coset (ifft, coset_fft); the owners send their
 * vectors to rank 3 mod world, which forms (a*b - c)/Z and the quotient's coefficients (bzk_groth16_h_combine_dev: a <- h) and
 * hands rank k the slice [(m-1)k/world, (m-1)(k+1)/world) of them.  The transport between GPUs is the caller's
 * (bazuka_b200.groth16.SplitShardedProver uses NCCL point-to-point through torch.distributed).
 *   bzk_groth16_shard_begin   z, the vectors in poly_mask into the caller's device buffers d_evals[s] (2^log_m scalars each),
 *                             and the l / a / b_g1 / b_g2 partial sums enqueued — they keep the GPU busy during the exchange
 *   bzk_groth16_shard_finish  the h partial sum over d_h_shard, then the four partial sums of bzk_groth16_prove_partial */
int32_t bzk_groth16_shard_begin(bzk_ctx *ctx, const bzk_groth16_params *params, const bzk_r1cs *r1cs, const void *inputs, const void *aux,
                                int32_t witness_on_device, uint32_t poly_mask, void *d_evals[3]);
int32_t bzk_groth16_h_combine_dev(bzk_ctx *ctx, void *d_a, void *d_b, void *d_c, uint32_t log_n);
int32_t bzk_groth16_shard_finish(bzk_ctx *ctx, const bzk_groth16_params *params, const bzk_r1cs *r1cs, const void *d_h_shard,
                                 bzk_g1_affine *a_sum, bzk_g1_affine *b1_sum, bzk_g2_affine *b2_sum, bzk_g1_affine *hl_sum);
int32_t bzk_groth16_finalize(const bzk_g1_affine *alpha_g1, const bzk_g1_affine *beta_g1, const bzk_g2_affine *beta_g2,
                             const bzk_g1_affine *delta_g1, const bzk_g2_affine *delta_g2,
                             const bzk_g1_affine *a_sum, const bzk_g1_affine *b1_sum, const bzk_g2_affine *b2_sum, const bzk_g1_affine *hl_sum,
                             const bzk_fr *r, const bzk_fr *s, bzk_g1_affine *proof_a, bzk_g2_affine *proof_b, bzk_g1_affine *proof_c);

/* ------------------------------------------------------------------ MPN ledger + update transition builder
 * Native host logic of `mpn::update::update` (/root/reference/src/mpn/update.rs:8-299) over the state model of
 * /root/reference/src/mpn/mod.rs:219-240 (accounts with a token sub-tree in a 4-ary sparse Poseidon tree): ledger
 * decisions first (no hashing), then all hashing in batches on the GPU (bzk_poseidon_hash + the versioned tree
 * update).  Scalars are CANONICAL 32-byte little-endian integers here (amounts and nonces are u64, as in the
 * reference).  bzk_mpn_update_build consumes up to 4^log4_batch acceptable transactions in order and writes
 *   raws[4^B][n_raw]  each slot's circuit inputs in UpdateCircuit's allocation order (n_raw = 32 + 9T + 6A,
 *                     bzk_mpn_update_raw_width) — the RAW operands of the witness program; null slots padded,
 *   ext[4^B][2]       {fee token, state root entering the slot} — the program's external slots,
 *   accepted[n_txs]   1 where the transaction was taken (rejected or beyond the batch: 0), optional,
 *   public3           {state before, aux_data = Poseidon(fee_token, fee sum), state after},
 * and advances the ledger.  BZK_ERR_NOT_ON_CURVE: a compressed key does not decompress. */
typedef struct bzk_mpn_state bzk_mpn_state;
typedef struct {
    uint64_t nonce, amount, fee;
    uint8_t src_pk_odd, dst_pk_odd, pad[6];
    bzk_fr src_pk_x, dst_pk_x;              /* PointCompressed(x, is_odd) of the two JubJub keys */
    bzk_fr amount_token_id, fee_token_id;
    bzk_fr sig_rx, sig_ry, sig_s;           /* EdDSA signature (checked in the circuit, not by the builder) */
} bzk_mpn_tx;
int32_t bzk_mpn_state_create(bzk_ctx *ctx, uint32_t log4_tree, uint32_t log4_token, const bzk_fr *jubjub_d, bzk_mpn_state **out);
int32_t bzk_mpn_state_free(bzk_mpn_state *state);
int32_t bzk_mpn_state_root(const bzk_mpn_state *state, bzk_fr *root);
int32_t bzk_mpn_state_set_account(bzk_ctx *ctx, bzk_mpn_state *state, uint64_t index, uint64_t tx_nonce, uint64_t withdraw_nonce,
                                  const bzk_fr *addr_x, const bzk_fr *addr_y, const uint32_t *token_index, const bzk_fr *token_id,
                                  const uint64_t *token_amount, uint32_t n_tokens);
int32_t bzk_mpn_update_raw_width(uint32_t log4_tree, uint32_t log4_token, uint32_t *n_raw);
/* Fork / introspection / block application for the ledger.  bzk_mpn_update_build WRITES the ledger it is given (state
 * tree, accounts, the fork's new-account map) before any proof exists: build a block's batches on a clone
 * (`db.fork_on_ram()`, /root/reference/src/mpn/mod.rs:313) and keep the clone only if the block is accepted; after a
 * failed proof or a reorg, drop it.  `info`: the `ZkCompressedState {state_hash, state_size}` that goes into
 * `MpnWork::new_root`, the chain's account count and the number of accounts created on this fork so far.
 * `commit_accounts`: the block was applied — the fork's new accounts enter the chain's address index
 * (`get_mpn_account_indices`), exactly what the builders consult first (/root/reference/src/mpn/update.rs:47-70). */
int32_t bzk_mpn_state_clone(const bzk_mpn_state *state, bzk_mpn_state **out);
int32_t bzk_mpn_state_info(const bzk_mpn_state *state, bzk_fr *state_hash, uint64_t *state_size, uint64_t *account_count, uint64_t *pending_accounts);
int32_t bzk_mpn_state_commit_accounts(bzk_mpn_state *state);
int32_t bzk_mpn_state_shape(const bzk_mpn_state *state, uint32_t out[2]);   /* {log4_tree, log4_token} */
/* `MpnWorkPool.final_delta` (/root/reference/src/mpn/mod.rs:17-45,416-417): the scalar leaves in which `after` (the fork
 * bzk_mpn_prepare_works returned) differs from `before`, as the bincode of `ZkDeltaPairs` = HashMap<ZkDataLocator(Vec<u64>),
 * Option<ZkScalar>>: [account, field] for the four account scalars, [account, 4, token slot, 0 | 1] for a token's id / balance;
 * a leaf that became zero is None.  Ascending locator order; release with bzk_buffer_free. */
int32_t bzk_mpn_state_delta(const bzk_mpn_state *before, const bzk_mpn_state *after, uint8_t **bytes, size_t *len, uint64_t *n_entries);
/* A block's MPN state delta applied to the ledger, as a full node does for every block (`update_contract` with
 * `index_mpn_accounts`, /root/reference/src/blockchain/ops/apply_tx/update_contract/mod.rs:130-144).
 *   delta        the bincode of ZkDeltaPairs, the image bzk_mpn_state_delta writes; None = the leaf becomes zero
 *                (`v.unwrap_or_default()`, /root/reference/src/zk/state/mod.rs:285-308).  Locators [i, f] (f < 4) and
 *                [i, 4, slot, 0 | 1] with i < 4^log4_tree, slot < 4^log4_token.  The result does not depend on entry order.
 *   indexing     (/root/reference/src/blockchain/ops/apply_tx/mod.rs:14-56) every index whose x and y are both in the delta
 *                records its (x, y); an address keeps its smallest index; indices equal to the account count advance it in
 *                ascending order.  An index above the count, or x without y (or y without x), is refused.
 *   expect_hash  canonical; with expect_size, the ZkCompressedState the block attested (update_contract/mod.rs:139-144); NULL:
 *                no check.
 *   n_entries    optional: the number of entries applied.
 * All hashing runs on the context's stream as one launch per tree level and one copy back.  All or nothing: on any refusal
 * or error the ledger is unchanged and bzk_last_error(ctx) says why.  BZK_ERR_BAD_ARG refuses a truncated image, trailing
 * bytes, an option tag other than 0 / 1, a duplicate locator, a locator outside the MPN state model, a non-canonical scalar,
 * a value the account model cannot hold (nonce or balance >= 2^64, a balance under token id zero), an indexing
 * inconsistency, a root or size other than expected, and a ledger holding a prepare_works fork's new accounts (apply to the
 * chain's ledger, not to a fork).  A snapshot is a delta too: bzk_mpn_state_delta(empty ledger, ledger) applied to a fresh
 * ledger rebuilds it. */
int32_t bzk_mpn_state_apply_delta(bzk_ctx *ctx, bzk_mpn_state *state, const uint8_t *delta, size_t len, const bzk_fr *expect_hash,
                                  const uint64_t *expect_size, uint64_t *n_entries);
/* Deposit and withdraw batches natively (`mpn::deposit::deposit`, /root/reference/src/mpn/deposit.rs:11-233; `mpn::withdraw::withdraw`,
 * /root/reference/src/mpn/withdraw.rs:10-259), next to the update builder: the same ledger, the same batched GPU hashing,
 * rows of circuit inputs out.  `bzk_mpn_deposit` / `bzk_mpn_withdraw` carry what the circuits consume of `MpnDeposit` /
 * `MpnWithdraw` (scalars canonical little-endian; `fingerprint` = `ContractWithdraw::fingerprint()` of the L1 payment).  The
 * withdraw builder checks nonces, balances and the EdDSA signature; neither touches L1 balances (chain state).
 *   raws1 / raws2   phase-1 / phase-2 inputs of every slot (widths 5 and 9+3T+3A for deposits, 12 and 12+6T+3A for withdrawals)
 *   roots[slots]    the state root entering each slot (phase 2's external)
 *   reveal          the rows the circuit reveals (4 / 7 per slot); public3 = {state, aux_data = their list root, next_state}
 * bzk_mpn_dw_witness then runs the three programs of bzk_mpn_dw_circuit_compile (phase 1, reveal, phase 2) into z. */
typedef struct {
    bzk_fr pk_x;
    uint8_t pk_odd, pad[7];
    bzk_fr token_id;
    uint64_t amount;
    uint64_t src_id;   /* caller's id of `payment.src`, the paying L1 account (0 = not tracked): after one rejected deposit the
                        * later deposits of the same source in the call are rejected too (deposit.rs:33,68-83) */
} bzk_mpn_deposit;
typedef struct {
    bzk_fr pk_x;
    uint8_t pk_odd, check_calldata, pad[2];   /* check_calldata: `calldata` below is the payment's and must equal
                                               * Poseidon(pk.x, pk.y, nonce, sig.r.x, sig.r.y, sig.s) (`verify_calldata`) */
    uint32_t nonce;
    bzk_fr sig_rx, sig_ry, sig_s;
    bzk_fr amount_token_id, fee_token_id, fingerprint;
    uint64_t amount, fee;
    bzk_fr calldata;
} bzk_mpn_withdraw;
int32_t bzk_mpn_deposit_build(bzk_ctx *ctx, bzk_mpn_state *state, const bzk_mpn_deposit *deposits, uint64_t n, uint32_t log4_batch, bzk_fr *raws1,
                              bzk_fr *raws2, bzk_fr *roots, bzk_fr *reveal, uint8_t *accepted, bzk_fr public3[3], uint64_t *n_accepted);
int32_t bzk_mpn_withdraw_build(bzk_ctx *ctx, bzk_mpn_state *state, const bzk_mpn_withdraw *withdraws, uint64_t n, uint32_t log4_batch, bzk_fr *raws1,
                               bzk_fr *raws2, bzk_fr *roots, bzk_fr *reveal, uint8_t *accepted, bzk_fr public3[3], uint64_t *n_accepted);
typedef struct bzk_witness_program bzk_witness_program;
int32_t bzk_mpn_dw_witness(bzk_ctx *ctx, const bzk_witness_program *phase1, const bzk_witness_program *phase2, const bzk_witness_program *reveal_prog,
                           uint64_t n_slots, const bzk_fr *raws1, const bzk_fr *raws2, const bzk_fr *roots, const int32_t *ext_src, uint32_t n_ext_src,
                           const bzk_fr *reveal_rows, const bzk_fr public5[5], void *d_inputs, void *d_aux);
/* `PublicKey::decompress` (/root/reference/src/crypto/jubjub/curve.rs:78-88) on the host field arithmetic, no
 * context: y = sqrt((1 + x^2) / (1 - d x^2)) with the parity rule; canonical scalars. */
int32_t bzk_jubjub_decompress(const bzk_fr *jubjub_d, const bzk_fr *x, int32_t y_is_odd, bzk_fr out_xy[2]);
/* `JubJub::verify` (/root/reference/src/crypto/jubjub/mod.rs:151-167) on the host (no context): h = Poseidon(R.x, R.y, A.x, A.y,
 * message), accept iff h*A + R == s*BASE and A, R are on the curve.  Canonical scalars; returns 1 / 0, negative on bad arguments. */
int32_t bzk_jubjub_eddsa_verify(const bzk_poseidon_host *hasher, const bzk_fr *jubjub_d, const bzk_fr pk_xy[2], const bzk_fr *message,
                                const bzk_fr sig_r_xy[2], const bzk_fr *sig_s);
/* ------------------------------------------------------------------ EdDSA signature checks in batches (device)
 * `JubJub::verify` on many signatures at once, one thread per signature: the key decompressed as `PointCompressed::decompress`
 * does, A and R on the curve, h = Poseidon(R.x, R.y, A.x, A.y, msg), accept iff [h] A + R == [s] BASE as points of the full
 * curve group (h and s as plain integers below r: no reduction modulo the prime order, no cofactor clearing).  A scalar that
 * is not canonical, or a key that does not decompress (where the reference panics), gives 0.
 *   bzk_jubjub_eddsa_verify_batch  the message as given (canonical scalars in every field)
 *   bzk_mpn_tx_verify_batch        `MpnTransaction::verify_signature`: msg = Poseidon(nonce, D.x, D.y, amount token, amount, fee token,
 *                                  fee), D the decompressed destination key (0 where it does not decompress)
 *   bzk_mpn_signatures_verify_bytes  the bincode of Vec<MpnWithdraw> (kind 1: `MpnWithdraw::verify_signature`,
 *                                  msg = Poseidon(fingerprint(payment), nonce)) or Vec<MpnTransaction> (kind 2), the images
 *                                  bzk_mpn_prepare_works takes; ok == NULL: only *n (the item count); cap < *n: BZK_ERR_BAD_ARG
 * ok[i] = 1 (accept) or 0 (reject); n_ok (optional) = the number accepted.  A rejected signature is a verdict: the call returns
 * BZK_OK.  BZK_ERR_BAD_ARG (nothing written to ok): a null pointer with n > 0, jubjub_d not canonical, kind 0 or above 2, a
 * malformed image (truncated, trailing bytes, a bad tag, an unreduced scalar).  BZK_ERR_NO_PARAMS: the context has no Poseidon
 * table.  Synchronous on the context's stream.  Items go through the context's arenas 2^18 at a time, so device memory stays
 * bounded for any n; the context keeps a fixed-base table of BASE (786 KB) for the last jubjub_d it was given. */
typedef struct {
    bzk_fr pk_x;
    uint8_t pk_odd, pad[7];   /* PublicKey = PointCompressed(pk_x, pk_odd) */
    bzk_fr message, sig_rx, sig_ry, sig_s;
} bzk_eddsa_item;             /* 168 B, canonical scalars */
int32_t bzk_jubjub_eddsa_verify_batch(bzk_ctx *ctx, const bzk_fr *jubjub_d, const bzk_eddsa_item *items, size_t n, uint8_t *ok, uint64_t *n_ok);
int32_t bzk_mpn_tx_verify_batch(bzk_ctx *ctx, const bzk_fr *jubjub_d, const bzk_mpn_tx *txs, size_t n, uint8_t *ok, uint64_t *n_ok);
int32_t bzk_mpn_signatures_verify_bytes(bzk_ctx *ctx, const bzk_fr *jubjub_d, uint32_t kind, const uint8_t *bytes, size_t len, uint8_t *ok,
                                        size_t cap, uint64_t *n, uint64_t *n_ok);
/* ------------------------------------------------------------------ Ed25519 signature checks (L1: deposits, transactions)
 * `Ed25519::verify` (src/crypto/ed25519.rs:81-83): ed25519-dalek 1.x `PublicKey::verify`, the non-strict, cofactorless check.
 * For pk (32 B), sig = R || s (64 B) and message M the verdict is 1 iff
 *   s (little-endian) < l = 2^252 + 27742317777372353535851937790883648493 (s is never reduced; bit 255 set gives 0);
 *   pk decompresses as curve25519-dalek 3.x does: y = the low 255 bits taken mod p (non-canonical y accepted), x =
 *     sqrt_ratio_i(y^2 - 1, d y^2 + 1) exists, the non-negative root negated when bit 255 is set ("-0" accepted); small-order
 *     and mixed-order keys are accepted;
 *   k = SHA-512(R || pk || M) as a 512-bit little-endian integer mod l;
 *   compress([k](-A) + [s]B) == R byte for byte, in the full group (no cofactor): a non-canonical, off-curve or "-0" R gives 0.
 *   bzk_ed25519_verify              one signature on the host, no context: 1 accept, 0 reject, < 0 bad argument (pk or sig
 *                                   NULL, msg NULL with len > 0)
 *   bzk_ed25519_verify_batch        on the GPU, one thread per signature: pks n x 32 B, sigs n x 64 B, message i =
 *                                   msgs[offsets[i] .. offsets[i+1]) with n + 1 offsets, offsets[0] = 0, non-decreasing (msgs
 *                                   may be NULL when offsets[n] = 0).  The TransactionAndDelta arm: M = bincode(sig_state_excluded()),
 *                                   src/core/transaction.rs:386-397
 *   bzk_mpn_deposits_verify_bytes   `ContractDeposit::verify_signature` (src/core/transaction.rs:192-201) of each payment of a
 *                                   bincode Vec<MpnDeposit>, the image bzk_mpn_prepare_works takes: M = bincode(payment with sig
 *                                   = None); 0 where sig is None or not 64 bytes.  ok == NULL: only *n (the item count); cap < *n:
 *                                   BZK_ERR_BAD_ARG
 * ok[i] = 1 (accept) or 0 (reject); n_ok (optional) = the number accepted.  A rejected signature is a verdict: the call returns
 * BZK_OK.  BZK_ERR_BAD_ARG (nothing written to ok): a null pointer with n > 0, bad offsets, a malformed image.  Synchronous on
 * the context's stream.  Items go through the context's arena at most 2^18 items and 64 MiB of messages at a time (a longer
 * single message goes alone), so device memory stays bounded for any batch; the context keeps a fixed-base table of B
 * (786 KB), built on first use. */
int32_t bzk_ed25519_verify(const uint8_t pk[32], const uint8_t *msg, size_t len, const uint8_t sig[64]);
int32_t bzk_ed25519_verify_batch(bzk_ctx *ctx, const uint8_t *pks, const uint8_t *sigs, const uint8_t *msgs, const uint64_t *offsets, size_t n,
                                 uint8_t *ok, uint64_t *n_ok);
int32_t bzk_mpn_deposits_verify_bytes(bzk_ctx *ctx, const uint8_t *bytes, size_t len, uint8_t *ok, size_t cap, uint64_t *n, uint64_t *n_ok);
int32_t bzk_mpn_update_build(bzk_ctx *ctx, bzk_mpn_state *state, const bzk_mpn_tx *txs, uint64_t n_txs, uint32_t log4_batch,
                             const bzk_fr *fee_token, bzk_fr *raws, bzk_fr *ext, uint8_t *accepted, bzk_fr public3[3],
                             uint64_t *n_accepted);

/* Whole-batch witness from the builder's rows, resident in device memory as z = d_inputs[6] ++ d_aux
 * (6 + n_slots*slot_vars + epilogue_vars elements): the six public / prologue values
 * prologue[6] = {commitment, height, state, fee_token, aux_data, next_state} (canonical), the slot program on
 * every slot, and the epilogue program (the fee-commitment Poseidon gadget; its externals are the fee token and
 * every slot's accepted fee, taken from the rows).  Feeds bzk_groth16_prove_dev directly. */
typedef struct bzk_witness_program bzk_witness_program;
int32_t bzk_mpn_update_witness(bzk_ctx *ctx, const bzk_witness_program *slot_prog, const bzk_witness_program *epilogue_prog,
                               uint64_t n_slots, uint32_t log4_token, uint64_t slot_vars, uint64_t epilogue_vars, const bzk_fr *raws,
                               const bzk_fr *ext, uint32_t n_raw, const bzk_fr prologue[6], void *d_inputs, void *d_aux);

/* ------------------------------------------------------------------ MPN update circuit, compiled natively
 * Structure-only synthesis (bellman's `KeypairAssembly` role) of `UpdateCircuit`
 * (/root/reference/src/mpn/circuits/update_circuit.rs:49-494) over the reference's gadgets and bellman's
 * AllocatedNum / AllocatedBit / Boolean / to_bits_le_strict, in C++: emits the R1CS of a 4^log4_batch-slot batch
 * (arrays for bzk_r1cs_upload) and the slot / epilogue witness programs (arrays for bzk_witness_program_upload).
 * poseidon_blob = the table bzk_poseidon_load_params takes; jubjub = {d, 8*BASE.x, 8*BASE.y}, canonical.  No GPU. */
typedef struct bzk_mpn_circuit bzk_mpn_circuit;
int32_t bzk_mpn_update_circuit_compile(uint32_t log4_tree, uint32_t log4_token, uint32_t log4_batch, const uint8_t *poseidon_blob,
                                       size_t blob_len, const bzk_fr jubjub[3], bzk_mpn_circuit **out);
/* DepositCircuit (kind 1) / WithdrawCircuit (kind 2) (/root/reference/src/mpn/circuits/{deposit,withdraw}_circuit.rs):
 * these walk the batch twice around the `reveal` of the batch root, so there are two slot programs — program 0 =
 * phase 1, program 1 = phase 2 (externals described by bzk_mpn_circuit_two_phase_info) — and the batch's aux layout is
 * [5 public-input copies][phase 1 x n][reveal][phase 2 x n].  In `shape`: slot_vars = phase-1 variables per slot,
 * epilogue_vars = phase-2 variables per slot, last entry = reveal variables. */
int32_t bzk_mpn_dw_circuit_compile(uint32_t kind, uint32_t log4_tree, uint32_t log4_token, uint32_t log4_batch, const uint8_t *poseidon_blob,
                                   size_t blob_len, const bzk_fr jubjub[3], bzk_mpn_circuit **out);
int32_t bzk_mpn_circuit_two_phase_info(const bzk_mpn_circuit *circuit, uint64_t counts[2], int32_t *row_local, int32_t *ext_src);
int32_t bzk_mpn_circuit_free(bzk_mpn_circuit *circuit);
/* out[4] = {kind: 0 UpdateCircuit, 1 DepositCircuit, 2 WithdrawCircuit; log4_tree; log4_token; log4_batch} */
int32_t bzk_mpn_circuit_kind(const bzk_mpn_circuit *circuit, uint32_t out[4]);
/* shape = {num_inputs, num_aux, num_constraints, nnz_a, nnz_b, nnz_c, prologue_aux, slot_vars, state_out (slot-local),
 *          final_fee (slot-local), epilogue_vars, reveal_vars (two-phase circuits; 0 for the update circuit)} */
int32_t bzk_mpn_circuit_shape(const bzk_mpn_circuit *circuit, uint64_t shape[12]);
int32_t bzk_mpn_circuit_matrix(const bzk_mpn_circuit *circuit, uint32_t side, uint64_t *rowptr, uint32_t *col, bzk_fr *val);
/* The update circuit in the blocked form of bzk_r1cs_upload_blocked: slots 2.. are not stored, so the matrices
 * (bzk_mpn_circuit_matrix) hold head | template | tail.  The witness programs and bzk_mpn_circuit_shape (the expanded
 * system's constraint and entry counts) equal bzk_mpn_update_circuit_compile's. */
int32_t bzk_mpn_update_circuit_compile_blocked(uint32_t log4_tree, uint32_t log4_token, uint32_t log4_batch, const uint8_t *poseidon_blob,
                                               size_t blob_len, const bzk_fr jubjub[3], bzk_mpn_circuit **out);
/* out = {head_rows, tmpl_rows, reps, tail_rows, var_lo, var_stride, stored nnz a, b, c} of an update circuit from either
 * compile (of an explicit one: where the blocks lie in its full matrices); BZK_ERR_BAD_ARG for the two-phase circuits */
int32_t bzk_mpn_circuit_blocks(const bzk_mpn_circuit *circuit, uint64_t out[9]);
/* which: 0 = slot program (two-phase circuits: phase 1), 1 = epilogue program (phase 2), 2 = the `reveal` of a two-phase
 * batch (one instance; externals = every slot's revealed row, slot-major); sizes = {n_ops, n_lc, n_terms, n_coefs, n_raw,
 * n_ext}; array outputs optional */
int32_t bzk_mpn_circuit_program(const bzk_mpn_circuit *circuit, uint32_t which, uint64_t sizes[6], int32_t *ops, int32_t *lc_ptr,
                                int32_t *lc_slot, int32_t *lc_coef, bzk_fr *coefs);

/* ------------------------------------------------------------------ witness generation (device)
 * bellman's `ProvingAssignment` runs `MpnCircuit::synthesize` with value closures
 * (/root/reference/src/mpn/circuits/update_circuit.rs:49-494).  Every slot of an update batch performs the
 * same allocations, so the host compiles one slot into a straight-line program (bazuka_b200/mpn/
 * witness_program.py) and the device interprets it with one thread per slot.
 *   ops[n_ops][6] = {opcode, lc0, lc1, lc2, lc3, imm}; op j defines block variable j.
 *     0 RAW  raws[slot][imm]           1 MUL lc0*lc1            2 BIT  bit imm of canonical(lc0)
 *     3 ISZERO lc0==0                  4 INVZ lc0^-1 (0 -> 0)   5 SELECT lc0 ? lc2 : lc1
 *     6 JJ   JubJub sum (lc0,lc1)+(lc2,lc3) -> variables j, j+1 ((0,0) if an operand is off-curve)   7 NOP
 *   linear combination l = sum_{k in [lc_ptr[l], lc_ptr[l+1])} coefs[lc_coef[k]] * V[lc_slot[k]]
 *   (coefs[0] must be the constant one); slots: 0 = ONE, 1..n_ext = variables the block reads but does not
 *   define (update circuit: the fee token and the state root entering the slot), 1 + n_ext + j = block
 *   variable j.  coefs and jj_d (the curve's d) are Montgomery images, each below r, and coefs[0] is the
 *   Montgomery image of one; the upload refuses a program that breaks either rule (BZK_ERR_BAD_ARG).
 * bzk_witness_run_dev: raws[ntx][n_raw] and ext[ntx][n_ext] are CANONICAL host images (converted on the
 * device); writes the Montgomery values of slot t's variables to d_aux_out[t*n_ops + j]. */
int32_t bzk_witness_program_upload(bzk_ctx *ctx, const int32_t *ops, uint64_t n_ops, const int32_t *lc_ptr, uint64_t n_lc,
                                   const int32_t *lc_slot, const int32_t *lc_coef, uint64_t n_terms, const bzk_fr *coefs,
                                   uint64_t n_coefs, uint32_t n_raw, uint32_t n_ext, const bzk_fr *jj_d, bzk_witness_program **out);
int32_t bzk_witness_program_free(bzk_ctx *ctx, bzk_witness_program *prog);
int32_t bzk_witness_run_dev(bzk_ctx *ctx, const bzk_witness_program *prog, const bzk_fr *raws, const bzk_fr *ext, uint64_t ntx,
                            void *d_aux_out);

/* ------------------------------------------------------------------ worker protocol (bincode), host only
 * What a node hands an MPN prover and takes back, in the reference's own wire format — `bincode::serialize` of
 *   MpnWork {config, public_inputs, data, new_root, reward}      /root/reference/src/mpn/mod.rs:264-270
 *   GetMpnWorkRequest / GetMpnWorkResponse {works: HashMap<usize, MpnWork>}
 *   PostMpnSolutionRequest {prover, proofs: HashMap<usize, ZkProof>} / PostMpnSolutionResponse {accepted}
 *                                                                  /root/reference/src/client/messages.rs:368-397
 * (`BazukaClient::{get_mpn_works, post_mpn_proof}`, /root/reference/src/client/mod.rs:428-464) — so a Rust node or worker
 * passes `&bincode::serialize(&work)?` across the FFI unconverted.  A decoded work re-encodes to the bytes it came from.
 * Scalars of the info struct and of the row functions are CANONICAL (like the builders' rows); `public_inputs` are
 * Montgomery images as the verifier takes them.  No GPU context: these run anywhere. */
typedef struct bzk_mpn_work bzk_mpn_work;
typedef struct {
    uint32_t kind;                  /* MpnWorkData variant: 0 deposit, 1 withdraw, 2 update */
    uint32_t log4_tree, log4_token; /* MpnConfig.log4_tree_size / log4_token_tree_size */
    uint32_t log4_batch;            /* the config's batch size for this kind */
    uint64_t n_transitions;
    uint64_t height;                /* ZkPublicInputs */
    bzk_fr state, aux_data, next_state;
    bzk_fr new_root_hash;           /* ZkCompressedState {state_hash, state_size} */
    uint64_t new_root_size;
    uint64_t reward;
} bzk_mpn_work_info;
/* consumed == NULL: the buffer must hold exactly one work; otherwise *consumed = bytes read (works back to back) */
int32_t bzk_mpn_work_decode(const uint8_t *bytes, size_t len, bzk_mpn_work **out, size_t *consumed);
int32_t bzk_mpn_work_free(bzk_mpn_work *work);
int32_t bzk_mpn_work_encode(const bzk_mpn_work *work, uint8_t *out, size_t cap, size_t *len);   /* out == NULL: size only */
int32_t bzk_mpn_work_get_info(const bzk_mpn_work *work, bzk_mpn_work_info *out);
/* `MpnWork::vk()`: the verifying-key image (878 + 97 n bytes, no enum tag) of the work's kind; valid while the work lives */
int32_t bzk_mpn_work_vk(const bzk_mpn_work *work, const uint8_t **vk, size_t *len);
/* `MpnWork::verify`'s commitment (/root/reference/src/mpn/mod.rs:283-285, chain side update_contract/mod.rs:29-32):
 * ZkScalar::new(sha3_256(bincode((prover, reward)))) — canonical */
int32_t bzk_mpn_commitment(const uint8_t prover[32], uint64_t reward, bzk_fr *out);
int32_t bzk_sha3_256(const uint8_t *data, size_t len, uint8_t out[32]);   /* `Hasher::hash` (/root/reference/src/core/hash.rs:29) */
/* [commitment, height, state, aux_data, next_state] for (work, prover): Montgomery, as bzk_groth16_verify_bytes takes them */
int32_t bzk_mpn_work_public_inputs(const bzk_mpn_work *work, const uint8_t prover[32], bzk_fr out[5]);
/* `MpnWork::verify(prover, proof)` (/root/reference/src/mpn/mod.rs:281-295): 1 accepted, 0 rejected, < 0 bad argument */
int32_t bzk_mpn_work_verify(const bzk_mpn_work *work, const uint8_t prover[32], const uint8_t *proof387);
/* A work's transitions as the rows the witness drivers consume — what the external prover does first with a work.  All 4^B
 * slots of the work's batch size are written: a work carries only the transitions its builder made, the rest are padded like
 * `{Update,Deposit,Withdraw}Transition::null` (/root/reference/src/mpn/mod.rs:440-537).
 *   update:             raws[4^B][32 + 9T + 6A], ext[4^B][2] = {fee token, state root entering the slot}  -> bzk_mpn_update_witness
 *   deposit / withdraw: raws1, raws2, roots[4^B], reveal (layouts of bzk_mpn_deposit_build / _withdraw_build) -> bzk_mpn_dw_witness
 * The entering roots do not travel: they are recomputed from each transition's own account, proof and index with the host
 * Poseidon.  BZK_ERR_NOT_ON_CURVE: a key of the work does not decompress; BZK_ERR_BAD_ARG: proofs of the wrong depth. */
int32_t bzk_mpn_work_update_rows(const bzk_mpn_work *work, const bzk_poseidon_host *hasher, const bzk_fr *jubjub_d, const bzk_fr *fee_token,
                                 bzk_fr *raws, bzk_fr *ext);
int32_t bzk_mpn_work_dw_rows(const bzk_mpn_work *work, const bzk_poseidon_host *hasher, const bzk_fr *jubjub_d, bzk_fr *raws1, bzk_fr *raws2,
                             bzk_fr *roots, bzk_fr *reveal);
/* the same rows with every hash in batched launches on a context (1 + A launches for the entering roots of the whole batch, one
 * for the calldata hashes) instead of (1 + A) dependent host hashes per transaction — what bzk_mpn_prover_prove_work uses */
int32_t bzk_mpn_work_update_rows_ctx(bzk_ctx *ctx, const bzk_mpn_work *work, const bzk_fr *jubjub_d, const bzk_fr *fee_token, bzk_fr *raws, bzk_fr *ext);
int32_t bzk_mpn_work_dw_rows_ctx(bzk_ctx *ctx, const bzk_mpn_work *work, const bzk_fr *jubjub_d, bzk_fr *raws1, bzk_fr *raws2, bzk_fr *roots,
                                 bzk_fr *reveal);
/* messages: up to `cap` works are decoded into ids[] / works[] (free each); *n = the number on the wire */
int32_t bzk_mpn_get_work_response_decode(const uint8_t *bytes, size_t len, uint64_t *ids, bzk_mpn_work **works, uint64_t cap, uint64_t *n);
int32_t bzk_mpn_get_work_request_encode(const uint8_t address[32], uint8_t out[40]);
/* proofs387 = n x 387-byte Groth16Proof images (sent as 391-byte ZkProof::Groth16); out == NULL: size only */
int32_t bzk_mpn_post_solution_request_encode(const uint8_t prover[32], const uint64_t *ids, const uint8_t *proofs387, uint64_t n, uint8_t *out,
                                             size_t cap, size_t *len);
int32_t bzk_mpn_post_solution_response_decode(const uint8_t *bytes, size_t len, uint64_t *accepted);

/* `mpn::prepare_works` (/root/reference/src/mpn/mod.rs:298-424) over the native ledger — the validator's side of the protocol.
 * On ONE fork of `state` (not modified; `db.fork_on_ram()`): mpn_num_deposit_batches deposit batches, then the withdraw batches,
 * then the update batches, every batch offered the whole list again, accounts created on the way visible to the later batches
 * (`new_account_indices`); every batch becomes an MpnWork {config, public_inputs, data, new_root, reward}.  Inputs are the
 * reference's wire images: `bincode::serialize` of the `MpnConfig`, of `&Vec<MpnDeposit>`, `&Vec<MpnWithdraw>` and
 * `&Vec<MpnTransaction>` (NULL = none); rewards = {deposit, withdraw, update}; fee_token canonical (Ziesha = 1).  What the
 * builders check of the L1 side is read from the payments (a deposit's source, a withdrawal's calldata and fingerprint).
 * Outputs: *works_bytes = bincode of `HashMap<usize, MpnWork>` numbered in building order (the body of GetMpnWorkResponse;
 * release with bzk_buffer_free), *fork_out = the ledger after all batches (bzk_mpn_state_free, or commit_accounts + keep).
 * The validator's own reward deposit and the L1 balances are chain state: prepend that deposit like mod.rs:338-351 does, and offer only
 * deposits whose L1 source can pay amount and fee (`check_balance`, /root/reference/src/mpn/deposit.rs:85-107 reads `db.get_balance`). */
int32_t bzk_mpn_prepare_works(bzk_ctx *ctx, const bzk_mpn_state *state, const uint8_t *config_bytes, size_t config_len, const uint8_t *deposits_bytes,
                              size_t deposits_len, const uint8_t *withdraws_bytes, size_t withdraws_len, const uint8_t *updates_bytes, size_t updates_len,
                              const uint64_t rewards[3], uint64_t height, const bzk_fr *fee_token, bzk_mpn_state **fork_out, uint8_t **works_bytes,
                              size_t *works_len, uint64_t *n_works);
int32_t bzk_buffer_free(uint8_t *buffer);

/* ------------------------------------------------------------------ the external prover's job as one call
 * `MpnWork` (bincode) in, `ZkProof::Groth16` (391 bytes, bincode) out — what the reference's workers do between
 * `GET /bincode/mpn/work` and `POST /bincode/mpn/solution` (/root/reference/src/client/mod.rs:428-464; `MpnWork::verify` on the
 * node side checks the result, /root/reference/src/mpn/mod.rs:281-295).  One prover per circuit (kind, A, T, B): it uploads the
 * natively compiled circuit's witness programs and R1CS (bzk_mpn_{update,dw}_circuit_compile) and keeps z resident; `params` is
 * that circuit's proving key (borrowed).  prove_work = bzk_mpn_work_decode -> bzk_mpn_work_{update,dw}_rows_ctx ->
 * bzk_mpn_{update,dw}_witness -> bzk_groth16_prove_dev -> bzk_groth16_proof_bytes.  r, s: Montgomery images.
 * BZK_ERR_BAD_ARG: malformed work, or a work of another kind / size than the prover's circuit. */
typedef struct bzk_mpn_prover bzk_mpn_prover;
int32_t bzk_mpn_prover_create(bzk_ctx *ctx, const bzk_mpn_circuit *circuit, const bzk_groth16_params *params, const bzk_fr *jubjub_d,
                              const bzk_fr *fee_token, bzk_mpn_prover **out);
int32_t bzk_mpn_prover_free(bzk_ctx *ctx, bzk_mpn_prover *prover);
int32_t bzk_mpn_prover_prove_work(bzk_ctx *ctx, bzk_mpn_prover *prover, const uint8_t *work_bytes, size_t work_len, const uint8_t prover_address[32],
                                  const bzk_fr *r, const bzk_fr *s, int32_t check_satisfied, uint8_t zkproof391[391]);

/* ------------------------------------------------------------------ the MPN worker: a node's work response in, the solution out
 * What a worker does on each poll (the reference's external prover, src/mpn/mod.rs:79-129): `GetMpnWorkResponse` bytes in,
 * `PostMpnSolutionRequest` bytes out, over one or more contexts, several of them on one GPU if wanted.
 *   bzk_mpn_worker_create   config = bincode(MpnConfig), the node's; devices[i] = a context and, per kind in MpnWorkData order
 *                           {deposit, withdraw, update}, that kind's proving key (borrowed, must outlive the worker) or NULL when
 *                           this context does not serve the kind.  Each served circuit is compiled once at the config's shape
 *                           (A, T, B of its kind): the update circuit always by the blocked compile, deposit and withdraw
 *                           explicit; one bzk_mpn_prover per context and kind.  poseidon_blob / jubjub as for the compilers,
 *                           fee_token canonical (Ziesha = 1).  Every context must have its Poseidon table loaded.
 *                           BZK_ERR_BAD_ARG: a malformed config, no context, a key whose five vector lengths are not the ones
 *                           its circuit's R1CS gives (h = m - 1, l = num_aux, a / b_g1 / b_g2 = density counts), or whose
 *                           alpha_g1, beta_g1, beta_g2, delta_g1 or delta_g2 differ from that kind's verifying key in the config.
 *   bzk_mpn_worker_prove_response
 *                           decodes the response (bzk_mpn_get_work_response_decode) and proves every work whose config is the
 *                           worker's (the same shape and the same verifying-key bytes for its kind), with the satisfiability
 *                           check on, one host thread per context, largest circuit first.  Before a proof is kept it is checked
 *                           against the work's verifying key and public inputs (one bzk_groth16_verify_batch per kind).  The proved
 *                           works are encoded with bzk_mpn_post_solution_request_encode into *solution (release with
 *                           bzk_buffer_free), in the order of the response.  status_each (optional, one per work on the wire, in
 *                           response order): BZK_OK proved; BZK_ERR_BAD_ARG a foreign config or a work of a kind no context serves;
 *                           BZK_ERR_UNSAT transitions that do not satisfy the circuit; BZK_ERR_REJECTED a proof that failed its own
 *                           verification (the key's point vectors or ic do not belong to the verifying key).  Such works are left
 *                           out and the call still returns BZK_OK.  A malformed response is BZK_ERR_BAD_ARG with no solution; a
 *                           device or memory error is returned as such, with no solution.
 *                           Blinding: seed == NULL draws r and s of every proof from the OS (getrandom, 64 bytes each, reduced mod
 *                           r).  A non-NULL seed (32 bytes) is a test hook that makes proofs reproducible: r = SHA3(seed || id ||
 *                           "r"), s = SHA3(seed || id || "s") as little-endian integers mod r, id = the work's u64 id (little-endian)
 *                           — never use it in production, a predictable r or s gives away the witness.
 * Each context is driven by one thread of the call at a time; the worker itself launches no kernel of its own. */
typedef struct bzk_mpn_worker bzk_mpn_worker;
typedef struct {
    bzk_ctx *ctx;
    const bzk_groth16_params *params[3];   /* deposit, withdraw, update; NULL = not served on this context */
} bzk_mpn_worker_device;
int32_t bzk_mpn_worker_create(const uint8_t *config_bytes, size_t config_len, const bzk_mpn_worker_device *devices, uint32_t n_devices,
                              const uint8_t *poseidon_blob, size_t blob_len, const bzk_fr jubjub[3], const bzk_fr *fee_token, bzk_mpn_worker **out);
int32_t bzk_mpn_worker_prove_response(bzk_mpn_worker *worker, const uint8_t *response, size_t len, const uint8_t prover_address[32],
                                      const uint8_t *seed32, uint8_t **solution, size_t *solution_len, int32_t *status_each, uint64_t status_cap,
                                      uint64_t *n_works);
int32_t bzk_mpn_worker_free(bzk_mpn_worker *worker);
/* Host wall-clock milliseconds of the last successful prove_response: {the whole call, rows + witness (summed over works, the
 * context synchronised after each witness), the rest of each proof (summed over works), the self-check}.  With several contexts
 * the two sums can exceed the call's time. */
int32_t bzk_mpn_worker_last_timing(const bzk_mpn_worker *worker, double ms[4]);

/* 387-byte bincode image of `Groth16Proof {a,b,c}` (/root/reference/src/zk/groth16/mod.rs:33-38);
 * prefix it with the u32 variant tag 0 for `ZkProof::Groth16` (391 B). */
int32_t bzk_groth16_proof_bytes(const bzk_g1_affine *a, const bzk_g2_affine *b, const bzk_g1_affine *c, uint8_t out[387]);
/* Verifier.  Replaces `zk::groth16::groth16_verify` / `zk::check_proof`
 * (/root/reference/src/zk/groth16/mod.rs:67-121, /root/reference/src/zk/mod.rs:157-193): bellman
 * `prepare_verifying_key` + `verify_proof` with public inputs [commitment, height, prev_state, aux_data,
 * next_state].  Host arithmetic (one verification is a scalar job; no GPU context needed).
 * Returns 1 = accepted, 0 = rejected, < 0 = BZK_ERR_BAD_ARG.  `_bytes` takes the reference's bincode
 * images: `Groth16VerifyingKey` (878 + 97*len B) and `Groth16Proof` (387 B). */
int32_t bzk_groth16_verify(const bzk_g1_affine *alpha_g1, const bzk_g2_affine *beta_g2, const bzk_g2_affine *gamma_g2,
                           const bzk_g2_affine *delta_g2, const bzk_g1_affine *ic, size_t n_ic,
                           const bzk_fr *public_inputs, size_t n_inputs,
                           const bzk_g1_affine *proof_a, const bzk_g2_affine *proof_b, const bzk_g1_affine *proof_c);
int32_t bzk_groth16_verify_bytes(const uint8_t *vk, size_t vk_len, const bzk_fr *public_inputs, size_t n_inputs, const uint8_t *proof387);
/* Prepared verifying key — bellman `PreparedVerifyingKey`, which the reference rebuilds on every `groth16_verify` call
 * (/root/reference/src/zk/groth16/mod.rs:97-108): e(alpha,beta) and the Miller-loop line coefficients of gamma and
 * delta, computed once.  The plain entry points above keep the 8 most recently used prepared keys in an internal
 * mutex-guarded cache; with an explicit handle there is no shared state. */
typedef struct bzk_groth16_pvk bzk_groth16_pvk;
int32_t bzk_groth16_pvk_create(const bzk_g1_affine *alpha_g1, const bzk_g2_affine *beta_g2, const bzk_g2_affine *gamma_g2,
                               const bzk_g2_affine *delta_g2, const bzk_g1_affine *ic, size_t n_ic, bzk_groth16_pvk **out);
int32_t bzk_groth16_pvk_from_bytes(const uint8_t *vk, size_t vk_len, bzk_groth16_pvk **out);
int32_t bzk_groth16_pvk_free(bzk_groth16_pvk *pvk);
int32_t bzk_groth16_verify_prepared(const bzk_groth16_pvk *pvk, const bzk_fr *public_inputs, size_t n_inputs,
                                    const bzk_g1_affine *proof_a, const bzk_g2_affine *proof_b, const bzk_g1_affine *proof_c);
/* Batch verification of m proofs under one key (a node syncing many blocks, SURVEY §8f-4): random linear combination
 *   prod_j e(r_j A_j, B_j) * e(-sum_j r_j acc_j, gamma) * e(-sum_j r_j C_j, delta) == e(alpha,beta)^(sum_j r_j)
 * with 127-bit r_j derived from `seed` (draw a fresh random seed per batch), m + 2 Miller loops over `threads` host
 * threads (<= 0: all) and ONE final exponentiation.  public_inputs: m rows of n_inputs Montgomery scalars; proofs387:
 * m x 387 bytes.  Returns 1 if every proof verifies, else 0; ok_each (optional, m bytes) receives per-proof verdicts
 * (on a failing batch the proofs are re-checked one by one). */
int32_t bzk_groth16_verify_batch(const bzk_groth16_pvk *pvk, const bzk_fr *public_inputs, size_t n_inputs, const uint8_t *proofs387, size_t m,
                                 uint64_t seed, int32_t threads, uint8_t *ok_each);
/* The same check with the m proof-dependent Miller loops on the GPU (one thread per proof); the key-dependent loops, the
 * product and the single final exponentiation stay on the host.  Same verdicts as the host version for the same seed. */
int32_t bzk_groth16_verify_batch_dev(bzk_ctx *ctx, const bzk_groth16_pvk *pvk, const bzk_fr *public_inputs, size_t n_inputs,
                                     const uint8_t *proofs387, size_t m, uint64_t seed, uint8_t *ok_each);
/* Building blocks also used by the GPU-side trusted-setup helper (bellman `generate_parameters`):
 * CSR sparse matrix-vector product over Fr (out[row] = sum val*vec[col]) and fixed-base scalar
 * multiplication out[i] = [k_i] base written as wire images. */
int32_t bzk_csr_spmv_dev(bzk_ctx *ctx, const void *d_rowptr, const void *d_col, const void *d_val, uint64_t nrows, const void *d_vec, void *d_out);
int32_t bzk_g1_fixed_base_mul_dev(bzk_ctx *ctx, const bzk_g1_affine *base, const void *d_scalars, size_t n, void *d_out);
int32_t bzk_g2_fixed_base_mul_dev(bzk_ctx *ctx, const bzk_g2_affine *base, const void *d_scalars, size_t n, void *d_out);
/* The same multiplications stored straight into a new resident base vector (d_scalars: n Montgomery Fr on the device),
 * so that a key vector is never held twice; enqueued on the context's stream. */
int32_t bzk_g1_bases_fixed_base_mul(bzk_ctx *ctx, const bzk_g1_affine *base, const void *d_scalars, size_t n, bzk_g1_bases **out);
int32_t bzk_g2_bases_fixed_base_mul(bzk_ctx *ctx, const bzk_g2_affine *base, const void *d_scalars, size_t n, bzk_g2_bases **out);

/* ------------------------------------------------------------------ elementwise Fr (device)
 * out[i] = a[i] (op) b[i]; used by the prover pipeline and the arithmetic parity tests. */
#define BZK_FR_ADD 0
#define BZK_FR_SUB 1
#define BZK_FR_MUL 2
int32_t bzk_fr_binop_dev(bzk_ctx *ctx, int32_t op, const void *d_a, const void *d_b, void *d_out, size_t n);
/* Fp product, for the 384-bit arithmetic parity test: out[i] = a[i]*b[i] (Montgomery images, 48 B) */
int32_t bzk_fp_mul_dev(bzk_ctx *ctx, const void *d_a, const void *d_b, void *d_out, size_t n);

#ifdef __cplusplus
}
#endif
#endif /* BZK_H */
