/* zkb200 — C ABI of the H100-native Groth16 prover hot path (libzkb200.so).
 *
 * Drop-in boundary for the path LayerXcom/zero-chain reaches through
 *     bellman::groth16::create_random_proof(circuit, &Parameters<Bls12>, rng)
 * (call sites core/proofs/src/confidential.rs:149, core/proofs/src/anonymous.rs:165; the CRS is
 * read at core/proofs/src/confidential.rs:95-103 by Parameters::read(buf, checked = true)).
 * bellman 0.1.0 itself is an un-vendored dependency (Cargo.lock:210-212), so each entry point
 * cites the upstream function it replaces and the reference call site that reaches it.
 *
 * Conventions
 *   - plain pointers and sizes only; the caller owns every input/output buffer for the duration
 *     of the call; handles (zk_ctx, zk_bases, zk_params) are owned by the library.
 *   - Fr scalars cross the ABI as canonical FrRepr: 4 little-endian u64 limbs, value < r
 *     (= Fr::into_repr(), core/pairing/src/bls12_381/fr.rs:290-303).  Montgomery form is internal.
 *   - the CRS crosses once as the exact Parameters::write byte stream (zface/params/conf_pk.dat);
 *     proofs come back as the exact Proof::write bytes (core/bellman-verifier/src/lib.rs:55-65).
 *   - "limb form" points (kernel-level entry points only): affine x|y in Montgomery limbs,
 *     96 B (G1: x[6] y[6] u64) or 192 B (G2: x.c0 x.c1 y.c0 y.c1), infinity = all zero.
 *   - every function returns ZK_OK (0) or a negative error; zk_last_error() gives the text.
 *     Error codes mirror bellman's SynthesisError / io::Error as seen at the call sites
 *     (zface/src/error.rs:17,45-48).
 *   - thread safety: a zk_ctx is single-threaded (one CUDA stream + its own workspace, NTT tables and lanes); zk_params /
 *     zk_bases / zk_pvk / zk_r1cs are read-only after creation and may be shared by several contexts on the same device.
 *     Concurrent proving on one zk_params (what bellman's Arc<Vec<..>> parameters allow, SURVEY.md §8b) = one zk_ctx per
 *     host thread, all passing the same zk_params (bench.py's two_batches_in_flight does exactly that).
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with
 *     ZK_ERR_CUDA.
 */
#ifndef ZKB200_H
#define ZKB200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define ZK_OK 0
#define ZK_ERR_CUDA (-1)                 /* no device / CUDA runtime failure */
#define ZK_ERR_INVALID (-2)              /* bad argument */
#define ZK_ERR_ASSIGNMENT_MISSING (-3)   /* SynthesisError::AssignmentMissing: vector sizes do not match the CRS */
#define ZK_ERR_POLY_DEGREE_TOO_LARGE (-4)/* SynthesisError::PolynomialDegreeTooLarge */
#define ZK_ERR_UNEXPECTED_IDENTITY (-5)  /* SynthesisError::UnexpectedIdentity (base or delta at infinity) */
#define ZK_ERR_IO (-6)                   /* SynthesisError::IoError: truncated / malformed Parameters stream */
#define ZK_ERR_DECODE (-7)               /* GroupDecodingError (not on curve, not in subgroup, bad flags, x >= q) */
#define ZK_ERR_NOT_CANONICAL (-8)        /* a scalar >= r (PrimeFieldDecodingError::NotInField) */
#define ZK_ERR_MALFORMED_VK (-9)         /* SynthesisError::MalformedVerifyingKey: inputs.len() + 1 != ic.len() */
#define ZK_ERR_BAD_SIGNATURE (-10)      /* zk_import_block: an extrinsic's signature fails (BadSignature) */

const char *zk_last_error(void);
int zk_device_count(void);
const char *zk_version(void);

/* ---- execution context: one per (device, stream) ------------------------------------------- */
typedef struct zk_ctx zk_ctx;
/* stream: a cudaStream_t to run on (e.g. the caller's current stream) or NULL to create one. */
int zk_ctx_create(int device, void *stream, zk_ctx **out);
void zk_ctx_destroy(zk_ctx *ctx);
int zk_ctx_sync(zk_ctx *ctx);
/* Tuning options of a context (and of the prover lanes it owns).  Results never depend on them.
 *   ZK_OPT_AFFINE_MIN_ENTRIES  MSMs with at least this many (term, window) entries reduce their buckets with batched-affine
 *                              rounds (6.4 field products per addition instead of 10, one shared serial inversion per round)
 *                              before the XYZZ pass: more throughput with several MSMs in flight or batched proving, more
 *                              latency for one blocking MSM.  Default 2^22;
 *                              -1 = never, 0 = always.
 *   ZK_OPT_AFFINE_LEVELS       number of rounds; -1 (default) = from the average bucket length.
 *   ZK_OPT_VERIFY_LANES        1 (default): the verifier's Miller loops and final exponentiations spread every Fq12 value over six
 *                              lanes of a warp; 0: one thread per proof (the round-1 kernels, kept as the A/B reference). */
#define ZK_OPT_AFFINE_MIN_ENTRIES 1
#define ZK_OPT_AFFINE_LEVELS 2
#define ZK_OPT_VERIFY_LANES 3
int zk_ctx_set_opt(zk_ctx *ctx, int opt, long value);
void *zk_ctx_stream(zk_ctx *ctx);

/* ---- multi-scalar multiplication (replaces bellman::multiexp::multiexp, SURVEY.md §8 a8) ----- */
typedef struct zk_bases zk_bases;
/* Upload n affine bases (limb form, HOST memory) and, if precompute != 0, build the window tables
 * 2^(c*w) * P_i on the device (the CRS is fixed, so this is done once, like Parameters::read).
 * window_bits = 0 picks c from n.  group = 1 (G1) or 2 (G2).  Infinity bases are rejected
 * (bellman: SynthesisError::UnexpectedIdentity). */
int zk_bases_upload(zk_ctx *ctx, int group, const uint64_t *bases_limbs, size_t n, int window_bits, int precompute,
                    zk_bases **out);
void zk_bases_free(zk_bases *b);
size_t zk_bases_len(const zk_bases *b);
int zk_bases_window_bits(const zk_bases *b);
/* sum_i scalars[i] * P_i over the first n bases.  scalars: canonical FrRepr in HOST memory
 * (host -> device copy is part of the call); out: uncompressed encoding (96 B for G1, 192 B for G2;
 * G1Uncompressed / G2Uncompressed::from_affine, core/pairing/src/bls12_381/ec.rs:686-752, 1343-1425). */
int zk_msm(zk_ctx *ctx, const zk_bases *b, const uint64_t *scalars, size_t n, uint8_t *out);
/* same with scalars already resident in DEVICE memory (kernel-only timing; prover-internal use) */
int zk_msm_device(zk_ctx *ctx, const zk_bases *b, const void *d_scalars, size_t n, uint8_t *out);
/* The same MSM as a future, which is what bellman's multiexp returns (multiexp.rs: Box<Future<Item = G>>): begin enqueues the
 * upload (host variant), the MSM, the affine conversion and the download of the encoded point, and returns; end waits and
 * hands out the 96 / 192 bytes.  One MSM may be in flight per context.  Everything after the bucket accumulation runs on a
 * high-priority stream of the context, so two contexts used alternately overlap the latency-bound tail of one MSM (and the
 * upload of the next scalars) with the accumulation of the other — results are identical to zk_msm / zk_msm_device. */
int zk_msm_begin(zk_ctx *ctx, const zk_bases *b, const uint64_t *scalars, size_t n);
int zk_msm_device_begin(zk_ctx *ctx, const zk_bases *b, const void *d_scalars, size_t n);
int zk_msm_end(zk_ctx *ctx, uint8_t *out);
/* multi-GPU form: the rank's partial (zk_partial_size bytes) lands in d_partial_out on zk_ctx_tail_stream(ctx); the caller enqueues
 * its all-gather on that stream, then zk_points_fold_begin (fold + encode + download on the same stream); zk_msm_end collects. */
void *zk_ctx_tail_stream(zk_ctx *ctx);
int zk_msm_partial_device_begin(zk_ctx *ctx, const zk_bases *b, const void *d_scalars, size_t n, void *d_partial_out);
int zk_points_fold_begin(zk_ctx *ctx, int group, const void *d_partials, size_t count);
/* batch of `batch` independent scalar vectors (each n long, contiguous) against the same bases;
 * out: batch encodings.  Used by the batched prover. */
int zk_msm_batch_device(zk_ctx *ctx, const zk_bases *b, const void *d_scalars, size_t n, size_t batch, uint8_t *out);
/* multi-GPU helper: the partial result as an XYZZ point in DEVICE memory is all-gathered by the
 * caller (NCCL, bytes) and folded with zk_points_fold: out = encoding of sum of `count` device
 * points of zk_partial_size(group) bytes each. */
size_t zk_partial_size(int group);
int zk_msm_partial_device(zk_ctx *ctx, const zk_bases *b, const void *d_scalars, size_t n, void *d_partial_out);
int zk_points_fold(zk_ctx *ctx, int group, const void *d_partials, size_t count, uint8_t *out);

/* ---- Fr radix-2 NTT (replaces bellman::domain::EvaluationDomain, SURVEY.md §8 a7) ----------- */
#define ZK_NTT_FFT 0         /* EvaluationDomain::fft        */
#define ZK_NTT_IFFT 1        /* EvaluationDomain::ifft       (includes the m^-1 scaling) */
#define ZK_NTT_COSET_FFT 2   /* EvaluationDomain::coset_fft  (distribute_powers(7) then fft) */
#define ZK_NTT_ICOSET_FFT 3  /* EvaluationDomain::icoset_fft (ifft then distribute_powers(7^-1)) */
/* data: 2^log_n Fr elements, MONTGOMERY limbs (the in-memory form of bellman's Scalar<E>), natural
 * order in and out, transformed in place.  Host-memory and device-memory flavours. */
int zk_ntt_fr(zk_ctx *ctx, uint64_t *data, unsigned log_n, int mode);
int zk_ntt_fr_device(zk_ctx *ctx, void *d_data, unsigned log_n, int mode);

/* ---- Groth16 (replaces bellman::groth16::{Parameters::read, create_proof}) ------------------ */
typedef struct zk_params zk_params;
/* Parses the exact Parameters::write stream (SURVEY.md §3.3; reference call
 * core/proofs/src/confidential.rs:99 `Parameters::read(&buf[..], true)`), decodes every point on
 * the device, with checked != 0 also tests on-curve and r-torsion membership
 * (core/pairing/src/bls12_381/ec.rs:675-685), rejects infinity in the query vectors, and keeps the
 * CRS (and its MSM window tables) resident on the context's device. */
int zk_params_load(zk_ctx *ctx, const uint8_t *pk_bytes, size_t len, int checked, zk_params **out);
void zk_params_free(zk_params *p);
/* counts[6] = { ic, h, l, a, b_g1, b_g2 } */
int zk_params_counts(const zk_params *p, uint64_t counts[6]);
/* Parameters::write (bellman groth16; reference call core/proofs/src/confidential.rs:73-93 `self.proving_key.write(..)`): the
 * resident CRS re-encoded as the exact byte stream Parameters::read consumes — zk_params_size bytes; loading a file and writing
 * it back reproduces the file byte for byte.  zk_params_write_vk emits only the VerifyingKey head (VerifyingKey::write: alpha_g1 |
 * beta_g1 | beta_g2 | gamma_g2 | delta_g1 | delta_g2 | u32 n | ic; zk_params_vk_size bytes) — what `params.vk`
 * (core/proofs/src/setup.rs:31, prepare_verifying_key(&params.vk)) needs on the host side. */
size_t zk_params_size(const zk_params *p);
size_t zk_params_vk_size(const zk_params *p);
int zk_params_write(zk_ctx *ctx, const zk_params *p, uint8_t *out);
int zk_params_write_vk(zk_ctx *ctx, const zk_params *p, uint8_t *out);
/* Parameters::read(buf, checked = true) with a decoded-CRS cache on disk (SURVEY.md §8 f1; the "FIX: too heavy" read at
 * core/proofs/src/crypto_components.rs:320-328).  If `cache_path` holds the decoded Montgomery points of exactly these bytes
 * (SHA-256 of the whole stream, length and vector counts are compared, and the cached points carry their own SHA-256), they are uploaded as they are — no decoding, no on-curve
 * or subgroup tests (*cache_hit = 1).  Otherwise the stream goes through the full CHECKED load and the cache file is (re)written
 * atomically (*cache_hit = 0); a cache that cannot be written is not an error.  cache_hit may be NULL.
 * Trust: the hashes guard against corruption and against a cache of another key, not against an adversary who can write
 * `cache_path` (they could store off-curve points with a matching body hash) — keep the file where the proving key itself lives. */
int zk_params_load_cached(zk_ctx *ctx, const uint8_t *pk_bytes, size_t len, const char *cache_path, int *cache_hit, zk_params **out);

/* create_proof for ONE already-synthesised witness (the Rust shim runs ProvingAssignment::synthesize
 * and the `input_i * 0 = 0` rows, then calls this; SURVEY.md §8b).
 *   a/b/c_evals      n_constraints canonical Fr each (<A_j,z>, <B_j,z>, <C_j,z>)
 *   input_assignment n_inputs canonical Fr, [0] = ONE;  aux_assignment n_aux canonical Fr
 *   *_density        one BYTE per variable (0/1): DensityTracker bits of the A-aux, B-input, B-aux queries
 *   r, s             the two blinding scalars create_random_proof draws (canonical)
 *   proof_out        192 B = Proof::write (compressed A | B | C) */
int zk_groth16_prove(zk_ctx *ctx, const zk_params *p,
                     const uint64_t *a_evals, const uint64_t *b_evals, const uint64_t *c_evals, size_t n_constraints,
                     const uint64_t *input_assignment, size_t n_inputs,
                     const uint64_t *aux_assignment, size_t n_aux,
                     const uint8_t *a_aux_density, const uint8_t *b_input_density, const uint8_t *b_aux_density,
                     const uint64_t r[4], const uint64_t s[4], uint8_t proof_out[192]);
/* `batch` witnesses of the same circuit (same sizes and densities), arrays concatenated per proof:
 * a_evals[batch][n_constraints][4] ... r[batch][4], s[batch][4]; proofs_out[batch][192]. */
int zk_groth16_prove_batch(zk_ctx *ctx, const zk_params *p, size_t batch,
                           const uint64_t *a_evals, const uint64_t *b_evals, const uint64_t *c_evals, size_t n_constraints,
                           const uint64_t *input_assignment, size_t n_inputs,
                           const uint64_t *aux_assignment, size_t n_aux,
                           const uint8_t *a_aux_density, const uint8_t *b_input_density, const uint8_t *b_aux_density,
                           const uint64_t *r, const uint64_t *s, uint8_t *proofs_out);

/* ---- proving straight from the witness (SURVEY.md §8 f4: synthesis off the critical path) --------------
 * For a FIXED circuit the constraint matrices A, B, C are known after one synthesis pass (bellman's
 * KeypairAssembly records them as at/bt/ct during parameter generation).  Loaded once in CSR form, the device
 * evaluates <A_j,z>, <B_j,z>, <C_j,z> itself, so per proof only the assignment z = (inputs | aux) crosses PCIe
 * (0.64 MB instead of 2.6 MB for confidential_transfer) and ProvingAssignment::enforce's host arithmetic disappears.
 *   row_ptr[n_constraints + 1], col[nnz] (variable index: < n_inputs = input, else n_inputs + aux index),
 *   coeff[nnz][4] canonical Fr.  The `input_i * 0 = 0` rows are appended by the library; densities are derived. */
typedef struct zk_r1cs zk_r1cs;
int zk_r1cs_load(zk_ctx *ctx, size_t n_constraints, size_t n_inputs, size_t n_aux,
                 const uint32_t *a_row_ptr, const uint32_t *a_col, const uint64_t *a_coeff,
                 const uint32_t *b_row_ptr, const uint32_t *b_col, const uint64_t *b_coeff,
                 const uint32_t *c_row_ptr, const uint32_t *c_col, const uint64_t *c_coeff, zk_r1cs **out);
void zk_r1cs_free(zk_r1cs *r1cs);
int zk_groth16_prove_witness_batch(zk_ctx *ctx, const zk_params *p, const zk_r1cs *r1cs, size_t batch,
                                   const uint64_t *input_assignment, const uint64_t *aux_assignment,
                                   const uint64_t *r, const uint64_t *s, uint8_t *proofs_out);

/* ---- utilities / diagnostics ------------------------------------------------------------------ */
/* out[i] = scalars[i] * base (limb form in, limb form out); group 1 or 2.  Used to build synthetic
 * CRS / test vectors on the device (fixed-base scalar multiplication). */
int zk_scalar_mul_many(zk_ctx *ctx, int group, const uint64_t *base_limbs, const uint64_t *scalars, size_t n,
                       uint64_t *out_limbs);
/* element-wise field ops on host arrays (parity tests of the device arithmetic):
 * field 0 = Fq (6 limbs), 1 = Fr (4 limbs); op 0 mul, 1 add, 2 sub, 3 sqr, 4 inverse, 5 from_repr, 6 into_repr */
int zk_field_op(zk_ctx *ctx, int field, int op, const uint64_t *a, const uint64_t *b, size_t n, uint64_t *out);
/* calibrates the modmul roofline: runs `iters` dependent-chain-free Montgomery products per thread
 * over blocks x threads threads, returns products per second (field 0 Fq, 1 Fr). */
int zk_bench_modmul(zk_ctx *ctx, int field, int blocks, int threads, int iters, double *modmul_per_s, double *ms);

/* Live timing of the dominant kernel (the MSM bucket accumulation) with CUDA events recorded on the
 * context's stream around each launch: enable, run the workload, read the summed duration and launch
 * count (bench.py's roofline block).  Disabled by default (no events are created). */
int zk_ctx_profile(zk_ctx *ctx, int enable);
int zk_ctx_profile_read(zk_ctx *ctx, double *total_ms, uint64_t *launches);
/* Work executed by the MSMs of this context (and of its prover lanes) since the last zk_ctx_profile call, counted on the device:
 * the number of bucket additions (= non-zero signed digits) in G1 and in G2, and how many of them were left to the XYZZ pass
 * (the others were done by batched-affine rounds).  bench.py turns them into executed Fq-modmul-equivalents for the rooflines:
 * an XYZZ mixed addition = 10 products in the base field, a batched-affine addition = 6.4. */
int zk_ctx_profile_counts(zk_ctx *ctx, uint64_t *g1_additions, uint64_t *g2_additions, uint64_t *g1_xyzz, uint64_t *g2_xyzz);

/* ---- Groth16 verification (SURVEY.md §8 f2: the step after the proving path) ----------------------------------
 * zk_pvk: bellman_verifier::PreparedVerifyingKey<Bls12> resident on the device — e(alpha_g1, beta_g2), the Miller-loop
 * line coefficients of -gamma_g2 and -delta_g2, ic, and a fixed-base table of ic[1..] for the public-input sums. */
typedef struct zk_pvk zk_pvk;
/* PreparedVerifyingKey::read (core/bellman-verifier/src/lib.rs:204-245): the bytes zface ships as conf_vk.dat /
 * anony_vk.dat and modules/zk-system keeps in storage.  ic points are checked (on curve, subgroup, not infinity). */
int zk_pvk_load(zk_ctx *ctx, const uint8_t *pvk_bytes, size_t len, zk_pvk **out);
/* prepare_verifying_key(&vk) (core/bellman-verifier/src/verifier.rs:15-30) computed on the device from the VerifyingKey
 * encoding (alpha_g1 | beta_g1 | beta_g2 | gamma_g2 | delta_g1 | delta_g2 | u32 n | ic) — the head of Parameters::write,
 * so a proving-key buffer can be passed as is (trailing bytes are ignored). */
int zk_pvk_prepare(zk_ctx *ctx, const uint8_t *vk_bytes, size_t len, zk_pvk **out);
/* PreparedVerifyingKey::write (lib.rs:183-202): zk_pvk_size bytes, byte-identical to the reference's file */
size_t zk_pvk_size(const zk_pvk *k);
int zk_pvk_write(const zk_pvk *k, uint8_t *out);
size_t zk_pvk_num_inputs(const zk_pvk *k);      /* ic.len() - 1 */
void zk_pvk_free(zk_pvk *k);
/* Proof::read (lib.rs:67-108) + verify_proof (verifier.rs:32-63) for n proofs against one key.
 * proofs: n * 192 bytes (Proof::write); inputs: n * n_inputs canonical Fr (4 LE u64 each, FrRepr);
 * verdicts[i]: 1 = Ok(true), 0 = Ok(false), 2 = Proof::read failed with InvalidData (bad flags, x >= q, not on curve,
 * not in the subgroup), 3 = Proof::read failed with PointInfinity.  Returns ZK_ERR_MALFORMED_VK when
 * n_inputs + 1 != ic.len(), ZK_ERR_NOT_CANONICAL when an input is >= r. */
int zk_groth16_verify_batch(zk_ctx *ctx, const zk_pvk *k, size_t n, const uint8_t *proofs, const uint64_t *inputs,
                            size_t n_inputs, uint8_t *verdicts);
/* same with device pointers; asynchronous on the context's stream (zk_ctx_sync reports a pending ZK_ERR_NOT_CANONICAL) */
int zk_groth16_verify_batch_device(zk_ctx *ctx, const zk_pvk *k, size_t n, const uint8_t *d_proofs, const uint64_t *d_inputs,
                                   size_t n_inputs, uint8_t *d_verdicts);
/* ---- Jubjub public inputs (what modules/zk-system/src/lib.rs:56-165 builds before verify_proof) ----------------
 * Point::read + as_prime_order + into_xy (core/jubjub/src/curve/edwards.rs:92-164, 319-352) for n 32-byte encodings.
 * xy: n * 2 canonical Fr (x then y; 4 LE u64 each); status[i]: 0 ok, 1 NotInField (y >= r), 2 NotOnCurve (no square root),
 * 3 not in the prime-order subgroup (as_prime_order == None).  A rejected point's x and y are zero. */
int zk_jubjub_into_xy(zk_ctx *ctx, size_t n, const uint8_t *points, uint64_t *xy, uint8_t *status);
/* verify_confidential_proof / verify_anonymous_proof (modules/zk-system/src/lib.rs:56-165) for n transactions:
 * points = n * n_points * 32 bytes in PublicInputBuilder push order; public inputs = (x0, y0, x1, y1, ...).
 * verdicts as zk_groth16_verify_batch, plus 4 = a public-input point was rejected (the reference builds the inputs
 * before Proof::read, so 4 takes precedence over 2 / 3).  ZK_ERR_MALFORMED_VK when 2 * n_points + 1 != ic.len(). */
int zk_groth16_verify_points_batch(zk_ctx *ctx, const zk_pvk *k, size_t n, const uint8_t *proofs, const uint8_t *points,
                                   size_t n_points, uint8_t *verdicts);
/* same with device pointers; asynchronous on the context's stream */
int zk_groth16_verify_points_batch_device(zk_ctx *ctx, const zk_pvk *k, size_t n, const uint8_t *d_proofs,
                                          const uint8_t *d_points, size_t n_points, uint8_t *d_verdicts);
/* ---- RedJubjub transaction signatures (what impl Verify for RedjubjubSignature runs per extrinsic) ---------------
 * PublicKey::try_from(vk) + PublicKey::verify(msg, sig, FixedGenerators::Diversifier) (core/primitives/src/signature.rs:65-82,
 * core/jubjub/src/redjubjub.rs:127-155) for n signatures.
 * vks: n * 32 B; sigs: n * 64 B (rbar | sbar); msgs: concatenated message bytes, message i = msgs[msg_off[i] .. msg_off[i+1]),
 * so msg_off has n + 1 entries and msgs holds msg_off[n] bytes; messages may be empty and start at any byte.
 * verdicts[i]: 1 = true; 0 = the equation fails; 2 = vk is not a curve point; 3 = rbar is not a curve point; 4 = sbar >= r_J.
 * (Every value other than 1 is the reference's `false`.  When several apply, the lowest of 2 / 3 / 4 wins, in the
 * reference's order.)  ZK_ERR_INVALID for a NULL pointer, or for offsets that decrease. */
int zk_redjubjub_verify_batch(zk_ctx *ctx, size_t n, const uint8_t *vks, const uint8_t *sigs, const uint8_t *msgs,
                              const uint64_t *msg_off, uint8_t *verdicts);
/* the same with device pointers; asynchronous on the context's stream.  The offsets are not checked: they must not decrease. */
int zk_redjubjub_verify_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_vks, const uint8_t *d_sigs, const uint8_t *d_msgs,
                                     const uint64_t *d_msg_off, uint8_t *d_verdicts);
/* sum_i scalars[i] * P_i over Jubjub (edwards::Point<Unknown>::mul + add).  points: n * 32 B Point::write encodings,
 * read without a subgroup test; scalars: n * 32 B little-endian canonical Fs (< r_J); out: 32 B Point::write.
 * ZK_ERR_DECODE (zk_last_error names the first bad index) for a point that fails Point::read, ZK_ERR_NOT_CANONICAL for a
 * scalar >= r_J (checked first), ZK_ERR_INVALID for NULL arguments with n > 0 or n > 2^26.  n = 0 gives the identity. */
int zk_jubjub_msm(zk_ctx *ctx, size_t n, const uint8_t *points, const uint8_t *scalars, uint8_t out[32]);
/* redjubjub::batch_verify(rng, batch, FixedGenerators::Diversifier) (core/jubjub/src/redjubjub.rs:166-204) for n entries,
 * with the per-entry randomizers z_i (the reference's E::Fs::rand(rng)) supplied by the caller: n * 32 B canonical Fs.
 * vks / sigs / msgs / msg_off exactly as zk_redjubjub_verify_batch.  On return:
 *   *verdict = 1  [8](sum z_i R_i + sum (z_i c_i) vk_i - (sum z_i S_i) P_G) == O      (the reference's true; also for n = 0)
 *            = 0  the combined equation fails
 *            = 2 / 3 / 4  some entry's vk / rbar / sbar is rejected (the codes of zk_redjubjub_verify_batch);
 *              *first_bad (may be NULL) = the lowest such index, and the code is that entry's, in the per-signature order.
 *   *first_bad = n when no entry is rejected.
 * The z_i MUST be unpredictable to the signers (drawn from a cryptographic RNG after the batch is fixed): the check only
 * bounds a forged entry's chance of passing by ~1 / r_J over the draw of z, and a z_i = 0 lets any entry i pass.  A verdict
 * other than 1 does not say which entry is wrong beyond the first rejected encoding: callers that need per-signature
 * verdicts fall back to zk_redjubjub_verify_batch.
 * ZK_ERR_NOT_CANONICAL for a z_i >= r_J; ZK_ERR_INVALID as zk_redjubjub_verify_batch (NULL, decreasing offsets) or for
 * n >= 2^25. */
int zk_redjubjub_batch_verify(zk_ctx *ctx, size_t n, const uint8_t *vks, const uint8_t *sigs, const uint8_t *msgs,
                              const uint64_t *msg_off, const uint8_t *zs, uint8_t *verdict, uint64_t *first_bad);
/* device pointers; asynchronous on the context's stream; d_verdict / d_first_bad in device memory (d_first_bad 8-byte
 * aligned, may be NULL).  The offsets and the z_i are not checked on the host: an entry with z_i >= r_J is rejected on the
 * device with *d_verdict = 5, ahead of that entry's own checks. */
int zk_redjubjub_batch_verify_device(zk_ctx *ctx, size_t n, const uint8_t *d_vks, const uint8_t *d_sigs,
                                     const uint8_t *d_msgs, const uint64_t *d_msg_off, const uint8_t *d_zs,
                                     uint8_t *d_verdict, uint64_t *d_first_bad);
/* ---- lifted-ElGamal balance decryption (what zface's BalanceQuery runs before every transfer) --------------------
 * DecryptionKey::read + Ciphertext::read (+ Ciphertext::read of the pending transfer and Ciphertext::add) +
 * Ciphertext::decrypt(dk, FixedGenerators::Diversifier)  (core/keys/src/lib.rs:125-132, core/crypto/src/elgamal.rs:87-136,
 * zface/src/utils/getter.rs:135-175) for n ciphertexts.
 * dks: n * 32 B (Fs, little-endian); cts: n * 64 B (left | right); pending: NULL (none) or n * 64 B, added to cts first.
 * values[i]: the amount when status[i] == 0, else 0.
 * status[i]: 0 = Some(values[i]); 1 = None (no i < 1 000 000 with i P_G = left - dk right); 2 = dk >= r_J;
 *            3 = cts[i] fails Ciphertext::read (either point: y >= r, not on the curve, or not of prime order);
 *            4 = pending[i] fails Ciphertext::read.  When several apply, the lowest of 2 / 3 / 4 wins, in zface's order.
 * ZK_ERR_INVALID for a NULL ctx / dks / cts / values / status when n > 0.  The first call on a context builds the table of
 * the 10^6 multiples of P_G on the device; it stays resident until zk_ctx_destroy: 32 MB of encodings and an 8 MB index
 * (about 45 MB with the allocator's headroom), plus 96 MB of scratch while it is built. */
int zk_elgamal_decrypt_batch(zk_ctx *ctx, size_t n, const uint8_t *dks, const uint8_t *cts, const uint8_t *pending,
                             uint32_t *values, uint8_t *status);
/* the same with device pointers (d_values 4-byte aligned); asynchronous on the context's stream */
int zk_elgamal_decrypt_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_dks, const uint8_t *d_cts, const uint8_t *d_pending,
                                    uint32_t *d_values, uint8_t *d_status);
/* ---- building confidential transfers (what zface's gen_proof / gen_xt run around the proof) -----------------------
 * All with the Diversifier generator P_G; scalars are 32 B little-endian Fs, points 32 B Point::write encodings.
 * SpendingKey::from_seed -> ProofGenerationKey -> DecryptionKey -> EncryptionKey (core/keys/src/lib.rs:64-71, 167-199) for n
 * seeds of any length: seed i = seeds[seed_off[i] .. seed_off[i+1]), as the messages of zk_redjubjub_verify_batch.
 * sks / dks / eks: n * 32 B.  ZK_ERR_INVALID for a NULL pointer with n > 0, or for offsets that decrease. */
int zk_keys_from_seed_batch(zk_ctx *ctx, size_t n, const uint8_t *seeds, const uint64_t *seed_off, uint8_t *sks, uint8_t *dks,
                            uint8_t *eks);
/* the same with device pointers; asynchronous on the context's stream.  The offsets are not checked: they must not decrease. */
int zk_keys_from_seed_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_seeds, const uint64_t *d_seed_off, uint8_t *d_sks,
                                   uint8_t *d_dks, uint8_t *d_eks);
/* GEpoch::group_hash(epochs[i]) (core/primitives/src/g_epoch.rs:102-145) for n epochs: g_epochs = n * 32 B.  ZK_ERR_DECODE,
 * naming the epoch, when no tag byte below 255 gives a point (the reference asserts there); ZK_ERR_INVALID for NULL. */
int zk_g_epoch_batch(zk_ctx *ctx, size_t n, const uint32_t *epochs, uint8_t *g_epochs);
/* the same with device pointers; asynchronous.  A row whose hash would need tag byte 255 is left as 32 bytes of 0xff. */
int zk_g_epoch_batch_device(zk_ctx *ctx, size_t n, const uint32_t *d_epochs, uint8_t *d_g_epochs);
/* The fields of n confidential transfers: MultiCiphertexts::<Confidential>::encrypt (core/crypto/src/elgamal.rs:48-66) and
 * ProofContext's rvk and nonce, from the sender's sk (n * 32 B), the recipient's encryption key (n * 32 B), amount and fee
 * (n uint32 each), the ElGamal randomness r and the re-randomizer alpha (n * 32 B each) and the call's g_epoch (32 B).
 * fields: n * 288 B, per row the 9 points in the order of groth16.ConfidentialTx's constructor: address_sender (= ek_s),
 *   address_recipient (copied), amount_sender = amount P_G + r ek_s, amount_recipient = amount P_G + r ek_r,
 *   fee_sender = fee P_G + r ek_s, randomness = r P_G, rvk = pgk + alpha P_G, g_epoch (copied), nonce = dk g_epoch.
 * rsks: n * 32 B, sk + alpha mod r_J; dks: n * 32 B, the sender's decryption key.
 * status[i]: 0, or the zk_jubjub_into_xy code (1 / 2 / 3) of a recipient key that fails EncryptionKey::read
 *   (Point::read + as_prime_order); that row's fields, rsk and dk are zero and the other rows are unaffected.
 * ZK_ERR_NOT_CANONICAL (zk_last_error names the array and the lowest index) for an sk, r or alpha >= r_J; ZK_ERR_DECODE
 * for a g_epoch that fails Point::read or is not of prime order (the outputs are then undefined); ZK_ERR_INVALID for NULL. */
int zk_confidential_fields_batch(zk_ctx *ctx, size_t n, const uint8_t *sks, const uint8_t *eks_recipient, const uint32_t *amounts,
                                 const uint32_t *fees, const uint8_t *rs, const uint8_t *alphas, const uint8_t *g_epoch, uint8_t *fields,
                                 uint8_t *rsks, uint8_t *dks, uint8_t *status);
/* the same with device pointers (d_g_epoch: 32 B on the device); asynchronous on the context's stream.  The next zk_ctx_sync
 * reports ZK_ERR_NOT_CANONICAL (a row with an sk, r or alpha >= r_J is left unwritten) or ZK_ERR_DECODE (g_epoch). */
int zk_confidential_fields_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_sks, const uint8_t *d_eks_recipient,
                                        const uint32_t *d_amounts, const uint32_t *d_fees, const uint8_t *d_rs, const uint8_t *d_alphas,
                                        const uint8_t *d_g_epoch, uint8_t *d_fields, uint8_t *d_rsks, uint8_t *d_dks, uint8_t *d_status);
/* The fields of n anonymous transfers: MultiCiphertexts::<Anonymous>::encrypt (core/proofs/src/crypto_components.rs:168-216)
 * placed in ring order as gen_proof places them (core/proofs/src/anonymous.rs:97-145), with ProofContext's rvk and nonce.
 * keys: a table of n_keys 32-byte encryption keys (a wallet's EncKeySet, or a block's account table); NULL only when
 *   n_keys = 0.  Each key an in-range ring index names is read (EncryptionKey::read) once per call; the others are not read.
 * rings: n * 11 uint32 indices into keys, in MultiEncKeys order: [0] the recipient, [1..11) the ten decoys in order.
 * positions: n * 2 bytes, s_index then t_index.  amounts: n uint32 (there is no fee).  sks, rs, alphas: n * 32 B of Fs
 *   (the sender's spending key, the ElGamal randomness r, the re-randomizer alpha).  g_epoch: 32 B.
 * fields: n * 864 B, per row 27 points in the argument order of groth16.AnonymousTx after the member indices:
 *   enc_keys[12] | left_ciphertexts[12] | right_ciphertext | rvk | nonce.  The sender sits at s, the recipient at t, and the
 *   decoys fill the other ten positions in their order.  enc_keys[s] = ek_s = dk P_G, enc_keys at the others are the
 *   table's bytes copied; left_ciphertexts[s] = -amount P_G + r ek_s (neg_encrypt), [t] = amount P_G + r ek_t (encrypt),
 *   a decoy's = r ek_d (encrypt of 0); right_ciphertext = r P_G, rvk = pgk + alpha P_G, nonce = dk g_epoch.
 * rsks: n * 32 B, sk + alpha mod r_J; dks: n * 32 B, the sender's decryption key.
 * status[i]: 0 built; 5 s >= 12, t >= 12 or s = t; 4 a ring index >= n_keys; else 1 / 2 / 3, the zk_jubjub_into_xy code of
 *   the row's first key, in MultiEncKeys order, that fails EncryptionKey::read.  5 comes before 4 and 4 before the key
 *   codes.  A row with a non-zero status gets all-zero fields, rsk and dk; the other rows are unaffected.
 * ZK_ERR_NOT_CANONICAL (zk_last_error names the array and the lowest index) for an sk, r or alpha >= r_J; ZK_ERR_DECODE
 * for a g_epoch that fails Point::read or is not of prime order (the outputs are then undefined); ZK_ERR_INVALID for NULL,
 * and for n above 2^22 or n_keys above 2^24. */
int zk_anonymous_fields_batch(zk_ctx *ctx, size_t n_keys, const uint8_t *keys, size_t n, const uint8_t *sks, const uint32_t *rings,
                              const uint8_t *positions, const uint32_t *amounts, const uint8_t *rs, const uint8_t *alphas,
                              const uint8_t *g_epoch, uint8_t *fields, uint8_t *rsks, uint8_t *dks, uint8_t *status);
/* the same with device pointers (d_rings and d_amounts 4-byte aligned, d_g_epoch: 32 B on the device); asynchronous on the
 * context's stream.  The next zk_ctx_sync reports ZK_ERR_NOT_CANONICAL (a row with an sk, r or alpha >= r_J is left
 * unwritten) or ZK_ERR_DECODE (g_epoch). */
int zk_anonymous_fields_batch_device(zk_ctx *ctx, size_t n_keys, const uint8_t *d_keys, size_t n, const uint8_t *d_sks,
                                     const uint32_t *d_rings, const uint8_t *d_positions, const uint32_t *d_amounts, const uint8_t *d_rs,
                                     const uint8_t *d_alphas, const uint8_t *d_g_epoch, uint8_t *d_fields, uint8_t *d_rsks,
                                     uint8_t *d_dks, uint8_t *d_status);
/* PrivateKey::sign(msg, rng, FixedGenerators::Diversifier) (core/jubjub/src/redjubjub.rs:73-103) for n messages, with the
 * 80 random bytes T of each signature supplied by the caller: ts = n * 80 B.  sks: n * 32 B; msgs / msg_off exactly as
 * zk_redjubjub_verify_batch; sigs: n * 64 B (rbar | sbar).  ZK_ERR_NOT_CANONICAL (naming the lowest index) for an
 * sk >= r_J; ZK_ERR_INVALID for NULL, or for offsets that decrease. */
int zk_redjubjub_sign_batch(zk_ctx *ctx, size_t n, const uint8_t *sks, const uint8_t *ts, const uint8_t *msgs, const uint64_t *msg_off,
                            uint8_t *sigs);
/* the same with device pointers; asynchronous.  The offsets are not checked; an sk >= r_J leaves its signature unwritten
 * and the next zk_ctx_sync reports ZK_ERR_NOT_CANONICAL. */
int zk_redjubjub_sign_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_sks, const uint8_t *d_ts, const uint8_t *d_msgs,
                                   const uint64_t *d_msg_off, uint8_t *d_sigs);
/* ---- wallet keys: zface's hierarchical key derivation (zface/src/derive/mod.rs, a ZIP-32-style scheme) ----------------
 * An extended key is written as 73 B: depth u8 | parent tag 4 B | child index u32 LE | chain code 32 B | key 32 B, the key an
 * sk (32 B Fs, an xsk) or a pgk (a Point::write encoding, an xpgk).  Child indices are raw u32: >= 2^31 is hardened.  All
 * multiples are of the Diversifier generator P_G.  dks / eks are an account's into_decryption_key(pgk) and dk P_G, the
 * keys zk_elgamal_decrypt_batch and zk_confidential_fields_batch take; ek is the account's address.
 * ExtendedSpendingKey::master(seeds[i]) (derive/mod.rs:48-64) for n seeds of any length, laid out as in
 * zk_keys_from_seed_batch.  xsks: n * 73 B.  xpgks (n * 73 B, From<&ExtendedSpendingKey>: the same header with key =
 * sk P_G), dks and eks (n * 32 B) are optional: NULL means not computed.  ZK_ERR_INVALID for a required NULL pointer with
 * n > 0, or for offsets that decrease. */
int zk_xsk_master_batch(zk_ctx *ctx, size_t n, const uint8_t *seeds, const uint64_t *seed_off, uint8_t *xsks, uint8_t *xpgks,
                        uint8_t *dks, uint8_t *eks);
/* the same with device pointers; asynchronous on the context's stream.  The offsets are not checked: they must not decrease. */
int zk_xsk_master_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_seeds, const uint64_t *d_seed_off, uint8_t *d_xsks,
                               uint8_t *d_xpgks, uint8_t *d_dks, uint8_t *d_eks);
/* ExtendedSpendingKey::derive_child (derive/mod.rs:66-104) for n rows: row i derives child child_idx[i] of the xsk
 * parents[parent_idx[i]] (parents: a table of n_parents xsks, NULL only when n_parents = 0).  Scanning accounts is one
 * parent with many indices; a path is one call per level, the previous level's xsks being the next level's parents.
 * Every parent an in-range row names is read once per call (its sk, pgk and tag); the others are not read.
 * xsks: n * 73 B; xpgks (n * 73 B), dks and eks (n * 32 B) as in zk_xsk_master_batch, optional.
 * status[i]: 0 derived; 4 parent_idx >= n_parents; 6 the parent is at depth 255 (its child's depth would not fit in a u8).
 *   A row with a non-zero status gets all-zero outputs; the other rows are unaffected.
 * ZK_ERR_NOT_CANONICAL, zk_last_error naming the lowest such parent index, for a named parent whose sk >= r_J
 * (SpendingKey::read fails); ZK_ERR_INVALID for a required NULL pointer, and for n above 2^26 or n_parents above 2^24. */
int zk_xsk_derive_batch(zk_ctx *ctx, size_t n_parents, const uint8_t *parents, size_t n, const uint32_t *parent_idx,
                        const uint32_t *child_idx, uint8_t *xsks, uint8_t *xpgks, uint8_t *dks, uint8_t *eks, uint8_t *status);
/* the same with device pointers (d_parent_idx and d_child_idx 4-byte aligned); asynchronous on the context's stream.  The
 * rows that name a parent whose sk >= r_J are left unwritten, status included, and the next zk_ctx_sync reports
 * ZK_ERR_NOT_CANONICAL.  No output may overlap d_parents: rows read their parents while other rows write, so a path chains
 * levels through separate buffers, never in place. */
int zk_xsk_derive_batch_device(zk_ctx *ctx, size_t n_parents, const uint8_t *d_parents, size_t n, const uint32_t *d_parent_idx,
                               const uint32_t *d_child_idx, uint8_t *d_xsks, uint8_t *d_xpgks, uint8_t *d_dks, uint8_t *d_eks,
                               uint8_t *d_status);
/* ExtendedProofGenerationKey::derive_child (derive/mod.rs:164-197), the watch-only derivation: parents is a table of
 * n_parents xpgks, and the rows work as in zk_xsk_derive_batch.  xpgks: n * 73 B; dks and eks (n * 32 B) optional.
 * status[i]: 0 derived; 4 parent_idx >= n_parents; else 1 / 2 / 3, the zk_jubjub_into_xy code of a parent whose pgk fails
 *   ProofGenerationKey::read (Point::read + as_prime_order); else 5 for a hardened index (the reference returns an error);
 *   else 6 for a parent at depth 255.  A row with a non-zero status gets all-zero outputs; the other rows are unaffected.
 * ZK_ERR_INVALID for a required NULL pointer, and for n above 2^26 or n_parents above 2^24. */
int zk_xpgk_derive_batch(zk_ctx *ctx, size_t n_parents, const uint8_t *parents, size_t n, const uint32_t *parent_idx,
                         const uint32_t *child_idx, uint8_t *xpgks, uint8_t *dks, uint8_t *eks, uint8_t *status);
/* the same with device pointers (d_parent_idx and d_child_idx 4-byte aligned); asynchronous on the context's stream.  As in
 * zk_xsk_derive_batch_device, no output may overlap d_parents. */
int zk_xpgk_derive_batch_device(zk_ctx *ctx, size_t n_parents, const uint8_t *d_parents, size_t n, const uint32_t *d_parent_idx,
                                const uint32_t *d_child_idx, uint8_t *d_xpgks, uint8_t *d_dks, uint8_t *d_eks, uint8_t *d_status);
/* ---- confidential-transfer balance updates of one block (what modules/encrypted-balances runs around each proof) ------
 * rollover + sub_enc_balance + add_pending_transfer (modules/encrypted-balances/src/lib.rs:25-96, 133-222) for n_tx
 * transactions, in order, over a table of n_accounts accounts.
 * balances / pendings: n_accounts * 64 B (Ciphertext: left | right); acct_flags[a]: bit 0 balance present, bit 1 pending
 * present, bit 2 rollover due (last_rollover < current_epoch, worked out by the caller).  An account is rolled over at its
 * first touch by any transaction, if due: balance = (balance or zero) + (pending or zero), present; pending absent.
 * sender / recipient: n_tx account indices; tx_points: n_tx * 128 B, amount_sender | amount_recipient | fee_sender |
 * randomness; applied[k]: 1 when transaction k passed its checks (the proof verdict), else 0.
 * balance_sender[k]: 64 B, the sender's balance that verify_confidential_proof reads (Ciphertext::zero() when absent).
 * balance_after[k]: 64 B, the sender's balance after the transaction (the ConfidentialTransfer event); written for applied
 *   transactions only, the other entries are left as they are.
 * tx_status[k]: 0 applied (balance -= (amount_sender + fee_sender, 2 randomness), an absent balance staying absent;
 *   pending(recipient) += (amount_recipient, randomness)); 1 not applied (applied[k] = 0); 2 a transaction point fails
 *   Point::read + as_prime_order (not applied: the verifier rejects the same point); 3 sender or recipient >= n_accounts
 *   (not applied, and it touches no account).  When several apply, 3 comes before 2 and 2 before 1.
 * new_balances / new_pendings / new_flags: the state after the block.  Untouched accounts are copied through byte for byte;
 *   a touched account's absent ciphertexts are 64 zero bytes, its flags keep bits 3-7, and bit 2 is cleared.
 * ZK_ERR_DECODE when a touched account's stored ciphertext (balance or pending, when present) fails Ciphertext::read;
 *   zk_last_error names the lowest such account, and the outputs are undefined.  ZK_ERR_INVALID for a NULL ctx, for a NULL
 *   account array when n_accounts > 0 or transaction array when n_tx > 0, and for n_accounts or n_tx above 2^22.  n_tx = 0
 *   gives the state back unchanged. */
int zk_balances_confidential_block(zk_ctx *ctx, size_t n_accounts, const uint8_t *balances, const uint8_t *pendings,
                                   const uint8_t *acct_flags, size_t n_tx, const uint32_t *sender, const uint32_t *recipient,
                                   const uint8_t *tx_points, const uint8_t *applied, uint8_t *balance_sender, uint8_t *balance_after,
                                   uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags);
/* the same with device pointers (d_sender / d_recipient 4-byte aligned); asynchronous on the context's stream.  A touched
 * account that fails to decode is reported by the next zk_ctx_sync (or the next call that reports the context's pending
 * device errors) as ZK_ERR_DECODE, with the account named in zk_last_error */
int zk_balances_confidential_block_device(zk_ctx *ctx, size_t n_accounts, const uint8_t *d_balances, const uint8_t *d_pendings,
                                          const uint8_t *d_acct_flags, size_t n_tx, const uint32_t *d_sender,
                                          const uint32_t *d_recipient, const uint8_t *d_tx_points, const uint8_t *d_applied,
                                          uint8_t *d_balance_sender, uint8_t *d_balance_after, uint8_t *d_tx_status,
                                          uint8_t *d_new_balances, uint8_t *d_new_pendings, uint8_t *d_new_flags);
/* ---- anonymous-transfer state updates of one block (what modules/anonymous-balances runs around each proof) ------------
 * anonymous_transfer (modules/anonymous-balances/src/lib.rs:23-82, 169-232) for n_tx transactions over the module's own
 * account table (AnonymousBalances storage, not EncryptedBalances).  ZK_ANON_RING = 12 members per transaction
 * (core/proofs/src/constants.rs:1; the only ring the shipped anony_vk.dat accepts).  Each transaction rolls over its 12
 * members (at an account's first touch, when due, as zk_balances_confidential_block does; the rollover stands whatever
 * the verdict), then verify_anonymous_proof reads the 12 members' balances, and an applied transaction adds
 * from_left_right(left_i, right_ciphertext) to member i's pending transfer.  A member listed twice is rolled over once and
 * receives both additions.
 * keys: n_accounts * 32 B, each account's EncKey: copied into the verifier inputs, never decoded here.
 * balances / pendings / acct_flags: as zk_balances_confidential_block (bits 0-2: balance, pending, rollover due).
 * members: n_tx * 12 account indices; tx_points: n_tx * 13 * 32 B = left_ciphertexts[0..12) | right_ciphertext;
 * tx_extra: n_tx * 64 B = rvk | nonce; g_epoch: 32 B (LastGEpoch, one value per block).
 * applied: n_tx bytes; transaction k is applied iff applied[k] == 1, so the verdicts of
 *   zk_groth16_verify_points_batch(_device) can be passed unchanged (0, 2, 3 and 4 are all "not applied").
 * enc_balances[k]: 12 * 64 B, the acc[] that verify_anonymous_proof reads (Ciphertext::zero() when absent).
 * verify_points[k]: 52 * 32 B in verify_anonymous_proof's push order (12 keys, 12 left ciphertexts, the 12 acc left
 *   points, the 12 acc right points, right_ciphertext, rvk, g_epoch, nonce), ready for zk_groth16_verify_points_batch with
 *   n_points = 52.  What the verifier reads does not depend on applied.
 * tx_status[k]: 0 applied; 1 not applied (applied[k] != 1); 2 a left / right point fails Point::read + as_prime_order (not
 *   applied); 3 a member index >= n_accounts (the transaction touches nothing; its enc_balances and verify_points rows are
 *   zero).  3 comes before 2 and 2 before 1.
 * new_balances / new_pendings / new_flags: as zk_balances_confidential_block.
 * ZK_ERR_DECODE when a touched account's stored ciphertext fails Ciphertext::read; zk_last_error names the lowest such
 *   account, and the outputs are undefined.  ZK_ERR_INVALID for a NULL ctx, for a NULL account array when n_accounts > 0
 *   or transaction array (g_epoch included) when n_tx > 0, for n_accounts above 2^22 and for n_tx above 2^18. */
#define ZK_ANON_RING 12
int zk_balances_anonymous_block(zk_ctx *ctx, size_t n_accounts, const uint8_t *keys, const uint8_t *balances, const uint8_t *pendings,
                                const uint8_t *acct_flags, size_t n_tx, const uint32_t *members, const uint8_t *tx_points,
                                const uint8_t *tx_extra, const uint8_t *g_epoch, const uint8_t *applied, uint8_t *enc_balances,
                                uint8_t *verify_points, uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags);
/* the same with device pointers (d_members 4-byte aligned); asynchronous on the context's stream.  A touched account that
 * fails to decode is reported by the next zk_ctx_sync as ZK_ERR_DECODE, with the account named in zk_last_error */
int zk_balances_anonymous_block_device(zk_ctx *ctx, size_t n_accounts, const uint8_t *d_keys, const uint8_t *d_balances,
                                       const uint8_t *d_pendings, const uint8_t *d_acct_flags, size_t n_tx, const uint32_t *d_members,
                                       const uint8_t *d_tx_points, const uint8_t *d_tx_extra, const uint8_t *d_g_epoch,
                                       const uint8_t *d_applied, uint8_t *d_enc_balances, uint8_t *d_verify_points, uint8_t *d_tx_status,
                                       uint8_t *d_new_balances, uint8_t *d_new_pendings, uint8_t *d_new_flags);
/* ---- both calls of modules/anonymous-balances in one block ---------------------------------------------------------------
 * anonymous_transfer and issue (modules/anonymous-balances/src/lib.rs:23-134) for n_tx transactions in block order: the
 * arguments of zk_balances_anonymous_block, plus
 * kind[k]: 0 anonymous_transfer, 1 issue.  An issue uses members[12 k] as its issuer (the other 11 entries are ignored),
 *   slot 0 of its tx_points row as total and slot 12 as randomness (the other slots are ignored); its tx_extra row is
 *   ignored.  The caller builds an issue's 11 verifier points from its extrinsic fields (verify_confidential_proof over
 *   (issuer, issuer, total, total, balance, rvk, fee, randomness, nonce)) and checks it with the confidential key.
 * issued[k]: 64 B, the Issued event's ciphertext from_left_right(total, randomness) as Point::write encodings; written for
 *   applied issues only, other entries are left as they are.
 * An applied issue sets the issuer's balance to that ciphertext and touches nothing else: no rollover, the pending balance
 *   and the due bit stay.  So the balance a transfer reads for member m is the last applied issue to m after m's first
 *   transfer touch and before the transfer, else m's rolled balance, where the rollover at the first touch starts from the
 *   last applied issue before it (or the stored balance).  The final balance follows the same rule at the end of the block.
 * tx_status[k]: as zk_balances_anonymous_block for a transfer.  An issue: 3 the issuer >= n_accounts, or an unknown kind; 2
 *   total or randomness fails Point::read + as_prime_order; 1 not applied (applied[k] != 1); 0 applied.  3 comes before 2
 *   and 2 before 1.  An issue's and an unknown kind's enc_balances and verify_points rows are zero bytes.
 * new_balances / new_pendings / new_flags: as zk_balances_anonymous_block.  An account only issues name is never decoded:
 *   without an applied issue it is copied through byte for byte; with one, its balance is the last issued encoding, its
 *   pending bytes are copied, and its flags gain bit 0 (bit 2 stays).
 * ZK_ERR_DECODE as zk_balances_anonymous_block: an account a transfer touches must have stored ciphertexts that read, even
 *   when an issue before the touch replaces the stored balance.  ZK_ERR_INVALID as zk_balances_anonymous_block, and for a
 *   NULL kind or issued when n_tx > 0.  With no issue and no unknown kind the outputs are zk_balances_anonymous_block's. */
#define ZK_ANON_TRANSFER 0
#define ZK_ANON_ISSUE 1
int zk_anonymous_calls_block(zk_ctx *ctx, size_t n_accounts, const uint8_t *keys, const uint8_t *balances, const uint8_t *pendings,
                             const uint8_t *acct_flags, size_t n_tx, const uint8_t *kind, const uint32_t *members, const uint8_t *tx_points,
                             const uint8_t *tx_extra, const uint8_t *g_epoch, const uint8_t *applied, uint8_t *enc_balances,
                             uint8_t *verify_points, uint8_t *issued, uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings,
                             uint8_t *new_flags);
/* the same with device pointers (d_members 4-byte aligned); asynchronous on the context's stream.  A touched account that
 * fails to decode is reported by the next zk_ctx_sync as ZK_ERR_DECODE, with the account named in zk_last_error */
int zk_anonymous_calls_block_device(zk_ctx *ctx, size_t n_accounts, const uint8_t *d_keys, const uint8_t *d_balances,
                                    const uint8_t *d_pendings, const uint8_t *d_acct_flags, size_t n_tx, const uint8_t *d_kind,
                                    const uint32_t *d_members, const uint8_t *d_tx_points, const uint8_t *d_tx_extra,
                                    const uint8_t *d_g_epoch, const uint8_t *d_applied, uint8_t *d_enc_balances, uint8_t *d_verify_points,
                                    uint8_t *d_issued, uint8_t *d_tx_status, uint8_t *d_new_balances, uint8_t *d_new_pendings,
                                    uint8_t *d_new_flags);
/* ---- encrypted-asset calls of one block (what modules/encrypted-assets runs around each proof) --------------------------
 * confidential_transfer, issue and destroy (modules/encrypted-assets/src/lib.rs:32-215, 266-358) for n_tx transactions, in
 * order, over a table of n_slots slots: one slot per (AssetId, EncKey), numbered by the caller.
 * balances / pendings: n_slots * 64 B; slot_flags[s]: bit 0 balance present, bit 1 pending present, bit 2 rollover due
 *   (LastRollOver, or 0 when absent, < current_epoch, worked out by the caller); bits 3-7 are kept.
 * kind[k]: 0 confidential_transfer, 1 issue, 2 destroy.
 * slot_a[k]: the sender's slot, the issuer's (new asset id, issuer) slot, or the owner's slot; slot_b[k]: the recipient's
 *   slot, read for transfers only.  Asset ids come from the caller, who knows the issue verdicts before choosing the
 *   issuer's slot; nothing here numbers assets.
 * tx_points: n_tx * 128 B.  Transfer: amount_sender | amount_recipient | fee_sender | randomness; issue: total | ignored |
 *   ignored | randomness; destroy: ignored.
 * applied[k]: transaction k is applied iff applied[k] == 1, so verifier verdicts pass unchanged.
 * A transfer rolls over its sender, then its recipient, at a due slot's first transfer touch (balance = (balance or zero) +
 *   (pending or zero), present; pending absent; the rollover stands whatever the verdict), then, when applied, balance(a)
 *   -= (amount_sender + fee_sender, 2 randomness), an absent balance staying absent, and pending(b) += (amount_recipient,
 *   randomness).  An applied issue sets balance(a) = (total, randomness) (TotalSupply holds the same ciphertext); an applied
 *   destroy takes balance(a) and pending(a), both absent after.  Neither rolls over, and neither clears the due bit.
 * balance_sender[k]: 64 B.  A transfer: the sender's balance verify_confidential_proof reads (Ciphertext::zero() when
 *   absent); 64 zero bytes for the other kinds.
 * balance_after[k]: 64 B, the sender's balance after an applied transfer (the event); other entries are left as they are.
 * event_ct[k] / event_flags[k]: 128 B / 1 B, written for applied issues and destroys only.  An issue: its total ciphertext
 *   | 64 zero bytes, flags 1.  A destroy: the taken balance | the taken pending, an absent one as 64 zero bytes; flags bit 0
 *   / bit 1 tell which were present.
 * tx_status[k]: 0 applied; 1 not applied (applied[k] != 1); 2 a point the call reads fails Point::read + as_prime_order (a
 *   transfer's four, an issue's total and randomness; not applied, and a transfer's rollovers still stand); 3 a slot index
 *   >= n_slots or an unknown kind (the transaction touches nothing).  3 comes before 2 and 2 before 1.
 * new_balances / new_pendings / new_flags: the state after the block.  A slot no valid transaction names is copied through
 *   byte for byte; a named slot's absent ciphertexts are 64 zero bytes, its flags keep bits 3-7, and bit 2 is cleared only
 *   when a transfer touched it.
 * Every ciphertext written is a Point::write encoding.  Where the module moves stored bytes unchanged (a rollover into an
 *   absent balance, destroy's take), this differs only for an identity point stored with the x-sign bit set, which
 *   Point::read accepts.
 * ZK_ERR_DECODE when a named slot's stored ciphertext (balance or pending, when present) fails Ciphertext::read;
 *   zk_last_error names the lowest such slot, and the outputs are undefined.  ZK_ERR_INVALID for a NULL ctx, for a NULL
 *   slot array when n_slots > 0 or transaction array when n_tx > 0, for n_slots above 2^22 and for n_tx above 2^20 (6 sort
 *   elements per transaction).  n_tx = 0 gives the state back unchanged. */
int zk_assets_block(zk_ctx *ctx, size_t n_slots, const uint8_t *balances, const uint8_t *pendings, const uint8_t *slot_flags,
                    size_t n_tx, const uint8_t *kind, const uint32_t *slot_a, const uint32_t *slot_b, const uint8_t *tx_points,
                    const uint8_t *applied, uint8_t *balance_sender, uint8_t *balance_after, uint8_t *event_ct, uint8_t *event_flags,
                    uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags);
/* the same with device pointers (d_slot_a / d_slot_b 4-byte aligned); asynchronous on the context's stream.  A named slot
 * that fails to decode is reported by the next zk_ctx_sync as ZK_ERR_DECODE, with the slot named in zk_last_error */
int zk_assets_block_device(zk_ctx *ctx, size_t n_slots, const uint8_t *d_balances, const uint8_t *d_pendings, const uint8_t *d_slot_flags,
                           size_t n_tx, const uint8_t *d_kind, const uint32_t *d_slot_a, const uint32_t *d_slot_b, const uint8_t *d_tx_points,
                           const uint8_t *d_applied, uint8_t *d_balance_sender, uint8_t *d_balance_after, uint8_t *d_event_ct,
                           uint8_t *d_event_flags, uint8_t *d_tx_status, uint8_t *d_new_balances, uint8_t *d_new_pendings,
                           uint8_t *d_new_flags);
/* ---- block import: the proofs and the state of encrypted-balances / encrypted-assets transfers in one call ----------------
 * A transfer's proof is checked against the sender's balance at that transaction, which depends on which of the sender's
 * earlier transfers passed.  So the call runs rounds: every transfer starts undecided and counts as applied; each round
 * runs the state pass with the current mask, verifies the undecided transfers against the balance_sender it gives
 * (zk_groth16_verify_points_batch with 11 points), and in each chain (the transfers of one sender) decides the undecided
 * transfers up to and including the first whose verdict is not 1; the rest waits for the next round.  A round without a
 * failure ends the import with its state pass; a round that leaves nothing undecided is followed by one last state pass.
 * A block takes 1 + (the most failures in one chain) rounds at most, one fewer when those failures end the chain, and one
 * when nothing fails; a block without transfers takes none.
 *
 * zk_import_confidential_block: the arguments of zk_balances_confidential_block, with the verifier's inputs in place of
 *   tx_points and applied.
 * rows: n_tx * 11 * 32 B, each transfer's verifier points in verify_confidential_proof's push order (address_sender,
 *   address_recipient, amount_sender, amount_recipient, randomness, fee_sender, balance_sender left, balance_sender right,
 *   rvk, g_epoch, nonce).  Slots 6-7 are ignored: the call fills them from the state.  The state pass's tx_points are
 *   slots 2, 3, 5, 4.
 * proofs: n_tx * 192 B.  pvk: a prepared key of 11-point proofs on the context's device, ready to use.
 * verdicts[k]: the verdict of transaction k, as zk_groth16_verify_points_batch gives it (1 passes).
 * balance_after, tx_status, new_balances, new_pendings, new_flags: zk_balances_confidential_block's outputs for the final
 *   mask; balance_after is zero for a transaction that is not applied.
 * rounds: the number of verification launches (may be NULL).
 * ZK_ERR_INVALID, naming the lowest such transaction in zk_last_error, when a sender or recipient is >= n_accounts; and as
 *   zk_balances_confidential_block for NULL arguments and sizes.  ZK_ERR_MALFORMED_VK for a key of other than 11 points.
 *   ZK_ERR_DECODE as zk_balances_confidential_block; the outputs are then undefined. */
int zk_import_confidential_block(zk_ctx *ctx, const zk_pvk *pvk, size_t n_accounts, const uint8_t *balances, const uint8_t *pendings,
                                 const uint8_t *acct_flags, size_t n_tx, const uint32_t *sender, const uint32_t *recipient,
                                 const uint8_t *rows, const uint8_t *proofs, uint8_t *verdicts, uint8_t *balance_after, uint8_t *tx_status,
                                 uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags, unsigned *rounds);
/* the same with device pointers (d_sender / d_recipient 4-byte aligned; rounds is a host pointer).  The call blocks on the
 * context's stream before the first round and after each round, to read a block of four counters, and returns with the
 * outputs complete; it reports ZK_ERR_DECODE itself. */
int zk_import_confidential_block_device(zk_ctx *ctx, const zk_pvk *pvk, size_t n_accounts, const uint8_t *d_balances,
                                        const uint8_t *d_pendings, const uint8_t *d_acct_flags, size_t n_tx, const uint32_t *d_sender,
                                        const uint32_t *d_recipient, const uint8_t *d_rows, const uint8_t *d_proofs, uint8_t *d_verdicts,
                                        uint8_t *d_balance_after, uint8_t *d_tx_status, uint8_t *d_new_balances, uint8_t *d_new_pendings,
                                        uint8_t *d_new_flags, unsigned *rounds);
/* zk_import_assets_block: the transfer rounds over zk_assets_block, with chains keyed by the sender slot (slot_a).  The
 *   arguments of zk_assets_block, with rows, proofs and fixed_verdicts in place of applied.  Asset ids and slots are the
 *   caller's, as for zk_assets_block: they depend on the issue verdicts, which the caller has before the call.
 * rows / proofs: as zk_import_confidential_block, read at transfers only.
 * fixed_verdicts[k]: the verdict of issue or destroy k: 1 passes and is applied, any other byte fails; ignored at transfers.
 * verdicts[k]: fixed_verdicts[k] for an issue or destroy, byte for byte, the transfer's verdict otherwise.  verdicts may be
 *   the fixed_verdicts buffer itself.
 * balance_after, event_ct, event_flags, tx_status, new_balances, new_pendings, new_flags: zk_assets_block's outputs for the
 *   final mask, with zero bytes where it writes nothing.
 * ZK_ERR_INVALID, naming the lowest such transaction, for an unknown kind, a transfer's slot_a or slot_b >= n_slots, or a
 *   passing issue's or destroy's slot_a >= n_slots (a failing one's slots are ignored); otherwise as
 *   zk_import_confidential_block. */
int zk_import_assets_block(zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const uint8_t *balances, const uint8_t *pendings,
                           const uint8_t *slot_flags, size_t n_tx, const uint8_t *kind, const uint32_t *slot_a, const uint32_t *slot_b,
                           const uint8_t *tx_points, const uint8_t *rows, const uint8_t *proofs, const uint8_t *fixed_verdicts,
                           uint8_t *verdicts, uint8_t *balance_after, uint8_t *event_ct, uint8_t *event_flags, uint8_t *tx_status,
                           uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags, unsigned *rounds);
/* the same with device pointers, blocking as zk_import_confidential_block_device does */
int zk_import_assets_block_device(zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const uint8_t *d_balances, const uint8_t *d_pendings,
                                  const uint8_t *d_slot_flags, size_t n_tx, const uint8_t *d_kind, const uint32_t *d_slot_a,
                                  const uint32_t *d_slot_b, const uint8_t *d_tx_points, const uint8_t *d_rows, const uint8_t *d_proofs,
                                  const uint8_t *d_fixed_verdicts, uint8_t *d_verdicts, uint8_t *d_balance_after, uint8_t *d_event_ct,
                                  uint8_t *d_event_flags, uint8_t *d_tx_status, uint8_t *d_new_balances, uint8_t *d_new_pendings,
                                  uint8_t *d_new_flags, unsigned *rounds);
/* zk_import_asset_calls: a block of encrypted-asset calls from the slot table as the module stores it and each transaction
 *   as its extrinsic carries it.  The call verifies the issues and destroys (zk_groth16_verify_points_batch, 11 points),
 *   numbers the passing issues, resolves every (AssetId, EncKey) a transaction names to a row of the slot table, appending
 *   new rows, and runs zk_import_assets_block's rounds on the grown table with those verdicts fixed.
 * Slot table, n_slots rows: slot_ids (uint32 AssetId), slot_keys (32 B EncKey); balances, pendings, slot_flags as
 *   zk_assets_block.  (slot_ids[r], slot_keys[r]) must be distinct across rows.
 * next_asset_id: NextAssetId before the block.  new_slot_flags: the flags of a row the block creates, less bits 0-1
 *   (ACCOUNT_DUE when current_epoch > 0).
 * kind[k]: 0 transfer, 1 issue, 2 destroy.  asset_id[k]: read at transfers and destroys, ignored at issues.
 * rows: n_tx * 11 * 32 B in zk_import_confidential_block's order, the only source of a transaction's fields: slot 0 is the
 *   sender, issuer or owner; slot 1 the recipient (read at transfers); an issue's total and randomness are slots 2 and 4.
 *   Slots 6-7 are ignored at transfers (the rounds fill them from the state) and read at issues and destroys (balance /
 *   dummy_balance).  proofs: n_tx * 192 B.  pvk: the 11-point key of all three kinds, on the context's device, ready to use.
 * A passing issue (verdict 1) gets the id next_asset_id + (the passing issues before it) and references (its id, issuer); a
 *   passing destroy references (asset_id, owner); a transfer (asset_id, sender) and (asset_id, recipient).  A failing issue
 *   or destroy references nothing and consumes no id.  A key in the table maps to its row; a new key gets row n_slots + (the
 *   new keys whose first reference comes earlier, in block order, sender before recipient), zero ciphertexts and flags
 *   new_slot_flags & ~3.
 * Outputs: verdicts, balance_after, event_ct, event_flags, tx_status, new_balances, new_pendings, new_flags as
 *   zk_import_assets_block, on the grown table; asset_ids[k]: the id of passing issue k, 0 elsewhere; new_slot_ids /
 *   new_slot_keys: the grown table's (id, key) per row, the first n_slots rows copied; *n_slots_out: its rows.  The table
 *   outputs need room for n_slots + 2 * n_tx rows.  rounds: as zk_import_assets_block (may be NULL).
 * ZK_ERR_INVALID, naming the lowest such transaction or row in zk_last_error, for an unknown kind, a passing issue whose id
 *   would pass 2^32 - 1, a table row whose (id, key) equals an earlier row's, and more than 2^22 rows after the block; for
 *   NULL arguments (n_slots_out always, the table's when n_slots > 0, the transactions' when n_tx > 0, the table outputs
 *   when either is) and sizes as zk_assets_block.  ZK_ERR_MALFORMED_VK for a key of other than 11 points.  ZK_ERR_DECODE
 *   as zk_assets_block; the outputs are then undefined. */
int zk_import_asset_calls(zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const uint32_t *slot_ids, const uint8_t *slot_keys,
                          const uint8_t *balances, const uint8_t *pendings, const uint8_t *slot_flags, uint32_t next_asset_id,
                          uint8_t new_slot_flags, size_t n_tx, const uint8_t *kind, const uint32_t *asset_id, const uint8_t *rows,
                          const uint8_t *proofs, uint8_t *verdicts, uint32_t *asset_ids, uint8_t *balance_after, uint8_t *event_ct,
                          uint8_t *event_flags, uint8_t *tx_status, uint32_t *new_slot_ids, uint8_t *new_slot_keys, uint8_t *new_balances,
                          uint8_t *new_pendings, uint8_t *new_flags, size_t *n_slots_out, unsigned *rounds);
/* the same with device pointers (the uint32 arrays 4-byte aligned; n_slots_out and rounds are host pointers).  The call
 * blocks on the context's stream twice before the rounds, to read a block of counters: after checking the kinds and the
 * table (the number of issues and destroys sizes their verification), and after resolving the slots (the new rows, an id
 * overflow); then as zk_import_assets_block_device.  It returns with the outputs complete. */
int zk_import_asset_calls_device(zk_ctx *ctx, const zk_pvk *pvk, size_t n_slots, const uint32_t *d_slot_ids, const uint8_t *d_slot_keys,
                                 const uint8_t *d_balances, const uint8_t *d_pendings, const uint8_t *d_slot_flags, uint32_t next_asset_id,
                                 uint8_t new_slot_flags, size_t n_tx, const uint8_t *d_kind, const uint32_t *d_asset_id, const uint8_t *d_rows,
                                 const uint8_t *d_proofs, uint8_t *d_verdicts, uint32_t *d_asset_ids, uint8_t *d_balance_after,
                                 uint8_t *d_event_ct, uint8_t *d_event_flags, uint8_t *d_tx_status, uint32_t *d_new_slot_ids,
                                 uint8_t *d_new_slot_keys, uint8_t *d_new_balances, uint8_t *d_new_pendings, uint8_t *d_new_flags,
                                 size_t *n_slots_out, unsigned *rounds);
/* ---- block import: the proofs and the state of anonymous-balances calls in one call -------------------------------------
 * zk_import_anonymous_block: anonymous_transfer and issue in block order, verified and applied.  No rounds: an issue's
 * proof reads only its own fields, and a transfer changes pending balances only, so nothing a proof is checked against
 * depends on a transfer's verdict.  The call verifies the issues (zk_groth16_verify_points_batch with conf_pvk, 11
 * points), runs the state pass (zk_anonymous_calls_block) with the issue verdicts as the mask and no transfer applied,
 * verifies the transfers on the 52 points that pass gives (anon_pvk), and runs the state pass again with all the verdicts.
 * A block without issues takes zk_balances_anonymous_block's passes; a block without transfers ends after the first pass.
 *
 * The arguments of zk_anonymous_calls_block, with the verifier's inputs in place of applied:
 * kind: as zk_anonymous_calls_block (0 transfer, 1 issue); NULL: every transaction is a transfer.
 * tx_extra[k]: rvk | nonce, read for issues too.
 * issue_fields: n_tx * 96 B, an issue's fee | balance; read at issues only, may be NULL when the block has no issue.
 * proofs: n_tx * 192 B.  anon_pvk: a prepared key of 52-point proofs; conf_pvk: one of 11-point proofs, or NULL when the
 *   block has no issue.  Both on the context's device, ready to use.
 * verdicts[k]: as zk_groth16_verify_points_batch gives it (1 passes).  An issue's from conf_pvk on (issuer, issuer, total,
 *   total, randomness, fee, balance, rvk, g_epoch, nonce), with issuer = keys[members[12 k]], total and randomness slots 0
 *   and 12 of its tx_points row; a transfer's from anon_pvk on its 52 verify_points of the first state pass.
 * enc_balances, issued, tx_status, new_balances, new_pendings, new_flags: zk_anonymous_calls_block's outputs for the final
 *   verdicts; issued is zero bytes where nothing is written.
 * ZK_ERR_INVALID, naming the lowest such transaction in zk_last_error, for an unknown kind, a transfer's member >=
 *   n_accounts, an issuer >= n_accounts (an issue's other 11 member entries are ignored), or an issue when conf_pvk or
 *   issue_fields is NULL; and as zk_anonymous_calls_block for NULL arguments (kind excepted) and sizes.
 *   ZK_ERR_MALFORMED_VK for an anon_pvk of other than 52 points or a conf_pvk of other than 11.  ZK_ERR_DECODE as
 *   zk_anonymous_calls_block; the outputs are then undefined. */
int zk_import_anonymous_block(zk_ctx *ctx, const zk_pvk *anon_pvk, const zk_pvk *conf_pvk, size_t n_accounts, const uint8_t *keys,
                              const uint8_t *balances, const uint8_t *pendings, const uint8_t *acct_flags, size_t n_tx, const uint8_t *kind,
                              const uint32_t *members, const uint8_t *tx_points, const uint8_t *tx_extra, const uint8_t *issue_fields,
                              const uint8_t *g_epoch, const uint8_t *proofs, uint8_t *verdicts, uint8_t *enc_balances, uint8_t *issued,
                              uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags);
/* the same with device pointers (d_members 4-byte aligned).  The call blocks on the context's stream once, to read the
 * number of issues and of transfers and the lowest bad transaction, and returns with the outputs complete; it reports
 * ZK_ERR_DECODE itself. */
int zk_import_anonymous_block_device(zk_ctx *ctx, const zk_pvk *anon_pvk, const zk_pvk *conf_pvk, size_t n_accounts, const uint8_t *d_keys,
                                     const uint8_t *d_balances, const uint8_t *d_pendings, const uint8_t *d_acct_flags, size_t n_tx,
                                     const uint8_t *d_kind, const uint32_t *d_members, const uint8_t *d_tx_points, const uint8_t *d_tx_extra,
                                     const uint8_t *d_issue_fields, const uint8_t *d_g_epoch, const uint8_t *d_proofs, uint8_t *d_verdicts,
                                     uint8_t *d_enc_balances, uint8_t *d_issued, uint8_t *d_tx_status, uint8_t *d_new_balances,
                                     uint8_t *d_new_pendings, uint8_t *d_new_flags);
/* ---- block import: the signatures and all three zk pallets' calls in one call --------------------------------------------
 * zk_import_block: what Executive::execute_block needs from the zk pallets for one block.  It checks every extrinsic's
 * signature (the block is rejected if one fails, modules/executive/src/lib.rs:168-183), then imports the block's
 * confidential transfers, encrypted-asset calls and anonymous-balances calls.  The pallets keep disjoint storage, so
 * each section's outputs equal, byte for byte, those of its own call on the same arguments:
 * zk_import_confidential_block, zk_import_asset_calls and zk_import_anonymous_block.  The call shares verifier launches
 * across sections.  L1 (conf_pvk) verifies the confidential transfers' first round, every asset issue and destroy, and
 * every anonymous issue.  One launch with anon_pvk verifies the anonymous transfers.  Each later conf_pvk launch verifies
 * the undecided transfers of both chain-keyed sections: confidential round r with asset round r - 1.  That is
 * max(R_conf, 1 + R_assets) launches with conf_pvk, R being a section's rounds in its own call, plus one with anon_pvk;
 * a launch with no proofs is skipped.
 *
 * Arguments, in order:
 *   conf_pvk: the 11-point key of the confidential transfers, the asset calls and the anonymous issues; may be NULL when
 *     no section has a transaction that uses it.  anon_pvk: the 52-point key; may be NULL when the anonymous section has
 *     no transaction.  Each key passed must have its shape (ZK_ERR_MALFORMED_VK).
 *   the signatures: n_sig, vks, sigs, msgs, msg_off, zs exactly as zk_redjubjub_batch_verify takes them (one per
 *     extrinsic, checked with FixedGenerators::Diversifier).
 *   c_*: zk_import_confidential_block's arguments less ctx and pvk; a_*: zk_import_asset_calls's less ctx and pvk;
 *     an_*: zk_import_anonymous_block's less ctx and the keys.  A section with no rows and no transactions is empty
 *     and needs no pointers beyond what its own call needs at zero size.
 *   first_bad_sig: the lowest extrinsic whose signature fails, n_sig when none does (may be NULL).
 *   launches: the verifier launches the call made, with both keys (may be NULL).
 * Checks, in this order:
 *   1. NULL arguments and sizes, per section as each call checks them (ZK_ERR_INVALID).
 *   2. Each section's kinds and indices (ZK_ERR_INVALID; zk_last_error names the section and the lowest transaction or
 *      table row, e.g. "zk_import_block: assets: transaction 17: ...").
 *   3. The signatures, as redjubjub_verify_batched: the batch check, then the per-signature verdicts when it fails.
 *      If any verdict is not 1 the call returns ZK_ERR_BAD_SIGNATURE.  It then verifies no proof and writes no
 *      output; zk_last_error names the extrinsic and its verdict (0 / 2 / 3 / 4).  Every z_i is checked first: a
 *      z_i >= r_J gives ZK_ERR_NOT_CANONICAL, naming the lowest such extrinsic.
 *   4. The proofs and the state passes.  The asset section's id overflow and table size (ZK_ERR_INVALID) and a
 *      stored ciphertext that does not read (ZK_ERR_DECODE) are reported as each call reports them. */
int zk_import_block(zk_ctx *ctx, const zk_pvk *conf_pvk, const zk_pvk *anon_pvk, size_t n_sig, const uint8_t *vks, const uint8_t *sigs,
                    const uint8_t *msgs, const uint64_t *msg_off, const uint8_t *zs, size_t c_n_accounts, const uint8_t *c_balances,
                    const uint8_t *c_pendings, const uint8_t *c_acct_flags, size_t c_n_tx, const uint32_t *c_sender,
                    const uint32_t *c_recipient, const uint8_t *c_rows, const uint8_t *c_proofs, uint8_t *c_verdicts,
                    uint8_t *c_balance_after, uint8_t *c_tx_status, uint8_t *c_new_balances, uint8_t *c_new_pendings, uint8_t *c_new_flags,
                    unsigned *c_rounds, size_t a_n_slots, const uint32_t *a_slot_ids, const uint8_t *a_slot_keys, const uint8_t *a_balances,
                    const uint8_t *a_pendings, const uint8_t *a_slot_flags, uint32_t a_next_asset_id, uint8_t a_new_slot_flags,
                    size_t a_n_tx, const uint8_t *a_kind, const uint32_t *a_asset_id, const uint8_t *a_rows, const uint8_t *a_proofs,
                    uint8_t *a_verdicts, uint32_t *a_asset_ids, uint8_t *a_balance_after, uint8_t *a_event_ct, uint8_t *a_event_flags,
                    uint8_t *a_tx_status, uint32_t *a_new_slot_ids, uint8_t *a_new_slot_keys, uint8_t *a_new_balances,
                    uint8_t *a_new_pendings, uint8_t *a_new_flags, size_t *a_n_slots_out, unsigned *a_rounds, size_t an_n_accounts,
                    const uint8_t *an_keys, const uint8_t *an_balances, const uint8_t *an_pendings, const uint8_t *an_acct_flags,
                    size_t an_n_tx, const uint8_t *an_kind, const uint32_t *an_members, const uint8_t *an_tx_points,
                    const uint8_t *an_tx_extra, const uint8_t *an_issue_fields, const uint8_t *an_g_epoch, const uint8_t *an_proofs,
                    uint8_t *an_verdicts, uint8_t *an_enc_balances, uint8_t *an_issued, uint8_t *an_tx_status, uint8_t *an_new_balances,
                    uint8_t *an_new_pendings, uint8_t *an_new_flags, size_t *first_bad_sig, unsigned *launches);
/* the same with device pointers (the uint32 and uint64 arrays aligned to their size; c_rounds, a_n_slots_out, a_rounds,
 * first_bad_sig and launches are host pointers; msg_off is not checked and must not decrease).  The call blocks on the
 * context's stream to read a block of counters: once before L1 (every section's kinds and indices, and the batch
 * verdict of the signatures), once more when that batch check fails, once after L1 when the confidential transfers
 * took part in it or the block has an asset section, and once after each later launch.  It returns with the outputs complete. */
int zk_import_block_device(zk_ctx *ctx, const zk_pvk *conf_pvk, const zk_pvk *anon_pvk, size_t n_sig, const uint8_t *d_vks,
                           const uint8_t *d_sigs, const uint8_t *d_msgs, const uint64_t *d_msg_off, const uint8_t *d_zs, size_t c_n_accounts,
                           const uint8_t *d_c_balances, const uint8_t *d_c_pendings, const uint8_t *d_c_acct_flags, size_t c_n_tx,
                           const uint32_t *d_c_sender, const uint32_t *d_c_recipient, const uint8_t *d_c_rows, const uint8_t *d_c_proofs,
                           uint8_t *d_c_verdicts, uint8_t *d_c_balance_after, uint8_t *d_c_tx_status, uint8_t *d_c_new_balances,
                           uint8_t *d_c_new_pendings, uint8_t *d_c_new_flags, unsigned *c_rounds, size_t a_n_slots,
                           const uint32_t *d_a_slot_ids, const uint8_t *d_a_slot_keys, const uint8_t *d_a_balances,
                           const uint8_t *d_a_pendings, const uint8_t *d_a_slot_flags, uint32_t a_next_asset_id, uint8_t a_new_slot_flags,
                           size_t a_n_tx, const uint8_t *d_a_kind, const uint32_t *d_a_asset_id, const uint8_t *d_a_rows,
                           const uint8_t *d_a_proofs, uint8_t *d_a_verdicts, uint32_t *d_a_asset_ids, uint8_t *d_a_balance_after,
                           uint8_t *d_a_event_ct, uint8_t *d_a_event_flags, uint8_t *d_a_tx_status, uint32_t *d_a_new_slot_ids,
                           uint8_t *d_a_new_slot_keys, uint8_t *d_a_new_balances, uint8_t *d_a_new_pendings, uint8_t *d_a_new_flags,
                           size_t *a_n_slots_out, unsigned *a_rounds, size_t an_n_accounts, const uint8_t *d_an_keys,
                           const uint8_t *d_an_balances, const uint8_t *d_an_pendings, const uint8_t *d_an_acct_flags, size_t an_n_tx,
                           const uint8_t *d_an_kind, const uint32_t *d_an_members, const uint8_t *d_an_tx_points,
                           const uint8_t *d_an_tx_extra, const uint8_t *d_an_issue_fields, const uint8_t *d_an_g_epoch,
                           const uint8_t *d_an_proofs, uint8_t *d_an_verdicts, uint8_t *d_an_enc_balances, uint8_t *d_an_issued,
                           uint8_t *d_an_tx_status, uint8_t *d_an_new_balances, uint8_t *d_an_new_pendings, uint8_t *d_an_new_flags,
                           size_t *first_bad_sig, unsigned *launches);
/* Engine::pairing (core/pairing/src/lib.rs:108-115, bls12_381/mod.rs:40-160) for n pairs of checked G1Uncompressed /
 * G2Uncompressed encodings; out: n * 576 bytes in Fq12::write order (fq12.rs:29-45). */
int zk_pairing_batch(zk_ctx *ctx, size_t n, const uint8_t *g1, const uint8_t *g2, uint8_t *out);

#ifdef __cplusplus
}
#endif
#endif /* ZKB200_H */
