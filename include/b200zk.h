/* b200zk.h -- C ABI of the H100-native Groth16 proving hot path (BN254).
 *
 * This is the drop-in boundary for the reference's hot path.  The reference (100% Rust, CPU only)
 * has no FFI of its own; each entry point below names the Rust item whose *body* it replaces, and
 * INTEGRATION.md shows the `extern "C"` block + call-site change a maintainer would add.
 *
 * Data layout (identical to arkworks' in-memory representation, so Rust slices can be passed
 * as-is with `as_ptr() as *const u64`):
 *   Fr / Fq element : 4 x u64 little-endian limbs, Montgomery form (R = 2^256)
 *   G1 affine       : x || y                       (8 limbs, 64 B)
 *   G2 affine       : x.c0 || x.c1 || y.c0 || y.c1 (16 limbs, 128 B)
 *   infinity        : all-zero coordinates (zkey convention, ark-circom/src/zkey.rs:353-373);
 *                     result points additionally report it through `*out_is_inf`.
 * Ownership: the caller owns every host buffer for the duration of the call (borrow semantics
 * of the Rust slices); the library owns all device memory behind `ctx` / `pk`.
 * Threading: calls that name different `stream` slots (0..2 = MultiplexedStreamID::{Zero,One,Two},
 * mpc-net/src/lib.rs:29-33) may be issued concurrently from different host threads, mirroring
 * `tokio::try_join!` in groth16/src/prove.rs:119-125; calls on one slot are serialised.
 * There is no CPU fallback: without a CUDA device every entry point fails with B200ZK_ERR_CUDA.
 */
#ifndef B200ZK_H
#define B200ZK_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200zk_ctx b200zk_ctx;
typedef struct b200zk_pk b200zk_pk;
typedef struct b200zk_group b200zk_group;         /* several GPUs of one box, one host process (csrc/group.cu) */
typedef struct b200zk_group_pk b200zk_group_pk;   /* a proving key sharded over a group */
typedef struct b200zk_group_r1cs b200zk_group_r1cs;   /* a circuit's A and B sharded over a group by QAP output slot */
typedef struct b200zk_zkey b200zk_zkey;   /* a snarkjs Groth16 .zkey resident in HBM: b200zk_pk + A, B in CSR */
typedef struct b200zk_group_zkey b200zk_group_zkey;   /* the same resident on a group: b200zk_group_pk + A, B sharded by slot */

enum {
    B200ZK_OK = 0,
    B200ZK_ERR_LENGTH = 1,  /* bases.len() != scalars.len(): arkworks `Err(min_len)`, surfaced by `?` at dmsm/mod.rs:82 */
    B200ZK_ERR_DOMAIN = 2,  /* log_n > 28 (Fr two-adicity) / size mismatch: `D::new` -> None, ext_wit.rs:31-32 */
    B200ZK_ERR_CUDA = 3,
    B200ZK_ERR_ARG = 4,
    B200ZK_ERR_OOM = 5,
    B200ZK_ERR_SHORT_BUFFER = 6   /* an output buffer is too small: the *_len arguments say what is needed */
};

/* ---- context (one per GPU; the reference's per-party `Net` handle plays this role) ---------- */
int b200zk_ctx_create(int device, b200zk_ctx** out);
void b200zk_ctx_destroy(b200zk_ctx* ctx);
const char* b200zk_last_error(const b200zk_ctx* ctx);
const char* b200zk_version(void);
/* Make slot `stream` (0..2) launch on a caller-provided cudaStream_t (e.g. torch's current stream).  Work already queued
 * through the slot is ordered before work on the new stream (an event wait, no host synchronisation), so the old stream
 * must still exist when the slot is re-bound. */
int b200zk_ctx_set_stream(b200zk_ctx* ctx, int stream, void* cuda_stream);
int b200zk_ctx_sync(b200zk_ctx* ctx, int stream);
/* Per-kernel CUDA-event profiling (used by bench.py for the roofline numbers). */
int b200zk_profile_enable(b200zk_ctx* ctx, int on);
int b200zk_profile_reset(b200zk_ctx* ctx);
/* Writes a JSON object {"kernel": {"launches": L, "ms": total}, ...} into buf. */
int b200zk_profile_json(b200zk_ctx* ctx, char* buf, size_t buf_len);
/* Total kernels launched by this ctx since creation / last reset (bench.py "gpu_launches"). */
uint64_t b200zk_launch_count(const b200zk_ctx* ctx);

/* ---- d_msm (dist-primitives/src/dmsm/mod.rs:70-98; hot line :82 `G::msm(bases, scalars)`) ---- */
/* Host buffers.  Returns B200ZK_ERR_LENGTH when n_bases != n_scalars (last_error = min_len). */
int b200zk_msm_g1(b200zk_ctx* ctx, int stream, const uint64_t* bases, size_t n_bases,
                  const uint64_t* scalars, size_t n_scalars, uint64_t out_affine[8], int* out_is_inf);
int b200zk_msm_g2(b200zk_ctx* ctx, int stream, const uint64_t* bases, size_t n_bases,
                  const uint64_t* scalars, size_t n_scalars, uint64_t out_affine[16], int* out_is_inf);
/* Host buffers in, this GPU's partial sum out (XYZZ, device memory, ordered on slot `stream`): the input travels over PCIe in
 * parts whose bucket kernels add into one bucket set, so the transfer hides behind the compute.  The multi-GPU callers use it
 * for their index range and combine the partials (b200zk_msm_exchange_sum_dev, b200zk_group_msm_*).  The staging copies
 * wait for earlier work on the slot's stream.  Returns once the host buffers may be reused. */
int b200zk_msm_staged_dev(b200zk_ctx* ctx, int stream, int g2, const uint64_t* bases, size_t n_bases, const uint64_t* scalars,
                          size_t n_scalars, void* d_out_xyzz);
/* Device buffers (inputs already resident in HBM).  `d_out_xyzz` receives the un-normalised
 * partial sum (G1: 4 x 32 B = X,Y,ZZ,ZZZ; G2: 4 x 64 B) so that rank partials can be exchanged
 * and combined with b200zk_g{1,2}_sum_dev -- the multi-GPU replacement of the king's gather +
 * `unpackexp` + sum at dmsm/mod.rs:87-97. */
int b200zk_msm_g1_dev(b200zk_ctx* ctx, int stream, const void* d_bases, const void* d_scalars, size_t n,
                      void* d_out_xyzz);
int b200zk_msm_g2_dev(b200zk_ctx* ctx, int stream, const void* d_bases, const void* d_scalars, size_t n,
                      void* d_out_xyzz);
/* Fixed-base window tables: for bases that never change between calls (the proving key's query vectors,
 * groth16/src/proving_key.rs:35-110) keep table[w * n + i] = 2^{c w} * bases[i], w < b200zk_msm_table_windows(c) =
 * ceil(255 / c), resident in HBM.  b200zk_msm_table_dev then computes the same sum as b200zk_msm_g{1,2}_dev with one
 * bucket set and no doublings (g2 = 0: G1, 64-byte points; 1: G2, 128-byte points).  d_table must hold
 * windows * n points. */
unsigned b200zk_msm_table_windows(unsigned c);
/* The window b200zk_pk_precompute picks for n bases (about log2 n, in [10, 20]). */
unsigned b200zk_msm_table_auto_window(size_t n);
int b200zk_msm_table_build_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_bases, size_t n, unsigned c,
                               void* d_table);
int b200zk_msm_table_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_table, const void* d_scalars, size_t n,
                         unsigned c, void* d_out_xyzz);
/* Sum `count` XYZZ partials (device) and normalise to affine (host). */
int b200zk_g1_sum_dev(b200zk_ctx* ctx, int stream, const void* d_xyzz, size_t count, uint64_t out_affine[8],
                      int* out_is_inf);
int b200zk_g2_sum_dev(b200zk_ctx* ctx, int stream, const void* d_xyzz, size_t count, uint64_t out_affine[16],
                      int* out_is_inf);

/* ---- d_fft / d_ifft (dist-primitives/src/dfft/mod.rs:17-54 / :56-95) -------------------------- */
/* In-place on a host buffer of (pad << log_n) x 4 limbs whose first 2^log_n elements are the input:
 *   out = dom.fft(x) / dom.ifft(x) for `dom = Radix2EvaluationDomain::new(2^log_n)` (natural order
 *   in and out); coset != 0 uses the coset domain `get_coset(Fr::GENERATOR)` (pss.rs:41-48);
 *   bitrev_in / bitrev_out apply `fft_in_place_rearrange` (dfft/mod.rs:258-271) to the input / to the
 *   (padded) output -- the `rearrange` flag; pad >= 1 zero-extends the result to pad * 2^log_n
 *   before the output rearrangement (dfft/mod.rs:225-227). */
int b200zk_ntt_fr(b200zk_ctx* ctx, int stream, uint64_t* data, unsigned log_n, int inverse, int coset,
                  int bitrev_in, int bitrev_out, unsigned pad);
/* Device-resident, natural order, out-of-place allowed (d_out may equal d_in); batch contiguous. */
int b200zk_ntt_fr_dev(b200zk_ctx* ctx, int stream, const void* d_in, void* d_out, unsigned log_n, int inverse,
                      int coset, unsigned batch);
/* Building blocks of the multi-GPU four-step NTT (SURVEY 8e); see parallel.py for the orchestration:
 * column transform of a [rows x cols] slab along `rows` with twiddle w_N^(global_col*k) applied. */
int b200zk_ntt_fr_fourstep_cols_dev(b200zk_ctx* ctx, int stream, const void* d_in, void* d_out, unsigned log_rows,
                                    unsigned log_cols_local, unsigned log_n, uint64_t global_col0, int inverse);

/* Fused compute + exchange (the GPU-native four-step): same column transform, but the last pass stores every
 * output element directly into the receive buffer of the rank that owns its row, through NVLink peer mappings --
 * no pack / NCCL all-to-all / unpack passes.  peer_out[g]: device pointer (valid in THIS process, see
 * b200zk_peer_open) to rank g's row-major [rows / n_peers][cols] receive buffer.  The caller orders the row step
 * after all ranks' column steps with a stream-ordered barrier (parallel.sharded_ntt_p2p uses a 1-element all-reduce). */
int b200zk_ntt_fr_fourstep_cols_p2p_dev(b200zk_ctx* ctx, int stream, const void* d_in, void* const* peer_out,
                                        unsigned n_peers, unsigned log_rows, unsigned log_cols_local, unsigned log_n,
                                        uint64_t global_col0, int inverse);
/* Peer-visible device memory (cudaMalloc + CUDA IPC): allocate locally and export a 64-byte handle; open a peer's
 * handle to obtain a pointer usable by this process's kernels. */
int b200zk_peer_alloc(b200zk_ctx* ctx, size_t bytes, void** d_ptr, uint8_t handle_out[64]);
int b200zk_peer_open(b200zk_ctx* ctx, const uint8_t handle[64], void** d_ptr);
int b200zk_peer_close(b200zk_ctx* ctx, void* d_ptr);
int b200zk_peer_free(b200zk_ctx* ctx, void* d_ptr);

/* d_msm's exchange step as one kernel over peer memory (dmsm/mod.rs:87-97: send_to_king, unpackexp, sum, recv_from_king):
 * every rank stores its XYZZ partial into every peer's mailbox, waits on sequence flags for the partials of all ranks, adds
 * them and normalises -- no NCCL call, no host round trip.  peer_mailboxes[g]: rank g's mailbox (b200zk_peer_alloc of
 * B200ZK_MAILBOX_BYTES, zero-filled; peers' opened with b200zk_peer_open).  seq: 1, 2, 3, ... the same on every rank.
 * d_out_affine: 64 / 128 bytes of canonical affine coordinates followed by one u64 infinity flag. */
#define B200ZK_MAILBOX_BYTES 8192
int b200zk_msm_exchange_sum_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_partial, void* const* peer_mailboxes,
                                unsigned n_peers, unsigned rank, uint64_t seq, void* d_out_affine);

/* Generalised building block: `batch` contiguous transforms of size 2^log_t; output k of transform b is
 * multiplied by base^((b + b0)(alpha k + beta) + gamma k) where base = w_{2^log_base} (direction of the
 * transform) or, with base_is_shift, the forward root w_{2^log_base} used by the h coefficient shift.
 * fourstep_cols == (b0 = global_col0, alpha = 1, beta = 0, gamma = 0, log_base = log_n). */
int b200zk_ntt_fr_batched_post_dev(b200zk_ctx* ctx, int stream, const void* d_in, void* d_out, unsigned log_t,
                                   unsigned batch, int inverse, unsigned log_base, int base_is_shift, uint64_t b0,
                                   uint64_t alpha, uint64_t beta, uint64_t gamma);
/* out[i] = a[i]*b[i] - c[i] on device-resident vectors (the king's pointwise step, ext_wit.rs:88-92). */
int b200zk_fr_mul_sub_dev(b200zk_ctx* ctx, int stream, const void* d_a, const void* d_b, const void* d_c, void* d_out,
                          size_t n);

/* ---- ext_wit::h (groth16/src/ext_wit.rs:16-101 == ark-circom/src/circom/qap.rs:64-89) --------- */
/* a, b, c: QAP evaluation vectors (2^log_m x 4 limbs each); h_out[i] = A(w^(2i+1)) B(..) - C(..). */
int b200zk_h_circom(b200zk_ctx* ctx, const uint64_t* a, const uint64_t* b, const uint64_t* c, unsigned log_m,
                    uint64_t* h_out);
int b200zk_h_circom_dev(b200zk_ctx* ctx, const void* d_a, const void* d_b, const void* d_c, unsigned log_m,
                        void* d_h_out);

/* ---- qap::qap (groth16/src/qap.rs:44-91): R1CS matrices x full assignment -> QAP evaluation vectors ----
 * A and B in CSR form (row_ptr: num_constraints + 1 x u32, col: nnz x u32 wire index, val: nnz x 4 limbs
 * Montgomery), z: full assignment (Montgomery).  Writes a, b, c (2^log_m x 4 limbs each):
 * a_i = <A_i, z>, b_i = <B_i, z>, c_i = a_i b_i for i < num_constraints; a[num_constraints + j] = z[j], j < num_inputs. */
int b200zk_qap_dev(b200zk_ctx* ctx, int stream, const void* d_a_row_ptr, const void* d_a_col, const void* d_a_val,
                   const void* d_b_row_ptr, const void* d_b_col, const void* d_b_val, size_t num_constraints,
                   size_t num_inputs, const void* d_z, unsigned log_m, void* d_a, void* d_b, void* d_c);
/* Montgomery <-> canonical conversion applied `times` times (zkey coefficients are stored times R^2:
 * ark-circom/src/zkey.rs:333-338 -> to_mont = 0, times = 1; .wtns / .r1cs values: to_mont = 1, times = 1). */
int b200zk_fr_convert_dev(b200zk_ctx* ctx, int stream, const void* d_in, void* d_out, size_t n, int to_mont, int times);
/* R1CS satisfaction, the check of snarkjs `wtns check <r1cs> <wtns>`: constraint i fails when
 * <A_i, w> <B_i, w> != <C_i, w> over Fr.  A, B and C in CSR form with the conventions of b200zk_qap_dev (row_ptr:
 * n_constraints + 1 x u32, col: nnz x u32 wire index, val: nnz x 4 limbs Montgomery; col / val may be null for a matrix
 * without terms); w: the full assignment (Montgomery), long enough for every column.  *n_failed = the number of failing
 * constraints, *first_failed = the lowest failing index (n_constraints when none fails).  n_constraints = 0: OK with no
 * failure; a null row_ptr, w or output with n_constraints > 0: B200ZK_ERR_ARG.  Returns once the counters are on the host. */
int b200zk_r1cs_check_dev(b200zk_ctx* ctx, int stream, const void* d_a_row_ptr, const void* d_a_col, const void* d_a_val,
                          const void* d_b_row_ptr, const void* d_b_col, const void* d_b_val, const void* d_c_row_ptr,
                          const void* d_c_col, const void* d_c_val, size_t n_constraints, const void* d_w, uint64_t* n_failed,
                          uint64_t* first_failed);

/* ---- proving key (what PackedProvingKeyShare carries, groth16/src/proving_key.rs:19-25,48-65) -- */
/* a_query, b_g1_query, b_g2_query: n_vars points; l_query: n_vars - n_inputs; h_query: m points.
 * vk_points = alpha_g1(8) beta_g1(8) delta_g1(8) beta_g2(16) delta_g2(16) limbs. */
int b200zk_pk_upload(b200zk_ctx* ctx, const uint64_t* a_query, const uint64_t* b_g1_query,
                     const uint64_t* b_g2_query, const uint64_t* l_query, const uint64_t* h_query, size_t n_vars,
                     size_t n_inputs, size_t m, const uint64_t* vk_points, b200zk_pk** out);
/* Same, from device-resident arrays (copied device-to-device; the caller keeps ownership of its buffers). */
int b200zk_pk_upload_dev(b200zk_ctx* ctx, const void* d_a_query, const void* d_b_g1_query, const void* d_b_g2_query,
                         const void* d_l_query, const void* d_h_query, size_t n_vars, size_t n_inputs, size_t m,
                         const uint64_t* vk_points, b200zk_pk** out);
void b200zk_pk_free(b200zk_ctx* ctx, b200zk_pk* pk);
/* (Re)build the key's fixed-base window tables (b200zk_msm_table_*): c = 0 picks b200zk_msm_table_auto_window(n)
 * per query, c = 0xFFFFFFFF drops the tables.  b200zk_pk_upload{,_dev} call this with c = 0 unless the environment
 * has B200ZK_PK_TABLES=0; tables that would exceed B200ZK_PK_TABLE_MAX_GB (default: 60% of the free HBM) are skipped and proving runs
 * the generic MSM on the queries.  The proof bytes do not depend on the choice.  b200zk_pk_table_bytes: HBM held by
 * the tables (0 = none). */
int b200zk_pk_precompute(b200zk_ctx* ctx, b200zk_pk* pk, unsigned c);
size_t b200zk_pk_table_bytes(const b200zk_pk* pk);

/* ---- packexp_from_public / unpackexp over whole vectors (dist-primitives/src/dmsm/mod.rs:7-68, applied chunk by chunk to
 * the proving key in groth16/src/proving_key.rs:35-110): out[k * rows + j] = sum_{i < l} matrix[j * l + i] * points[k * l + i]
 * for every chunk k < n_chunks.  matrix: rows x l Fr elements (Montgomery) -- the pack (n x l) or unpack (l x n) matrix of
 * the PackedSharingParams; points / out affine (G1 8, G2 16 u64 limbs). */
int b200zk_points_matmul_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_points, size_t n_chunks, size_t l,
                             const void* d_matrix, size_t rows, void* d_out);

/* ---- Groth16::verify_with_processed_vk (groth16/examples/sha256.rs:229-254, mpc-api/src/main.rs:187-247) ----------
 * e(A, B) == e(alpha_g1, beta_g2) * e(gamma_abc_g1[0] + sum_i x_i gamma_abc_g1[i+1], gamma_g2) * e(C, delta_g2), evaluated as
 * one product of four Miller loops and one final exponentiation on the device.  Host buffers: affine points as Montgomery
 * u64 limbs (G1 8, G2 16; infinity all-zero), public inputs n_public x 4 Montgomery limbs.  *is_valid = 1 / 0.  Points
 * are taken as given (decompress with b200zk_points_decompress_dev(check_subgroup = 1) for arkworks' validation). */
int b200zk_groth16_verify(b200zk_ctx* ctx, const uint64_t* alpha_g1, const uint64_t* beta_g2, const uint64_t* gamma_g2,
                          const uint64_t* delta_g2, const uint64_t* gamma_abc_g1, size_t n_public,
                          const uint64_t* public_inputs, const uint64_t* proof_a, const uint64_t* proof_b,
                          const uint64_t* proof_c, int* is_valid);
/* vk_alphabeta_12 of the verification key snarkjs `zkey export verificationkey` writes: e(alpha_g1, beta_g2) as snarkjs
 * computes it, i.e. the pairing of b200zk_groth16_verify raised to ffjavascript's hard-part multiple m = 2u(6u^2 + 3u + 1).
 * Host buffers: alpha_g1 8, beta_g2 16 Montgomery u64 limbs (infinity all-zero); out: 12 canonical Fq elements (4 u64 limbs
 * each) in snarkjs's nesting [[c0.a, c0.b, c0.c], [c1.a, c1.b, c1.c]] of Fq2 pairs (c0, c1), over the tower
 * Fq12 = Fq6[w]/(w^2 - v), Fq6 = Fq2[v]/(v^3 - (9 + u)). */
int b200zk_vk_alphabeta_12(b200zk_ctx* ctx, const uint64_t alpha_g1[8], const uint64_t beta_g2[16], uint64_t out[48]);

/* ---- ark-serialize Compress::Yes point codec (common/src/utils/serializer.rs:20-49: every proving / verifying key and
 * proof of the reference travels in this form; zk-cli/src/main.rs:130-136) --------------------------------------------
 * G1: 32 bytes = x little-endian, top bits of the last byte 0x80 (y is the larger of y, -y) / 0x40 (infinity);
 * G2: 64 bytes = x.c0 || x.c1, flags in the last byte.  Affine points: 8 / 16 Montgomery u64 limbs, infinity all-zero.
 * decompress: one square root per point on the device; *n_invalid = encodings that are not curve points (then the call
 * returns B200ZK_ERR_ARG and those slots hold infinity).  check_subgroup != 0 also multiplies every G2 point by r
 * (G1 has cofactor 1), i.e. arkworks' Validate::Yes. */
int b200zk_points_compress_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_affine, size_t n, void* d_bytes);
int b200zk_points_decompress_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_bytes, size_t n, int check_subgroup,
                                 void* d_affine, size_t* n_invalid);

/* ---- prove::{A,B,C}::compute + assembly (groth16/src/prove.rs:21-136, examples/sha256.rs:208-212)
 * z: full assignment (n_vars x 4 limbs, z[0] = 1); a, b, c: QAP evaluation vectors (m x 4 limbs);
 * r, s: 4 limbs (Montgomery; the reference always passes zero).  mirror_bg1 != 0 also runs the
 * MSM over b_g1_query when r == 0, as the reference does unconditionally (prove.rs:123).
 * proof_out: Proof<Bn254> in ark-serialize Compress::Yes form (A 32 || B 64 || C 32 bytes). */
int b200zk_groth16_prove(b200zk_ctx* ctx, const b200zk_pk* pk, const uint64_t* z, const uint64_t* a,
                         const uint64_t* b, const uint64_t* c, const uint64_t r[4], const uint64_t s[4],
                         int mirror_bg1, uint8_t proof_out[128]);

/* Same with z, a, b, c already resident in HBM. */
int b200zk_groth16_prove_dev(b200zk_ctx* ctx, const b200zk_pk* pk, const void* d_z, const void* d_a, const void* d_b,
                             const void* d_c, const uint64_t r[4], const uint64_t s[4], int mirror_bg1,
                             uint8_t proof_out[128]);

/* ---- snarkjs `groth16 prove <zkey> <wtns> <proof.json> <public.json>` from the files' bytes (csrc/zkey.cu) ---------------
 * b200zk_zkey_load: parse a Groth16 .zkey (zkey_len bytes; the caller may unmap it on return) and keep it in HBM: the point
 * sections go to the device as they are (Montgomery, little-endian, infinity all-zero), and the coefficient section is sorted
 * into A and B in CSR form on the device, dropping the public-input rows snarkjs appends; num_constraints = the largest
 * constraint index - n_public.  table_window as b200zk_pk_precompute's c: 0 = the automatic table policy of
 * b200zk_pk_upload (B200ZK_PK_TABLES, B200ZK_PK_TABLE_MAX_GB), 0xFFFFFFFF = no fixed-base tables (a caller that proves once:
 * the tables cost more to build than one proof saves).  Refused before any launch (B200ZK_ERR_ARG, the message of
 * formats.read_zkey): a bad magic, a section past zkey_len, a missing or short section, a protocol other than Groth16 (1),
 * a field other than BN254, n_public + 1 > n_vars, a domain size that is not a power of two; a domain above 2^27:
 * B200ZK_ERR_DOMAIN.  A coefficient record with matrix > 1, signal >= n_vars or constraint >= domain size: B200ZK_ERR_ARG
 * with the count and the first index.  Peak device memory while loading: 80 bytes per coefficient record + 16 bytes per
 * constraint, then the proving key and its tables; held afterwards: the key, its tables, 36 bytes per record + 8 per
 * constraint. */
int  b200zk_zkey_load(b200zk_ctx* ctx, const void* zkey, size_t zkey_len, unsigned table_window, b200zk_zkey** out);
void b200zk_zkey_free(b200zk_ctx* ctx, b200zk_zkey* zk);
int  b200zk_zkey_info(const b200zk_zkey* zk, size_t* n_vars, size_t* n_public, size_t* domain_size, size_t* num_constraints);
/* The longest proof.json plus its NUL: every coordinate below q has at most 77 digits.  The longest public.json of n public
 * signals plus its NUL: "[", n lines of up to 77 digits in quotes, n - 1 commas, "\n]" (n = 0: "[]"). */
#define B200ZK_PROOF_JSON_MAX 810
#define B200ZK_PUBLIC_JSON_MAX(n_public) (3 + 82 * (size_t)(n_public))
/* Prove from a .wtns (n8 = 32, prime = r, n_vars entries, each < r) with the key: the proof of circom.groth16_prove.
 * r, s: 4 Montgomery limbs each (as b200zk_groth16_prove); NULL draws the value uniformly mod r from getrandom, so that the
 * proof is zero-knowledge.  proof_out (128 bytes, ark-serialize Compress::Yes), proof_json and public_json may each be NULL.
 * The JSON is snarkjs's text (one-space indent, no trailing newline, infinity ["0","1","0"] / [["0","0"],["1","0"],["0","0"]]),
 * NUL-terminated; public.json holds w[1..n_public] of the witness.  *proof_json_len / *public_json_len: in, the buffer sizes;
 * out, the text lengths without the NUL.  Buffers of B200ZK_PROOF_JSON_MAX / B200ZK_PUBLIC_JSON_MAX(n_public) bytes always
 * suffice.  A buffer under B200ZK_PROOF_JSON_MAX / the exact public.json size + 1 is refused
 * before any launch with B200ZK_ERR_SHORT_BUFFER, both lengths then set to the sizes needed.  Refused before any launch: a
 * malformed wtns (B200ZK_ERR_ARG, formats.read_wtns's message), an entry count other than n_vars (B200ZK_ERR_LENGTH,
 * "witness has N entries, the key expects M"); an entry >= r: B200ZK_ERR_ARG naming the count and the first index.  One key
 * may prove any number of witnesses and several keys may be live on one context; calls are serialised as
 * b200zk_groth16_prove's (slots 0, 1 and 2). */
int  b200zk_zkey_prove(b200zk_ctx* ctx, const b200zk_zkey* zk, const void* wtns, size_t wtns_len, const uint64_t r[4],
                       const uint64_t s[4], uint8_t proof_out[128], char* proof_json, size_t* proof_json_len, char* public_json,
                       size_t* public_json_len);

/* Multi-GPU prove building blocks: sum `count` XYZZ partials spaced `stride` points apart into one XYZZ point,
 * and run only the final assembly (prove.rs:36-44,75-83,128-134 + sha256.rs:208-212 + Compress::Yes) on MSM results
 * that were combined across ranks.  include_zero_terms = 0 when the MSMs already covered index 0 (z[0] = 1). */
int b200zk_xyzz_sum_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_in, size_t count, size_t stride, void* d_out);
int b200zk_groth16_assemble_dev(b200zk_ctx* ctx, const b200zk_pk* pk, const void* d_msm_a, const void* d_msm_b2,
                                const void* d_msm_l, const void* d_msm_h, const void* d_msm_b1_or_null,
                                const uint64_t r[4], const uint64_t s[4], int include_zero_terms, uint8_t proof_out[128]);

/* ---- circuit-specific setup building blocks (Groth16::circuit_specific_setup in the reference's drivers,
 *      groth16/examples/sha256.rs:133-137; h-query per ark-circom/src/circom/qap.rs:94-110) ------------------------ */
/* out[i] = scalars[i] * G (generator of G1, or of G2 when g2 != 0); scalars Montgomery, out affine. */
int b200zk_fixed_base_mul_dev(b200zk_ctx* ctx, int g2, const void* d_scalars, size_t n, void* d_out);
/* out[i] = scale * base^i  (base, scale: 4 limbs Montgomery, host). */
int b200zk_fr_powers_dev(b200zk_ctx* ctx, const uint64_t base[4], const uint64_t scale[4], size_t n, void* d_out);
/* Generic CSR mat-vec over Fr: out[r] = sum val[k] x[idx[k]], k in [ptr[r], ptr[r+1]). */
int b200zk_fr_spmv_dev(b200zk_ctx* ctx, const void* d_ptr, const void* d_idx, const void* d_val, const void* d_x,
                       size_t n_rows, void* d_out);
/* The same CSR product over group elements: out[r] = sum val[k] points[idx[k]], k in [ptr[r], ptr[r+1]) -- the step of
 * snarkjs `zkey new` that turns a Powers-of-Tau file's Lagrange bases into the query vectors, and (over the odd points of
 * the doubled domain) the h-query convention of ark-circom/src/circom/qap.rs:11-15.  Conventions as
 * b200zk_fr_spmv_dev: ptr n_rows + 1 x u32, idx nnz x u32, val nnz x 4 limbs Montgomery; points / out affine (g2 = 0: G1,
 * 8 u64 limbs; 1: G2, 16), infinity all-zero, an empty row gives infinity; idx and val may be null when
 * nnz = ptr[n_rows] = 0.  Rows of more than 256 entries go through the MSM.  Reads ptr to the host and returns once out is complete; temporary device memory: nnz XYZZ points. */
int b200zk_points_spmv_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_ptr, const void* d_idx, const void* d_val,
                           const void* d_points, size_t n_rows, void* d_out);
/* One scalar times many points, out[i] = k * points[i] -- the step of a snarkjs `zkey contribute` / `zkey beacon` that
 * multiplies the L and H sections by delta^-1.  k: 4 u64 limbs, a plain little-endian integer (not Montgomery, not
 * reduced), host.  Affine in and out (G1 8 / G2 16 u64 limbs, Montgomery), infinity all-zero; out may equal points.
 * G1 reduces k mod r and uses the GLV split (every G1 point has order r); G2 runs the plain 256-bit ladder on k as given,
 * so it is right for twist points outside the order-r subgroup too (cofactor clearing).  Enqueued on the slot's stream. */
int b200zk_points_scale_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_points, size_t n, const uint64_t k[4],
                            void* d_out);
/* out[i] = n^-1 * sum_j omega_n^(-i j) * in[j],  n = 2^log_n: the Lagrange basis in the exponent that snarkjs
 * `powersoftau prepare phase2` writes.  Affine Montgomery points in natural order, infinity all-zero (also as input).
 * omega_n is the root of unity of b200zk_ntt_fr_dev, so points_intt(k_j G) == fixed_base_mul(ntt(k, inverse)) point for
 * point.  g2 = 0: G1 (8 u64 limbs per point), 1: G2 (16); the points must lie in the order-r subgroup (every G1 point
 * does; the GLV split is used on both groups).  d_out may equal d_in (in place); no other overlap is allowed.
 * Temporary device memory: 2^(log_n - 1) x 64 bytes, allocated before anything is launched (B200ZK_ERR_OOM with a message
 * when it does not fit).  log_n > 28: B200ZK_ERR_DOMAIN; a null pointer: B200ZK_ERR_ARG.  Returns once out is complete. */
int b200zk_points_intt_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_in, unsigned log_n, void* d_out);
/* out[i] = sum_j omega_n^(i j) * in[j],  n = 2^log_n, unscaled: the forward transform of b200zk_points_intt_dev, the step
 * of a snarkjs `zkey export bellman` that moves the H query from the zkey's Lagrange form to the tau basis of the MPC
 * params.  points_ntt(k_j G) == fixed_base_mul(ntt(k)) point for point, and points_intt(points_ntt(P)) == P.  Points,
 * order, subgroup, aliasing, temporary memory and error codes as b200zk_points_intt_dev.  Returns once out is complete. */
int b200zk_points_ntt_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_in, unsigned log_n, void* d_out);
/* out[i] = (first * ratio^i) * points[i], i < n: the step of a snarkjs `powersoftau contribute` that multiplies every point
 * of a ceremony section by its own power of the secret (ffjavascript G.batchApplyKey).  first, ratio: 4 u64 limbs, plain
 * little-endian integers (reduced mod r by the call, like b200zk_points_scale_dev's k), host.  Affine Montgomery points
 * (G1 8 / G2 16 u64 limbs), infinity all-zero (also as input); a zero scalar gives infinity, ratio = 0 gives first * P_0
 * at i = 0 (0^0 = 1) and infinity elsewhere.  out may equal points.  On G2 the GLV split is only right for points of the
 * order-r subgroup, which every ceremony point is.  A section may be processed in chunks: the call on points [a, b) with
 * first * ratio^a as `first` equals that slice of one call over the whole section.  Temporary device memory: n x 64 bytes,
 * allocated before anything is launched (B200ZK_ERR_OOM with a message when it does not fit).  A null pointer with n > 0:
 * B200ZK_ERR_ARG; n = 0 does nothing.  Returns once out is complete. */
int b200zk_points_mul_powers_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_points, size_t n, const uint64_t first[4],
                                 const uint64_t ratio[4], void* d_out);
/* out[i] = a[i] - b[i], i < n: the step of snarkjs `zkey new` that makes the circuit hash's H points tau^(n+i) G1 - tau^i G1
 * from a ceremony's tau powers.  Affine Montgomery points (g2 = 0: G1, 8 u64 limbs; 1: G2, 16), infinity all-zero (also
 * as input); a[i] = b[i] gives infinity, a[i] = -b[i] gives 2 a[i].  out may equal a or b; no other overlap is allowed.
 * A null pointer with n > 0: B200ZK_ERR_ARG; n = 0 does nothing.  Enqueued on the slot's stream. */
int b200zk_points_sub_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_a, const void* d_b, size_t n, void* d_out);
/* ffjavascript's point encodings, the bytes a phase-1 ceremony hashes.  fmt 0 = toRprUncompressed: canonical big-endian
 * x || y (G2: x.c1 x.c0 y.c1 y.c0), 64 / 128 bytes; fmt 1 = toRprCompressed: canonical big-endian x (G2: x.c1 x.c0) with
 * 0x80 in byte 0 when y is the larger of (y, -y) (Fq2: decided by c1 unless c1 = 0, then by c0), 32 / 64 bytes.
 * Infinity: 0x40 then zeros in both.  d_affine: n affine Montgomery points; d_bytes: n encodings back to back (16-byte
 * aligned).  Enqueued on the slot's stream. */
int b200zk_points_encode_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_affine, size_t n, int fmt, void* d_bytes);
/* The inverse of b200zk_points_encode_dev: the step of a snarkjs `challenge contribute` (fmt 0) and `import response`
 * (fmt 1) that reads ffjavascript's encodings back into points, one thread per point.  Valid: infinity is 0x40 then zeros
 * (both formats); fmt 0 is x || y with both < q, byte 0's top two bits clear and y^2 = x^3 + b; fmt 1 is x < q (after
 * masking 0x80) with a curve point, y the square root whose "larger" rule (as in encode) agrees with the 0x80 flag.
 * check_subgroup != 0 also requires [r] P == O on G2 (G1 has cofactor 1).  d_bytes: n encodings back to back; d_affine:
 * n affine Montgomery points (G1 8 / G2 16 u64 limbs, infinity all-zero); both 16-byte aligned.  *n_invalid = the number
 * of invalid encodings, *first_invalid = the lowest invalid index (n when there is none); either may be null.  Any invalid
 * encoding: B200ZK_ERR_ARG with a message giving the count and the first index, and those slots hold infinity.  A null
 * pointer with n > 0: B200ZK_ERR_ARG; n = 0 does nothing.  Returns once the counters are on the host. */
int b200zk_points_decode_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_bytes, size_t n, int fmt, int check_subgroup,
                             void* d_affine, size_t* n_invalid, size_t* first_invalid);
/* Blake2b-512 (RFC 7693) whose state is a caller-owned 216-byte buffer, so that hashing can be suspended and resumed (a
 * phase-1 contribution record stores the response hasher's state as its partialHash).  Layout: buffer[128] || h[8] (u64
 * LE) || t[2] (u64 LE) || c (u32 LE) || outlen (u32 LE), with the reference implementation's lazy rule (a full buffer is
 * compressed only when more input arrives); believed to be blake2b-wasm's context, not checked against snarkjs.  Host
 * only: no context and no GPU.  B200ZK_ERR_ARG for a null pointer or a state no init / update can produce. */
int b200zk_blake2b512_init(uint8_t state[216]);
int b200zk_blake2b512_update(uint8_t state[216], const void* data, size_t len);
int b200zk_blake2b512_final(const uint8_t state[216], uint8_t out[64]);
/* out[i] = (a[i] s0 + b[i] s1 + c[i] s2) s3   (s: 16 limbs = 4 Montgomery scalars, host). */
int b200zk_fr_lincomb_dev(b200zk_ctx* ctx, const void* d_a, const void* d_b, const void* d_c, const uint64_t s[16], size_t n,
                          void* d_out);

/* ---- deterministic dummy inputs (groth16/examples/local_groth_bench.rs:21-52,
 *      groth16/src/proving_key.rs:112-155 generate dummy CRS points the same way: not a setup) ---- */
int b200zk_g1_generate_dev(b200zk_ctx* ctx, uint64_t seed, size_t n, void* d_out);
int b200zk_g2_generate_dev(b200zk_ctx* ctx, uint64_t seed, size_t n, void* d_out);
int b200zk_fr_generate_dev(b200zk_ctx* ctx, uint64_t seed, size_t n, void* d_out);

/* ---- multi-GPU group: the sharded hot path behind ONE call each (SURVEY 8b `device_ids, n_dev`; BASELINE config 5) ------
 * One host process owns n_dev GPUs (1, 2, 4 or 8) with NVLink peer access; the king/client star of mpc-net/src/lib.rs:61-139
 * is replaced by index-range sharding of the MSMs and a four-step NTT whose column kernels store straight into the owning
 * peer's memory.  Host buffers hold the WHOLE vectors (what the Rust caller has); results are the same group elements /
 * field vectors / proof bytes as the single-GPU calls.  Calls on one group are serialised by the caller. */
int b200zk_group_create(const int* device_ids, int n_dev, b200zk_group** out);
void b200zk_group_destroy(b200zk_group* group);
int b200zk_group_size(const b200zk_group* group);
b200zk_ctx* b200zk_group_ctx(b200zk_group* group, int rank);            /* rank's single-GPU context (borrowed) */
const char* b200zk_group_last_error(const b200zk_group* group);
/* d_msm (dist-primitives/src/dmsm/mod.rs:70-98) over all GPUs of the group. */
int b200zk_group_msm_g1(b200zk_group* group, const uint64_t* bases, size_t n_bases, const uint64_t* scalars, size_t n_scalars,
                        uint64_t out_affine[8], int* out_is_inf);
int b200zk_group_msm_g2(b200zk_group* group, const uint64_t* bases, size_t n_bases, const uint64_t* scalars, size_t n_scalars,
                        uint64_t out_affine[16], int* out_is_inf);
/* d_fft / d_ifft (dist-primitives/src/dfft/mod.rs:17-95): natural order in and out, in place, 2^log_n elements. */
int b200zk_group_ntt_fr(b200zk_group* group, uint64_t* data, unsigned log_n, int inverse);
/* ext_wit::h (groth16/src/ext_wit.rs:16-101): a, b, c, h_out: 2^log_m x 4 limbs. */
int b200zk_group_h_circom(b200zk_group* group, const uint64_t* a, const uint64_t* b, const uint64_t* c, unsigned log_m,
                          uint64_t* h_out);
/* Proving key sharded over the group (arguments as b200zk_pk_upload): GPU g keeps rows [g n / P, (g+1) n / P) of every
 * query (h_query in the column layout of the sharded h) plus their fixed-base tables. */
int b200zk_group_pk_upload(b200zk_group* group, const uint64_t* a_query, const uint64_t* b_g1_query, const uint64_t* b_g2_query,
                           const uint64_t* l_query, const uint64_t* h_query, size_t n_vars, size_t n_inputs, size_t m,
                           const uint64_t* vk_points, b200zk_group_pk** out);
void b200zk_group_pk_free(b200zk_group* group, b200zk_group_pk* pk);
size_t b200zk_group_pk_table_bytes(const b200zk_group_pk* pk);
/* prove::{A,B,C} + assembly + Compress::Yes (groth16/src/prove.rs:21-136, examples/sha256.rs:208-212), arguments as
 * b200zk_groth16_prove: sharded h, five partial MSMs per GPU, peer copies of the partials to GPU 0, assembly there. */
int b200zk_group_groth16_prove(b200zk_group* group, const b200zk_group_pk* pk, const uint64_t* z, const uint64_t* a,
                               const uint64_t* b, const uint64_t* c, const uint64_t r[4], const uint64_t s[4],
                               uint8_t proof_out[128]);
/* A and B of the circuit in CSR form (conventions of b200zk_qap_dev: row_ptr num_constraints + 1 x u32, col nnz x u32,
 * val nnz x 4 limbs), for a key of domain 2^log_m (log_m <= 27) and n_vars variables.  values_montgomery_depth as
 * groth16.qap.ConstraintMatrices: 1 = zkey words (value R^2), 0 = Montgomery, -1 = canonical; the conversion runs on each
 * GPU after upload.  GPU g keeps the rows of its column-layout slice of the domain (rows = 2^ceil(log_m / 2),
 * cols = 2^floor(log_m / 2), cg = cols / P: local slot c rows + r is global row r cols + g cg + c), reordered on the host once.
 * Refused before any launch: num_constraints + num_inputs > 2^log_m or log_m > 27 (B200ZK_ERR_DOMAIN); cols < P, a column
 * index >= n_vars (the message names the matrix and the term), a row_ptr that does not start at 0 or decreases, or
 * num_inputs outside 1..n_vars (B200ZK_ERR_ARG). */
int  b200zk_group_r1cs_upload(b200zk_group* group, const uint32_t* a_row_ptr, const uint32_t* a_col, const uint64_t* a_val,
                              const uint32_t* b_row_ptr, const uint32_t* b_col, const uint64_t* b_val, size_t num_constraints,
                              size_t num_inputs, size_t n_vars, unsigned log_m, int values_montgomery_depth,
                              b200zk_group_r1cs** out);
void b200zk_group_r1cs_free(b200zk_group* group, b200zk_group_r1cs* matrices);
/* Host only (no device is touched): the 2^log_m / n_gpus + 1 entries of the CSR row_ptr that GPU `rank` of b200zk_group_r1cs_upload
 * keeps, from the global row_ptr (num_constraints + 1 entries).  B200ZK_ERR_DOMAIN / B200ZK_ERR_ARG as the upload. */
int  b200zk_group_r1cs_local_row_ptr(const uint32_t* row_ptr, size_t num_constraints, unsigned log_m, int n_gpus, int rank,
                                     uint32_t* local_row_ptr);
/* b200zk_group_groth16_prove from the witness: d_z is the full assignment (n_vars x 4 limbs, Montgomery) resident on the
 * group's device 0 and written on the slot-0 stream of b200zk_group_ctx(group, 0).  The call copies it to every other GPU
 * (peer copies), runs the sharded QAP (each GPU computes its column-layout slice of a, b, c), then exactly the rest of
 * b200zk_group_groth16_prove; the host waits only for the proof bytes.  Refused before any launch: a key or matrices uploaded
 * to another group, n_inputs or n_vars differing between key and matrices (B200ZK_ERR_ARG), different domain sizes
 * (B200ZK_ERR_DOMAIN). */
int  b200zk_group_groth16_prove_r1cs_dev(b200zk_group* group, const b200zk_group_pk* pk, const b200zk_group_r1cs* matrices,
                                         const void* d_z, const uint64_t r[4], const uint64_t s[4], uint8_t proof_out[128]);

/* ---- snarkjs `groth16 prove` from the files' bytes on a group (csrc/group.cu, csrc/zkey.cu): b200zk_zkey_* sharded -------
 * b200zk_group_zkey_load: b200zk_zkey_load on a group.  The header checks, messages and codes are b200zk_zkey_load's
 * (B200ZK_ERR_ARG / B200ZK_ERR_DOMAIN before any launch); a domain whose cols = 2^floor(log m / 2) is below the group size is
 * refused before any launch with B200ZK_ERR_ARG, "domain too small for this many GPUs".  The coefficient section is sorted
 * once on GPU 0, keyed (owner GPU, matrix, slot), so that every GPU's A and B are one contiguous slice, which is copied to
 * that GPU; the layout is b200zk_group_r1cs_upload's (local slot c rows + r is global row r cols + g cg + c).  The point
 * sections are sharded from the caller's bytes as b200zk_group_pk_upload shards them (a, b1, b2, l by index range, h in the
 * column layout); the vk points come from the header.  table_window as b200zk_zkey_load's, on every shard: 0 = the
 * automatic policy (B200ZK_PK_TABLES), 0xFFFFFFFF = no tables, else the window c.  The caller may unmap the file on return.
 * Device memory, n coefficient records, m the domain size, P GPUs: peak on GPU 0 while sorting about 80 n + 16 m bytes (raw
 * records, counters, the whole CSR and its own slice); held afterwards by GPU g, 36 bytes per record it owns + 8 m / P + 4
 * bytes, plus its proving-key shard and tables (in an emulated group, `b200zk_group_create` with one device id repeated,
 * every rank's share is on that device).  Errors: b200zk_group_last_error, "device N: " before device-side messages. */
int    b200zk_group_zkey_load(b200zk_group* group, const void* zkey, size_t zkey_len, unsigned table_window,
                              b200zk_group_zkey** out);
void   b200zk_group_zkey_free(b200zk_group* group, b200zk_group_zkey* zk);
int    b200zk_group_zkey_info(const b200zk_group_zkey* zk, size_t* n_vars, size_t* n_public, size_t* domain_size,
                              size_t* num_constraints);
size_t b200zk_group_zkey_table_bytes(const b200zk_group_zkey* zk);
/* b200zk_zkey_prove on a group: the same arguments, texts, bytes, codes, messages and *_len outputs.  The witness goes to
 * GPU 0, is checked and converted there and peer-copied to the other GPUs; then the sharded QAP, h and MSMs of
 * b200zk_group_groth16_prove_r1cs_dev, and the JSON encodings on GPU 0.  A key loaded on another group: B200ZK_ERR_ARG
 * before any launch. */
int    b200zk_group_zkey_prove(b200zk_group* group, const b200zk_group_zkey* zk, const void* wtns, size_t wtns_len,
                               const uint64_t r[4], const uint64_t s[4], uint8_t proof_out[128], char* proof_json,
                               size_t* proof_json_len, char* public_json, size_t* public_json_len);

/* ---- the parties' local share arithmetic (n-party compatibility mirrors, SURVEY 8f4) ----------------------------------
 * Element-wise Fr operation on host buffers of n x 4 Montgomery limbs: op 0 = a * b (share-wise product of two sharings,
 * e.g. the degree-2 input of d_fft, dfft/mod.rs:207-211), 1 = a + b, 2 = a - b (with 0 the butterflies of fft1_in_place,
 * dfft/mod.rs:122-135, one call per stage for all of a party's butterflies). */
int b200zk_fr_op(b200zk_ctx* ctx, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n);

/* ---- self-test hooks (tests only): element-wise field ops on device ------------------------- */
/* op: 0 mul, 1 add, 2 sub; field: 0 Fq, 1 Fr.  a, b, out: n x 4 limbs host buffers. */
int b200zk_test_field_op(b200zk_ctx* ctx, int field, int op, const uint64_t* a, const uint64_t* b, uint64_t* out,
                         size_t n);
/* One device primitive of csrc/fp.cuh, codec.cuh, pairing.cuh, glv.cuh or ec.cuh per element (csrc/selftest.cu), for the
 * exact tests against big integers.  in: n records of IN u64 words, out: n records of OUT words (host buffers).  Field
 * elements are raw Montgomery limbs (Fq / Fr 4 words, Fq2 c0 c1 8, Fq6 a b c 24, Fq12 c0 c1 48); points affine_t (x y:
 * G1 8 words, G2 16) or xyzz_t (x y zz zzz: G1 16, G2 32).  F = Fq at op s, Fr at op 32 + s:
 *   s  0 add (a, b)   1 sub   2 neg (a)   3 dbl   4 mul (a, b)   5 mul_ni   6 sqr (a)   7 mul, b any value < 2^256
 *   s  8/9/10 mul_k<2/3/4> (K (a, b) pairs -> K products)   11 mul_wide + redc<1> (a, b -> 512-bit a b (8 words), result)
 *   s 12 redc<2> (512-bit t < 2 p 2^256)   13 inv   14 inv_fermat   15 to_mont   16 from_mont   17 from_u32 (1 word)
 *   s 18 pow_u64 (a, u64 e)
 *   64 fr_root_of_unity (1 word: log_n | inverse << 8, log_n <= 28)                                       [device only]
 *   70 Fq2 mul (a, b)  71 sqr  72 inv  73..76 mul_group<1..4> (K pairs -> K)  77 fq2_mul_xi  78 fq2_conj
 *   79 glv_phi_x on Fq (G1)  80 glv_phi_x on Fq2 (G2)
 *   84 fq_pow_p1_4  85 fq_sqrt -> (flag, root)  86 fq2_sqrt -> (flag, root, zero when false)  87 fq_half
 *   88 fq_is_larger -> flag  89 fq2_is_larger -> flag  90 fq_from_bytes (32 bytes, top_mask) -> (flag, value)
 *   96 Fq6 mul  97 Fq6 inv  98 Fq6 mul_v  99 Fq12 mul  100 Fq12 inv  101 Fq12 conj  102 Fq12 frob2
 *   103 final_exponentiation  104 final_exponentiation(miller_loop(P, Q)) (G1 affine, G2 affine)  105 g2_frobenius_twist
 *   108 glv_decompose (canonical k < r) -> (|k1| 2 words, neg1, |k2| 2 words, neg2)
 * Group law, G1 at 112 + s, G2 at 128 + s, xyzz_t in and out unless noted:
 *   s  0 dbl  1 add (a, b)  2 dbl_ilp  3 add_ilp  4 madd (acc, affine p, u64 negate)  5 dbl_affine (affine)
 *   s  6 to_affine -> affine  7 mul_scalar (p, 4 canonical words k < 2^256)
 *   s  8 quad_ops<F, false>::add  9 ::dbl (one element per quad)  10 quad_ops<F, true>::add  11 ::dbl (one element per
 *      warp)                                                                                               [device only]
 * BAD_ARG for an unknown op. */
int b200zk_test_arith(b200zk_ctx* ctx, int op, const uint64_t* in, size_t n, uint64_t* out);

#ifdef __cplusplus
}
#endif
#endif /* B200ZK_H */
