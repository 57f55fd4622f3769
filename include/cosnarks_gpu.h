/* cosnarks_gpu.h -- C ABI of libcosnarks_gpu.so, the H100 (sm_90a) backend for the co-snarks hot path.
 *
 * The reference (TaceoLabs/co-snarks @ 2b4592e) is pure Rust and has no FFI; its seams for this path
 * are (1) the crate `taceo-ark-algebra 0.1.0` (msm + fft), (2) the `R1CSToQAP` trait and (3) the
 * `CircomGroth16Prover` driver trait.  Each entry point below names the reference interface it
 * replaces; INTEGRATION.md shows the Rust `extern "C"` bindings a maintainer would add.
 *
 * Conventions
 *  - Field elements are little-endian arrays of 64-bit limbs in MONTGOMERY form with R = 2^(64*limbs),
 *    i.e. byte-identical to arkworks' `Fp<MontBackend<_, N>>.0.0` ([u64; N]): BN254 Fr/Fq and
 *    BLS12-381 Fr = 4 limbs, BLS12-381 Fq = 6 limbs.  "canonical" = the plain integer (BigInt).
 *  - G1 affine = x || y ; G2 affine = x.c0 || x.c1 || y.c0 || y.c1 ; the all-zero encoding is the
 *    point at infinity (same marker as snarkjs .zkey files).
 *  - Rep3 share = a || b (Rep3PrimeFieldShare, mpc-core/src/protocols/rep3/arithmetic/types.rs:21-28).
 *  - All functions return 0 on success and a negative code on failure; cs_last_error() gives the
 *    message for the calling thread.  No exceptions cross the boundary.  There is no CPU fallback:
 *    without a CUDA device every compute call fails with CS_ERR_CUDA.
 *  - `h_` pointers are host memory (pinned or pageable), `d_` pointers are device memory of the
 *    context's device.  Calls on one cs_ctx are serialised by the caller; use one ctx per host thread
 *    for concurrency (the reference calls msm/fft from several rayon workers, groth16.rs:227).
 */
#ifndef COSNARKS_GPU_H
#define COSNARKS_GPU_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CS_OK 0
#define CS_ERR_ARG (-1)
#define CS_ERR_CUDA (-2)
#define CS_ERR_LIMIT (-3)
#define CS_ERR_STATE (-4)

typedef enum { CS_BN254 = 0, CS_BLS12_381 = 1 } cs_curve;
typedef enum { CS_G1 = 0, CS_G2 = 1 } cs_group;
typedef enum { CS_NTT_IN_TO_OUT = 0, CS_NTT_OUT_TO_IN = 1 } cs_ntt_order;
typedef enum { CS_PLAIN = 0, CS_REP3 = 1 } cs_share_kind;

typedef struct cs_ctx cs_ctx;
typedef struct cs_bases cs_bases;
typedef struct cs_domain cs_domain;
typedef struct cs_groth16_pk cs_groth16_pk;
typedef struct cs_net cs_net; /* party-to-party transport, see "party-to-party transport" below */

/* ---- library / context ------------------------------------------------------------------------ */
const char* cs_last_error(void);
/* version string, e.g. "cosnarks-b200 0.1 (sm_90a)" */
const char* cs_version(void);
/* `stream` = an existing cudaStream_t the context should run on (e.g. torch's current stream), or NULL
 * to let the context create its own. */
int cs_ctx_create(int device, void* stream, cs_ctx** out);
void cs_ctx_destroy(cs_ctx* ctx);
int cs_ctx_synchronize(cs_ctx* ctx);
/* kernels launched by this context since creation (bench.py's "gpu_launches") */
uint64_t cs_ctx_launch_count(const cs_ctx* ctx);

/* device memory helpers so a host language needs no CUDA binding of its own */
int cs_dev_alloc(cs_ctx* ctx, size_t bytes, void** d_out);
int cs_dev_free(cs_ctx* ctx, void* d_ptr);
int cs_host_alloc_pinned(size_t bytes, void** h_out);
int cs_host_free_pinned(void* h_ptr);
int cs_memcpy_h2d(cs_ctx* ctx, void* d_dst, const void* h_src, size_t bytes);
int cs_memcpy_d2h(cs_ctx* ctx, void* h_dst, const void* d_src, size_t bytes);

/* ---- MSM: taceo_ark_algebra::msm::{msm_unchecked, msm_bigint} --------------------------------------
 * Reference call sites: co-groth16/src/mpc/plain.rs:66-74, rep3.rs:124-132, shamir.rs:111-119,
 * co-groth16/src/groth16.rs:194, mpc-core/src/protocols/rep3/pointshare.rs:201-222,
 * co-noir/co-noir-common/src/honk_curve.rs:81-83.
 *
 * cs_bases_upload: upload `n` affine points (Montgomery) once per proving key / SRS; the library
 * expands them into the per-window table it keeps resident in HBM.  window_bits = 0 picks a default
 * (at most 16); an explicit window_bits must lie in [2, 20], the widest window the bucket sort takes, and
 * anything else fails here with CS_ERR_ARG (so does a Groth16 key created with such a window).
 * cs_msm: sum_{i<n} scalars[i] * bases[offset + i]; the reference "chops to the shorter slice"
 * (honk_curve.rs:33-34) -- pass n = min(len).  scalars_montgomery = 1 for `&[Fr]` (msm_unchecked),
 * 0 for canonical `&[BigInt]` (msm_bigint; must be < r).  Result: affine point (Montgomery), all-zero
 * + *out_is_infinity = 1 for the identity. */
int cs_bases_upload(cs_ctx* ctx, cs_curve curve, cs_group group, const uint64_t* h_points_mont, size_t n,
                    int window_bits, cs_bases** out);
void cs_bases_free(cs_bases* bases);
size_t cs_bases_len(const cs_bases* bases);
int cs_msm(cs_ctx* ctx, const cs_bases* bases, size_t offset, const uint64_t* h_scalars, size_t n,
           int scalars_montgomery, uint64_t* h_out_affine_mont, int* out_is_infinity);
int cs_msm_device(cs_ctx* ctx, const cs_bases* bases, size_t offset, const uint64_t* d_scalars, size_t n,
                  int scalars_montgomery, uint64_t* h_out_affine_mont, int* out_is_infinity);

/* rep3::pointshare::msm_public_points (mpc-core/src/protocols/rep3/pointshare.rs:201-222; used by co-plonk
 * mpc/rep3.rs:170-175 and co-noir-common mpc/rep3.rs:259-266): shares = n Rep3 shares a||b (Montgomery);
 * returns the point share {a: sum a_i P_i, b: sum b_i P_i} as two affine points. */
int cs_msm_rep3_shares(cs_ctx* ctx, const cs_bases* bases, size_t offset, const uint64_t* h_shares, size_t n,
                       uint64_t* h_out_a_affine, uint64_t* h_out_b_affine);

/* Measurement hooks (bench.py): when enabled, cs_msm / cs_msm_device record CUDA events at the five stage
 * boundaries of the MSM on its launching stream; cs_msm_stage_ms returns the last MSM's stage durations
 * {digits+histogram, scan+scatter, bucket accumulation (k_msm_accum0), partial folding, bucket reduction}. */
int cs_msm_profile(cs_ctx* ctx, int enable);
int cs_msm_stage_ms(cs_ctx* ctx, float* out_ms5);
/* While profiling is on: where the stage boundaries of the five MSM workspaces (Groth16: A, B1, B2, L, H) fell in the
 * last fork/join section, in ms after the fork -- out_ms[w * 6 + i], i = 0..5 (start, after digits, sort, accumulate,
 * fold, reduce); -1 where no event exists.  Synchronises the device. */
int cs_msm_timeline_ms(cs_ctx* ctx, float* out_ms);

/* out[i] = scalars[i] * base (affine Montgomery), i < n.  No counterpart on the reference's prover path:
 * it is the fixed-base multiplication a Groth16/KZG setup performs, provided so that tests and bench.py
 * can synthesise proving keys of any size on the device (SURVEY.md 8d). */
int cs_fixed_base_mul(cs_ctx* ctx, cs_curve curve, cs_group group, const uint64_t* h_base_affine_mont,
                      const uint64_t* h_scalars, size_t n, int scalars_montgomery, uint64_t* h_out_points);

/* ---- NTT: taceo_ark_algebra::fft::{Domain, bit_reverse} ---------------------------------------------
 * Domain::with_group_gen(size, gen) (co-groth16/src/groth16/reduction.rs:93), ::new (:249), size()
 * (:251), ifft_in_to_out / fft_out_to_in (:141-175, :270-327), bit_reverse (:58, :328).
 * `batch` = interleaved components per element: 1 for Fr / half shares, 2 for Rep3 shares
 * (DomainCoeff impl, rep3/arithmetic/ops.rs:5-114).  The inverse includes the 1/n scaling.
 * group_gen (Montgomery) must be a primitive 2^log_n-th root of unity; NULL selects arkworks' default
 * generator for the field (Domain::new). */
int cs_domain_create(cs_ctx* ctx, cs_curve curve, unsigned log_n, const uint64_t* group_gen_mont,
                     cs_domain** out);
void cs_domain_free(cs_domain* dom);
size_t cs_domain_size(const cs_domain* dom);
int cs_ifft_in_to_out(cs_ctx* ctx, const cs_domain* dom, uint64_t* d_data, unsigned batch);
int cs_fft_out_to_in(cs_ctx* ctx, const cs_domain* dom, uint64_t* d_data, unsigned batch);
int cs_bit_reverse(cs_ctx* ctx, cs_curve curve, uint64_t* d_data, unsigned log_n, unsigned batch);
/* Natural-order transforms as co-plonk uses them (`T::fft / T::ifft` = domain.fft / domain.ifft on the
 * snarkjs-rooted Radix2EvaluationDomain, co-plonk/src/mpc/rep3.rs:140-152, types.rs:76-100): natural in,
 * natural out; data must hold domain-size elements (zero-pad shorter inputs as arkworks does). */
int cs_fft(cs_ctx* ctx, const cs_domain* dom, uint64_t* d_data, unsigned batch);
int cs_ifft(cs_ctx* ctx, const cs_domain* dom, uint64_t* d_data, unsigned batch);
/* evaluate_poly_public / rep3::poly::eval_poly (mpc-core/src/protocols/rep3/poly.rs:42-68): evaluate the
 * (shared) polynomial with n coefficients (`batch` components each, device memory) at a public point;
 * h_out receives `batch` field elements (the share of the evaluation). */
int cs_eval_poly(cs_ctx* ctx, cs_curve curve, const uint64_t* d_coeffs, size_t n, unsigned batch,
                 const uint64_t* h_point_mont, uint64_t* h_out);
/* host-buffer convenience wrappers (copy in, transform, copy out) -- what a drop-in for the
 * `&mut [T]` signatures of the reference binds to */
int cs_ifft_in_to_out_host(cs_ctx* ctx, const cs_domain* dom, uint64_t* h_data, unsigned batch);
int cs_fft_out_to_in_host(cs_ctx* ctx, const cs_domain* dom, uint64_t* h_data, unsigned batch);

/* ---- share-wise vector kernels ------------------------------------------------------------------
 * cs_vec_mul/add/sub: elementwise on Fr (plain driver local_mul_vec, co-groth16/src/mpc/plain.rs:83-89;
 *   `ab -= c`, reduction.rs:185-190).
 * cs_vec_scale_table: x[i] *= table[i] per component (distribute_powers_and_mul_by_const,
 *   co-groth16/src/mpc/rep3.rs:95-106; reduction.rs:166-171).
 * cs_rep3_local_mul_vec: rep3::arithmetic::local_mul_vec (mpc-core/.../rep3/arithmetic.rs:132-146):
 *   out_i = a_i.a*b_i.a + a_i.a*b_i.b + a_i.b*b_i.a + mask_i; d_mask may be NULL (zero masks);
 *   the masks themselves come from the caller's Rep3Rand (rngs.rs:137-156).
 * cs_rep3_to_shamir: bridges/rep3_to_shamir.rs:43-63, out_i = ca*x_i.a + cb*x_i.b. */
int cs_vec_mul(cs_ctx* ctx, cs_curve curve, const uint64_t* d_a, const uint64_t* d_b, uint64_t* d_out, size_t n);
int cs_vec_add(cs_ctx* ctx, cs_curve curve, const uint64_t* d_a, const uint64_t* d_b, uint64_t* d_out, size_t n);
int cs_vec_sub(cs_ctx* ctx, cs_curve curve, const uint64_t* d_a, const uint64_t* d_b, uint64_t* d_out, size_t n);
int cs_vec_scale_table(cs_ctx* ctx, cs_curve curve, uint64_t* d_x, const uint64_t* d_table, size_t n, unsigned batch);
int cs_rep3_local_mul_vec(cs_ctx* ctx, cs_curve curve, const uint64_t* d_a, const uint64_t* d_b,
                          const uint64_t* d_mask, uint64_t* d_out, size_t n);
/* out_i = sum_{j<k} w_j * in_j[i]  (k <= 8, weights Montgomery on the host, vectors on the device).
 * Shamir degree reduction (mpc-core/src/protocols/shamir/network.rs:150-243) in three uses: consuming a
 * double-sharing pair (`inp += r_2t`, `share -= r_t`: weights 1, +-1), the king's Lagrange-weighted sum of the
 * 2t+1 received vectors (:170-187), and the fresh share `acc * c_id` sent back to each party (:196-214). */
int cs_vec_lincomb(cs_ctx* ctx, cs_curve curve, const uint64_t* const* d_inputs, const uint64_t* h_weights_mont,
                   unsigned k, size_t n, uint64_t* d_out);
/* Rep3Rand::masking_field_elements_vec on the device (mpc-core/src/protocols/rep3/rngs.rs:137-156,
 * RngType = rand_chacha::ChaCha12Rng): seeds = the two ChaCha keys (own stream / previous party's stream),
 * word_pos = each rng's current position in 32-bit words (ChaCha12Rng::get_word_pos), rounds = 12.
 * Writes n masks a_i - b_i (Montgomery) to device memory; the caller advances both rngs by 8 n words.
 * cs_chacha_keystream is the test hook for the block function (RFC 7539 vector with rounds = 20). */
int cs_rep3_masks_device(cs_ctx* ctx, cs_curve curve, const uint8_t* h_seed1, uint64_t word_pos1,
                         const uint8_t* h_seed2, uint64_t word_pos2, unsigned rounds, size_t n, uint64_t* d_out);
int cs_chacha_keystream(cs_ctx* ctx, const uint8_t* h_key, uint64_t first_block, unsigned rounds, unsigned nblocks,
                        uint32_t* h_out_words);
int cs_rep3_to_shamir(cs_ctx* ctx, cs_curve curve, const uint64_t* d_x, const uint64_t* h_ca_mont,
                      const uint64_t* h_cb_mont, uint64_t* d_out, size_t n);

/* ---- Groth16: R1CSToQAP::witness_map_from_matrices + CoGroth16::prove ------------------------------
 * cs_groth16_pk_create uploads ark_groth16::ProvingKey + ConstraintMatrices once
 * (fields used by the prover: co-groth16/src/groth16.rs:219-225,234-290; lib.rs:262-272).
 *   matrices in CSR: row_ptr[num_constraints+1], col[nnz] (variable index, publics first), coeff[nnz]
 *   (Fr Montgomery).  Query arrays are affine Montgomery points.
 * cs_groth16_witness_map = CircomReduction::witness_map_from_matrices (reduction.rs:77-193):
 *   kind = CS_PLAIN: witness = Fr values, masks ignored;  kind = CS_REP3: witness = shares {a,b},
 *   party = 0..2, h_mask1/h_mask2 = the two local_mul_vec mask vectors (NULL = zero).  Output: the
 *   `domain_size` half shares of h, left on the device inside the pk scratch and (if h_out != NULL)
 *   copied to the host. */
typedef struct {
  cs_curve curve;
  size_t num_constraints, num_instance_variables, num_witness_variables;
  const uint32_t* a_row_ptr; const uint32_t* a_col; const uint64_t* a_coeff; size_t a_nnz;
  const uint32_t* b_row_ptr; const uint32_t* b_col; const uint64_t* b_coeff; size_t b_nnz;
  const uint64_t* alpha_g1; const uint64_t* beta_g1; const uint64_t* beta_g2;
  const uint64_t* delta_g1; const uint64_t* delta_g2;
  const uint64_t* a_query; size_t a_query_len;
  const uint64_t* b_g1_query; size_t b_g1_query_len;
  const uint64_t* b_g2_query; size_t b_g2_query_len;
  const uint64_t* l_query; size_t l_query_len;
  const uint64_t* h_query; size_t h_query_len;
  int window_bits; /* 0 = default */
  /* optional: the C matrix, needed only by LibSnarkReduction (groth16/reduction.rs:241-342); NULL otherwise */
  const uint32_t* c_row_ptr; const uint32_t* c_col; const uint64_t* c_coeff; size_t c_nnz;
} cs_groth16_key_desc;

int cs_groth16_pk_create(cs_ctx* ctx, const cs_groth16_key_desc* desc, cs_groth16_pk** out);
void cs_groth16_pk_free(cs_groth16_pk* pk);
size_t cs_groth16_domain_size(const cs_groth16_pk* pk);
/* the curve the key was built for (cs_curve; read from the zkey's base-field modulus by cs_groth16_pk_from_zkey) */
int cs_groth16_pk_curve(const cs_groth16_pk* pk);

/* snarkjs file ingest (what co-circom does with taceo-circom-types before calling prove,
 * co-circom/co-circom/src/bin/co-circom.rs:1005-1016): a Groth16 .zkey goes straight to the device-resident
 * key (its point sections already are Montgomery limb arrays), a .wtns to Montgomery field elements.
 * cs_wtns_read with out_mont == NULL only reports the element count. */
int cs_groth16_pk_from_zkey(cs_ctx* ctx, const char* zkey_path, int window_bits, cs_groth16_pk** out,
                            size_t* out_n_public);
int cs_wtns_read(const char* wtns_path, cs_curve curve, uint64_t* out_mont, size_t capacity, size_t* out_n);

int cs_groth16_witness_map(cs_ctx* ctx, cs_groth16_pk* pk, cs_share_kind kind, int party,
                           const uint64_t* h_public_inputs, const uint64_t* h_witness,
                           const uint64_t* h_mask1, const uint64_t* h_mask2, uint64_t* h_out);

/* LibSnarkReduction::witness_map_from_matrices (groth16/reduction.rs:241-342; the arkworks/libsnark-style
 * witness map, not used by the CLI: co-circom.rs:1020): Domain::new + coset GENERATOR, a and b from A/B,
 * c from the C matrix as half shares, ONE local_mul_vec (one mask vector), h = coefficients of
 * (a*b - c) / Z over the coset, natural order.  Requires c_* in the key descriptor. */
int cs_groth16_witness_map_libsnark(cs_ctx* ctx, cs_groth16_pk* pk, cs_share_kind kind, int party,
                                    const uint64_t* h_public_inputs, const uint64_t* h_witness,
                                    const uint64_t* h_mask, uint64_t* h_out);

/* Groth16::plain_prove (co-groth16/src/groth16.rs:484-490) with the randomness (r, s) supplied by
 * the caller (the reference draws it from thread_rng, mpc/plain.rs:23-26).  public_inputs includes
 * the leading 1; witness = the private part.  Outputs: proof A (G1), B (G2), C (G1) affine Montgomery. */
int cs_groth16_prove_plain(cs_ctx* ctx, cs_groth16_pk* pk, const uint64_t* h_public_inputs,
                           const uint64_t* h_witness, const uint64_t* h_r_mont, const uint64_t* h_s_mont,
                           uint64_t* out_a, uint64_t* out_b, uint64_t* out_c);

/* Same with the private witness already resident in device memory (e.g. left there by a GPU witness
 * extension); public inputs stay on the host (they feed the host-side public-input MSM). */
int cs_groth16_prove_plain_device(cs_ctx* ctx, cs_groth16_pk* pk, const uint64_t* h_public_inputs,
                                  const uint64_t* d_witness, const uint64_t* h_r_mont, const uint64_t* h_s_mont,
                                  uint64_t* out_a, uint64_t* out_b, uint64_t* out_c);

/* One party's LOCAL part of Rep3CoGroth16::prove up to the first network round
 * (groth16.rs:151-163 + the rayon_join5 block :227-294): witness map, then the five MSMs.
 *   r_share/s_share: this party's Rep3 shares {a,b} of r and s (T::rand, mpc/rep3.rs:27-29).
 * Outputs (affine Montgomery half shares): g_a = r_g1, g1_b = s_g1 (G1), g2_b = s_g2 (G2),
 * l_acc, h_acc (G1).  The two network legs and the final sums (groth16.rs:296-337) are run by the
 * host-side driver (co_snarks_b200/rep3.py <-> mpc-net Network). */
int cs_groth16_rep3_local(cs_ctx* ctx, cs_groth16_pk* pk, int party, const uint64_t* h_public_inputs,
                          const uint64_t* h_witness_shares, const uint64_t* h_mask1, const uint64_t* h_mask2,
                          const uint64_t* h_r_share, const uint64_t* h_s_share,
                          uint64_t* out_g_a, uint64_t* out_g1_b, uint64_t* out_g2_b,
                          uint64_t* out_l_acc, uint64_t* out_h_acc);

/* The same, restricted to a subset of the five MSMs, so that one party's local phase can be split over two
 * GPUs (SURVEY.md 8e: GPU0 takes {A, B1, L}, GPU1 takes {witness map -> H, B2}); outputs of parts that
 * were not requested are the identity.  CS_PART_H includes the witness map. */
#define CS_PART_A 1u
#define CS_PART_B1 2u
#define CS_PART_B2 4u
#define CS_PART_L 8u
#define CS_PART_H 16u
#define CS_PART_ALL 31u
int cs_groth16_rep3_local_parts(cs_ctx* ctx, cs_groth16_pk* pk, int party, unsigned parts,
                                const uint64_t* h_public_inputs, const uint64_t* h_witness_shares,
                                const uint64_t* h_mask1, const uint64_t* h_mask2, const uint64_t* h_r_share,
                                const uint64_t* h_s_share, uint64_t* out_g_a, uint64_t* out_g1_b,
                                uint64_t* out_g2_b, uint64_t* out_l_acc, uint64_t* out_h_acc);

/* The same with the two witness-map mask vectors drawn ON THE DEVICE from the party's correlated ChaCha
 * streams (Rep3Rand, rngs.rs:86-156): mask1 uses words [pos, pos + 8n) of each stream, mask2 the next 8n
 * words (two consecutive masking_field_elements_vec calls, reduction.rs:160,182); the caller advances
 * both rngs by 16 n words.  prf == NULL falls back to the host-supplied h_mask1 / h_mask2. */
typedef struct {
  uint8_t seed1[32]; uint64_t word_pos1;   /* this party's stream  (rng1) */
  uint8_t seed2[32]; uint64_t word_pos2;   /* previous party's stream (rng2) */
  unsigned rounds;                         /* 12 = ChaCha12Rng */
} cs_rep3_prf;
int cs_groth16_rep3_local_prf(cs_ctx* ctx, cs_groth16_pk* pk, int party, unsigned parts,
                              const uint64_t* h_public_inputs, const uint64_t* h_witness_shares,
                              const uint64_t* h_mask1, const uint64_t* h_mask2, const cs_rep3_prf* prf,
                              const uint64_t* h_r_share, const uint64_t* h_s_share, uint64_t* out_g_a,
                              uint64_t* out_g1_b, uint64_t* out_g2_b, uint64_t* out_l_acc, uint64_t* out_h_acc);

/* mul_vec on large share vectors as ONE kernel over NVLink peer memory
 * (rep3::arithmetic::local_mul_vec + reshare_vec, mpc-core/src/protocols/rep3/arithmetic.rs:132-160; the
 * call pattern of co-plonk/src/mpc/rep3.rs:185-196 and round3.rs): z_i = a_i*b_i + mask_i with the masks
 * drawn in registers from `prf` (NULL = no masks), d_out[i].a = z_i, and -- when d_next_out is not NULL --
 * d_next_out[i].b = z_i, where d_next_out is the NEXT party's d_out mapped with cs_ipc_open (or any device
 * pointer this GPU can store to).  Asynchronous on the context stream: once all three parties' kernels have
 * completed (stream sync + barrier), every d_out holds full Rep3PrimeFieldShare{a,b} elements.  The caller
 * advances both rngs by 8 n words.  cs_rep3_set_b is the staging-buffer variant of the second half
 * (d_out[i].b = d_recv[i]) for transports that deliver the b-halves as a contiguous vector. */
int cs_rep3_mul_vec_reshare(cs_ctx* ctx, cs_curve curve, const uint64_t* d_a, const uint64_t* d_b, size_t n,
                            const cs_rep3_prf* prf, uint64_t* d_out, uint64_t* d_next_out);
int cs_rep3_set_b(cs_ctx* ctx, cs_curve curve, const uint64_t* d_recv, size_t n, uint64_t* d_out);
/* One process per GPU: export a cs_malloc'ed buffer as a 64-byte CUDA IPC handle / map a peer's handle
 * (peer access over NVLink is enabled on first use) / unmap it. */
int cs_ipc_export(cs_ctx* ctx, const void* d_ptr, uint8_t* out_handle64);
int cs_ipc_open(cs_ctx* ctx, const uint8_t* handle64, void** out_peer_ptr);
int cs_ipc_close(cs_ctx* ctx, void* peer_ptr);

/* ---- sharing on the device (SURVEY.md 8f rank 2) -----------------------------------------------------------
 * cs_share_rep3_device: rep3::share_field_elements (mpc-core/src/protocols/rep3.rs:281-293; what split-witness /
 * CompressedRep3SharedWitness::share_rep3 with Compression::None produce, co-circom-types/src/lib.rs:279-382) for a
 * device-resident witness: a, b uniform by rejection sampling (F::rand), c = val - a - b; d_share0/1/2 receive the
 * three parties' n x {a, b} vectors (they may live on other GPUs: any pointer this GPU can store to).  seed32 = the
 * ChaCha12 key of the dealer's rng (NULL: OS entropy); element i draws from the sub-streams 2i and 2i + 1.
 * cs_fr_rand_device: n uniform elements (F::rand), element i from sub-stream stream_base + i. */
int cs_share_rep3_device(cs_ctx* ctx, cs_curve curve, const uint64_t* d_witness, size_t n, const uint8_t* h_seed32,
                         uint64_t* d_share0, uint64_t* d_share1, uint64_t* d_share2);
int cs_fr_rand_device(cs_ctx* ctx, cs_curve curve, const uint8_t* h_seed32, uint64_t stream_base, uint64_t* d_out, size_t n);

/* ---- share files: CompressedRep3SharedWitness (co-circom-types/src/lib.rs:162-219; written by `co-circom
 * split-witness`, read by generate-proof with bincode::deserialize_from, co-circom.rs:1014-1016) -----------------
 * bincode 1 (fixed-width little-endian integers) over serde derives: public_inputs = bytes(ark-compressed Vec<F>),
 * then the Rep3ShareVecType variant (u32): 0 Replicated(bytes(Vec<{a, b}>)), 1 SeededReplicated{a, b: SeededType},
 * 2 Additive(bytes(Vec<F>)), 3 SeededAdditive(SeededType); SeededType = 0 Shares(bytes) | 1 Seed([u8; 32], u64 len),
 * expanded as len x F::rand over ChaCha12Rng::from_seed (rep3.rs:181-196).  ark field elements are 32 canonical
 * little-endian bytes.  Output: public inputs and shares in Montgomery form; *out_kind = CS_REP3 for replicated
 * shares (n_witness x {a, b}) or CS_PLAIN for additive half shares (n_witness x Fr) that still need
 * cs_rep3_replicate_additive (uncompress_shared_witness reshares once, co-circom/src/lib.rs:64-73).
 * Pass out buffers = NULL to query the sizes.  No reference fixture of this format exists in the repository: the
 * layout is restated from the serde derives ("parity unpinned" at the byte level; round-trip tested). */
int cs_rep3_witness_read(const char* path, cs_curve curve, uint64_t* out_public, size_t public_capacity,
                         uint64_t* out_shares, size_t shares_capacity_elems, size_t* out_n_public, size_t* out_n_witness,
                         cs_share_kind* out_kind);
/* additive -> replicated: send my additive share vector to the next party, receive the previous party's:
 * share_i = (mine_i, prev_i)  (Rep3NetworkExt::reshare_many) */
int cs_rep3_replicate_additive(cs_net* net, const uint64_t* h_additive, size_t n, uint64_t* h_out_shares);

/* ---- batched witness-extension VM operations (circom-mpc-vm/src/mpc/batched_rep3.rs:124-188, 322-337) ----------
 * BatchedCircomRep3VmWitnessExtension runs one circuit on a batch of inputs, so every VM opcode acts on a vector of
 * `batch_size` values.  These are its arithmetic opcodes on device-resident vectors: shares = n x {a, b}, publics =
 * n x Fr (Montgomery).  `op` selects the reference function:
 *   CS_R3B_ADD / CS_R3B_SUB            arithmetic::add / sub                         (shared, shared)
 *   CS_R3B_ADD_PUBLIC                  arithmetic::add_public                        (shared, public)
 *   CS_R3B_SUB_PUBLIC                  arithmetic::sub_shared_by_public              (shared - public)
 *   CS_R3B_PUBLIC_SUB                  arithmetic::sub_public_by_shared              (public - shared)
 *   CS_R3B_MUL_PUBLIC                  arithmetic::mul_public
 *   CS_R3B_NEG                         -shared                                        (d_y = NULL)
 *   CS_R3B_PROMOTE                     arithmetic::promote_to_trivial_share          (d_x = NULL, d_y = publics)
 * The secret x secret `mul` (batched_rep3.rs:185 -> arithmetic::mul_vec) is cs_rep3_mul_vec_reshare above: product,
 * masks and the store into the next party's vector in one kernel.
 * `open` (batched_rep3.rs:322-327 -> open_vec): cs_rep3_batch_open_send copies the b-components into d_next_recv
 * (the NEXT party's receive buffer mapped with cs_ipc_open, or a local staging buffer for other transports);
 * after the parties have met, cs_rep3_batch_open_finish adds a + b + received. */
typedef enum {
  CS_R3B_ADD = 0, CS_R3B_SUB = 1, CS_R3B_ADD_PUBLIC = 2, CS_R3B_SUB_PUBLIC = 3, CS_R3B_PUBLIC_SUB = 4,
  CS_R3B_MUL_PUBLIC = 5, CS_R3B_NEG = 6, CS_R3B_PROMOTE = 7
} cs_rep3_batch_op;
int cs_rep3_batch(cs_ctx* ctx, cs_curve curve, cs_rep3_batch_op op, int party, const uint64_t* d_x,
                  const uint64_t* d_y, uint64_t* d_out, size_t n);
int cs_rep3_batch_open_send(cs_ctx* ctx, cs_curve curve, const uint64_t* d_shares, size_t n, uint64_t* d_next_recv);
int cs_rep3_batch_open_finish(cs_ctx* ctx, cs_curve curve, const uint64_t* d_shares, const uint64_t* d_recv,
                              uint64_t* d_out_public, size_t n);

/* ---- UltraHonk commitments: CoUtils::commit / commit_and_send (co-noir/co-noir-common/src/lib.rs:57-101) ->
 * T::msm_public_points(&crs.monomials[..poly.len()], poly) -> HonkCurve::fast_msm = msm_unchecked
 * (honk_curve.rs:81-83; the reference chops to the shorter slice, :33-34).  The Oink prover commits the wire,
 * lookup and permutation polynomials one after the other (co_oink_prover.rs:547-700: w_l, w_r, w_o,
 * lookup_read_counts, lookup_read_tags, w_4, lookup_inverses, z_perm); here a round's polynomials are committed
 * concurrently (one stream and MSM workspace each) against the resident CRS table (cs_bases_from_crs_file).
 *   share_kind CS_PLAIN: polys[k] = lens[k] x Fr                -> out_points[k]            (plain / Shamir shares)
 *              CS_REP3 : polys[k] = lens[k] x {a, b}            -> out_points[2k], [2k+1]   (Rep3PointShare a, b:
 *                                                                   co-noir-common/src/mpc/rep3.rs:259-266)
 * polys are device pointers; k <= 4 per call. */
int cs_honk_commit_batch(cs_ctx* ctx, const cs_bases* crs, cs_share_kind kind, const uint64_t* const* d_polys,
                         const size_t* lens, unsigned k, uint64_t* h_out_points);

/* ---- party-to-party transport: mpc_net::Network (mpc-net/src/lib.rs:34-63: id / send / recv) -------------
 * A cs_net is one n-party mesh.  Two implementations:
 *  (1) callbacks -- the host language hands over its own transport (the Rust shim wraps `&N: Network`,
 *      the CPU tests wrap torch.distributed/gloo); `send` must not block on the receiver (mpc-net queues),
 *      `recv` blocks until `bytes` bytes from `from_party` have arrived.  Return 0 on success.
 *  (2) peer mailboxes -- mpc-net replaced on-box: every party owns a small mailbox in the HBM of its GPU;
 *      a send is a copy into the RECEIVER's mailbox through a CUDA-IPC mapping (NVLink peer memory; same-GPU
 *      processes work too), ordered payload-then-sequence-number on a dedicated copy stream, with credits so
 *      a slow receiver is never overrun.  Messages of any size (chunked); the Groth16 legs send 64..192 bytes.
 *      Bootstrap: create, exchange the 64-byte handles by any means (torch.distributed, files), connect.
 *      Parties living in ONE process (threads) connect with cs_net_peer_connect_local instead. */
typedef struct {
  void* user;
  int (*send)(void* user, int to_party, const void* data, size_t bytes);
  int (*recv)(void* user, int from_party, void* data, size_t bytes);
} cs_net_callbacks;
int cs_net_from_callbacks(int id, int n_parties, const cs_net_callbacks* cb, cs_net** out);
int cs_net_peer_create(cs_ctx* ctx, int id, int n_parties, cs_net** out);
int cs_net_peer_handle(cs_net* net, uint8_t* out_handle64);
/* handles: n_parties x 64 bytes, indexed by party id (the own entry is ignored) */
int cs_net_peer_connect(cs_net* net, const uint8_t* handles);
int cs_net_peer_connect_local(cs_net* net, cs_net* const* peers /* n_parties entries, own may be NULL */);
int cs_net_send(cs_net* net, int to_party, const void* data, size_t bytes);
int cs_net_recv(cs_net* net, int from_party, void* data, size_t bytes);
/* Send to `to` and receive from `from` in one call; on mailbox nets both directions advance chunk by chunk, so an
 * all-to-all of messages larger than the credit window (8 x 64 KB per channel) cannot dead-lock with every party
 * sending first.  Callback nets: send then recv (the transport queues sends, like mpc_net::Network::send). */
int cs_net_sendrecv(cs_net* net, int to, const void* sdata, size_t sbytes, int from, void* rdata, size_t rbytes);
uint64_t cs_net_bytes_sent(const cs_net* net);
void cs_net_free(cs_net* net);

/* ---- Rep3State (mpc-core/src/protocols/rep3.rs:43-75): the party's correlated randomness --------------
 * rng1 = this party's ChaCha12 stream, rng2 = the previous party's (Rep3Rand, rngs.rs:86-98).
 * cs_rep3_state_create draws seed1 from the OS entropy pool (getrandom(2); the reference:
 * ChaCha12Rng::from_entropy) and exchanges it exactly like setup_prf: seed2 = net.reshare(seed1).
 * cs_rep3_state_from_seeds is the deterministic constructor for tests and for callers whose Rust side
 * already holds a Rep3State (pass the two seeds and word positions).  fork mirrors MpcState::fork:
 * both parties derive the child seeds from their streams, no communication. */
typedef struct cs_rep3_state cs_rep3_state;
int cs_rep3_state_create(cs_net* net, cs_rep3_state** out);
int cs_rep3_state_from_seeds(int party, const uint8_t* seed_own32, uint64_t word_pos_own,
                             const uint8_t* seed_prev32, uint64_t word_pos_prev, cs_rep3_state** out);
int cs_rep3_state_fork(cs_rep3_state* st, cs_rep3_state** out);
/* current (seed, word position) of both streams -- what cs_*_prf entry points take */
int cs_rep3_state_prf(const cs_rep3_state* st, cs_rep3_prf* out);
int cs_rep3_state_advance(cs_rep3_state* st, uint64_t nwords);
/* arithmetic::rand (rep3/arithmetic.rs:357-360): share (a, b) = (F::rand(rng1), F::rand(rng2)), Montgomery;
 * ark-ff's Fp::rand = rejection sampling on the top-masked 64-bit limbs. */
int cs_rep3_state_rand(cs_rep3_state* st, cs_curve curve, uint64_t* out_share /* a || b */);
void cs_rep3_state_free(cs_rep3_state* st);
/* 32 bytes from the OS entropy pool (seeds for tests that want fresh randomness; r, s of plain_prove) */
int cs_os_random(uint8_t* out, size_t bytes);

/* ---- Rep3CoGroth16::prove (co-groth16/src/groth16.rs:360-379 -> prove_inner :125-177 ->
 * create_proof_with_assignment :207-338), the whole party: local phase on the GPU, then the reference's two
 * network legs inside the library -- round 1: open_half_point(g_a) on net0 | scalar_mul(g1_b, r) on net1
 * (:305-308); round 2: open_half_point(g_c) on net0 | open_half_point(g2_b) on net1 (:325-328) -- four
 * point-sized messages per party, and the final sums (:314-322) on the host while nothing else waits.
 *   net0, net1  two 3-party meshes as in the CLI's TcpNetwork::networks::<2> (co-circom.rs:1003); the same
 *               handle may be passed twice.
 *   state       Rep3State of this party (consumed: advanced by the 16 n mask words + the r, s, rs-mask and
 *               EC-mask draws, in the reference's order).
 *   witness     h_witness_shares (host, [nw][a||b]) or d_witness_shares (already resident); exactly one.
 *   out_rs      optional [4][limbs]: r.a, r.b, s.a, s.b -- lets a test reconstruct r = sum r_i.a.
 * Every party returns the same opened proof (A, B, C affine Montgomery). */
int cs_groth16_rep3_prove(cs_ctx* ctx, cs_groth16_pk* pk, cs_net* net0, cs_net* net1, cs_rep3_state* state,
                          const uint64_t* h_public_inputs, const uint64_t* h_witness_shares,
                          const uint64_t* d_witness_shares, uint64_t* out_a, uint64_t* out_b, uint64_t* out_c,
                          uint64_t* out_rs);
/* Two GPUs per party (SURVEY.md 8e-2): the party's second GPU runs {witness map -> H, B2} and hands the two
 * points to the first through `pair` (a 2-party cs_net: id 0 = the protocol GPU, id 1 = the helper); the first
 * runs {A, B1, L} and the protocol.  Both are given states with identical seeds (cs_rep3_state_from_seeds from
 * cs_rep3_state_prf of the main's state) so that their draws stay in lock-step. */
int cs_groth16_rep3_prove_main(cs_ctx* ctx, cs_groth16_pk* pk, cs_net* net0, cs_net* net1, cs_net* pair,
                               cs_rep3_state* state, const uint64_t* h_public_inputs,
                               const uint64_t* h_witness_shares, const uint64_t* d_witness_shares,
                               uint64_t* out_a, uint64_t* out_b, uint64_t* out_c, uint64_t* out_rs);
int cs_groth16_rep3_prove_helper(cs_ctx* ctx, cs_groth16_pk* pk, int party, cs_net* pair, cs_rep3_state* state,
                                 const uint64_t* h_public_inputs, const uint64_t* h_witness_shares,
                                 const uint64_t* d_witness_shares);

/* ---- Shamir(n, t): ShamirPreprocessing / ShamirState (mpc-core/src/protocols/shamir.rs:26-186), the DN07 double
 * sharings (shamir/rngs.rs:334-470), king-based degree reduction (shamir/network.rs:150-301) and the openings
 * (shamir/pointshare.rs:102-111) over an n-party cs_net.  num_parties >= 2 threshold + 1 (shamir.rs:41-43).
 * `amount` pairs are preprocessed at creation (rounded up to batches of t + 1); get_pair refills on demand. */
typedef struct cs_shamir_state cs_shamir_state;
int cs_shamir_state_create(cs_net* net, cs_curve curve, int num_parties, int threshold, size_t amount, cs_shamir_state** out);
int cs_shamir_state_fork(cs_shamir_state* st, size_t amount, cs_shamir_state** out);
size_t cs_shamir_state_pairs(const cs_shamir_state* st);
void cs_shamir_state_free(cs_shamir_state* st);
/* ShamirState::rand: a degree-t share of a value no party knows (the r_t half of a pair) */
int cs_shamir_state_rand(cs_shamir_state* st, cs_net* net, uint64_t* out_share);
/* the party's opening weights: open_lagrange_t (t + 1 entries) or open_lagrange_2t (2t + 1), for the parties
 * id, id-1, id-2, ... (mod n) in that order */
int cs_shamir_open_lagrange(const cs_shamir_state* st, int degree_2t, uint64_t* out, size_t capacity_elems, size_t* out_n);
/* degree_reduce_many on a device vector of degree-2t values (the result of a local share product): consumes one pair
 * per element; inp += r_2t, parties 1..2t send to the king (party 0), the king accumulates with the Lagrange weights
 * (one k_vec_lincomb launch), shares the result as a known polynomial with t zero shares and sends acc * P(id + 1)
 * to parties 0..n-t-1; share -= r_t.  Vector arithmetic on the GPU, traffic through cs_net. */
int cs_shamir_degree_reduce_many(cs_ctx* ctx, cs_shamir_state* st, cs_net* net, const uint64_t* d_in, size_t len, uint64_t* d_out);
/* degree_reduce_point: the same for one point share; `base_affine` is the public point the pair is lifted with
 * (the reference uses the group generator) */
int cs_shamir_degree_reduce_point(cs_shamir_state* st, cs_net* net, cs_group group, const uint64_t* base_affine,
                                  const uint64_t* in_affine, uint64_t* out_affine);
/* open_half_point: broadcast_next over 2t + 1 parties + reconstruct_point with open_lagrange_2t */
int cs_shamir_open_half_point(cs_shamir_state* st, cs_net* net, cs_group group, const uint64_t* in_affine, uint64_t* out_affine);

/* ShamirCoGroth16::prove (co-groth16/src/groth16.rs:439-463 -> prove_inner -> create_proof_with_assignment with
 * ShamirGroth16Driver, mpc/shamir.rs): three pairs are preprocessed over net0 (two rand calls, one for scalar_mul's
 * degree_reduce_point), state1 = state0.fork(1); local phase on the GPU (cs_groth16_shamir_local), then
 * open_half_point(g_a) | scalar_mul(g1_b, r) = degree_reduce_point + local product, then the openings of g_c and
 * g2_b as degree-2t sharings.  out_rs (optional, 2 x Fr): this party's shares of r and s. */
int cs_groth16_shamir_prove(cs_ctx* ctx, cs_groth16_pk* pk, cs_net* net0, cs_net* net1, int num_parties, int threshold,
                            const uint64_t* h_public_inputs, const uint64_t* h_witness_shares, uint64_t* out_a,
                            uint64_t* out_b, uint64_t* out_c, uint64_t* out_rs);
/* CoGroth16::prove_with_shamir_bridge (groth16.rs:394-417): a Rep3-shared witness is translated locally to
 * Shamir(t = 1, n = 3) shares (bridges/rep3_to_shamir.rs:31-63; k_rep3_to_shamir on the device) and proved with the
 * Shamir driver. */
int cs_groth16_prove_with_shamir_bridge(cs_ctx* ctx, cs_groth16_pk* pk, cs_net* net0, cs_net* net1,
                                        const uint64_t* h_public_inputs, const uint64_t* h_witness_rep3_shares,
                                        uint64_t* out_a, uint64_t* out_b, uint64_t* out_c, uint64_t* out_rs);

/* ShamirGroth16Driver's local phase (co-groth16/src/mpc/shamir.rs:29-119): identical arithmetic to the plain
 * driver on degree-t shares -- every party adds the public terms/points; outputs are degree-2t point shares
 * that the host protocol opens (shamir/pointshare.rs:86-113). */
int cs_groth16_shamir_local(cs_ctx* ctx, cs_groth16_pk* pk, const uint64_t* h_public_inputs,
                            const uint64_t* h_witness_shares, const uint64_t* h_r_share, const uint64_t* h_s_share,
                            uint64_t* out_g_a, uint64_t* out_g1_b, uint64_t* out_g2_b,
                            uint64_t* out_l_acc, uint64_t* out_h_acc);

/* ---- Plonk (snarkjs) prover, plain driver: co-circom/co-plonk/src/lib.rs:80-115 (prove_inner) with
 * PlainPlonkDriver (mpc/plain.rs) == Plonk::plain_prove (lib.rs:271-281) ----------------------------------
 * cs_plonk_pk_create uploads circom_types::plonk::Zkey once (fields read by the prover: round1.rs:109-224
 * additions + wire maps, round2.rs:99-160 sigma evaluations, round3.rs:330-420 selector / sigma / Lagrange
 * evaluations on the extended domain, round4.rs:143-144 + round5.rs:150-230 coefficient forms, p_tau) and
 * allocates the per-proof workspace.  All field elements Montgomery, points affine Montgomery, (0,0) = infinity.
 * Polynomials: `coeffs` = domain_size values, `evals` = 4 * domain_size values (the zkey stores both). */
typedef struct cs_plonk_pk cs_plonk_pk;
typedef struct {
  cs_curve curve;
  uint32_t n_vars, n_public, domain_size, n_additions, n_constraints;
  const uint64_t* k1_mont;            /* verifying_key.k1, k2 */
  const uint64_t* k2_mont;
  const uint64_t* vk_points;          /* Qm Ql Qr Qo Qc S1 S2 S3 (G1), hashed into the transcript (round2.rs:211-218) */
  const uint32_t* additions_ids;      /* n_additions x (signal_id1, signal_id2) */
  const uint64_t* additions_factors;  /* n_additions x (factor1, factor2) */
  const uint32_t* map_a;              /* n_constraints wire -> signal maps */
  const uint32_t* map_b;
  const uint32_t* map_c;
  const uint64_t* q_coeffs[5];        /* qm ql qr qo qc */
  const uint64_t* q_evals[5];
  const uint64_t* s_coeffs[3];        /* sigma 1..3 */
  const uint64_t* s_evals[3];
  const uint64_t* lagrange_evals;     /* max(1, n_public) x 4 * domain_size */
  const uint64_t* p_tau;              /* SRS powers, n_p_tau >= domain_size + 6 G1 points */
  size_t n_p_tau;
} cs_plonk_key_desc;
int cs_plonk_pk_create(cs_ctx* ctx, const cs_plonk_key_desc* desc, cs_plonk_pk** out);
/* Base set straight from a Barretenberg / Ignition CRS file (co-noir/co-noir-common/src/crs/parse.rs:93-101,
 * 154-158: 64 B per G1 point, x then y, big-endian canonical): points [offset, offset + n) become a cs_bases. */
int cs_bases_from_crs_file(cs_ctx* ctx, const char* path, size_t offset, size_t n, int window_bits, cs_bases** out);
/* The same straight from a snarkjs Plonk .zkey (circom_types::plonk::Zkey::from_reader, co-circom.rs:1053-1060);
 * out_n_witness = number of private witness values a proof takes (nVars - nAdditions - nPublic - 1). */
int cs_plonk_pk_from_zkey(cs_ctx* ctx, const char* path, cs_plonk_pk** out, size_t* out_n_public, size_t* out_n_witness);
void cs_plonk_pk_free(cs_plonk_pk* pk);
int cs_plonk_pk_curve(const cs_plonk_pk* pk);
/* what a driver needs to know about an uploaded key: counts and the eight verification-key commitments
 * (Qm Ql Qr Qo Qc S1 S2 S3, affine Montgomery) that open the transcript; any output pointer may be NULL */
int cs_plonk_pk_info(const cs_plonk_pk* pk, size_t* n_public, size_t* n_witness, size_t* domain_size, uint64_t* vk_points);
/* One proof.  h_public_inputs: n_public + 1 values as in SharedWitness.public_inputs (entry 0, the constant one,
 * is replaced by zero like types.rs:118-120); h_witness: the remaining n_vars - n_additions - n_public - 1
 * values; h_blinders_mont: the 11 round-1 blinding scalars b[0..11) (Round1Challenges, round1.rs:45-47) -- the
 * caller draws them, which is what makes proofs reproducible against the oracle / the reference's KATs.
 * out_points: 9 G1 affine points A B C Z T1 T2 T3 Wxi Wxiw; out_evals: eval_a eval_b eval_c eval_s1 eval_s2
 * eval_zw (PlonkProof, round5.rs:50-70).  Errors mirror PlonkProofError (lib.rs:40-69).
 * The key object owns the per-proof workspace: one proof at a time per cs_plonk_pk (use one key object per
 * concurrent prover thread; Rep3 sessions carry their own workspace and may share a key). */
int cs_plonk_prove_plain(cs_ctx* ctx, cs_plonk_pk* pk, const uint64_t* h_public_inputs, size_t n_public_inputs,
                         const uint64_t* h_witness, size_t n_witness, const uint64_t* h_blinders_mont,
                         uint64_t* out_points, uint64_t* out_evals);
/* ---- Rep3 co-Plonk (Rep3CoPlonk::prove, co-plonk/src/lib.rs:222-240; driver traits co-plonk/src/mpc.rs:16-185,
 * Rep3 implementation mpc/rep3.rs) -- one session per party, stepped by the host protocol driver
 * (co_snarks_b200/plonk.py), which opens what each step returns and hashes the transcript.
 * Shares are interleaved {a, b} (4 limbs each).  Products that must become replicated shares again are written
 * into this party's arena slot (.a) and the NEXT party's (.b): pass the next party's arena (cs_ipc_open'ed or a
 * same-process pointer) to cs_plonk_rep3_connect, or NULL to move the a-halves yourself (cs_rep3_set_b).
 * Slots written per step: ROUND2_A {0,1}, ROUND2_B {2,3}, ROUND2_D {4,5}, ROUND2_E {6}: n shares each;
 * ROUND3_A {0..11}: 4n shares each.  All parties must finish a step before any starts the next one.
 * Step inputs / outputs (host, Montgomery):
 *   ROUND2_A in beta, gamma                    ROUND2_B -
 *   ROUND2_C out g (n) | q (n+1) additive      ROUND2_D in the opened sums G | Q
 *   ROUND2_E -                                 ROUND2_F out y (n) additive
 *   ROUND2_G in the opened Y; out partial [z]  ROUND3_A in alpha
 *   ROUND3_B out partial [t1] [t2] [t3]        ROUND4 in xi; out partial eval a b c zw, then public eval s1 s2
 *   ROUND5 in xi, v, eval_a eval_b eval_c eval_s1 eval_s2 eval_zw (opened); out partial [Wxi] [Wxiw]
 * "partial" = this party's additive share of the point / scalar: the sum over the parties is the proof element
 * (open_point_g1 / open_vec, mpc/rep3.rs:113-138).  round1 takes the party's correlated ChaCha streams
 * (masks and the random shares of round 2 are drawn on the device); cs_plonk_rep3_prf_words = words consumed. */
typedef struct cs_plonk_rep3 cs_plonk_rep3;
enum {
  CS_PLONK_R3_ROUND2_A = 1, CS_PLONK_R3_ROUND2_B, CS_PLONK_R3_ROUND2_C, CS_PLONK_R3_ROUND2_D, CS_PLONK_R3_ROUND2_E,
  CS_PLONK_R3_ROUND2_F, CS_PLONK_R3_ROUND2_G, CS_PLONK_R3_ROUND3_A, CS_PLONK_R3_ROUND3_B, CS_PLONK_R3_ROUND4,
  CS_PLONK_R3_ROUND5
};
int cs_plonk_rep3_create(cs_ctx* ctx, cs_plonk_pk* pk, int party, cs_plonk_rep3** out);
void cs_plonk_rep3_free(cs_plonk_rep3* s);
int cs_plonk_rep3_arena(cs_plonk_rep3* s, void** d_arena, size_t* slot_bytes, unsigned* n_slots);
int cs_plonk_rep3_connect(cs_plonk_rep3* s, void* d_next_arena);
/* Device-resident openings of the two large masked vectors: ROUND2_C / ROUND2_F leave their additive output at
 * *d_additive_out (h_out may be NULL); ROUND2_D / ROUND2_G called with h_in == NULL read the opened sum from
 * *d_opened_in, where the driver has added up the three parties' vectors (e.g. ncclAllGather + cs_vec_add). */
int cs_plonk_rep3_io(cs_plonk_rep3* s, void** d_additive_out, void** d_opened_in);
int cs_plonk_rep3_round1(cs_plonk_rep3* s, const cs_rep3_prf* prf, const uint64_t* h_public_inputs, size_t n_public_inputs,
                         const uint64_t* h_witness_shares, size_t n_witness, const uint64_t* h_blinder_shares,
                         uint64_t* out_points);
int cs_plonk_rep3_step(cs_plonk_rep3* s, int step, const uint64_t* h_in, uint64_t* h_out);
uint64_t cs_plonk_rep3_prf_words(const cs_plonk_rep3* s);

/* The previous and the next party's additive-out vectors (their cs_plonk_rep3_io d_additive_out; CUDA-IPC-mapped or
 * same-process pointers): openings of n-sized vectors then READ THE PEERS' HBM (two vector additions over NVLink,
 * fenced by token rounds) instead of travelling through the net.  NULL, NULL = through the net. */
int cs_plonk_rep3_connect_io(cs_plonk_rep3* s, void* d_prev_out, void* d_next_out);

/* Rep3CoPlonk::prove for one party (co-plonk/src/lib.rs:222-240; prove_inner :80-115; openings mpc/rep3.rs:113-138):
 * the whole step sequence above, the Keccak-256 transcript (types.rs:140-190) and the openings, inside the library
 * over `net` (3 parties; the session's party id must equal the net's).  `state`: the party's correlated streams -- the
 * eleven round-1 blinder shares are drawn from it with T::rand unless h_blinder_shares (11 x {a, b}) is given, the
 * device kernels draw their masks from the positions that follow, and the streams are advanced past everything
 * consumed even when the call fails.  out_points: A B C Z T1 T2 T3 Wxi Wxiw (affine, Montgomery); out_evals:
 * eval_a eval_b eval_c eval_s1 eval_s2 eval_zw.  Every party returns the same opened proof. */
int cs_plonk_rep3_prove(cs_plonk_rep3* s, cs_net* net, cs_rep3_state* state, const uint64_t* h_public_inputs,
                        size_t n_public_inputs, const uint64_t* h_witness_shares, size_t n_witness,
                        const uint64_t* h_blinder_shares, uint64_t* out_points, uint64_t* out_evals);
/* sha3::Keccak256 of a host buffer (the transcript hash, types.rs:13-14); test hook. */
int cs_keccak256(const uint8_t* data, size_t len, uint8_t* out32);

/* ---- single-point helpers used by the host-side protocol code (latency-only, run on the host) -----
 * scalar_mul_public_point_hs (mpc/rep3.rs:141-146), point addition / negation for
 * open_half_point (pointshare.rs:152-155) and the final sums (groth16.rs:314-322).
 * scalar is Fr in Montgomery form. */
int cs_point_scalar_mul(cs_curve curve, cs_group group, const uint64_t* point_affine_mont,
                        const uint64_t* scalar_mont, uint64_t* out_affine_mont);
int cs_point_add(cs_curve curve, cs_group group, const uint64_t* p_affine_mont, const uint64_t* q_affine_mont,
                 uint64_t* out_affine_mont);
int cs_point_neg(cs_curve curve, cs_group group, const uint64_t* p_affine_mont, uint64_t* out_affine_mont);
/* Fr helpers: Montgomery <-> canonical, multiplication, and the snarkjs roots of unity
 * (groth16_roots_of_unity, co-groth16/src/groth16.rs:91-100). */
int cs_fr_to_mont(cs_curve curve, const uint64_t* in_canonical, uint64_t* out_mont, size_t n);
int cs_fr_from_mont(cs_curve curve, const uint64_t* in_mont, uint64_t* out_canonical, size_t n);
int cs_fq_to_mont(cs_curve curve, const uint64_t* in_canonical, uint64_t* out_mont, size_t n);
int cs_fq_from_mont(cs_curve curve, const uint64_t* in_mont, uint64_t* out_canonical, size_t n);
/* single-element Fr arithmetic in Montgomery form (r*s of groth16.rs:297, share algebra of the host protocol) */
int cs_fr_mul(cs_curve curve, const uint64_t* a_mont, const uint64_t* b_mont, uint64_t* out_mont);
int cs_fr_inv(cs_curve curve, const uint64_t* a_mont, uint64_t* out_mont);
int cs_fr_add(cs_curve curve, const uint64_t* a_mont, const uint64_t* b_mont, uint64_t* out_mont);
int cs_fr_sub(cs_curve curve, const uint64_t* a_mont, const uint64_t* b_mont, uint64_t* out_mont);
int cs_groth16_roots_of_unity(cs_curve curve, unsigned pow, uint64_t* out_group_gen_mont,
                              uint64_t* out_coset_shift_mont);

/* ---------------------------------------------------------------------------------------------------------------
 * UltraHonk sumcheck, prover side (co-noir/co-ultrahonk/src/co_decider/co_sumcheck/*; plain prover:
 * co-noir/ultrahonk/src/decider/sumcheck/*).  Field elements are Montgomery Fr; a Rep3 share is {a, b}.
 * ------------------------------------------------------------------------------------------------------------- */

/* GateSeparatorPolynomial::new (ultrahonk/src/decider/types.rs:53-67): d_out[j] = prod over the set bits i of j of
 * betas[i], j < 2^log_n (d_out: device, 2^log_n elements). */
int cs_sumcheck_gate_separator(cs_ctx* ctx, cs_curve curve, const uint64_t* h_betas_mont, unsigned log_n, uint64_t* d_out);

/* partially_evaluate_init / partially_evaluate_inplace (co_sumcheck_prover.rs:33-97) for a batch of polynomials of
 * the same current length `len` (even): d_out[k][i] = d_in[k][2i] + (d_in[k][2i+1] - d_in[k][2i]) * u, i < len/2.
 * d_in / d_out: host arrays of n_polys device pointers; shared = 0: public values, 1: Rep3 shares (both components).
 * When len == 2 a zero is written behind the single result, as the reference keeps two entries (:75-77, :91-93), so
 * output buffers hold at least two elements.  An output may not alias its input: callers ping-pong two buffers where
 * the reference folds in place.  Runs on the context's stream, asynchronously. */
int cs_sumcheck_fold(cs_ctx* ctx, cs_curve curve, const uint64_t* const* d_in, uint64_t* const* d_out, size_t n_polys,
                     int shared, size_t len, const uint64_t* h_challenge_mont);

/* The polynomials UltraArithmeticRelation::add_entities batches (relations/ultra_arithmetic_relation.rs:252-268):
 * device pointers, `round_size` rows each.  Witness columns are Fr values (CS_PLAIN) or Rep3 shares (CS_REP3);
 * selectors are public. */
typedef struct {
  const uint64_t *w_l, *w_r, *w_o, *w_4, *w_l_shift, *w_4_shift;
  const uint64_t *q_m, *q_l, *q_r, *q_o, *q_4, *q_c, *q_arith;
} cs_honk_arith_polys;

/* One sumcheck round of the UltraArithmeticRelation over all edges (row pairs) of the round:
 * SumcheckRound::compute_univariate_inner's loop (co_sumcheck_round.rs:261-305: extend_edges, scaling factor
 * beta_products[(edge >> 1) * periodicity], accumulate) restricted to that relation.
 *   h_r0: 6 evaluations of sub-relation 0 -- Fr values (plain) or this party's ADDITIVE share (Rep3: the half-shared
 *         accumulator UltraArithmeticRelationAccHalfShared::r0); h_r1: 5 evaluations of sub-relation 1 -- Fr values
 *         (plain, 5 x Fr) or Rep3 shares (5 x {a, b}).
 *   prf (Rep3, optional): the party's two ChaCha12 streams; words [pos, pos + 48) of each become one zero share per
 *         r0 evaluation (the reference masks every product inside local_mul_vec; only the sum reaches the protocol).
 *         The caller advances both streams by 48 words.  NULL: no mask (tests).
 * Edges whose q_arith is zero contribute zero, which is what the reference's can_skip filter leaves out.
 * Shamir parties call this with CS_PLAIN on their degree-t shares: public terms enter every party's share, products
 * are local, so h_r0 is a degree-2t sharing (degree_reduce next) and h_r1 a degree-t sharing. */
int cs_sumcheck_arith_round(cs_ctx* ctx, cs_curve curve, cs_share_kind kind, int party, const cs_honk_arith_polys* d_polys,
                            size_t round_size, const uint64_t* d_beta_products, size_t periodicity, const cs_rep3_prf* prf,
                            uint64_t* h_r0, uint64_t* h_r1);

#ifdef __cplusplus
}
#endif
#endif /* COSNARKS_GPU_H */
