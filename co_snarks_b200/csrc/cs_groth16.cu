// Groth16 prover hot path: device-resident proving key, CircomReduction witness map, the five MSMs
// and the proof assembly.
//
// Mirrors co-circom/co-groth16/src/groth16.rs:125-338 (prove_inner, calculate_coeff,
// create_proof_with_assignment) and groth16/reduction.rs:77-193 (CircomReduction) for the Plain and
// Rep3 drivers (mpc/plain.rs, mpc/rep3.rs).  Everything between the witness upload and the five MSM
// results stays in HBM; only points come back.  Single-point work (scalar_mul_public_point_hs,
// add_assign_points_public_hs, the public-input MSM over query[1..=pub], the final sums) runs on
// the host while the GPU works -- it is latency-only in the reference too (SURVEY.md 8a, a12).
#include <functional>
#include "cs_lib.cuh"
#include "cs_net.h"

using namespace cs;

struct cs_groth16_pk {
  int curve = 0;
  size_t nc = 0, ni = 0, nw = 0, n = 0;
  unsigned log_n = 0;
  DevBuf a_rowptr, a_col, a_coeff, b_rowptr, b_col, b_coeff;
  cs_bases *a_query = nullptr, *b_g1 = nullptr, *b_g2 = nullptr, *l_query = nullptr, *h_query = nullptr;
  std::vector<uint64_t> alpha_g1, beta_g1, beta_g2, delta_g1, delta_g2;
  std::vector<uint64_t> a_head, b1_head, b2_head;  // query[0..ni] host copies
  cs_domain* dom = nullptr;
  DevBuf coset_tab;  // shift^bitrev(p) / n
  DevBuf d_pub, d_wit, d_a, d_b, d_c, d_m1, d_m2;
  // LibSnarkReduction (reduction.rs:241-342): C matrix, arkworks domain, coset = GENERATOR
  DevBuf c_rowptr, c_col, c_coeff;
  bool have_c = false;
  bool share_b_sort = false;  // B1 and B2 sort identically (same infinity pattern): B2 reuses B1's sorted entries
  cs_domain* dom_ark = nullptr;
  DevBuf coset_tab_ark, ginv_pows, vinv_over_n;
};

namespace {

// ---- host-side point helpers on raw limb buffers (Montgomery affine) --------------------------
template <class Cfg, int G>
struct HostGroup {
  typedef typename GroupOf<Cfg, G>::HF HF;
  typedef host::HXyzz<HF> X;
  typedef host::HAffine<HF> A;
  typedef host::HFp<typename Cfg::FrP> HR;
  static X load(const uint64_t* p) {
    A a;
    memcpy(&a, p, sizeof(a));
    return X::from_affine(a);
  }
  static void store(uint64_t* out, const X& x) {
    A a = host::haffine(x);
    memcpy(out, &a, sizeof(a));
  }
  // scalar in Montgomery form
  static X mul(const X& p, const uint64_t* s_mont) {
    HR s;
    memcpy(s.l, s_mont, sizeof(s.l));
    HR c = s.from_mont();
    return host::hmul(p, c.l, HR::N);
  }
};

template <class Cfg>
int build_coset_table(cs_ctx* ctx, cs_groth16_pk* pk) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HF;
  uint64_t gen[HF::N], shift[HF::N];
  CS_TRY(cs_groth16_roots_of_unity((cs_curve)pk->curve, pk->log_n, gen, shift));
  CS_TRY(cs_domain_create(ctx, (cs_curve)pk->curve, pk->log_n, gen, &pk->dom));
  if (pk->log_n == 0) return 0;
  HF s;
  memcpy(s.l, shift, sizeof(s.l));
  std::vector<HF> pw(33);
  for (int j = 0; j < 32; j++) {
    pw[j] = s;
    s = s.sqr();
  }
  pw[32] = HF::from_u64(pk->n).inverse();  // scale = 1/n
  DevBuf dpw;
  CS_TRY(dpw.reserve(pw.size() * sizeof(HF)));
  CS_CUDA(cudaMemcpyAsync(dpw.p, pw.data(), pw.size() * sizeof(HF), cudaMemcpyHostToDevice, ctx->stream));
  CS_TRY(pk->coset_tab.reserve(pk->n * sizeof(HF)));
  CS_LAUNCH(k_ntt_coset_table<FrP>, ceil_div(pk->n, 256), 256, 0, ctx->stream, dpw.as<uint32_t>(),
            dpw.as<uint32_t>() + 32 * FrP::N, pk->log_n, pk->coset_tab.as<uint32_t>());
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  dpw.release();
  return 0;
}

int upload(cs_ctx* ctx, DevBuf& buf, const void* src, size_t bytes) {
  CS_TRY(buf.reserve(bytes ? bytes : 4));
  if (bytes) CS_CUDA(cudaMemcpyAsync(buf.p, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return 0;
}

// CircomReduction::witness_map_from_matrices on the device.  Leaves h (n half shares) in pk->d_c.
// d_pub / d_wit must already hold the inputs; masks (Rep3) in d_m1 / d_m2 or null.
template <class Cfg>
int witness_map_device(cs_ctx* ctx, cs_groth16_pk* pk, int kind, int party, const uint32_t* d_wit, bool have_m1,
                       bool have_m2, cudaStream_t st) {
  typedef typename Cfg::FrP FrP;
  const unsigned batch = kind == CS_REP3 ? 2 : 1;
  const int pub_comp = kind == CS_REP3 ? (party == 0 ? 0 : (party == 1 ? 1 : -1)) : 0;
  const uint32_t n = (uint32_t)pk->n;
  CS_TRY(pk->d_a.reserve((size_t)n * batch * 32));
  CS_TRY(pk->d_b.reserve((size_t)n * batch * 32));
  CS_TRY(pk->d_c.reserve((size_t)n * 32));
  // a = A w (+ promoted public rows, reduction.rs:104-113), b = B w   (evaluate_constraint)
  CS_SPAN("witness map from matrices");
  {
  CS_SPAN("evaluate constraints + coset table computation");
  CS_LAUNCH(k_spmv<FrP>, ceil_div(n, 128), 128, 0, st, pk->a_rowptr.as<uint32_t>(), pk->a_col.as<uint32_t>(),
            pk->a_coeff.as<uint32_t>(), pk->d_pub.as<uint32_t>(), (uint32_t)pk->ni, d_wit, batch, batch,
            pub_comp, (uint32_t)pk->nc, (uint32_t)pk->ni, n, pk->d_a.as<uint32_t>());
  CS_LAUNCH(k_spmv<FrP>, ceil_div(n, 128), 128, 0, st, pk->b_rowptr.as<uint32_t>(), pk->b_col.as<uint32_t>(),
            pk->b_coeff.as<uint32_t>(), pk->d_pub.as<uint32_t>(), (uint32_t)pk->ni, d_wit, batch, batch,
            pub_comp, (uint32_t)pk->nc, 0u, n, pk->d_b.as<uint32_t>());
  }
  unsigned blocks = ceil_div(n, 256);
  if (blocks > CS_NUM_SMS * 16) blocks = CS_NUM_SMS * 16;
  // c = local_mul_vec(a, b)   (reduction.rs:160)
  CS_SPAN("c: local_mul_vec / a, b, c: distribute powers (fft/ifft)");
  if (kind == CS_REP3)
    CS_LAUNCH(k_rep3_local_mul<FrP>, blocks, 256, 0, st, pk->d_a.as<uint32_t>(), pk->d_b.as<uint32_t>(),
              have_m1 ? pk->d_m1.as<uint32_t>() : (const uint32_t*)nullptr, (const uint32_t*)nullptr,
              pk->d_c.as<uint32_t>(), (size_t)n);
  else
    CS_LAUNCH(k_plain_mul_sub<FrP>, blocks, 256, 0, st, pk->d_a.as<uint32_t>(), pk->d_b.as<uint32_t>(),
              (const uint32_t*)nullptr, pk->d_c.as<uint32_t>(), (size_t)n);
  // each of a, b, c: ifft_in_to_out -> * coset table -> fft_out_to_in   (reduction.rs:135-178);
  // the table multiply and the 1/n are fused into the last iNTT pass.
  const uint32_t* post = pk->log_n ? pk->coset_tab.as<uint32_t>() : nullptr;
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_a.as<uint32_t>(), batch, true, post, st));
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_a.as<uint32_t>(), batch, false, nullptr, st));
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_b.as<uint32_t>(), batch, true, post, st));
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_b.as<uint32_t>(), batch, false, nullptr, st));
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_c.as<uint32_t>(), 1, true, post, st));
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_c.as<uint32_t>(), 1, false, nullptr, st));
  // h = local_mul_vec(a', b') - c'   (reduction.rs:182-190), in place over c
  CS_SPAN("ab: local_mul_vec + compute ab");
  if (kind == CS_REP3)
    CS_LAUNCH(k_rep3_local_mul<FrP>, blocks, 256, 0, st, pk->d_a.as<uint32_t>(), pk->d_b.as<uint32_t>(),
              have_m2 ? pk->d_m2.as<uint32_t>() : (const uint32_t*)nullptr, pk->d_c.as<uint32_t>(),
              pk->d_c.as<uint32_t>(), (size_t)n);
  else
    CS_LAUNCH(k_plain_mul_sub<FrP>, blocks, 256, 0, st, pk->d_a.as<uint32_t>(), pk->d_b.as<uint32_t>(),
              pk->d_c.as<uint32_t>(), pk->d_c.as<uint32_t>(), (size_t)n);
  CS_CUDA(cudaGetLastError());
  return 0;
}

// Lazily builds what LibSnarkReduction needs: Domain::new (arkworks generator), the bit-reversed coset
// table GENERATOR^rev(p) / n, the natural-order powers GENERATOR^-i and the constant (g^n - 1)^-1 / n.
template <class Cfg>
int ensure_libsnark(cs_ctx* ctx, cs_groth16_pk* pk) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HF;
  if (pk->dom_ark) return 0;
  if (!pk->have_c) return fail(CS_ERR_STATE, "LibSnarkReduction needs the C matrix (cs_groth16_key_desc.c_*)");
  CS_TRY(cs_domain_create(ctx, (cs_curve)pk->curve, pk->log_n, nullptr, &pk->dom_ark));
  const size_t n = pk->n;
  HF g = HF::from_u64(std::is_same<Cfg, Bn254Cfg>::value ? 5 : 7);  // F::GENERATOR
  HF ginv = g.inverse();
  HF ninv = HF::from_u64(n).inverse();
  uint64_t e[HF::N] = {0};
  e[0] = n;
  HF vinv = (g.pow(e, HF::N) - HF::one()).inverse();  // vanishing polynomial over the coset, inverted
  HF c = vinv * ninv;
  std::vector<HF> pw(32 + 1 + 32);
  HF a = g, b = ginv;
  for (int j = 0; j < 32; j++) { pw[j] = a; pw[33 + j] = b; a = a.sqr(); b = b.sqr(); }
  pw[32] = ninv;
  DevBuf dpw;
  CS_TRY(dpw.reserve(pw.size() * sizeof(HF)));
  CS_CUDA(cudaMemcpyAsync(dpw.p, pw.data(), pw.size() * sizeof(HF), cudaMemcpyHostToDevice, ctx->stream));
  CS_TRY(pk->coset_tab_ark.reserve(n * sizeof(HF)));
  CS_TRY(pk->ginv_pows.reserve(n * sizeof(HF)));
  CS_TRY(pk->vinv_over_n.reserve(sizeof(HF)));
  CS_CUDA(cudaMemcpyAsync(pk->vinv_over_n.p, c.l, sizeof(HF), cudaMemcpyHostToDevice, ctx->stream));
  if (pk->log_n)
    CS_LAUNCH(k_ntt_coset_table<FrP>, ceil_div(n, 256), 256, 0, ctx->stream, dpw.as<uint32_t>(), dpw.as<uint32_t>() + 32 * FrP::N,
              pk->log_n, pk->coset_tab_ark.as<uint32_t>());
  CS_LAUNCH(k_ntt_twiddles<FrP>, ceil_div(n, 256), 256, 0, ctx->stream, dpw.as<uint32_t>() + 33 * FrP::N, (uint32_t)n,
            pk->ginv_pows.as<uint32_t>());
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  dpw.release();
  return 0;
}

// LibSnarkReduction::witness_map_from_matrices on the device; h (coefficients of H, natural order) in pk->d_c.
template <class Cfg>
int witness_map_libsnark_device(cs_ctx* ctx, cs_groth16_pk* pk, int kind, int party, const uint32_t* d_wit, bool have_mask,
                                cudaStream_t st) {
  typedef typename Cfg::FrP FrP;
  CS_TRY(ensure_libsnark<Cfg>(ctx, pk));
  const unsigned batch = kind == CS_REP3 ? 2 : 1;
  const int pub_comp = kind == CS_REP3 ? (party == 0 ? 0 : (party == 1 ? 1 : -1)) : 0;
  const int pub_comp_hs = kind == CS_REP3 ? (party == 0 ? 0 : -1) : 0;
  const uint32_t n = (uint32_t)pk->n;
  CS_TRY(pk->d_a.reserve((size_t)n * batch * 32));
  CS_TRY(pk->d_b.reserve((size_t)n * batch * 32));
  CS_TRY(pk->d_c.reserve((size_t)n * 32));
  CS_LAUNCH(k_spmv<FrP>, ceil_div(n, 128), 128, 0, st, pk->a_rowptr.as<uint32_t>(), pk->a_col.as<uint32_t>(),
            pk->a_coeff.as<uint32_t>(), pk->d_pub.as<uint32_t>(), (uint32_t)pk->ni, d_wit, batch, batch, pub_comp,
            (uint32_t)pk->nc, (uint32_t)pk->ni, n, pk->d_a.as<uint32_t>());
  CS_LAUNCH(k_spmv<FrP>, ceil_div(n, 128), 128, 0, st, pk->b_rowptr.as<uint32_t>(), pk->b_col.as<uint32_t>(),
            pk->b_coeff.as<uint32_t>(), pk->d_pub.as<uint32_t>(), (uint32_t)pk->ni, d_wit, batch, batch, pub_comp,
            (uint32_t)pk->nc, 0u, n, pk->d_b.as<uint32_t>());
  // c from the C matrix as HALF shares (reduction.rs:292-298)
  CS_LAUNCH(k_spmv<FrP>, ceil_div(n, 128), 128, 0, st, pk->c_rowptr.as<uint32_t>(), pk->c_col.as<uint32_t>(),
            pk->c_coeff.as<uint32_t>(), pk->d_pub.as<uint32_t>(), (uint32_t)pk->ni, d_wit, 1u, batch, pub_comp_hs,
            (uint32_t)pk->nc, 0u, n, pk->d_c.as<uint32_t>());
  const uint32_t* post = pk->log_n ? pk->coset_tab_ark.as<uint32_t>() : nullptr;
  CS_TRY(ntt_run(ctx, pk->dom_ark, pk->d_a.as<uint32_t>(), batch, true, post, st));
  CS_TRY(ntt_run(ctx, pk->dom_ark, pk->d_a.as<uint32_t>(), batch, false, nullptr, st));
  CS_TRY(ntt_run(ctx, pk->dom_ark, pk->d_b.as<uint32_t>(), batch, true, post, st));
  CS_TRY(ntt_run(ctx, pk->dom_ark, pk->d_b.as<uint32_t>(), batch, false, nullptr, st));
  CS_TRY(ntt_run(ctx, pk->dom_ark, pk->d_c.as<uint32_t>(), 1, true, post, st));
  CS_TRY(ntt_run(ctx, pk->dom_ark, pk->d_c.as<uint32_t>(), 1, false, nullptr, st));
  unsigned blocks = ceil_div(n, 256);
  if (blocks > CS_NUM_SMS * 16) blocks = CS_NUM_SMS * 16;
  // ab = local_mul_vec(a, b) - c   (reduction.rs:289, :316-322; the constant factor is folded into the iNTT below)
  if (kind == CS_REP3)
    CS_LAUNCH(k_rep3_local_mul<FrP>, blocks, 256, 0, st, pk->d_a.as<uint32_t>(), pk->d_b.as<uint32_t>(),
              have_mask ? pk->d_m1.as<uint32_t>() : (const uint32_t*)nullptr, pk->d_c.as<uint32_t>(), pk->d_c.as<uint32_t>(),
              (size_t)n);
  else
    CS_LAUNCH(k_plain_mul_sub<FrP>, blocks, 256, 0, st, pk->d_a.as<uint32_t>(), pk->d_b.as<uint32_t>(),
              pk->d_c.as<uint32_t>(), pk->d_c.as<uint32_t>(), (size_t)n);
  // interpolate over the coset: iNTT scaled by (g^n - 1)^-1 / n, bit_reverse, times g^-i  (reduction.rs:324-339)
  if (pk->log_n) {
    CS_TRY((ntt_enqueue<FrP>(pk->d_c.as<uint32_t>(), pk->dom_ark->tw_inv.as<uint32_t>(), pk->log_n, 1, false, nullptr,
                             pk->vinv_over_n.as<uint32_t>(), st)));
    CS_LAUNCH(k_bit_reverse<FrP>, ceil_div(n, 256), 256, 0, st, pk->d_c.as<uint32_t>(), pk->log_n, 1u);
  } else {
    CS_LAUNCH(k_vec_scale_table<FrP>, 1, 32, 0, st, pk->d_c.as<uint32_t>(), pk->vinv_over_n.as<uint32_t>(), (size_t)1, 1u);
  }
  CS_LAUNCH(k_vec_scale_table<FrP>, blocks, 256, 0, st, pk->d_c.as<uint32_t>(), pk->ginv_pows.as<uint32_t>(), (size_t)n, 1u);
  CS_CUDA(cudaGetLastError());
  return 0;
}

int upload_inputs(cs_ctx* ctx, cs_groth16_pk* pk, int kind, const uint64_t* h_pub, const uint64_t* h_wit,
                  const uint64_t* h_m1, const uint64_t* h_m2) {
  const unsigned batch = kind == CS_REP3 ? 2 : 1;
  CS_TRY(upload(ctx, pk->d_pub, h_pub, pk->ni * 32));
  if (h_wit) CS_TRY(upload(ctx, pk->d_wit, h_wit, pk->nw * batch * 32));
  if (kind == CS_REP3 && h_m1) CS_TRY(upload(ctx, pk->d_m1, h_m1, pk->n * 32));
  if (kind == CS_REP3 && h_m2) CS_TRY(upload(ctx, pk->d_m2, h_m2, pk->n * 32));
  return 0;
}

// The local, GPU-heavy part shared by plain_prove and the Rep3 party: witness map + five MSMs.
// r_hs / s_hs: half shares (Montgomery Fr) of r and s.  add_public: plain driver or Rep3 party 0
// (add_assign_points_public_hs, mpc/rep3.rs:108-118).  Outputs are affine Montgomery points.
template <class Cfg>
int local_phase(cs_ctx* ctx, cs_groth16_pk* pk, int kind, int party, const uint64_t* h_pub, const uint64_t* h_wit,
                const uint64_t* d_wit_in, const uint64_t* h_m1, const uint64_t* h_m2, const uint64_t* r_hs, const uint64_t* s_hs,
                uint64_t* out_a, uint64_t* out_b1, uint64_t* out_b2, uint64_t* out_l, uint64_t* out_h,
                unsigned parts = CS_PART_ALL, const cs_rep3_prf* prf = nullptr, const uint64_t* rs_mont = nullptr,
                uint64_t* out_rs_delta = nullptr, const std::function<void()>* overlap = nullptr,
                const std::function<int(const uint64_t*, const uint64_t*)>* mid = nullptr) {
  typedef HostGroup<Cfg, 0> H1;
  typedef HostGroup<Cfg, 1> H2;
  const unsigned batch = kind == CS_REP3 ? 2 : 1;
  const bool add_public = (kind == CS_PLAIN) || party == 0;
  const bool have_aux = pk->nw > 0;
  const bool do_a = parts & CS_PART_A, do_b1 = parts & CS_PART_B1, do_b2 = parts & CS_PART_B2,
             do_l = parts & CS_PART_L, do_h = parts & CS_PART_H;
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_TRY(upload_inputs(ctx, pk, kind, h_pub, h_wit, do_h ? h_m1 : nullptr, do_h ? h_m2 : nullptr));
  // fork: A, B1, B2, L need only the witness.  The witness map -> H chain is the longest dependency chain of the proof
  // (6-10 NTTs, then a full MSM), so it is enqueued FIRST and on the highest-priority stream: its passes interleave
  // with the other MSMs' accumulation grids instead of queueing behind all of them (otherwise H starts only after the
  // four side MSMs have drained).
  CS_TRY(ctx_fork(ctx, 4));
  cudaStream_t wm = ctx->wm;
  CS_CUDA(cudaStreamWaitEvent(wm, ctx->ev_fork, 0));
  // witness either uploaded from the host just above, or already resident in HBM (d_wit_in)
  const uint32_t* wit = d_wit_in ? reinterpret_cast<const uint32_t*>(d_wit_in) : pk->d_wit.as<uint32_t>();
  if (do_h) {
    bool have_m1 = h_m1 != nullptr, have_m2 = h_m2 != nullptr;
    if (prf && kind == CS_REP3) {
      // masks drawn on the device from the party's two ChaCha streams (rngs.rs:137-156); the second
      // vector continues 8 n words further, exactly as two consecutive fill_bytes calls would
      typedef typename Cfg::FrP FrP;
      const size_t n = pk->n;
      CS_TRY(pk->d_m1.reserve(n * 32));
      CS_TRY(pk->d_m2.reserve(n * 32));
      CS_TRY(ctx->prf_keys.reserve(64));
      CS_CUDA(cudaMemcpyAsync(ctx->prf_keys.p, prf->seed1, 32, cudaMemcpyHostToDevice, wm));
      CS_CUDA(cudaMemcpyAsync((char*)ctx->prf_keys.p + 32, prf->seed2, 32, cudaMemcpyHostToDevice, wm));
      CS_LAUNCH(k_rep3_masks<FrP>, ceil_div(n, 128), 128, 0, wm, ctx->prf_keys.as<uint32_t>(), prf->word_pos1,
                prf->word_pos2, prf->rounds, n, pk->d_m1.as<uint32_t>());
      CS_LAUNCH(k_rep3_masks<FrP>, ceil_div(n, 128), 128, 0, wm, ctx->prf_keys.as<uint32_t>(),
                prf->word_pos1 + 8 * n, prf->word_pos2 + 8 * n, prf->rounds, n, pk->d_m2.as<uint32_t>());
      have_m1 = have_m2 = true;
    }
    CS_TRY((witness_map_device<Cfg>(ctx, pk, kind, party, wit, have_m1, have_m2, wm)));
    {
      CS_SPAN("msm h_query");
      CS_TRY(msm_enqueue_dyn(ctx, 4, wm, pk->h_query, 0, pk->d_c.as<uint32_t>(), 1, pk->n, 1));
    }
  }
  if (have_aux) {
    // query[1 + pub_len ..] = query[ni ..]  (groth16.rs:193)
    CS_SPAN("compute A, B/G1, B/G2 in create proof with assignment + msm l_query");
    if (do_a) CS_TRY(msm_enqueue_dyn(ctx, 0, ctx->side[0], pk->a_query, pk->ni, wit, batch, pk->nw, 1));
    if (do_b1) CS_TRY(msm_enqueue_dyn(ctx, 1, ctx->side[1], pk->b_g1, pk->ni, wit, batch, pk->nw, 1));
    if (do_b2)
      CS_TRY(msm_enqueue_dyn(ctx, 2, ctx->side[2], pk->b_g2, pk->ni, wit, batch, pk->nw, 1,
                             (do_b1 && pk->share_b_sort) ? 1 : -1));
    if (do_l) CS_TRY(msm_enqueue_dyn(ctx, 3, ctx->side[3], pk->l_query, 0, wit, batch, pk->nw, 1));
  }
  CS_TRY(ctx_join(ctx, 4));
  CS_CUDA(cudaEventRecord(ctx->ev_wm, wm));
  CS_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_wm, 0));

  // ---- host work overlapped with the GPU: scalar_mul_public_point_hs + public parts (groth16.rs:232-276)
  const size_t g1l = 2 * H1::HF::N, g2l = 4 * H1::HF::N;
  typename H1::X a_acc = H1::X::inf(), b1_acc = H1::X::inf();
  typename H2::X b2_acc = H2::X::inf();
  if (do_a) {
    a_acc = H1::mul(H1::load(pk->delta_g1.data()), r_hs);
    if (add_public) {
      a_acc = host::hadd(a_acc, H1::load(pk->a_head.data()));
      a_acc = host::hadd(a_acc, H1::load(pk->alpha_g1.data()));
      // msm_unchecked(&query[1..=pub_len], input_assignment) with input_assignment = public_inputs[1..]
      for (size_t k = 1; k < pk->ni; k++)
        a_acc = host::hadd(a_acc, H1::mul(H1::load(pk->a_head.data() + k * g1l), h_pub + k * 4));
    }
  }
  if (do_b1) {
    b1_acc = H1::mul(H1::load(pk->delta_g1.data()), s_hs);
    if (add_public) {
      b1_acc = host::hadd(b1_acc, H1::load(pk->b1_head.data()));
      b1_acc = host::hadd(b1_acc, H1::load(pk->beta_g1.data()));
      for (size_t k = 1; k < pk->ni; k++)
        b1_acc = host::hadd(b1_acc, H1::mul(H1::load(pk->b1_head.data() + k * g1l), h_pub + k * 4));
    }
  }
  if (do_b2) {
    b2_acc = H2::mul(H2::load(pk->delta_g2.data()), s_hs);
    if (add_public) {
      b2_acc = host::hadd(b2_acc, H2::load(pk->b2_head.data()));
      b2_acc = host::hadd(b2_acc, H2::load(pk->beta_g2.data()));
      for (size_t k = 1; k < pk->ni; k++)
        b2_acc = host::hadd(b2_acc, H2::mul(H2::load(pk->b2_head.data() + k * g2l), h_pub + k * 4));
    }
  }
  CS_SPAN("r*s without networking");
  if (rs_mont && out_rs_delta)  // (r s) * delta_1 (groth16.rs:297-298), also while the GPU is busy
    H1::store(out_rs_delta, H1::mul(H1::load(pk->delta_g1.data()), rs_mont));
  if (overlap) (*overlap)();  // caller's single-point work that does not depend on the MSM results
  uint64_t tmp[24];
  int inf = 0;
  // A and B1 run on side streams that started before the witness map and finish well before H: the caller's work
  // that needs only those two (the first network round, s*A and r*B1) is done while the GPU still computes L, B2, H
  bool ab_done = false;
  if (mid && have_aux && do_a && do_b1) {
    CS_CUDA(cudaEventSynchronize(ctx->ev_side[0]));
    CS_CUDA(cudaEventSynchronize(ctx->ev_side[1]));
    CS_TRY(msm_finish_dyn(ctx, 0, pk->a_query, tmp, &inf)); a_acc = host::hadd(a_acc, H1::load(tmp));
    CS_TRY(msm_finish_dyn(ctx, 1, pk->b_g1, tmp, &inf)); b1_acc = host::hadd(b1_acc, H1::load(tmp));
    H1::store(out_a, a_acc);
    H1::store(out_b1, b1_acc);
    CS_TRY((*mid)(out_a, out_b1));
    ab_done = true;
  }
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  memset(out_l, 0, g1l * 8);
  memset(out_h, 0, g1l * 8);
  if (have_aux) {
    if (do_a && !ab_done) { CS_TRY(msm_finish_dyn(ctx, 0, pk->a_query, tmp, &inf)); a_acc = host::hadd(a_acc, H1::load(tmp)); }
    if (do_b1 && !ab_done) { CS_TRY(msm_finish_dyn(ctx, 1, pk->b_g1, tmp, &inf)); b1_acc = host::hadd(b1_acc, H1::load(tmp)); }
    if (do_b2) { CS_TRY(msm_finish_dyn(ctx, 2, pk->b_g2, tmp, &inf)); b2_acc = host::hadd(b2_acc, H2::load(tmp)); }
    if (do_l) CS_TRY(msm_finish_dyn(ctx, 3, pk->l_query, out_l, &inf));
  }
  if (do_h) CS_TRY(msm_finish_dyn(ctx, 4, pk->h_query, out_h, &inf));
  if (!ab_done) {
    H1::store(out_a, a_acc);
    H1::store(out_b1, b1_acc);
  }
  H2::store(out_b2, b2_acc);
  if (mid && !ab_done) CS_TRY((*mid)(out_a, out_b1));  // no early window (empty witness): same call, after the fact
  return 0;
}

template <class Cfg>
int prove_plain_t(cs_ctx* ctx, cs_groth16_pk* pk, const uint64_t* h_pub, const uint64_t* h_wit,
                  const uint64_t* d_wit, const uint64_t* r, const uint64_t* s, uint64_t* out_a, uint64_t* out_b,
                  uint64_t* out_c) {
  typedef HostGroup<Cfg, 0> H1;
  typedef host::HFp<typename Cfg::FrP> HR;
  uint64_t a[12], b1[12], l[12], h[12], rsd[12];
  HR rr, ss;
  memcpy(rr.l, r, sizeof(rr.l));
  memcpy(ss.l, s, sizeof(ss.l));
  HR rs = rr * ss;
  // groth16.rs:296-322 with the plain driver: C = s*A + r*B1 - (r s)*delta1 + L + H; the two scalar
  // multiplications run on the host as soon as A and B1 are there, while the GPU finishes L, B2 and H
  typename H1::X c = H1::X::inf();
  std::function<int(const uint64_t*, const uint64_t*)> mid = [&](const uint64_t* pa, const uint64_t* pb1) -> int {
    c = host::hadd(H1::mul(H1::load(pa), s), H1::mul(H1::load(pb1), r));
    return 0;
  };
  CS_TRY((local_phase<Cfg>(ctx, pk, CS_PLAIN, 0, h_pub, h_wit, d_wit, nullptr, nullptr, r, s, a, b1, out_b, l, h,
                           CS_PART_ALL, nullptr, rs.l, rsd, nullptr, &mid)));
  c = host::hadd(c, host::hneg(H1::load(rsd)));
  c = host::hadd(c, H1::load(l));
  c = host::hadd(c, H1::load(h));
  memcpy(out_a, a, 2 * H1::HF::N * 8);
  H1::store(out_c, c);
  return 0;
}


// Rep3CoGroth16::prove for one party (groth16.rs:360-379, prove_inner :125-177, create_proof_with_assignment
// :207-338 with Rep3Groth16Driver, mpc/rep3.rs).  role: 0 = the whole party on one GPU, 1 = the party's
// protocol GPU ({A, B1, L} + both network legs; receives g2_b and h_acc from the helper over `pair`),
// 2 = the helper GPU ({witness map -> H, B2}).
template <class Cfg>
int rep3_prove_t(cs_ctx* ctx, cs_groth16_pk* pk, cs_net* net0, cs_net* net1, cs_net* pair, int role, int party,
                 cs_rep3_state* state0, const uint64_t* h_pub, const uint64_t* h_wit, const uint64_t* d_wit,
                 uint64_t* out_a, uint64_t* out_b, uint64_t* out_c, uint64_t* out_rs) {
  typedef HostGroup<Cfg, 0> H1;
  typedef HostGroup<Cfg, 1> H2;
  typedef host::HFp<typename Cfg::FrP> HR;
  typedef typename Cfg::FrP FrP;
  constexpr size_t G1L = 2 * H1::HF::N, G2L = 4 * H1::HF::N;  // 64-bit limbs of an affine point
  const size_t n = pk->n;
  // state1 = state0.fork(0) (groth16.rs:368): the scalar_mul leg draws its EC mask from the fork
  cs_rep3_state* st1p = nullptr;
  CS_TRY(cs_rep3_state_fork(state0, &st1p));
  std::unique_ptr<cs_rep3_state> state1(st1p);
  // ---- correlated randomness in the order the reference consumes it
  // two n-element mask vectors of the witness map (reduction.rs:160,182): drawn on the device from
  // (seed, word position); the streams move past the 2 x 8n words
  cs_rep3_prf prf;
  CS_TRY(cs_rep3_state_prf(state0, &prf));
  CS_TRY(cs_rep3_state_advance(state0, 16 * (uint64_t)n));
  uint64_t r_sh[2 * HR::N], s_sh[2 * HR::N];  // T::rand x2 (groth16.rs:157)
  CS_TRY(cs_rep3_state_rand(state0, (cs_curve)pk->curve, r_sh));
  CS_TRY(cs_rep3_state_rand(state0, (cs_curve)pk->curve, s_sh));
  if (out_rs) { memcpy(out_rs, r_sh, sizeof(r_sh)); memcpy(out_rs + 2 * HR::N, s_sh, sizeof(s_sh)); }
  // rs = local_mul_vec([r], [s]) (groth16.rs:297): r.a s.a + r.a s.b + r.b s.a + (F(rng1) - F(rng2))
  HR ra, rb, sa, sb;
  memcpy(ra.l, r_sh, sizeof(ra.l)); memcpy(rb.l, r_sh + HR::N, sizeof(rb.l));
  memcpy(sa.l, s_sh, sizeof(sa.l)); memcpy(sb.l, s_sh + HR::N, sizeof(sb.l));
  HR m1 = state0->rng1.template fr_be_mod_order<FrP>(), m2 = state0->rng2.template fr_be_mod_order<FrP>();
  HR rs = ra * (sa + sb) + rb * sa + (m1 - m2);
  // EC mask of scalar_mul_local (pointshare.rs:119-125, rngs.rs:177-186): C::rand(rng1) - C::rand(rng2), realised
  // as k1 P - k2 P with k_i = F::rand(rng_i) and P = alpha_1 of the key, a public generator of the prime-order
  // group, so k P is uniform (arkworks samples curve points by x-coordinate; the three parties' masks cancel
  // either way)
  uint64_t k1[HR::N], k2[HR::N];
  state1->rng1.template fr_rand<FrP>(k1, Cfg::FR_BITS);
  state1->rng2.template fr_rand<FrP>(k2, Cfg::FR_BITS);
  if (role == 2) {
    // helper GPU: {witness map -> H, B2}; same draws as the main GPU (lock-step), results over the pair link
    uint64_t a[G1L], b1[G1L], b2[G2L], l[G1L], h[G1L];
    CS_TRY((local_phase<Cfg>(ctx, pk, CS_REP3, party, h_pub, h_wit, d_wit, nullptr, nullptr, r_sh, s_sh, a, b1, b2, l, h,
                             CS_PART_B2 | CS_PART_H, &prf)));
    uint64_t msg[G2L + G1L];
    memcpy(msg, b2, G2L * 8);
    memcpy(msg + G2L, h, G1L * 8);
    return cs_net_send(pair, 0, msg, sizeof(msg));
  }
  typename H1::X ec_mask = H1::X::inf();
  std::function<void()> overlap = [&]() {
    typename H1::X g = H1::load(pk->alpha_g1.data());
    HR a1, a2;
    memcpy(a1.l, k1, sizeof(a1.l)); memcpy(a2.l, k2, sizeof(a2.l));
    HR d = a1 - a2;  // (k1 - k2) G: one scalar multiplication instead of two
    HR dc = d.from_mont();
    ec_mask = host::hmul(g, dc.l, HR::N);
  };
  uint64_t g_a[G1L], g1_b[G1L], g2_b[G2L], l_acc[G1L], h_acc[G1L], rsd[G1L];
  const unsigned parts = role == 1 ? (CS_PART_A | CS_PART_B1 | CS_PART_L) : CS_PART_ALL;
  Rep3Net n0(net0), n1(net1);
  typename H1::X A_open = H1::X::inf(), g_c = H1::X::inf();
  // ---- network round 1 (groth16.rs:305-308): open_half_point(g_a) on net0 | scalar_mul(g1_b, r) on net1, run as soon
  // as THIS party's A and B1 are there -- the GPU is still busy with L, B2 and H, so the round trip and the three
  // scalar multiplications that follow it are off the critical path.  All sends first (they do not block).
  std::function<int(const uint64_t*, const uint64_t*)> mid = [&](const uint64_t* pa, const uint64_t* pb1) -> int {
    CS_SPAN("network round after calc coeff");
    CS_TRY(n0.send_next(pa, G1L * 8));
    CS_TRY(n0.send_prev(pa, G1L * 8));
    CS_TRY(n1.send_next(pb1, G1L * 8));
    // what can be done before the answers arrive: rhs.a * self.b
    typename H1::X B1 = H1::load(pb1);
    typename H1::X t = H1::mul(B1, r_sh + HR::N);
    uint64_t ga_prev[G1L], ga_next[G1L], g1b_prev[G1L];
    CS_TRY(n0.recv_prev(ga_prev, G1L * 8));
    CS_TRY(n0.recv_next(ga_next, G1L * 8));
    CS_TRY(n1.recv_prev(g1b_prev, G1L * 8));
    A_open = host::hadd(host::hadd(H1::load(pa), H1::load(ga_prev)), H1::load(ga_next));
    // scalar_mul_local: b * point + mask, (a, b) * (pa, pb) = pa b.a + pb b.a + pa b.b  (rep3 share product)
    typename H1::X r_g1_b = host::hadd(host::hadd(H1::mul(host::hadd(B1, H1::load(g1b_prev)), r_sh), t), ec_mask);
    g_c = host::hadd(H1::mul(A_open, s_sh), r_g1_b);  // groth16.rs:314-317
    return 0;
  };
  CS_TRY((local_phase<Cfg>(ctx, pk, CS_REP3, party, h_pub, h_wit, d_wit, nullptr, nullptr, r_sh, s_sh, g_a, g1_b, g2_b,
                           l_acc, h_acc, parts, role == 1 ? nullptr : &prf, rs.l, rsd, &overlap, &mid)));
  if (role == 1) {
    uint64_t msg[G2L + G1L];
    CS_TRY(cs_net_recv(pair, 1, msg, sizeof(msg)));
    memcpy(g2_b, msg, G2L * 8);
    memcpy(h_acc, msg + G2L, G1L * 8);
  }
  CS_SPAN("finish - open two points and some adds");
  // ---- groth16.rs:318-322
  g_c = host::hadd(g_c, host::hneg(H1::load(rsd)));
  g_c = host::hadd(g_c, H1::load(l_acc));
  g_c = host::hadd(g_c, H1::load(h_acc));
  uint64_t gc[G1L];
  H1::store(gc, g_c);
  // ---- network round 2 (groth16.rs:325-328): open_half_point(g_c) on net0 | open_half_point(g2_b) on net1
  CS_TRY(n0.send_next(gc, G1L * 8));
  CS_TRY(n0.send_prev(gc, G1L * 8));
  CS_TRY(n1.send_next(g2_b, G2L * 8));
  CS_TRY(n1.send_prev(g2_b, G2L * 8));
  uint64_t gc_prev[G1L], gc_next[G1L], b2_prev[G2L], b2_next[G2L];
  CS_TRY(n0.recv_prev(gc_prev, G1L * 8));
  CS_TRY(n0.recv_next(gc_next, G1L * 8));
  CS_TRY(n1.recv_prev(b2_prev, G2L * 8));
  CS_TRY(n1.recv_next(b2_next, G2L * 8));
  H1::store(out_a, A_open);
  H1::store(out_c, host::hadd(host::hadd(g_c, H1::load(gc_prev)), H1::load(gc_next)));
  H2::store(out_b, host::hadd(host::hadd(H2::load(g2_b), H2::load(b2_prev)), H2::load(b2_next)));
  return 0;
}

// ShamirCoGroth16::prove (groth16.rs:439-463): preprocessing of three pairs over net0, state1 = state0.fork(1),
// then prove_inner / create_proof_with_assignment with ShamirGroth16Driver (mpc/shamir.rs).
template <class Cfg>
int shamir_prove_t(cs_ctx* ctx, cs_groth16_pk* pk, cs_net* net0, cs_net* net1, int n_parties, int threshold,
                   const uint64_t* h_pub, const uint64_t* h_wit, const uint64_t* d_wit, uint64_t* out_a, uint64_t* out_b,
                   uint64_t* out_c, uint64_t* out_rs) {
  typedef HostGroup<Cfg, 0> H1;
  typedef host::HFp<typename Cfg::FrP> HR;
  constexpr size_t G1L = 2 * H1::HF::N, G2L = 4 * H1::HF::N;
  // we need 3 corr rand pairs: 2 for the two rand calls, 1 for scalar_mul (groth16.rs:448-452)
  cs_shamir_state* s0 = nullptr;
  CS_TRY(cs_shamir_state_create(net0, (cs_curve)pk->curve, n_parties, threshold, 3, &s0));
  struct Guard { cs_shamir_state* a = nullptr; cs_shamir_state* b = nullptr; ~Guard() { cs_shamir_state_free(a); cs_shamir_state_free(b); } } guard;
  guard.a = s0;
  cs_shamir_state* s1 = nullptr;
  CS_TRY(cs_shamir_state_fork(s0, 1, &s1));
  guard.b = s1;
  uint64_t r[HR::N], sv[HR::N];
  CS_TRY(cs_shamir_state_rand(s0, net0, r));   // groth16.rs:157
  CS_TRY(cs_shamir_state_rand(s0, net0, sv));
  if (out_rs) { memcpy(out_rs, r, sizeof(r)); memcpy(out_rs + HR::N, sv, sizeof(sv)); }
  HR rr, ss;
  memcpy(rr.l, r, sizeof(r));
  memcpy(ss.l, sv, sizeof(sv));
  HR rs = rr * ss;  // local_mul_vec([r], [s]): a degree-2t share (shamir/arithmetic.rs:73-80)
  uint64_t g_a[G1L], g1_b[G1L], g2_b[G2L], l_acc[G1L], h_acc[G1L], rsd[G1L];
  // the Shamir driver's local computation is the plain driver's on degree-t shares: every party adds the public terms
  CS_TRY((local_phase<Cfg>(ctx, pk, CS_PLAIN, 0, h_pub, h_wit, d_wit, nullptr, nullptr, r, sv, g_a, g1_b, g2_b, l_acc, h_acc,
                           CS_PART_ALL, nullptr, rs.l, rsd)));
  // round 1 (groth16.rs:305-308): open_half_point(g_a) on net0 | scalar_mul(g1_b, r) on net1 with state1
  uint64_t a_open[G1L], g1_b_red[G1L];
  CS_TRY(cs_shamir_open_half_point(s0, net0, CS_G1, g_a, a_open));
  CS_TRY(cs_shamir_degree_reduce_point(s1, net1, CS_G1, pk->alpha_g1.data(), g1_b, g1_b_red));  // mpc/shamir.rs:146-148
  typename H1::X r_g1_b = H1::mul(H1::load(g1_b_red), r);                                      // scalar_mul_local
  typename H1::X g_c = H1::mul(H1::load(a_open), sv);
  g_c = host::hadd(g_c, r_g1_b);
  g_c = host::hadd(g_c, host::hneg(H1::load(rsd)));
  g_c = host::hadd(g_c, H1::load(l_acc));
  g_c = host::hadd(g_c, H1::load(h_acc));
  uint64_t gc[G1L];
  H1::store(gc, g_c);
  // round 2 (groth16.rs:325-328)
  CS_TRY(cs_shamir_open_half_point(s0, net0, CS_G1, gc, out_c));
  CS_TRY(cs_shamir_open_half_point(s1, net1, CS_G2, g2_b, out_b));
  memcpy(out_a, a_open, sizeof(a_open));
  return 0;
}

int rep3_prove_dispatch(cs_ctx* ctx, cs_groth16_pk* pk, cs_net* net0, cs_net* net1, cs_net* pair, int role, int party,
                        cs_rep3_state* state, const uint64_t* h_pub, const uint64_t* h_wit, const uint64_t* d_wit,
                        uint64_t* out_a, uint64_t* out_b, uint64_t* out_c, uint64_t* out_rs) {
  if (!ctx || !pk || !state || !h_pub) return fail(CS_ERR_ARG, "cs_groth16_rep3_prove: NULL argument");
  if (pk->nw && !h_wit == !d_wit) return fail(CS_ERR_ARG, "cs_groth16_rep3_prove: pass the witness shares either on the host or on the device");
  if (role != 2) {
    if (!net0 || !net1 || !out_a || !out_b || !out_c) return fail(CS_ERR_ARG, "cs_groth16_rep3_prove: NULL argument");
    if (net0->n != 3 || net1->n != 3 || net0->id != net1->id) return fail(CS_ERR_ARG, "cs_groth16_rep3_prove: net0/net1 must be 3-party meshes of the same party");
    if (net0->id != state->id) return fail(CS_ERR_ARG, "cs_groth16_rep3_prove: state belongs to party %d, net to party %d", state->id, net0->id);
  }
  if (role != 0 && (!pair || pair->n != 2 || pair->id != role - 1)) return fail(CS_ERR_ARG, "cs_groth16_rep3_prove: pair must be the 2-party link (id %d)", role - 1);
  if (party < 0 || party > 2) return fail(CS_ERR_ARG, "cs_groth16_rep3_prove: party must be 0..2");
  switch (pk->curve) {
    case CS_BN254:
      return rep3_prove_t<Bn254Cfg>(ctx, pk, net0, net1, pair, role, party, state, h_pub, h_wit, d_wit, out_a, out_b, out_c, out_rs);
#if defined(CS_ENABLE_BLS12_381)
    case CS_BLS12_381:
      return rep3_prove_t<Bls381Cfg>(ctx, pk, net0, net1, pair, role, party, state, h_pub, h_wit, d_wit, out_a, out_b, out_c, out_rs);
#endif
    default: return fail(CS_ERR_ARG, "unsupported curve");
  }
}

}  // namespace

extern "C" {

int cs_groth16_rep3_prove(cs_ctx* ctx, cs_groth16_pk* pk, cs_net* net0, cs_net* net1, cs_rep3_state* state,
                          const uint64_t* h_pub, const uint64_t* h_wit, const uint64_t* d_wit, uint64_t* out_a,
                          uint64_t* out_b, uint64_t* out_c, uint64_t* out_rs) {
  return rep3_prove_dispatch(ctx, pk, net0, net1, nullptr, 0, state ? state->id : 0, state, h_pub, h_wit, d_wit, out_a, out_b,
                             out_c, out_rs);
}

int cs_groth16_rep3_prove_main(cs_ctx* ctx, cs_groth16_pk* pk, cs_net* net0, cs_net* net1, cs_net* pair,
                               cs_rep3_state* state, const uint64_t* h_pub, const uint64_t* h_wit, const uint64_t* d_wit,
                               uint64_t* out_a, uint64_t* out_b, uint64_t* out_c, uint64_t* out_rs) {
  return rep3_prove_dispatch(ctx, pk, net0, net1, pair, 1, state ? state->id : 0, state, h_pub, h_wit, d_wit, out_a, out_b,
                             out_c, out_rs);
}

int cs_groth16_rep3_prove_helper(cs_ctx* ctx, cs_groth16_pk* pk, int party, cs_net* pair, cs_rep3_state* state,
                                 const uint64_t* h_pub, const uint64_t* h_wit, const uint64_t* d_wit) {
  if (state && state->id != party) return fail(CS_ERR_ARG, "cs_groth16_rep3_prove_helper: state belongs to party %d", state->id);
  return rep3_prove_dispatch(ctx, pk, nullptr, nullptr, pair, 2, party, state, h_pub, h_wit, d_wit, nullptr, nullptr, nullptr,
                             nullptr);
}

int cs_groth16_pk_create(cs_ctx* ctx, const cs_groth16_key_desc* d, cs_groth16_pk** out) {
  if (!ctx || !d || !out) return fail(CS_ERR_ARG, "cs_groth16_pk_create: NULL argument");
  if (d->curve != CS_BN254
#if defined(CS_ENABLE_BLS12_381)
      && d->curve != CS_BLS12_381
#endif
  )
    return fail(CS_ERR_ARG, "cs_groth16_pk_create: unsupported curve %d", (int)d->curve);
  const size_t nc = d->num_constraints, ni = d->num_instance_variables, nw = d->num_witness_variables;
  if (ni == 0) return fail(CS_ERR_ARG, "cs_groth16_pk_create: num_instance_variables must be >= 1");
  // lengths the prover indexes (groth16.rs:190-200, 283, 290)
  if (d->a_query_len != ni + nw || d->b_g1_query_len != ni + nw || d->b_g2_query_len != ni + nw)
    return fail(CS_ERR_ARG, "cs_groth16_pk_create: a/b query length must be %zu", ni + nw);
  if (d->l_query_len != nw) return fail(CS_ERR_ARG, "cs_groth16_pk_create: l_query length must be %zu", nw);
  CS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<cs_groth16_pk> pk(new cs_groth16_pk());
  pk->curve = d->curve;
  pk->nc = nc; pk->ni = ni; pk->nw = nw;
  size_t n = 1;
  unsigned lg = 0;
  while (n < nc + ni) { n <<= 1; lg++; }  // next_power_of_two (reduction.rs:85)
  pk->n = n;
  pk->log_n = lg;
  if (d->h_query_len < n) return fail(CS_ERR_ARG, "cs_groth16_pk_create: h_query has %zu points, domain needs %zu", d->h_query_len, n);
  const unsigned max_adicity = d->curve == CS_BN254 ? 28 : 32;
  if (lg > max_adicity) return fail(CS_ERR_ARG, "Polynomial Degree too large");  // reduction.rs:87-89
  const size_t fq = fq_limbs64(d->curve), g1b = 2 * fq * 8, g2b = 4 * fq * 8;
  CS_TRY(upload(ctx, pk->a_rowptr, d->a_row_ptr, (nc + 1) * 4));
  CS_TRY(upload(ctx, pk->a_col, d->a_col, d->a_nnz * 4));
  CS_TRY(upload(ctx, pk->a_coeff, d->a_coeff, d->a_nnz * 32));
  CS_TRY(upload(ctx, pk->b_rowptr, d->b_row_ptr, (nc + 1) * 4));
  CS_TRY(upload(ctx, pk->b_col, d->b_col, d->b_nnz * 4));
  CS_TRY(upload(ctx, pk->b_coeff, d->b_coeff, d->b_nnz * 32));
  if (d->c_row_ptr) {
    CS_TRY(upload(ctx, pk->c_rowptr, d->c_row_ptr, (nc + 1) * 4));
    CS_TRY(upload(ctx, pk->c_col, d->c_col, d->c_nnz * 4));
    CS_TRY(upload(ctx, pk->c_coeff, d->c_coeff, d->c_nnz * 32));
    pk->have_c = true;
  }
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  pk->alpha_g1.assign(d->alpha_g1, d->alpha_g1 + 2 * fq);
  pk->beta_g1.assign(d->beta_g1, d->beta_g1 + 2 * fq);
  pk->beta_g2.assign(d->beta_g2, d->beta_g2 + 4 * fq);
  pk->delta_g1.assign(d->delta_g1, d->delta_g1 + 2 * fq);
  pk->delta_g2.assign(d->delta_g2, d->delta_g2 + 4 * fq);
  pk->a_head.assign(d->a_query, d->a_query + ni * 2 * fq);
  pk->b1_head.assign(d->b_g1_query, d->b_g1_query + ni * 2 * fq);
  pk->b2_head.assign(d->b_g2_query, d->b_g2_query + ni * 4 * fq);
  (void)g1b; (void)g2b;
  const int wb = d->window_bits;
  CS_TRY(cs_bases_upload(ctx, d->curve, CS_G1, d->a_query, d->a_query_len, wb, &pk->a_query));
  CS_TRY(cs_bases_upload(ctx, d->curve, CS_G1, d->b_g1_query, d->b_g1_query_len, wb, &pk->b_g1));
  CS_TRY(cs_bases_upload(ctx, d->curve, CS_G2, d->b_g2_query, d->b_g2_query_len, wb, &pk->b_g2));
  if (nw) CS_TRY(cs_bases_upload(ctx, d->curve, CS_G1, d->l_query, d->l_query_len, wb, &pk->l_query));
  CS_TRY(cs_bases_upload(ctx, d->curve, CS_G1, d->h_query, n, wb, &pk->h_query));
  {
    static int share_env = -1;  // CS_SHARE_B_SORT=0 disables the shared sort (A/B comparison)
    if (share_env < 0) { const char* e = getenv("CS_SHARE_B_SORT"); share_env = e ? atoi(e) : 1; }
    if (share_env) CS_TRY(bases_sort_compatible(ctx, pk->b_g1, pk->b_g2, &pk->share_b_sort));
  }
  switch (d->curve) {
    case CS_BN254: CS_TRY(build_coset_table<Bn254Cfg>(ctx, pk.get())); break;
#if defined(CS_ENABLE_BLS12_381)
    case CS_BLS12_381: CS_TRY(build_coset_table<Bls381Cfg>(ctx, pk.get())); break;
#endif
    default: break;
  }
  *out = pk.release();
  return 0;
}

void cs_groth16_pk_free(cs_groth16_pk* pk) {
  if (!pk) return;
  DevBuf* bufs[] = {&pk->a_rowptr, &pk->a_col, &pk->a_coeff, &pk->b_rowptr, &pk->b_col, &pk->b_coeff, &pk->coset_tab,
                    &pk->d_pub, &pk->d_wit, &pk->d_a, &pk->d_b, &pk->d_c, &pk->d_m1, &pk->d_m2,
                    &pk->c_rowptr, &pk->c_col, &pk->c_coeff, &pk->coset_tab_ark, &pk->ginv_pows, &pk->vinv_over_n};
  for (DevBuf* b : bufs) b->release();
  cs_bases_free(pk->a_query);
  cs_bases_free(pk->b_g1);
  cs_bases_free(pk->b_g2);
  cs_bases_free(pk->l_query);
  cs_bases_free(pk->h_query);
  cs_domain_free(pk->dom);
  cs_domain_free(pk->dom_ark);
  delete pk;
}

size_t cs_groth16_domain_size(const cs_groth16_pk* pk) { return pk ? pk->n : 0; }
int cs_groth16_pk_curve(const cs_groth16_pk* pk) { return pk ? pk->curve : CS_ERR_ARG; }

int cs_groth16_witness_map(cs_ctx* ctx, cs_groth16_pk* pk, cs_share_kind kind, int party, const uint64_t* h_pub,
                           const uint64_t* h_wit, const uint64_t* h_m1, const uint64_t* h_m2, uint64_t* h_out) {
  if (!ctx || !pk || !h_pub || (pk->nw && !h_wit)) return fail(CS_ERR_ARG, "cs_groth16_witness_map: NULL argument");
  if (kind != CS_PLAIN && kind != CS_REP3) return fail(CS_ERR_ARG, "cs_groth16_witness_map: bad share kind");
  if (kind == CS_REP3 && (party < 0 || party > 2)) return fail(CS_ERR_ARG, "cs_groth16_witness_map: party must be 0..2");
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_TRY(upload_inputs(ctx, pk, kind, h_pub, h_wit, h_m1, h_m2));
  switch (pk->curve) {
    case CS_BN254:
      CS_TRY((witness_map_device<Bn254Cfg>(ctx, pk, kind, party, pk->d_wit.as<uint32_t>(), h_m1 != nullptr,
                                           h_m2 != nullptr, ctx->stream)));
      break;
#if defined(CS_ENABLE_BLS12_381)
    case CS_BLS12_381:
      CS_TRY((witness_map_device<Bls381Cfg>(ctx, pk, kind, party, pk->d_wit.as<uint32_t>(), h_m1 != nullptr,
                                            h_m2 != nullptr, ctx->stream)));
      break;
#endif
    default: return fail(CS_ERR_ARG, "unsupported curve");
  }
  if (h_out) CS_CUDA(cudaMemcpyAsync(h_out, pk->d_c.p, pk->n * 32, cudaMemcpyDeviceToHost, ctx->stream));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return 0;
}

int cs_groth16_witness_map_libsnark(cs_ctx* ctx, cs_groth16_pk* pk, cs_share_kind kind, int party, const uint64_t* h_pub,
                                    const uint64_t* h_wit, const uint64_t* h_mask, uint64_t* h_out) {
  if (!ctx || !pk || !h_pub || (pk->nw && !h_wit)) return fail(CS_ERR_ARG, "cs_groth16_witness_map_libsnark: NULL argument");
  if (kind != CS_PLAIN && kind != CS_REP3) return fail(CS_ERR_ARG, "cs_groth16_witness_map_libsnark: bad share kind");
  if (kind == CS_REP3 && (party < 0 || party > 2)) return fail(CS_ERR_ARG, "cs_groth16_witness_map_libsnark: party must be 0..2");
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_TRY(upload_inputs(ctx, pk, kind, h_pub, h_wit, h_mask, nullptr));
  switch (pk->curve) {
    case CS_BN254:
      CS_TRY((witness_map_libsnark_device<Bn254Cfg>(ctx, pk, kind, party, pk->d_wit.as<uint32_t>(), h_mask != nullptr, ctx->stream)));
      break;
#if defined(CS_ENABLE_BLS12_381)
    case CS_BLS12_381:
      CS_TRY((witness_map_libsnark_device<Bls381Cfg>(ctx, pk, kind, party, pk->d_wit.as<uint32_t>(), h_mask != nullptr, ctx->stream)));
      break;
#endif
    default: return fail(CS_ERR_ARG, "unsupported curve");
  }
  if (h_out) CS_CUDA(cudaMemcpyAsync(h_out, pk->d_c.p, pk->n * 32, cudaMemcpyDeviceToHost, ctx->stream));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return 0;
}

int cs_groth16_prove_plain(cs_ctx* ctx, cs_groth16_pk* pk, const uint64_t* h_pub, const uint64_t* h_wit,
                           const uint64_t* r, const uint64_t* s, uint64_t* out_a, uint64_t* out_b, uint64_t* out_c) {
  if (!ctx || !pk || !h_pub || (pk->nw && !h_wit) || !r || !s || !out_a || !out_b || !out_c)
    return fail(CS_ERR_ARG, "cs_groth16_prove_plain: NULL argument");
  switch (pk->curve) {
    case CS_BN254: return prove_plain_t<Bn254Cfg>(ctx, pk, h_pub, h_wit, nullptr, r, s, out_a, out_b, out_c);
#if defined(CS_ENABLE_BLS12_381)
    case CS_BLS12_381: return prove_plain_t<Bls381Cfg>(ctx, pk, h_pub, h_wit, nullptr, r, s, out_a, out_b, out_c);
#endif
    default: return fail(CS_ERR_ARG, "unsupported curve");
  }
}

int cs_groth16_prove_plain_device(cs_ctx* ctx, cs_groth16_pk* pk, const uint64_t* h_pub, const uint64_t* d_wit,
                                  const uint64_t* r, const uint64_t* s, uint64_t* out_a, uint64_t* out_b,
                                  uint64_t* out_c) {
  if (!ctx || !pk || !h_pub || (pk->nw && !d_wit) || !r || !s || !out_a || !out_b || !out_c)
    return fail(CS_ERR_ARG, "cs_groth16_prove_plain_device: NULL argument");
  switch (pk->curve) {
    case CS_BN254: return prove_plain_t<Bn254Cfg>(ctx, pk, h_pub, nullptr, d_wit, r, s, out_a, out_b, out_c);
#if defined(CS_ENABLE_BLS12_381)
    case CS_BLS12_381: return prove_plain_t<Bls381Cfg>(ctx, pk, h_pub, nullptr, d_wit, r, s, out_a, out_b, out_c);
#endif
    default: return fail(CS_ERR_ARG, "unsupported curve");
  }
}

// ShamirGroth16Driver's local computation is the plain driver's, applied to degree-t shares
// (mpc/shamir.rs:29-103: public terms and public points are added by EVERY party, local_mul_vec = a*b,
// to_half_share = identity); only rand / degree_reduce_point / open_half_point touch the network.
int cs_groth16_shamir_local(cs_ctx* ctx, cs_groth16_pk* pk, const uint64_t* h_pub, const uint64_t* h_wit_shares,
                            const uint64_t* r_share, const uint64_t* s_share, uint64_t* out_g_a, uint64_t* out_g1_b,
                            uint64_t* out_g2_b, uint64_t* out_l, uint64_t* out_h) {
  if (!ctx || !pk || !h_pub || (pk->nw && !h_wit_shares) || !r_share || !s_share || !out_g_a || !out_g1_b ||
      !out_g2_b || !out_l || !out_h)
    return fail(CS_ERR_ARG, "cs_groth16_shamir_local: NULL argument");
  switch (pk->curve) {
    case CS_BN254:
      return local_phase<Bn254Cfg>(ctx, pk, CS_PLAIN, 0, h_pub, h_wit_shares, nullptr, nullptr, nullptr, r_share,
                                   s_share, out_g_a, out_g1_b, out_g2_b, out_l, out_h);
#if defined(CS_ENABLE_BLS12_381)
    case CS_BLS12_381:
      return local_phase<Bls381Cfg>(ctx, pk, CS_PLAIN, 0, h_pub, h_wit_shares, nullptr, nullptr, nullptr, r_share,
                                    s_share, out_g_a, out_g1_b, out_g2_b, out_l, out_h);
#endif
    default: return fail(CS_ERR_ARG, "unsupported curve");
  }
}

int cs_groth16_rep3_local(cs_ctx* ctx, cs_groth16_pk* pk, int party, const uint64_t* h_pub,
                          const uint64_t* h_wit_shares, const uint64_t* h_m1, const uint64_t* h_m2,
                          const uint64_t* r_share, const uint64_t* s_share, uint64_t* out_g_a, uint64_t* out_g1_b,
                          uint64_t* out_g2_b, uint64_t* out_l, uint64_t* out_h) {
  return cs_groth16_rep3_local_parts(ctx, pk, party, CS_PART_ALL, h_pub, h_wit_shares, h_m1, h_m2, r_share, s_share,
                                     out_g_a, out_g1_b, out_g2_b, out_l, out_h);
}

int cs_groth16_rep3_local_parts(cs_ctx* ctx, cs_groth16_pk* pk, int party, unsigned parts, const uint64_t* h_pub,
                                const uint64_t* h_wit_shares, const uint64_t* h_m1, const uint64_t* h_m2,
                                const uint64_t* r_share, const uint64_t* s_share, uint64_t* out_g_a,
                                uint64_t* out_g1_b, uint64_t* out_g2_b, uint64_t* out_l, uint64_t* out_h) {
  return cs_groth16_rep3_local_prf(ctx, pk, party, parts, h_pub, h_wit_shares, h_m1, h_m2, nullptr, r_share, s_share,
                                   out_g_a, out_g1_b, out_g2_b, out_l, out_h);
}

int cs_groth16_rep3_local_prf(cs_ctx* ctx, cs_groth16_pk* pk, int party, unsigned parts, const uint64_t* h_pub,
                              const uint64_t* h_wit_shares, const uint64_t* h_m1, const uint64_t* h_m2,
                              const cs_rep3_prf* prf, const uint64_t* r_share, const uint64_t* s_share,
                              uint64_t* out_g_a, uint64_t* out_g1_b, uint64_t* out_g2_b, uint64_t* out_l,
                              uint64_t* out_h) {
  if (prf && (prf->rounds == 0 || (prf->rounds & 1) || prf->rounds > 20))
    return fail(CS_ERR_ARG, "cs_groth16_rep3_local_prf: rounds must be even and <= 20");
  if (!ctx || !pk || !h_pub || (pk->nw && !h_wit_shares) || !r_share || !s_share || !out_g_a || !out_g1_b ||
      !out_g2_b || !out_l || !out_h)
    return fail(CS_ERR_ARG, "cs_groth16_rep3_local: NULL argument");
  if (party < 0 || party > 2) return fail(CS_ERR_ARG, "cs_groth16_rep3_local: party must be 0..2");
  // to_half_share = the `a` component (mpc/rep3.rs:120-122): first Fr of the share
  switch (pk->curve) {
    case CS_BN254:
      return local_phase<Bn254Cfg>(ctx, pk, CS_REP3, party, h_pub, h_wit_shares, nullptr, h_m1, h_m2, r_share, s_share,
                                   out_g_a, out_g1_b, out_g2_b, out_l, out_h, parts, prf);
#if defined(CS_ENABLE_BLS12_381)
    case CS_BLS12_381:
      return local_phase<Bls381Cfg>(ctx, pk, CS_REP3, party, h_pub, h_wit_shares, nullptr, h_m1, h_m2, r_share, s_share,
                                    out_g_a, out_g1_b, out_g2_b, out_l, out_h, parts, prf);
#endif
    default: return fail(CS_ERR_ARG, "unsupported curve");
  }
}

int cs_groth16_shamir_prove(cs_ctx* ctx, cs_groth16_pk* pk, cs_net* net0, cs_net* net1, int num_parties, int threshold,
                            const uint64_t* h_pub, const uint64_t* h_wit, uint64_t* out_a, uint64_t* out_b, uint64_t* out_c,
                            uint64_t* out_rs) {
  if (!ctx || !pk || !net0 || !net1 || !h_pub || (pk->nw && !h_wit) || !out_a || !out_b || !out_c)
    return fail(CS_ERR_ARG, "cs_groth16_shamir_prove: NULL argument");
  if (net0->n != num_parties || net1->n != num_parties || net0->id != net1->id)
    return fail(CS_ERR_ARG, "cs_groth16_shamir_prove: net0/net1 must be %d-party meshes of the same party", num_parties);
  switch (pk->curve) {
    case CS_BN254: return shamir_prove_t<Bn254Cfg>(ctx, pk, net0, net1, num_parties, threshold, h_pub, h_wit, nullptr, out_a, out_b, out_c, out_rs);
#if defined(CS_ENABLE_BLS12_381)
    case CS_BLS12_381: return shamir_prove_t<Bls381Cfg>(ctx, pk, net0, net1, num_parties, threshold, h_pub, h_wit, nullptr, out_a, out_b, out_c, out_rs);
#endif
    default: return fail(CS_ERR_ARG, "unsupported curve");
  }
}

int cs_groth16_prove_with_shamir_bridge(cs_ctx* ctx, cs_groth16_pk* pk, cs_net* net0, cs_net* net1, const uint64_t* h_pub,
                                        const uint64_t* h_wit_rep3, uint64_t* out_a, uint64_t* out_b, uint64_t* out_c,
                                        uint64_t* out_rs) {
  if (!ctx || !pk || !net0 || !net1 || !h_pub || (pk->nw && !h_wit_rep3) || !out_a || !out_b || !out_c)
    return fail(CS_ERR_ARG, "cs_groth16_prove_with_shamir_bridge: NULL argument");
  if (net0->n != 3 || net0->id < 0 || net0->id > 2) return fail(CS_ERR_ARG, "not a valid party id");  // groth16.rs:403-404
  CS_CUDA(cudaSetDevice(ctx->device));
  // get_translation_points (bridges/rep3_to_shamir.rs:14-29): f(X) = 1 - X / z evaluated at id + 1
  const uint64_t id = (uint64_t)net0->id;
  const uint64_t z1 = id == 0 ? 3 : id, z2 = id == 2 ? 1 : id + 2, e = id + 1;
  uint64_t ca[4], cb[4];
  auto coeff = [&](uint64_t z, uint64_t* out) -> int {
    uint64_t zc[4] = {z, 0, 0, 0}, ec[4] = {e, 0, 0, 0}, onec[4] = {1, 0, 0, 0}, zm[4], em[4], onem[4], q[4];
    CS_TRY(cs_fr_to_mont((cs_curve)pk->curve, zc, zm, 1));
    CS_TRY(cs_fr_to_mont((cs_curve)pk->curve, ec, em, 1));
    CS_TRY(cs_fr_to_mont((cs_curve)pk->curve, onec, onem, 1));
    CS_TRY(cs_fr_inv((cs_curve)pk->curve, zm, q));
    CS_TRY(cs_fr_mul((cs_curve)pk->curve, q, em, q));
    return cs_fr_sub((cs_curve)pk->curve, onem, q, out);
  };
  CS_TRY(coeff(z1, ca));
  CS_TRY(coeff(z2, cb));
  // translate_primefield_repshare_vec on the device: share_i = a_i x + b_i y (k_rep3_to_shamir)
  DevBuf d_in, d_out;
  CS_TRY(d_in.reserve(pk->nw * 64 + 64));
  CS_TRY(d_out.reserve(pk->nw * 32 + 32));
  int rc = 0;
  if (pk->nw) {
    CS_CUDA(cudaMemcpyAsync(d_in.p, h_wit_rep3, pk->nw * 64, cudaMemcpyHostToDevice, ctx->stream));
    rc = cs_rep3_to_shamir(ctx, (cs_curve)pk->curve, d_in.as<uint64_t>(), ca, cb, d_out.as<uint64_t>(), pk->nw);
  }
  if (!rc) {
    switch (pk->curve) {
      case CS_BN254: rc = shamir_prove_t<Bn254Cfg>(ctx, pk, net0, net1, 3, 1, h_pub, nullptr, d_out.as<uint64_t>(), out_a, out_b, out_c, out_rs); break;
#if defined(CS_ENABLE_BLS12_381)
      case CS_BLS12_381: rc = shamir_prove_t<Bls381Cfg>(ctx, pk, net0, net1, 3, 1, h_pub, nullptr, d_out.as<uint64_t>(), out_a, out_b, out_c, out_rs); break;
#endif
      default: rc = fail(CS_ERR_ARG, "unsupported curve");
    }
  }
  d_in.release();
  d_out.release();
  return rc;
}

}  // extern "C"
