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
  // Whose sorted entries each witness MSM (A, B1, B2, L) accumulates, decided once from the infinity masks
  // (plan_witness_views): -1 = the shared witness sort as it is; its own index = its own filtered view of that sort;
  // another index = that MSM's view (same table geometry and infinity pattern, as B2 has with B1)
  int wit_src[4] = {0, 1, 2, 3};
  cs_domain* dom_ark = nullptr;
  DevBuf coset_tab_ark, ginv_pows, vinv_over_n;
  DevBuf d_pt;  // the single-point work of a batch of proofs (batch_points)
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
// K > 1 (plain values only): the witness maps of K proofs at once -- public inputs [K][ni] in d_pub, witnesses [K][nw]
// from d_wit -- with a, b, c and h as K interleaved columns ([n][K]), so that each transform is one NTT call.
template <class Cfg>
int witness_map_device(cs_ctx* ctx, cs_groth16_pk* pk, int kind, int party, const uint32_t* d_wit, bool have_m1,
                       bool have_m2, cudaStream_t st, uint32_t K = 1) {
  typedef typename Cfg::FrP FrP;
  const unsigned batch = kind == CS_REP3 ? 2 : 1;
  const int pub_comp = kind == CS_REP3 ? (party == 0 ? 0 : (party == 1 ? 1 : -1)) : 0;
  const uint32_t n = (uint32_t)pk->n;
  if (K > 1 && kind != CS_PLAIN) return fail(CS_ERR_ARG, "witness map: batches are of plain witnesses");
  CS_TRY(pk->d_a.reserve((size_t)n * batch * K * 32));
  CS_TRY(pk->d_b.reserve((size_t)n * batch * K * 32));
  CS_TRY(pk->d_c.reserve((size_t)n * K * 32));
  // a = A w (+ promoted public rows, reduction.rs:104-113), b = B w   (evaluate_constraint)
  CS_SPAN("witness map from matrices");
  {
  CS_SPAN("evaluate constraints + coset table computation");
  const dim3 grid(ceil_div(n, 128), K);
  const uint32_t wps = (uint32_t)pk->nw * batch;
  CS_LAUNCH(k_spmv<FrP>, grid, 128, 0, st, pk->a_rowptr.as<uint32_t>(), pk->a_col.as<uint32_t>(),
            pk->a_coeff.as<uint32_t>(), pk->d_pub.as<uint32_t>(), (uint32_t)pk->ni, d_wit, batch, batch,
            pub_comp, (uint32_t)pk->nc, (uint32_t)pk->ni, n, wps, batch * K, pk->d_a.as<uint32_t>());
  CS_LAUNCH(k_spmv<FrP>, grid, 128, 0, st, pk->b_rowptr.as<uint32_t>(), pk->b_col.as<uint32_t>(),
            pk->b_coeff.as<uint32_t>(), pk->d_pub.as<uint32_t>(), (uint32_t)pk->ni, d_wit, batch, batch,
            pub_comp, (uint32_t)pk->nc, 0u, n, wps, batch * K, pk->d_b.as<uint32_t>());
  }
  unsigned blocks = ceil_div((size_t)n * K, 256);
  if (blocks > CS_NUM_SMS * 16) blocks = CS_NUM_SMS * 16;
  // c = local_mul_vec(a, b)   (reduction.rs:160)
  CS_SPAN("c: local_mul_vec / a, b, c: distribute powers (fft/ifft)");
  if (kind == CS_REP3)
    CS_LAUNCH(k_rep3_local_mul<FrP>, blocks, 256, 0, st, pk->d_a.as<uint32_t>(), pk->d_b.as<uint32_t>(),
              have_m1 ? pk->d_m1.as<uint32_t>() : (const uint32_t*)nullptr, (const uint32_t*)nullptr,
              pk->d_c.as<uint32_t>(), (size_t)n);
  else
    CS_LAUNCH(k_plain_mul_sub<FrP>, blocks, 256, 0, st, pk->d_a.as<uint32_t>(), pk->d_b.as<uint32_t>(),
              (const uint32_t*)nullptr, pk->d_c.as<uint32_t>(), (size_t)n * K);
  // each of a, b, c: ifft_in_to_out -> * coset table -> fft_out_to_in   (reduction.rs:135-178);
  // the table multiply and the 1/n are fused into the last iNTT pass.
  const uint32_t* post = pk->log_n ? pk->coset_tab.as<uint32_t>() : nullptr;
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_a.as<uint32_t>(), batch * K, true, post, st));
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_a.as<uint32_t>(), batch * K, false, nullptr, st));
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_b.as<uint32_t>(), batch * K, true, post, st));
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_b.as<uint32_t>(), batch * K, false, nullptr, st));
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_c.as<uint32_t>(), K, true, post, st));
  CS_TRY(ntt_run(ctx, pk->dom, pk->d_c.as<uint32_t>(), K, false, nullptr, st));
  // h = local_mul_vec(a', b') - c'   (reduction.rs:182-190), in place over c
  CS_SPAN("ab: local_mul_vec + compute ab");
  if (kind == CS_REP3)
    CS_LAUNCH(k_rep3_local_mul<FrP>, blocks, 256, 0, st, pk->d_a.as<uint32_t>(), pk->d_b.as<uint32_t>(),
              have_m2 ? pk->d_m2.as<uint32_t>() : (const uint32_t*)nullptr, pk->d_c.as<uint32_t>(),
              pk->d_c.as<uint32_t>(), (size_t)n);
  else
    CS_LAUNCH(k_plain_mul_sub<FrP>, blocks, 256, 0, st, pk->d_a.as<uint32_t>(), pk->d_b.as<uint32_t>(),
              pk->d_c.as<uint32_t>(), pk->d_c.as<uint32_t>(), (size_t)n * K);
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
            (uint32_t)pk->nc, (uint32_t)pk->ni, n, 0u, batch, pk->d_a.as<uint32_t>());
  CS_LAUNCH(k_spmv<FrP>, ceil_div(n, 128), 128, 0, st, pk->b_rowptr.as<uint32_t>(), pk->b_col.as<uint32_t>(),
            pk->b_coeff.as<uint32_t>(), pk->d_pub.as<uint32_t>(), (uint32_t)pk->ni, d_wit, batch, batch, pub_comp,
            (uint32_t)pk->nc, 0u, n, 0u, batch, pk->d_b.as<uint32_t>());
  // c from the C matrix as HALF shares (reduction.rs:292-298)
  CS_LAUNCH(k_spmv<FrP>, ceil_div(n, 128), 128, 0, st, pk->c_rowptr.as<uint32_t>(), pk->c_col.as<uint32_t>(),
            pk->c_coeff.as<uint32_t>(), pk->d_pub.as<uint32_t>(), (uint32_t)pk->ni, d_wit, 1u, batch, pub_comp_hs,
            (uint32_t)pk->nc, 0u, n, 0u, 1u, pk->d_c.as<uint32_t>());
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

// Fills pk->wit_src.  A witness MSM reads the shared witness sort as it is when its table slots are that sort's
// entries (w * nw + i: nw bases, offset 0) and none of its bases is infinite -- L of a key in which every witness
// variable occurs.  Any other MSM filters the sort for its table, and MSMs whose tables agree in length, offset and
// infinity pattern share one filtered view (B1 and B2: B_i(tau) G1 and B_i(tau) G2 vanish together).
int plan_witness_views(cs_ctx* ctx, cs_groth16_pk* pk) {
  const size_t ni = pk->ni, nw = pk->nw;
  if (!nw) return 0;
  const cs_bases* q[4] = {pk->a_query, pk->b_g1, pk->b_g2, pk->l_query};
  const size_t off[4] = {ni, ni, ni, 0};
  std::vector<uint8_t> inf[4];
  for (int j = 0; j < 4; j++) {
    if (q[j]->sh.c != q[0]->sh.c || q[j]->sh.W != q[0]->sh.W || q[j]->sh.k != q[0]->sh.k)
      return fail(CS_ERR_STATE, "cs_groth16_pk_create: the witness MSMs' tables differ in window shape");
    std::vector<uint32_t> words((q[j]->n + 31) / 32);
    CS_CUDA(cudaMemcpyAsync(words.data(), q[j]->infmask.p, words.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CS_CUDA(cudaStreamSynchronize(ctx->stream));
    inf[j].resize(nw);
    bool any = false;
    for (size_t i = 0; i < nw; i++) {
      const size_t k = off[j] + i;
      inf[j][i] = (words[k >> 5] >> (k & 31)) & 1;
      any = any || inf[j][i];
    }
    pk->wit_src[j] = j;
    if (q[j]->n == nw && off[j] == 0 && !any) {
      pk->wit_src[j] = -1;
      continue;
    }
    for (int k = 0; k < j; k++)
      if (pk->wit_src[k] == k && q[k]->n == q[j]->n && off[k] == off[j] && inf[k] == inf[j]) {
        pk->wit_src[j] = k;
        break;
      }
  }
  return 0;
}

// Device bytes of a key whose tables keep one row per k windows: its five tables, and what its proofs reserve, sized by
// the code that reserves it -- the five MSM workspaces and the shared witness sort (msm_sort_bytes, msm_accum_bytes),
// the witness-map vectors of a Rep3 proof (the larger share kind: two components, two masks), the coset table and
// the domain's twiddles.  cw / ch: windows of the witness tables and of H.
template <class Cfg>
size_t key_bytes(size_t ni, size_t nw, size_t n, unsigned cw, unsigned ch, unsigned k) {
  typedef typename GroupOf<Cfg, 0>::F F1;
  typedef typename GroupOf<Cfg, 1>::F F2;
  const MsmShape sw = msm_shape(Cfg::FR_BITS, cw, k), shh = msm_shape(Cfg::FR_BITS, ch, k);
  size_t b = 2 * bases_bytes<Cfg, 0>(ni + nw, sw) + bases_bytes<Cfg, 1>(ni + nw, sw) + bases_bytes<Cfg, 0>(n, shh);
  if (nw) {
    b += bases_bytes<Cfg, 0>(nw, sw);
    b += 5 * msm_sort_bytes(sw, (uint32_t)nw) + 3 * msm_accum_bytes<F1>(sw, (uint32_t)nw) + msm_accum_bytes<F2>(sw, (uint32_t)nw);
  }
  b += msm_sort_bytes(shh, (uint32_t)n) + msm_accum_bytes<F1>(shh, (uint32_t)n);
  const size_t fr = 32;
  b += DevBuf::alloc_size(ni * fr) + DevBuf::alloc_size(nw * 2 * fr) + 2 * DevBuf::alloc_size(n * 2 * fr) +
       4 * DevBuf::alloc_size(n * fr) + 2 * DevBuf::alloc_size(n / 2 * fr);
  return b;
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
  CS_TRY(ctx_fork(ctx, 5));
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
    // the four MSMs take the same scalars: their digits are sorted once, on side stream 4, and each MSM reads that
    // sort as it is or filters it for its own table (msm_enqueue)
    const unsigned part[4] = {CS_PART_A, CS_PART_B1, CS_PART_B2, CS_PART_L};
    const cs_bases* q[4] = {pk->a_query, pk->b_g1, pk->b_g2, pk->l_query};
    const size_t off[4] = {pk->ni, pk->ni, pk->ni, 0};
    if (do_a || do_b1 || do_b2 || do_l)
      CS_TRY(msm_sort_shared_dyn(ctx, CS_WIT_SORT, ctx->side[4], pk->a_query, wit, batch, pk->nw, 1));
    for (int j = 0; j < 4; j++) {
      if (!(parts & part[j])) continue;
      int src = pk->wit_src[j];
      if (src >= 0 && !(parts & part[src])) src = j;  // the MSM that builds the view is not part of this call
      const int sort_slot = src < 0 || src == j ? CS_WIT_SORT : src;
      CS_TRY(msm_enqueue_dyn(ctx, j, ctx->side[j], q[j], off[j], wit, batch, pk->nw, 1, sort_slot, src == j));
    }
  }
  CS_TRY(ctx_join(ctx, 5));
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


// ---- batches of plain proofs: CoGroth16::prove (plain driver) applied to K witnesses of one circuit
// A sub-batch of K proofs runs one witness map over K interleaved columns, one sort and one accumulation per MSM
// with a proof dimension (msm_enqueue's K), and does every proof's single-point work on the device (k_point_*).

// Carves the point work's device buffers for K proofs out of one allocation; null base = sizes only.
template <class Cfg>
struct BatchPoints {
  typedef typename GroupOf<Cfg, 0>::F F1;
  typedef typename GroupOf<Cfg, 1>::F F2;
  Affine<F1> *b1, *cst1, *cb, *out_c;  // A and B1 term bases [2K][ni], their shared points [2], C's bases [K][3], C [K]
  Affine<F2> *b2, *cst2, *out_b2;      // B2 term bases [K][ni], its shared point, B2 [K]
  uint32_t *sc1, *sc3;                 // scalars: A and B1 terms [2K][ni] (B2's are B1's), C's terms [K][3]
  Xyzz<F1> *prod1, *prod3, *sum1;
  Xyzz<F2> *prod2, *sum2;
  size_t bytes = 0;
  BatchPoints(char* base, size_t K, size_t ni) {
    auto take = [&](size_t n) { char* p = base ? base + bytes : nullptr; bytes += (n + 255) & ~(size_t)255; return p; };
    b1 = (Affine<F1>*)take(2 * K * ni * sizeof(Affine<F1>));
    cst1 = (Affine<F1>*)take(2 * sizeof(Affine<F1>));
    cb = (Affine<F1>*)take(3 * K * sizeof(Affine<F1>));
    out_c = (Affine<F1>*)take(K * sizeof(Affine<F1>));
    b2 = (Affine<F2>*)take(K * ni * sizeof(Affine<F2>));
    cst2 = (Affine<F2>*)take(sizeof(Affine<F2>));
    out_b2 = (Affine<F2>*)take(K * sizeof(Affine<F2>));
    sc1 = (uint32_t*)take(2 * K * ni * 32);
    sc3 = (uint32_t*)take(3 * K * 32);
    prod1 = (Xyzz<F1>*)take(2 * K * ni * sizeof(Xyzz<F1>));
    prod3 = (Xyzz<F1>*)take(3 * K * sizeof(Xyzz<F1>));
    sum1 = (Xyzz<F1>*)take(2 * K * sizeof(Xyzz<F1>));
    prod2 = (Xyzz<F2>*)take(K * ni * sizeof(Xyzz<F2>));
    sum2 = (Xyzz<F2>*)take(K * sizeof(Xyzz<F2>));
  }
};

// Device bytes of the scratch of a sub-batch of K proofs: the witness-map vectors and inputs, the workspaces of the
// shared witness sort and the five MSMs (bounded as in key_bytes) and the point work.
template <class Cfg>
size_t batch_bytes(const cs_groth16_pk* pk, size_t K, bool host_wit) {
  typedef typename GroupOf<Cfg, 0>::F F1;
  typedef typename GroupOf<Cfg, 1>::F F2;
  const size_t n = pk->n, nw = pk->nw;
  size_t b = 3 * DevBuf::alloc_size(n * K * 32) + DevBuf::alloc_size(pk->ni * K * 32) +
             (host_wit ? DevBuf::alloc_size(nw * K * 32) : 0) + DevBuf::alloc_size(BatchPoints<Cfg>(nullptr, K, pk->ni).bytes);
  if (nw) {
    const MsmShape sw = pk->a_query->sh;
    b += 5 * msm_sort_bytes(sw, nw, K) + 3 * msm_accum_bytes<F1>(sw, nw, K) + msm_accum_bytes<F2>(sw, nw, K);
  }
  const MsmShape shh = pk->h_query->sh;
  return b + msm_sort_bytes(shh, n, K) + msm_accum_bytes<F1>(shh, n, K);
}

// Proofs per sub-batch: the most, up to K, that the MSM limits (msm_max_batch), the NTT's pass tile and the device
// memory allow.  The memory is what the table budget leaves (table_budget) plus the scratch the key and the context
// already hold, which a larger sub-batch reallocates.  One proof always runs: it fails where a single proof would.
template <class Cfg>
int pick_sub_batch(cs_ctx* ctx, cs_groth16_pk* pk, size_t K, bool host_wit, size_t* out) {
  size_t kmax = K;
  if (pk->nw) kmax = std::min<size_t>(kmax, msm_max_batch(pk->a_query->sh, (uint32_t)pk->nw));
  kmax = std::min<size_t>(kmax, msm_max_batch(pk->h_query->sh, (uint32_t)pk->n));
  if (pk->log_n)
    while (kmax > 1 && !ntt_max_stages((uint32_t)kmax, true)) kmax--;
  size_t held = pk->d_a.cap + pk->d_b.cap + pk->d_c.cap + pk->d_pub.cap + pk->d_wit.cap + pk->d_pt.cap, budget = 0;
  for (int i = 0; i <= CS_NSIDE; i++) held += ctx->msm_ws[i].bytes();
  CS_TRY(table_budget(ctx, &budget, held));
  size_t lo = 1, hi = kmax;  // largest K' in [1, kmax] whose scratch fits, or 1
  while (lo < hi) {
    const size_t mid = lo + (hi - lo + 1) / 2;
    if (batch_bytes<Cfg>(pk, mid, host_wit) <= budget) lo = mid; else hi = mid - 1;
  }
  *out = lo;
  return 0;
}

template <class Cfg>
int prove_plain_batch_t(cs_ctx* ctx, cs_groth16_pk* pk, size_t K, const uint64_t* h_pub, const uint64_t* h_wit,
                        const uint64_t* d_wit, const uint64_t* r, const uint64_t* s, uint64_t* out_a, uint64_t* out_b,
                        uint64_t* out_c) {
  typedef HostGroup<Cfg, 0> H1;
  typedef HostGroup<Cfg, 1> H2;
  typedef host::HFp<typename Cfg::FrP> HR;
  typedef typename GroupOf<Cfg, 0>::F F1;
  typedef typename GroupOf<Cfg, 1>::F F2;
  typedef typename Cfg::FrP FrP;
  constexpr size_t G1L = 2 * H1::HF::N, G2L = 4 * H1::HF::N, FR = HR::N;
  const size_t ni = pk->ni, nw = pk->nw;
  CS_CUDA(cudaSetDevice(ctx->device));
  size_t Kb = 1;
  CS_TRY(pick_sub_batch<Cfg>(ctx, pk, K, h_wit != nullptr, &Kb));
  CS_TRY(pk->d_pt.reserve(BatchPoints<Cfg>(nullptr, Kb, ni).bytes));
  const BatchPoints<Cfg> bp(pk->d_pt.as<char>(), Kb, ni);
  // the fixed points: term bases of every proof (delta and the public-input heads), the shared sums (alpha_1 +
  // query[0], ...) and delta_1 in C's bases; the same for every sub-batch
  {
    std::vector<uint64_t> b1(2 * Kb * ni * G1L), b2(Kb * ni * G2L), cb(3 * Kb * G1L, 0), cst1(2 * G1L), cst2(G2L);
    for (size_t p = 0; p < Kb; p++)
      for (size_t j = 0; j < ni; j++) {
        const uint64_t* a = j ? pk->a_head.data() + j * G1L : pk->delta_g1.data();
        const uint64_t* b = j ? pk->b1_head.data() + j * G1L : pk->delta_g1.data();
        const uint64_t* c = j ? pk->b2_head.data() + j * G2L : pk->delta_g2.data();
        memcpy(&b1[(p * ni + j) * G1L], a, G1L * 8);
        memcpy(&b1[((Kb + p) * ni + j) * G1L], b, G1L * 8);
        memcpy(&b2[(p * ni + j) * G2L], c, G2L * 8);
      }
    for (size_t p = 0; p < Kb; p++) memcpy(&cb[(3 * p + 2) * G1L], pk->delta_g1.data(), G1L * 8);
    H1::store(cst1.data(), host::hadd(H1::load(pk->alpha_g1.data()), H1::load(pk->a_head.data())));
    H1::store(cst1.data() + G1L, host::hadd(H1::load(pk->beta_g1.data()), H1::load(pk->b1_head.data())));
    H2::store(cst2.data(), host::hadd(H2::load(pk->beta_g2.data()), H2::load(pk->b2_head.data())));
    CS_CUDA(cudaMemcpyAsync(bp.b1, b1.data(), b1.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    CS_CUDA(cudaMemcpyAsync(bp.b2, b2.data(), b2.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    CS_CUDA(cudaMemcpyAsync(bp.cb, cb.data(), cb.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    CS_CUDA(cudaMemcpyAsync(bp.cst1, cst1.data(), cst1.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    CS_CUDA(cudaMemcpyAsync(bp.cst2, cst2.data(), cst2.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    CS_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  std::vector<uint64_t> sc1(2 * Kb * ni * FR), sc3(3 * Kb * FR), cb(3 * Kb * G1L), ob2(Kb * G2L), oc(Kb * G1L);
  for (size_t j0 = 0; j0 < K; j0 += Kb) {
    const size_t k = std::min(Kb, K - j0);
    const uint32_t kk = (uint32_t)k;
    // scalars of the point work: A [r, pub[1..]], B1 and B2 [s, pub[1..]], C [s, r, -(r s)]
    for (size_t p = 0; p < k; p++) {
      const uint64_t *rp = r + (j0 + p) * FR, *sp = s + (j0 + p) * FR, *pub = h_pub + (j0 + p) * ni * FR;
      memcpy(&sc1[p * ni * FR], rp, FR * 8);
      memcpy(&sc1[(k + p) * ni * FR], sp, FR * 8);
      for (size_t j = 1; j < ni; j++) {
        memcpy(&sc1[(p * ni + j) * FR], pub + j * FR, FR * 8);
        memcpy(&sc1[((k + p) * ni + j) * FR], pub + j * FR, FR * 8);
      }
      HR rr, ss;
      memcpy(rr.l, rp, sizeof(rr.l));
      memcpy(ss.l, sp, sizeof(ss.l));
      const HR nrs = HR::zero() - rr * ss;
      memcpy(&sc3[3 * p * FR], sp, FR * 8);
      memcpy(&sc3[(3 * p + 1) * FR], rp, FR * 8);
      memcpy(&sc3[(3 * p + 2) * FR], nrs.l, FR * 8);
    }
    // inputs: public [k][ni] always from the host, the witness [k][nw] from the host or in place
    CS_TRY(upload(ctx, pk->d_pub, h_pub + j0 * ni * FR, k * ni * 32));
    const uint32_t* wit = d_wit ? reinterpret_cast<const uint32_t*>(d_wit + j0 * nw * FR) : nullptr;
    if (h_wit) {
      CS_TRY(upload(ctx, pk->d_wit, h_wit + j0 * nw * FR, k * nw * 32));
      wit = pk->d_wit.as<uint32_t>();
    }
    CS_CUDA(cudaMemcpyAsync(bp.sc1, sc1.data(), 2 * k * ni * 32, cudaMemcpyHostToDevice, ctx->stream));
    CS_CUDA(cudaMemcpyAsync(bp.sc3, sc3.data(), 3 * k * 32, cudaMemcpyHostToDevice, ctx->stream));
    // the MSMs, laid out on the streams as in local_phase: witness map -> H first, on the highest-priority stream
    CS_TRY(ctx_fork(ctx, 5));
    cudaStream_t wm = ctx->wm;
    CS_CUDA(cudaStreamWaitEvent(wm, ctx->ev_fork, 0));
    CS_TRY((witness_map_device<Cfg>(ctx, pk, CS_PLAIN, 0, wit, false, false, wm, kk)));
    CS_TRY(msm_enqueue_dyn(ctx, 4, wm, pk->h_query, 0, pk->d_c.as<uint32_t>(), kk, pk->n, 1, -1, false, kk, 1));
    if (nw) {
      const cs_bases* q[4] = {pk->a_query, pk->b_g1, pk->b_g2, pk->l_query};
      const size_t off[4] = {ni, ni, ni, 0};
      CS_TRY(msm_sort_shared_dyn(ctx, CS_WIT_SORT, ctx->side[4], pk->a_query, wit, 1, nw, 1, kk, nw));
      for (int j = 0; j < 4; j++) {
        const int src = pk->wit_src[j];
        CS_TRY(msm_enqueue_dyn(ctx, j, ctx->side[j], q[j], off[j], wit, 1, nw, 1, src < 0 || src == j ? CS_WIT_SORT : src,
                               src == j, kk, nw));
      }
    }
    CS_TRY(ctx_join(ctx, 5));
    CS_CUDA(cudaEventRecord(ctx->ev_wm, wm));
    CS_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_wm, 0));
    // the point work (groth16.rs:232-322 with the plain driver), after the MSMs:
    //   A = alpha_1 + query[0] + sum_j pub_j query[j] + r delta_1 + msm_A      (B1, B2 alike with s)
    //   C = s A + r B1 - (r s) delta_1 + L + H
    cudaStream_t st = ctx->stream;
    auto res1 = [&](int slot) { return nw || slot == 4 ? ctx->msm_ws[slot].result.template as<Xyzz<F1>>() : nullptr; };
    const Xyzz<F2>* res_b2 = nw ? ctx->msm_ws[2].result.as<Xyzz<F2>>() : nullptr;
    const uint32_t T = (uint32_t)ni, nt = kk * T;
    const uint32_t* sc_b = bp.sc1 + (size_t)nt * FrP::N;  // B1's and B2's scalars
    CS_LAUNCH((k_point_terms<F1, FrP>), ceil_div(nt, 128), 128, 0, st, bp.b1, bp.sc1, nt, bp.prod1);
    CS_LAUNCH((k_point_terms<F1, FrP>), ceil_div(nt, 128), 128, 0, st, bp.b1 + Kb * ni, sc_b, nt, bp.prod1 + nt);
    CS_LAUNCH((k_point_terms<F2, FrP>), ceil_div(nt, 128), 128, 0, st, bp.b2, sc_b, nt, bp.prod2);
    CS_LAUNCH(k_point_sum<F1>, ceil_div(kk, 128), 128, 0, st, bp.prod1, T, kk, res1(0), (const Xyzz<F1>*)nullptr, bp.cst1,
              bp.sum1);
    CS_LAUNCH(k_point_sum<F1>, ceil_div(kk, 128), 128, 0, st, bp.prod1 + nt, T, kk, res1(1),
              (const Xyzz<F1>*)nullptr, bp.cst1 + 1, bp.sum1 + kk);
    CS_LAUNCH(k_point_sum<F2>, ceil_div(kk, 128), 128, 0, st, bp.prod2, T, kk, res_b2, (const Xyzz<F2>*)nullptr, bp.cst2,
              bp.sum2);
    const uint32_t runs = ceil_div(kk, POINT_INV_RUN);
    CS_LAUNCH(k_point_affine<F1>, ceil_div(runs, 128), 128, 0, st, bp.sum1, kk, 3u, bp.cb);
    CS_LAUNCH(k_point_affine<F1>, ceil_div(runs, 128), 128, 0, st, bp.sum1 + kk, kk, 3u, bp.cb + 1);
    CS_LAUNCH(k_point_affine<F2>, ceil_div(runs, 128), 128, 0, st, bp.sum2, kk, 1u, bp.out_b2);
    CS_LAUNCH((k_point_terms<F1, FrP>), ceil_div(3 * kk, 128), 128, 0, st, bp.cb, bp.sc3, 3 * kk, bp.prod3);
    CS_LAUNCH(k_point_sum<F1>, ceil_div(kk, 128), 128, 0, st, bp.prod3, 3u, kk, res1(3), res1(4), (const Affine<F1>*)nullptr,
              bp.sum1);
    CS_LAUNCH(k_point_affine<F1>, ceil_div(runs, 128), 128, 0, st, bp.sum1, kk, 1u, bp.out_c);
    CS_CUDA(cudaGetLastError());
    CS_CUDA(cudaMemcpyAsync(cb.data(), bp.cb, 3 * k * G1L * 8, cudaMemcpyDeviceToHost, st));
    CS_CUDA(cudaMemcpyAsync(ob2.data(), bp.out_b2, k * G2L * 8, cudaMemcpyDeviceToHost, st));
    CS_CUDA(cudaMemcpyAsync(oc.data(), bp.out_c, k * G1L * 8, cudaMemcpyDeviceToHost, st));
    CS_CUDA(cudaStreamSynchronize(st));
    for (size_t p = 0; p < k; p++) memcpy(out_a + (j0 + p) * G1L, &cb[3 * p * G1L], G1L * 8);
    memcpy(out_b + j0 * G2L, ob2.data(), k * G2L * 8);
    memcpy(out_c + j0 * G1L, oc.data(), k * G1L * 8);
  }
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
  return cs::groth16_pk_create(ctx, d, 0, out);
}

}  // extern "C"

int cs::groth16_pk_create(cs_ctx* ctx, const cs_groth16_key_desc* d, unsigned k, cs_groth16_pk** out) {
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
  if (d->window_bits && (d->window_bits < 2 || d->window_bits > (int)MSM_MAX_WINDOW))
    return fail(CS_ERR_ARG, "cs_bases_upload: window_bits %d out of range [2,%u] (0 = automatic)", d->window_bits, MSM_MAX_WINDOW);
  CS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<cs_groth16_pk, void (*)(cs_groth16_pk*)> pk(new cs_groth16_pk(), cs_groth16_pk_free);
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
  // A, B1, B2 and L share one sort of the witness digits, so their tables share one window shape: the one the
  // nw witness scalars would get (the MSMs run over nw scalars; the result does not depend on the window)
  int wwb = wb, hwb = wb;
  // one k (windows per table row) for the five tables: the smallest with which the key fits the table budget
  CS_DISPATCH_CURVE(d->curve, {
    if (!wwb) wwb = (int)msm_auto_window(nw, Cfg::FR_BITS);
    if (!hwb) hwb = (int)msm_auto_window(n, Cfg::FR_BITS);
    const unsigned cmax = wwb > hwb ? wwb : hwb;
    const unsigned W = msm_shape(Cfg::FR_BITS, wwb < hwb ? wwb : hwb).W;  // the more windows of the two shapes
    if (!k)
      CS_TRY(pick_table_rows(ctx, cmax, W, [&](unsigned kk) { return key_bytes<Cfg>(ni, nw, n, wwb, hwb, kk); },
                             "cs_groth16_pk_create", &k));
  });
  CS_TRY(bases_upload(ctx, d->curve, CS_G1, d->a_query, d->a_query_len, wwb, k, &pk->a_query));
  CS_TRY(bases_upload(ctx, d->curve, CS_G1, d->b_g1_query, d->b_g1_query_len, wwb, k, &pk->b_g1));
  CS_TRY(bases_upload(ctx, d->curve, CS_G2, d->b_g2_query, d->b_g2_query_len, wwb, k, &pk->b_g2));
  if (nw) CS_TRY(bases_upload(ctx, d->curve, CS_G1, d->l_query, d->l_query_len, wwb, k, &pk->l_query));
  CS_TRY(bases_upload(ctx, d->curve, CS_G1, d->h_query, n, hwb, k, &pk->h_query));
  CS_TRY(plan_witness_views(ctx, pk.get()));
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

extern "C" {

void cs_groth16_pk_free(cs_groth16_pk* pk) {
  if (!pk) return;
  DevBuf* bufs[] = {&pk->a_rowptr, &pk->a_col, &pk->a_coeff, &pk->b_rowptr, &pk->b_col, &pk->b_coeff, &pk->coset_tab,
                    &pk->d_pub, &pk->d_wit, &pk->d_a, &pk->d_b, &pk->d_c, &pk->d_m1, &pk->d_m2,
                    &pk->c_rowptr, &pk->c_col, &pk->c_coeff, &pk->coset_tab_ark, &pk->ginv_pows, &pk->vinv_over_n,
                    &pk->d_pt};
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

int cs_groth16_pk_table_info(const cs_groth16_pk* pk, unsigned* table_rows, size_t* table_bytes) {
  if (!pk) return fail(CS_ERR_ARG, "cs_groth16_pk_table_info: pk is NULL");
  const cs_bases* q[5] = {pk->a_query, pk->b_g1, pk->b_g2, pk->l_query, pk->h_query};
  size_t bytes = 0;
  for (const cs_bases* b : q)
    if (b) bytes += b->table.cap + b->infmask.cap;
  if (table_rows) *table_rows = pk->a_query->sh.T;
  if (table_bytes) *table_bytes = bytes;
  return 0;
}
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

int cs_groth16_prove_plain_batch(cs_ctx* ctx, cs_groth16_pk* pk, size_t num_proofs, const uint64_t* h_public_inputs,
                                 size_t num_public, const uint64_t* h_witness, const uint64_t* d_witness, size_t num_witness,
                                 const uint64_t* h_r_mont, const uint64_t* h_s_mont, uint64_t* out_a, uint64_t* out_b,
                                 uint64_t* out_c) {
  if (!ctx || !pk || !h_public_inputs || !h_r_mont || !h_s_mont || !out_a || !out_b || !out_c)
    return fail(CS_ERR_ARG, "cs_groth16_prove_plain_batch: NULL argument");
  if (num_proofs == 0) return fail(CS_ERR_ARG, "cs_groth16_prove_plain_batch: a batch needs at least one proof");
  if (num_public != pk->ni || num_witness != pk->nw)
    return fail(CS_ERR_ARG, "cs_groth16_prove_plain_batch: the key takes %zu public inputs (incl. the leading one) and %zu "
                "witness values per proof, got %zu and %zu", pk->ni, pk->nw, num_public, num_witness);
  if (pk->nw && !h_witness == !d_witness)
    return fail(CS_ERR_ARG, "cs_groth16_prove_plain_batch: pass the witnesses either on the host or on the device");
  CS_DISPATCH_CURVE(pk->curve, {
    return prove_plain_batch_t<Cfg>(ctx, pk, num_proofs, h_public_inputs, h_witness, d_witness, h_r_mont, h_s_mont, out_a,
                                    out_b, out_c);
  });
  return 0;
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
