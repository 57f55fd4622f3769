// C-ABI entry points of the UltraHonk sumcheck kernels (cs_sumcheck.cuh); contract in include/cosnarks_gpu.h.
#include "cs_lib.cuh"
#include "cs_net.h"
#include "cs_sumcheck.cuh"

using namespace cs;

namespace {

template <class Cfg>
int gate_separator_t(cs_ctx* ctx, const uint64_t* h_betas, unsigned log_n, uint64_t* d_out) {
  typedef typename Cfg::FrP FrP;
  CS_TRY(ctx->io.reserve((size_t)(log_n ? log_n : 1) * 32));
  if (log_n) CS_CUDA(cudaMemcpyAsync(ctx->io.p, h_betas, (size_t)log_n * 32, cudaMemcpyHostToDevice, ctx->stream));
  const size_t n = (size_t)1 << log_n;
  CS_LAUNCH(k_sc_gate_separator<FrP>, ceil_div(n, 128), 128, 0, ctx->stream, ctx->io.as<uint32_t>(), log_n,
            reinterpret_cast<uint32_t*>(d_out));
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaStreamSynchronize(ctx->stream));  // ctx->io is reused by the next convenience call
  return 0;
}

template <class Cfg>
int fold_t(cs_ctx* ctx, const uint64_t* const* d_in, uint64_t* const* d_out, size_t n_polys, int shared, size_t len,
           const uint64_t* h_challenge) {
  typedef typename Cfg::FrP FrP;
  Fp<FrP> u;
  memcpy(u.l, h_challenge, sizeof(u.l));
  const uint32_t comps = shared ? 2 : 1;
  const size_t half = len / 2;
  unsigned blocks = ceil_div(half * comps, 256);
  if (blocks > CS_NUM_SMS * 8) blocks = CS_NUM_SMS * 8;
  for (size_t base = 0; base < n_polys; base += SC_FOLD_MAX) {
    const size_t cnt = n_polys - base < (size_t)SC_FOLD_MAX ? n_polys - base : (size_t)SC_FOLD_MAX;
    ScFoldArgs a;
    memset(&a, 0, sizeof(a));
    for (size_t k = 0; k < cnt; k++) {
      a.in[k] = reinterpret_cast<const uint32_t*>(d_in[base + k]);
      a.out[k] = reinterpret_cast<uint32_t*>(d_out[base + k]);
    }
    CS_LAUNCH(k_sc_fold<FrP>, dim3(blocks, (unsigned)cnt), 256, 0, ctx->stream, a, comps, half, u, half == 1 ? 1 : 0);
  }
  CS_CUDA(cudaGetLastError());
  return 0;
}

template <class Cfg>
int arith_round_t(cs_ctx* ctx, int kind, int party, const cs_honk_arith_polys* dp, size_t round_size,
                  const uint64_t* d_beta_products, size_t periodicity, const cs_rep3_prf* prf, uint64_t* h_r0, uint64_t* h_r1) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HR;
  const size_t n_edges = round_size / 2;
  const unsigned blocks = ceil_div(n_edges, 128);
  ScArithPolys p;
  const uint64_t* const src[13] = {dp->w_l, dp->w_r, dp->w_o, dp->w_4, dp->w_l_shift, dp->w_4_shift, dp->q_m,
                                   dp->q_l, dp->q_r, dp->q_o, dp->q_4, dp->q_c, dp->q_arith};
  const uint32_t** dst[13] = {&p.w_l, &p.w_r, &p.w_o, &p.w_4, &p.w_l_shift, &p.w_4_shift, &p.q_m,
                              &p.q_l, &p.q_r, &p.q_o, &p.q_4, &p.q_c, &p.q_arith};
  for (int k = 0; k < 13; k++) {
    if (!src[k]) return fail(CS_ERR_ARG, "cs_sumcheck_arith_round: polynomial %d is NULL", k);
    *dst[k] = reinterpret_cast<const uint32_t*>(src[k]);
  }
  // -1/2 in Montgomery form
  HR two = HR::one() + HR::one();
  HR nh = HR::zero() - two.inverse();
  Fp<FrP> neg_half;
  memcpy(neg_half.l, nh.l, sizeof(neg_half.l));
  DevBuf& part = ctx->sc_part;  // grown once, reused by every round (no cudaMalloc / cudaFree on the per-round path)
  DevBuf& res = ctx->sc_res;
  CS_TRY(part.reserve((size_t)blocks * SC_SLOTS * 32));
  CS_TRY(res.reserve((size_t)SC_SLOTS * 32));
  auto done = [&](int r) { return r; };
  if (kind == CS_REP3)
    CS_LAUNCH_SYNC((k_sc_arith_round<FrP, true>), blocks, 128, 0, ctx->stream, p, n_edges,
                   reinterpret_cast<const uint32_t*>(d_beta_products), periodicity, party, neg_half, part.as<uint32_t>());
  else
    CS_LAUNCH_SYNC((k_sc_arith_round<FrP, false>), blocks, 128, 0, ctx->stream, p, n_edges,
                   reinterpret_cast<const uint32_t*>(d_beta_products), periodicity, party, neg_half, part.as<uint32_t>());
  CS_LAUNCH_SYNC(k_sc_sum_partials<FrP>, SC_SLOTS, 256, 0, ctx->stream, part.as<uint32_t>(), (size_t)blocks, res.as<uint32_t>());
  uint64_t host[SC_SLOTS * 4];
  cudaError_t e = cudaMemcpyAsync(host, res.p, sizeof(host), cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) return done(fail(CS_ERR_CUDA, "cs_sumcheck_arith_round: %s", cudaGetErrorString(e)));
  for (int k = 0; k < SC_R0_LEN; k++) {
    HR v;
    memcpy(v.l, host + 4 * k, 32);
    if (kind == CS_REP3 && prf) {
      // one fresh zero share per evaluation: masking_field_element = PRF1 - PRF2 (rngs.rs:137-146); the three
      // parties' masks cancel, so the opened univariate is the plain one
      HostChaCha c1, c2;
      c1.init(prf->seed1, prf->word_pos1 + 8 * (uint64_t)k);
      c2.init(prf->seed2, prf->word_pos2 + 8 * (uint64_t)k);
      v = v + (c1.fr_be_mod_order<FrP>() - c2.fr_be_mod_order<FrP>());
    }
    memcpy(h_r0 + 4 * k, v.l, 32);
  }
  const int rc1 = kind == CS_REP3 ? 2 : 1;
  for (int k = 0; k < SC_R1_LEN; k++)
    for (int c = 0; c < rc1; c++) memcpy(h_r1 + 4 * (rc1 * k + c), host + 4 * (SC_R0_LEN + 2 * k + c), 32);
  return done(0);
}

}  // namespace

extern "C" {

int cs_sumcheck_gate_separator(cs_ctx* ctx, cs_curve curve, const uint64_t* h_betas_mont, unsigned log_n, uint64_t* d_out) {
  if (!ctx || !d_out || (log_n && !h_betas_mont)) return fail(CS_ERR_ARG, "cs_sumcheck_gate_separator: NULL argument");
  if (log_n > 30) return fail(CS_ERR_LIMIT, "cs_sumcheck_gate_separator: log_n = %u too large", log_n);
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_DISPATCH_CURVE(curve, return gate_separator_t<Cfg>(ctx, h_betas_mont, log_n, d_out));
  return 0;
}

int cs_sumcheck_fold(cs_ctx* ctx, cs_curve curve, const uint64_t* const* d_in, uint64_t* const* d_out, size_t n_polys, int shared,
                     size_t len, const uint64_t* h_challenge_mont) {
  if (!ctx || !h_challenge_mont || (n_polys && (!d_in || !d_out))) return fail(CS_ERR_ARG, "cs_sumcheck_fold: NULL argument");
  if (len < 2 || (len & 1)) return fail(CS_ERR_ARG, "cs_sumcheck_fold: the length must be even and >= 2 (got %zu)", len);
  for (size_t k = 0; k < n_polys; k++) {
    if (!d_in[k] || !d_out[k]) return fail(CS_ERR_ARG, "cs_sumcheck_fold: polynomial %zu is NULL", k);
    if (d_in[k] == d_out[k]) return fail(CS_ERR_ARG, "cs_sumcheck_fold: polynomial %zu: the output may not alias the input", k);
  }
  if (n_polys == 0) return 0;
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_DISPATCH_CURVE(curve, return fold_t<Cfg>(ctx, d_in, d_out, n_polys, shared, len, h_challenge_mont));
  return 0;
}

int cs_sumcheck_arith_round(cs_ctx* ctx, cs_curve curve, cs_share_kind kind, int party, const cs_honk_arith_polys* d_polys,
                            size_t round_size, const uint64_t* d_beta_products, size_t periodicity, const cs_rep3_prf* prf,
                            uint64_t* h_r0, uint64_t* h_r1) {
  if (!ctx || !d_polys || !d_beta_products || !h_r0 || !h_r1) return fail(CS_ERR_ARG, "cs_sumcheck_arith_round: NULL argument");
  if (kind != CS_PLAIN && kind != CS_REP3) return fail(CS_ERR_ARG, "cs_sumcheck_arith_round: bad share kind %d", (int)kind);
  if (kind == CS_REP3 && (party < 0 || party > 2)) return fail(CS_ERR_ARG, "cs_sumcheck_arith_round: bad party id %d", party);
  if (round_size < 2 || (round_size & 1)) return fail(CS_ERR_ARG, "cs_sumcheck_arith_round: the round size must be even and >= 2");
  if (periodicity == 0) return fail(CS_ERR_ARG, "cs_sumcheck_arith_round: periodicity is 0");
  if (prf && (prf->rounds == 0 || (prf->rounds & 1) || prf->rounds > 20)) return fail(CS_ERR_ARG, "cs_sumcheck_arith_round: bad PRF rounds");
  if (prf && prf->rounds != 12) return fail(CS_ERR_ARG, "cs_sumcheck_arith_round: the host mask path implements ChaCha12 only");
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_DISPATCH_CURVE(curve, return arith_round_t<Cfg>(ctx, kind, party, d_polys, round_size, d_beta_products, periodicity, prf, h_r0, h_r1));
  return 0;
}

}  // extern "C"
