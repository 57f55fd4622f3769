// Plonk prover (plain driver) on the device: co-plonk's five rounds with a device-resident proving key.
//
// Mirrors co-circom/co-plonk/src/lib.rs:80-115 (prove_inner) and round1.rs .. round5.rs for
// PlainPlonkDriver (mpc/plain.rs); the Keccak-256 transcript (types.rs:140-190) and the handful of scalar
// formulas of round 5 run on the host, every vector stays in HBM between the witness upload and the nine
// commitments.  Orderings: an inverse NTT leaves coefficients in bit-reversed order; the 4n-point evaluation
// consumes exactly that order spread at stride 4 (bitrev_4n(j) = 4 bitrev_n(j) for j < n), so only the
// coefficient vectors that are committed / evaluated are permuted back.
#include <algorithm>
#include <chrono>
#include "cs_lib.cuh"
#include "cs_net.h"
#include "cs_plonk.cuh"
#include "cs_plonk_rep3.cuh"
#include "cs_shamir.cuh"

using namespace cs;

namespace cs {
template <class Cfg>
int eval_poly_t(cs_ctx* ctx, const uint64_t* d_coeffs, size_t n, unsigned batch, const uint64_t* h_point, uint64_t* h_out);
}

namespace {

// One prover's per-proof device workspace, reserved once: the plain prover's in the key, each party's in its session.
// w, buf, poly and ev hold `comps` field elements per entry (1: values or Shamir shares, 2: Rep3 share pairs); the
// quotient and opening vectors t .. tmp1 hold one.
struct PlonkWork {
  DevBuf w, buf[3], poly[4], ev[4], t, tz, t1, t2, t3, tmp0, tmp1, totals, small;

  int reserve(size_t n, size_t n_vars, size_t comps) {
    CS_TRY(w.reserve(n_vars * comps * 32));
    for (DevBuf& b : buf) CS_TRY(b.reserve(n * comps * 32));
    for (int i = 0; i < 4; i++) {
      CS_TRY(poly[i].reserve((n + 8) * comps * 32));
      CS_TRY(ev[i].reserve(4 * n * comps * 32));
    }
    CS_TRY(t.reserve(4 * n * 32));
    CS_TRY(tz.reserve(4 * n * 32));
    for (DevBuf* b : {&t1, &t2, &t3, &tmp0, &tmp1}) CS_TRY(b->reserve((n + 8) * 32));
    return small.reserve(8192);  // divide_by_linear's table, then r3_batch_inverse's inverse at 4 KB
  }
  std::vector<const DevBuf*> all() const {
    return {&w, &buf[0], &buf[1], &buf[2], &poly[0], &poly[1], &poly[2], &poly[3], &ev[0], &ev[1], &ev[2], &ev[3],
            &t, &tz, &t1, &t2, &t3, &tmp0, &tmp1, &totals, &small};
  }
  void release() {
    for (const DevBuf* b : all()) const_cast<DevBuf*>(b)->release();
  }
  size_t bytes() const {
    size_t s = 0;
    for (const DevBuf* b : all()) s += b->cap;
    return s;
  }
};

}  // namespace

struct cs_plonk_pk {
  int curve = 0;
  uint32_t n_vars = 0, n_public = 0, n = 0, n_additions = 0, n_constraints = 0, nlag = 0;
  unsigned log_n = 0;
  std::vector<uint64_t> k1, k2, vk_points;  // Montgomery
  cs_bases* p_tau = nullptr;
  cs_domain *dom = nullptr, *dom4 = nullptr;
  DevBuf add_ids, add_factors, add_order;
  std::vector<uint32_t> level_ends;  // additions sorted by dependency level
  DevBuf map_a, map_b, map_c;
  DevBuf q_coeffs[5], q_evals[5], s_coeffs[3], s_evals[3], lagrange;
  PlonkWork ws;  // the plain prover's

  uint32_t n_witness() const { return n_vars - n_additions - n_public - 1; }  // private inputs: no leading one, no additions
};

namespace {

// ---- Keccak-256 (sha3::Keccak256: original 0x01 padding) and the transcript of types.rs:140-190 -------
void keccak_f(uint64_t s[25]) {
  static const uint64_t RC[24] = {
      0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808AULL, 0x8000000080008000ULL, 0x000000000000808BULL,
      0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL, 0x000000000000008AULL, 0x0000000000000088ULL,
      0x0000000080008009ULL, 0x000000008000000AULL, 0x000000008000808BULL, 0x800000000000008BULL, 0x8000000000008089ULL,
      0x8000000000008003ULL, 0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800AULL, 0x800000008000000AULL,
      0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};
  static const int ROT[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};
  auto rol = [](uint64_t x, int n) { return n ? (x << n) | (x >> (64 - n)) : x; };
  for (int round = 0; round < 24; round++) {
    uint64_t C[5], D[5], B[25];
    for (int x = 0; x < 5; x++) C[x] = s[x] ^ s[x + 5] ^ s[x + 10] ^ s[x + 15] ^ s[x + 20];
    for (int x = 0; x < 5; x++) D[x] = C[(x + 4) % 5] ^ rol(C[(x + 1) % 5], 1);
    for (int i = 0; i < 25; i++) s[i] ^= D[i % 5];
    for (int x = 0; x < 5; x++)
      for (int y = 0; y < 5; y++) B[y + 5 * ((2 * x + 3 * y) % 5)] = rol(s[x + 5 * y], ROT[x + 5 * y]);
    for (int x = 0; x < 5; x++)
      for (int y = 0; y < 5; y++) s[x + 5 * y] = B[x + 5 * y] ^ ((~B[(x + 1) % 5 + 5 * y]) & B[(x + 2) % 5 + 5 * y]);
    s[0] ^= RC[round];
  }
}

void keccak256(const std::vector<uint8_t>& data, uint8_t out[32]) {
  const size_t rate = 136;
  std::vector<uint8_t> msg(data);
  msg.push_back(0x01);
  while (msg.size() % rate) msg.push_back(0);
  msg.back() |= 0x80;
  uint64_t s[25];
  memset(s, 0, sizeof(s));
  for (size_t off = 0; off < msg.size(); off += rate) {
    for (size_t i = 0; i < rate / 8; i++) {
      uint64_t v = 0;
      for (int b = 0; b < 8; b++) v |= (uint64_t)msg[off + 8 * i + b] << (8 * b);
      s[i] ^= v;
    }
    keccak_f(s);
  }
  for (int i = 0; i < 4; i++)
    for (int b = 0; b < 8; b++) out[8 * i + b] = (uint8_t)(s[i] >> (8 * b));
}

template <class Cfg>
struct Transcript {
  typedef host::HFp<typename Cfg::FrP> HR;
  typedef host::HFp<typename Cfg::FqP> HQ;
  std::vector<uint8_t> buf;
  template <class H>
  void put_be(const H& canonical) {  // fixed-width big-endian
    for (int i = H::N - 1; i >= 0; i--)
      for (int b = 7; b >= 0; b--) buf.push_back((uint8_t)(canonical.l[i] >> (8 * b)));
  }
  void add_scalar(const HR& mont) { put_be(mont.from_mont()); }
  void add_point(const uint64_t* affine_mont) {  // (0, 0) = infinity -> 2 * byte_len zero bytes (types.rs:168-176)
    HQ x, y;
    memcpy(x.l, affine_mont, sizeof(x.l));
    memcpy(y.l, affine_mont + HQ::N, sizeof(y.l));
    put_be(x.from_mont());
    put_be(y.from_mont());
  }
  HR get_challenge() {  // from_be_bytes_mod_order of the 32-byte digest
    uint8_t d[32];
    keccak256(buf, d);
    HR v = HR::zero();
    for (int i = 0; i < 32; i++) v.l[(31 - i) / 8] |= (uint64_t)d[i] << (8 * ((31 - i) % 8));
    // v < 2^256 is unreduced; r2 * v keeps the CIOS rows in range and lands in [0, r) as v R mod r
    return HR::r2() * v;
  }
};

int upload(cs_ctx* ctx, DevBuf& buf, const void* src, size_t bytes) {
  CS_TRY(buf.reserve(bytes ? bytes : 4));
  if (bytes) CS_CUDA(cudaMemcpyAsync(buf.p, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return 0;
}

template <class HR>
void put(uint32_t* dst, const HR& v) { memcpy(dst, v.l, sizeof(v.l)); }

// scratch: the workspace's `totals`
template <class FrP, int OP>
int scan(cs_ctx* ctx, PlonkWork& ws, const uint32_t* in, uint32_t* out, uint32_t n, int rev) {
  const uint32_t nb = ceil_div(n, SCAN_TILE);
  CS_TRY(ws.totals.reserve((size_t)nb * 32));
  uint32_t* totals = ws.totals.as<uint32_t>();
  CS_LAUNCH_SYNC(k_scan_block<FrP COMMA OP>, nb, SCAN_THREADS, (size_t)SCAN_THREADS * 32, ctx->stream, in, out, n, rev, totals);
  if (nb > 1) {
    CS_LAUNCH_SYNC(k_scan_totals<FrP COMMA OP>, 1, 256, (size_t)256 * 32, ctx->stream, totals, nb);
    CS_LAUNCH(k_scan_apply<FrP COMMA OP>, ceil_div(n, 256), 256, 0, ctx->stream, out, n, rev, totals);
  }
  CS_CUDA(cudaGetLastError());
  return 0;
}

template <class FrP>
CS_GLOBAL void k_spread4(const uint32_t* __restrict__ in, uint32_t n, uint32_t batch, uint32_t* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;  // over 4n outputs
  if (i >= 4 * n) return;
  for (uint32_t c = 0; c < batch; c++) {
    Fp<FrP> v = Fp<FrP>::zero();
    if ((i & 3) == 0) v = ld_fr<FrP>(in + ((size_t)(i >> 2) * batch + c) * FrP::N);
    st_fr<FrP>(out + ((size_t)i * batch + c) * FrP::N, v);
  }
}

// evaluations (natural order, n points) -> coefficients: `poly` natural order, and -- when ev4 != NULL -- the
// 4n-point evaluations of the same (unblinded) polynomial, without permuting in between.
template <class Cfg>
int interpolate_and_extend(cs_ctx* ctx, cs_plonk_pk* pk, uint32_t* poly, uint32_t* ev4, unsigned batch = 1) {
  typedef typename Cfg::FrP FrP;
  const uint32_t n = pk->n;
  CS_TRY(ntt_run(ctx, pk->dom, poly, batch, true, nullptr, ctx->stream));  // bit-reversed coefficients
  if (ev4) {
    CS_LAUNCH(k_spread4<FrP>, ceil_div((size_t)4 * n, 256), 256, 0, ctx->stream, poly, n, batch, ev4);
    CS_TRY(ntt_run(ctx, pk->dom4, ev4, batch, false, nullptr, ctx->stream));
  }
  CS_LAUNCH(k_bit_reverse<FrP>, ceil_div(n, 256), 256, 0, ctx->stream, poly, pk->log_n, batch);
  CS_CUDA(cudaGetLastError());
  return 0;
}

// b: `count` blinders of `batch` components each (component-major per blinder: b[i * batch + c])
template <class Cfg>
int blind(cs_ctx* ctx, uint32_t* poly, uint32_t n, const host::HFp<typename Cfg::FrP>* b, int count, unsigned batch = 1) {
  PlonkBlind rev;
  memset(&rev, 0, sizeof(rev));
  for (int i = 0; i < count; i++)
    for (unsigned c = 0; c < batch; c++) put(rev.v[i * batch + c], b[(count - 1 - i) * batch + c]);
  CS_LAUNCH(k_plonk_blind<typename Cfg::FrP>, 1, 32, 0, ctx->stream, poly, n, batch, rev, (uint32_t)count);
  return 0;
}

struct Commit { const uint32_t* d_scalars; size_t len; uint64_t* out; };
// msm_public_points_g1 over p_tau[..len] for up to CS_NSIDE polynomials at once, one stream each
template <class Cfg>
int commit_many(cs_ctx* ctx, cs_plonk_pk* pk, const Commit* c, int k) {
  if (k > CS_NSIDE) return fail(CS_ERR_ARG, "commit_many: too many polynomials");
  CS_TRY(ctx_fork(ctx, k));
  for (int i = 0; i < k; i++) {
    if (c[i].len > pk->p_tau->n) return fail(CS_ERR_ARG, "Polynomial Degree too large: %zu coefficients, %zu SRS points", c[i].len, pk->p_tau->n);
    CS_TRY(msm_enqueue_dyn(ctx, i, ctx->side[i], pk->p_tau, 0, c[i].d_scalars, 1, c[i].len, 1));
  }
  CS_TRY(ctx_join(ctx, k));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < k; i++) CS_TRY(msm_finish_dyn(ctx, i, pk->p_tau, c[i].out, nullptr));
  return 0;
}

template <class Cfg>
int plonk_pk_create_t(cs_ctx* ctx, const cs_plonk_key_desc* d, cs_plonk_pk* pk) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HR;
  const uint32_t n = d->domain_size;
  if (n == 0 || (n & (n - 1))) return fail(CS_ERR_ARG, "Invalid domain size %u", n);  // types.rs:79-81
  unsigned lg = 0;
  while ((1u << lg) < n) lg++;
  if (lg + 2 > Cfg::TWO_ADICITY) return fail(CS_ERR_ARG, "Polynomial Degree too large");
  if (d->n_p_tau < (size_t)n + 6) return fail(CS_ERR_ARG, "cs_plonk_pk_create: %zu SRS points, need domain_size + 6", d->n_p_tau);
  if (d->n_constraints > n) return fail(CS_ERR_ARG, "cs_plonk_pk_create: more constraints than the domain holds");
  if (d->n_vars < d->n_public + 1 + d->n_additions) return fail(CS_ERR_ARG, "cs_plonk_pk_create: inconsistent variable counts");
  pk->n_vars = d->n_vars; pk->n_public = d->n_public; pk->n = n; pk->n_additions = d->n_additions;
  pk->n_constraints = d->n_constraints; pk->log_n = lg;
  pk->nlag = d->n_public ? d->n_public : 1;
  pk->k1.assign(d->k1_mont, d->k1_mont + HR::N);
  pk->k2.assign(d->k2_mont, d->k2_mont + HR::N);
  const size_t pl = point_limbs64(pk->curve, CS_G1);
  pk->vk_points.assign(d->vk_points, d->vk_points + 8 * pl);
  // snarkjs roots: domain n uses roots[pow], the extended domain roots[pow + 2] (types.rs:94-100)
  uint64_t gen[HR::N], shift[HR::N];
  CS_TRY(cs_groth16_roots_of_unity((cs_curve)pk->curve, lg, gen, shift));
  CS_TRY(cs_domain_create(ctx, (cs_curve)pk->curve, lg, gen, &pk->dom));
  CS_TRY(cs_groth16_roots_of_unity((cs_curve)pk->curve, lg + 2, gen, shift));
  CS_TRY(cs_domain_create(ctx, (cs_curve)pk->curve, lg + 2, gen, &pk->dom4));
  CS_TRY(cs_bases_upload(ctx, (cs_curve)pk->curve, CS_G1, d->p_tau, d->n_p_tau, 0, &pk->p_tau));
  // additions: dependency levels (an addition may read earlier additions, round1.rs:191-224)
  const uint32_t na = d->n_additions, first_add = d->n_vars - na;
  std::vector<uint32_t> level(na, 0);
  uint32_t maxl = 0;
  for (uint32_t k = 0; k < na; k++) {
    uint32_t l = 0;
    for (int s = 0; s < 2; s++) {
      uint32_t id = d->additions_ids[2 * k + s];
      if (id >= d->n_vars) return fail(CS_ERR_ARG, "Cannot index into witness %u", id);
      if (id >= first_add) {
        if (id - first_add >= k) return fail(CS_ERR_ARG, "cs_plonk_pk_create: addition %u reads a later addition", k);
        l = std::max(l, level[id - first_add] + 1);
      }
    }
    level[k] = l;
    maxl = std::max(maxl, l);
  }
  std::vector<uint32_t> order(na);
  for (uint32_t k = 0; k < na; k++) order[k] = k;
  std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return level[x] < level[y]; });
  pk->level_ends.clear();
  for (uint32_t t = 0; t < na; t++)
    if (t + 1 == na || level[order[t + 1]] != level[order[t]]) pk->level_ends.push_back(t + 1);
  CS_TRY(upload(ctx, pk->add_ids, d->additions_ids, (size_t)na * 8));
  CS_TRY(upload(ctx, pk->add_factors, d->additions_factors, (size_t)na * 64));
  CS_TRY(upload(ctx, pk->add_order, order.data(), (size_t)na * 4));
  for (uint32_t i = 0; i < d->n_constraints; i++)
    if (d->map_a[i] >= d->n_vars || d->map_b[i] >= d->n_vars || d->map_c[i] >= d->n_vars)
      return fail(CS_ERR_ARG, "Cannot index into witness (wire map row %u)", i);
  CS_TRY(upload(ctx, pk->map_a, d->map_a, (size_t)d->n_constraints * 4));
  CS_TRY(upload(ctx, pk->map_b, d->map_b, (size_t)d->n_constraints * 4));
  CS_TRY(upload(ctx, pk->map_c, d->map_c, (size_t)d->n_constraints * 4));
  for (int i = 0; i < 5; i++) {
    CS_TRY(upload(ctx, pk->q_coeffs[i], d->q_coeffs[i], (size_t)n * 32));
    CS_TRY(upload(ctx, pk->q_evals[i], d->q_evals[i], (size_t)4 * n * 32));
  }
  for (int i = 0; i < 3; i++) {
    CS_TRY(upload(ctx, pk->s_coeffs[i], d->s_coeffs[i], (size_t)n * 32));
    CS_TRY(upload(ctx, pk->s_evals[i], d->s_evals[i], (size_t)4 * n * 32));
  }
  CS_TRY(upload(ctx, pk->lagrange, d->lagrange_evals, (size_t)pk->nlag * 4 * n * 32));
  CS_TRY(pk->ws.reserve(n, d->n_vars, 1));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  (void)maxl;
  return 0;
}

// q(X) = p(X) / (X - x) in place over `p` (len entries -> len - 1), optionally subtracting *sub0 from p[0] first
template <class Cfg>
int divide_by_linear(cs_ctx* ctx, PlonkWork& ws, uint32_t* p, uint32_t len, const host::HFp<typename Cfg::FrP>& x,
                     const host::HFp<typename Cfg::FrP>* sub0) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HR;
  if (x.is_zero()) return fail(CS_ERR_ARG, "plonk: evaluation challenge is zero");
  std::vector<HR> tab(2 * 33 + 1);
  HR a = x, b = x.inverse();
  for (int j = 0; j < 33; j++) { tab[j] = a; tab[33 + j] = b; a = a.sqr(); b = b.sqr(); }
  if (sub0) tab[66] = *sub0;
  uint32_t* d_tab = ws.small.as<uint32_t>();
  CS_CUDA(cudaMemcpyAsync(d_tab, tab.data(), tab.size() * sizeof(HR), cudaMemcpyHostToDevice, ctx->stream));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));  // `tab` is a stack-owned vector
  const unsigned blocks = ceil_div(ceil_div(len, 8), 128);
  CS_LAUNCH(k_scale_by_powers<FrP>, blocks, 128, 0, ctx->stream, p, d_tab, 0u, 0, sub0 ? d_tab + 66 * FrP::N : (const uint32_t*)nullptr,
            len, p);
  CS_TRY((scan<FrP, 1>(ctx, ws, p, p, len, 0)));
  CS_LAUNCH(k_scale_by_powers<FrP>, blocks, 128, 0, ctx->stream, p, d_tab + 33 * FrP::N, 1u, 1, (const uint32_t*)nullptr, len - 1, p);
  CS_CUDA(cudaGetLastError());
  return 0;
}

// Z_H weights of the blinding terms on the four cosets of the extended domain (mul4vec_post, round3.rs:20-108), from
// the 4th root of unity roots[2] (types.rs:105)
template <class Cfg>
int quotient_consts(int curve, PlonkConsts& K) {
  typedef host::HFp<typename Cfg::FrP> HR;
  uint64_t g4[HR::N], unused[HR::N];
  CS_TRY(cs_groth16_roots_of_unity((cs_curve)curve, 2, g4, unused));
  HR w4, one = HR::one(), two = one + one, zero = HR::zero();
  memcpy(w4.l, g4, sizeof(w4.l));
  HR z1[4] = {zero, w4 - one, zero - two, zero - one - w4};
  HR z2[4] = {zero, zero - two * w4, two + two, two * w4};
  HR z3[4] = {zero, two + two * w4, zero - (two + two + two + two), two - two * w4};
  for (int i = 0; i < 4; i++) { put(K.z1[i], z1[i]); put(K.z2[i], z2[i]); put(K.z3[i], z3[i]); }
  return 0;
}

template <class Cfg>
host::HFp<typename Cfg::FrP> domain_gen(const cs_plonk_pk* pk) {  // w_n, the generator of the n-point domain
  host::HFp<typename Cfg::FrP> w;
  memcpy(w.l, pk->dom->group_gen.data(), sizeof(w.l));
  return w;
}

// Round 5's scalars (round5.rs:284-340; calculate_lagrange_evaluations / calculate_pi, lib.rs:181-219): the weights of
// the linearisation polynomial's terms.  pub: the key's n_public public inputs without the leading slot; ev: the opened
// eval_a eval_b eval_c eval_s1 eval_s2 eval_zw; beta, gamma, alpha, alpha2, k1, k2 are read from K.
template <class Cfg>
int lin_weights(const cs_plonk_pk* pk, const uint64_t* pub, const PlonkConsts& K, const host::HFp<typename Cfg::FrP>& xi,
                const host::HFp<typename Cfg::FrP>& v0, const host::HFp<typename Cfg::FrP>* ev, PlonkLinW& W) {
  typedef host::HFp<typename Cfg::FrP> HR;
  auto ld = [](const uint32_t* w) { HR x; memcpy(x.l, w, sizeof(x.l)); return x; };
  const HR beta = ld(K.beta), gamma = ld(K.gamma), alpha = ld(K.alpha), alpha2 = ld(K.alpha2), k1 = ld(K.k1), k2 = ld(K.k2);
  const HR ea = ev[0], eb = ev[1], ec = ev[2], es1 = ev[3], es2 = ev[4], ezw = ev[5];
  HR v[5];
  v[0] = v0;
  for (int i = 1; i < 5; i++) v[i] = v[i - 1] * v[0];
  const HR w_n = domain_gen<Cfg>(pk);
  HR xin = xi;
  for (unsigned q = 0; q < pk->log_n; q++) xin = xin.sqr();
  const HR zh = xin - HR::one();
  const HR nn = HR::from_u64(pk->n);
  std::vector<HR> ls(pk->nlag);
  {
    HR wi = HR::one();
    for (uint32_t i = 0; i < pk->nlag; i++) {
      HR dnm = nn * (xi - wi);
      if (dnm.is_zero()) return fail(CS_ERR_ARG, "plonk: xi hit the evaluation domain");
      ls[i] = wi * zh * dnm.inverse();
      wi = wi * w_n;
    }
  }
  HR eval_pi = HR::zero();
  for (uint32_t i = 0; i < pk->n_public && i < pk->nlag; i++) {
    HR val;
    memcpy(val.l, pub + (size_t)i * HR::N, sizeof(val.l));
    eval_pi = eval_pi - ls[i] * val;
  }
  const HR betaxi = beta * xi;
  const HR e2 = (ea + betaxi + gamma) * (eb + betaxi * k1 + gamma) * (ec + betaxi * k2 + gamma) * alpha;
  const HR e3 = (ea + beta * es1 + gamma) * (eb + beta * es2 + gamma) * ezw * alpha;
  const HR e4 = alpha2 * ls[0];
  const HR r0 = eval_pi - e3 * (ec + gamma) - e4;
  memset(&W, 0, sizeof(W));
  put(W.ab, ea * eb); put(W.ea, ea); put(W.eb, eb); put(W.ec, ec); put(W.e3beta, e3 * beta); put(W.e24, e2 + e4);
  put(W.zh, zh); put(W.xin, xin); put(W.xin2, xin.sqr());
  for (int i = 0; i < 5; i++) put(W.v[i], v[i]);
  put(W.c0, r0 - v[0] * ea - v[1] * eb - v[2] * ec - v[3] * es1 - v[4] * es2);
  return 0;
}

// the commitments of p[0..k) (at most three), `len` coefficients each, into k consecutive points at `out`
template <class Cfg>
int commit_polys(cs_ctx* ctx, cs_plonk_pk* pk, const DevBuf* p, int k, size_t len, uint64_t* out) {
  Commit c[3];
  for (int i = 0; i < k; i++) c[i] = Commit{p[i].as<uint32_t>(), len, out + i * point_limbs64(pk->curve, CS_G1)};
  return commit_many<Cfg>(ctx, pk, c, k);
}

// The Fiat-Shamir challenges of rounds 2-5 (round2.rs:226-245, round3.rs:560-610, round4.rs:108-165, round5.rs:284-340),
// each the Keccak hash of its own transcript.  What enters each transcript, and in which order, is the protocol's format.
template <class Cfg>
struct Challenges {
  typedef host::HFp<typename Cfg::FrP> HR;
  static constexpr size_t PL = 2 * host::HFp<typename Cfg::FqP>::N;  // limbs of an affine G1 point
  HR beta, gamma, alpha, xi, v;

  void round2(const cs_plonk_pk* pk, const uint64_t* pub, const uint64_t* abc) {  // pub: with the leading slot
    Transcript<Cfg> t;
    for (int i = 0; i < 8; i++) t.add_point(pk->vk_points.data() + i * PL);
    for (uint32_t i = 1; i <= pk->n_public; i++) {
      HR x;
      memcpy(x.l, pub + (size_t)i * HR::N, sizeof(x.l));
      t.add_scalar(x);
    }
    for (int i = 0; i < 3; i++) t.add_point(abc + i * PL);
    beta = t.get_challenge();
    Transcript<Cfg> tg;
    tg.add_scalar(beta);
    gamma = tg.get_challenge();
  }
  void round3(const uint64_t* z) {
    Transcript<Cfg> t;
    t.add_scalar(beta);
    t.add_scalar(gamma);
    t.add_point(z);
    alpha = t.get_challenge();
  }
  void round4(const uint64_t* t123) {
    Transcript<Cfg> t;
    t.add_scalar(alpha);
    for (int i = 0; i < 3; i++) t.add_point(t123 + i * PL);
    xi = t.get_challenge();
  }
  void round5(const HR* ev) {  // ev: the opened a b c s1 s2 zw
    Transcript<Cfg> t;
    t.add_scalar(xi);
    for (int i = 0; i < 6; i++) t.add_scalar(ev[i]);
    v = t.get_challenge();
  }
};

// Init round (round1.rs:191-252): w = 0 | public inputs | witness | additions, `comps` elements per variable.  The public
// values go into component pub_comp, or nowhere when it is negative (Rep3 promote_to_trivial_share,
// rep3/arithmetic.rs:41-50); the leading one reads as zero (types.rs:118-120).
template <class Cfg>
int load_witness(cs_ctx* ctx, const cs_plonk_pk* pk, PlonkWork& ws, const uint64_t* h_pub, const uint64_t* h_wit,
                 unsigned comps, int pub_comp) {
  typedef typename Cfg::FrP FrP;
  constexpr int NW = FrP::N, N = host::HFp<FrP>::N;
  cudaStream_t st = ctx->stream;
  const uint32_t npub = pk->n_public, n_priv = pk->n_witness();
  uint32_t* w = ws.w.as<uint32_t>();
  std::vector<uint64_t> stage;
  if (comps == 1 && pub_comp == 0) {  // the caller's layout: copy the public inputs as they are
    CS_CUDA(cudaMemsetAsync(w, 0, 32, st));
    if (npub) CS_CUDA(cudaMemcpyAsync(w + NW, h_pub + N, (size_t)npub * 32, cudaMemcpyHostToDevice, st));
  } else {
    stage.assign((size_t)(npub + 1) * comps * N, 0);
    for (uint32_t j = 1; j <= npub && pub_comp >= 0; j++)
      memcpy(&stage[((size_t)j * comps + pub_comp) * N], h_pub + (size_t)j * N, N * 8);
    CS_CUDA(cudaMemcpyAsync(w, stage.data(), stage.size() * 8, cudaMemcpyHostToDevice, st));
  }
  if (n_priv)
    CS_CUDA(cudaMemcpyAsync(w + (size_t)(npub + 1) * comps * NW, h_wit, (size_t)n_priv * comps * 32, cudaMemcpyHostToDevice, st));
  if (!stage.empty()) CS_CUDA(cudaStreamSynchronize(st));  // `stage` is a local vector
  uint32_t lo = 0;
  for (uint32_t hi : pk->level_ends) {
    CS_LAUNCH(k_plonk_additions<FrP>, ceil_div(hi - lo, 128), 128, 0, st, pk->add_order.as<uint32_t>(), lo, hi,
              pk->add_ids.as<uint32_t>(), pk->add_factors.as<uint32_t>(), pk->n_vars - pk->n_additions, (uint32_t)comps, w);
    lo = hi;
  }
  return 0;
}

// Round 1 for wire k (round1.rs:108-189, 255-320): gathered from w into buf[k]; poly[k] = its coefficients blinded by
// b[0], b[1] (`comps` components each, component-major); ev[k] = the 4n-point evaluations of the unblinded polynomial
template <class Cfg>
int wire_poly(cs_ctx* ctx, cs_plonk_pk* pk, PlonkWork& ws, int k, unsigned comps, const host::HFp<typename Cfg::FrP>* b) {
  const uint32_t n = pk->n;
  const DevBuf* maps[3] = {&pk->map_a, &pk->map_b, &pk->map_c};
  uint32_t *buf = ws.buf[k].as<uint32_t>(), *poly = ws.poly[k].as<uint32_t>();
  CS_LAUNCH(k_plonk_gather<typename Cfg::FrP>, ceil_div(n, 256), 256, 0, ctx->stream, maps[k]->as<uint32_t>(), pk->n_constraints,
            n, (uint32_t)comps, ws.w.as<uint32_t>(), buf);
  CS_CUDA(cudaMemcpyAsync(poly, buf, (size_t)n * comps * 32, cudaMemcpyDeviceToDevice, ctx->stream));
  CS_TRY(interpolate_and_extend<Cfg>(ctx, pk, poly, ws.ev[k].as<uint32_t>(), comps));
  return blind<Cfg>(ctx, poly, n, b, 2, comps);
}

// Z from its n values in poly[3] (round2.rs:197-250): coefficients blinded by b[0..3), and ev[3] = the 4n-point
// evaluations of the unblinded polynomial
template <class Cfg>
int z_poly(cs_ctx* ctx, cs_plonk_pk* pk, PlonkWork& ws, unsigned comps, const host::HFp<typename Cfg::FrP>* b) {
  CS_TRY(interpolate_and_extend<Cfg>(ctx, pk, ws.poly[3].as<uint32_t>(), ws.ev[3].as<uint32_t>(), comps));
  return blind<Cfg>(ctx, ws.poly[3].as<uint32_t>(), pk->n, b, 3, comps);
}

// K before the challenges: the eleven blinders b[0], b[stride], .. (a Rep3 pair's additive half at stride 2), k1, k2
template <class Cfg>
void init_consts(PlonkConsts& K, const cs_plonk_pk* pk, const host::HFp<typename Cfg::FrP>* b, int stride) {
  memset(&K, 0, sizeof(K));
  for (int i = 0; i < 11; i++) put(K.b[i], b[stride * i]);
  memcpy(K.k1, pk->k1.data(), sizeof(K.k1));
  memcpy(K.k2, pk->k2.data(), sizeof(K.k2));
}

template <class Cfg>
int set_alpha(const cs_plonk_pk* pk, PlonkConsts& K, const host::HFp<typename Cfg::FrP>& alpha) {
  put(K.alpha, alpha);
  put(K.alpha2, alpha.sqr());
  return quotient_consts<Cfg>(pk->curve, K);
}

// the round kernels' views of the key and the workspace
R3Round2In r3_round2_in(const cs_plonk_pk* pk, const PlonkWork& ws) {
  return R3Round2In{ws.buf[0].as<uint32_t>(),     ws.buf[1].as<uint32_t>(),     ws.buf[2].as<uint32_t>(),
                    pk->s_evals[0].as<uint32_t>(), pk->s_evals[1].as<uint32_t>(), pk->s_evals[2].as<uint32_t>(),
                    pk->dom4->tw_fwd.as<uint32_t>()};
}
R3QuotIn r3_quot_in(const cs_plonk_pk* pk, const PlonkWork& ws) {
  return R3QuotIn{ws.ev[0].as<uint32_t>(), ws.ev[1].as<uint32_t>(), ws.ev[2].as<uint32_t>(), ws.ev[3].as<uint32_t>(),
                  pk->dom4->tw_fwd.as<uint32_t>()};
}
R3KeyEvals key_evals(const cs_plonk_pk* pk, const PlonkWork& ws) {
  const DevBuf *q = pk->q_evals, *s = pk->s_evals;
  return R3KeyEvals{q[0].as<uint32_t>(), q[1].as<uint32_t>(), q[2].as<uint32_t>(), q[3].as<uint32_t>(),
                    q[4].as<uint32_t>(), s[0].as<uint32_t>(), s[1].as<uint32_t>(), s[2].as<uint32_t>(),
                    pk->lagrange.as<uint32_t>(), ws.buf[0].as<uint32_t>()};
}

// Round 3's tail (round3.rs:560-610): t and tz from 4n evaluations to coefficients, split into T1 T2 T3, committed into
// three points at `out`
template <class Cfg>
int split_and_commit(cs_ctx* ctx, cs_plonk_pk* pk, PlonkWork& ws, const PlonkConsts& K, uint64_t* out) {
  typedef typename Cfg::FrP FrP;
  cudaStream_t st = ctx->stream;
  const uint32_t n = pk->n, n4 = 4 * n;
  const size_t pl = point_limbs64(pk->curve, CS_G1);
  uint32_t *t = ws.t.as<uint32_t>(), *tz = ws.tz.as<uint32_t>();
  uint32_t *t1 = ws.t1.as<uint32_t>(), *t2 = ws.t2.as<uint32_t>(), *t3 = ws.t3.as<uint32_t>();
  CS_TRY(ntt_run(ctx, pk->dom4, t, 1, true, nullptr, st));
  CS_TRY(ntt_run(ctx, pk->dom4, tz, 1, true, nullptr, st));
  CS_LAUNCH(k_bit_reverse<FrP>, ceil_div(n4, 256), 256, 0, st, t, pk->log_n + 2, 1u);
  CS_LAUNCH(k_bit_reverse<FrP>, ceil_div(n4, 256), 256, 0, st, tz, pk->log_n + 2, 1u);
  CS_LAUNCH(k_plonk_tsplit<FrP>, ceil_div(n, 128), 128, 0, st, t, tz, n, K, t1, t2, t3);
  Commit c[3] = {{t1, (size_t)n + 1, out}, {t2, (size_t)n + 1, out + pl}, {t3, (size_t)n + 6, out + 2 * pl}};
  return commit_many<Cfg>(ctx, pk, c, 3);
}

// Round 4 (round4.rs:108-165): out = a b c at xi, z at xi w, s1 s2 at xi.  p: the coefficients of a b c z
template <class Cfg>
int evaluate(cs_ctx* ctx, const cs_plonk_pk* pk, const DevBuf* p, const host::HFp<typename Cfg::FrP>& xi, uint64_t* out) {
  typedef host::HFp<typename Cfg::FrP> HR;
  const size_t n = pk->n;
  const HR xiw = xi * domain_gen<Cfg>(pk);
  for (int k = 0; k < 3; k++) CS_TRY((eval_poly_t<Cfg>(ctx, p[k].as<uint64_t>(), n + 2, 1, xi.l, out + k * HR::N)));
  CS_TRY((eval_poly_t<Cfg>(ctx, p[3].as<uint64_t>(), n + 3, 1, xiw.l, out + 3 * HR::N)));
  CS_TRY((eval_poly_t<Cfg>(ctx, pk->s_coeffs[0].as<uint64_t>(), n, 1, xi.l, out + 4 * HR::N)));
  return eval_poly_t<Cfg>(ctx, pk->s_coeffs[1].as<uint64_t>(), n, 1, xi.l, out + 5 * HR::N);
}

// Round 5 (round5.rs:284-340): Wxi = (linearisation numerator) / (X - xi) and Wxiw = (z - eval_zw) / (X - xi w),
// committed into two points at `out`.  p: the coefficients of a b c z; pub: the public inputs after the leading slot;
// ev: the opened a b c s1 s2 zw.  pub_terms = 0 leaves out the public polynomials, the constants and eval_zw, which
// enter at one party only when the shares are additive (add_with_public on x_0).
template <class Cfg>
int opening_polys(cs_ctx* ctx, cs_plonk_pk* pk, PlonkWork& ws, const DevBuf* p, const uint64_t* pub, const PlonkConsts& K,
                  const host::HFp<typename Cfg::FrP>& xi, const host::HFp<typename Cfg::FrP>& v,
                  const host::HFp<typename Cfg::FrP>* ev, int pub_terms, uint64_t* out) {
  typedef typename Cfg::FrP FrP;
  const uint32_t n = pk->n;
  const size_t pl = point_limbs64(pk->curve, CS_G1);
  PlonkLinW W;
  CS_TRY(lin_weights<Cfg>(pk, pub, K, xi, v, ev, W));
  const DevBuf *q = pk->q_coeffs, *s = pk->s_coeffs;
  const PlonkLinIn li{q[0].as<uint32_t>(),  q[1].as<uint32_t>(),  q[2].as<uint32_t>(),  q[3].as<uint32_t>(),
                      q[4].as<uint32_t>(),  s[0].as<uint32_t>(),  s[1].as<uint32_t>(),  s[2].as<uint32_t>(),
                      p[0].as<uint32_t>(),  p[1].as<uint32_t>(),  p[2].as<uint32_t>(),  p[3].as<uint32_t>(),
                      ws.t1.as<uint32_t>(), ws.t2.as<uint32_t>(), ws.t3.as<uint32_t>()};
  uint32_t *wxi = ws.tmp0.as<uint32_t>(), *wxiw = ws.tmp1.as<uint32_t>();
  CS_LAUNCH(k_plonk_wxi_numerator<FrP>, ceil_div(n + 6, 128), 128, 0, ctx->stream, li, W, n, pub_terms, wxi);
  CS_TRY(divide_by_linear<Cfg>(ctx, ws, wxi, n + 6, xi, nullptr));
  CS_CUDA(cudaMemcpyAsync(wxiw, p[3].as<uint32_t>(), (size_t)(n + 3) * 32, cudaMemcpyDeviceToDevice, ctx->stream));
  CS_TRY(divide_by_linear<Cfg>(ctx, ws, wxiw, n + 3, xi * domain_gen<Cfg>(pk), pub_terms ? &ev[5] : nullptr));
  Commit c[2] = {{wxi, (size_t)n + 5, out}, {wxiw, (size_t)n + 2, out + pl}};
  return commit_many<Cfg>(ctx, pk, c, 2);
}

template <class Cfg>
int plonk_prove_plain_t(cs_ctx* ctx, cs_plonk_pk* pk, const uint64_t* h_pub, const uint64_t* h_wit, const uint64_t* h_blind,
                        uint64_t* out_points, uint64_t* out_evals) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HR;
  constexpr int NW = FrP::N;
  PlonkWork& ws = pk->ws;
  const uint32_t n = pk->n;
  const size_t pl = point_limbs64(pk->curve, CS_G1);
  cudaStream_t st = ctx->stream;
  CS_CUDA(cudaSetDevice(ctx->device));
  HR b[11];
  memcpy(b, h_blind, sizeof(b));
  uint64_t* P = out_points;  // A B C Z T1 T2 T3 Wxi Wxiw
  // ---- init round, round 1
  CS_TRY(load_witness<Cfg>(ctx, pk, ws, h_pub, h_wit, 1, 0));
  for (int k = 0; k < 3; k++) CS_TRY(wire_poly<Cfg>(ctx, pk, ws, k, 1, b + 2 * k));
  CS_TRY(commit_polys<Cfg>(ctx, pk, ws.poly, 3, (size_t)n + 2, P));
  // ---- round 2 (round2.rs:197-250)
  Challenges<Cfg> ch;
  ch.round2(pk, h_pub, P);
  PlonkConsts K;
  init_consts<Cfg>(K, pk, b, 1);
  put(K.beta, ch.beta);
  put(K.gamma, ch.gamma);
  uint32_t *num = ws.t.as<uint32_t>(), *den = num + (size_t)n * NW, *sden = den + (size_t)n * NW;  // scratch inside t (4n)
  const R3Round2In in = r3_round2_in(pk, ws);
  CS_LAUNCH(k_plonk_numden<FrP>, ceil_div(n, 128), 128, 0, st, in.a, in.b, in.c, in.s1, in.s2, in.s3, in.tw4, n, K, num, den);
  CS_TRY((scan<FrP, 0>(ctx, ws, num, num, n, 0)));    // running products of the numerators (in place)
  CS_TRY((scan<FrP, 0>(ctx, ws, den, sden, n, 1)));   // suffix products of the denominators
  HR total;
  CS_CUDA(cudaMemcpyAsync(total.l, sden, sizeof(total.l), cudaMemcpyDeviceToHost, st));
  CS_CUDA(cudaStreamSynchronize(st));
  if (total.is_zero()) return fail(CS_ERR_ARG, "Cannot invert zero");  // mpc/plain.rs:206-208
  HR inv_total = total.inverse();
  uint32_t* d_small = ws.small.as<uint32_t>();
  CS_CUDA(cudaMemcpyAsync(d_small, inv_total.l, sizeof(inv_total.l), cudaMemcpyHostToDevice, st));
  CS_LAUNCH(k_plonk_zbuf<FrP>, ceil_div(n, 128), 128, 0, st, num, sden, d_small, n, ws.poly[3].as<uint32_t>());
  CS_CUDA(cudaStreamSynchronize(st));  // inv_total is a stack variable
  CS_TRY(z_poly<Cfg>(ctx, pk, ws, 1, b + 6));
  CS_TRY(commit_polys<Cfg>(ctx, pk, ws.poly + 3, 1, (size_t)n + 3, P + 3 * pl));
  // ---- round 3 (round3.rs:560-610)
  ch.round3(P + 3 * pl);
  CS_TRY(set_alpha<Cfg>(pk, K, ch.alpha));
  const R3QuotIn q = r3_quot_in(pk, ws);
  const R3KeyEvals E = key_evals(pk, ws);
  const PlonkQuotIn qi{q.a, q.b, q.c, q.z, E.qm, E.ql, E.qr, E.qo, E.qc, E.s1, E.s2, E.s3, E.lagrange, E.buf_a, q.tw4};
  CS_LAUNCH(k_plonk_quotient<FrP>, ceil_div(4 * n, 128), 128, 0, st, qi, n, pk->nlag, K, ws.t.as<uint32_t>(), ws.tz.as<uint32_t>());
  CS_TRY(split_and_commit<Cfg>(ctx, pk, ws, K, P + 4 * pl));
  // ---- round 4
  ch.round4(P + 4 * pl);
  HR e[6];  // a b c zw s1 s2
  CS_TRY(evaluate<Cfg>(ctx, pk, ws.poly, ch.xi, e[0].l));
  // ---- round 5
  const HR ev[6] = {e[0], e[1], e[2], e[4], e[5], e[3]};  // the proof's order: a b c s1 s2 zw
  ch.round5(ev);
  CS_TRY(opening_polys<Cfg>(ctx, pk, ws, ws.poly, h_pub + HR::N, K, ch.xi, ch.v, ev, 1, P + 7 * pl));
  memcpy(out_evals, ev, sizeof(ev));
  return 0;
}


// ======================================================================================================
// Rep3 co-Plonk: one session per party (Rep3CoPlonk::prove, co-plonk/src/lib.rs:222-240 with
// Rep3PlonkDriver, mpc/rep3.rs).  The session owns the party's share vectors and the arena that the next
// party's products are stored into; the host driver (co_snarks_b200/plonk.py) sequences the steps, opens the
// partial commitments / evaluations / masked vectors and hashes the transcript.  See cs_plonk_rep3.cuh.
// ======================================================================================================
}  // namespace

struct cs_plonk_rep3 {
  cs_ctx* ctx = nullptr;
  cs_plonk_pk* pk = nullptr;
  int party = 0;
  PlonkWork ws;       // w, buf, poly and ev hold share pairs
  DevBuf polyadd[4];  // component 0 of a b c z: this party's additive share, what it commits and evaluates
  DevBuf arena, addv, pubv;
  uint32_t* next_arena = nullptr;
  const uint32_t* peer_out[2] = {nullptr, nullptr};  // previous / next party's additive-out vector (cs_plonk_rep3_connect_io)
  size_t slot_words = 0;  // 32-bit words per arena slot (4n shares)
  cs::PrfArgs prf;
  uint64_t ctr = 0;       // field elements drawn from each stream so far
  uint64_t rbase = 0;     // first random share of round 2
  cs::PlonkConsts K;
  cs::R3Blinders B;
  std::vector<uint64_t> pub;  // public inputs (Montgomery), without the leading slot
};

namespace {

constexpr int R3_SLOTS = 12;

int r3_create(cs_plonk_rep3* s) {
  const size_t n = s->pk->n;
  CS_TRY(s->ws.reserve(n, s->pk->n_vars, 2));
  for (DevBuf& p : s->polyadd) CS_TRY(p.reserve((n + 8) * 32));
  s->slot_words = 4 * n * 2 * 8;
  CS_TRY(s->arena.reserve((size_t)R3_SLOTS * s->slot_words * 4));
  CS_CUDA(cudaMemsetAsync(s->arena.p, 0, (size_t)R3_SLOTS * s->slot_words * 4, s->ctx->stream));
  CS_TRY(s->addv.reserve((2 * n + 2) * 32));
  CS_TRY(s->pubv.reserve((8 * n + 16) * 32));  // 1/G | 1/Q | scan scratch (2n + 2) | opened vectors (2n + 1)
  CS_CUDA(cudaStreamSynchronize(s->ctx->stream));
  return 0;
}

inline uint32_t* r3_slot(cs_plonk_rep3* s, int k) { return s->arena.as<uint32_t>() + (size_t)k * s->slot_words; }
inline uint32_t* r3_peer(cs_plonk_rep3* s, int k) { return s->next_arena ? s->next_arena + (size_t)k * s->slot_words : nullptr; }

template <class Cfg>
int r3_round1_t(cs_plonk_rep3* s, const uint64_t* h_pub, const uint64_t* h_wit_shares, const uint64_t* h_blind, uint64_t* out_points) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HR;
  cs_ctx* ctx = s->ctx;
  cs_plonk_pk* pk = s->pk;
  const uint32_t n = pk->n;
  s->pub.assign(h_pub + HR::N, h_pub + (size_t)(pk->n_public + 1) * HR::N);
  CS_TRY(load_witness<Cfg>(ctx, pk, s->ws, h_pub, h_wit_shares, 2, s->party < 2 ? s->party : -1));
  HR bsh[22];
  memcpy(bsh, h_blind, sizeof(bsh));
  init_consts<Cfg>(s->K, pk, bsh, 2);
  memset(&s->B, 0, sizeof(s->B));
  for (int i = 0; i < 9; i++) { put(s->B.b[i].v[0], bsh[2 * i]); put(s->B.b[i].v[1], bsh[2 * i + 1]); }
  for (int k = 0; k < 3; k++) {
    CS_TRY(wire_poly<Cfg>(ctx, pk, s->ws, k, 2, bsh + 4 * k));
    CS_LAUNCH(k_extract_component<FrP>, ceil_div(n + 2, 256), 256, 0, ctx->stream, s->ws.poly[k].as<uint32_t>(), n + 2, 2u, 0u,
              s->polyadd[k].as<uint32_t>());
  }
  return commit_polys<Cfg>(ctx, pk, s->polyadd, 3, (size_t)n + 2, out_points);
}

// elementwise inverse of `cnt` public values at `v` (device) into `out`; scratch: 2 cnt elements at `scr`
template <class Cfg>
int r3_batch_inverse(cs_ctx* ctx, PlonkWork& ws, const uint32_t* v, uint32_t cnt, uint32_t* scr, uint32_t* out) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HR;
  uint32_t *pre = scr, *suf = scr + (size_t)cnt * FrP::N;
  CS_TRY((scan<FrP, 0>(ctx, ws, v, pre, cnt, 0)));
  CS_TRY((scan<FrP, 0>(ctx, ws, v, suf, cnt, 1)));
  HR total;
  CS_CUDA(cudaMemcpyAsync(total.l, suf, sizeof(total.l), cudaMemcpyDeviceToHost, ctx->stream));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  if (total.is_zero()) return fail(CS_ERR_ARG, "Cannot invert zero");  // rep3 inv_vec, arithmetic.rs:245-262
  HR it = total.inverse();
  uint32_t* d_it = ws.small.as<uint32_t>() + 128 * FrP::N;
  CS_CUDA(cudaMemcpyAsync(d_it, it.l, sizeof(it.l), cudaMemcpyHostToDevice, ctx->stream));
  CS_LAUNCH(k_batch_inverse<FrP>, ceil_div(cnt, 128), 128, 0, ctx->stream, pre, suf, d_it, cnt, out);
  CS_CUDA(cudaStreamSynchronize(ctx->stream));  // `it` is a stack variable
  return 0;
}

template <class Cfg>
int r3_step_t(cs_plonk_rep3* s, int step, const uint64_t* h_in, uint64_t* h_out) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HR;
  constexpr int NW = FrP::N;
  cs_ctx* ctx = s->ctx;
  cs_plonk_pk* pk = s->pk;
  PlonkWork& ws = s->ws;
  cudaStream_t st = ctx->stream;
  const uint32_t n = pk->n, n4 = 4 * n;
  const unsigned gb = ceil_div(n, 128);
  uint32_t *addv = s->addv.as<uint32_t>(), *pubv = s->pubv.as<uint32_t>();
  // public vectors: [0, n) 1/G | [n, 2n+1) 1/Q | then scratch
  uint32_t *ginv = pubv, *qinv = pubv + (size_t)n * NW, *pscr = pubv + (size_t)(2 * n + 1) * NW;
  switch (step) {
    case CS_PLONK_R3_ROUND2_A: {  // in: beta, gamma
      memcpy(s->K.beta, h_in, 32);
      memcpy(s->K.gamma, h_in + HR::N, 32);
      CS_LAUNCH(k_r3_round2_a<Rep3Pol<FrP>>, gb, 128, 0, st, r3_round2_in(pk, ws), s->K, n, s->party, s->prf, s->ctr, r3_slot(s, 0),
                r3_slot(s, 1), r3_peer(s, 0), r3_peer(s, 1));
      s->ctr += 2 * (uint64_t)n;
      break;
    }
    case CS_PLONK_R3_ROUND2_B: {
      CS_LAUNCH(k_r3_round2_b<Rep3Pol<FrP>>, gb, 128, 0, st, r3_round2_in(pk, ws), s->K, n, s->party, s->prf, s->ctr, r3_slot(s, 0),
                r3_slot(s, 1), r3_slot(s, 2), r3_slot(s, 3), r3_peer(s, 2), r3_peer(s, 3));
      s->ctr += 2 * (uint64_t)n;
      break;
    }
    case CS_PLONK_R3_ROUND2_C: {  // out: g (n) | q (n + 1), additive
      s->rbase = s->ctr;
      s->ctr += 2 * (3 * (uint64_t)n + 2);  // 3n + 2 random shares s, r, s' of 64 bytes each (two element slots)
      CS_LAUNCH(k_r3_round2_c<Rep3Pol<FrP>>, ceil_div(n + 1, 128), 128, 0, st, r3_slot(s, 3), n, s->prf, s->rbase, s->ctr, addv,
                addv + (size_t)n * NW);
      s->ctr += 2 * (uint64_t)n + 1;
      if (h_out) CS_CUDA(cudaMemcpyAsync(h_out, addv, (size_t)(2 * n + 1) * 32, cudaMemcpyDeviceToHost, st));
      CS_CUDA(cudaStreamSynchronize(st));
      return 0;
    }
    case CS_PLONK_R3_ROUND2_D: {  // in: opened G (n) | Q (n + 1)
      uint32_t* opened = pscr + (size_t)(4 * n + 4) * NW;  // h_in == NULL: the driver summed the parties' vectors in place
      if (h_in) CS_CUDA(cudaMemcpyAsync(opened, h_in, (size_t)(2 * n + 1) * 32, cudaMemcpyHostToDevice, st));
      CS_TRY(r3_batch_inverse<Cfg>(ctx, ws, opened, n, pscr, ginv));
      CS_TRY(r3_batch_inverse<Cfg>(ctx, ws, opened + (size_t)n * NW, n + 1, pscr, qinv));
      CS_LAUNCH(k_r3_round2_d<Rep3Pol<FrP>>, gb, 128, 0, st, r3_slot(s, 2), ginv, qinv, n, s->prf, s->rbase, s->ctr, r3_slot(s, 4),
                r3_slot(s, 5), r3_peer(s, 4), r3_peer(s, 5));
      s->ctr += 2 * (uint64_t)n;
      break;
    }
    case CS_PLONK_R3_ROUND2_E: {
      CS_LAUNCH(k_r3_round2_e<Rep3Pol<FrP>>, gb, 128, 0, st, r3_slot(s, 4), n, s->prf, s->rbase, s->ctr, r3_slot(s, 6), r3_peer(s, 6));
      s->ctr += n;
      break;
    }
    case CS_PLONK_R3_ROUND2_F: {  // out: y (n), additive
      CS_LAUNCH(k_r3_round2_f<Rep3Pol<FrP>>, gb, 128, 0, st, r3_slot(s, 6), qinv, n, s->prf, s->rbase, s->ctr, addv);
      s->ctr += n;
      if (h_out) CS_CUDA(cudaMemcpyAsync(h_out, addv, (size_t)n * 32, cudaMemcpyDeviceToHost, st));
      CS_CUDA(cudaStreamSynchronize(st));
      return 0;
    }
    case CS_PLONK_R3_ROUND2_G: {  // in: opened Y (n); out: partial [z]
      uint32_t* y = pscr;
      if (h_in) CS_CUDA(cudaMemcpyAsync(y, h_in, (size_t)n * 32, cudaMemcpyHostToDevice, st));
      else CS_CUDA(cudaMemcpyAsync(y, pscr + (size_t)(4 * n + 4) * NW, (size_t)n * 32, cudaMemcpyDeviceToDevice, st));
      CS_TRY((scan<FrP, 0>(ctx, ws, y, y, n, 0)));
      CS_LAUNCH(k_r3_round2_g<Rep3Pol<FrP>>, gb, 128, 0, st, y, r3_slot(s, 5), n, ws.poly[3].as<uint32_t>());
      HR bsh[6];
      for (int i = 0; i < 3; i++) { memcpy(bsh[2 * i].l, s->B.b[6 + i].v[0], 32); memcpy(bsh[2 * i + 1].l, s->B.b[6 + i].v[1], 32); }
      CS_TRY(z_poly<Cfg>(ctx, pk, ws, 2, bsh));
      CS_LAUNCH(k_extract_component<FrP>, ceil_div(n + 3, 256), 256, 0, st, ws.poly[3].as<uint32_t>(), n + 3, 2u, 0u,
                s->polyadd[3].as<uint32_t>());
      return commit_polys<Cfg>(ctx, pk, s->polyadd + 3, 1, (size_t)n + 3, h_out);
    }
    case CS_PLONK_R3_ROUND3_A: {  // in: alpha
      HR alpha;
      memcpy(alpha.l, h_in, 32);
      CS_TRY(set_alpha<Cfg>(pk, s->K, alpha));
      CS_LAUNCH(k_r3_quot_l1<Rep3Pol<FrP>>, ceil_div(n4, 64), 64, 0, st, r3_quot_in(pk, ws), s->B, n, s->prf, s->ctr,
                s->arena.as<uint32_t>(), s->next_arena, s->slot_words);
      s->ctr += 12 * (uint64_t)n4;
      break;
    }
    case CS_PLONK_R3_ROUND3_B: {  // out: partial [t1] [t2] [t3]
      CS_LAUNCH(k_r3_quot_l2<Rep3Pol<FrP>>, ceil_div(n4, 64), 64, 0, st, r3_quot_in(pk, ws), s->B, key_evals(pk, ws), n, pk->nlag,
                s->K, s->party, s->prf, s->ctr, s->arena.as<uint32_t>(), s->slot_words, ws.t.as<uint32_t>(), ws.tz.as<uint32_t>());
      s->ctr += 2 * (uint64_t)n4;
      return split_and_commit<Cfg>(ctx, pk, ws, s->K, h_out);
    }
    case CS_PLONK_R3_ROUND4: {  // in: xi; out: partial eval_a eval_b eval_c eval_zw, then public eval_s1 eval_s2
      HR xi;
      memcpy(xi.l, h_in, 32);
      return evaluate<Cfg>(ctx, pk, s->polyadd, xi, h_out);
    }
    case CS_PLONK_R3_ROUND5: {  // in: xi, v0, eval_a eval_b eval_c eval_s1 eval_s2 eval_zw (opened); out: partial [Wxi] [Wxiw]
      HR in[8];
      memcpy(in, h_in, sizeof(in));
      // the public polynomials and constants enter once (add_with_public on x_0)
      return opening_polys<Cfg>(ctx, pk, ws, s->polyadd, s->pub.data(), s->K, in[0], in[1], in + 2, s->party == 0, h_out);
    }
    default:
      return fail(CS_ERR_ARG, "cs_plonk_rep3_step: unknown step %d", step);
  }
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// Rep3CoPlonk::prove for one party (co-plonk/src/lib.rs:222-240; prove_inner :80-115; openings mpc/rep3.rs:113-138):
// the step sequence of the device session, the Keccak transcript and the openings, over a cs_net.
//  * "reshare" of first-layer products: with the next party's arena connected the kernels have already stored them
//    there (NVLink peer stores) and the exchange is a token round; otherwise the a-halves travel through the net.
//  * opening of an m-element additive vector: with the peers' out-vectors connected (cs_plonk_rep3_connect_io) the sum
//    is two vector additions that READ THE PEERS' HBM, fenced by token rounds; otherwise host-staged through the net.
namespace {

int r3_token_round(cs_net* net) {  // broadcast of one byte: nobody passes before everybody has arrived
  const int id = net->id, nx = (id + 1) % 3, pv = (id + 2) % 3;
  uint8_t one = 1, a = 0, b = 0;
  CS_TRY(cs_net_send(net, nx, &one, 1));
  CS_TRY(cs_net_send(net, pv, &one, 1));
  CS_TRY(cs_net_recv(net, pv, &a, 1));
  return cs_net_recv(net, nx, &b, 1);
}

template <class Cfg>
int r3_prove_t(cs_plonk_rep3* s, cs_net* net, cs_rep3_state* state, const uint64_t* h_pub, size_t n_pub, const uint64_t* h_wit,
               size_t n_wit, const uint64_t* h_blind, uint64_t* out_points, uint64_t* out_evals) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HR;
  typedef host::HFp<typename Cfg::FqP> HQ;
  typedef host::HAffine<HQ> A1;
  typedef host::HXyzz<HQ> X1;
  cs_ctx* ctx = s->ctx;
  const cs_plonk_pk* pk = s->pk;
  const cs_curve cv = (cs_curve)pk->curve;
  const size_t n = pk->n, pl = 2 * HQ::N;
  const int id = net->id, nx = (id + 1) % 3, pv = (id + 2) % 3;
  // Round1Challenges::random (round1.rs:82-92): eleven T::rand shares, unless the caller brings them (known-answer tests)
  uint64_t blind[11 * 2 * HR::N];
  if (h_blind) memcpy(blind, h_blind, sizeof(blind));
  else for (int i = 0; i < 11; i++) CS_TRY(cs_rep3_state_rand(state, cv, blind + (size_t)i * 2 * HR::N));
  cs_rep3_prf prf;
  CS_TRY(cs_rep3_state_prf(state, &prf));
  // whatever happens below, the streams move past what the device kernels may have consumed: PRF output is never reused
  struct Advance {
    cs_plonk_rep3* s; cs_rep3_state* st;
    ~Advance() { cs_rep3_state_advance(st, cs_plonk_rep3_prf_words(s)); }
  } advance{s, state};

  // open_point_vec_g1 / open_vec: every party sends its k partial values (`len` limbs each) to both others, then adds
  auto open = [&](uint64_t* v, int k, size_t len, auto add) -> int {
    std::vector<uint64_t> a(k * len), b(k * len);
    CS_TRY(cs_net_send(net, nx, v, k * len * 8));
    CS_TRY(cs_net_send(net, pv, v, k * len * 8));
    CS_TRY(cs_net_recv(net, pv, a.data(), k * len * 8));
    CS_TRY(cs_net_recv(net, nx, b.data(), k * len * 8));
    for (int i = 0; i < k; i++) add(v + i * len, a.data() + i * len, b.data() + i * len);
    return 0;
  };
  auto add_points = [](uint64_t* x, const uint64_t* y, const uint64_t* z) {
    A1 p[3];
    memcpy(&p[0], x, sizeof(A1)); memcpy(&p[1], y, sizeof(A1)); memcpy(&p[2], z, sizeof(A1));
    p[0] = host::haffine(host::hadd(host::hadd(X1::from_affine(p[0]), X1::from_affine(p[1])), X1::from_affine(p[2])));
    memcpy(x, &p[0], sizeof(A1));
  };
  auto add_scalars = [](uint64_t* x, const uint64_t* y, const uint64_t* z) {
    HR s[3];
    memcpy(s[0].l, x, sizeof(s[0].l)); memcpy(s[1].l, y, sizeof(s[1].l)); memcpy(s[2].l, z, sizeof(s[2].l));
    s[0] = s[0] + s[1] + s[2];
    memcpy(x, s[0].l, sizeof(s[0].l));
  };
  void *d_out_v = nullptr, *d_in_v = nullptr;
  CS_TRY(cs_plonk_rep3_io(s, &d_out_v, &d_in_v));
  uint64_t* d_out = (uint64_t*)d_out_v;
  uint64_t* d_in = (uint64_t*)d_in_v;
  auto open_device_vector = [&](size_t m) -> int {  // sum of the parties' additive vectors at d_out -> d_in
    CS_CUDA(cudaStreamSynchronize(ctx->stream));
    if (s->peer_out[0]) {
      CS_TRY(r3_token_round(net));  // all three vectors are complete
      CS_TRY(cs_vec_add(ctx, cv, d_out, (const uint64_t*)s->peer_out[0], d_in, m));
      CS_TRY(cs_vec_add(ctx, cv, d_in, (const uint64_t*)s->peer_out[1], d_in, m));
      CS_CUDA(cudaStreamSynchronize(ctx->stream));
      net->bytes_sent += 2 * m * 32;  // what the two peers pulled from this party over NVLink
      return r3_token_round(net);     // nobody overwrites its vector while a peer still reads it
    }
    std::vector<uint64_t> mine(m * HR::N), a(m * HR::N), b(m * HR::N);
    CS_CUDA(cudaMemcpyAsync(mine.data(), d_out, m * 32, cudaMemcpyDeviceToHost, ctx->stream));
    CS_CUDA(cudaStreamSynchronize(ctx->stream));
    // ring order with both directions progressing: messages may exceed the mailbox credit window
    CS_TRY(cs_net_sendrecv(net, nx, mine.data(), m * 32, pv, a.data(), m * 32));
    CS_TRY(cs_net_sendrecv(net, pv, mine.data(), m * 32, nx, b.data(), m * 32));
    DevBuf da, db;
    int rc = da.reserve(m * 32);
    if (!rc) rc = db.reserve(m * 32);
    if (!rc) {
      cudaMemcpyAsync(da.p, a.data(), m * 32, cudaMemcpyHostToDevice, ctx->stream);
      cudaMemcpyAsync(db.p, b.data(), m * 32, cudaMemcpyHostToDevice, ctx->stream);
      rc = cs_vec_add(ctx, cv, d_out, da.as<uint64_t>(), d_in, m);
      if (!rc) rc = cs_vec_add(ctx, cv, d_in, db.as<uint64_t>(), d_in, m);
      cudaStreamSynchronize(ctx->stream);
    }
    da.release(); db.release();
    return rc;
  };
  auto reshare = [&](std::initializer_list<int> slots, size_t count) -> int {
    CS_CUDA(cudaStreamSynchronize(ctx->stream));
    if (s->next_arena) return r3_token_round(net);
    // staged: the a-halves of every slot go to the next party, the previous party's arrive as our b-halves
    std::vector<uint64_t> za(count * HR::N), zb(count * HR::N);
    DevBuf d;
    CS_TRY(d.reserve(count * 32));
    int rc = 0;
    for (int k : slots) {
      uint8_t* base = (uint8_t*)s->arena.p + (size_t)k * s->slot_words * 4;
      cudaMemcpy2DAsync(za.data(), 32, base, 64, 32, count, cudaMemcpyDeviceToHost, ctx->stream);
      cudaStreamSynchronize(ctx->stream);
      rc = cs_net_sendrecv(net, nx, za.data(), count * 32, pv, zb.data(), count * 32);
      if (rc) break;
      cudaMemcpyAsync(d.p, zb.data(), count * 32, cudaMemcpyHostToDevice, ctx->stream);
      rc = cs_rep3_set_b(ctx, cv, d.as<uint64_t>(), count, (uint64_t*)base);
      if (rc) break;
      cudaStreamSynchronize(ctx->stream);
    }
    d.release();
    return rc;
  };
  auto step = [&](int st, const uint64_t* in, uint64_t* out) { return cs_plonk_rep3_step(s, st, in, out); };

  uint64_t* pts = out_points;  // A B C Z T1 T2 T3 Wxi Wxiw
  // ---- round 1
  CS_TRY(cs_plonk_rep3_round1(s, &prf, h_pub, n_pub, h_wit, n_wit, blind, pts));
  CS_TRY(open(pts, 3, pl, add_points));
  // ---- round 2
  Challenges<Cfg> ch;
  ch.round2(pk, h_pub, pts);
  const HR bg[2] = {ch.beta, ch.gamma};
  CS_TRY(step(CS_PLONK_R3_ROUND2_A, bg[0].l, nullptr)); CS_TRY(reshare({0, 1}, n));
  CS_TRY(step(CS_PLONK_R3_ROUND2_B, nullptr, nullptr)); CS_TRY(reshare({2, 3}, n));
  CS_TRY(step(CS_PLONK_R3_ROUND2_C, nullptr, nullptr));
  CS_TRY(open_device_vector(2 * n + 1));
  CS_TRY(step(CS_PLONK_R3_ROUND2_D, nullptr, nullptr)); CS_TRY(reshare({4, 5}, n));
  CS_TRY(step(CS_PLONK_R3_ROUND2_E, nullptr, nullptr)); CS_TRY(reshare({6}, n));
  CS_TRY(step(CS_PLONK_R3_ROUND2_F, nullptr, nullptr));
  CS_TRY(open_device_vector(n));
  CS_TRY(step(CS_PLONK_R3_ROUND2_G, nullptr, pts + 3 * pl));
  CS_TRY(open(pts + 3 * pl, 1, pl, add_points));
  // ---- round 3
  ch.round3(pts + 3 * pl);
  CS_TRY(step(CS_PLONK_R3_ROUND3_A, ch.alpha.l, nullptr));
  CS_TRY(reshare({0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}, 4 * n));
  CS_TRY(step(CS_PLONK_R3_ROUND3_B, nullptr, pts + 4 * pl));
  CS_TRY(open(pts + 4 * pl, 3, pl, add_points));
  // ---- round 4
  ch.round4(pts + 4 * pl);
  HR e[6];  // partial a b c zw | public s1 s2
  CS_TRY(step(CS_PLONK_R3_ROUND4, ch.xi.l, e[0].l));
  CS_TRY(open(e[0].l, 4, HR::N, add_scalars));
  // ---- round 5
  const HR ev[6] = {e[0], e[1], e[2], e[4], e[5], e[3]};  // the proof's order: a b c s1 s2 zw
  ch.round5(ev);
  const HR in5[8] = {ch.xi, ch.v, ev[0], ev[1], ev[2], ev[3], ev[4], ev[5]};
  CS_TRY(step(CS_PLONK_R3_ROUND5, in5[0].l, pts + 7 * pl));
  CS_TRY(open(pts + 7 * pl, 2, pl, add_points));
  memcpy(out_evals, ev, sizeof(ev));
  return 0;
}

}  // namespace

// ======================================================================================================
// Shamir co-Plonk (ShamirCoPlonk::prove, co-plonk/src/lib.rs:237-260 with ShamirPlonkDriver, mpc/shamir.rs): one
// session per party of a Shamir(n, t) sharing, the whole proof inside the library over a cs_net.  A share is one Fr
// element, so every linear step -- additions, gather, iNTT / extension, blinding, tsplit, evaluation, the Wxi numerator,
// division by (X - xi), the commitments -- is the plain prover's kernel on shares, with public values added by every
// party.  Products follow the Rep3 session's layering (cs_plonk_rep3.cuh, ShamirPol): a local product (degree 2t), then
// ONE device degree reduction per product layer covering all of its slots (one king round each):
//   round 2  n12 d12 | num den | x u | m      7n reductions; G = den s, Q = r s' and Y = m / r_{i+1} open at degree 2t;
//            s, r, s' are 3n + 2 random shares (the r_t halves of double sharings)
//   round 3  the twelve first-layer products  48n reductions; t and tz stay at degree 2t
// Degree-2t results (T1 T2 T3 Wxi) open with 2t + 1 parties; a b c Z Wxiw and the four evaluations with t + 1.
// Pairs per proof: 10n + 2 (made on the device when round 2 starts) + 48n (when round 3 starts) = 58n + 2, plus the
// 11 blinders from the state's host pool (ShamirState::rand) unless the caller brings them: 58n + 13.
// ======================================================================================================
struct cs_plonk_shamir {
  cs_ctx* ctx = nullptr;
  cs_plonk_pk* pk = nullptr;
  int n_parties = 0, thr = 0, party = 0;
  cs_shamir_state* state = nullptr;  // created over the first proof's net, kept for the next ones
  PlonkWork ws;
  DevBuf arena, pair_t, pair_2t, addv, pubv;
  size_t pairs = 0;    // pairs the last proof consumed
  double pair_ms = 0;  // wall time of the last proof's device pair generation
};

namespace {

int sh_create(cs_plonk_shamir* s) {
  const size_t n = s->pk->n;
  CS_TRY(s->ws.reserve(n, s->pk->n_vars, 1));
  CS_TRY(s->arena.reserve(48 * n * 32));  // round 3: twelve slots of 4n; round 2: seven slots of n
  CS_TRY(s->addv.reserve((2 * n + 2) * 32));
  return s->pubv.reserve((8 * n + 16) * 32);  // 1/G | 1/Q | scan scratch | opened G | Q
}

template <class Cfg>
int sh_prove_t(cs_plonk_shamir* s, cs_net* net, const uint64_t* h_pub, const uint64_t* h_wit, const uint64_t* h_blind,
               uint64_t* out_points, uint64_t* out_evals, uint64_t* out_blind) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HR;
  typedef ShamirPol<FrP> Pol;
  constexpr int NW = FrP::N;
  cs_ctx* ctx = s->ctx;
  cs_plonk_pk* pk = s->pk;
  PlonkWork& ws = s->ws;
  cudaStream_t st = ctx->stream;
  const cs_curve cv = (cs_curve)pk->curve;
  const uint32_t n = pk->n, n4 = 4 * n;
  const size_t pl = point_limbs64(pk->curve, CS_G1);
  const unsigned gb = ceil_div(n, 128);
  s->pairs = 0;
  s->pair_ms = 0;
  if (!s->state) CS_TRY(cs_shamir_state_create(net, cv, s->n_parties, s->thr, 0, &s->state));
  cs_shamir_state* sst = s->state;
  // Round1Challenges::random (round1.rs:82-92): eleven ShamirState::rand shares unless the caller brings them
  HR b[11];
  if (h_blind) memcpy(b, h_blind, sizeof(b));
  else {
    for (int i = 0; i < 11; i++) CS_TRY(cs_shamir_state_rand(sst, net, b[i].l));
    s->pairs += 11;
  }
  if (out_blind) memcpy(out_blind, b, sizeof(b));
  auto make_pairs = [&](size_t count) -> int {
    CS_TRY(s->pair_t.reserve(count * 32));
    CS_TRY(s->pair_2t.reserve(count * 32));
    const auto t0 = std::chrono::steady_clock::now();
    CS_TRY(shamir_double_sharings(ctx, sst, net, count, s->pair_t.as<uint64_t>(), s->pair_2t.as<uint64_t>()));
    s->pair_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    s->pairs += count;
    return 0;
  };
  auto reduce = [&](uint32_t* v, size_t len, size_t first_pair) {  // in place, pairs [first_pair, first_pair + len)
    CS_CUDA(cudaStreamSynchronize(st));
    return shamir_degree_reduce(ctx, sst, net, (const uint64_t*)v, len, (uint64_t*)v, s->pair_t.as<uint64_t>() + first_pair * 4,
                                s->pair_2t.as<uint64_t>() + first_pair * 4);
  };
  auto open_points = [&](uint64_t* p, int k, int degree_2t) {
    return shamir_open_points(sst, net, CS_G1, degree_2t, p, k);
  };
  uint64_t* P = out_points;  // A B C Z T1 T2 T3 Wxi Wxiw
  // ---- init round (every party holds the public values themselves), round 1
  CS_TRY(load_witness<Cfg>(ctx, pk, ws, h_pub, h_wit, 1, 0));
  for (int k = 0; k < 3; k++) CS_TRY(wire_poly<Cfg>(ctx, pk, ws, k, 1, b + 2 * k));
  CS_TRY(commit_polys<Cfg>(ctx, pk, ws.poly, 3, (size_t)n + 2, P));
  CS_TRY(open_points(P, 3, 0));
  // ---- round 2 (round2.rs:197-250)
  Challenges<Cfg> ch;
  ch.round2(pk, h_pub, P);
  PlonkConsts K;
  init_consts<Cfg>(K, pk, b, 1);
  put(K.beta, ch.beta);
  put(K.gamma, ch.gamma);
  CS_TRY(make_pairs(10 * (size_t)n + 2));
  const ShamirRnd R{s->pair_t.as<uint32_t>()};  // s, r, s' = the r_t halves of pairs [0, 3n + 2)
  const size_t first = 3 * (size_t)n + 2;         // the reductions take the pairs after them
  uint32_t* arena = s->arena.as<uint32_t>();
  auto slot = [&](int k) { return arena + (size_t)k * n * NW; };  // round 2: slots of n, a layer's slots adjacent
  uint32_t *pubv = s->pubv.as<uint32_t>(), *addv = s->addv.as<uint32_t>();
  uint32_t *ginv = pubv, *qinv = pubv + (size_t)n * NW, *pscr = pubv + (size_t)(2 * n + 1) * NW;
  uint32_t* opened = pscr + (size_t)(4 * n + 4) * NW;
  const R3Round2In in = r3_round2_in(pk, ws);
  uint32_t* none = nullptr;
  CS_LAUNCH(k_r3_round2_a<Pol>, gb, 128, 0, st, in, K, n, s->party, R, 0ull, slot(0), slot(1), none, none);
  CS_TRY(reduce(slot(0), 2 * (size_t)n, first));
  CS_LAUNCH(k_r3_round2_b<Pol>, gb, 128, 0, st, in, K, n, s->party, R, 0ull, slot(0), slot(1), slot(2), slot(3), none, none);
  CS_TRY(reduce(slot(2), 2 * (size_t)n, first + 2 * (size_t)n));
  CS_LAUNCH(k_r3_round2_c<Pol>, ceil_div(n + 1, 128), 128, 0, st, slot(3), n, R, 0ull, 0ull, addv, addv + (size_t)n * NW);
  CS_CUDA(cudaStreamSynchronize(st));
  CS_TRY(shamir_open_vec(ctx, sst, net, 1, (const uint64_t*)addv, 2 * (size_t)n + 1, (uint64_t*)opened));
  CS_TRY(r3_batch_inverse<Cfg>(ctx, ws, opened, n, pscr, ginv));
  CS_TRY(r3_batch_inverse<Cfg>(ctx, ws, opened + (size_t)n * NW, n + 1, pscr, qinv));
  CS_LAUNCH(k_r3_round2_d<Pol>, gb, 128, 0, st, slot(2), ginv, qinv, n, R, 0ull, 0ull, slot(4), slot(5), none, none);
  CS_TRY(reduce(slot(4), 2 * (size_t)n, first + 4 * (size_t)n));
  CS_LAUNCH(k_r3_round2_e<Pol>, gb, 128, 0, st, slot(4), n, R, 0ull, 0ull, slot(6), none);
  CS_TRY(reduce(slot(6), n, first + 6 * (size_t)n));
  CS_LAUNCH(k_r3_round2_f<Pol>, gb, 128, 0, st, slot(6), qinv, n, R, 0ull, 0ull, addv);
  CS_CUDA(cudaStreamSynchronize(st));
  uint32_t* y = pscr;
  CS_TRY(shamir_open_vec(ctx, sst, net, 1, (const uint64_t*)addv, n, (uint64_t*)y));
  CS_TRY((scan<FrP, 0>(ctx, ws, y, y, n, 0)));
  CS_LAUNCH(k_r3_round2_g<Pol>, gb, 128, 0, st, y, slot(5), n, ws.poly[3].as<uint32_t>());
  CS_TRY(z_poly<Cfg>(ctx, pk, ws, 1, b + 6));
  CS_TRY(commit_polys<Cfg>(ctx, pk, ws.poly + 3, 1, (size_t)n + 3, P + 3 * pl));
  CS_TRY(open_points(P + 3 * pl, 1, 0));
  // ---- round 3 (round3.rs:560-610)
  ch.round3(P + 3 * pl);
  CS_TRY(set_alpha<Cfg>(pk, K, ch.alpha));
  CS_TRY(make_pairs(48 * (size_t)n));
  const R3QuotIn qi = r3_quot_in(pk, ws);
  R3Blinders B;
  memset(&B, 0, sizeof(B));
  for (int i = 0; i < 9; i++) put(B.b[i].v[0], b[i]);
  const size_t slot_words = (size_t)n4 * NW;
  const ShamirRnd R3{nullptr};  // round 3 draws no random shares; round 2's pair buffer has been replaced
  CS_LAUNCH(k_r3_quot_l1<Pol>, ceil_div(n4, 64), 64, 0, st, qi, B, n, R3, 0ull, arena, none, slot_words);
  CS_TRY(reduce(arena, 12 * (size_t)n4, 0));
  CS_LAUNCH(k_r3_quot_l2<Pol>, ceil_div(n4, 64), 64, 0, st, qi, B, key_evals(pk, ws), n, pk->nlag, K, s->party, R3, 0ull, arena,
            slot_words, ws.t.as<uint32_t>(), ws.tz.as<uint32_t>());
  CS_TRY(split_and_commit<Cfg>(ctx, pk, ws, K, P + 4 * pl));
  CS_TRY(open_points(P + 4 * pl, 3, 1));
  // ---- round 4
  ch.round4(P + 4 * pl);
  HR e[6];  // a b c zw (shares, then opened) | public s1 s2
  CS_TRY(evaluate<Cfg>(ctx, pk, ws.poly, ch.xi, e[0].l));
  CS_TRY(shamir_open_scalars(sst, net, 0, e[0].l, 4));
  // ---- round 5
  const HR ev[6] = {e[0], e[1], e[2], e[4], e[5], e[3]};  // the proof's order: a b c s1 s2 zw
  ch.round5(ev);
  CS_TRY(opening_polys<Cfg>(ctx, pk, ws, ws.poly, h_pub + HR::N, K, ch.xi, ch.v, ev, 1, P + 7 * pl));  // public terms at every party
  CS_TRY(open_points(P + 7 * pl, 1, 1));  // Wxi: degree 2t (it carries T1 T2 T3)
  CS_TRY(open_points(P + 8 * pl, 1, 0));  // Wxiw: degree t
  memcpy(out_evals, ev, sizeof(ev));
  return 0;
}

// the caller's public inputs (the leading one included) and witness entries against the key
int check_counts(const cs_plonk_pk* pk, size_t n_public_inputs, size_t n_witness, const char* fn) {
  if (n_public_inputs != (size_t)pk->n_public + 1)
    return fail(CS_ERR_ARG, "%s: %zu public inputs, the key expects %u (incl. the leading one)", fn, n_public_inputs,
                pk->n_public + 1);
  if (n_witness != pk->n_witness()) return fail(CS_ERR_ARG, "%s: %zu witness values, the key expects %u", fn, n_witness, pk->n_witness());
  return 0;
}

}  // namespace

extern "C" {

int cs_plonk_pk_create(cs_ctx* ctx, const cs_plonk_key_desc* d, cs_plonk_pk** out) {
  if (!ctx || !d || !out) return fail(CS_ERR_ARG, "cs_plonk_pk_create: NULL argument");
  if (!d->k1_mont || !d->k2_mont || !d->vk_points || !d->p_tau || !d->lagrange_evals ||
      (d->n_additions && (!d->additions_ids || !d->additions_factors)) ||
      (d->n_constraints && (!d->map_a || !d->map_b || !d->map_c)))
    return fail(CS_ERR_ARG, "cs_plonk_pk_create: NULL array in the key description");
  for (int i = 0; i < 5; i++)
    if (!d->q_coeffs[i] || !d->q_evals[i]) return fail(CS_ERR_ARG, "cs_plonk_pk_create: NULL selector polynomial");
  for (int i = 0; i < 3; i++)
    if (!d->s_coeffs[i] || !d->s_evals[i]) return fail(CS_ERR_ARG, "cs_plonk_pk_create: NULL sigma polynomial");
  CS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<cs_plonk_pk> pk(new cs_plonk_pk());
  pk->curve = d->curve;
  int rc = 0;
  CS_DISPATCH_CURVE(d->curve, rc = plonk_pk_create_t<Cfg>(ctx, d, pk.get()));
  if (rc) {
    cs_plonk_pk_free(pk.release());
    return rc;
  }
  *out = pk.release();
  return 0;
}

void cs_plonk_pk_free(cs_plonk_pk* pk) {
  if (!pk) return;
  cs_bases_free(pk->p_tau);
  cs_domain_free(pk->dom);
  cs_domain_free(pk->dom4);
  DevBuf* all[] = {&pk->add_ids, &pk->add_factors, &pk->add_order, &pk->map_a, &pk->map_b, &pk->map_c, &pk->lagrange};
  for (DevBuf* b : all) b->release();
  for (int i = 0; i < 5; i++) { pk->q_coeffs[i].release(); pk->q_evals[i].release(); }
  for (int i = 0; i < 3; i++) { pk->s_coeffs[i].release(); pk->s_evals[i].release(); }
  pk->ws.release();
  delete pk;
}

int cs_plonk_pk_curve(const cs_plonk_pk* pk) { return pk ? pk->curve : CS_ERR_ARG; }

int cs_plonk_pk_info(const cs_plonk_pk* pk, size_t* n_public, size_t* n_witness, size_t* domain_size, uint64_t* vk_points) {
  if (!pk) return fail(CS_ERR_ARG, "cs_plonk_pk_info: NULL key");
  if (n_public) *n_public = pk->n_public;
  if (n_witness) *n_witness = pk->n_witness();
  if (domain_size) *domain_size = pk->n;
  if (vk_points) memcpy(vk_points, pk->vk_points.data(), pk->vk_points.size() * 8);
  return 0;
}

int cs_keccak256(const uint8_t* data, size_t len, uint8_t* out32) {
  if ((len && !data) || !out32) return fail(CS_ERR_ARG, "cs_keccak256: NULL argument");
  std::vector<uint8_t> v(data, data + len);
  keccak256(v, out32);
  return 0;
}

int cs_plonk_prove_plain(cs_ctx* ctx, cs_plonk_pk* pk, const uint64_t* h_public_inputs, size_t n_public_inputs,
                         const uint64_t* h_witness, size_t n_witness, const uint64_t* h_blinders_mont,
                         uint64_t* out_points, uint64_t* out_evals) {
  if (!ctx || !pk || !h_public_inputs || !h_blinders_mont || !out_points || !out_evals || (n_witness && !h_witness))
    return fail(CS_ERR_ARG, "cs_plonk_prove_plain: NULL argument");
  CS_TRY(check_counts(pk, n_public_inputs, n_witness, "cs_plonk_prove_plain"));
  CS_DISPATCH_CURVE(pk->curve, return plonk_prove_plain_t<Cfg>(ctx, pk, h_public_inputs, h_witness, h_blinders_mont, out_points, out_evals));
  return 0;
}


int cs_plonk_rep3_create(cs_ctx* ctx, cs_plonk_pk* pk, int party, cs_plonk_rep3** out) {
  if (!ctx || !pk || !out) return fail(CS_ERR_ARG, "cs_plonk_rep3_create: NULL argument");
  if (party < 0 || party > 2) return fail(CS_ERR_ARG, "cs_plonk_rep3_create: party id %d", party);
  CS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<cs_plonk_rep3> s(new cs_plonk_rep3());
  s->ctx = ctx; s->pk = pk; s->party = party;
  memset(&s->prf, 0, sizeof(s->prf));
  const int rc = r3_create(s.get());
  if (rc) { cs_plonk_rep3_free(s.release()); return rc; }
  *out = s.release();
  return 0;
}

void cs_plonk_rep3_free(cs_plonk_rep3* s) {
  if (!s) return;
  DevBuf* all[] = {&s->arena, &s->addv, &s->pubv, &s->polyadd[0], &s->polyadd[1], &s->polyadd[2], &s->polyadd[3]};
  for (DevBuf* b : all) b->release();
  s->ws.release();
  delete s;
}

int cs_plonk_rep3_arena(cs_plonk_rep3* s, void** d_arena, size_t* slot_bytes, unsigned* n_slots) {
  if (!s || !d_arena || !slot_bytes || !n_slots) return fail(CS_ERR_ARG, "cs_plonk_rep3_arena: NULL argument");
  *d_arena = s->arena.p;
  *slot_bytes = s->slot_words * 4;
  *n_slots = R3_SLOTS;
  return 0;
}

int cs_plonk_rep3_io(cs_plonk_rep3* s, void** d_additive_out, void** d_opened_in) {
  if (!s || !d_additive_out || !d_opened_in) return fail(CS_ERR_ARG, "cs_plonk_rep3_io: NULL argument");
  *d_additive_out = s->addv.p;
  *d_opened_in = s->pubv.as<uint32_t>() + ((size_t)(2 * s->pk->n + 1) + (size_t)(4 * s->pk->n + 4)) * 8;
  return 0;
}

int cs_plonk_rep3_connect(cs_plonk_rep3* s, void* d_next_arena) {
  if (!s) return fail(CS_ERR_ARG, "cs_plonk_rep3_connect: NULL argument");
  s->next_arena = reinterpret_cast<uint32_t*>(d_next_arena);
  return 0;
}

int cs_plonk_rep3_round1(cs_plonk_rep3* s, const cs_rep3_prf* prf, const uint64_t* h_public_inputs, size_t n_public_inputs,
                         const uint64_t* h_witness_shares, size_t n_witness, const uint64_t* h_blinder_shares,
                         uint64_t* out_points) {
  if (!s || !prf || !h_public_inputs || !h_blinder_shares || !out_points || (n_witness && !h_witness_shares))
    return fail(CS_ERR_ARG, "cs_plonk_rep3_round1: NULL argument");
  CS_TRY(check_counts(s->pk, n_public_inputs, n_witness, "cs_plonk_rep3_round1"));
  if (prf->rounds == 0 || (prf->rounds & 1) || prf->rounds > 20) return fail(CS_ERR_ARG, "cs_plonk_rep3_round1: bad ChaCha round count");
  CS_CUDA(cudaSetDevice(s->ctx->device));
  memcpy(s->prf.keys.k, prf->seed1, 32);
  memcpy(s->prf.keys.k + 8, prf->seed2, 32);
  s->prf.pos1 = prf->word_pos1; s->prf.pos2 = prf->word_pos2; s->prf.rounds = prf->rounds;
  s->ctr = 0;
  CS_DISPATCH_CURVE(s->pk->curve, return r3_round1_t<Cfg>(s, h_public_inputs, h_witness_shares, h_blinder_shares, out_points));
  return 0;
}

int cs_plonk_rep3_step(cs_plonk_rep3* s, int step, const uint64_t* h_in, uint64_t* h_out) {
  if (!s) return fail(CS_ERR_ARG, "cs_plonk_rep3_step: NULL session");
  CS_CUDA(cudaSetDevice(s->ctx->device));
  // which steps read h_in / write h_out: a missing buffer is an argument error, not a crash
  {
    const bool needs_in = step == CS_PLONK_R3_ROUND2_A || step == CS_PLONK_R3_ROUND3_A || step == CS_PLONK_R3_ROUND4 ||
                          step == CS_PLONK_R3_ROUND5;
    const bool needs_out = step == CS_PLONK_R3_ROUND2_G || step == CS_PLONK_R3_ROUND3_B || step == CS_PLONK_R3_ROUND4 ||
                           step == CS_PLONK_R3_ROUND5;
    if (needs_in && !h_in) return fail(CS_ERR_ARG, "cs_plonk_rep3_step: step %d reads h_in, which is NULL", step);
    if (needs_out && !h_out) return fail(CS_ERR_ARG, "cs_plonk_rep3_step: step %d writes h_out, which is NULL", step);
  }
  CS_DISPATCH_CURVE(s->pk->curve, return r3_step_t<Cfg>(s, step, h_in, h_out));
  return 0;
}

uint64_t cs_plonk_rep3_prf_words(const cs_plonk_rep3* s) { return s ? 8 * s->ctr : 0; }

int cs_plonk_rep3_connect_io(cs_plonk_rep3* s, void* d_prev_out, void* d_next_out) {
  if (!s) return fail(CS_ERR_ARG, "cs_plonk_rep3_connect_io: NULL argument");
  if ((d_prev_out == nullptr) != (d_next_out == nullptr)) return fail(CS_ERR_ARG, "cs_plonk_rep3_connect_io: give both peers or neither");
  s->peer_out[0] = reinterpret_cast<const uint32_t*>(d_prev_out);
  s->peer_out[1] = reinterpret_cast<const uint32_t*>(d_next_out);
  return 0;
}

int cs_plonk_rep3_prove(cs_plonk_rep3* s, cs_net* net, cs_rep3_state* state, const uint64_t* h_public_inputs, size_t n_public_inputs,
                        const uint64_t* h_witness_shares, size_t n_witness, const uint64_t* h_blinder_shares, uint64_t* out_points,
                        uint64_t* out_evals) {
  if (!s || !net || !state || !h_public_inputs || !out_points || !out_evals || (n_witness && !h_witness_shares))
    return fail(CS_ERR_ARG, "cs_plonk_rep3_prove: NULL argument");
  if (net->n != 3 || net->id != s->party) return fail(CS_ERR_ARG, "cs_plonk_rep3_prove: the net is party %d of %d, the session is party %d of 3", net->id, net->n, s->party);
  CS_CUDA(cudaSetDevice(s->ctx->device));
  CS_DISPATCH_CURVE(s->pk->curve, return r3_prove_t<Cfg>(s, net, state, h_public_inputs, n_public_inputs, h_witness_shares, n_witness,
                                                         h_blinder_shares, out_points, out_evals));
  return 0;
}

int cs_plonk_shamir_create(cs_ctx* ctx, cs_plonk_pk* pk, int num_parties, int threshold, int party, cs_plonk_shamir** out) {
  if (!ctx || !pk || !out) return fail(CS_ERR_ARG, "cs_plonk_shamir_create: NULL argument");
  if (threshold < 1 || 2 * threshold + 1 > num_parties) return fail(CS_ERR_ARG, "Threshold too large for number of parties");
  if (num_parties > (int)LINCOMB_MAX) return fail(CS_ERR_LIMIT, "cs_plonk_shamir_create: %d parties exceed %u", num_parties, LINCOMB_MAX);
  if (party < 0 || party >= num_parties) return fail(CS_ERR_ARG, "cs_plonk_shamir_create: party id %d of %d", party, num_parties);
  CS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<cs_plonk_shamir> s(new cs_plonk_shamir());
  s->ctx = ctx; s->pk = pk; s->n_parties = num_parties; s->thr = threshold; s->party = party;
  const int rc = sh_create(s.get());
  if (rc) { cs_plonk_shamir_free(s.release()); return rc; }
  *out = s.release();
  return 0;
}

void cs_plonk_shamir_free(cs_plonk_shamir* s) {
  if (!s) return;
  DevBuf* all[] = {&s->arena, &s->pair_t, &s->pair_2t, &s->addv, &s->pubv};
  for (DevBuf* b : all) b->release();
  s->ws.release();
  cs_shamir_state_free(s->state);
  delete s;
}

int cs_plonk_shamir_prove(cs_plonk_shamir* s, cs_net* net, const uint64_t* h_public_inputs, size_t n_public_inputs,
                          const uint64_t* h_witness_shares, size_t n_witness, const uint64_t* h_blinder_shares,
                          uint64_t* out_points, uint64_t* out_evals, uint64_t* out_blinder_shares) {
  if (!s || !net || !h_public_inputs || !out_points || !out_evals || (n_witness && !h_witness_shares))
    return fail(CS_ERR_ARG, "cs_plonk_shamir_prove: NULL argument");
  if (net->n != s->n_parties || net->id != s->party)
    return fail(CS_ERR_ARG, "cs_plonk_shamir_prove: the net is party %d of %d, the session is party %d of %d", net->id, net->n,
                s->party, s->n_parties);
  CS_TRY(check_counts(s->pk, n_public_inputs, n_witness, "cs_plonk_shamir_prove"));
  CS_CUDA(cudaSetDevice(s->ctx->device));
  CS_DISPATCH_CURVE(s->pk->curve, return sh_prove_t<Cfg>(s, net, h_public_inputs, h_witness_shares, h_blinder_shares, out_points,
                                                         out_evals, out_blinder_shares));
  return 0;
}

size_t cs_plonk_shamir_pairs(const cs_plonk_shamir* s) { return s ? s->pairs : 0; }

double cs_plonk_shamir_pair_ms(const cs_plonk_shamir* s) { return s ? s->pair_ms : 0.0; }

size_t cs_plonk_shamir_device_bytes(const cs_plonk_shamir* s) {
  if (!s) return 0;
  return shamir_state_device_bytes(s->state) + s->ws.bytes() + s->arena.cap + s->pair_t.cap + s->pair_2t.cap + s->addv.cap +
         s->pubv.cap;
}

}  // extern "C"
