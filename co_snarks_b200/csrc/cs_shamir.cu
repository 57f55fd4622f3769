// Shamir(n, t) protocol pieces of the co-snarks provers inside the library:
//   ShamirPreprocessing / ShamirState   mpc-core/src/protocols/shamir.rs:26-186
//   DN07 double sharings (r_t, r_2t)    mpc-core/src/protocols/shamir/rngs.rs:334-470 (random_double_share, buffer_triples)
//   king-based degree reduction         mpc-core/src/protocols/shamir/network.rs:150-301 (degree_reduce_many / _point)
//   openings                            mpc-core/src/protocols/shamir/pointshare.rs:102-111, network.rs:96-126 (broadcast_next)
// over a cs_net of n parties.  Vector-sized work (the pair consumption `inp += r_2t`, the king's Lagrange-weighted
// accumulation, the fresh shares `acc * c_id`, `share -= r_t`) runs on the GPU through k_vec_binop / k_vec_lincomb;
// single points and scalars stay on the host, as in the reference.
//
// One deliberate simplification against rngs.rs: the reference compresses the dealing of the double sharings with
// pairwise PRG seeds (t parties derive their shares locally); here every dealer sends every share explicitly.  The
// resulting objects -- t + 1 uniformly random double sharings per batch, extracted with the (t+1) x n Vandermonde
// matrix -- are the same, only the preprocessing traffic is larger (2 field elements per pair and recipient).
//
// Plonk-sized consumers (cs_plonk_shamir) take their pairs from the device: shamir_double_sharings deals, exchanges and
// extracts whole vectors of pairs with k_fr_rand and k_vec_lincomb (no host arithmetic per pair), and
// shamir_degree_reduce / shamir_open_vec work on device vectors.  The host pair pool below stays for point-sized
// consumers (degree_reduce_point, cs_shamir_state_rand).
#include <algorithm>
#include "cs_lib.cuh"
#include "cs_net.h"
#include "cs_shamir.cuh"

using namespace cs;

struct cs_shamir_state {
  int curve = 0, id = 0, n = 0, t = 0;
  // Montgomery Fr, 4 x u64 each
  std::vector<uint64_t> open_lagrange_t, open_lagrange_2t, mul_lagrange_2t, mul_reconstruct_with_zeros;
  std::vector<uint64_t> r_t, r_2t;  // buffered pairs
  size_t generation_amount = 1024;  // ShamirState::DEFAULT_PAIR_GEN_AMOUNT, doubled on every refill
  HostChaCha rng;
  ShamirWorkspace ws;  // staging of the vector routines, kept between calls
};

namespace {

template <class FrP>
struct ShamirOps {
  typedef host::HFp<FrP> HR;
  static HR from_u(uint64_t v) { return HR::from_u64(v); }
  static HR load(const uint64_t* p) { HR r; memcpy(r.l, p, sizeof(r.l)); return r; }
  static void push(std::vector<uint64_t>& v, const HR& x) { v.insert(v.end(), x.l, x.l + HR::N); }

  // lagrange_from_coeff (shamir.rs:442-461): weights at 0 for the evaluation points `pts`
  static std::vector<uint64_t> lagrange_from_coeff(const std::vector<size_t>& pts) {
    std::vector<uint64_t> out;
    for (size_t i : pts) {
      HR num = HR::one(), den = HR::one();
      const HR fi = from_u(i);
      for (size_t j : pts)
        if (i != j) { const HR fj = from_u(j); num = num * fj; den = den * (fj - fi); }
      push(out, num * den.inverse());
    }
    return out;
  }
  // interpolation_poly_from_zero_points (shamir.rs:571-589): P(0) = 1, P(z) = 0 for z in zero_points
  static std::vector<uint64_t> poly_from_zero_points(const std::vector<size_t>& zeros) {
    std::vector<HR> num{HR::one()};
    HR d = HR::one();
    for (size_t z : zeros) {
      const HR zf = from_u(z);
      num.insert(num.begin(), HR::zero());           // poly_times_root_inplace: multiply by (x - z)
      for (size_t i = 1; i < num.size(); i++) num[i - 1] = num[i - 1] - num[i] * zf;
      d = d * zf.neg();
    }
    const HR c = d.inverse();
    std::vector<uint64_t> out;
    for (auto& x : num) push(out, x * c);
    return out;
  }
  static HR eval_poly(const std::vector<HR>& poly, const HR& x) {  // shamir.rs:335-344
    HR e = poly.back();
    for (size_t i = poly.size() - 1; i-- > 0;) e = e * x + poly[i];
    return e;
  }
  static HR rand(HostChaCha& rng, unsigned bits) {
    HR r;
    rng.template fr_rand<FrP>(r.l, bits);
    return r;
  }
};

unsigned fr_bits(int curve) { return curve == CS_BN254 ? 254 : 255; }

// random_double_share + buffer_triples: `batches` x (t + 1) new pairs
template <class FrP>
int buffer_pairs_t(cs_shamir_state* st, cs_net* net, size_t batches) {
  typedef ShamirOps<FrP> O;
  typedef typename O::HR HR;
  const int n = st->n, t = st->t, id = st->id;
  const unsigned bits = fr_bits(st->curve);
  // my dealings: f_k of degree t, g_k of degree 2t, same constant term
  std::vector<std::vector<HR>> f(batches), g(batches);
  for (size_t k = 0; k < batches; k++) {
    const HR s = O::rand(st->rng, bits);
    f[k].push_back(s);
    g[k].push_back(s);
    for (int d = 0; d < t; d++) f[k].push_back(O::rand(st->rng, bits));
    for (int d = 0; d < 2 * t; d++) g[k].push_back(O::rand(st->rng, bits));
  }
  // rcv[k][src]: the share dealer `src` gave me
  std::vector<std::vector<HR>> rcv_t(batches, std::vector<HR>(n)), rcv_2t(batches, std::vector<HR>(n));
  // all-to-all in n - 1 rounds: round k sends my dealing to party id + k and takes party id - k's (cs_net_sendrecv moves
  // both directions chunk by chunk, so dealings larger than the mailbox credit window cannot dead-lock)
  std::vector<uint64_t> msg(batches * 2 * HR::N), rmsg(batches * 2 * HR::N);
  {
    const HR xi = O::from_u((uint64_t)id + 1);
    for (size_t k = 0; k < batches; k++) { rcv_t[k][id] = O::eval_poly(f[k], xi); rcv_2t[k][id] = O::eval_poly(g[k], xi); }
  }
  for (int round = 1; round < n; round++) {
    const int j = (id + round) % n, src = (id + n - round) % n;
    const HR xj = O::from_u((uint64_t)j + 1);
    for (size_t k = 0; k < batches; k++) {
      const HR a = O::eval_poly(f[k], xj), b = O::eval_poly(g[k], xj);
      memcpy(&msg[(2 * k) * HR::N], a.l, sizeof(a.l));
      memcpy(&msg[(2 * k + 1) * HR::N], b.l, sizeof(b.l));
    }
    CS_TRY(cs_net_sendrecv(net, j, msg.data(), msg.size() * 8, src, rmsg.data(), rmsg.size() * 8));
    for (size_t k = 0; k < batches; k++) {
      rcv_t[k][src] = O::load(&rmsg[(2 * k) * HR::N]);
      rcv_2t[k][src] = O::load(&rmsg[(2 * k + 1) * HR::N]);
    }
  }
  // DN07 extraction with the (t + 1) x n Vandermonde matrix M[row][col] = (col + 1)^row  (rngs.rs:140-157, matmul)
  for (size_t k = 0; k < batches; k++)
    for (int row = 0; row <= t; row++) {
      HR at = HR::zero(), a2t = HR::zero();
      for (int col = 0; col < n; col++) {
        HR m = HR::one();
        const HR c = O::from_u((uint64_t)col + 1);
        for (int e = 0; e < row; e++) m = m * c;
        at = at + rcv_t[k][col] * m;
        a2t = a2t + rcv_2t[k][col] * m;
      }
      O::push(st->r_t, at);
      O::push(st->r_2t, a2t);
    }
  return 0;
}

int buffer_pairs(cs_shamir_state* st, cs_net* net, size_t batches) {
  switch (st->curve) {
    case CS_BN254: return buffer_pairs_t<Bn254Fr>(st, net, batches);
#if defined(CS_ENABLE_BLS12_381)
    case CS_BLS12_381: return buffer_pairs_t<Bls381Fr>(st, net, batches);
#endif
    default: return fail(CS_ERR_ARG, "unsupported curve");
  }
}

// ShamirState::get_pair (shamir.rs:127-143): pops from the back, refills (doubling) when empty
int get_pair(cs_shamir_state* st, cs_net* net, uint64_t* r_t, uint64_t* r_2t) {
  if (st->r_t.empty()) {
    CS_TRY(buffer_pairs(st, net, (st->generation_amount + st->t) / (st->t + 1)));
    st->generation_amount *= 2;
  }
  memcpy(r_t, &st->r_t[st->r_t.size() - 4], 32);
  memcpy(r_2t, &st->r_2t[st->r_2t.size() - 4], 32);
  st->r_t.resize(st->r_t.size() - 4);
  st->r_2t.resize(st->r_2t.size() - 4);
  return 0;
}

template <class FrP>
int state_init_t(cs_shamir_state* st) {
  typedef ShamirOps<FrP> O;
  const size_t n = st->n, t = st->t, id = st->id;
  std::vector<size_t> pts;
  // we send in circles, so we receive from the previous parties (shamir.rs:70-82)
  for (size_t i = 0; i <= t; i++) pts.push_back((id + n - i) % n + 1);
  st->open_lagrange_t = O::lagrange_from_coeff(pts);
  pts.clear();
  for (size_t i = 0; i <= 2 * t; i++) pts.push_back((id + n - i) % n + 1);
  st->open_lagrange_2t = O::lagrange_from_coeff(pts);
  pts.clear();
  for (size_t i = 1; i <= 2 * t + 1; i++) pts.push_back(i);
  st->mul_lagrange_2t = O::lagrange_from_coeff(pts);
  // the king shares <acc> as a known polynomial with t zero shares (shamir.rs:87-91)
  const size_t num_non_zero = n - t;
  pts.clear();
  for (size_t z = num_non_zero + 1; z <= n; z++) pts.push_back(z);
  st->mul_reconstruct_with_zeros = O::poly_from_zero_points(pts);
  return 0;
}

constexpr int KING_ID = 0;

// degree_reduce_point (network.rs:246-301) for a G1/G2 point given as affine Montgomery limbs
template <class Cfg, int G>
int degree_reduce_point_t(cs_shamir_state* st, cs_net* net, const uint64_t* base, const uint64_t* in, uint64_t* out) {
  typedef typename GroupOf<Cfg, G>::HF HF;
  typedef host::HXyzz<HF> X;
  typedef host::HAffine<HF> A;
  typedef host::HFp<typename Cfg::FrP> HR;
  const size_t PL = sizeof(A) / 8;
  auto load = [](const uint64_t* p) { A a; memcpy(&a, p, sizeof(a)); return X::from_affine(a); };
  auto store = [](uint64_t* o, const X& x) { A a = host::haffine(x); memcpy(o, &a, sizeof(a)); };
  auto mul_mont = [](const X& p, const uint64_t* s) { HR v; memcpy(v.l, s, sizeof(v.l)); HR c = v.from_mont(); return host::hmul(p, c.l, HR::N); };
  const int n = st->n, t = st->t, id = st->id;
  const int num_non_zero = n - t;
  uint64_t rt[4], r2t[4];
  CS_TRY(get_pair(st, net, rt, r2t));
  const X Gb = load(base);
  const X Rt = mul_mont(Gb, rt), R2t = mul_mont(Gb, r2t);
  const X input = host::hadd(load(in), R2t);
  X mine = X::inf();
  std::vector<uint64_t> buf(PL);
  if (id == KING_ID) {
    X acc = X::inf();
    for (int other = 0; other <= 2 * t; other++) {  // mul_lagrange_2t has 2t + 1 entries: parties 0..2t
      X v = input;
      if (other != KING_ID) { CS_TRY(cs_net_recv(net, other, buf.data(), PL * 8)); v = load(buf.data()); }
      acc = host::hadd(acc, mul_mont(v, &st->mul_lagrange_2t[4 * other]));
    }
    // poly = acc * precomputed (poly_with_zeros_from_precomputed_point), evaluated at id + 1 (Horner on points)
    const size_t plen = st->mul_reconstruct_with_zeros.size() / 4;
    for (int rid = 0; rid < num_non_zero; rid++) {
      HR x = HR::from_u64((uint64_t)rid + 1);
      // scalar Horner first, then one point multiplication: sum_k acc c_k x^k = acc * P(x)
      HR e;
      memcpy(e.l, &st->mul_reconstruct_with_zeros[4 * (plen - 1)], sizeof(e.l));
      for (size_t k = plen - 1; k-- > 0;) { HR c; memcpy(c.l, &st->mul_reconstruct_with_zeros[4 * k], sizeof(c.l)); e = e * x + c; }
      const X val = mul_mont(acc, e.l);
      if (rid == id) mine = val;
      else { store(buf.data(), val); CS_TRY(cs_net_send(net, rid, buf.data(), PL * 8)); }
    }
  } else {
    if (id <= 2 * t) { store(buf.data(), input); CS_TRY(cs_net_send(net, KING_ID, buf.data(), PL * 8)); }
    if (id < num_non_zero) { CS_TRY(cs_net_recv(net, KING_ID, buf.data(), PL * 8)); mine = load(buf.data()); }
  }
  store(out, host::hadd(mine, host::hneg(Rt)));
  return 0;
}

// open_point_many (pointshare.rs:129) / open_half_point (:102-111): broadcast_next over d + 1 parties (d = t or 2t),
// Lagrange-weighted sum, for `k` points in place
template <class Cfg, int G>
int open_points_t(cs_shamir_state* st, cs_net* net, int degree_2t, uint64_t* pts, size_t k) {
  typedef typename GroupOf<Cfg, G>::HF HF;
  typedef host::HXyzz<HF> X;
  typedef host::HAffine<HF> A;
  typedef host::HFp<typename Cfg::FrP> HR;
  const size_t PL = sizeof(A) / 8;
  auto load = [](const uint64_t* p) { A a; memcpy(&a, p, sizeof(a)); return X::from_affine(a); };
  auto mul_mont = [](const X& p, const uint64_t* s) { HR v; memcpy(v.l, s, sizeof(v.l)); HR c = v.from_mont(); return host::hmul(p, c.l, HR::N); };
  const int n = st->n, num = (degree_2t ? 2 * st->t : st->t) + 1, id = st->id;
  const std::vector<uint64_t>& lag = degree_2t ? st->open_lagrange_2t : st->open_lagrange_t;
  for (int s = 1; s < num; s++) CS_TRY(cs_net_send(net, (id + s) % n, pts, k * PL * 8));
  std::vector<X> acc(k);
  for (size_t i = 0; i < k; i++) acc[i] = mul_mont(load(pts + i * PL), &lag[0]);
  std::vector<uint64_t> buf(k * PL);
  for (int r = 1; r < num; r++) {
    CS_TRY(cs_net_recv(net, (id + n - r) % n, buf.data(), k * PL * 8));
    for (size_t i = 0; i < k; i++) acc[i] = host::hadd(acc[i], mul_mont(load(buf.data() + i * PL), &lag[4 * r]));
  }
  for (size_t i = 0; i < k; i++) {
    A a = host::haffine(acc[i]);
    memcpy(pts + i * PL, &a, sizeof(a));
  }
  return 0;
}

}  // namespace

namespace cs {

// Batches (t + 1 pairs each) per dealing round: bounds the device and host staging of one round to ~(3t + 2n + 3)
// x 32 MB and makes every round take a fresh seed.
constexpr size_t PAIR_BATCHES_MAX = (size_t)1 << 20;

// random_double_share + buffer_triples (rngs.rs:334-470) on device vectors.  Coefficient vectors, structure of arrays
// over the B batches of a round: [0] s, [1..t] f_1..f_t, [t+1..3t] g_1..g_2t, so that f = s + f_1 x + ... and
// g = s + g_1 x + ... share their constant term.  Dealing at x = j + 1 is one k_vec_lincomb per degree, the
// extraction one per Vandermonde row; pair (row, k) lands at index row B + k of the round's output range.
int shamir_double_sharings(cs_ctx* ctx, cs_shamir_state* st, cs_net* net, size_t count, uint64_t* d_rt, uint64_t* d_r2t) {
  if (count == 0) return 0;
  const int n = st->n, t = st->t, id = st->id;
  if (n > (int)LINCOMB_MAX) return fail(CS_ERR_LIMIT, "shamir_double_sharings: %d parties exceed %u", n, LINCOMB_MAX);
  const cs_curve cv = (cs_curve)st->curve;
  const size_t nc = 3 * (size_t)t + 1;
  CS_CUDA(cudaSetDevice(ctx->device));
  const size_t bmax = std::min(PAIR_BATCHES_MAX, (count + t) / (t + 1));
  ShamirWorkspace& ws = st->ws;
  DevBuf &coef = ws.coef, &rcv = ws.rcv, &msg = ws.msg;
  CS_TRY(coef.reserve(nc * bmax * 32));
  CS_TRY(rcv.reserve(2 * (size_t)n * bmax * 32));
  CS_TRY(msg.reserve(2 * bmax * 32));
  uint64_t* hs = ws.host0(2 * bmax * 4);
  uint64_t* hr = ws.host1(2 * bmax * 4);
  // w[e] = x^e in Montgomery form, e <= 2t
  auto powers = [&](uint64_t x, uint64_t* w, int m) {
    uint64_t c[4] = {x, 0, 0, 0}, xm[4];
    cs_fr_to_mont(cv, c, xm, 1);
    const uint64_t one[4] = {1, 0, 0, 0};
    cs_fr_to_mont(cv, one, w, 1);
    for (int e = 1; e < m; e++) cs_fr_mul(cv, w + 4 * (e - 1), xm, w + 4 * e);
  };
  auto cvec = [&](size_t j, size_t B) { return coef.as<uint64_t>() + j * B * 4; };
  for (size_t done = 0; done < count;) {
    const size_t todo = std::min(count - done, (size_t)(t + 1) * bmax);
    const size_t B = (todo + t) / (t + 1);
    uint8_t seed[32];
    st->rng.gen_seed(seed);  // one seed per dealing round, never reused
    CS_TRY(cs_fr_rand_device(ctx, cv, seed, 0, coef.as<uint64_t>(), nc * B));
    auto deal = [&](int j, uint64_t* out_t, uint64_t* out_2t) -> int {  // f(j + 1), g(j + 1)
      uint64_t w[4 * LINCOMB_MAX];
      powers((uint64_t)j + 1, w, 2 * t + 1);
      const uint64_t* in[LINCOMB_MAX];
      for (int d = 0; d <= t; d++) in[d] = cvec(d, B);
      CS_TRY(cs_vec_lincomb(ctx, cv, in, w, t + 1, B, out_t));
      for (int d = 1; d <= 2 * t; d++) in[d] = cvec(t + d, B);
      return cs_vec_lincomb(ctx, cv, in, w, 2 * t + 1, B, out_2t);
    };
    auto rt_of = [&](int src) { return rcv.as<uint64_t>() + (size_t)src * B * 4; };
    auto r2t_of = [&](int src) { return rcv.as<uint64_t>() + (size_t)(n + src) * B * 4; };
    CS_TRY(deal(id, rt_of(id), r2t_of(id)));
    // all-to-all in n - 1 rounds: round k sends my dealing to party id + k and takes party id - k's
    for (int round = 1; round < n; round++) {
      const int j = (id + round) % n, src = (id + n - round) % n;
      CS_TRY(deal(j, msg.as<uint64_t>(), msg.as<uint64_t>() + B * 4));
      CS_CUDA(cudaMemcpyAsync(hs, msg.p, 2 * B * 32, cudaMemcpyDeviceToHost, ctx->stream));
      CS_CUDA(cudaStreamSynchronize(ctx->stream));
      CS_TRY(cs_net_sendrecv(net, j, hs, 2 * B * 32, src, hr, 2 * B * 32));
      CS_CUDA(cudaMemcpyAsync(rt_of(src), hr, B * 32, cudaMemcpyHostToDevice, ctx->stream));
      CS_CUDA(cudaMemcpyAsync(r2t_of(src), hr + B * 4, B * 32, cudaMemcpyHostToDevice, ctx->stream));
      CS_CUDA(cudaStreamSynchronize(ctx->stream));  // hr is reused by the next round
    }
    // DN07 extraction with the (t + 1) x n Vandermonde matrix M[row][col] = (col + 1)^row  (rngs.rs:140-157)
    for (int row = 0; row <= t; row++) {
      const size_t lo = (size_t)row * B;
      if (lo >= todo) break;
      const size_t len = std::min(B, todo - lo);
      uint64_t w[4 * LINCOMB_MAX];
      const uint64_t* in_t[LINCOMB_MAX];
      const uint64_t* in_2t[LINCOMB_MAX];
      for (int col = 0; col < n; col++) {
        uint64_t p[4 * (2 * LINCOMB_MAX)];
        powers((uint64_t)col + 1, p, row + 1);
        memcpy(w + 4 * col, p + 4 * row, 32);
        in_t[col] = rt_of(col);
        in_2t[col] = r2t_of(col);
      }
      CS_TRY(cs_vec_lincomb(ctx, cv, in_t, w, n, len, d_rt + (done + lo) * 4));
      CS_TRY(cs_vec_lincomb(ctx, cv, in_2t, w, n, len, d_r2t + (done + lo) * 4));
    }
    done += todo;
  }
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return 0;
}

// degree_reduce_many (network.rs:150-243): inp += r_2t; parties 1..2t send to the king (party 0), which accumulates
// with the Lagrange weights (one k_vec_lincomb launch, k = 2t + 1), shares the result as a known polynomial with t zero
// shares and sends acc * P(id + 1) to parties 0..n-t-1; share -= r_t.
int shamir_degree_reduce(cs_ctx* ctx, cs_shamir_state* st, cs_net* net, const uint64_t* d_in, size_t len, uint64_t* d_out,
                         const uint64_t* d_rt, uint64_t* d_r2t) {
  if (len == 0) return 0;
  const int n = st->n, t = st->t, id = st->id, num_non_zero = n - t;
  CS_CUDA(cudaSetDevice(ctx->device));
  const cs_curve cv = (cs_curve)st->curve;
  DevBuf* d_stage = st->ws.stage;
  // inp += r_2t
  CS_TRY(cs_vec_add(ctx, cv, d_in, d_r2t, d_out, len));
  uint64_t* host = st->ws.host0(len * 4);
  int rc = 0;
  if (id == KING_ID) {
    // acc = sum_j lagrange_j * inputs_j over parties 0..2t: one k_vec_lincomb launch with k = 2t + 1
    const uint64_t* ins[LINCOMB_MAX];
    ins[0] = d_out;
    for (int other = 1; other <= 2 * t && !rc; other++) {
      rc = cs_net_recv(net, other, host, len * 32);
      if (rc) break;
      rc = d_stage[other].reserve(len * 32);
      if (rc) break;
      CS_CUDA(cudaMemcpyAsync(d_stage[other].p, host, len * 32, cudaMemcpyHostToDevice, ctx->stream));
      CS_CUDA(cudaStreamSynchronize(ctx->stream));  // `host` is reused for the next party
      ins[other] = d_stage[other].as<uint64_t>();
    }
    DevBuf& d_acc = st->ws.acc;
    if (!rc) rc = d_acc.reserve(len * 32);
    if (!rc) rc = cs_vec_lincomb(ctx, cv, ins, st->mul_lagrange_2t.data(), 2 * t + 1, len, d_acc.as<uint64_t>());
    // fresh shares: poly = acc * precomputed, share_id = acc * P(id + 1) -- one scalar per recipient
    for (int rid = 0; rid < num_non_zero && !rc; rid++) {
      uint64_t c[4];
      {
        const size_t plen = st->mul_reconstruct_with_zeros.size() / 4;
        // Horner in Fr on the host through the ABI's scalar helpers
        memcpy(c, &st->mul_reconstruct_with_zeros[4 * (plen - 1)], 32);
        uint64_t x_can[4] = {(uint64_t)rid + 1, 0, 0, 0}, x[4];
        cs_fr_to_mont(cv, x_can, x, 1);
        for (size_t k = plen - 1; k-- > 0;) {
          cs_fr_mul(cv, c, x, c);
          cs_fr_add(cv, c, &st->mul_reconstruct_with_zeros[4 * k], c);
        }
      }
      const uint64_t* one_in[1] = {d_acc.as<uint64_t>()};
      uint64_t* dst = rid == id ? d_out : d_r2t;  // r_2t is no longer needed: reuse as staging
      rc = cs_vec_lincomb(ctx, cv, one_in, c, 1, len, dst);
      if (rc || rid == id) continue;
      CS_CUDA(cudaMemcpyAsync(host, dst, len * 32, cudaMemcpyDeviceToHost, ctx->stream));
      CS_CUDA(cudaStreamSynchronize(ctx->stream));
      rc = cs_net_send(net, rid, host, len * 32);
    }
  } else {
    if (id <= 2 * t) {  // only send if my items are required
      CS_CUDA(cudaMemcpyAsync(host, d_out, len * 32, cudaMemcpyDeviceToHost, ctx->stream));
      CS_CUDA(cudaStreamSynchronize(ctx->stream));
      rc = cs_net_send(net, KING_ID, host, len * 32);
    }
    if (!rc) {
      if (id < num_non_zero) {
        rc = cs_net_recv(net, KING_ID, host, len * 32);
        if (!rc) CS_CUDA(cudaMemcpyAsync(d_out, host, len * 32, cudaMemcpyHostToDevice, ctx->stream));
      } else {
        CS_CUDA(cudaMemsetAsync(d_out, 0, len * 32, ctx->stream));
      }
    }
  }
  // share -= r_t
  if (!rc) rc = cs_vec_sub(ctx, cv, d_out, d_rt, d_out, len);
  if (!rc) CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return rc;
}

// open_vec (shamir/arithmetic.rs:191) on a device vector: my shares go to the next d parties, the previous d parties'
// arrive (one sendrecv per distance, so vectors larger than the mailbox credit window cannot dead-lock), and the
// Lagrange sum is one k_vec_lincomb launch with k = d + 1.  mul_open_vec (:262) is a local product kernel, then this.
int shamir_open_vec(cs_ctx* ctx, cs_shamir_state* st, cs_net* net, int degree_2t, const uint64_t* d_in, size_t len, uint64_t* d_out) {
  if (len == 0) return 0;
  const int n = st->n, id = st->id, d = degree_2t ? 2 * st->t : st->t;
  const cs_curve cv = (cs_curve)st->curve;
  CS_CUDA(cudaSetDevice(ctx->device));
  uint64_t* mine = st->ws.host0(len * 4);
  uint64_t* rcv = st->ws.host1(len * 4);
  CS_CUDA(cudaMemcpyAsync(mine, d_in, len * 32, cudaMemcpyDeviceToHost, ctx->stream));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  DevBuf* stage = st->ws.stage;
  const uint64_t* ins[LINCOMB_MAX];
  ins[0] = d_in;
  int rc = 0;
  for (int r = 1; r <= d && !rc; r++) {
    rc = cs_net_sendrecv(net, (id + r) % n, mine, len * 32, (id + n - r) % n, rcv, len * 32);
    if (!rc) rc = stage[r].reserve(len * 32);
    if (rc) break;
    CS_CUDA(cudaMemcpyAsync(stage[r].p, rcv, len * 32, cudaMemcpyHostToDevice, ctx->stream));
    CS_CUDA(cudaStreamSynchronize(ctx->stream));  // rcv is reused
    ins[r] = stage[r].as<uint64_t>();
  }
  const std::vector<uint64_t>& lag = degree_2t ? st->open_lagrange_2t : st->open_lagrange_t;
  if (!rc) rc = cs_vec_lincomb(ctx, cv, ins, lag.data(), d + 1, len, d_out);
  if (!rc) CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return rc;
}

// open_vec on a handful of scalars (host)
int shamir_open_scalars(cs_shamir_state* st, cs_net* net, int degree_2t, uint64_t* v, size_t k) {
  const int n = st->n, id = st->id, d = degree_2t ? 2 * st->t : st->t;
  const cs_curve cv = (cs_curve)st->curve;
  const std::vector<uint64_t>& lag = degree_2t ? st->open_lagrange_2t : st->open_lagrange_t;
  for (int s = 1; s <= d; s++) CS_TRY(cs_net_send(net, (id + s) % n, v, k * 32));
  std::vector<uint64_t> acc(k * 4), buf(k * 4), term(4);
  for (size_t i = 0; i < k; i++) CS_TRY(cs_fr_mul(cv, v + 4 * i, &lag[0], &acc[4 * i]));
  for (int r = 1; r <= d; r++) {
    CS_TRY(cs_net_recv(net, (id + n - r) % n, buf.data(), k * 32));
    for (size_t i = 0; i < k; i++) {
      CS_TRY(cs_fr_mul(cv, &buf[4 * i], &lag[4 * r], term.data()));
      CS_TRY(cs_fr_add(cv, &acc[4 * i], term.data(), &acc[4 * i]));
    }
  }
  memcpy(v, acc.data(), k * 32);
  return 0;
}

int shamir_open_points(cs_shamir_state* st, cs_net* net, cs_group group, int degree_2t, uint64_t* pts, size_t k) {
  CS_DISPATCH_CURVE(st->curve, {
    if (group == CS_G1) return open_points_t<Cfg, 0>(st, net, degree_2t, pts, k);
    return open_points_t<Cfg, 1>(st, net, degree_2t, pts, k);
  });
  return 0;
}

size_t shamir_state_device_bytes(const cs_shamir_state* st) { return st ? st->ws.device_bytes() : 0; }

}  // namespace cs

extern "C" {

int cs_shamir_state_create(cs_net* net, cs_curve curve, int num_parties, int threshold, size_t amount, cs_shamir_state** out) {
  if (!net || !out) return fail(CS_ERR_ARG, "cs_shamir_state_create: NULL argument");
  if (curve != CS_BN254 && curve != CS_BLS12_381) return fail(CS_ERR_ARG, "cs_shamir_state_create: unsupported curve");
  if (threshold < 1 || 2 * threshold + 1 > num_parties) return fail(CS_ERR_ARG, "Threshold too large for number of parties");  // shamir.rs:41-43
  if (net->n != num_parties) return fail(CS_ERR_ARG, "cs_shamir_state_create: the net has %d parties, %d expected", net->n, num_parties);
  if (2 * threshold + 1 > (int)LINCOMB_MAX) return fail(CS_ERR_LIMIT, "cs_shamir_state_create: 2t + 1 = %d exceeds %u", 2 * threshold + 1, LINCOMB_MAX);
  std::unique_ptr<cs_shamir_state> st(new cs_shamir_state());
  st->curve = curve; st->id = net->id; st->n = num_parties; st->t = threshold;
  uint8_t seed[32];
  CS_TRY(cs_os_random(seed, 32));  // RngType::from_entropy (shamir.rs:46)
  st->rng.init(seed, 0);
  if (curve == CS_BN254) CS_TRY(state_init_t<Bn254Fr>(st.get()));
#if defined(CS_ENABLE_BLS12_381)
  else CS_TRY(state_init_t<Bls381Fr>(st.get()));
#endif
  if (amount) CS_TRY(buffer_pairs(st.get(), net, (amount + threshold) / (threshold + 1)));
  *out = st.release();
  return 0;
}

void cs_shamir_state_free(cs_shamir_state* st) { delete st; }

size_t cs_shamir_state_pairs(const cs_shamir_state* st) { return st ? st->r_t.size() / 4 : 0; }

// MpcState::fork (shamir.rs:172-186): the child takes `amount` pairs from the front of the parent's buffer
int cs_shamir_state_fork(cs_shamir_state* st, size_t amount, cs_shamir_state** out) {
  if (!st || !out) return fail(CS_ERR_ARG, "cs_shamir_state_fork: NULL argument");
  if (amount * 4 > st->r_t.size()) return fail(CS_ERR_STATE, "not enough corr rand pairs");
  std::unique_ptr<cs_shamir_state> c(new cs_shamir_state(*st));
  c->r_t.assign(st->r_t.begin(), st->r_t.begin() + amount * 4);
  c->r_2t.assign(st->r_2t.begin(), st->r_2t.begin() + amount * 4);
  st->r_t.erase(st->r_t.begin(), st->r_t.begin() + amount * 4);
  st->r_2t.erase(st->r_2t.begin(), st->r_2t.begin() + amount * 4);
  uint8_t s[32];
  st->rng.gen_seed(s);
  c->rng.init(s, 0);
  *out = c.release();
  return 0;
}

// ShamirState::rand (shamir.rs:160-163)
int cs_shamir_state_rand(cs_shamir_state* st, cs_net* net, uint64_t* out_share) {
  if (!st || !net || !out_share) return fail(CS_ERR_ARG, "cs_shamir_state_rand: NULL argument");
  uint64_t r2t[4];
  return get_pair(st, net, out_share, r2t);
}

int cs_shamir_open_lagrange(const cs_shamir_state* st, int degree_2t, uint64_t* out, size_t capacity_elems, size_t* out_n) {
  if (!st || !out_n) return fail(CS_ERR_ARG, "cs_shamir_open_lagrange: NULL argument");
  const std::vector<uint64_t>& v = degree_2t ? st->open_lagrange_2t : st->open_lagrange_t;
  *out_n = v.size() / 4;
  if (!out) return 0;
  if (capacity_elems < v.size() / 4) return fail(CS_ERR_ARG, "cs_shamir_open_lagrange: buffer too small");
  memcpy(out, v.data(), v.size() * 8);
  return 0;
}

// degree_reduce_many (network.rs:150-243) on a device-resident vector of degree-2t values, pairs uploaded from the
// host pool in the order get_pair hands them out; the reduction itself is shamir_degree_reduce.
int cs_shamir_degree_reduce_many(cs_ctx* ctx, cs_shamir_state* st, cs_net* net, const uint64_t* d_in, size_t len, uint64_t* d_out) {
  if (!ctx || !st || !net || (len && (!d_in || !d_out))) return fail(CS_ERR_ARG, "cs_shamir_degree_reduce_many: NULL argument");
  if (len == 0) return 0;
  CS_CUDA(cudaSetDevice(ctx->device));
  std::vector<uint64_t> rt(len * 4), r2t(len * 4);
  for (size_t i = 0; i < len; i++) CS_TRY(get_pair(st, net, &rt[4 * i], &r2t[4 * i]));
  ScopedBuf d_rt, d_r2t;
  CS_TRY(d_rt.reserve(len * 32));
  CS_TRY(d_r2t.reserve(len * 32));
  CS_CUDA(cudaMemcpyAsync(d_rt.p, rt.data(), len * 32, cudaMemcpyHostToDevice, ctx->stream));
  CS_CUDA(cudaMemcpyAsync(d_r2t.p, r2t.data(), len * 32, cudaMemcpyHostToDevice, ctx->stream));
  return shamir_degree_reduce(ctx, st, net, d_in, len, d_out, d_rt.as<uint64_t>(), d_r2t.as<uint64_t>());
}

int cs_shamir_double_sharings(cs_ctx* ctx, cs_shamir_state* st, cs_net* net, size_t count, uint64_t* d_rt, uint64_t* d_r2t) {
  if (!ctx || !st || !net || (count && (!d_rt || !d_r2t))) return fail(CS_ERR_ARG, "cs_shamir_double_sharings: NULL argument");
  if (net->n != st->n || net->id != st->id)
    return fail(CS_ERR_ARG, "cs_shamir_double_sharings: the net is party %d of %d, the state party %d of %d", net->id, net->n, st->id, st->n);
  return shamir_double_sharings(ctx, st, net, count, d_rt, d_r2t);
}

int cs_shamir_degree_reduce_point(cs_shamir_state* st, cs_net* net, cs_group group, const uint64_t* base_affine,
                                  const uint64_t* in_affine, uint64_t* out_affine) {
  if (!st || !net || !base_affine || !in_affine || !out_affine) return fail(CS_ERR_ARG, "cs_shamir_degree_reduce_point: NULL argument");
  CS_DISPATCH_CURVE(st->curve, {
    if (group == CS_G1) return degree_reduce_point_t<Cfg, 0>(st, net, base_affine, in_affine, out_affine);
    return degree_reduce_point_t<Cfg, 1>(st, net, base_affine, in_affine, out_affine);
  });
  return 0;
}

int cs_shamir_open_half_point(cs_shamir_state* st, cs_net* net, cs_group group, const uint64_t* in_affine, uint64_t* out_affine) {
  if (!st || !net || !in_affine || !out_affine) return fail(CS_ERR_ARG, "cs_shamir_open_half_point: NULL argument");
  if (out_affine != in_affine) memmove(out_affine, in_affine, point_limbs64(st->curve, group) * 8);
  return shamir_open_points(st, net, group, 1, out_affine, 1);
}

}  // extern "C"
