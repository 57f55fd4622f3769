// Rep3 co-Plonk: the share-level kernels.  A party holds replicated shares {a, b} = (x_i, x_{i-1}) interleaved
// (mpc-core/src/protocols/rep3/arithmetic/types.rs:21-28).  Linear steps act per component; a product is the
// local cross-term sum a.a b.a + a.a b.b + a.b b.a plus a zero-sum ChaCha mask (rep3/arithmetic.rs:132-146,
// rngs.rs:103-106), and when the result is needed as a replicated share again it is stored both into this
// party's vector (.a) and into the NEXT party's (.b) through a peer pointer (reshare_vec, arithmetic.rs:149-160).
//
// What the reference computes with ~60 mul_vec round trips per proof (round2.rs:150-190 array_prod_mul,
// round3.rs:20-108 mul4vec) is organised here so that a share only crosses NVLink when a later product needs
// both of its halves:
//   round 2: two product layers for num/den, one masked inversion, one masked prefix product  (6 exchanges)
//   round 3: twelve first-layer products per extended-domain point (one exchange); every product above them
//            is evaluated locally into ADDITIVE shares of t and tz -- from there to the opened commitments and
//            evaluations everything is linear, so rounds 3b-5 run the plain kernels on additive shares.
// The opened proof equals the plain prover's for blinders b = sum of the parties' shares (masks cancel), which
// is what the parity tests check.
//
// The Shamir session (cs_plonk_shamir) runs the same kernel bodies over ShamirPol: a share is one element of a
// degree-t sharing, a product is the plain local product (degree 2t) and the caller degree-reduces each product layer
// with one king round; the layer above the last reduction (t, tz in round 3) stays at degree 2t.
#pragma once
#include "cs_plonk.cuh"
#include "cs_prf.cuh"

namespace cs {

template <class FrP>
struct Sh {
  Fp<FrP> a, b;
};
struct PrfArgs {
  PrfKeys keys;          // key1 = own stream, key2 = previous party's
  uint64_t pos1, pos2;   // word positions of element 0
  uint32_t rounds;
};
struct ShConst { uint32_t v[2][8]; };  // a share passed by value

template <class FrP> CS_D Sh<FrP> ld_sh(const uint32_t* p, size_t i) {
  Sh<FrP> s;
  s.a = ld_fr<FrP>(p + (2 * i) * FrP::N);
  s.b = ld_fr<FrP>(p + (2 * i + 1) * FrP::N);
  return s;
}
template <class FrP> CS_D void st_sh(uint32_t* p, size_t i, const Sh<FrP>& s) {
  st_fr<FrP>(p + (2 * i) * FrP::N, s.a);
  st_fr<FrP>(p + (2 * i + 1) * FrP::N, s.b);
}
// product result z: this party's .a, the next party's .b
template <class FrP> CS_D void st_reshare(uint32_t* mine, uint32_t* next, size_t i, const Fp<FrP>& z) {
  st_fr<FrP>(mine + (2 * i) * FrP::N, z);
  if (next) st_fr<FrP>(next + (2 * i + 1) * FrP::N, z);
}
template <class FrP> CS_D Sh<FrP> sh_const(const ShConst& c) {
  Sh<FrP> s;
  s.a = cload<FrP>(c.v[0]);
  s.b = cload<FrP>(c.v[1]);
  return s;
}
template <class FrP> CS_D Sh<FrP> sh_add(const Sh<FrP>& x, const Sh<FrP>& y) { return Sh<FrP>{x.a + y.a, x.b + y.b}; }
template <class FrP> CS_D Sh<FrP> sh_mulp(const Sh<FrP>& x, const Fp<FrP>& p) { return Sh<FrP>{x.a * p, x.b * p}; }
// add_with_public (rep3/arithmetic.rs:52-58): the public value lives in x_0 = party 0's a = party 1's b
template <class FrP> CS_D Sh<FrP> sh_addp(const Sh<FrP>& x, const Fp<FrP>& p, int party) {
  Sh<FrP> r = x;
  if (party == 0) r.a = r.a + p;
  if (party == 1) r.b = r.b + p;
  return r;
}
template <class FrP> CS_D Fp<FrP> sh_lmul(const Sh<FrP>& x, const Sh<FrP>& y) { return Fp<FrP>::dot2(x.a, y.a + y.b, x.b, y.a); }  // one reduction for both products
template <class FrP> CS_D Fp<FrP> prf_mask(const PrfArgs& P, uint64_t idx) {
  return prf_field_element<FrP>(P.keys.k, P.pos1 + 8 * idx, P.rounds) - prf_field_element<FrP>(P.keys.k + 8, P.pos2 + 8 * idx, P.rounds);
}
// arithmetic::rand: (F(rng1), F(rng2)).  Random share number `j` of the region that starts at element index `rbase`
// takes TWO element slots (64 bytes) of each stream: a 64-byte draw is uniform up to 2^-256 (the reference uses
// F::rand's rejection sampling, arithmetic.rs:357-360).
template <class FrP> CS_D Sh<FrP> prf_share(const PrfArgs& P, uint64_t rbase, uint64_t j) {
  const uint64_t w = 8 * (rbase + 2 * j);
  return Sh<FrP>{prf_field_element_wide<FrP>(P.keys.k, P.pos1 + w, P.rounds), prf_field_element_wide<FrP>(P.keys.k + 8, P.pos2 + w, P.rounds)};
}

// ---- share policies -------------------------------------------------------------------------------------
// The round-2/3 kernels below are written once over a share policy:
//   Rep3Pol<FrP>    replicated {a, b}; a product is the masked cross-term sum, stored into this party's .a and the
//                   next party's .b; random shares come from the correlated ChaCha streams; public values enter the
//                   x_0 component; the additive part of a linear expression is .a
//   ShamirPol<FrP>  one Fr element of a degree-t sharing; a product is the plain local product (degree 2t, reduced by
//                   the caller); random shares are r_t halves of device double sharings; every party adds public values
template <class FrP_>
struct Rep3Pol {
  typedef FrP_ FrP;
  typedef Fp<FrP> F;
  typedef Sh<FrP> S;
  typedef PrfArgs Rnd;
  static CS_D S ld(const uint32_t* p, size_t i) { return ld_sh<FrP>(p, i); }
  static CS_D void st(uint32_t* p, size_t i, const S& s) { st_sh<FrP>(p, i, s); }
  static CS_D S cnst(const ShConst& c) { return sh_const<FrP>(c); }
  static CS_D S add(const S& x, const S& y) { return sh_add<FrP>(x, y); }
  static CS_D S mulp(const S& x, const F& p) { return sh_mulp<FrP>(x, p); }
  static CS_D S addp(const S& x, const F& p, int party) { return sh_addp<FrP>(x, p, party); }
  static CS_D F lmul(const S& x, const S& y) { return sh_lmul<FrP>(x, y); }
  static CS_D F part(const S& x) { return x.a; }
  static CS_D bool pub(int party) { return party == 0; }
  static CS_D F masked(const F& z, const Rnd& P, uint64_t idx) { return z + prf_mask<FrP>(P, idx); }
  static CS_D S rand(const Rnd& P, uint64_t rbase, uint64_t j) { return prf_share<FrP>(P, rbase, j); }
  static CS_D void st_prod(uint32_t* mine, uint32_t* next, size_t i, const F& z) { st_reshare<FrP>(mine, next, i, z); }
};
struct ShamirRnd { const uint32_t* r; };  // random degree-t shares
template <class FrP_>
struct ShamirPol {
  typedef FrP_ FrP;
  typedef Fp<FrP> F;
  typedef Fp<FrP> S;
  typedef ShamirRnd Rnd;
  static CS_D S ld(const uint32_t* p, size_t i) { return ld_fr<FrP>(p + i * FrP::N); }
  static CS_D void st(uint32_t* p, size_t i, const S& s) { st_fr<FrP>(p + i * FrP::N, s); }
  static CS_D S cnst(const ShConst& c) { return cload<FrP>(c.v[0]); }
  static CS_D S add(const S& x, const S& y) { return x + y; }
  static CS_D S mulp(const S& x, const F& p) { return x * p; }
  static CS_D S addp(const S& x, const F& p, int) { return x + p; }
  static CS_D F lmul(const S& x, const S& y) { return x * y; }
  static CS_D F part(const S& x) { return x; }
  static CS_D bool pub(int) { return true; }
  static CS_D F masked(const F& z, const Rnd&, uint64_t) { return z; }
  static CS_D S rand(const Rnd& P, uint64_t rbase, uint64_t j) { return ld_fr<FrP>(P.r + (rbase + j) * FrP::N); }
  static CS_D void st_prod(uint32_t* mine, uint32_t*, size_t i, const F& z) { st_fr<FrP>(mine + i * FrP::N, z); }
};

struct R3Round2In {
  const uint32_t *a, *b, *c;        // wire buffers, n shares each
  const uint32_t *s1, *s2, *s3;     // sigma evaluations (4n, read at stride 4)
  const uint32_t* tw4;
};
// numerator / denominator factors of z (round2.rs:113-146), k = 0..2
template <class Pol>
CS_D void r3_factors(const R3Round2In& in, const PlonkConsts& K, uint32_t n, uint32_t i, int party, int k, typename Pol::S& nf,
                     typename Pol::S& df) {
  typedef typename Pol::FrP FrP;
  typedef Fp<FrP> F;
  constexpr int NW = FrP::N;
  F beta = cload<FrP>(K.beta), gamma = cload<FrP>(K.gamma);
  F bw = beta * root_pow<FrP>(in.tw4, 2 * n, 4 * i);
  const uint32_t* wire = k == 0 ? in.a : (k == 1 ? in.b : in.c);
  const uint32_t* sig = k == 0 ? in.s1 : (k == 1 ? in.s2 : in.s3);
  typename Pol::S x = Pol::ld(wire, i);
  F kk = k == 0 ? F::one() : cload<FrP>(k == 1 ? K.k1 : K.k2);
  nf = Pol::addp(x, kk * bw + gamma, party);
  df = Pol::addp(x, beta * ld_fr<FrP>(sig + (size_t)(4 * i) * NW) + gamma, party);
}

// layer 1: n12 = n1 n2, d12 = d1 d2  -> slots o_n, o_d (reshared)
template <class Pol>
CS_GLOBAL void k_r3_round2_a(R3Round2In in, PlonkConsts K, uint32_t n, int party, typename Pol::Rnd P, uint64_t mbase,
                              uint32_t* on, uint32_t* od, uint32_t* pn, uint32_t* pd) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  typename Pol::S n1, d1, n2, d2;
  r3_factors<Pol>(in, K, n, i, party, 0, n1, d1);
  r3_factors<Pol>(in, K, n, i, party, 1, n2, d2);
  Pol::st_prod(on, pn, i, Pol::masked(Pol::lmul(n1, n2), P, mbase + i));
  Pol::st_prod(od, pd, i, Pol::masked(Pol::lmul(d1, d2), P, mbase + n + i));
}
// layer 2: num = n12 n3, den = d12 d3
template <class Pol>
CS_GLOBAL void k_r3_round2_b(R3Round2In in, PlonkConsts K, uint32_t n, int party, typename Pol::Rnd P, uint64_t mbase,
                              const uint32_t* n12, const uint32_t* d12, uint32_t* on, uint32_t* od, uint32_t* pn, uint32_t* pd) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  typename Pol::S n3, d3;
  r3_factors<Pol>(in, K, n, i, party, 2, n3, d3);
  Pol::st_prod(on, pn, i, Pol::masked(Pol::lmul(Pol::ld(n12, i), n3), P, mbase + i));
  Pol::st_prod(od, pd, i, Pol::masked(Pol::lmul(Pol::ld(d12, i), d3), P, mbase + n + i));
}
// masked values to open: g_i = den_i s_i (i < n), q_k = r_k s'_k (k <= n); s, r, s' are fresh random shares
// (Rep3: drawn from the correlated streams at rbase; s: [0,n), r: [n, 2n+1), s': [2n+1, 3n+2)).  Additive (Rep3) or
// degree-2t (Shamir) outputs.
template <class Pol>
CS_GLOBAL void k_r3_round2_c(const uint32_t* den, uint32_t n, typename Pol::Rnd P, uint64_t rbase, uint64_t mbase,
                              uint32_t* out_g, uint32_t* out_q) {
  typedef typename Pol::FrP FrP;
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  typename Pol::S r = Pol::rand(P, rbase, n + i), sp = Pol::rand(P, rbase, 2 * n + 1 + i);
  st_fr<FrP>(out_q + (size_t)i * FrP::N, Pol::masked(Pol::lmul(r, sp), P, mbase + n + i));
  if (i < n) {
    typename Pol::S s = Pol::rand(P, rbase, i);
    st_fr<FrP>(out_g + (size_t)i * FrP::N, Pol::masked(Pol::lmul(Pol::ld(den, i), s), P, mbase + i));
  }
}
// with G^-1, Q^-1 public: 1/den_i = s_i / G_i,  x_i = num_i / den_i;  u_{i+1} = (s'_0 / Q_0) r_{i+1}
template <class Pol>
CS_GLOBAL void k_r3_round2_d(const uint32_t* num, const uint32_t* ginv, const uint32_t* qinv, uint32_t n, typename Pol::Rnd P,
                              uint64_t rbase, uint64_t mbase, uint32_t* ox, uint32_t* ou, uint32_t* px, uint32_t* pu) {
  typedef typename Pol::FrP FrP;
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  constexpr int NW = FrP::N;
  typename Pol::S deninv = Pol::mulp(Pol::rand(P, rbase, i), ld_fr<FrP>(ginv + (size_t)i * NW));
  Pol::st_prod(ox, px, i, Pol::masked(Pol::lmul(Pol::ld(num, i), deninv), P, mbase + i));
  typename Pol::S rinv0 = Pol::mulp(Pol::rand(P, rbase, 2 * n + 1), ld_fr<FrP>(qinv));
  Pol::st_prod(ou, pu, i, Pol::masked(Pol::lmul(rinv0, Pol::rand(P, rbase, n + i + 1)), P, mbase + n + i));
}
// m_i = r_i x_i
template <class Pol>
CS_GLOBAL void k_r3_round2_e(const uint32_t* x, uint32_t n, typename Pol::Rnd P, uint64_t rbase, uint64_t mbase, uint32_t* om,
                              uint32_t* pm) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Pol::st_prod(om, pm, i, Pol::masked(Pol::lmul(Pol::rand(P, rbase, n + i), Pol::ld(x, i)), P, mbase + i));
}
// y_i = m_i / r_{i+1} = m_i (s'_{i+1} / Q_{i+1}), to be opened
template <class Pol>
CS_GLOBAL void k_r3_round2_f(const uint32_t* m, const uint32_t* qinv, uint32_t n, typename Pol::Rnd P, uint64_t rbase,
                              uint64_t mbase, uint32_t* out_y) {
  typedef typename Pol::FrP FrP;
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  typename Pol::S rinv = Pol::mulp(Pol::rand(P, rbase, 2 * n + 1 + i + 1), ld_fr<FrP>(qinv + (size_t)(i + 1) * FrP::N));
  st_fr<FrP>(out_y + (size_t)i * FrP::N, Pol::masked(Pol::lmul(Pol::ld(m, i), rinv), P, mbase + i));
}
// prod_{j<=i} x_j = Y_0..Y_i * u_{i+1}  (Y public running products);  buffer_z is that rotated right by one
template <class Pol>
CS_GLOBAL void k_r3_round2_g(const uint32_t* ypref, const uint32_t* u, uint32_t n, uint32_t* zbuf) {
  typedef typename Pol::FrP FrP;
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Pol::st(zbuf, (i + 1) % n, Pol::mulp(Pol::ld(u, i), ld_fr<FrP>(ypref + (size_t)i * FrP::N)));
}

// elementwise inverse of a public vector from its prefix / suffix products and 1/total
template <class FrP>
CS_GLOBAL void k_batch_inverse(const uint32_t* pre, const uint32_t* suf, const uint32_t* inv_total, uint32_t n, uint32_t* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fp<FrP> v = ld_fr<FrP>(inv_total);
  if (i > 0) v = v * ld_fr<FrP>(pre + (size_t)(i - 1) * FrP::N);
  if (i + 1 < n) v = v * ld_fr<FrP>(suf + (size_t)(i + 1) * FrP::N);
  st_fr<FrP>(out + (size_t)i * FrP::N, v);
}

// ---- round 3 -------------------------------------------------------------------------------------------
struct R3QuotIn {
  const uint32_t *a, *b, *c, *z;   // 4n shares each (extended evaluations of the unblinded polynomials)
  const uint32_t* tw4;
};
struct R3Blinders { ShConst b[9]; };
template <class Pol>
struct R3Point {
  typename Pol::S a, b, c, z, zw, ap, bp, cp, zp, zwp;
  Fp<typename Pol::FrP> w;
};
template <class Pol>
CS_D R3Point<Pol> r3_point(const R3QuotIn& in, const R3Blinders& B, uint32_t n, uint32_t i) {
  typedef typename Pol::FrP FrP;
  typedef Fp<FrP> F;
  const uint32_t n4 = 4 * n;
  R3Point<Pol> p;
  p.w = root_pow<FrP>(in.tw4, 2 * n, i);
  F ww = root_pow<FrP>(in.tw4, 2 * n, (i + 4) % n4);
  p.a = Pol::ld(in.a, i); p.b = Pol::ld(in.b, i); p.c = Pol::ld(in.c, i); p.z = Pol::ld(in.z, i);
  p.zw = Pol::ld(in.z, (i + 4) % n4);
  p.ap = Pol::add(Pol::cnst(B.b[1]), Pol::mulp(Pol::cnst(B.b[0]), p.w));
  p.bp = Pol::add(Pol::cnst(B.b[3]), Pol::mulp(Pol::cnst(B.b[2]), p.w));
  p.cp = Pol::add(Pol::cnst(B.b[5]), Pol::mulp(Pol::cnst(B.b[4]), p.w));
  typename Pol::S b6 = Pol::cnst(B.b[6]), b7 = Pol::cnst(B.b[7]), b8 = Pol::cnst(B.b[8]);
  p.zp = Pol::add(Pol::add(Pol::mulp(b6, p.w.sqr()), Pol::mulp(b7, p.w)), b8);
  p.zwp = Pol::add(Pol::add(Pol::mulp(b6, ww.sqr()), Pol::mulp(b7, ww)), b8);
  return p;
}
// the twelve first-layer products: ab a.bp ap.b ap.bp | cz c.zp cp.z cp.zp | c.zw c.zwp cp.zw cp.zwp
// slot k of the arena holds product k (4n shares); masks at mbase + k 4n + i
template <class Pol>
CS_GLOBAL void k_r3_quot_l1(R3QuotIn in, R3Blinders B, uint32_t n, typename Pol::Rnd P, uint64_t mbase, uint32_t* arena,
                             uint32_t* peer, size_t slot_words) {
  typedef typename Pol::S S;
  const uint32_t n4 = 4 * n;
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  R3Point<Pol> p = r3_point<Pol>(in, B, n, i);
  const S* L[12] = {&p.a, &p.a, &p.ap, &p.ap, &p.c, &p.c, &p.cp, &p.cp, &p.c, &p.c, &p.cp, &p.cp};
  const S* R[12] = {&p.b, &p.bp, &p.b, &p.bp, &p.z, &p.zp, &p.z, &p.zp, &p.zw, &p.zwp, &p.zw, &p.zwp};
  for (int k = 0; k < 12; k++)
    Pol::st_prod(arena + (size_t)k * slot_words, peer ? peer + (size_t)k * slot_words : (uint32_t*)nullptr, i,
                 Pol::masked(Pol::lmul(*L[k], *R[k]), P, mbase + (uint64_t)k * n4 + i));
}

struct R3KeyEvals {
  const uint32_t *qm, *ql, *qr, *qo, *qc, *s1, *s2, *s3, *lagrange, *buf_a;  // buf_a: n shares
};
// e = (A)(B)(C)(D) with blinding parts, from the four (a,b)-type and four (c,d)-type products:
// value r and, for m != 0, the Z_H-weighted blinding sum (mul4vec / mul4vec_post, round3.rs:20-108)
template <class Pol>
CS_D void r3_mul4(const typename Pol::S& ab, const typename Pol::S& abp, const typename Pol::S& apb, const typename Pol::S& apbp,
                  const typename Pol::S& cd, const typename Pol::S& cdp, const typename Pol::S& cpd, const typename Pol::S& cpdp,
                  uint32_t m, const PlonkConsts& K, Fp<typename Pol::FrP>& r, Fp<typename Pol::FrP>& rz) {
  typedef typename Pol::FrP FrP;
  typename Pol::S s1 = Pol::add(apb, abp), s2 = Pol::add(cpd, cdp);
  r = Pol::lmul(ab, cd);
  rz = Pol::lmul(s1, cd) + Pol::lmul(ab, s2);
  if (m) {
    Fp<FrP> x1 = Pol::lmul(apbp, cd) + Pol::lmul(s1, s2) + Pol::lmul(ab, cpdp);
    Fp<FrP> x2 = Pol::lmul(s1, cpdp) + Pol::lmul(apbp, s2);
    Fp<FrP> x3 = Pol::lmul(apbp, cpdp);
    rz = rz + x1 * cload<FrP>(K.z1[m]) + x2 * cload<FrP>(K.z2[m]) + x3 * cload<FrP>(K.z3[m]);
  }
}
// layer 2: t and tz at every extended-domain point (compute_t, round3.rs:300-520) -- additive shares (Rep3) or
// degree-2t shares (Shamir).
// Operands are fetched where they are used (first-layer products from the arena, wire / z evaluations and their
// blinding parts recomputed from the nine blinders): holding the twelve products and the ten point values at once
// needed ~350 registers and spilled; the re-reads hit L1/L2.
template <class Pol>
CS_GLOBAL void k_r3_quot_l2(R3QuotIn in, R3Blinders B, R3KeyEvals E, uint32_t n, uint32_t nlag, PlonkConsts K, int party,
                             typename Pol::Rnd P, uint64_t mbase, const uint32_t* arena, size_t slot_words, uint32_t* t_out,
                             uint32_t* tz_out) {
  typedef typename Pol::FrP FrP;
  typedef Fp<FrP> F;
  typedef typename Pol::S S;
  constexpr int NW = FrP::N;
  const uint32_t n4 = 4 * n;
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const uint32_t m = i & 3;
  const F w = root_pow<FrP>(in.tw4, 2 * n, i);
  auto PR = [&](int k) { return Pol::ld(arena + (size_t)k * slot_words, i); };
  auto lin = [&](int hi, int lo) { return Pol::add(Pol::cnst(B.b[lo]), Pol::mulp(Pol::cnst(B.b[hi]), w)); };
  auto quad = [&](const F& x) {  // b6 x^2 + b7 x + b8
    return Pol::add(Pol::add(Pol::mulp(Pol::cnst(B.b[6]), x.sqr()), Pol::mulp(Pol::cnst(B.b[7]), x)), Pol::cnst(B.b[8]));
  };
  const F beta = cload<FrP>(K.beta), gamma = cload<FrP>(K.gamma);
  // e1, e1z: linear in the first-layer products -> this party's part of them (Rep3: the .a component)
  F e1, e1z;
  {
    const F qm = ld_fr<FrP>(E.qm + (size_t)i * NW), ql = ld_fr<FrP>(E.ql + (size_t)i * NW), qr = ld_fr<FrP>(E.qr + (size_t)i * NW),
            qo = ld_fr<FrP>(E.qo + (size_t)i * NW);
    e1 = Pol::part(PR(0)) * qm + Pol::part(Pol::ld(in.a, i)) * ql + Pol::part(Pol::ld(in.b, i)) * qr + Pol::part(Pol::ld(in.c, i)) * qo;
    F a0 = Pol::part(PR(1)) + Pol::part(PR(2));
    if (m) a0 = a0 + Pol::part(PR(3)) * cload<FrP>(K.z1[m]);
    e1z = a0 * qm + Pol::part(lin(0, 1)) * ql + Pol::part(lin(2, 3)) * qr + Pol::part(lin(4, 5)) * qo;
    for (uint32_t j = 0; j < nlag; j++)
      e1 = e1 - Pol::part(Pol::ld(E.buf_a, j)) * ld_fr<FrP>(E.lagrange + ((size_t)j * n4 + i) * NW);
    if (Pol::pub(party)) e1 = e1 + ld_fr<FrP>(E.qc + (size_t)i * NW);
  }
  // e2: (a + oa)(b + ob)(c + oc) z with oa = beta w + gamma, ...
  F e2, e2z, e3, e3z;
  {
    const F bw = beta * w;
    const F oa = bw + gamma, ob = bw * cload<FrP>(K.k1) + gamma, oc = bw * cload<FrP>(K.k2) + gamma;
    S ab = Pol::addp(Pol::add(PR(0), Pol::add(Pol::mulp(Pol::ld(in.a, i), ob), Pol::mulp(Pol::ld(in.b, i), oa))), oa * ob, party);
    S abp = Pol::add(PR(1), Pol::mulp(lin(2, 3), oa));
    S apb = Pol::add(PR(2), Pol::mulp(lin(0, 1), ob));
    S cd = Pol::add(PR(4), Pol::mulp(Pol::ld(in.z, i), oc));
    S cdp = Pol::add(PR(5), Pol::mulp(quad(w), oc));
    r3_mul4<Pol>(ab, abp, apb, PR(3), cd, cdp, PR(6), PR(7), m, K, e2, e2z);
  }
  {
    const F o1 = ld_fr<FrP>(E.s1 + (size_t)i * NW) * beta + gamma, o2 = ld_fr<FrP>(E.s2 + (size_t)i * NW) * beta + gamma,
            o3 = ld_fr<FrP>(E.s3 + (size_t)i * NW) * beta + gamma;
    S ab = Pol::addp(Pol::add(PR(0), Pol::add(Pol::mulp(Pol::ld(in.a, i), o2), Pol::mulp(Pol::ld(in.b, i), o1))), o1 * o2, party);
    S abp = Pol::add(PR(1), Pol::mulp(lin(2, 3), o1));
    S apb = Pol::add(PR(2), Pol::mulp(lin(0, 1), o2));
    S cd = Pol::add(PR(8), Pol::mulp(Pol::ld(in.z, (i + 4) % n4), o3));
    S cdp = Pol::add(PR(9), Pol::mulp(quad(root_pow<FrP>(in.tw4, 2 * n, (i + 4) % n4)), o3));
    r3_mul4<Pol>(ab, abp, apb, PR(3), cd, cdp, PR(10), PR(11), m, K, e3, e3z);
  }
  const F alpha = cload<FrP>(K.alpha);
  const F l0a2 = ld_fr<FrP>(E.lagrange + (size_t)i * NW) * cload<FrP>(K.alpha2);
  F zm1 = Pol::part(Pol::ld(in.z, i));
  if (Pol::pub(party)) zm1 = zm1 - F::one();
  const F e4 = zm1 * l0a2, e4z = Pol::part(quad(w)) * l0a2;
  st_fr<FrP>(t_out + (size_t)i * NW, Pol::masked(e1 + (e2 - e3) * alpha + e4, P, mbase + i));
  st_fr<FrP>(tz_out + (size_t)i * NW, Pol::masked(e1z + (e2z - e3z) * alpha + e4z, P, mbase + n4 + i));
}

}  // namespace cs
