// Quadratic extension and short-Weierstrass (a = 0) point arithmetic, device side.
//
// Replaces what `ark_ec::short_weierstrass::{Affine, Projective}` provide to
// `taceo_ark_algebra::msm::msm_unchecked` (reference call sites: co-groth16/src/mpc/rep3.rs:124-132,
// co-groth16/src/groth16.rs:190-200).  Accumulators use extended Jacobian "XYZZ" coordinates
// (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2): a mixed addition costs 8M + 2S and needs no inversion, and
// every special case (infinity, P + P, P + (-P)) is handled exactly because parity with the
// reference is bit-exact on the affine result.
#pragma once
#include "cs_field.cuh"

namespace cs {

// Fq2 = Fq[u]/(u^2 + 1)   (BN254 and BLS12-381)
template <class P>
struct Fp2 {
  typedef Fp<P> F;
  static constexpr int N = 2 * P::N;
  F c0, c1;
  static CS_D Fp2 zero() { Fp2 r; r.c0 = F::zero(); r.c1 = F::zero(); return r; }
  static CS_D Fp2 one() { Fp2 r; r.c0 = F::one(); r.c1 = F::zero(); return r; }
  CS_D bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
  CS_D bool operator==(const Fp2& b) const { return c0 == b.c0 && c1 == b.c1; }
  CS_D bool operator!=(const Fp2& b) const { return !(*this == b); }
  friend CS_D Fp2 operator+(const Fp2& a, const Fp2& b) { Fp2 r; r.c0 = a.c0 + b.c0; r.c1 = a.c1 + b.c1; return r; }
  friend CS_D Fp2 operator-(const Fp2& a, const Fp2& b) { Fp2 r; r.c0 = a.c0 - b.c0; r.c1 = a.c1 - b.c1; return r; }
  // mul / sqr / mul_sub are out-of-line (one copy per kernel) to keep the G2 point formulas in the I-cache.
  friend CS_D Fp2 operator*(const Fp2& a, const Fp2& b) { return mul_ool(a, b); }
  // Karatsuba on unreduced 2N-word products with one Montgomery reduction per coefficient: 5 N^2 wide multiply-adds
  // instead of the 6 N^2 of three reduced products.
  //   v0 = a0 b0, v1 = a1 b1 < p^2;  v2 = (a0 + a1)(b0 + b1) < 4 p^2 (sums < 2p, left unreduced)
  //   c1 = v2 - v0 - v1 = a0 b1 + a1 b0 < 2 p^2;  c0 = v0 + p^2 - v1 in (0, 2 p^2)
  // F::redc needs its input below p 2^(32N): 2 p^2 is, since 2 p < 2^(32N).
  static CS_DN Fp2 mul_ool(Fp2 a, Fp2 b) {
    constexpr int W = 2 * P::N;
    uint32_t v0[W], v1[W], v2[W];
    F::mul_wide(v0, a.c0, b.c0);
    F::mul_wide(v1, a.c1, b.c1);
    F::mul_wide(v2, F::add_unreduced(a.c0, a.c1), F::add_unreduced(b.c0, b.c1));
    sub_n<W>(v2, v0);
    sub_n<W>(v2, v1);
    add_mod_sq<P, 1>(v0);
    sub_n<W>(v0, v1);
    Fp2 r;
    r.c0 = F::redc(v0);
    r.c1 = F::redc(v2);
    return r;
  }
  // a b - c d with two Montgomery reductions (8 N^2 wide multiply-adds instead of the 12 N^2 of two reduced Fp2
  // products and a subtraction).  With u = the Karatsuba products of a b and w those of c d (as in mul_ool):
  //   t0 = 2 p^2 + (u0 - u1) - (w0 - w1)                       in (0, 4 p^2): both differences lie in (-p^2, p^2)
  //   t1 = 2 p^2 + (u2 - u0 - u1) - (w2 - w0 - w1)            in (0, 4 p^2): both cross sums lie in [0, 2 p^2)
  // The partial sums may wrap modulo 2^(64N); the totals do not.  F::redc needs t < p 2^(32N), i.e. 4 p < 2^(32N):
  // 2^256 / q = 5.3 for BN254 and 2^384 / p = 9.8 for BLS12-381.
  static CS_DN Fp2 mul_sub_ool(Fp2 a, Fp2 b, Fp2 c, Fp2 d) {
    constexpr int W = 2 * P::N;
    uint32_t t0[W], t1[W], t[W];
    CS_UNROLL
    for (int i = 0; i < W; i++) t0[i] = t1[i] = mod_sq<P, 2>(i);
    F::mul_wide(t, a.c0, b.c0);  // u0
    add_n<W>(t0, t);
    sub_n<W>(t1, t);
    F::mul_wide(t, a.c1, b.c1);  // u1
    sub_n<W>(t0, t);
    sub_n<W>(t1, t);
    F::mul_wide(t, F::add_unreduced(a.c0, a.c1), F::add_unreduced(b.c0, b.c1));  // u2
    add_n<W>(t1, t);
    F::mul_wide(t, c.c0, d.c0);  // w0
    sub_n<W>(t0, t);
    add_n<W>(t1, t);
    F::mul_wide(t, c.c1, d.c1);  // w1
    add_n<W>(t0, t);
    add_n<W>(t1, t);
    F::mul_wide(t, F::add_unreduced(c.c0, c.c1), F::add_unreduced(d.c0, d.c1));  // w2
    sub_n<W>(t1, t);
    Fp2 r;
    r.c0 = F::redc(t0);
    r.c1 = F::redc(t1);
    return r;
  }
  CS_D Fp2 sqr() const { return sqr_ool(*this); }
  static CS_DN Fp2 sqr_ool(Fp2 a) {
    // (c0 + c1 u)^2 = (c0 + c1)(c0 - c1) + 2 c0 c1 u
    Fp2 r;
    F t = F::mul_inline(a.c0, a.c1);
    r.c0 = F::mul_inline(a.c0 + a.c1, a.c0 - a.c1);
    r.c1 = t + t;
    return r;
  }
  CS_D Fp2 neg() const { Fp2 r; r.c0 = c0.neg(); r.c1 = c1.neg(); return r; }
  CS_D Fp2 dbl() const { Fp2 r; r.c0 = c0.dbl(); r.c1 = c1.dbl(); return r; }
  CS_D Fp2 inverse() const {
    F n = (c0.sqr() + c1.sqr()).inverse();
    Fp2 r;
    r.c0 = c0 * n;
    r.c1 = (c1 * n).neg();
    return r;
  }
};

// a b - c d: one fused reduction in the base field (Fp::dot2), one per coefficient in the extension
template <class P>
CS_D Fp<P> mul_sub(const Fp<P>& a, const Fp<P>& b, const Fp<P>& c, const Fp<P>& d) { return Fp<P>::dot2(a, b, c.neg(), d); }
template <class P>
CS_D Fp2<P> mul_sub(const Fp2<P>& a, const Fp2<P>& b, const Fp2<P>& c, const Fp2<P>& d) {
  return Fp2<P>::mul_sub_ool(a, b, c, d);
}

// Affine point; (0, 0) encodes infinity (never on y^2 = x^3 + b with b != 0) -- the same marker
// snarkjs .zkey files use.
template <class F>
struct Affine {
  F x, y;
  CS_D bool is_inf() const { return x.is_zero() && y.is_zero(); }
  static CS_D Affine inf() { Affine r; r.x = F::zero(); r.y = F::zero(); return r; }
};

template <class F>
struct Xyzz {
  F x, y, zz, zzz;
  CS_D bool is_inf() const { return zz.is_zero(); }
  static CS_D Xyzz inf() {
    Xyzz r;
    r.x = F::zero(); r.y = F::zero(); r.zz = F::zero(); r.zzz = F::zero();
    return r;
  }
  static CS_D Xyzz from_affine(const Affine<F>& p) {
    if (p.is_inf()) return inf();
    Xyzz r;
    r.x = p.x; r.y = p.y; r.zz = F::one(); r.zzz = F::one();
    return r;
  }
};

// 2 * (affine p), p != inf  (mdbl-2008-s-1, a = 0)
template <class F>
CS_DN Xyzz<F> dbl_affine(const Affine<F>& p) {
  Xyzz<F> r;
  if (p.y.is_zero()) return Xyzz<F>::inf();
  F U = p.y.dbl();
  F V = U.sqr();
  F W = U * V;
  F S = p.x * V;
  F X2 = p.x.sqr();
  F M = X2.dbl() + X2;
  r.x = M.sqr() - S.dbl();
  r.y = mul_sub(M, S - r.x, W, p.y);
  r.zz = V;
  r.zzz = W;
  return r;
}

// 2 * (xyzz p)  (dbl-2008-s-1, a = 0)
template <class F>
CS_DN Xyzz<F> dbl_xyzz(const Xyzz<F>& p) {
  if (p.is_inf() || p.y.is_zero()) return Xyzz<F>::inf();
  Xyzz<F> r;
  F U = p.y.dbl();
  F V = U.sqr();
  F W = U * V;
  F S = p.x * V;
  F X2 = p.x.sqr();
  F M = X2.dbl() + X2;
  r.x = M.sqr() - S.dbl();
  r.y = mul_sub(M, S - r.x, W, p.y);
  r.zz = V * p.zz;
  r.zzz = W * p.zzz;
  return r;
}

// acc += p  (madd-2008-s), p affine, optionally negated
template <class F>
CS_D void madd(Xyzz<F>& acc, const Affine<F>& p_in, bool negate) {
  if (p_in.is_inf()) return;
  Affine<F> p = p_in;
  if (negate) p.y = p.y.neg();
  if (acc.is_inf()) {
    acc.x = p.x; acc.y = p.y; acc.zz = F::one(); acc.zzz = F::one();
    return;
  }
  F U2 = p.x * acc.zz;
  F S2 = p.y * acc.zzz;
  F Pp = U2 - acc.x;
  F R = S2 - acc.y;
  if (Pp.is_zero()) {
    if (R.is_zero()) acc = dbl_affine(p);
    else acc = Xyzz<F>::inf();
    return;
  }
  F PP = Pp.sqr();
  F PPP = Pp * PP;
  F Q = acc.x * PP;
  F X3 = R.sqr() - PPP - Q.dbl();
  acc.y = mul_sub(R, Q - X3, acc.y, PPP);
  acc.x = X3;
  acc.zz = acc.zz * PP;
  acc.zzz = acc.zzz * PPP;
}

// acc += q  (add-2008-s), both XYZZ
template <class F>
CS_D void padd(Xyzz<F>& acc, const Xyzz<F>& q) {
  if (q.is_inf()) return;
  if (acc.is_inf()) { acc = q; return; }
  F U1 = acc.x * q.zz;
  F U2 = q.x * acc.zz;
  F S1 = acc.y * q.zzz;
  F S2 = q.y * acc.zzz;
  F Pp = U2 - U1;
  F R = S2 - S1;
  if (Pp.is_zero()) {
    if (R.is_zero()) acc = dbl_xyzz(acc);
    else acc = Xyzz<F>::inf();
    return;
  }
  F PP = Pp.sqr();
  F PPP = Pp * PP;
  F Q = U1 * PP;
  F X3 = R.sqr() - PPP - Q.dbl();
  acc.y = mul_sub(R, Q - X3, S1, PPP);
  acc.x = X3;
  acc.zz = acc.zz * q.zz * PP;
  acc.zzz = acc.zzz * q.zzz * PPP;
}

// A point held by the lane `delta` above this one (warp shuffle, whole warp takes part); lanes whose source falls
// outside the warp get their own value back, as __shfl_down_sync does.
template <class P>
CS_D Fp<P> shfl_down(const Fp<P>& a, unsigned delta) {
  Fp<P> r;
#if defined(CS_EMU)  // test emulation: one block-wide exchange per element instead of one per 32-bit word
  cs::emu::shfl_bytes(&a, &r, sizeof(r), 1, delta);
  return r;
#endif
  CS_UNROLL
  for (int i = 0; i < P::N; i++) r.l[i] = __shfl_down_sync(0xffffffffu, a.l[i], delta);
  return r;
}
template <class P>
CS_D Fp2<P> shfl_down(const Fp2<P>& a, unsigned delta) {
  Fp2<P> r;
  r.c0 = shfl_down(a.c0, delta);
  r.c1 = shfl_down(a.c1, delta);
  return r;
}
template <class F>
CS_D Xyzz<F> shfl_down(const Xyzz<F>& p, unsigned delta) {
  Xyzz<F> r;
#if defined(CS_EMU)  // test emulation: one block-wide exchange for the whole point instead of one per 32-bit word
  cs::emu::shfl_bytes(&p, &r, sizeof(r), 1, delta);
  return r;
#endif
  r.x = shfl_down(p.x, delta); r.y = shfl_down(p.y, delta);
  r.zz = shfl_down(p.zz, delta); r.zzz = shfl_down(p.zzz, delta);
  return r;
}

// XYZZ -> affine (one inversion); off the per-proof path
template <class F>
CS_DN Affine<F> to_affine(const Xyzz<F>& p) {
  if (p.is_inf()) return Affine<F>::inf();
  F zi = p.zzz.inverse();       // 1/ZZZ
  F zzi = (zi * p.zz).sqr();    // (ZZ/ZZZ)^2 = 1/ZZ   (ZZ^3 = ZZZ^2)
  Affine<F> r;
  r.x = p.x * zzi;
  r.y = p.y * zi;
  return r;
}

}  // namespace cs
