// Prime-field arithmetic in Montgomery form on 32-bit limbs (device side).
//
// Replaces the arkworks `Fp<MontBackend<_, N>>` arithmetic that every reference function on the
// hot path bottoms out in (field elements are `[u64; N]` little-endian Montgomery limbs with
// R = 2^(64 N); a `[u64; N]` is bit-identical to our `uint32_t[2 N]`, so buffers cross the C ABI
// without conversion).  SURVEY.md 8(a): "F_r element = 32 B ... Montgomery form, R = 2^256".
//
// mul(): word-serial Montgomery product with the even/odd accumulator split, so every
// 32x32->64 partial product is one IMAD.WIDE in a single carry chain (no carry-save fix-ups).
// All results are fully reduced to [0, p), which the exact equality tests in the point formulas need.
//
// Attribution: the even/odd-accumulator word-serial product below (mul_n, cmad_n, madc_n_rshift,
// mad_n_redc and the way mul_inline drives them) follows the structure and helper naming of
// Supranational's sppark, ff/mont_t.cuh (Copyright Supranational LLC, Apache License 2.0,
// https://github.com/supranational/sppark); see NOTICE at the repository root.  The product-scanning
// squaring, the conversions and everything else in this file are this repository's own.
#pragma once
#include "cs_prims.cuh"

namespace cs {

// ---- generic N-limb helpers ---------------------------------------------------------------------
template <int N>
CS_D void mul_n(uint32_t* acc, const uint32_t* a, uint32_t bi) {
  CS_UNROLL
  for (int j = 0; j < N; j += 2) {
    acc[j] = mul_lo(a[j], bi);
    acc[j + 1] = mul_hi(a[j], bi);
  }
}

// acc[0..N) += (a[0], a[2], ...) * bi   (pairs (lo,hi) land on (j, j+1)); carry-out stays in CC.
template <int N>
CS_D void cmad_n(uint32_t* acc, const uint32_t* a, uint32_t bi) {
  acc[0] = mad_lo_cc(a[0], bi, acc[0]);
  acc[1] = madc_hi_cc(a[0], bi, acc[1]);
  CS_UNROLL
  for (int j = 2; j < N; j += 2) {
    acc[j] = madc_lo_cc(a[j], bi, acc[j]);
    acc[j + 1] = madc_hi_cc(a[j], bi, acc[j + 1]);
  }
}

// odd = (odd >> 64) + (a[0], a[2], ...) * bi + CC      (no carry-out possible, see DESIGN.md)
template <int N>
CS_D void madc_n_rshift(uint32_t* odd, const uint32_t* a, uint32_t bi) {
  CS_UNROLL
  for (int j = 0; j < N - 2; j += 2) {
    odd[j] = madc_lo_cc(a[j], bi, odd[j + 2]);
    odd[j + 1] = madc_hi_cc(a[j], bi, odd[j + 3]);
  }
  odd[N - 2] = madc_lo_cc(a[N - 2], bi, 0);
  odd[N - 1] = madc_hi(a[N - 2], bi, 0);
}

// One row of the interleaved Montgomery product.  X is the accumulator aligned with bit 0 of the
// running value T, Y the one aligned 32 bits up (T = X + Y * 2^32); the roles swap every row.
template <class P, bool FIRST>
CS_D void mad_n_redc(uint32_t* X, uint32_t* Y, const uint32_t* a, uint32_t bi) {
  constexpr int N = P::N;
  if (FIRST) {
    mul_n<N>(Y, a + 1, bi);
    mul_n<N>(X, a, bi);
  } else {
    X[0] = add_cc(X[0], Y[1]);
    madc_n_rshift<N>(Y, a + 1, bi);
    cmad_n<N>(X, a, bi);
    Y[N - 1] = addc(Y[N - 1], 0);
  }
  uint32_t mi = mul_lo(X[0], P::M0);
  uint32_t mod[N];
  CS_UNROLL
  for (int i = 0; i < N; i++) mod[i] = P::mod(i);
  cmad_n<N>(Y, mod + 1, mi);
  cmad_n<N>(X, mod, mi);
  Y[N - 1] = addc(Y[N - 1], 0);
}

// The product half of a mad_n_redc row (the unreduced product Fp::mul_wide): X gets the low word of the shifted value
template <int N>
CS_D void mad_n(uint32_t* X, uint32_t* Y, const uint32_t* a, uint32_t bi) {
  X[0] = add_cc(X[0], Y[1]);
  madc_n_rshift<N>(Y, a + 1, bi);
  cmad_n<N>(X, a, bi);
  Y[N - 1] = addc(Y[N - 1], 0);
}
// A row of the reduction alone (Fp::redc): the one-word shift of mad_n_redc moves into the chain that adds m p
template <class P>
CS_D void redc_row(uint32_t* X, uint32_t* Y, const uint32_t* mod) {
  constexpr int N = P::N;
  const uint32_t m = mul_lo(X[0] + Y[1], P::M0);
  X[0] = add_cc(X[0], Y[1]);
  madc_n_rshift<N>(Y, mod + 1, m);
  cmad_n<N>(X, mod, m);
  Y[N - 1] = addc(Y[N - 1], 0);
}

// r[0..M) += a[0..M)  /  r[0..M) -= a[0..M), modulo 2^(32 M)
template <int M>
CS_D void add_n(uint32_t* r, const uint32_t* a) {
  r[0] = add_cc(r[0], a[0]);
  CS_UNROLL
  for (int i = 1; i < M - 1; i++) r[i] = addc_cc(r[i], a[i]);
  r[M - 1] = addc(r[M - 1], a[M - 1]);
}
template <int M>
CS_D void sub_n(uint32_t* r, const uint32_t* a) {
  r[0] = sub_cc(r[0], a[0]);
  CS_UNROLL
  for (int i = 1; i < M - 1; i++) r[i] = subc_cc(r[i], a[i]);
  r[M - 1] = subc(r[M - 1], a[M - 1]);
}

// K p^2 as 2N little-endian words, evaluated by the compiler: the offsets that keep the lazy Fp2 sums non-negative
template <class P, int K>
struct ModSq {
  uint32_t v[2 * P::N];
  CS_HD constexpr ModSq() : v{} {
    for (int i = 0; i < P::N; i++) {
      uint64_t carry = 0;
      for (int j = 0; j < P::N; j++) {
        const uint64_t s = (uint64_t)P::mod(i) * P::mod(j) + v[i + j] + carry;
        v[i + j] = (uint32_t)s;
        carry = s >> 32;
      }
      v[i + P::N] = (uint32_t)carry;
    }
    uint64_t carry = 0;
    for (int k = 0; k < 2 * P::N; k++) {
      const uint64_t s = (uint64_t)v[k] * K + carry;
      v[k] = (uint32_t)s;
      carry = s >> 32;
    }
  }
};
template <class P, int K>
CS_HD constexpr uint32_t mod_sq(int k) {
  constexpr ModSq<P, K> t;
  return t.v[k];
}
// r[0..2N) += K p^2
template <class P, int K>
CS_D void add_mod_sq(uint32_t* r) {
  constexpr int M = 2 * P::N;
  r[0] = add_cc(r[0], mod_sq<P, K>(0));
  CS_UNROLL
  for (int i = 1; i < M - 1; i++) r[i] = addc_cc(r[i], mod_sq<P, K>(i));
  r[M - 1] = addc(r[M - 1], mod_sq<P, K>(M - 1));
}

template <class P>
struct Fp {
  static constexpr int N = P::N;
  uint32_t l[N];

  // ---- constants
  static CS_D Fp zero() { Fp r; CS_UNROLL for (int i = 0; i < N; i++) r.l[i] = 0; return r; }
  static CS_D Fp one() { Fp r; CS_UNROLL for (int i = 0; i < N; i++) r.l[i] = P::one(i); return r; }
  static CS_D Fp r2() { Fp r; CS_UNROLL for (int i = 0; i < N; i++) r.l[i] = P::r2(i); return r; }

  CS_D bool is_zero() const {
    uint32_t o = 0;
    CS_UNROLL
    for (int i = 0; i < N; i++) o |= l[i];
    return o == 0;
  }
  CS_D bool operator==(const Fp& b) const {
    uint32_t o = 0;
    CS_UNROLL
    for (int i = 0; i < N; i++) o |= l[i] ^ b.l[i];
    return o == 0;
  }
  CS_D bool operator!=(const Fp& b) const { return !(*this == b); }

  // r = (r >= p) ? r - p : r
  CS_D void final_sub() {
    uint32_t t[N];
    t[0] = sub_cc(l[0], P::mod(0));
    CS_UNROLL
    for (int i = 1; i < N; i++) t[i] = subc_cc(l[i], P::mod(i));
    uint32_t borrow = subc(0, 0);  // 0xffffffff if l < p
    CS_UNROLL
    for (int i = 0; i < N; i++) l[i] = borrow ? l[i] : t[i];
  }

  friend CS_D Fp operator+(const Fp& a, const Fp& b) {
    Fp r;
    r.l[0] = add_cc(a.l[0], b.l[0]);
    CS_UNROLL
    for (int i = 1; i < N; i++) r.l[i] = addc_cc(a.l[i], b.l[i]);
    // p has at least one spare top bit (254/255/381-bit moduli), so no carry-out here
    r.final_sub();
    return r;
  }
  friend CS_D Fp operator-(const Fp& a, const Fp& b) {
    Fp r;
    r.l[0] = sub_cc(a.l[0], b.l[0]);
    CS_UNROLL
    for (int i = 1; i < N; i++) r.l[i] = subc_cc(a.l[i], b.l[i]);
    uint32_t borrow = subc(0, 0);
    r.l[0] = add_cc(r.l[0], borrow & P::mod(0));
    CS_UNROLL
    for (int i = 1; i < N; i++) r.l[i] = addc_cc(r.l[i], borrow & P::mod(i));
    return r;
  }
  CS_D Fp neg() const { return is_zero() ? *this : (zero() - *this); }
  CS_D Fp dbl() const { return *this + *this; }

  // Out-of-line on purpose: one ~230-instruction copy per kernel keeps the point formulas (10-42
  // multiplications each) inside the instruction cache; operands travel by value in registers.
  friend CS_D Fp operator*(const Fp& a, const Fp& b) { return mul_ool(a, b); }
  static CS_DN Fp mul_ool(Fp a, Fp b) { return mul_inline(a, b); }
  static CS_D Fp mul_inline(const Fp& a, const Fp& b) {
    uint32_t even[N], odd[N];
    mad_n_redc<P, true>(even, odd, a.l, b.l[0]);
    mad_n_redc<P, false>(odd, even, a.l, b.l[1]);
    CS_UNROLL
    for (int i = 2; i < N; i += 2) {
      mad_n_redc<P, false>(even, odd, a.l, b.l[i]);
      mad_n_redc<P, false>(odd, even, a.l, b.l[i + 1]);
    }
    // result = even + (odd >> 32)
    Fp r;
    r.l[0] = add_cc(even[0], odd[1]);
    CS_UNROLL
    for (int i = 1; i < N - 1; i++) r.l[i] = addc_cc(even[i], odd[i + 1]);
    r.l[N - 1] = addc(even[N - 1], 0);
    r.final_sub();
    return r;
  }
  // Squaring: product-scanning (Comba) form so that the 28 symmetric cross products a_i a_j (i < j) are
  // computed once and doubled: 36 + 64 (reduction) IMAD.WIDE instead of 128.  Each column keeps a 3-word
  // accumulator; the cross-product sum is doubled in a second 3-word register set before it is merged.
  CS_D Fp sqr() const { return sqr_ool(*this); }
  static CS_DN Fp sqr_ool(Fp a) {
    uint32_t c0 = 0, c1 = 0, c2 = 0;
    uint32_t m[N];
    Fp r;
    CS_UNROLL
    for (int k = 0; k < 2 * N - 1; k++) {
      // cross terms 2 * sum_{i < j, i + j = k} a_i a_j
      uint32_t t0 = 0, t1 = 0, t2 = 0;
      CS_UNROLL
      for (int i = 0; i < N; i++) {
        int j = k - i;
        if (j > i && j < N) {
          t0 = mad_lo_cc(a.l[i], a.l[j], t0);
          t1 = madc_hi_cc(a.l[i], a.l[j], t1);
          t2 = addc(t2, 0);
        }
      }
      t2 = (t2 << 1) | (t1 >> 31);
      t1 = (t1 << 1) | (t0 >> 31);
      t0 = t0 << 1;
      c0 = add_cc(c0, t0);
      c1 = addc_cc(c1, t1);
      c2 = addc(c2, t2);
      if ((k & 1) == 0) {  // square term a_{k/2}^2
        c0 = mad_lo_cc(a.l[k / 2], a.l[k / 2], c0);
        c1 = madc_hi_cc(a.l[k / 2], a.l[k / 2], c1);
        c2 = addc(c2, 0);
      }
      // reduction terms sum_i m_i p_{k-i}
      CS_UNROLL
      for (int i = 0; i < N; i++) {
        int j = k - i;
        if (i < k && i < N && j >= 0 && j < N && (k < N ? i < k : true)) {
          if (k < N || i >= k - N + 1) {
            c0 = mad_lo_cc(m[i], P::mod(j), c0);
            c1 = madc_hi_cc(m[i], P::mod(j), c1);
            c2 = addc(c2, 0);
          }
        }
      }
      if (k < N) {
        m[k] = mul_lo(c0, P::M0);
        c0 = mad_lo_cc(m[k], P::mod(0), c0);
        c1 = madc_hi_cc(m[k], P::mod(0), c1);
        c2 = addc(c2, 0);
      } else {
        r.l[k - N] = c0;
      }
      c0 = c1; c1 = c2; c2 = 0;
    }
    r.l[N - 1] = c0;
    r.final_sub();
    return r;
  }

  // a b + c d with ONE Montgomery reduction (product scanning: both partial-product sets and the reduction terms of
  // a column meet in one 3-word accumulator): 2 N^2 + N^2 wide multiply-adds instead of the 4 N^2 of two products.
  // Needs 2 p < 2^(32 N), true for every modulus here (254 / 255 / 381 bits in 256 / 256 / 384).
  static CS_D Fp dot2(const Fp& a, const Fp& b, const Fp& c, const Fp& d) { return dot2_ool(a, b, c, d); }
  static CS_DN Fp dot2_ool(Fp a, Fp b, Fp c, Fp d) {
    uint32_t c0 = 0, c1 = 0, c2 = 0;
    uint32_t m[N];
    Fp r;
    CS_UNROLL
    for (int k = 0; k < 2 * N - 1; k++) {
      CS_UNROLL
      for (int i = 0; i < N; i++) {
        const int j = k - i;
        if (j >= 0 && j < N) {
          c0 = mad_lo_cc(a.l[i], b.l[j], c0);
          c1 = madc_hi_cc(a.l[i], b.l[j], c1);
          c2 = addc(c2, 0);
          c0 = mad_lo_cc(c.l[i], d.l[j], c0);
          c1 = madc_hi_cc(c.l[i], d.l[j], c1);
          c2 = addc(c2, 0);
        }
      }
      // reduction terms m_i p_j, i + j = k, of the rows already determined (j >= 1)
      CS_UNROLL
      for (int i = 0; i < N; i++) {
        const int j = k - i;
        if (j >= 1 && j < N) {
          c0 = mad_lo_cc(m[i], P::mod(j), c0);
          c1 = madc_hi_cc(m[i], P::mod(j), c1);
          c2 = addc(c2, 0);
        }
      }
      if (k < N) {
        m[k] = mul_lo(c0, P::M0);
        c0 = mad_lo_cc(m[k], P::mod(0), c0);
        c1 = madc_hi_cc(m[k], P::mod(0), c1);
        c2 = addc(c2, 0);
      } else {
        r.l[k - N] = c0;
      }
      c0 = c1; c1 = c2; c2 = 0;
    }
    r.l[N - 1] = c0;
    r.final_sub();
    return r;
  }

  // ---- lazy reduction (the Fp2 products of cs_curve.cuh): an unreduced product and a separate reduction
  // a + b without the final subtraction: < 2p, which still fits N words (2p < 2^(32N) for every modulus here)
  static CS_D Fp add_unreduced(const Fp& a, const Fp& b) {
    Fp r;
    r.l[0] = add_cc(a.l[0], b.l[0]);
    CS_UNROLL
    for (int i = 1; i < N - 1; i++) r.l[i] = addc_cc(a.l[i], b.l[i]);
    r.l[N - 1] = addc(a.l[N - 1], b.l[N - 1]);
    return r;
  }
  // t[0..2N) = a b, unreduced, for a < 2^(32N - 1) (an unreduced sum < 2p qualifies) and any N-word b.  The rows of
  // mul_inline without their reduction halves: N^2 wide multiply-adds in one carry chain per half-row, and the word
  // that leaves the bottom of each row is the next word of t.
  static CS_D void mul_wide(uint32_t* t, const Fp& a, const Fp& b) {
    uint32_t even[N], odd[N];
    mul_n<N>(odd, a.l + 1, b.l[0]);
    mul_n<N>(even, a.l, b.l[0]);
    t[0] = even[0];
    CS_UNROLL
    for (int i = 1; i < N; i += 2) {
      mad_n<N>(odd, even, a.l, b.l[i]);
      t[i] = odd[0];
      if (i + 1 < N) {
        mad_n<N>(even, odd, a.l, b.l[i + 1]);
        t[i + 1] = even[0];
      }
    }
    // t[N..2N) = even + (odd >> 32)
    t[N] = add_cc(even[0], odd[1]);
    CS_UNROLL
    for (int k = 1; k < N - 1; k++) t[N + k] = addc_cc(even[k], odd[k + 1]);
    t[2 * N - 1] = addc(even[N - 1], 0);
  }
  // t R^-1 mod p (R = 2^(32N)) of a 2N-word t < p R, fully reduced.  The reduction rows of mul_inline run over the
  // low half (N^2 wide multiply-adds; the shift of each row rides in its reduction chain), which leaves
  // (t_lo + m p) / R <= p; adding t_hi < p stays below 2p, so one final subtraction suffices.
  static CS_D Fp redc(const uint32_t* t) {
    uint32_t even[N], odd[N], mod[N];
    CS_UNROLL
    for (int i = 0; i < N; i++) { even[i] = t[i]; mod[i] = P::mod(i); }
    const uint32_t m = mul_lo(even[0], P::M0);
    mul_n<N>(odd, mod + 1, m);
    cmad_n<N>(even, mod, m);
    odd[N - 1] = addc(odd[N - 1], 0);
    CS_UNROLL
    for (int i = 1; i < N; i += 2) {
      redc_row<P>(odd, even, mod);
      if (i + 1 < N) redc_row<P>(even, odd, mod);
    }
    Fp r;
    r.l[0] = add_cc(even[0], odd[1]);
    CS_UNROLL
    for (int k = 1; k < N - 1; k++) r.l[k] = addc_cc(even[k], odd[k + 1]);
    r.l[N - 1] = addc(even[N - 1], 0);
    r.l[0] = add_cc(r.l[0], t[N]);
    CS_UNROLL
    for (int k = 1; k < N - 1; k++) r.l[k] = addc_cc(r.l[k], t[N + k]);
    r.l[N - 1] = addc(r.l[N - 1], t[2 * N - 1]);
    r.final_sub();
    return r;
  }

  // Montgomery <-> canonical
  CS_D Fp to_mont() const { return (*this) * r2(); }
  CS_D Fp from_mont() const {
    Fp o = zero();
    o.l[0] = 1;
    return (*this) * o;
  }

  // a^(p-2); only used off the per-proof path (table precomputation)
  CS_D Fp inverse() const {
    Fp res = one();
    Fp base = *this;
    for (int i = 0; i < N; i++) {
      uint32_t e = P::mod(i);
      if (i == 0) e -= 2;  // all supported moduli have mod[0] >= 2 (they are odd and > 2)
      for (int b = 0; b < 32; b++) {
        if ((e >> b) & 1) res = res * base;
        base = base.sqr();
      }
    }
    return res;
  }
};

}  // namespace cs
