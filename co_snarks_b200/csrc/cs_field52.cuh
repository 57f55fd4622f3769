// Prime-field multiplication on the FP64 pipe: 5 limbs of 52 bits, Montgomery radix R = 2^260.
//
// Why: IMAD.WIDE.U32 -- the instruction the 8 x 32-bit CIOS product is made of -- issues at HALF the IMAD rate
// (4 cycles per warp instruction per SM sub-partition), while DFMA issues at the full rate (2 cycles);
// tools/pipe_probe.cu measures both.  A 52 x 52 -> 104-bit limb product costs two DFMA + one DADD (6 pipe
// cycles for 2704 bit^2) against 4 cycles per 1024 bit^2 for IMAD.WIDE: the same modular product needs
// ~170 FP64-pipe instructions (340 cycles) instead of ~150 IMAD-pipe instructions (600 cycles).
//
// The limb product (N. Emmart's double-precision split): for integer-valued doubles x, y in [0, 2^52)
//     hi = fma_rz(x, y, 2^104)            = 2^104 + floor(x y / 2^52) 2^52   (exact under round-to-zero)
//     lo = fma_rz(x, y, (2^104 + 2^52) - hi) = 2^52 + (x y mod 2^52)          (exact)
// so the IEEE bit patterns are E1 + H and E0 + L with E1 = bits(2^104), E0 = bits(2^52); sums of bit patterns
// are taken with 64-bit integer adds into ten column accumulators that start at minus the sum of the E
// constants they will receive.  Montgomery reduction is word-serial in the same columns (m_i = t_i * (-p^-1)
// mod 2^52, its low product with p_0 is never computed: it cancels t_i by construction).
//
// Value ranges: limbs are integers in [0, 2^52) ("normalized"); operands of mul/sqr must be < 8 p; since
// p / R < 2^-6 the result is < p (1 + X Y / 64) < 2 p for operands < X p, Y p.  Elements are kept lazily in
// [0, 8 p) -- callers add multiples of p before subtracting and only test "== 0 mod p" through zero_mod_p().
//
// Host build (tests/emu, tests of this file): the same code with fesetround-based emulation of the rounding
// modes, so exactness is checked against big integers on a box without a GPU.
#pragma once
#include <stdint.h>
#include "cs_prims.cuh"
#include "cs_field.cuh"

#if defined(CS_EMU) || !defined(__CUDA_ARCH__)
#include <cfenv>
#include <cmath>
#include <cstring>
#endif

namespace cs {

#if defined(__CUDA_ARCH__) && !defined(CS_EMU)
CS_D double f52_fma_rz(double a, double b, double c) { return __fma_rz(a, b, c); }
CS_D double f52_add(double a, double b) { return __dadd_rn(a, b); }
CS_D uint64_t f52_bits(double a) { return (uint64_t)__double_as_longlong(a); }
CS_D double f52_dbl(uint64_t b) { return __longlong_as_double((long long)b); }
#else
inline double f52_fma_rz(double a, double b, double c) {
  const int old = fegetround();
  fesetround(FE_TOWARDZERO);
  volatile double va = a, vb = b, vc = c;
  volatile double r = std::fma(va, vb, vc);
  fesetround(old);
  return r;
}
inline double f52_add(double a, double b) { volatile double va = a, vb = b; volatile double r = va + vb; return r; }
inline uint64_t f52_bits(double a) { uint64_t b; memcpy(&b, &a, 8); return b; }
inline double f52_dbl(uint64_t b) { double a; memcpy(&a, &b, 8); return a; }
#endif

constexpr uint64_t F52_E0 = 0x4330000000000000ull;  // bits(2^52)
constexpr uint64_t F52_E1 = 0x4670000000000000ull;  // bits(2^104)
constexpr uint64_t F52_MASK = (1ull << 52) - 1;
#define F52_C1 0x1p104
#define F52_C2 (0x1p104 + 0x1p52)
#define F52_W 0x1p52

// Integer limbs (the stored form) and their double form (what a multiplicand must be).
struct I52 { uint64_t l[5]; };
struct D52 { double l[5]; };

CS_D D52 f52_to_double(const I52& a) {
  D52 r;
  CS_UNROLL
  for (int k = 0; k < 5; k++) r.l[k] = f52_add(f52_dbl(a.l[k] | F52_E0), -F52_W);  // (2^52 + t) - 2^52
  return r;
}

// P52: constants of one prime, all as 52-bit limbs:  mod(k), np (= -p^-1 mod 2^52), kp(K, k) = limbs of K p
template <class P52, bool SQR>
CS_D I52 f52_mul_core(const D52& a, const D52& b) {
  // columns start at minus the sum of the E constants they will receive; the counts are fixed at compile time
  uint64_t c[10];
  CS_UNROLL
  for (int k = 0; k < 10; k++) {
    int nlo = 0, nhi = 0;
    for (int i = 0; i < 5; i++)
      for (int j = 0; j < 5; j++) {
        if (i + j == k) nlo++;                 // a_i b_j, low half
        if (i + j + 1 == k) nhi++;             // a_i b_j, high half
        if (i + j == k && j >= 1) nlo++;       // m_i p_j, low half (j = 0 is never formed)
        if (i + j + 1 == k) nhi++;             // m_i p_j, high half
      }
    c[k] = 0ull - ((uint64_t)nlo * F52_E0 + (uint64_t)nhi * F52_E1);
  }
  // ---- a * b
  CS_UNROLL
  for (int i = 0; i < 5; i++) {
    CS_UNROLL
    for (int j = 0; j < 5; j++) {
      if (SQR && j < i) continue;
      const double hi = f52_fma_rz(a.l[i], b.l[j], F52_C1);
      const double lo = f52_fma_rz(a.l[i], b.l[j], f52_add(F52_C2, -hi));
      const uint64_t hb = f52_bits(hi), lb = f52_bits(lo);
      if (SQR && j > i) {  // the symmetric term a_j a_i: same bit patterns once more
        c[i + j] += lb + lb;
        c[i + j + 1] += hb + hb;
      } else {
        c[i + j] += lb;
        c[i + j + 1] += hb;
      }
    }
  }
  // ---- word-serial Montgomery reduction
  CS_UNROLL
  for (int i = 0; i < 5; i++) {
    const uint64_t t = c[i] & F52_MASK;
    const double td = f52_add(f52_dbl(t | F52_E0), -F52_W);
    // m = (t * np) mod 2^52: only the low half of the product is needed
    const double mh = f52_fma_rz(td, P52::np(), F52_C1);
    const double ml = f52_fma_rz(td, P52::np(), f52_add(F52_C2, -mh));
    const double md = f52_add(ml, -F52_W);
    // column i becomes a multiple of 2^52 once m p_0's low half is added: carry = ceil(c_i / 2^52)
    c[i + 1] += (c[i] + F52_MASK) >> 52;
    c[i + 1] += f52_bits(f52_fma_rz(md, P52::mod_d(0), F52_C1));
    CS_UNROLL
    for (int j = 1; j < 5; j++) {
      const double hi = f52_fma_rz(md, P52::mod_d(j), F52_C1);
      const double lo = f52_fma_rz(md, P52::mod_d(j), f52_add(F52_C2, -hi));
      c[i + j] += f52_bits(lo);
      c[i + j + 1] += f52_bits(hi);
    }
  }
  // ---- result = columns 5..9, carries propagated
  I52 r;
  uint64_t carry = 0;
  CS_UNROLL
  for (int k = 0; k < 5; k++) {
    const uint64_t v = c[5 + k] + carry;
    r.l[k] = v & F52_MASK;
    carry = v >> 52;
  }
  return r;
}

template <class P52> CS_DN I52 f52_mul(D52 a, D52 b) { return f52_mul_core<P52, false>(a, b); }
template <class P52> CS_DN I52 f52_sqr(D52 a) { return f52_mul_core<P52, true>(a, a); }

// r = a - b + K p  (limbs signed in flight, normalized on the way out).  Requires b <= K p so that the value
// stays non-negative; the result is < a + K p.
template <class P52, int K>
CS_D I52 f52_sub(const I52& a, const I52& b) {
  I52 r;
  int64_t carry = 0;
  CS_UNROLL
  for (int k = 0; k < 5; k++) {
    const int64_t v = (int64_t)a.l[k] - (int64_t)b.l[k] + (int64_t)P52::kp(K, k) + carry;
    r.l[k] = (uint64_t)v & F52_MASK;
    carry = v >> 52;  // arithmetic shift: floor
  }
  return r;
}
// r = a + b (normalized; caller keeps the value below 8 p)
template <class P52>
CS_D I52 f52_add_i(const I52& a, const I52& b) {
  I52 r;
  uint64_t carry = 0;
  CS_UNROLL
  for (int k = 0; k < 5; k++) {
    const uint64_t v = a.l[k] + b.l[k] + carry;
    r.l[k] = v & F52_MASK;
    carry = v >> 52;
  }
  return r;
}

// Cheap NECESSARY condition for v == 0 (mod p) with v in [0, 8 p): the low 32 bits match one of k p, k = 0..7.
// A hit (probability 2^-29 for unrelated values) sends the caller to its exact slow path.
template <class P52>
CS_D bool f52_maybe_zero_mod_p(const I52& v) {
  const uint32_t w = (uint32_t)v.l[0];
  bool hit = false;
  CS_UNROLL
  for (int k = 0; k < 8; k++) hit = hit || (w == (uint32_t)(P52::kp(k, 0)));
  return hit;
}

// ---- 8 x 32-bit Montgomery (R = 2^256, canonical) <-> 5 x 52-bit Montgomery (R = 2^260, lazy) ------------
// in:  x 2^256 (canonical, 8 words) -> limbs -> * (2^264 mod p) / 2^260 = x 2^260
// out: x 2^260 (< 8 p)             -> * (2^256 mod p) / 2^260 = x 2^256 (< 1.125 p) -> words -> one subtraction
template <class P52, class P32>
CS_D I52 f52_from_fp(const Fp<P32>& x) {
  static_assert(P32::N == 8, "5 x 52-bit limbs cover 256-bit fields only");
  I52 v;
  const uint64_t w0 = x.l[0] | ((uint64_t)x.l[1] << 32), w1 = x.l[2] | ((uint64_t)x.l[3] << 32);
  const uint64_t w2 = x.l[4] | ((uint64_t)x.l[5] << 32), w3 = x.l[6] | ((uint64_t)x.l[7] << 32);
  v.l[0] = w0 & F52_MASK;
  v.l[1] = ((w0 >> 52) | (w1 << 12)) & F52_MASK;
  v.l[2] = ((w1 >> 40) | (w2 << 24)) & F52_MASK;
  v.l[3] = ((w2 >> 28) | (w3 << 36)) & F52_MASK;
  v.l[4] = w3 >> 16;
  I52 cin;
  CS_UNROLL
  for (int k = 0; k < 5; k++) cin.l[k] = P52::c_in(k);
  return f52_mul<P52>(f52_to_double(v), f52_to_double(cin));
}

template <class P52, class P32>
CS_D Fp<P32> f52_to_fp(const I52& x) {
  I52 cout;
  CS_UNROLL
  for (int k = 0; k < 5; k++) cout.l[k] = P52::c_out(k);
  const I52 v = f52_mul<P52>(f52_to_double(x), f52_to_double(cout));  // < 1.125 p < 2^255
  const uint64_t w0 = v.l[0] | (v.l[1] << 52), w1 = (v.l[1] >> 12) | (v.l[2] << 40);
  const uint64_t w2 = (v.l[2] >> 24) | (v.l[3] << 28), w3 = (v.l[3] >> 36) | (v.l[4] << 16);
  Fp<P32> r;
  r.l[0] = (uint32_t)w0; r.l[1] = (uint32_t)(w0 >> 32); r.l[2] = (uint32_t)w1; r.l[3] = (uint32_t)(w1 >> 32);
  r.l[4] = (uint32_t)w2; r.l[5] = (uint32_t)(w2 >> 32); r.l[6] = (uint32_t)w3; r.l[7] = (uint32_t)(w3 >> 32);
  r.final_sub();
  return r;
}

}  // namespace cs
