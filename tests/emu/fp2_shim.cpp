// Host-side test shim for the lazy-reduced Fp2 arithmetic (TEST INFRASTRUCTURE): the unreduced product and the
// separate Montgomery reduction of cs_field.cuh, and the Fp2 product and a b - c d of cs_curve.cuh, compiled with
// the emulated carry chain and exported for ctypes.  Every function works on n consecutive operands.
#include "cs_emu.h"
#include "cs_params.cuh"
#include "cs_curve.cuh"
using namespace cs;

template <class P>
static Fp<P> ld(const uint32_t* a) {
  Fp<P> r;
  for (int i = 0; i < P::N; i++) r.l[i] = a[i];
  return r;
}
template <class P>
static Fp2<P> ld2(const uint32_t* a) {
  Fp2<P> r;
  r.c0 = ld<P>(a);
  r.c1 = ld<P>(a + P::N);
  return r;
}
template <class P>
static void st2(const Fp2<P>& x, uint32_t* out) {
  for (int i = 0; i < P::N; i++) { out[i] = x.c0.l[i]; out[P::N + i] = x.c1.l[i]; }
}

#define FP2_SHIM(name, P)                                                                                           \
  extern "C" void name##_mul_wide(int n, const uint32_t* a, const uint32_t* b, uint32_t* t) {                       \
    for (int k = 0; k < n; k++) Fp<P>::mul_wide(t + 2 * P::N * k, ld<P>(a + P::N * k), ld<P>(b + P::N * k));        \
  }                                                                                                                 \
  extern "C" void name##_redc(int n, const uint32_t* t, uint32_t* out) {                                            \
    for (int k = 0; k < n; k++) {                                                                                   \
      Fp<P> r = Fp<P>::redc(t + 2 * P::N * k);                                                                      \
      for (int i = 0; i < P::N; i++) out[P::N * k + i] = r.l[i];                                                    \
    }                                                                                                               \
  }                                                                                                                 \
  extern "C" void name##_fp2_mul(int n, const uint32_t* a, const uint32_t* b, uint32_t* out) {                      \
    for (int k = 0; k < n; k++) st2<P>(ld2<P>(a + 2 * P::N * k) * ld2<P>(b + 2 * P::N * k), out + 2 * P::N * k);   \
  }                                                                                                                 \
  extern "C" void name##_fp2_mul_sub(int n, const uint32_t* a, const uint32_t* b, const uint32_t* c,               \
                                     const uint32_t* d, uint32_t* out) {                                            \
    for (int k = 0; k < n; k++) {                                                                                   \
      const int o = 2 * P::N * k;                                                                                   \
      st2<P>(mul_sub(ld2<P>(a + o), ld2<P>(b + o), ld2<P>(c + o), ld2<P>(d + o)), out + o);                         \
    }                                                                                                               \
  }

FP2_SHIM(bn254, Bn254Fq)
FP2_SHIM(bls381, Bls381Fq)
