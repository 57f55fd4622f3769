// Carry-chain primitives for multi-limb integer arithmetic on sm_90a.
//
// Device build: one PTX instruction each (add.cc / addc.cc / mad.lo.cc / madc.hi.cc ...); ptxas fuses
// mad.lo.cc + madc.hi.cc pairs into IMAD.WIDE.U32(.X) chains on the FMA pipe.
// CS_EMU build (g++, tests/emu only): the same primitives with an explicit thread-local carry flag so
// the exact device algorithms can be exercised on a CPU-only box.  The emulation build is test
// infrastructure; the product library never contains it.
#pragma once
#include <stdint.h>

#if defined(CS_EMU)
#include "cs_emu.h"
#define CS_D inline
#define CS_DN __attribute__((noinline))
#define CS_HD inline
#define CS_GLOBAL
#define CS_UNROLL
#else
#include <cuda_runtime.h>
#define CS_D __device__ __forceinline__
#define CS_DN __device__ __noinline__
#define CS_HD __host__ __device__ __forceinline__
#define CS_GLOBAL __global__
#define CS_UNROLL _Pragma("unroll")
#endif

namespace cs {

#if defined(CS_EMU)
// ---- emulation: explicit carry flag ---------------------------------------------------------
inline uint32_t& cf_() { static thread_local uint32_t cf = 0; return cf; }
inline uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t s = (uint64_t)a + b; cf_() = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { uint64_t s = (uint64_t)a + b + cf_(); cf_() = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t addc(uint32_t a, uint32_t b) { return (uint32_t)((uint64_t)a + b + cf_()); }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t d = (uint64_t)a - b; cf_() = (uint32_t)((d >> 32) & 1); return (uint32_t)d; }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { uint64_t d = (uint64_t)a - b - cf_(); cf_() = (uint32_t)((d >> 32) & 1); return (uint32_t)d; }
inline uint32_t subc(uint32_t a, uint32_t b) { return (uint32_t)((uint64_t)a - b - cf_()); }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return (uint32_t)((uint64_t)a * b); }
inline uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return add_cc(mul_lo(a, b), c); }
inline uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return addc_cc(mul_lo(a, b), c); }
inline uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) { return add_cc(mul_hi(a, b), c); }
inline uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { return addc_cc(mul_hi(a, b), c); }
inline uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return addc(mul_hi(a, b), c); }
#else
// ---- device: PTX ------------------------------------------------------------------------------
CS_D uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CS_D uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CS_D uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CS_D uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CS_D uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CS_D uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CS_D uint32_t mul_lo(uint32_t a, uint32_t b) { uint32_t r; asm volatile("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CS_D uint32_t mul_hi(uint32_t a, uint32_t b) { uint32_t r; asm volatile("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CS_D uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
CS_D uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
CS_D uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
CS_D uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
CS_D uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
#endif

}  // namespace cs
