// Issue-rate probe for the pipes a 256-bit modular multiplication can use on H100 (sm_90a):
//   * IMAD.WIDE.U32 without carries, with carry-out only, and the carry-in/out (.X) form the CIOS product uses
//   * DFMA (FP64 pipe) alone and interleaved with IMAD.WIDE -- do the two pipes overlap?
//   * IADD3 / IADD3.X (ALU pipe) alone and interleaved with IMAD.WIDE
//   * a Fermat inversion in units of Montgomery products (break-even of batched-affine additions, DESIGN.md)
// Output: one JSON object; rates in T instr/s over the whole chip.  Build as tools/imad_peak.cu.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../co_snarks_b200/csrc/cs_params.cuh"
#include "../co_snarks_b200/csrc/cs_field.cuh"

using namespace cs;

constexpr int CH = 8;

__global__ void k_wide_plain(uint64_t* out, uint32_t a, uint32_t b, int iters) {
  uint64_t acc[CH];
  uint32_t x[CH];
#pragma unroll
  for (int c = 0; c < CH; c++) { acc[c] = threadIdx.x + c; x[c] = a * (c + 1) + threadIdx.x; }
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CH; c++) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[c]) : "r"((uint32_t)acc[(c + 1) % CH]), "r"(b));
  }
  uint64_t s = 0;
#pragma unroll
  for (int c = 0; c < CH; c++) s += acc[c] + x[c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// all three operands distinct registers per instruction (no operand-reuse cache help)
__global__ void k_wide_noreuse(uint64_t* out, uint32_t a, uint32_t b, int iters) {
  uint64_t acc[CH];
  uint32_t x[CH], y[CH];
#pragma unroll
  for (int c = 0; c < CH; c++) { acc[c] = threadIdx.x + c; x[c] = a * (c + 1) + threadIdx.x; y[c] = b * (c + 3) + threadIdx.x; }
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CH; c++) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[c]) : "r"((uint32_t)acc[(c + 1) % CH]), "r"((uint32_t)(acc[(c + 3) % CH] >> 32)));
  }
  uint64_t s = 0;
#pragma unroll
  for (int c = 0; c < CH; c++) s += acc[c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// the carry chain of the library's product: 1 IMAD.WIDE with carry-out + 3 IMAD.WIDE.X per row of 8 limbs
__global__ void k_wide_carry(uint32_t* out, uint32_t a, uint32_t b, int iters) {
  uint32_t acc[2][8], x[8];
#pragma unroll
  for (int c = 0; c < 8; c++) { acc[0][c] = threadIdx.x + c; acc[1][c] = threadIdx.x * 3 + c; x[c] = a * (c + 1) + threadIdx.x; }
  for (int i = 0; i < iters; i++) {
    cmad_n<8>(acc[0], x, b);
    cmad_n<8>(acc[1], x + 1 - 1, b + 1);
  }
  uint32_t s = 0;
#pragma unroll
  for (int c = 0; c < 8; c++) s += acc[0][c] ^ acc[1][c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_dfma(double* out, double a, double b, int iters) {
  double acc[CH];
#pragma unroll
  for (int c = 0; c < CH; c++) acc[c] = threadIdx.x + c;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CH; c++) asm volatile("fma.rz.f64 %0, %1, %2, %0;" : "+d"(acc[c]) : "d"(acc[(c + 1) % CH]), "d"(b));
  }
  double s = 0;
#pragma unroll
  for (int c = 0; c < CH; c++) s += acc[c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// NI IMAD.WIDE and ND DFMA per inner step, independent chains
template <int NI, int ND>
__global__ void k_mix_dfma(uint64_t* out, uint32_t a, uint32_t b, double da, double db, int iters) {
  uint64_t acc[NI > 0 ? NI : 1];
  double dacc[ND > 0 ? ND : 1];
#pragma unroll
  for (int c = 0; c < NI; c++) acc[c] = threadIdx.x + c;
#pragma unroll
  for (int c = 0; c < ND; c++) dacc[c] = threadIdx.x + c;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < (NI > ND ? NI : ND); c++) {
      if (c < NI) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[c]) : "r"((uint32_t)acc[(c + 1) % (NI > 0 ? NI : 1)]), "r"(b));
      if (c < ND) asm volatile("fma.rz.f64 %0, %1, %2, %0;" : "+d"(dacc[c]) : "d"(dacc[(c + 1) % (ND > 0 ? ND : 1)]), "d"(db));
    }
  }
  uint64_t s = 0;
#pragma unroll
  for (int c = 0; c < NI; c++) s += acc[c];
#pragma unroll
  for (int c = 0; c < ND; c++) s += (uint64_t)dacc[c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// 64-bit adds as IADD3 + IADD3.X pairs (ALU pipe), optionally interleaved with IMAD.WIDE
template <int NI, int NA>
__global__ void k_mix_alu(uint64_t* out, uint32_t a, uint32_t b, int iters) {
  uint64_t acc[NI > 0 ? NI : 1];
  uint32_t lo[NA > 0 ? NA : 1], hi[NA > 0 ? NA : 1];
#pragma unroll
  for (int c = 0; c < NI; c++) acc[c] = threadIdx.x + c;
#pragma unroll
  for (int c = 0; c < NA; c++) { lo[c] = threadIdx.x + c; hi[c] = c; }
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < (NI > NA ? NI : NA); c++) {
      if (c < NI) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[c]) : "r"((uint32_t)acc[(c + 1) % (NI > 0 ? NI : 1)]), "r"(b));
      if (c < NA) asm volatile("add.cc.u32 %0, %0, %2; addc.u32 %1, %1, %3;" : "+r"(lo[c]), "+r"(hi[c]) : "r"(hi[(c + 1) % (NA > 0 ? NA : 1)]), "r"(lo[(c + 3) % (NA > 0 ? NA : 1)]));
    }
  }
  uint64_t s = 0;
#pragma unroll
  for (int c = 0; c < NI; c++) s += acc[c];
#pragma unroll
  for (int c = 0; c < NA; c++) s += lo[c] + ((uint64_t)hi[c] << 32);
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// d = a * b (IMAD.WIDE.U32 with RZ addend), operands taken from other chains' results
__global__ void k_mulwide_rz(uint64_t* out, uint32_t a, uint32_t b, int iters) {
  uint64_t acc[CH];
#pragma unroll
  for (int c = 0; c < CH; c++) acc[c] = ((uint64_t)(threadIdx.x + c + a) << 32) | (b + c);
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CH; c++)
      asm volatile("mul.wide.u32 %0, %1, %2;" : "=l"(acc[c]) : "r"((uint32_t)acc[(c + 1) % CH]), "r"((uint32_t)(acc[(c + 3) % CH] >> 32)));
  }
  uint64_t s = 0;
#pragma unroll
  for (int c = 0; c < CH; c++) s += acc[c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int HI>
__global__ void k_imad32(uint32_t* out, uint32_t a, uint32_t b, int iters) {
  uint32_t acc[CH];
#pragma unroll
  for (int c = 0; c < CH; c++) acc[c] = threadIdx.x * 2654435761u + c * 40503u + a;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CH; c++) {
      if (HI) asm volatile("mad.hi.u32 %0, %1, %2, %0;" : "+r"(acc[c]) : "r"(acc[(c + 1) % CH]), "r"(acc[(c + 3) % CH]));
      else asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(acc[c]) : "r"(acc[(c + 1) % CH]), "r"(acc[(c + 3) % CH]));
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int c = 0; c < CH; c++) s += acc[c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// product with RZ addend + the two words added into a running 3-word column by carry-chained adds
__global__ void k_mulwide_plus_adds(uint32_t* out, uint32_t a, uint32_t b, int iters) {
  uint32_t c0[4], c1[4], c2[4], x[4], y[4];
#pragma unroll
  for (int c = 0; c < 4; c++) { c0[c] = threadIdx.x + c; c1[c] = c; c2[c] = 0; x[c] = a * (c + 1) + threadIdx.x; y[c] = b + c; }
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < 4; c++) {
      uint32_t lo, hi;
      asm volatile("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;" : "=r"(lo), "=r"(hi) : "r"(x[c] ^ c0[(c + 1) % 4]), "r"(y[c]));
      asm volatile("add.cc.u32 %0, %0, %3; addc.cc.u32 %1, %1, %4; addc.u32 %2, %2, 0;" : "+r"(c0[c]), "+r"(c1[c]), "+r"(c2[c]) : "r"(lo), "r"(hi));
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int c = 0; c < 4; c++) s += c0[c] ^ c1[c] ^ c2[c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_inverse(uint32_t* out, int iters) {
  typedef Fp<Bn254Fq> F;
  F x;
  for (int i = 0; i < 8; i++) x.l[i] = threadIdx.x * 77 + i + blockIdx.x;
  x.l[7] &= 0x0fffffff;
  for (int i = 0; i < iters; i++) x = x.inverse() + F::one();
  out[blockIdx.x * blockDim.x + threadIdx.x] = x.l[0] ^ x.l[7];
}

__global__ void k_mulchain(uint32_t* out, int iters) {
  typedef Fp<Bn254Fq> F;
  F x, y;
  for (int i = 0; i < 8; i++) { x.l[i] = threadIdx.x * 77 + i; y.l[i] = blockIdx.x + i * 3 + 1; }
  for (int i = 0; i < iters; i++) x = x * y;
  out[blockIdx.x * blockDim.x + threadIdx.x] = x.l[0] ^ x.l[7];
}

template <class K>
float time_ms(K launch) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  launch();
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  launch();
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms;
  cudaEventElapsedTime(&ms, e0, e1);
  return ms;
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  const int sms = p.multiProcessorCount;
  void* buf;
  cudaMalloc(&buf, (size_t)sms * 2048 * 8);
  const int threads = 512, blocks = sms * 4, iters = 4096;
  const double thr = (double)blocks * threads;
  printf("{\"device\": \"%s\", \"sms\": %d", p.name, sms);
  float ms;
  ms = time_ms([&] { k_wide_plain<<<blocks, threads>>>((uint64_t*)buf, 3, 5, iters); });
  printf(", \"imad_wide_plain_tops\": %.3f", thr * CH * iters / (ms * 1e-3) / 1e12);
  ms = time_ms([&] { k_wide_noreuse<<<blocks, threads>>>((uint64_t*)buf, 3, 5, iters); });
  printf(", \"imad_wide_noreuse_tops\": %.3f", thr * CH * iters / (ms * 1e-3) / 1e12);
  ms = time_ms([&] { k_wide_carry<<<blocks, threads>>>((uint32_t*)buf, 3, 5, iters); });
  printf(", \"imad_wide_carrychain_tops\": %.3f", thr * 8 * iters / (ms * 1e-3) / 1e12);
  ms = time_ms([&] { k_mulwide_rz<<<blocks, threads>>>((uint64_t*)buf, 3, 5, iters); });
  printf(", \"imad_wide_rz_tops\": %.3f", thr * CH * iters / (ms * 1e-3) / 1e12);
  ms = time_ms([&] { k_imad32<0><<<blocks, threads>>>((uint32_t*)buf, 3, 5, iters); });
  printf(", \"imad_lo_tops\": %.3f", thr * CH * iters / (ms * 1e-3) / 1e12);
  ms = time_ms([&] { k_imad32<1><<<blocks, threads>>>((uint32_t*)buf, 3, 5, iters); });
  printf(", \"imad_hi_tops\": %.3f", thr * CH * iters / (ms * 1e-3) / 1e12);
  ms = time_ms([&] { k_mulwide_plus_adds<<<blocks, threads>>>((uint32_t*)buf, 3, 5, iters); });
  printf(", \"mulwide_plus_3adds_tops\": %.3f", thr * 4 * iters / (ms * 1e-3) / 1e12);
  ms = time_ms([&] { k_dfma<<<blocks, threads>>>((double*)buf, 1.000001, 0.999999, iters); });
  printf(", \"dfma_tops\": %.3f", thr * CH * iters / (ms * 1e-3) / 1e12);
  ms = time_ms([&] { k_mix_dfma<8, 8><<<blocks, threads>>>((uint64_t*)buf, 3, 5, 1.000001, 0.999999, iters); });
  printf(", \"mix_imad8_dfma8_ms\": %.3f", ms);
  ms = time_ms([&] { k_mix_dfma<8, 0><<<blocks, threads>>>((uint64_t*)buf, 3, 5, 1.000001, 0.999999, iters); });
  printf(", \"mix_imad8_dfma0_ms\": %.3f", ms);
  ms = time_ms([&] { k_mix_dfma<0, 8><<<blocks, threads>>>((uint64_t*)buf, 3, 5, 1.000001, 0.999999, iters); });
  printf(", \"mix_imad0_dfma8_ms\": %.3f", ms);
  ms = time_ms([&] { k_mix_dfma<8, 4><<<blocks, threads>>>((uint64_t*)buf, 3, 5, 1.000001, 0.999999, iters); });
  printf(", \"mix_imad8_dfma4_ms\": %.3f", ms);
  ms = time_ms([&] { k_mix_alu<0, 8><<<blocks, threads>>>((uint64_t*)buf, 3, 5, iters); });
  printf(", \"alu_add64_tops\": %.3f, \"mix_imad0_add8_ms\": %.3f", thr * 8 * iters / (ms * 1e-3) / 1e12, ms);
  ms = time_ms([&] { k_mix_alu<8, 8><<<blocks, threads>>>((uint64_t*)buf, 3, 5, iters); });
  printf(", \"mix_imad8_add8_ms\": %.3f", ms);
  ms = time_ms([&] { k_mix_alu<8, 0><<<blocks, threads>>>((uint64_t*)buf, 3, 5, iters); });
  printf(", \"mix_imad8_add0_ms\": %.3f", ms);
  {
    const int t2 = 128, b2 = sms * 16, it = 8;
    float mi = time_ms([&] { k_inverse<<<b2, t2>>>((uint32_t*)buf, it); });
    float mm = time_ms([&] { k_mulchain<<<b2, t2>>>((uint32_t*)buf, it * 256); });
    printf(", \"fermat_inverse_in_products\": %.1f, \"inverse_ginv_s\": %.4f", mi / (mm / 256.0), (double)b2 * t2 * it / (mi * 1e-3) / 1e9);
  }
  printf("}\n");
  return 0;
}
