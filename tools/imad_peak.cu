// Integer-pipe microbenchmark for the MSM/NTT roofline: sustained IMAD (32x32+32) and IMAD.WIDE
// (32x32+64) issue rate on H100, and the throughput of the library's Montgomery multiplication.
// HBM and tensor-core peaks say nothing here: 256-bit modular arithmetic is bound by this
// pipe instead (DESIGN.md "Rooflines").  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../co_snarks_b200/csrc/cs_params.cuh"
#include "../co_snarks_b200/csrc/cs_field.cuh"

template <int CHAINS>
__global__ void k_imad_wide(uint64_t* out, uint32_t a, uint32_t b, int iters) {
  uint64_t acc[CHAINS];
#pragma unroll
  for (int c = 0; c < CHAINS; c++) acc[c] = threadIdx.x + c;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CHAINS; c++)
      asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[c]) : "r"(a + c), "r"(b));
  }
  uint64_t s = 0;
#pragma unroll
  for (int c = 0; c < CHAINS; c++) s += acc[c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int CHAINS>
__global__ void k_imad_lo(uint32_t* out, uint32_t a, uint32_t b, int iters) {
  uint32_t acc[CHAINS];
#pragma unroll
  for (int c = 0; c < CHAINS; c++) acc[c] = threadIdx.x + c;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CHAINS; c++)
      asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(acc[c]) : "r"(a + c), "r"(b));
  }
  uint32_t s = 0;
#pragma unroll
  for (int c = 0; c < CHAINS; c++) s += acc[c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// CH independent Montgomery-multiplication chains per thread
template <int CH>
__global__ void k_montmul(uint32_t* out, int iters) {
  typedef cs::Fp<cs::Bn254Fq> F;
  F x[CH], y;
  for (int c = 0; c < CH; c++)
    for (int i = 0; i < 8; i++) x[c].l[i] = threadIdx.x * 77 + i + c;
  for (int i = 0; i < 8; i++) y.l[i] = blockIdx.x + i * 3 + 1;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CH; c++) x[c] = x[c] * y;
  }
  uint32_t s = 0;
  for (int c = 0; c < CH; c++) s += x[c].l[0] ^ x[c].l[7];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}


// ---- experiment: unsaturated 9 x 29-bit limbs, carry-free IMAD.WIDE column accumulation
__device__ __forceinline__ void mul29(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr uint32_t MASK = (1u << 29) - 1;
  constexpr uint32_t N0P = 75916169u;
  const uint32_t P[9] = {410844487u, 17064118u, 477274959u, 47522512u, 361093496u, 47923392u, 10936641u, 240920116u, 3171406u};
  uint64_t t[18];
#pragma unroll
  for (int k = 0; k < 18; k++) t[k] = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) {
#pragma unroll
    for (int j = 0; j < 9; j++) t[i + j] += (uint64_t)a[j] * b[i];
    uint32_t m = ((uint32_t)t[i] * N0P) & MASK;
#pragma unroll
    for (int j = 0; j < 9; j++) t[i + j] += (uint64_t)m * P[j];
    t[i + 1] += t[i] >> 29;
  }
#pragma unroll
  for (int k = 9; k < 17; k++) { t[k + 1] += t[k] >> 29; r[k - 9] = (uint32_t)t[k] & MASK; }
  r[8] = (uint32_t)t[17];
}
__device__ __noinline__ void mul29_ool(uint32_t* r, const uint32_t* a, const uint32_t* b) { mul29(r, a, b); }

template <int CH>
__global__ void k_montmul29(uint32_t* out, int iters) {
  uint32_t x[CH][9], y[9];
  for (int c = 0; c < CH; c++)
    for (int i = 0; i < 9; i++) x[c][i] = (threadIdx.x * 77 + i + c) & 0x1fffffff;
  for (int i = 0; i < 9; i++) y[i] = (blockIdx.x + i * 3 + 1) & 0x1fffffff;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CH; c++) { uint32_t r[9]; mul29(r, x[c], y); for (int k = 0; k < 9; k++) x[c][k] = r[k]; }
  }
  uint32_t s = 0;
  for (int c = 0; c < CH; c++) s += x[c][0] ^ x[c][8];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// ---- experiment: product-scanning (Comba / FIPS) Montgomery multiplication, 8 x 32-bit limbs.
// Each partial product is added into a 3-word column accumulator: IMAD.WIDE with carry-OUT only
// (no carry-in) + one IADD3.X on the ALU pipe, instead of the carry-in/out IMAD.WIDE.X chains.
template <class P>
__device__ __forceinline__ void mul_comba(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  using namespace cs;
  constexpr int N = 8;
  uint32_t c0 = 0, c1 = 0, c2 = 0;
  uint32_t m[N];
#pragma unroll
  for (int k = 0; k < N; k++) {
#pragma unroll
    for (int i = 0; i <= k; i++) {
      c0 = mad_lo_cc(a[i], b[k - i], c0); c1 = madc_hi_cc(a[i], b[k - i], c1); c2 = addc(c2, 0);
    }
#pragma unroll
    for (int i = 0; i < k; i++) {
      c0 = mad_lo_cc(m[i], P::mod(k - i), c0); c1 = madc_hi_cc(m[i], P::mod(k - i), c1); c2 = addc(c2, 0);
    }
    m[k] = mul_lo(c0, P::M0);
    c0 = mad_lo_cc(m[k], P::mod(0), c0); c1 = madc_hi_cc(m[k], P::mod(0), c1); c2 = addc(c2, 0);
    c0 = c1; c1 = c2; c2 = 0;
  }
#pragma unroll
  for (int k = N; k < 2 * N - 1; k++) {
#pragma unroll
    for (int i = k - N + 1; i < N; i++) {
      c0 = mad_lo_cc(a[i], b[k - i], c0); c1 = madc_hi_cc(a[i], b[k - i], c1); c2 = addc(c2, 0);
    }
#pragma unroll
    for (int i = k - N + 1; i < N; i++) {
      c0 = mad_lo_cc(m[i], P::mod(k - i), c0); c1 = madc_hi_cc(m[i], P::mod(k - i), c1); c2 = addc(c2, 0);
    }
    r[k - N] = c0;
    c0 = c1; c1 = c2; c2 = 0;
  }
  r[N - 1] = c0;
  // conditional subtraction
  uint32_t t[N];
  t[0] = sub_cc(r[0], P::mod(0));
#pragma unroll
  for (int i = 1; i < N; i++) t[i] = subc_cc(r[i], P::mod(i));
  uint32_t borrow = subc(0, 0);
#pragma unroll
  for (int i = 0; i < N; i++) r[i] = borrow ? r[i] : t[i];
}

template <int CH>
__global__ void k_montmul_comba(uint32_t* out, int iters, int* mismatch) {
  typedef cs::Fp<cs::Bn254Fq> F;
  F x[CH], y;
  for (int c = 0; c < CH; c++)
    for (int i = 0; i < 8; i++) x[c].l[i] = threadIdx.x * 77 + i + c;
  for (int i = 0; i < 8; i++) y.l[i] = blockIdx.x + i * 3 + 1;
  x[0].l[7] &= 0x0fffffff; y.l[7] &= 0x0fffffff;
  if (blockIdx.x == 0) {  // correctness vs the library multiplication
    F ref = x[0] * y; F got; mul_comba<cs::Bn254Fq>(got.l, x[0].l, y.l);
    if (!(ref == got)) atomicAdd(mismatch, 1);
  }
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CH; c++) { F r; mul_comba<cs::Bn254Fq>(r.l, x[c].l, y.l); x[c] = r; }
  }
  uint32_t s = 0;
  for (int c = 0; c < CH; c++) s += x[c].l[0] ^ x[c].l[7];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
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
  int sms = p.multiProcessorCount;
  void* buf;
  cudaMalloc(&buf, (size_t)sms * 16 * 1024 * 8);
  printf("{\"device\": \"%s\", \"sms\": %d", p.name, sms);
  const int iters = 4096;
  for (int threads : {256, 512, 1024}) {
    int blocks = sms * (2048 / threads);
    float ms = time_ms([&] { k_imad_wide<8><<<blocks, threads>>>((uint64_t*)buf, 3, 5, iters); });
    double ops = (double)blocks * threads * 8 * iters;
    printf(", \"imad_wide_tops_t%d\": %.3f", threads, ops / (ms * 1e-3) / 1e12);
    ms = time_ms([&] { k_imad_lo<8><<<blocks, threads>>>((uint32_t*)buf, 3, 5, iters); });
    printf(", \"imad_lo_tops_t%d\": %.3f", threads, ops / (ms * 1e-3) / 1e12);
  }
  for (int wps : {1, 2, 3, 4, 8}) {  // warps per SM sub-partition
    int threads = 128, blocks = sms * wps;  // 128 threads = 1 warp per SMSP per block
    float ms = time_ms([&] { k_montmul<1><<<blocks, threads>>>((uint32_t*)buf, 2048); });
    double muls = (double)blocks * threads * 2048;
    printf(", \"montmul_gmuls_ch1_w%d\": %.2f", wps, muls / (ms * 1e-3) / 1e9);
    ms = time_ms([&] { k_montmul<2><<<blocks, threads>>>((uint32_t*)buf, 2048); });
    printf(", \"montmul_gmuls_ch2_w%d\": %.2f", wps, 2 * muls / (ms * 1e-3) / 1e9);
  }
  for (int wps : {1, 2, 4, 8}) {
    int threads = 128, blocks = sms * wps;
    float ms = time_ms([&] { k_montmul29<1><<<blocks, threads>>>((uint32_t*)buf, 2048); });
    double muls = (double)blocks * threads * 2048;
    printf(", \"montmul29_gmuls_ch1_w%d\": %.2f", wps, muls / (ms * 1e-3) / 1e9);
    ms = time_ms([&] { k_montmul29<2><<<blocks, threads>>>((uint32_t*)buf, 2048); });
    printf(", \"montmul29_gmuls_ch2_w%d\": %.2f", wps, 2 * muls / (ms * 1e-3) / 1e9);
  }
  int* d_mis; cudaMalloc(&d_mis, 4); cudaMemset(d_mis, 0, 4);
  for (int wps : {1, 2, 4, 8}) {
    int threads = 128, blocks = sms * wps;
    float ms = time_ms([&] { k_montmul_comba<1><<<blocks, threads>>>((uint32_t*)buf, 2048, d_mis); });
    double muls = (double)blocks * threads * 2048;
    printf(", \"comba_gmuls_ch1_w%d\": %.2f", wps, muls / (ms * 1e-3) / 1e9);
    ms = time_ms([&] { k_montmul_comba<2><<<blocks, threads>>>((uint32_t*)buf, 2048, d_mis); });
    printf(", \"comba_gmuls_ch2_w%d\": %.2f", wps, 2 * muls / (ms * 1e-3) / 1e9);
  }
  int mis = -1; cudaMemcpy(&mis, d_mis, 4, cudaMemcpyDeviceToHost);
  printf(", \"comba_mismatches\": %d", mis);
  printf("}\n");
  return 0;
}
