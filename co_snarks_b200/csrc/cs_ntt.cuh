// Radix-2 NTT over the scalar field, shared-memory staged.
//
// Replaces `taceo_ark_algebra::fft::Domain::{ifft_in_to_out, fft_out_to_in}` (call sites
// co-groth16/src/groth16/reduction.rs:141-175,270-327) and, with the bit-reversal kernel, the
// natural-order `domain.fft/ifft` of co-plonk (co-plonk/src/mpc/rep3.rs:140-152).
//   in_to_out : natural order in  -> bit-reversed order out  (decimation in frequency)
//   out_to_in : bit-reversed in   -> natural order out       (decimation in time)
// so the iNTT -> coset scale -> NTT chain of the witness map needs no permutation, exactly as the
// reference arranges it (reduction.rs:70-72).  The caller supplies the group generator (snarkjs
// roots, groth16.rs:60-100); twiddles w^k, k < n/2, are precomputed once per (n, generator) in HBM.
//
// A pass runs up to NTT_MAX_K butterfly stages on a 2^k-row tile held in shared memory (two uint4
// planes per element, conflict-free for LDS.128), so 2^20 takes two passes.  `batch` interleaved
// components (1 = field elements, 2 = Rep3 shares {a,b}) ride along as tile columns, so a share
// vector is transformed in place without a transpose.
#pragma once
#include "cs_common.cuh"
#include "cs_field.cuh"

namespace cs {

constexpr unsigned NTT_MAX_K = 10;

template <class FrP>
CS_D Fp<FrP> ld_fr(const uint32_t* p) {
  Fp<FrP> r;
  const uint4* q = reinterpret_cast<const uint4*>(p);
  CS_UNROLL
  for (int k = 0; k < FrP::N / 4; k++) {
    uint4 v = q[k];
    r.l[4 * k] = v.x; r.l[4 * k + 1] = v.y; r.l[4 * k + 2] = v.z; r.l[4 * k + 3] = v.w;
  }
  return r;
}
template <class FrP>
CS_D void st_fr(uint32_t* p, const Fp<FrP>& v) {
  uint4* q = reinterpret_cast<uint4*>(p);
  CS_UNROLL
  for (int k = 0; k < FrP::N / 4; k++) q[k] = make_uint4(v.l[4 * k], v.l[4 * k + 1], v.l[4 * k + 2], v.l[4 * k + 3]);
}

// tw[k] = g^k for k < count, from the squarings table pw[j] = g^(2^j)
template <class FrP>
CS_GLOBAL void k_ntt_twiddles(const uint32_t* __restrict__ pw, uint32_t count, uint32_t* __restrict__ tw) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  Fp<FrP> acc = Fp<FrP>::one();
  for (uint32_t j = 0; (k >> j) != 0; j++)
    if ((k >> j) & 1) acc = acc * ld_fr<FrP>(pw + (size_t)j * FrP::N);
  st_fr<FrP>(tw + (size_t)k * FrP::N, acc);
}

// tab[p] = scale * g^(bitrev(p))   (bit-reversed coset table with the 1/n of the inverse NTT folded in;
// reduction.rs:45-60 builds shift^i and permutes it the same way)
template <class FrP>
CS_GLOBAL void k_ntt_coset_table(const uint32_t* __restrict__ pw, const uint32_t* __restrict__ scale,
                                 uint32_t logn, uint32_t* __restrict__ tab) {
  uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (1u << logn)) return;
  uint32_t k = logn ? (__brev(p) >> (32 - logn)) : 0;
  Fp<FrP> acc = ld_fr<FrP>(scale);
  for (uint32_t j = 0; (k >> j) != 0; j++)
    if ((k >> j) & 1) acc = acc * ld_fr<FrP>(pw + (size_t)j * FrP::N);
  st_fr<FrP>(tab + (size_t)p * FrP::N, acc);
}

// One pass = stages on index bits [log_stride, log_stride + k).  Tile rows r in [0, 2^k):
//   g = hi * (2^k * stride) + r * stride + lo.   Block = one (hi, lo) pair, all `batch` components.
// DIT=false: decimation in frequency (half-size shrinks);  DIT=true: decimation in time.
// post (optional): out[g] *= post[g]   (per-element table, e.g. the scaled coset table)
// scale (optional): out[g] *= *scale   (e.g. 1/n)
// TWS: the pass's 2^k - 1 twiddles are staged in shared memory next to the tile (heap order: the stage with
// local half-size mm uses entries [mm - 1, 2 mm - 1)), so the stage loop never waits on L2.
template <class FrP, bool DIT, bool TWS>
CS_GLOBAL void __launch_bounds__(512) k_ntt_pass(uint32_t* __restrict__ data, const uint32_t* __restrict__ tw, uint32_t logn,
                          uint32_t log_stride, uint32_t k, uint32_t batch,
                          const uint32_t* __restrict__ post, const uint32_t* __restrict__ scale) {
  typedef Fp<FrP> F;
  constexpr int NW = FrP::N;  // words per element (8)
  CS_DYN_SMEM(uint4, sm);
  const uint32_t rows = 1u << k;
  const uint32_t stride = 1u << log_stride;
  const uint32_t cols = batch;
  uint4* pl0 = sm;
  uint4* pl1 = sm + (size_t)rows * cols;
  const uint32_t tile = blockIdx.x;
  const uint32_t lo = tile & (stride - 1);
  const uint32_t hi = tile >> log_stride;
  const size_t gbase = ((size_t)hi << (k + log_stride)) + lo;
  const uint32_t T = blockDim.x;
  uint4* tp0 = pl1 + (size_t)rows * cols;
  uint4* tp1 = tp0 + rows;
  if (TWS) {
    for (uint32_t idx = threadIdx.x; idx + 1 < rows; idx += T) {
      uint32_t e = idx + 1;
      uint32_t lmm = 31 - __clz(e);
      uint32_t jj = (e - (1u << lmm)) * stride + lo;
      const uint4* src = reinterpret_cast<const uint4*>(tw + ((size_t)jj << (logn - 1 - (lmm + log_stride))) * NW);
      tp0[idx] = src[0];
      tp1[idx] = src[1];
    }
  }
  // load
  for (uint32_t idx = threadIdx.x; idx < rows * cols; idx += T) {
    uint32_t r = idx / cols, cix = idx - r * cols;
    size_t g = gbase + (size_t)r * stride;
    const uint4* src = reinterpret_cast<const uint4*>(data + (g * batch + cix) * NW);
    pl0[idx] = src[0];
    pl1[idx] = src[1];
  }
  __syncthreads();
  const uint32_t nbf = (rows >> 1) * cols;
  for (uint32_t q = 0; q < k; q++) {
    const uint32_t lmm = DIT ? q : (k - 1 - q);  // log2 of the local half-size
    const uint32_t mm = 1u << lmm;
    // global half-size m = mm * stride; twiddle index = jj * (n / (2m))
    const uint32_t tshift = logn - 1 - (lmm + log_stride);
    for (uint32_t b = threadIdx.x; b < nbf; b += T) {
      uint32_t bf = b / cols, cix = b - bf * cols;
      uint32_t r0 = ((bf >> lmm) << (lmm + 1)) | (bf & (mm - 1));
      uint32_t r1 = r0 + mm;
      uint32_t i0 = r0 * cols + cix, i1 = r1 * cols + cix;
      uint32_t jj = (r0 & (mm - 1)) * stride + lo;
      F x, y, w;
      {
        uint4 a = pl0[i0], c = pl1[i0];
        x.l[0] = a.x; x.l[1] = a.y; x.l[2] = a.z; x.l[3] = a.w; x.l[4] = c.x; x.l[5] = c.y; x.l[6] = c.z; x.l[7] = c.w;
        a = pl0[i1]; c = pl1[i1];
        y.l[0] = a.x; y.l[1] = a.y; y.l[2] = a.z; y.l[3] = a.w; y.l[4] = c.x; y.l[5] = c.y; y.l[6] = c.z; y.l[7] = c.w;
      }
      if (TWS) {
        uint32_t ti = (mm - 1) + (r0 & (mm - 1));
        uint4 a = tp0[ti], c = tp1[ti];
        w.l[0] = a.x; w.l[1] = a.y; w.l[2] = a.z; w.l[3] = a.w; w.l[4] = c.x; w.l[5] = c.y; w.l[6] = c.z; w.l[7] = c.w;
      } else {
        w = ld_fr<FrP>(tw + ((size_t)jj << tshift) * NW);
      }
      F o0, o1;
      if (DIT) {
        F t = y * w;
        o0 = x + t;
        o1 = x - t;
      } else {
        o0 = x + y;
        o1 = (x - y) * w;
      }
      pl0[i0] = make_uint4(o0.l[0], o0.l[1], o0.l[2], o0.l[3]);
      pl1[i0] = make_uint4(o0.l[4], o0.l[5], o0.l[6], o0.l[7]);
      pl0[i1] = make_uint4(o1.l[0], o1.l[1], o1.l[2], o1.l[3]);
      pl1[i1] = make_uint4(o1.l[4], o1.l[5], o1.l[6], o1.l[7]);
    }
    __syncthreads();
  }
  // store (+ optional fused scaling)
  for (uint32_t idx = threadIdx.x; idx < rows * cols; idx += T) {
    uint32_t r = idx / cols, cix = idx - r * cols;
    size_t g = gbase + (size_t)r * stride;
    uint4 a = pl0[idx], c = pl1[idx];
    if (post || scale) {
      F v;
      v.l[0] = a.x; v.l[1] = a.y; v.l[2] = a.z; v.l[3] = a.w; v.l[4] = c.x; v.l[5] = c.y; v.l[6] = c.z; v.l[7] = c.w;
      if (post) v = v * ld_fr<FrP>(post + g * NW);
      if (scale) v = v * ld_fr<FrP>(scale);
      a = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
      c = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
    }
    uint4* dst = reinterpret_cast<uint4*>(data + (g * batch + cix) * NW);
    dst[0] = a;
    dst[1] = c;
  }
}

// In-place bit-reversal permutation of n = 2^logn elements of `batch` components (fft::bit_reverse,
// reduction.rs:58,328).
template <class FrP>
CS_GLOBAL void k_bit_reverse(uint32_t* __restrict__ data, uint32_t logn, uint32_t batch) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1u << logn)) return;
  uint32_t j = logn ? (__brev(i) >> (32 - logn)) : 0;
  if (i >= j) return;
  for (uint32_t c = 0; c < batch; c++) {
    uint32_t* pi = data + ((size_t)i * batch + c) * FrP::N;
    uint32_t* pj = data + ((size_t)j * batch + c) * FrP::N;
    Fp<FrP> a = ld_fr<FrP>(pi), b = ld_fr<FrP>(pj);
    st_fr<FrP>(pi, b);
    st_fr<FrP>(pj, a);
  }
}

// Enqueue a whole transform.  tw = forward or inverse twiddle table (n/2 entries).
// dit=false: natural -> bit-reversed;  dit=true: bit-reversed -> natural.
template <class FrP>
int ntt_enqueue(uint32_t* d_data, const uint32_t* d_tw, uint32_t logn, uint32_t batch, bool dit,
                const uint32_t* d_post, const uint32_t* d_scale, cudaStream_t st) {
  if (logn == 0) {
    if (d_post || d_scale) return fail(-3, "ntt: size-1 transform with scaling is not supported on device");
    return 0;
  }
  // split logn into passes of <= NTT_MAX_K stages
  uint32_t npass = (logn + NTT_MAX_K - 1) / NTT_MAX_K;
  uint32_t base = logn / npass, extra = logn % npass;
  uint32_t done = 0;
  for (uint32_t p = 0; p < npass; p++) {
    uint32_t k = base + (p < extra ? 1 : 0);
    // DIF walks index bits from the top, DIT from the bottom
    uint32_t log_stride = dit ? done : (logn - done - k);
    bool last = (p + 1 == npass);
    uint32_t rows = 1u << k;
    static int tws_env = -1, thr_env = -1;  // tuning hooks
    if (tws_env < 0) { const char* e = getenv("CS_NTT_TWS"); tws_env = e ? atoi(e) : 1; }
    if (thr_env < 0) { const char* e = getenv("CS_NTT_THREADS"); thr_env = e ? atoi(e) : 512; }
    const bool tws = tws_env != 0;
    uint32_t threads = (rows / 2) * batch;
    if (threads > (uint32_t)thr_env) threads = thr_env;
    if (threads < 32) threads = 32;
    size_t smem = (size_t)rows * batch * 32 + (tws ? (size_t)rows * 32 : 0);
    uint32_t blocks = 1u << (logn - k);
    const uint32_t* post = last ? d_post : nullptr;
    const uint32_t* scale = last ? d_scale : nullptr;
#define CS_NTT_GO(D, S) \
  CS_LAUNCH_SYNC(k_ntt_pass<FrP COMMA D COMMA S>, blocks, threads, smem, st, d_data, d_tw, logn, log_stride, k, batch, post, scale)
    if (dit) { if (tws) CS_NTT_GO(true, true); else CS_NTT_GO(true, false); }
    else     { if (tws) CS_NTT_GO(false, true); else CS_NTT_GO(false, false); }
#undef CS_NTT_GO
    done += k;
  }
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
