// Multi-scalar multiplication  sum_i s_i * P_i  on sm_90a.
//
// Replaces `taceo_ark_algebra::msm::{msm_unchecked, msm_bigint}` (taceo-ark-algebra 0.1.0, not
// vendored; call sites co-groth16/src/mpc/{plain.rs:66-74, rep3.rs:124-132, shamir.rs:111-119},
// co-groth16/src/groth16.rs:190-200, mpc-core/src/protocols/rep3/pointshare.rs:201-222).
//
// Design (DESIGN.md "MSM"):
//  * The base set is a proving key / SRS: it is uploaded once and expanded to a table of
//    2^(c w) * P_i for every window w (W x the key size: ~6.4 GB for a 2^20 Groth16 key, which 80 GB of HBM affords).  All
//    windows then share ONE bucket set, so there is no per-window reduction and no window-combine
//    doubling chain on the per-proof path.
//  * Per MSM: signed c-bit digits -> counting sort by bucket (histogram, scan, scatter) -> bucket
//    accumulation as a load-balanced segmented reduction over fixed-size slices of the sorted entry
//    list (robust to skewed scalars) -> weighted bucket reduction sum_b b * S_b.
//  * Arithmetic is exact 256/381-bit Montgomery on the integer pipe; no tensor cores.
#pragma once
#include <stdlib.h>
#include "cs_common.cuh"
#include "cs_curve.cuh"

namespace cs {

constexpr unsigned MSM_SLICE_MAX = 64;  // entries per slice (levels 0 and 1 of the segmented reduction): 32 or 64
constexpr unsigned MSM_ORDER_BLOCK = 256;
constexpr unsigned MSM_RED_SEG = 4;     // buckets per thread in the weighted bucket reduction
constexpr unsigned MSM_SIGN = 0x80000000u;

// --------------------------------------------------------------------------- digits + histogram
// One thread per scalar: optional Montgomery -> canonical, signed c-bit recoding, histogram.
template <class FrP>
CS_GLOBAL void k_msm_digits(const uint32_t* __restrict__ scalars, uint32_t sstride, uint32_t n, int mont,
                            uint32_t c, uint32_t W, const uint32_t* __restrict__ infmask, uint32_t offset,
                            uint32_t* __restrict__ dig, uint32_t* __restrict__ count) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // bases at infinity (sparse Groth16 B-queries: B_i(tau) = 0 for variables absent from B) contribute
  // nothing: drop their entries before the sort instead of carrying them through the accumulation
  if ((infmask[(offset + i) >> 5] >> ((offset + i) & 31)) & 1) {
    for (uint32_t w = 0; w < W; w++) dig[(size_t)w * n + i] = 0;
    return;
  }
  Fp<FrP> s;
  // sstride = elements between consecutive scalars (2 reads the `a` component of Rep3 shares in place)
  const uint4* src = reinterpret_cast<const uint4*>(scalars) + (size_t)i * sstride * (FrP::N / 4);
  CS_UNROLL
  for (int k = 0; k < FrP::N / 4; k++) {
    uint4 v = src[k];
    s.l[4 * k] = v.x; s.l[4 * k + 1] = v.y; s.l[4 * k + 2] = v.z; s.l[4 * k + 3] = v.w;
  }
  if (mont) s = s.from_mont();
  uint32_t lim[FrP::N + 1];
  CS_UNROLL
  for (int k = 0; k < FrP::N; k++) lim[k] = s.l[k];
  lim[FrP::N] = 0;
  const uint32_t half = 1u << (c - 1);
  const uint32_t mask = (1u << c) - 1;
  uint32_t carry = 0;
  for (uint32_t w = 0; w < W; w++) {
    uint32_t pos = w * c;
    uint32_t li = pos >> 5, sh = pos & 31;
    uint32_t lo = li < FrP::N ? lim[li] : 0;
    uint32_t hi = li + 1 < FrP::N ? lim[li + 1] : 0;
    uint32_t d = (__funnelshift_r(lo, hi, sh) & mask) + carry;
    uint32_t out;
    if (d > half) {
      out = ((1u << c) - d) | MSM_SIGN;
      carry = 1;
    } else {
      out = d;
      carry = 0;
    }
    dig[(size_t)w * n + i] = out;
    uint32_t b = out & ~MSM_SIGN;
    if (b) atomicAdd(&count[b], 1u);
  }
}

// infmask bit i = (base i is the point at infinity); one thread per 32 bases, once per upload
template <class F>
CS_GLOBAL void k_msm_infmask(const Affine<F>* __restrict__ table, uint32_t n, uint32_t* __restrict__ mask) {
  uint32_t wd = blockIdx.x * blockDim.x + threadIdx.x;
  if (wd * 32 >= n) return;
  uint32_t m = 0;
  for (uint32_t k = 0; k < 32 && wd * 32 + k < n; k++)
    if (table[wd * 32 + k].is_inf()) m |= 1u << k;
  mask[wd] = m;
}

// --------------------------------------------------------------------------- scans
// From count[0..B]: start = exclusive scan of count; ns0[b] = ceil(count[b]/S), ns1 = ceil(ns0/S),
// ns2 = ceil(ns1/S) (three fold levels keep the last, serial, per-bucket fold short even when most scalars
// share one digit: 2^24 entries in ONE bucket leave 512 partials); sstart0 / sstart1 / sstart2 = exclusive scans.  Arrays have B + 2 entries (last = total).
// Two launches over ceil((B + 1) / 1024) blocks: coalesced block-local scans (warp shuffles, then the warp totals by
// the first warp) that leave each block's totals in aux[block][4], then the block offsets are added.
constexpr unsigned MSM_SCAN_T = 1024;
constexpr unsigned MSM_SCAN_MAX_BLOCKS = 1024;  // 2^20 buckets
CS_D void msm_scan_terms(const uint32_t* __restrict__ count, uint32_t k, uint32_t nb1, uint32_t S, uint32_t* v) {
  uint32_t cnt = (k && k < nb1) ? count[k] : 0;  // bucket 0 (zero digits) is dropped
  uint32_t n0 = (cnt + S - 1) / S;
  uint32_t n1 = (n0 + S - 1) / S;
  v[0] = cnt; v[1] = n0; v[2] = n1; v[3] = (n1 + S - 1) / S;
}
static CS_GLOBAL void k_msm_scan1(const uint32_t* __restrict__ count, uint32_t nb1 /* B + 1 */, uint32_t S,
                                  uint32_t* __restrict__ start, uint32_t* __restrict__ sstart0,
                                  uint32_t* __restrict__ sstart1, uint32_t* __restrict__ sstart2, uint32_t* __restrict__ aux) {
  __shared__ uint32_t sm[4][32];
  const uint32_t t = threadIdx.x, lane = t & 31, wid = t >> 5, nwarp = blockDim.x >> 5;
  const uint32_t k = blockIdx.x * blockDim.x + t;
  uint32_t v[4], inc[4];
  msm_scan_terms(count, k, nb1, S, v);
  CS_UNROLL
  for (int q = 0; q < 4; q++) {
    uint32_t x = v[q];
    CS_UNROLL
    for (uint32_t d = 1; d < 32; d <<= 1) {
      uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    inc[q] = x;
    if (lane == 31) sm[q][wid] = x;
  }
  __syncthreads();
  uint32_t w[4], x[4];
  CS_UNROLL
  for (int q = 0; q < 4; q++) {
    w[q] = (wid == 0 && lane < nwarp) ? sm[q][lane] : 0;
    x[q] = w[q];
    CS_UNROLL
    for (uint32_t d = 1; d < 32; d <<= 1) {
      uint32_t y = __shfl_up_sync(0xffffffffu, x[q], d);
      if (lane >= d) x[q] += y;
    }
  }
  __syncthreads();
  if (wid == 0 && lane < nwarp) {
    CS_UNROLL
    for (int q = 0; q < 4; q++) sm[q][lane] = x[q] - w[q];  // exclusive prefix of the warp totals
    if (lane == nwarp - 1) {
      CS_UNROLL
      for (int q = 0; q < 4; q++) aux[blockIdx.x * 4 + q] = x[q];  // block total
    }
  }
  __syncthreads();
  if (k < nb1) {
    start[k] = sm[0][wid] + inc[0] - v[0];
    sstart0[k] = sm[1][wid] + inc[1] - v[1];
    sstart1[k] = sm[2][wid] + inc[2] - v[2];
    sstart2[k] = sm[3][wid] + inc[3] - v[3];
  }
}
static CS_GLOBAL void k_msm_scan2(const uint32_t* __restrict__ count, uint32_t nb1, uint32_t S,
                                  uint32_t* __restrict__ start, uint32_t* __restrict__ sstart0,
                                  uint32_t* __restrict__ sstart1, uint32_t* __restrict__ sstart2,
                                  const uint32_t* __restrict__ aux) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nb1) return;
  uint32_t off[4] = {0, 0, 0, 0};
  for (uint32_t b = 0; b < blockIdx.x; b++) {
    CS_UNROLL
    for (int q = 0; q < 4; q++) off[q] += aux[b * 4 + q];
  }
  uint32_t a = start[k] + off[0], b0 = sstart0[k] + off[1], b1 = sstart1[k] + off[2], b2 = sstart2[k] + off[3];
  start[k] = a; sstart0[k] = b0; sstart1[k] = b1; sstart2[k] = b2;
  if (k == nb1 - 1) {
    uint32_t v[4];
    msm_scan_terms(count, k, nb1, S, v);
    start[nb1] = a + v[0]; sstart0[nb1] = b0 + v[1]; sstart1[nb1] = b1 + v[2]; sstart2[nb1] = b2 + v[3];
  }
}

// --------------------------------------------------------------------------- scatter
// grid.y = window.  sorted[pos] = table index | sign, grouped by bucket.
static CS_GLOBAL void k_msm_scatter(const uint32_t* __restrict__ dig, uint32_t n, uint32_t nbases,
                             uint32_t offset, const uint32_t* __restrict__ start,
                             uint32_t* __restrict__ cursor, uint32_t* __restrict__ sorted) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t w = blockIdx.y;
  if (i >= n) return;
  uint32_t d = dig[(size_t)w * n + i];
  uint32_t b = d & ~MSM_SIGN;
  if (!b) return;
  uint32_t pos = start[b] + atomicAdd(&cursor[b], 1u);
  sorted[pos] = (w * nbases + offset + i) | (d & MSM_SIGN);
}

// largest b in [0, nb1) with arr[b] <= s   (arr non-decreasing, arr[0] = 0)
CS_D uint32_t find_bucket(const uint32_t* __restrict__ arr, uint32_t nb1, uint32_t s) {
  uint32_t lo = 0, hi = nb1;  // invariant arr[lo] <= s < arr[hi]  (arr[nb1] = total > s)
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (arr[mid] <= s) lo = mid; else hi = mid;
  }
  return lo;
}

// --------------------------------------------------------------------------- slice order (by length)
// Slices of one warp should have the same length, otherwise every lane waits for the longest one
// (bucket loads are Poisson: with 2^19 buckets and ~26 entries each the warp maximum is ~1.4x the
// mean).  A counting sort of the slices by length, longest first: per-block shared-memory histograms
// (k_msm_slice_hist), one thread per length scanning the block columns (k_msm_slice_offsets), then a
// scatter with block-local ranks (k_msm_slice_order).  order[] = slice id, order_b[] = its bucket.
static CS_GLOBAL void k_msm_slice_hist(const uint32_t* __restrict__ count, const uint32_t* __restrict__ sstart0,
                                       uint32_t nb1, uint32_t S, uint32_t* __restrict__ slice_len,
                                       uint32_t* __restrict__ slice_bkt, uint32_t* __restrict__ block_hist) {
  __shared__ uint32_t h[MSM_SLICE_MAX + 1];
  for (uint32_t k = threadIdx.x; k <= MSM_SLICE_MAX; k += blockDim.x) h[k] = 0;
  __syncthreads();
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < sstart0[nb1]) {
    uint32_t lo = 0, hi = nb1;  // largest b with sstart0[b] <= s
    while (hi - lo > 1) {
      uint32_t mid = (lo + hi) >> 1;
      if (sstart0[mid] <= s) lo = mid; else hi = mid;
    }
    uint32_t j = s - sstart0[lo];
    uint32_t len = count[lo] - j * S;
    if (len > S) len = S;
    slice_len[s] = len;
    slice_bkt[s] = lo;
    atomicAdd(&h[len], 1u);
  }
  __syncthreads();
  for (uint32_t k = threadIdx.x; k <= MSM_SLICE_MAX; k += blockDim.x)
    block_hist[(size_t)blockIdx.x * (MSM_SLICE_MAX + 1) + k] = h[k];
}

// Column L of block_hist (one column per slice length) -> exclusive offsets over the histogram blocks, in
// three barrier-free steps: chunk sums (thread = (L, chunk)), a short serial scan per length, chunk write-back.
constexpr unsigned MSM_OFF_CHUNKS = 64;
static CS_GLOBAL void k_msm_slice_off1(const uint32_t* __restrict__ block_hist, uint32_t nblocks,
                                       uint32_t* __restrict__ chunk_sum) {
  uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (MSM_SLICE_MAX + 1) * MSM_OFF_CHUNKS) return;
  uint32_t L = id / MSM_OFF_CHUNKS, ch = id % MSM_OFF_CHUNKS;
  uint32_t per = (nblocks + MSM_OFF_CHUNKS - 1) / MSM_OFF_CHUNKS;
  uint32_t lo = ch * per, hi = lo + per < nblocks ? lo + per : nblocks;
  uint32_t sum = 0;
  for (uint32_t b = lo; b < hi; b++) sum += block_hist[(size_t)b * (MSM_SLICE_MAX + 1) + L];
  chunk_sum[id] = sum;
}
// one thread: per-length chunk prefixes and len_base[L] = start of the length-L region of `order` (longest first)
static CS_GLOBAL void k_msm_slice_off2(uint32_t* __restrict__ chunk_sum, uint32_t* __restrict__ len_base) {
  uint32_t L = blockIdx.x * blockDim.x + threadIdx.x;
  if (L > MSM_SLICE_MAX) return;
  uint32_t run = 0;
  for (uint32_t c = 0; c < MSM_OFF_CHUNKS; c++) {
    uint32_t v = chunk_sum[L * MSM_OFF_CHUNKS + c];
    chunk_sum[L * MSM_OFF_CHUNKS + c] = run;
    run += v;
  }
  len_base[MSM_SLICE_MAX + 1 + L] = run;  // column totals, consumed by k_msm_slice_off3's thread 0
}
static CS_GLOBAL void k_msm_slice_off3(uint32_t* __restrict__ block_hist, uint32_t nblocks,
                                       const uint32_t* __restrict__ chunk_sum, uint32_t* __restrict__ len_base) {
  uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id == 0) {
    uint32_t run = 0;
    for (int k = MSM_SLICE_MAX; k >= 0; k--) { len_base[k] = run; run += len_base[MSM_SLICE_MAX + 1 + k]; }
  }
  if (id >= (MSM_SLICE_MAX + 1) * MSM_OFF_CHUNKS) return;
  uint32_t L = id / MSM_OFF_CHUNKS, ch = id % MSM_OFF_CHUNKS;
  uint32_t per = (nblocks + MSM_OFF_CHUNKS - 1) / MSM_OFF_CHUNKS;
  uint32_t lo = ch * per, hi = lo + per < nblocks ? lo + per : nblocks;
  uint32_t run = chunk_sum[id];
  for (uint32_t b = lo; b < hi; b++) {
    uint32_t v = block_hist[(size_t)b * (MSM_SLICE_MAX + 1) + L];
    block_hist[(size_t)b * (MSM_SLICE_MAX + 1) + L] = run;
    run += v;
  }
}

static CS_GLOBAL void k_msm_slice_order(const uint32_t* __restrict__ slice_len, const uint32_t* __restrict__ slice_bkt,
                                        uint32_t nslices_max, const uint32_t* __restrict__ sstart0, uint32_t nb1,
                                        const uint32_t* __restrict__ block_off, const uint32_t* __restrict__ len_base,
                                        uint32_t* __restrict__ order, uint32_t* __restrict__ order_b) {
  __shared__ uint32_t h[MSM_SLICE_MAX + 1];
  for (uint32_t k = threadIdx.x; k <= MSM_SLICE_MAX; k += blockDim.x) h[k] = 0;
  __syncthreads();
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < sstart0[nb1]) {
    uint32_t len = slice_len[s];
    uint32_t rank = atomicAdd(&h[len], 1u);
    uint32_t pos = len_base[len] + block_off[(size_t)blockIdx.x * (MSM_SLICE_MAX + 1) + len] + rank;
    order[pos] = s;
    order_b[pos] = slice_bkt[s];
  }
}

// --------------------------------------------------------------------------- accumulation level 0
// One thread per slice of <= S sorted entries of ONE bucket: mixed additions from the table.  Threads take
// slices in length order (order[]), so the lanes of a warp run the same number of additions.
template <class F, int MINB>
CS_GLOBAL void __launch_bounds__(128, MINB) k_msm_accum0(const Affine<F>* __restrict__ table,
                                                         const uint32_t* __restrict__ sorted,
                                                         const uint32_t* __restrict__ count,
                                                         const uint32_t* __restrict__ start,
                                                         const uint32_t* __restrict__ sstart0, uint32_t nb1, uint32_t S,
                                                         const uint32_t* __restrict__ order,
                                                         const uint32_t* __restrict__ order_b,
                                                         Xyzz<F>* __restrict__ part0) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= sstart0[nb1]) return;
  uint32_t s = order[t];
  uint32_t b = order_b[t];
  uint32_t j = s - sstart0[b];
  uint32_t beg = start[b] + j * S;
  uint32_t end = start[b] + count[b];
  if (end > beg + S) end = beg + S;
  Xyzz<F> acc = Xyzz<F>::inf();
  uint32_t e = sorted[beg];
  Affine<F> p = table[e & ~MSM_SIGN];
  for (uint32_t k = beg; k < end; k++) {
    uint32_t e_cur = e;
    Affine<F> p_cur = p;
    if (k + 1 < end) {  // prefetch the next point while this addition runs
      e = sorted[k + 1];
      p = table[e & ~MSM_SIGN];
    }
    madd(acc, p_cur, (e_cur & MSM_SIGN) != 0);
  }
  part0[s] = acc;
}

// --------------------------------------------------------------------------- accumulation level 1
template <class F>
CS_GLOBAL void __launch_bounds__(128) k_msm_accum1(const Xyzz<F>* __restrict__ part0,
                                                   const uint32_t* __restrict__ sstart0,
                                                   const uint32_t* __restrict__ sstart1, uint32_t nb1, uint32_t S,
                                                   Xyzz<F>* __restrict__ part1) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= sstart1[nb1]) return;
  uint32_t b = find_bucket(sstart1, nb1, s);
  uint32_t j = s - sstart1[b];
  uint32_t beg = sstart0[b] + j * S;
  uint32_t end = sstart0[b + 1];
  if (end > beg + S) end = beg + S;
  Xyzz<F> acc = part0[beg];
  for (uint32_t k = beg + 1; k < end; k++) padd(acc, part0[k]);
  part1[s] = acc;
}

// --------------------------------------------------------------------------- accumulation level 2
// One thread per bucket: fold the (normally single) level-1 partial(s) into the bucket sum.
template <class F>
CS_GLOBAL void __launch_bounds__(128) k_msm_accum2(const Xyzz<F>* __restrict__ part1,
                                                   const uint32_t* __restrict__ sstart1, uint32_t nb1,
                                                   Xyzz<F>* __restrict__ bucket) {
  uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb1) return;
  uint32_t beg = sstart1[b], end = sstart1[b + 1];
  Xyzz<F> acc = Xyzz<F>::inf();
  if (beg < end) {
    acc = part1[beg];
    for (uint32_t k = beg + 1; k < end; k++) padd(acc, part1[k]);
  }
  bucket[b] = acc;
}

// --------------------------------------------------------------------------- bucket reduction
// Thread t owns buckets (t L, (t+1) L]:  out[t] = sum_{b} b * S_b  over its segment
//   = tot + (t L) * acc,   acc = sum S_b,  tot = sum (b - t L) S_b  by a running sum.
template <class F>
CS_GLOBAL void __launch_bounds__(128) k_msm_reduce_seg(const Xyzz<F>* __restrict__ bucket, uint32_t B,
                                                       uint32_t L, Xyzz<F>* __restrict__ red) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t lo = t * L;
  if (lo >= B) return;
  uint32_t hi = lo + L < B ? lo + L : B;
  Xyzz<F> acc = Xyzz<F>::inf(), tot = Xyzz<F>::inf();
  for (uint32_t b = hi; b > lo; b--) {
    padd(acc, bucket[b]);
    padd(tot, acc);
  }
  // tot += lo * acc   (double-and-add, lo < 2^31)
  if (lo != 0 && !acc.is_inf()) {
    Xyzz<F> m = Xyzz<F>::inf();
    int top = 31 - __clz(lo);
    for (int bit = top; bit >= 0; bit--) {
      m = dbl_xyzz(m);
      if ((lo >> bit) & 1) padd(m, acc);
    }
    padd(tot, m);
  }
  red[t] = tot;
}

// No warp-shuffle tree here: every lane would pay the full point addition in every round, and moving a 128/256-byte
// XYZZ point is 32/64 SHFL, so a shuffle tree is slower than the shared-memory tree below.
// Block b sums red[k] for k = b*T + t, stride gridDim.x*T, into out[b] (shared-memory tree); launched
// twice: many blocks, then one block over the block results.
template <class F>
CS_GLOBAL void k_msm_final_sum(const Xyzz<F>* __restrict__ red, uint32_t cnt,
                                                      Xyzz<F>* __restrict__ out) {
  CS_DYN_SMEM(Xyzz<F>, sm);
  const uint32_t T = blockDim.x, t = threadIdx.x;
  Xyzz<F> acc = Xyzz<F>::inf();
  for (uint32_t k = blockIdx.x * T + t; k < cnt; k += gridDim.x * T) padd(acc, red[k]);
  sm[t] = acc;
  __syncthreads();
  for (uint32_t step = T >> 1; step > 0; step >>= 1) {
    if (t < step) {
      Xyzz<F> a = sm[t];
      padd(a, sm[t + step]);
      sm[t] = a;
    }
    __syncthreads();
  }
  if (t == 0) out[blockIdx.x] = sm[0];
}

// --------------------------------------------------------------------------- table precomputation
// table[w * n + i] = 2^(c w) * P_i  (affine), w = 0..W-1.  One thread per base point; runs once per
// proving key (cs_bases_upload), off the per-proof path.  The affine conversions of up to MSM_PRE_CHUNK consecutive
// windows share ONE field inversion (Montgomery's trick on their ZZZ values): 2 inversions of 356 products per base
// at W = 16 instead of 15.
constexpr int MSM_PRE_CHUNK = 8;
template <class F>
CS_GLOBAL void __launch_bounds__(128) k_msm_precompute(Affine<F>* __restrict__ table, uint32_t n,
                                                       uint32_t c, uint32_t W) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<F> p = table[i];
  if (p.is_inf()) {
    for (uint32_t w = 1; w < W; w++) table[(size_t)w * n + i] = Affine<F>::inf();
    return;
  }
  Xyzz<F> cur = Xyzz<F>::from_affine(p);
  uint32_t w = 1;
  while (w < W) {
    Xyzz<F> pts[MSM_PRE_CHUNK];
    F pre[MSM_PRE_CHUNK];
    int cnt = 0;
    bool degenerate = false;
    for (; cnt < MSM_PRE_CHUNK && w + cnt < W; cnt++) {
      for (uint32_t k = 0; k < c; k++) cur = dbl_xyzz(cur);
      pts[cnt] = cur;
      degenerate = degenerate || cur.is_inf();
    }
    Affine<F> last;
    if (degenerate) {  // a multiple hit the point at infinity (not on the curves in use): one inversion per point
      for (int j = 0; j < cnt; j++) {
        last = to_affine(pts[j]);
        table[(size_t)(w + j) * n + i] = last;
      }
    } else {
      pre[0] = pts[0].zzz;
      for (int j = 1; j < cnt; j++) pre[j] = pre[j - 1] * pts[j].zzz;
      F inv = pre[cnt - 1].inverse();  // 1 / (zzz_0 ... zzz_{cnt-1})
      for (int j = cnt - 1; j >= 0; j--) {
        F zi = j ? inv * pre[j - 1] : inv;   // 1 / zzz_j
        inv = inv * pts[j].zzz;              // 1 / (zzz_0 ... zzz_{j-1})
        F zzi = (zi * pts[j].zz).sqr();      // (ZZ / ZZZ)^2 = 1 / ZZ   (ZZ^3 = ZZZ^2)
        Affine<F> a;
        a.x = pts[j].x * zzi;
        a.y = pts[j].y * zi;
        table[(size_t)(w + j) * n + i] = a;
        if (j == cnt - 1) last = a;
      }
    }
    cur = Xyzz<F>::from_affine(last);  // ZZ = ZZZ = 1 again: the next chunk's first doublings stay cheap
    w += cnt;
  }
}

// --------------------------------------------------------------------------- fixed-base batch mul
// out[i] = scalars[i] * base  (affine).  Used to synthesise proving keys / SRS (a trusted setup is n
// fixed-base multiplications); off the per-proof path.
template <class F, class FrP>
CS_GLOBAL void __launch_bounds__(128) k_fixed_base_mul(const Affine<F>* __restrict__ base,
                                                       const uint32_t* __restrict__ scalars, uint32_t n,
                                                       int mont, Affine<F>* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fp<FrP> s;
  const uint4* src = reinterpret_cast<const uint4*>(scalars) + (size_t)i * (FrP::N / 4);
  CS_UNROLL
  for (int k = 0; k < FrP::N / 4; k++) {
    uint4 v = src[k];
    s.l[4 * k] = v.x; s.l[4 * k + 1] = v.y; s.l[4 * k + 2] = v.z; s.l[4 * k + 3] = v.w;
  }
  if (mont) s = s.from_mont();
  uint32_t lim[FrP::N];
  CS_UNROLL
  for (int k = 0; k < FrP::N; k++) lim[k] = s.l[k];
  Affine<F> b = base[0];
  Xyzz<F> acc = Xyzz<F>::inf();
  for (int bit = FrP::N * 32 - 1; bit >= 0; bit--) {
    acc = dbl_xyzz(acc);
    if ((lim[bit >> 5] >> (bit & 31)) & 1) madd(acc, b, false);
  }
  out[i] = to_affine(acc);
}

// --------------------------------------------------------------------------- host driver
struct MsmShape {
  uint32_t c, W, B;  // window bits, windows, buckets (1..B)
};

static inline MsmShape msm_shape(uint32_t scalar_bits, uint32_t c) {
  MsmShape s;
  s.c = c;
  s.W = (scalar_bits + 1 + c - 1) / c;  // top window keeps <= c-1 bits so the signed recoding never overflows
  s.B = 1u << (c - 1);
  return s;
}

// Window size.  The work is W n mixed additions + ~4 * 2^(c-1) full additions in the bucket reduction
// (running sums + the per-segment scalar multiple).  Wider windows cut the accumulation but the 2^(c-1)-bucket
// phases (sort, fold, reduce) grow with them, so 16 is the cap (window_bits overrides).
// Below 2^15 points the window shrinks with the input (lg n - 4) so that tiny MSMs do not pay for 2^15 buckets.
// A window size whose TOP window is only a few bits wide is avoided: its 2^k digit values send n / 2^k scalars
// each into the same handful of buckets and their fold becomes a serial chain (e.g. 254 + 1 = 18 * 14 + 3).
static inline uint32_t msm_auto_window(size_t n, uint32_t scalar_bits) {
  int lg = 0;
  while ((1ull << (lg + 1)) <= n) lg++;
  int c = lg >= 15 ? 16 : lg - 4;
  if (c < 4) c = 4;
  while (c < 16) {
    const uint32_t W = (scalar_bits + 1 + c - 1) / c;
    const uint32_t top = scalar_bits + 1 - (W - 1) * c;
    if (2 * top >= (uint32_t)c) break;
    c++;
  }
  return (uint32_t)c;
}
static inline uint32_t msm_slice(const MsmShape& sh) {
  const char* e = getenv("CS_MSM_SLICE");  // test hook: exercise the 64-entry path with few buckets
  if (e && atoi(e) == 64) return 64u;
  if (e && atoi(e) == 32) return 32u;
  return sh.c >= 18 ? 64u : 32u;
}

constexpr int MSM_NSTAGE = 5;  // digits | scan+scatter | accum0 | accum1+2 | reduce+final
struct MsmWorkspace {
  DevBuf dig, sorted, meta, part0, part1, part2, bucket, red, scal, result, order;
  void* h_result = nullptr;  // pinned, holds one Xyzz
  size_t h_result_cap = 0;
  bool profile = false;      // record CUDA events at the stage boundaries (bench.py roofline)
  cudaEvent_t ev[MSM_NSTAGE + 1] = {};
  cudaEvent_t sorted_ev = nullptr;  // recorded once the sorted entries / slice order of this MSM are final
  bool sorted_ev_made = false, sorted_once = false;
  cudaEvent_t acc_in = nullptr, acc_out = nullptr;  // hand-off to / from the accumulation stream (msm_enqueue's st_acc)
  int mark(int i, cudaStream_t st) {
    if (!profile) return 0;
    if (!ev[i]) CS_CUDA(cudaEventCreateWithFlags(&ev[i], 0));
    CS_CUDA(cudaEventRecord(ev[i], st));
    return 0;
  }
  void release() {
    for (int i = 0; i <= MSM_NSTAGE; i++) {
      if (ev[i]) cudaEventDestroy(ev[i]);
      ev[i] = nullptr;
    }
    if (sorted_ev_made) cudaEventDestroy(sorted_ev);
    if (acc_in) cudaEventDestroy(acc_in);
    if (acc_out) cudaEventDestroy(acc_out);
    acc_in = acc_out = nullptr;
    sorted_ev = nullptr;
    sorted_ev_made = sorted_once = false;
    dig.release(); sorted.release(); meta.release(); part0.release(); part1.release(); part2.release();
    bucket.release(); red.release(); scal.release(); result.release(); order.release();
    if (h_result) cudaFreeHost(h_result);
    h_result = nullptr;
    h_result_cap = 0;
  }
};

// FP64-pipe accumulation (cs_msm52.cuh); defined for the fields that have 52-bit-limb constants
template <class F>
int msm_accum0_f52(const Affine<F>* table, const uint32_t* sorted, const uint32_t* count, const uint32_t* start,
                   const uint32_t* sstart0, uint32_t nb1, uint32_t S, const uint32_t* order, const uint32_t* order_b,
                   Xyzz<F>* part0, uint32_t max_s0, cudaStream_t st);

// Enqueue one MSM on `st`.  d_scalars: device, n elements of Fr (8 x u32).  The XYZZ result lands in
// ws.h_result (pinned) after the stream drains.
// sort_from (optional): another workspace whose MSM was enqueued over the SAME scalars with the same table
// geometry (nbases, offset, n, window) and the same infinity pattern -- Groth16's B1 / B2 pair.  Its sorted
// entries and slice order are reused (they index table slots, not points), so this MSM starts at the
// accumulation; `st` waits for that workspace's sort to finish.
// st_acc (optional): a second, LOWER-priority stream for the accumulation kernel alone.  When several MSMs share the
// GPU, the block scheduler serves equal-priority grids in launch order, so the short sort / fold / reduce kernels of
// one MSM queue behind the full-GPU accumulation grids of all the others (measured: folds of an MSM finished at 3 ms
// ran long after their own accumulation); with the accumulation on a lower-priority stream they slip in between.
template <class F, class FrP>
int msm_enqueue(MsmWorkspace& ws, const Affine<F>* table, const uint32_t* infmask, uint32_t nbases, MsmShape sh,
                uint32_t offset,
                const uint32_t* d_scalars, uint32_t sstride, uint32_t n, int mont, cudaStream_t st,
                MsmWorkspace* sort_from = nullptr, bool table_m260 = false, cudaStream_t st_acc = nullptr) {
  const uint32_t nb1 = sh.B + 1;
  const size_t nent = (size_t)sh.W * n;
  if (nent >= (1ull << 31) || (size_t)sh.W * nbases >= (1ull << 31))
    return fail(-3, "msm: W*n = %zu exceeds 2^31 entries", nent);
  const uint32_t S = msm_slice(sh);
  const size_t max_s0 = nent / S + nb1;
  const size_t max_s1 = max_s0 / S + nb1;
  const size_t max_s2 = max_s1 / S + nb1;
  MsmWorkspace& so = sort_from ? *sort_from : ws;  // owner of the sort buffers
  // meta: count[nb1] cursor[nb1] | start[nb1+1] sstart0[nb1+1] sstart1[nb1+1] sstart2[nb1+1] | aux[4 * scan blocks]
  const size_t meta_words = 2 * (size_t)nb1 + 4 * ((size_t)nb1 + 1) + 4 * MSM_SCAN_MAX_BLOCKS;  // + the scan's block totals
  if (!sort_from) {
    CS_TRY(ws.dig.reserve(nent * 4));
    CS_TRY(ws.sorted.reserve(nent * 4));
    CS_TRY(ws.meta.reserve(meta_words * 4));
  }
  CS_TRY(ws.part0.reserve(max_s0 * sizeof(Xyzz<F>)));
  CS_TRY(ws.part1.reserve(max_s1 * sizeof(Xyzz<F>)));
  CS_TRY(ws.part2.reserve(max_s2 * sizeof(Xyzz<F>)));
  CS_TRY(ws.bucket.reserve((size_t)nb1 * sizeof(Xyzz<F>)));
  const uint32_t L = sh.B < MSM_RED_SEG ? sh.B : MSM_RED_SEG;
  const uint32_t nseg = (sh.B + L - 1) / L;
  const uint32_t fs_threads = sizeof(Xyzz<F>) > 128 ? 128 : 256;  // <= 32 KB of dynamic shared memory
  const uint32_t fs_blocks = nseg > 4 * fs_threads ? (nseg + fs_threads - 1) / fs_threads : 1;
  CS_TRY(ws.red.reserve(((size_t)nseg + fs_blocks) * sizeof(Xyzz<F>)));
  CS_TRY(ws.result.reserve(sizeof(Xyzz<F>)));
  // slice order: slice_len | slice_bkt | order | order_b (max_s0 each) | block_hist | len_base
  const uint32_t ob = ceil_div(max_s0, MSM_ORDER_BLOCK);
  const size_t order_words = 4 * max_s0 + (size_t)ob * (MSM_SLICE_MAX + 1) + 2 * (MSM_SLICE_MAX + 1) +
                             (size_t)(MSM_SLICE_MAX + 1) * MSM_OFF_CHUNKS;
  if (!sort_from) CS_TRY(ws.order.reserve(order_words * 4));
  if (ws.h_result_cap < sizeof(Xyzz<F>)) {
    if (ws.h_result) cudaFreeHost(ws.h_result);
    CS_CUDA(cudaMallocHost(&ws.h_result, sizeof(Xyzz<F>)));
    ws.h_result_cap = sizeof(Xyzz<F>);
  }
  uint32_t* slice_len = so.order.as<uint32_t>();
  uint32_t* slice_bkt = slice_len + max_s0;
  uint32_t* order = slice_bkt + max_s0;
  uint32_t* order_b = order + max_s0;
  uint32_t* block_hist = order_b + max_s0;
  uint32_t* len_base = block_hist + (size_t)ob * (MSM_SLICE_MAX + 1);
  uint32_t* chunk_sum = len_base + 2 * (MSM_SLICE_MAX + 1);
  uint32_t* count = so.meta.as<uint32_t>();
  uint32_t* cursor = count + nb1;
  uint32_t* start = cursor + nb1;
  uint32_t* sstart0 = start + nb1 + 1;
  uint32_t* sstart1 = sstart0 + nb1 + 1;
  uint32_t* sstart2 = sstart1 + nb1 + 1;
  if (sort_from) {
    if (!sort_from->sorted_once) return fail(-1, "msm: the workspace to share a sort with has not been enqueued");
    CS_TRY(ws.mark(0, st));
    CS_CUDA(cudaStreamWaitEvent(st, sort_from->sorted_ev, 0));
    CS_TRY(ws.mark(1, st));
  } else {
    CS_TRY(ws.mark(0, st));
    CS_CUDA(cudaMemsetAsync(count, 0, 2 * (size_t)nb1 * 4, st));
    CS_LAUNCH(k_msm_digits<FrP>, ceil_div(n, 256), 256, 0, st, d_scalars, sstride, n, mont, sh.c, sh.W, infmask, offset,
              ws.dig.as<uint32_t>(), count);
    CS_TRY(ws.mark(1, st));
    {
      const uint32_t sb = ceil_div(nb1, MSM_SCAN_T);
      if (sb > MSM_SCAN_MAX_BLOCKS) return fail(-3, "msm: %u buckets exceed the scan's limit", sh.B);
      uint32_t* aux = sstart2 + nb1 + 1;
      CS_LAUNCH_SYNC(k_msm_scan1, sb, MSM_SCAN_T, 0, st, count, nb1, S, start, sstart0, sstart1, sstart2, aux);
      CS_LAUNCH(k_msm_scan2, sb, MSM_SCAN_T, 0, st, count, nb1, S, start, sstart0, sstart1, sstart2, aux);
    }
    CS_LAUNCH(k_msm_scatter, dim3(ceil_div(n, 256), sh.W), 256, 0, st, ws.dig.as<uint32_t>(), n, nbases,
              offset, start, cursor, ws.sorted.as<uint32_t>());
    CS_LAUNCH_SYNC(k_msm_slice_hist, ob, MSM_ORDER_BLOCK, 0, st, count, sstart0, nb1, S, slice_len, slice_bkt, block_hist);
    {
      const uint32_t nt = (MSM_SLICE_MAX + 1) * MSM_OFF_CHUNKS;
      CS_LAUNCH(k_msm_slice_off1, ceil_div(nt, 128), 128, 0, st, block_hist, ob, chunk_sum);
      CS_LAUNCH(k_msm_slice_off2, 1, 128, 0, st, chunk_sum, len_base);
      CS_LAUNCH(k_msm_slice_off3, ceil_div(nt, 128), 128, 0, st, block_hist, ob, chunk_sum, len_base);
    }
    CS_LAUNCH_SYNC(k_msm_slice_order, ob, MSM_ORDER_BLOCK, 0, st, slice_len, slice_bkt, (uint32_t)max_s0, sstart0, nb1,
                   block_hist, len_base, order, order_b);
    if (!ws.sorted_ev_made) {
      CS_CUDA(cudaEventCreateWithFlags(&ws.sorted_ev, cudaEventDisableTiming));
      ws.sorted_ev_made = true;
    }
    CS_CUDA(cudaEventRecord(ws.sorted_ev, st));
    ws.sorted_once = true;
  }
  CS_TRY(ws.mark(2, st));
  cudaStream_t st_main = st;
  if (st_acc) {
    if (!ws.acc_in) {
      CS_CUDA(cudaEventCreateWithFlags(&ws.acc_in, cudaEventDisableTiming));
      CS_CUDA(cudaEventCreateWithFlags(&ws.acc_out, cudaEventDisableTiming));
    }
    CS_CUDA(cudaEventRecord(ws.acc_in, st));
    CS_CUDA(cudaStreamWaitEvent(st_acc, ws.acc_in, 0));
    st = st_acc;
  }
  {
    // resident blocks per SM (register cap), overridable for experiments
    static int minb_env = -1;
    if (minb_env < 0) { const char* e = getenv("CS_ACCUM0_MINB"); minb_env = e ? atoi(e) : 0; }
    const int minb = minb_env ? minb_env : 4;
    if (table_m260) {
      CS_TRY((msm_accum0_f52<F>(table, so.sorted.as<uint32_t>(), count, start, sstart0, nb1, S, order, order_b,
                                ws.part0.as<Xyzz<F>>(), (uint32_t)max_s0, st)));
    } else {
#define CS_ACC0(M)                                                                                              \
  CS_LAUNCH(k_msm_accum0<F COMMA M>, ceil_div(max_s0, 128), 128, 0, st, table, so.sorted.as<uint32_t>(), count, \
            start, sstart0, nb1, S, order, order_b, ws.part0.as<Xyzz<F>>())
    switch (minb) {
      case 2: CS_ACC0(2); break;
      case 3: CS_ACC0(3); break;
      case 5: CS_ACC0(5); break;
      case 6: CS_ACC0(6); break;
      default: CS_ACC0(4); break;
    }
#undef CS_ACC0
    }
  }
  if (st_acc) {
    CS_CUDA(cudaEventRecord(ws.acc_out, st_acc));
    st = st_main;
    CS_CUDA(cudaStreamWaitEvent(st, ws.acc_out, 0));
  }
  CS_TRY(ws.mark(3, st));
  CS_LAUNCH(k_msm_accum1<F>, ceil_div(max_s1, 128), 128, 0, st, ws.part0.as<Xyzz<F>>(), sstart0, sstart1,
            nb1, S, ws.part1.as<Xyzz<F>>());
  CS_LAUNCH(k_msm_accum1<F>, ceil_div(max_s2, 128), 128, 0, st, ws.part1.as<Xyzz<F>>(), sstart1, sstart2,
            nb1, S, ws.part2.as<Xyzz<F>>());
  CS_LAUNCH(k_msm_accum2<F>, ceil_div(nb1, 128), 128, 0, st, ws.part2.as<Xyzz<F>>(), sstart2, nb1,
            ws.bucket.as<Xyzz<F>>());
  CS_TRY(ws.mark(4, st));
  CS_LAUNCH(k_msm_reduce_seg<F>, ceil_div(nseg, 128), 128, 0, st, ws.bucket.as<Xyzz<F>>(), sh.B, L,
            ws.red.as<Xyzz<F>>());
  if (fs_blocks > 1) {
    Xyzz<F>* stage = ws.red.as<Xyzz<F>>() + nseg;
    CS_LAUNCH_SYNC(k_msm_final_sum<F>, fs_blocks, fs_threads, fs_threads * sizeof(Xyzz<F>), st, ws.red.as<Xyzz<F>>(), nseg,
                   stage);
    CS_LAUNCH_SYNC(k_msm_final_sum<F>, 1, fs_threads, fs_threads * sizeof(Xyzz<F>), st, stage, fs_blocks,
                   ws.result.as<Xyzz<F>>());
  } else {
    CS_LAUNCH_SYNC(k_msm_final_sum<F>, 1, fs_threads, fs_threads * sizeof(Xyzz<F>), st, ws.red.as<Xyzz<F>>(), nseg,
                   ws.result.as<Xyzz<F>>());
  }
  CS_TRY(ws.mark(5, st));
  CS_CUDA(cudaMemcpyAsync(ws.h_result, ws.result.p, sizeof(Xyzz<F>), cudaMemcpyDeviceToHost, st));
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
