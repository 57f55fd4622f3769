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
//    doubling chain on the per-proof path.  A key whose full tables do not fit keeps one row per k windows and k
//    bucket groups, combined by c (k - 1) doublings (MsmShape).
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

// --------------------------------------------------------------------------- digits
// Scalar i: optional Montgomery -> canonical, then signed c-bit recoding; f(row, digit) for every window w, where the
// digit is bucket | MSM_SIGN and bucket 0 is a zero digit.  A table of one row per k windows (MsmShape) puts window w
// in row w / k and its digits d in bucket group w % k: bucket (w % k) B + d.  k = 1: row w, bucket d.
template <class FrP, class Fn>
CS_D void msm_recode(const uint32_t* __restrict__ scalars, uint32_t sstride, uint32_t i, int mont, uint32_t c,
                     uint32_t W, uint32_t k, Fn&& f) {
  Fp<FrP> s;
  // sstride = elements between consecutive scalars (2 reads the `a` component of Rep3 shares in place)
  const uint4* src = reinterpret_cast<const uint4*>(scalars) + (size_t)i * sstride * (FrP::N / 4);
  CS_UNROLL
  for (int q = 0; q < FrP::N / 4; q++) {
    uint4 v = src[q];
    s.l[4 * q] = v.x; s.l[4 * q + 1] = v.y; s.l[4 * q + 2] = v.z; s.l[4 * q + 3] = v.w;
  }
  if (mont) s = s.from_mont();
  const uint32_t half = 1u << (c - 1);
  const uint32_t mask = (1u << c) - 1;
  uint32_t carry = 0, row = 0, gb = 0;  // gb = first bucket of the group - 1
  for (uint32_t w = 0; w < W; w++) {
    uint32_t pos = w * c;
    uint32_t li = pos >> 5, sh = pos & 31;
    uint32_t lo = li < FrP::N ? s.l[li] : 0;
    uint32_t hi = li + 1 < FrP::N ? s.l[li + 1] : 0;
    uint32_t d = (__funnelshift_r(lo, hi, sh) & mask) + carry;
    uint32_t out;
    if (d > half) {
      out = ((1u << c) - d) | MSM_SIGN;  // d = 2^c: a zero digit with a carry
      carry = 1;
    } else {
      out = d;
      carry = 0;
    }
    f(row, out & ~MSM_SIGN ? out + gb : 0);
    gb += half;
    if (gb == k * half) {
      gb = 0;
      row++;
    }
  }
}

// bases at infinity (sparse Groth16 B-queries: B_i(tau) = 0 for variables absent from B) contribute nothing: their
// entries are dropped before the sort instead of being carried through the accumulation.  infmask = null keeps every
// entry (the witness sort that several base sets share, filtered per table by k_msm_view_*).
CS_D bool msm_base_inf(const uint32_t* __restrict__ infmask, uint32_t k) {
  return infmask && ((infmask[k >> 5] >> (k & 31)) & 1);
}

// --------------------------------------------------------------------------- bucket sort
// A counting sort of the W n entries by bucket in three passes, with no global atomics:
//  * k_msm_bin_count: block x takes scalars [x tile, (x + 1) tile), recodes them and counts its entries per bucket in a
//    shared-memory histogram; the histogram becomes row x of tab (nblk rows of B words, column b - 1 = bucket b).
//  * k_msm_bin_scan: per bucket, the rows become exclusive prefixes (block x's first slot inside the bucket) and the
//    column total becomes count[b].
//  * k_msm_bin_scatter: the block recodes its tile again and places every entry at start[b] + its row's prefix + a
//    rank from a shared-memory cursor.
// A histogram covers MSM_BIN_SPAN buckets (128 KB); wider windows split the buckets over grid.y, and each block
// re-reads its tile for its share of the buckets.
// K scalar vectors over one base set (a batch of K proofs; proof p's scalars start pstride elements after proof
// p - 1's) sort as one: bucket (p k + g) B + d.  Each tile belongs to one proof (blocks [p nblk_p, (p + 1) nblk_p)), so
// its table row covers only that proof's k B buckets, and the table is K times one MSM's.
// The scatter takes MSM_SCATTER_SPAN buckets per grid.y slice even at c = 16: its scattered 4-byte stores, not the
// recoding, bound it, and with a quarter of the buckets at a time the output lines being written stay fewer (measured at 2^20 scalars on the H100: 412 us in four slices against 509 us
// in one, although each slice recodes the tile again).
constexpr unsigned MSM_BIN_T = 1024;             // threads per block of k_msm_bin_count / k_msm_bin_scatter
constexpr unsigned MSM_BIN_TILE = 4096;          // scalars per block, unless the count table would outgrow W n words
constexpr unsigned MSM_BIN_SPAN = 1u << 15;      // buckets per shared-memory histogram: all of them up to c = 16
constexpr unsigned MSM_SCATTER_SPAN = 1u << 13;  // buckets per grid.y slice of k_msm_bin_scatter

template <class FrP>
CS_GLOBAL void __launch_bounds__(MSM_BIN_T) k_msm_bin_count(const uint32_t* __restrict__ scalars, uint32_t sstride,
                                                            uint32_t n, int mont, uint32_t c, uint32_t W, uint32_t kw,
                                                            const uint32_t* __restrict__ infmask, uint32_t offset,
                                                            uint32_t tile, uint32_t nblk_p, uint32_t pstride, uint32_t B,
                                                            uint32_t* __restrict__ tab) {
  CS_DYN_SMEM(uint32_t, h);
  const uint32_t bt = blockIdx.x % nblk_p;  // tile within proof blockIdx.x / nblk_p
  scalars += (size_t)(blockIdx.x / nblk_p) * pstride * FrP::N;
  const uint32_t lo = blockIdx.y * MSM_BIN_SPAN + 1;  // buckets [lo, lo + span)
  const uint32_t span = B + 1 - lo < MSM_BIN_SPAN ? B + 1 - lo : MSM_BIN_SPAN;
  for (uint32_t k = threadIdx.x; k < span; k += blockDim.x) h[k] = 0;
  __syncthreads();
  const uint32_t i1 = (bt + 1) * tile < n ? (bt + 1) * tile : n;
  for (uint32_t i = bt * tile + threadIdx.x; i < i1; i += blockDim.x) {
    if (msm_base_inf(infmask, offset + i)) continue;
    msm_recode<FrP>(scalars, sstride, i, mont, c, W, kw, [&](uint32_t, uint32_t d) {
      const uint32_t k = (d & ~MSM_SIGN) - lo;  // wraps past span for bucket 0 and for buckets below lo
      if (k < span) atomicAdd(&h[k], 1u);
    });
  }
  __syncthreads();
  uint32_t* row = tab + (size_t)blockIdx.x * B + (lo - 1);
  for (uint32_t k = threadIdx.x; k < span; k += blockDim.x) row[k] = h[k];
}

// One thread per bucket, down the nblk rows of its proof's table (B buckets per proof, NB in all); count[0] = 0 (zero
// digits are dropped).
constexpr unsigned MSM_BIN_SCAN_U = 16;  // rows loaded before any is rewritten: loads in flight per thread
static CS_GLOBAL void k_msm_bin_scan(uint32_t* __restrict__ tab, uint32_t nblk, uint32_t B, uint32_t NB,
                                     uint32_t* __restrict__ count) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b == 0) count[0] = 0;
  if (b >= NB) return;
  uint32_t* col = tab + (size_t)(b / B) * nblk * B + b % B;
  uint32_t run = 0, r = 0;
  for (; r + MSM_BIN_SCAN_U <= nblk; r += MSM_BIN_SCAN_U) {
    uint32_t v[MSM_BIN_SCAN_U];
    CS_UNROLL
    for (uint32_t u = 0; u < MSM_BIN_SCAN_U; u++) v[u] = col[(size_t)(r + u) * B];
    CS_UNROLL
    for (uint32_t u = 0; u < MSM_BIN_SCAN_U; u++) {
      col[(size_t)(r + u) * B] = run;
      run += v[u];
    }
  }
  for (; r < nblk; r++) {
    const uint32_t v = col[(size_t)r * B];
    col[(size_t)r * B] = run;
    run += v;
  }
  count[b + 1] = run;
}

// sorted[pos] = table slot row * nbases + offset + i | sign, grouped by bucket
template <class FrP>
CS_GLOBAL void __launch_bounds__(MSM_BIN_T) k_msm_bin_scatter(const uint32_t* __restrict__ scalars, uint32_t sstride,
                                                              uint32_t n, int mont, uint32_t c, uint32_t W, uint32_t kw,
                                                              const uint32_t* __restrict__ infmask, uint32_t offset,
                                                              uint32_t tile, uint32_t nblk_p, uint32_t pstride,
                                                              uint32_t B, uint32_t nbases,
                                                              const uint32_t* __restrict__ tab,
                                                              const uint32_t* __restrict__ start,
                                                              uint32_t* __restrict__ sorted) {
  CS_DYN_SMEM(uint32_t, cur);
  const uint32_t p = blockIdx.x / nblk_p, bt = blockIdx.x % nblk_p;
  scalars += (size_t)p * pstride * FrP::N;
  const uint32_t lo = blockIdx.y * MSM_SCATTER_SPAN + 1;
  const uint32_t span = B + 1 - lo < MSM_SCATTER_SPAN ? B + 1 - lo : MSM_SCATTER_SPAN;
  const uint32_t* row = tab + (size_t)blockIdx.x * B + (lo - 1);
  for (uint32_t k = threadIdx.x; k < span; k += blockDim.x) cur[k] = start[p * B + lo + k] + row[k];
  __syncthreads();
  const uint32_t i1 = (bt + 1) * tile < n ? (bt + 1) * tile : n;
  for (uint32_t i = bt * tile + threadIdx.x; i < i1; i += blockDim.x) {
    if (msm_base_inf(infmask, offset + i)) continue;
    msm_recode<FrP>(scalars, sstride, i, mont, c, W, kw, [&](uint32_t row, uint32_t d) {
      const uint32_t k = (d & ~MSM_SIGN) - lo;
      if (k < span) sorted[atomicAdd(&cur[k], 1u)] = (row * nbases + offset + i) | (d & MSM_SIGN);
    });
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

// --------------------------------------------------------------------------- filtered view of a shared sort
// Groth16's A, B1, B2 and L MSMs take the same witness scalars over different tables.  Their digits are sorted ONCE
// without an infinity mask (msm_sort with infmask = null, entries j * n + i: table row j, scalar i); a table with
// infinity bases, or whose slots are not j * n + i, gets a stream compaction of those entries that drops the entries
// of its infinite bases and rewrites the rest to its own slots, j * nbases + offset + i (the tables share one window
// shape: c, W and windows per row k).  The compaction keeps the order, so the view is grouped by bucket as the shared
// entries are, and its bucket counts follow from the kept entries before each shared bucket start: per-block counts
// and keep bitmaps, no per-entry global atomics.
constexpr unsigned MSM_VIEW_T = 256;  // entries per block of the view kernels, one per thread
constexpr unsigned MSM_VIEW_WORDS = MSM_VIEW_T / 32;

CS_D uint32_t popc32(uint32_t x) {
#if defined(CS_EMU)
  return (uint32_t)__builtin_popcount(x);
#else
  return __popc(x);
#endif
}
// bit l = pred of lane l; every lane of the warp calls it
CS_D uint32_t warp_bits(bool pred) {
#if defined(CS_EMU)
  uint32_t x = pred ? 1u << (threadIdx.x & 31) : 0u;  // distinct bits: the butterfly sum is the OR
  for (uint32_t d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(0xffffffffu, x, d);
  return x;
#else
  return __ballot_sync(0xffffffffu, pred);
#endif
}

// keep[] bit p = shared entry p belongs to a finite base of this table; blk_cnt[block] = kept entries of the block
static CS_GLOBAL void k_msm_view_flags(const uint32_t* __restrict__ sorted, const uint32_t* __restrict__ src_start,
                                       uint32_t nb1, uint32_t n, const uint32_t* __restrict__ infmask, uint32_t offset,
                                       uint32_t* __restrict__ keep, uint32_t* __restrict__ blk_cnt) {
  __shared__ uint32_t cnt[MSM_VIEW_WORDS];
  const uint32_t t = threadIdx.x;
  const uint32_t p = blockIdx.x * MSM_VIEW_T + t;
  bool k = false;
  if (p < src_start[nb1]) {  // total shared entries
    const uint32_t i = (sorted[p] & ~MSM_SIGN) % n;
    k = !((infmask[(offset + i) >> 5] >> ((offset + i) & 31)) & 1);
  }
  const uint32_t bits = warp_bits(k);
  if ((t & 31) == 0) {
    keep[(size_t)blockIdx.x * MSM_VIEW_WORDS + (t >> 5)] = bits;
    cnt[t >> 5] = popc32(bits);
  }
  __syncthreads();
  if (t == 0) {
    uint32_t c = 0;
    for (uint32_t w = 0; w < MSM_VIEW_WORDS; w++) c += cnt[w];
    blk_cnt[blockIdx.x] = c;
  }
}

// one block: blk_off = exclusive scan of blk_cnt[0..nblk), blk_off[nblk] = total
static CS_GLOBAL void k_msm_view_scan(const uint32_t* __restrict__ blk_cnt, uint32_t nblk, uint32_t* __restrict__ blk_off) {
  __shared__ uint32_t sm[MSM_SCAN_T];
  const uint32_t t = threadIdx.x, T = blockDim.x;
  const uint32_t per = (nblk + T - 1) / T;
  const uint32_t lo = t * per < nblk ? t * per : nblk, hi = lo + per < nblk ? lo + per : nblk;
  uint32_t s = 0;
  for (uint32_t b = lo; b < hi; b++) s += blk_cnt[b];
  sm[t] = s;
  __syncthreads();
  for (uint32_t d = 1; d < T; d <<= 1) {
    const uint32_t v = t >= d ? sm[t - d] : 0;
    __syncthreads();
    sm[t] += v;
    __syncthreads();
  }
  uint32_t run = sm[t] - s;
  for (uint32_t b = lo; b < hi; b++) {
    const uint32_t c = blk_cnt[b];
    blk_off[b] = run;
    run += c;
  }
  if (t == T - 1) blk_off[nblk] = run;
}

// kept entries among shared positions [0, p)
CS_D uint32_t view_kept_before(uint32_t p, const uint32_t* __restrict__ keep, const uint32_t* __restrict__ blk_off) {
  const uint32_t blk = p / MSM_VIEW_T;
  uint32_t r = blk_off[blk];
  for (uint32_t w = blk * MSM_VIEW_WORDS; w < (p >> 5); w++) r += popc32(keep[w]);
  if (p & 31) r += popc32(keep[p >> 5] & ((1u << (p & 31)) - 1));
  return r;
}

// count[b] of the view: kept entries of shared bucket b
static CS_GLOBAL void k_msm_view_counts(const uint32_t* __restrict__ src_start, uint32_t nb1, const uint32_t* __restrict__ keep,
                                        const uint32_t* __restrict__ blk_off, uint32_t* __restrict__ count) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb1) return;
  count[b] = b ? view_kept_before(src_start[b + 1], keep, blk_off) - view_kept_before(src_start[b], keep, blk_off) : 0;
}

// kept shared entry p -> position blk_off[block] + rank in the block, rewritten to this table's slot
static CS_GLOBAL void k_msm_view_scatter(const uint32_t* __restrict__ sorted, uint32_t n, uint32_t nbases, uint32_t offset,
                                         const uint32_t* __restrict__ keep, const uint32_t* __restrict__ blk_off,
                                         uint32_t* __restrict__ out) {
  const uint32_t t = threadIdx.x;
  const uint32_t* kb = keep + (size_t)blockIdx.x * MSM_VIEW_WORDS;
  const uint32_t word = kb[t >> 5];
  if (!((word >> (t & 31)) & 1)) return;
  uint32_t pos = blk_off[blockIdx.x] + popc32(word & ((1u << (t & 31)) - 1));
  for (uint32_t k = 0; k < (t >> 5); k++) pos += popc32(kb[k]);
  const uint32_t e = sorted[blockIdx.x * MSM_VIEW_T + t];
  const uint32_t v = e & ~MSM_SIGN, w = v / n, i = v - w * n;
  out[pos] = (w * nbases + offset + i) | (e & MSM_SIGN);
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
  if constexpr (sizeof(Affine<F>) > 64) {
    // G2: the 64-register accumulator leaves no room for a register copy of the next 128-byte point, so the next point
    // is only prefetched into L1 (no registers held) and loaded when its addition starts
    for (uint32_t k = beg; k < end; k++) {
      const uint32_t e_cur = e;
      if (k + 1 < end) {
        e = sorted[k + 1];
        prefetch_l1(table + (e & ~MSM_SIGN));
      }
      madd(acc, table[e_cur & ~MSM_SIGN], (e_cur & MSM_SIGN) != 0);
    }
    part0[s] = acc;
    return;
  }
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
// Thread t owns buckets (t L, (t+1) L] of the NB = k B buckets:  out[t] = sum_{b} (b - g B) * S_b  over its segment,
// g = the bucket group (L divides B, so a segment lies in one group)
//   = tot + (t L - g B) * acc,   acc = sum S_b,  tot = sum (b - t L) S_b  by a running sum.
template <class F>
CS_GLOBAL void __launch_bounds__(128) k_msm_reduce_seg(const Xyzz<F>* __restrict__ bucket, uint32_t NB, uint32_t B,
                                                       uint32_t L, Xyzz<F>* __restrict__ red) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t lo = t * L;
  if (lo >= NB) return;
  uint32_t hi = lo + L < NB ? lo + L : NB;
  const uint32_t w = lo & (B - 1);  // t L - g B (B is a power of two)
  Xyzz<F> acc = Xyzz<F>::inf(), tot = Xyzz<F>::inf();
  for (uint32_t b = hi; b > lo; b--) {
    padd(acc, bucket[b]);
    padd(tot, acc);
  }
  // tot += w * acc   (double-and-add, w < 2^31)
  if (w != 0 && !acc.is_inf()) {
    Xyzz<F> m = Xyzz<F>::inf();
    int top = 31 - __clz(w);
    for (int bit = top; bit >= 0; bit--) {
      m = dbl_xyzz(m);
      if ((w >> bit) & 1) padd(m, acc);
    }
    padd(tot, m);
  }
  red[t] = tot;
}

// No warp-shuffle tree here: every lane would pay the full point addition in every round, and moving a 128/256-byte
// XYZZ point is 32/64 SHFL, so a shuffle tree is slower than the shared-memory tree below.
// Block b sums red[k] for k = b*T + t, stride gridDim.x*T, into out[b] (shared-memory tree); launched
// twice: many blocks, then one block over the block results.  grid.y = bucket groups, each over its own cnt inputs.
template <class F>
CS_GLOBAL void k_msm_final_sum(const Xyzz<F>* __restrict__ red, uint32_t cnt,
                                                      Xyzz<F>* __restrict__ out) {
  CS_DYN_SMEM(Xyzz<F>, sm);
  const uint32_t T = blockDim.x, t = threadIdx.x;
  red += (size_t)blockIdx.y * cnt;
  out += (size_t)blockIdx.y * gridDim.x;
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

// One thread: the k group sums R_g of a table with one row per k windows -> sum_g 2^(c g) R_g by Horner's rule
// (c (k - 1) doublings).
template <class F>
CS_GLOBAL void k_msm_combine_groups(const Xyzz<F>* __restrict__ gsum, uint32_t k, uint32_t c, Xyzz<F>* __restrict__ out) {
  Xyzz<F> acc = gsum[k - 1];
  for (uint32_t g = k - 1; g-- > 0;) {
    for (uint32_t d = 0; d < c; d++) acc = dbl_xyzz(acc);
    padd(acc, gsum[g]);
  }
  out[0] = acc;
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

// --------------------------------------------------------------------------- scalar multiplication
// s P by double-and-add over the bits of s (canonical, not Montgomery), one thread.  p may be a register copy or a
// point in memory, which is then read at each addition (fewer registers held: what the G2 point terms need)
template <class F, class FrP>
CS_D Xyzz<F> scalar_mul(const Affine<F>& p, const Fp<FrP>& s) {
  Xyzz<F> acc = Xyzz<F>::inf();
  for (int bit = FrP::N * 32 - 1; bit >= 0; bit--) {
    acc = dbl_xyzz(acc);
    if ((s.l[bit >> 5] >> (bit & 31)) & 1) madd(acc, p, false);
  }
  return acc;
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
  const Affine<F> b = base[0];
  out[i] = to_affine(scalar_mul<F, FrP>(b, s));
}

// --------------------------------------------------------------------------- small point linear combinations
// out[o] = sum_j s_oj P_oj (+ per-output XYZZ addends, + one shared point) for a batch of outputs with a few terms each:
// the single-point work of a batch of proofs (r delta_1, s A, the public-input terms, ...).  Three launches:
//  * k_point_terms: one thread per term, prod[t] = s_t P_t by double-and-add over the bits of the (Montgomery) scalar;
//  * k_point_sum: one thread per output, the sum of its T products, its addends and `shared`;
//  * k_point_affine: Montgomery's trick over runs of POINT_INV_RUN outputs, one field inversion per run.
constexpr uint32_t POINT_INV_RUN = 32;

template <class F, class FrP>
CS_GLOBAL void __launch_bounds__(128) k_point_terms(const Affine<F>* __restrict__ base, const uint32_t* __restrict__ scalars,
                                                    uint32_t nterms, Xyzz<F>* __restrict__ prod) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nterms) return;
  Fp<FrP> s;
  CS_UNROLL
  for (int k = 0; k < FrP::N; k++) s.l[k] = scalars[(size_t)t * FrP::N + k];
  prod[t] = scalar_mul<F, FrP>(base[t], s.from_mont());
}

template <class F>
CS_GLOBAL void __launch_bounds__(128) k_point_sum(const Xyzz<F>* __restrict__ prod, uint32_t T, uint32_t nout,
                                                  const Xyzz<F>* __restrict__ add0, const Xyzz<F>* __restrict__ add1,
                                                  const Affine<F>* __restrict__ shared, Xyzz<F>* __restrict__ out) {
  const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= nout) return;
  Xyzz<F> acc = shared ? Xyzz<F>::from_affine(*shared) : Xyzz<F>::inf();
  for (uint32_t j = 0; j < T + 2; j++) {  // one call site of padd: a G2 addition inlined three times spills more
    const Xyzz<F>* q = j < T ? prod + (size_t)o * T + j : (j == T ? add0 : add1);
    if (q && j >= T) q += o;
    if (q) padd(acc, *q);
  }
  out[o] = acc;
}

// out[o ostride] = affine(in[o]).  The running products of the ZZZ coordinates are kept in the outputs' x until the
// backward pass overwrites them; points at infinity are skipped by the products and come out as (0, 0).
template <class F>
CS_GLOBAL void __launch_bounds__(128) k_point_affine(const Xyzz<F>* __restrict__ in, uint32_t nout, uint32_t ostride,
                                                     Affine<F>* __restrict__ out) {
  const uint32_t lo = (blockIdx.x * blockDim.x + threadIdx.x) * POINT_INV_RUN;
  if (lo >= nout) return;
  const uint32_t hi = lo + POINT_INV_RUN < nout ? lo + POINT_INV_RUN : nout;
  F run = F::one();
  for (uint32_t o = lo; o < hi; o++) {
    if (!in[o].is_inf()) run = run * in[o].zzz;
    out[(size_t)o * ostride].x = run;
  }
  F inv = run.inverse();  // 1 / (product of every finite ZZZ of the run)
  for (uint32_t o = hi; o-- > lo;) {  // the coordinates are loaded where they are used: no point held in registers
    Affine<F> a = Affine<F>::inf();
    if (!in[o].is_inf()) {
      const F zi = o > lo ? inv * out[(size_t)(o - 1) * ostride].x : inv;  // 1 / ZZZ_o
      inv = inv * in[o].zzz;
      const F zzi = (zi * in[o].zz).sqr();  // (ZZ / ZZZ)^2 = 1 / ZZ
      a.x = in[o].x * zzi;
      a.y = in[o].y * zi;
    }
    out[(size_t)o * ostride] = a;
  }
}

// --------------------------------------------------------------------------- host driver
// A table keeps one row per k windows, T = ceil(W / k) rows: row j = 2^(c k j) P_i (k_msm_precompute with window c k).
// Window w reads row w / k and accumulates into bucket group w % k (k B buckets in all); the group sums are combined
// as sum_g 2^(c g) R_g.  k = 1 is the full table: a row per window and one bucket group.
struct MsmShape {
  uint32_t c, W, B;  // window bits, windows, buckets per group (1..B)
  uint32_t k = 1, T = 0;  // windows per table row, table rows
  uint32_t nb() const { return k * B; }  // buckets of all groups (1..k B)
};

static inline MsmShape msm_shape(uint32_t scalar_bits, uint32_t c, uint32_t k = 1) {
  MsmShape s;
  s.c = c;
  s.W = (scalar_bits + 1 + c - 1) / c;  // top window keeps <= c-1 bits so the signed recoding never overflows
  s.B = 1u << (c - 1);
  s.k = k < s.W ? k : s.W;
  s.T = (s.W + s.k - 1) / s.k;
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
  size_t bytes() const {
    return dig.cap + sorted.cap + meta.cap + part0.cap + part1.cap + part2.cap + bucket.cap + red.cap + scal.cap +
           result.cap + order.cap;
  }
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

// Buffer sizes of K MSMs over n scalars each (K W n entries, K k B buckets) and the layout of their sort buffers.
struct MsmSizes {
  uint32_t nb1, S, ob, K;
  size_t nent, max_s0, max_s1, max_s2;
  MsmSizes(const MsmShape& sh, uint32_t n, uint32_t K_ = 1) {
    K = K_;
    nb1 = K * sh.nb() + 1;
    nent = (size_t)K * sh.W * n;
    S = msm_slice(sh);
    max_s0 = nent / S + nb1;
    max_s1 = max_s0 / S + nb1;
    max_s2 = max_s1 / S + nb1;
    ob = ceil_div(max_s0, MSM_ORDER_BLOCK);
  }
  // meta: count[nb1] | start[nb1+1] sstart0[nb1+1] sstart1[nb1+1] sstart2[nb1+1] | aux[4 * scan blocks]
  size_t meta_words() const { return (size_t)nb1 + 4 * ((size_t)nb1 + 1) + 4 * MSM_SCAN_MAX_BLOCKS; }
  // slice order: slice_len | slice_bkt | order | order_b (max_s0 each) | block_hist | len_base | chunk_sum
  size_t order_words() const {
    return 4 * max_s0 + (size_t)ob * (MSM_SLICE_MAX + 1) + 2 * (MSM_SLICE_MAX + 1) + (size_t)(MSM_SLICE_MAX + 1) * MSM_OFF_CHUNKS;
  }
};
struct MsmSortBufs {
  uint32_t *count, *start, *sstart0, *sstart1, *sstart2, *aux;
  uint32_t *slice_len, *slice_bkt, *order, *order_b, *block_hist, *len_base, *chunk_sum;
  MsmSortBufs(const MsmWorkspace& w, const MsmSizes& z) {
    count = w.meta.as<uint32_t>();
    start = count + z.nb1;
    sstart0 = start + z.nb1 + 1;
    sstart1 = sstart0 + z.nb1 + 1;
    sstart2 = sstart1 + z.nb1 + 1;
    aux = sstart2 + z.nb1 + 1;
    slice_len = w.order.as<uint32_t>();
    slice_bkt = slice_len + z.max_s0;
    order = slice_bkt + z.max_s0;
    order_b = order + z.max_s0;
    block_hist = order_b + z.max_s0;
    len_base = block_hist + (size_t)z.ob * (MSM_SLICE_MAX + 1);
    chunk_sum = len_base + 2 * (MSM_SLICE_MAX + 1);
  }
};

// Largest batch of MSMs one sort and accumulation can take in shape sh: K k B + 1 bucket slots for the scan, K W n < 2^31
// entries, K k bucket groups over k_msm_final_sum's grid.y
static inline uint32_t msm_max_batch(const MsmShape& sh, uint32_t n) {
  size_t K = ((size_t)MSM_SCAN_MAX_BLOCKS * MSM_SCAN_T - 1) / sh.nb();
  if (n) K = K < ((1ull << 31) - 1) / ((size_t)sh.W * n) ? K : ((1ull << 31) - 1) / ((size_t)sh.W * n);
  K = K < 65535 / sh.k ? K : 65535 / sh.k;
  return (uint32_t)K;
}

static inline int msm_check_limits(const MsmShape& sh, uint32_t n, uint32_t nbases, uint32_t K = 1) {
  const size_t nent = (size_t)K * sh.W * n;
  if (nent >= (1ull << 31) || (size_t)sh.T * nbases >= (1ull << 31))
    return fail(-3, "msm: K*W*n = %zu entries or T*nbases = %zu table slots exceed 2^31", nent, (size_t)sh.T * nbases);
  if (K > 1 && K > msm_max_batch(sh, n))
    return fail(-3, "msm: a batch of %u MSMs exceeds the %u that one sort takes in this window shape (K*k*B + 1 <= 2^20 "
                    "buckets, K*k <= 65535 groups)", K, msm_max_batch(sh, n));
  return 0;
}

// count[] -> bucket starts and slice offsets (start, sstart0..2)
static inline int msm_scan(const MsmSortBufs& q, const MsmSizes& z, uint32_t NB, cudaStream_t st) {
  const uint32_t sb = ceil_div(z.nb1, MSM_SCAN_T);
  if (sb > MSM_SCAN_MAX_BLOCKS) return fail(-3, "msm: %u buckets exceed the scan's limit", NB);
  CS_LAUNCH_SYNC(k_msm_scan1, sb, MSM_SCAN_T, 0, st, q.count, z.nb1, z.S, q.start, q.sstart0, q.sstart1, q.sstart2, q.aux);
  CS_LAUNCH(k_msm_scan2, sb, MSM_SCAN_T, 0, st, q.count, z.nb1, z.S, q.start, q.sstart0, q.sstart1, q.sstart2, q.aux);
  return 0;
}

// Slice order by length; then ws.sorted_ev marks the sorted entries and the order as final.
static inline int msm_slice_order(MsmWorkspace& ws, const MsmSortBufs& q, const MsmSizes& z, cudaStream_t st) {
  CS_LAUNCH_SYNC(k_msm_slice_hist, z.ob, MSM_ORDER_BLOCK, 0, st, q.count, q.sstart0, z.nb1, z.S, q.slice_len, q.slice_bkt,
                 q.block_hist);
  const uint32_t nt = (MSM_SLICE_MAX + 1) * MSM_OFF_CHUNKS;
  CS_LAUNCH(k_msm_slice_off1, ceil_div(nt, 128), 128, 0, st, q.block_hist, z.ob, q.chunk_sum);
  CS_LAUNCH(k_msm_slice_off2, 1, 128, 0, st, q.chunk_sum, q.len_base);
  CS_LAUNCH(k_msm_slice_off3, ceil_div(nt, 128), 128, 0, st, q.block_hist, z.ob, q.chunk_sum, q.len_base);
  CS_LAUNCH_SYNC(k_msm_slice_order, z.ob, MSM_ORDER_BLOCK, 0, st, q.slice_len, q.slice_bkt, (uint32_t)z.max_s0, q.sstart0,
                 z.nb1, q.block_hist, q.len_base, q.order, q.order_b);
  if (!ws.sorted_ev_made) {
    CS_CUDA(cudaEventCreateWithFlags(&ws.sorted_ev, cudaEventDisableTiming));
    ws.sorted_ev_made = true;
  }
  CS_CUDA(cudaEventRecord(ws.sorted_ev, st));
  ws.sorted_once = true;
  return 0;
}

// The bucket sort's histograms take more than the default 48 KB of shared memory; once per device and scalar field.
template <class FrP>
int msm_smem_optin() {
#if !defined(CS_EMU)
  CS_CUDA(cudaFuncSetAttribute(k_msm_bin_count<FrP>, cudaFuncAttributeMaxDynamicSharedMemorySize, MSM_BIN_SPAN * 4));
  CS_CUDA(cudaFuncSetAttribute(k_msm_bin_scatter<FrP>, cudaFuncAttributeMaxDynamicSharedMemorySize, MSM_SCATTER_SPAN * 4));
#endif
  return 0;
}

// Scalars per block of the bucket sort: MSM_BIN_TILE, or more where nblk rows of B counts would exceed the W n words
// the table has (windows above 16 at small n).  The table then takes at most max(W n, B) words.
static inline uint32_t msm_bin_tile(const MsmShape& sh, const MsmSizes& z, uint32_t n) {
  const size_t ent = z.nent / z.K;  // entries of one MSM of the batch
  const size_t rows = ent / sh.nb() > 1 ? ent / sh.nb() : 1;
  const size_t nblk = ceil_div(n, MSM_BIN_TILE) < rows ? ceil_div(n, MSM_BIN_TILE) : rows;
  return n ? ceil_div(n, nblk) : 1;
}

// Words of ws.dig: msm_sort's per-block count table (or W n words, whichever is larger) and msm_view's keep bitmap
// and block counts
static inline size_t msm_sort_dig_words(const MsmShape& sh, const MsmSizes& z, uint32_t n) {
  const size_t tab_words = (size_t)z.K * (n ? ceil_div(n, msm_bin_tile(sh, z, n)) : 0) * sh.nb();
  return tab_words > z.nent ? tab_words : z.nent;
}
static inline size_t msm_view_dig_words(const MsmSizes& z) {
  const size_t nblk = ceil_div(z.nent, MSM_VIEW_T);
  return nblk * MSM_VIEW_WORDS + 2 * nblk + 1;
}

// Bucket reduction tail of msm_enqueue: segments of L buckets (L divides B), then k_msm_final_sum over each group's
// nseg_g segment sums in fs_blocks blocks; red holds the segment sums, the block sums and, for k > 1, the group sums.
// A batch of K MSMs has K k groups, proof p's being [p k, (p + 1) k).
template <class F>
struct MsmReduce {
  uint32_t L, nseg_g, nseg, ngroups, fs_threads, fs_blocks;
  size_t red_elems;
  explicit MsmReduce(const MsmShape& sh, uint32_t K = 1) {
    L = sh.B < MSM_RED_SEG ? sh.B : MSM_RED_SEG;
    nseg_g = sh.B / L;
    ngroups = K * sh.k;
    nseg = ngroups * nseg_g;
    fs_threads = sizeof(Xyzz<F>) > 128 ? 128 : 256;  // <= 32 KB of dynamic shared memory
    fs_blocks = nseg_g > 4 * fs_threads ? (nseg_g + fs_threads - 1) / fs_threads : 1;
    red_elems = (size_t)nseg + (size_t)ngroups * fs_blocks + (sh.k > 1 ? ngroups : 0);
  }
};

// Device bytes msm_sort / msm_view (sort) and msm_enqueue (accumulation) reserve in a workspace for K MSMs of n scalars
static inline size_t msm_sort_bytes(const MsmShape& sh, uint32_t n, uint32_t K = 1) {
  const MsmSizes z(sh, n, K);
  const size_t dig = msm_sort_dig_words(sh, z, n) > msm_view_dig_words(z) ? msm_sort_dig_words(sh, z, n) : msm_view_dig_words(z);
  return DevBuf::alloc_size(dig * 4) + DevBuf::alloc_size(z.nent * 4) + DevBuf::alloc_size(z.meta_words() * 4) +
         DevBuf::alloc_size(z.order_words() * 4);
}
template <class F>
size_t msm_accum_bytes(const MsmShape& sh, uint32_t n, uint32_t K = 1) {
  const MsmSizes z(sh, n, K);
  const size_t x = sizeof(Xyzz<F>);
  return DevBuf::alloc_size(z.max_s0 * x) + DevBuf::alloc_size(z.max_s1 * x) + DevBuf::alloc_size(z.max_s2 * x) +
         DevBuf::alloc_size((size_t)z.nb1 * x) + DevBuf::alloc_size(MsmReduce<F>(sh, K).red_elems * x) +
         DevBuf::alloc_size(K * x);
}

// Digits, bucket sort and slice order of n scalars into ws; the entries index table slots row * nbases + offset + i.
// infmask = null keeps the entries of every base: with nbases = n and offset = 0 that is the shared witness sort,
// which msm_enqueue reads as it is (a table without infinity bases and slots row * n + i) or through msm_view.
// K > 1: K scalar vectors (proof p's scalar i at (i sstride + p pstride) elements) sorted as one over K k B buckets.
template <class FrP>
int msm_sort(MsmWorkspace& ws, const uint32_t* infmask, uint32_t nbases, MsmShape sh, uint32_t offset,
             const uint32_t* d_scalars, uint32_t sstride, uint32_t n, int mont, cudaStream_t st, uint32_t K = 1,
             uint32_t pstride = 0) {
  CS_TRY(msm_check_limits(sh, n, nbases, K));
  const MsmSizes z(sh, n, K);
  const uint32_t tile = msm_bin_tile(sh, z, n);
  const uint32_t nblk_p = n ? ceil_div(n, tile) : 0, nblk = K * nblk_p;
  const uint32_t NB = sh.nb();  // buckets of one proof
  const dim3 grid(nblk, ceil_div(NB, MSM_BIN_SPAN)), grid_sc(nblk, ceil_div(NB, MSM_SCATTER_SPAN));
  const uint32_t smem = (NB < MSM_BIN_SPAN ? NB : MSM_BIN_SPAN) * 4;
  const uint32_t smem_sc = (NB < MSM_SCATTER_SPAN ? NB : MSM_SCATTER_SPAN) * 4;
  // dig holds the per-block count table (k_msm_bin_*)
  CS_TRY(ws.dig.reserve(msm_sort_dig_words(sh, z, n) * 4));
  CS_TRY(ws.sorted.reserve(z.nent * 4));
  CS_TRY(ws.meta.reserve(z.meta_words() * 4));
  CS_TRY(ws.order.reserve(z.order_words() * 4));
  const MsmSortBufs q(ws, z);
  uint32_t* tab = ws.dig.as<uint32_t>();
  CS_TRY(ws.mark(0, st));
  if (nblk)
    CS_LAUNCH_SYNC(k_msm_bin_count<FrP>, grid, MSM_BIN_T, smem, st, d_scalars, sstride, n, mont, sh.c, sh.W, sh.k,
                   infmask, offset, tile, nblk_p, pstride, NB, tab);
  CS_TRY(ws.mark(1, st));
  CS_LAUNCH(k_msm_bin_scan, ceil_div(K * NB, 256), 256, 0, st, tab, nblk_p, NB, K * NB, q.count);
  CS_TRY(msm_scan(q, z, K * NB, st));
  if (nblk)
    CS_LAUNCH_SYNC(k_msm_bin_scatter<FrP>, grid_sc, MSM_BIN_T, smem_sc, st, d_scalars, sstride, n, mont, sh.c, sh.W, sh.k,
                   infmask, offset, tile, nblk_p, pstride, NB, nbases, tab, q.start, ws.sorted.as<uint32_t>());
  return msm_slice_order(ws, q, z, st);
}

// This table's entries out of the shared witness sort in src (k_msm_view_*): entries of its infinite bases dropped,
// the others rewritten to its slots row * nbases + offset + i; then bucket offsets and a slice order of its own.
static inline int msm_view(MsmWorkspace& ws, const MsmWorkspace& src, const uint32_t* infmask, uint32_t nbases,
                           MsmShape sh, uint32_t offset, uint32_t n, cudaStream_t st, uint32_t K = 1) {
  const MsmSizes z(sh, n, K);
  const uint32_t nblk = ceil_div(z.nent, MSM_VIEW_T);
  // dig: keep bitmap | blk_cnt[nblk] | blk_off[nblk + 1]
  CS_TRY(ws.dig.reserve(msm_view_dig_words(z) * 4));
  CS_TRY(ws.sorted.reserve(z.nent * 4));
  CS_TRY(ws.meta.reserve(z.meta_words() * 4));
  CS_TRY(ws.order.reserve(z.order_words() * 4));
  const MsmSortBufs q(ws, z), s(src, z);
  uint32_t* keep = ws.dig.as<uint32_t>();
  uint32_t* blk_cnt = keep + (size_t)nblk * MSM_VIEW_WORDS;
  uint32_t* blk_off = blk_cnt + nblk;
  const uint32_t* src_sorted = src.sorted.as<uint32_t>();
  CS_LAUNCH_SYNC(k_msm_view_flags, nblk, MSM_VIEW_T, 0, st, src_sorted, s.start, z.nb1, n, infmask, offset, keep, blk_cnt);
  CS_LAUNCH_SYNC(k_msm_view_scan, 1, MSM_SCAN_T, 0, st, blk_cnt, nblk, blk_off);
  CS_LAUNCH(k_msm_view_counts, ceil_div(z.nb1, 256), 256, 0, st, s.start, z.nb1, keep, blk_off, q.count);
  CS_LAUNCH(k_msm_view_scatter, nblk, MSM_VIEW_T, 0, st, src_sorted, n, nbases, offset, keep, blk_off,
            ws.sorted.as<uint32_t>());
  CS_TRY(msm_scan(q, z, K * sh.nb(), st));
  return msm_slice_order(ws, q, z, st);
}

// Enqueue one MSM on `st`.  d_scalars: device, n elements of Fr (8 x u32).  The XYZZ result lands in ws.result and
// ws.h_result (pinned) after the stream drains.  K > 1: a batch of K MSMs over the same bases (scalar layout as in
// msm_sort), one sort and accumulation for all; K results.
// sort_from (optional): a workspace holding a sort of the SAME scalars, enqueued earlier; `st` waits for it.
//  * view = false: its sorted entries and slice order are used as they are (they index table slots, not points), so
//    this MSM starts at the accumulation.  Table geometry (nbases, offset, n, window) and infinity pattern must
//    match: Groth16's B2 on B1's entries, or L (no infinity base, slots w * n + i) on the shared witness sort.
//  * view = true: sort_from holds the shared witness sort (msm_sort without a mask), and this MSM accumulates its
//    own filtered view of it (msm_view).
// st_acc (optional): a second, LOWER-priority stream for the accumulation kernel alone.  When several MSMs share the
// GPU, the block scheduler serves equal-priority grids in launch order, so the short sort / fold / reduce kernels of
// one MSM queue behind the full-GPU accumulation grids of all the others (measured: folds of an MSM finished at 3 ms
// ran long after their own accumulation); with the accumulation on a lower-priority stream they slip in between.
template <class F, class FrP>
int msm_enqueue(MsmWorkspace& ws, const Affine<F>* table, const uint32_t* infmask, uint32_t nbases, MsmShape sh,
                uint32_t offset,
                const uint32_t* d_scalars, uint32_t sstride, uint32_t n, int mont, cudaStream_t st,
                MsmWorkspace* sort_from = nullptr, bool view = false, bool table_m260 = false, cudaStream_t st_acc = nullptr,
                uint32_t K = 1, uint32_t pstride = 0) {
  CS_TRY(msm_check_limits(sh, n, nbases, K));
  const MsmSizes z(sh, n, K);
  const uint32_t nb1 = z.nb1, S = z.S;
  const size_t max_s0 = z.max_s0, max_s1 = z.max_s1, max_s2 = z.max_s2;
  CS_TRY(ws.part0.reserve(max_s0 * sizeof(Xyzz<F>)));
  CS_TRY(ws.part1.reserve(max_s1 * sizeof(Xyzz<F>)));
  CS_TRY(ws.part2.reserve(max_s2 * sizeof(Xyzz<F>)));
  CS_TRY(ws.bucket.reserve((size_t)nb1 * sizeof(Xyzz<F>)));
  const MsmReduce<F> rd(sh, K);
  const uint32_t L = rd.L, nseg = rd.nseg, fs_threads = rd.fs_threads, fs_blocks = rd.fs_blocks, G = rd.ngroups;
  CS_TRY(ws.red.reserve(rd.red_elems * sizeof(Xyzz<F>)));
  CS_TRY(ws.result.reserve(K * sizeof(Xyzz<F>)));
  if (ws.h_result_cap < K * sizeof(Xyzz<F>)) {
    if (ws.h_result) cudaFreeHost(ws.h_result);
    ws.h_result = nullptr;
    ws.h_result_cap = 0;
    CS_CUDA(cudaMallocHost(&ws.h_result, K * sizeof(Xyzz<F>)));
    ws.h_result_cap = K * sizeof(Xyzz<F>);
  }
  if (sort_from) {
    if (!sort_from->sorted_once) return fail(-1, "msm: the workspace to share a sort with has not been enqueued");
    CS_TRY(ws.mark(0, st));
    CS_CUDA(cudaStreamWaitEvent(st, sort_from->sorted_ev, 0));
    CS_TRY(ws.mark(1, st));
    if (view) CS_TRY(msm_view(ws, *sort_from, infmask, nbases, sh, offset, n, st, K));
  } else {
    CS_TRY(msm_sort<FrP>(ws, infmask, nbases, sh, offset, d_scalars, sstride, n, mont, st, K, pstride));
  }
  MsmWorkspace& so = sort_from && !view ? *sort_from : ws;  // owner of the sorted entries
  const MsmSortBufs q(so, z);
  const uint32_t *count = q.count, *start = q.start, *sstart0 = q.sstart0, *sstart1 = q.sstart1, *sstart2 = q.sstart2;
  const uint32_t *order = q.order, *order_b = q.order_b;
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
    // resident blocks per SM (register cap), overridable for experiments.  G2 at 2: the cap under which its kernel does
    // not spill, and the fastest in a sweep on the H100 (DESIGN.md 4.2)
    static int minb_env = -1;
    if (minb_env < 0) { const char* e = getenv("CS_ACCUM0_MINB"); minb_env = e ? atoi(e) : 0; }
    const int minb = minb_env ? minb_env : (sizeof(Affine<F>) > 64 ? 2 : 4);
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
  CS_LAUNCH(k_msm_reduce_seg<F>, ceil_div(nseg, 128), 128, 0, st, ws.bucket.as<Xyzz<F>>(), K * sh.nb(), sh.B, L,
            ws.red.as<Xyzz<F>>());
  // one sum per bucket group: the MSM results themselves when k = 1, else the group sums that k_msm_combine_groups weights
  Xyzz<F>* gsum = sh.k > 1 ? ws.red.as<Xyzz<F>>() + nseg + (size_t)G * fs_blocks : ws.result.as<Xyzz<F>>();
  if (fs_blocks > 1) {
    Xyzz<F>* stage = ws.red.as<Xyzz<F>>() + nseg;
    CS_LAUNCH_SYNC(k_msm_final_sum<F>, dim3(fs_blocks, G), fs_threads, fs_threads * sizeof(Xyzz<F>), st,
                   ws.red.as<Xyzz<F>>(), rd.nseg_g, stage);
    CS_LAUNCH_SYNC(k_msm_final_sum<F>, dim3(1, G), fs_threads, fs_threads * sizeof(Xyzz<F>), st, stage, fs_blocks, gsum);
  } else {
    CS_LAUNCH_SYNC(k_msm_final_sum<F>, dim3(1, G), fs_threads, fs_threads * sizeof(Xyzz<F>), st, ws.red.as<Xyzz<F>>(),
                   rd.nseg_g, gsum);
  }
  // one launch per MSM of a batch: a batch index in the kernel makes its G2 instantiations spill more
  for (uint32_t p = 0; sh.k > 1 && p < K; p++)
    CS_LAUNCH(k_msm_combine_groups<F>, 1, 1, 0, st, gsum + (size_t)p * sh.k, sh.k, sh.c, ws.result.as<Xyzz<F>>() + p);
  CS_TRY(ws.mark(5, st));
  CS_CUDA(cudaMemcpyAsync(ws.h_result, ws.result.p, K * sizeof(Xyzz<F>), cudaMemcpyDeviceToHost, st));
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
