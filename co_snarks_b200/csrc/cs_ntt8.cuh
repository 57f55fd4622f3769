// NTT pass, second generation: TMA-staged tiles + register radix-8 butterflies.
//
// Same transform as k_ntt_pass (cs_ntt.cuh; replaces taceo_ark_algebra::fft::Domain::{ifft_in_to_out,
// fft_out_to_in}, call sites co-groth16/src/groth16/reduction.rs:141-175) -- a pass runs k <= 7 stages on index
// bits [log_stride, log_stride + k) -- with three changes that the round-1 profile asked for:
//  * a CTA owns a 32 KB tile of 1024 field elements: 2^k rows x CB columns, where the columns are NEIGHBOURING
//    indices (strided passes: consecutive `lo`, so a row is CB * 32 contiguous bytes instead of one 32-byte
//    sector; stride-1 pass: consecutive tiles, the whole tile is one contiguous range);
//  * the tile is brought into shared memory by the TMA unit: every thread issues ONE `cp.async.bulk` for its
//    256-byte piece, all completing on one mbarrier (`mbarrier.arrive.expect_tx`), and written back with
//    `cp.async.bulk.global.shared::cta` -- no LDG -> register -> STS round trip, no address arithmetic per element;
//  * butterflies run three stages at a time in registers (radix-8: 8 elements, 12 products, 7 twiddles per
//    thread and round), so a 7-stage pass synchronises 3 times instead of 7 and touches shared memory 3 times.
// Shared-memory bank conflicts are left alone on purpose: a butterfly costs ~600 issue cycles of Montgomery
// product per warp, a 2-way conflicted LDS.128 pair ~16.
#pragma once
#include "cs_common.cuh"
#include "cs_field.cuh"
#include "cs_ntt.cuh"

namespace cs {

constexpr uint32_t NTT8_ELEMS = 1024;   // field elements per CTA tile (32 KB)
constexpr uint32_t NTT8_THREADS = 128;  // 8 elements per thread and round
constexpr uint32_t NTT8_MAX_K = 7;

#if !defined(CS_EMU)
CS_D uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
CS_D void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
CS_D void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
CS_D void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// global -> shared, completion counted on the mbarrier (TMA bulk copy, no tensor map: 1-D, 16-byte granules)
CS_D void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
CS_D void tma_store_1d(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
CS_D void tma_store_commit_wait() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
CS_D void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#endif

template <class FrP>
CS_D Fp<FrP> ld_sm(const uint4* sm, uint32_t e) {
  Fp<FrP> r;
  const uint4 a = sm[2 * e], c = sm[2 * e + 1];
  r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w; r.l[4] = c.x; r.l[5] = c.y; r.l[6] = c.z; r.l[7] = c.w;
  return r;
}
template <class FrP>
CS_D void st_sm(uint4* sm, uint32_t e, const Fp<FrP>& v) {
  sm[2 * e] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
  sm[2 * e + 1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}

// one stage on a pair held in registers
template <class FrP, bool DIT>
CS_D void bfly(Fp<FrP>& x, Fp<FrP>& y, const Fp<FrP>& w) {
  if (DIT) {
    const Fp<FrP> t = y * w;
    y = x - t;
    x = x + t;
  } else {
    const Fp<FrP> d = x - y;
    x = x + y;
    y = d * w;
  }
}

struct Ntt8Ctx {
  uint4* sm;
  const uint32_t *tw, *post, *scale;
  uint32_t logn, log_stride, k, batch, R, CB, C, stride, lo0, tile, t;
  bool contiguous;
  size_t gbase;
};

// One round: L stages on groups of 2^L elements spaced s = 2^lmm_lo rows apart; every thread takes 8 / 2^L groups.
template <class FrP, bool DIT, int L>
CS_D void ntt8_round(const Ntt8Ctx& c, uint32_t done) {
  typedef Fp<FrP> F;
  constexpr int NW = FrP::N;
  constexpr int Gs = 1 << L;
  // local half-sizes of this round's stages: DIF takes them from the top (k-1-done ...), DIT from the bottom
  const uint32_t lmm_lo = DIT ? done : (c.k - done - L);  // log2 of the SMALLEST half-size in the round
  const uint32_t s = 1u << lmm_lo;                         // row spacing inside a group
  const bool last_round = (done + L == c.k);
  for (uint32_t u = 0; u < (8u >> L); u++) {
    const uint32_t gid = c.t + NTT8_THREADS * u;
    const uint32_t cc = gid % c.CB, q = gid / c.CB;
    const uint32_t o = q & (s - 1), b = q >> lmm_lo;
    const uint32_t base = (b << (lmm_lo + L)) + o;
    const uint32_t lo = c.contiguous ? 0 : c.lo0 + cc / c.batch;
    auto eidx = [&](uint32_t r) -> uint32_t {
      return c.contiguous ? ((cc / c.batch) * c.R + r) * c.batch + (cc % c.batch) : r * c.CB + cc;
    };
    F v[Gs];
    CS_UNROLL
    for (int j = 0; j < Gs; j++) v[j] = ld_sm<FrP>(c.sm, eidx(base + j * s));
    CS_UNROLL
    for (int st = 0; st < L; st++) {
      const int hbit = DIT ? st : (L - 1 - st);            // pairs differ in bit hbit of j
      const uint32_t lmm = lmm_lo + hbit;                   // log2 local half-size
      const uint32_t tshift = c.logn - 1 - (lmm + c.log_stride);
      CS_UNROLL
      for (int j = 0; j < Gs; j++) {
        if ((j >> hbit) & 1) continue;
        const int j2 = j | (1 << hbit);
        const uint32_t r0 = base + j * s;
        const uint32_t jj = (r0 & ((1u << lmm) - 1)) * c.stride + lo;
        const F w = ld_fr<FrP>(c.tw + ((size_t)jj << tshift) * NW);
        bfly<FrP, DIT>(v[j], v[j2], w);
      }
    }
    CS_UNROLL
    for (int j = 0; j < Gs; j++) {
      const uint32_t r = base + j * s;
      if (last_round && (c.post || c.scale)) {
        const size_t g = c.contiguous ? ((size_t)c.tile * c.C + cc / c.batch) * c.R + r : c.gbase + (size_t)r * c.stride + cc / c.batch;
        if (c.post) v[j] = v[j] * ld_fr<FrP>(c.post + g * NW);
        if (c.scale) v[j] = v[j] * ld_fr<FrP>(c.scale);
      }
      st_sm<FrP>(c.sm, eidx(r), v[j]);
    }
  }
}

// rounds[i] = number of stages done in registers in round i (1..3); sum = k
template <class FrP, bool DIT>
CS_GLOBAL void __launch_bounds__(NTT8_THREADS) k_ntt_pass8(uint32_t* __restrict__ data, const uint32_t* __restrict__ tw,
                                                           uint32_t logn, uint32_t log_stride, uint32_t k, uint32_t batch,
                                                           uint32_t rounds_packed, const uint32_t* __restrict__ post,
                                                           const uint32_t* __restrict__ scale) {
  typedef Fp<FrP> F;
  constexpr int NW = FrP::N;
  CS_DYN_SMEM(uint4, sm);
  const uint32_t R = 1u << k;
  const uint32_t CB = NTT8_ELEMS >> k;     // field elements per row
  const uint32_t C = CB / batch;            // indices per row
  const uint32_t stride = 1u << log_stride;
  const bool contiguous = log_stride == 0;
  const uint32_t t = threadIdx.x;
  // ---- tile geometry
  //   strided:    tile -> (hi, lo0), element (r, cc): index g = hi R stride + r stride + lo0 + cc / batch, component cc % batch
  //   contiguous: tile -> C consecutive row blocks, element (r, cc): g = (tile C + cc / batch) R + r
  uint32_t hi = 0, lo0 = 0;
  if (!contiguous) {
    const uint32_t per_hi = stride / C;
    hi = blockIdx.x / per_hi;
    lo0 = (blockIdx.x % per_hi) * C;
  }
  const size_t gbase = contiguous ? (size_t)blockIdx.x * NTT8_ELEMS / batch : ((size_t)hi << (k + log_stride)) + lo0;
  // ---- load: 128 threads x 256 bytes through the TMA unit
  const uint32_t piece = NTT8_ELEMS * 32 / NTT8_THREADS;  // 256 B
  char* smb = reinterpret_cast<char*>(sm);
#if defined(CS_EMU)
  {
    for (uint32_t b = 0; b < piece; b += 16) {
      const uint32_t off = t * piece + b;  // byte offset inside the tile image
      size_t goff;
      if (contiguous) goff = gbase * batch * 32 + off;
      else { const uint32_t r = off / (CB * 32), in_row = off % (CB * 32); goff = ((gbase + (size_t)r * stride) * batch) * 32 + in_row; }
      *reinterpret_cast<uint4*>(smb + off) = *reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(data) + goff);
    }
  }
  __syncthreads();
#else
  uint64_t* bar = reinterpret_cast<uint64_t*>(smb + NTT8_ELEMS * 32);
  if (t == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (t == 0) mbar_expect_tx(bar, NTT8_ELEMS * 32);
  __syncthreads();  // the expectation is registered before any copy can complete
  {
    const uint32_t row_bytes = CB * 32;
    // a thread's 256-byte piece never straddles two rows: row_bytes is 256 (k = 7, batch 1), 512, ... or the tile is contiguous
    const uint32_t off = t * piece;
    const char* g = reinterpret_cast<const char*>(data);
    size_t goff;
    if (contiguous) goff = gbase * batch * 32 + off;
    else { const uint32_t r = off / row_bytes, in_row = off % row_bytes; goff = ((gbase + (size_t)r * stride) * batch) * 32 + in_row; }
    tma_load_1d(smb + off, g + goff, piece, bar);
  }
  mbar_wait(bar, 0);
#endif
  // ---- rounds (the per-round code is instantiated for L = 1, 2, 3 so that the 2^L elements stay in registers)
  Ntt8Ctx cx;
  cx.sm = sm; cx.tw = tw; cx.post = post; cx.scale = scale;
  cx.logn = logn; cx.log_stride = log_stride; cx.k = k; cx.batch = batch; cx.R = R; cx.CB = CB; cx.C = C; cx.stride = stride;
  cx.contiguous = contiguous; cx.lo0 = lo0; cx.gbase = gbase; cx.tile = blockIdx.x; cx.t = t;
  uint32_t done = 0;  // stages finished
  for (uint32_t rd = 0; rd < 4; rd++) {
    const uint32_t L = (rounds_packed >> (4 * rd)) & 15;
    if (!L) break;
    if (L == 3) ntt8_round<FrP, DIT, 3>(cx, done);
    else if (L == 2) ntt8_round<FrP, DIT, 2>(cx, done);
    else ntt8_round<FrP, DIT, 1>(cx, done);
    done += L;
    __syncthreads();
  }
  // ---- store
#if defined(CS_EMU)
  for (uint32_t b = 0; b < piece; b += 16) {
    const uint32_t off = t * piece + b;
    size_t goff;
    if (contiguous) goff = gbase * batch * 32 + off;
    else { const uint32_t r = off / (CB * 32), in_row = off % (CB * 32); goff = ((gbase + (size_t)r * stride) * batch) * 32 + in_row; }
    *reinterpret_cast<uint4*>(reinterpret_cast<char*>(data) + goff) = *reinterpret_cast<const uint4*>(smb + off);
  }
#else
  fence_proxy_async();  // the generic-proxy writes above must be visible to the TMA unit
  __syncthreads();
  {
    const uint32_t row_bytes = CB * 32;
    const uint32_t off = t * piece;
    char* g = reinterpret_cast<char*>(data);
    size_t goff;
    if (contiguous) goff = gbase * batch * 32 + off;
    else { const uint32_t r = off / row_bytes, in_row = off % row_bytes; goff = ((gbase + (size_t)r * stride) * batch) * 32 + in_row; }
    tma_store_1d(g + goff, smb + off, piece);
    tma_store_commit_wait();  // shared memory must stay valid until the unit has read it
  }
#endif
}

// pass plan for the TMA / radix-8 kernel; returns false when the geometry does not fit (small transforms use k_ntt_pass)
static inline bool ntt8_plan(uint32_t logn, uint32_t batch, bool dit, uint32_t* ks, uint32_t* strides, uint32_t* npass_out) {
  if (logn < 12 || logn > 31) return false;
  const uint32_t npass = (logn + NTT8_MAX_K - 1) / NTT8_MAX_K;
  uint32_t base = logn / npass, extra = logn % npass, done = 0;
  // index bits are consumed from the top (DIF) or from the bottom (DIT); give the extra stages to the strided passes
  uint32_t kk[8];
  for (uint32_t p = 0; p < npass; p++) kk[p] = base;
  for (uint32_t e = 0; e < extra; e++) kk[e] += 1;  // p = 0 .. extra-1: strided passes in DIF order
  // DIF order: pass p has log_stride = logn - done - k; the LAST DIF pass is the stride-1 pass (kk[npass-1] = base)
  for (uint32_t p = 0; p < npass; p++) {
    const uint32_t k = dit ? kk[npass - 1 - p] : kk[p];
    const uint32_t log_stride = dit ? done : (logn - done - k);
    const uint32_t C = (NTT8_ELEMS >> k) / batch;
    if (k > NTT8_MAX_K || k < 3 || C == 0) return false;
    if (log_stride != 0 && (1u << log_stride) < C) return false;
    // a 256-byte piece must stay inside one row of a strided tile
    if (log_stride != 0 && (NTT8_ELEMS >> k) * 32 < 256) return false;
    ks[p] = k;
    strides[p] = log_stride;
    done += k;
  }
  *npass_out = npass;
  return true;
}

static inline uint32_t ntt8_rounds(uint32_t k) {  // k = 3..7 -> stages per round, 4 bits each
  switch (k) {
    case 3: return 0x3;
    case 4: return 0x22;
    case 5: return 0x23;   // rounds: 3, then 2
    case 6: return 0x33;
    default: return 0x223; // 7: 3, 2, 2
  }
}

template <class FrP>
int ntt_enqueue8(uint32_t* d_data, const uint32_t* d_tw, uint32_t logn, uint32_t batch, bool dit, const uint32_t* d_post,
                 const uint32_t* d_scale, cudaStream_t st, bool* used) {
  uint32_t ks[8], ls[8], npass = 0;
  *used = false;
  if (!ntt8_plan(logn, batch, dit, ks, ls, &npass)) return 0;
  *used = true;
  const size_t smem = NTT8_ELEMS * 32 + 16;
  const uint32_t blocks = (uint32_t)((((size_t)1 << logn) * batch) / NTT8_ELEMS);
  for (uint32_t p = 0; p < npass; p++) {
    const bool last = p + 1 == npass;
    const uint32_t* post = last ? d_post : nullptr;
    const uint32_t* scale = last ? d_scale : nullptr;
    if (dit)
      CS_LAUNCH_SYNC(k_ntt_pass8<FrP COMMA true>, blocks, NTT8_THREADS, smem, st, d_data, d_tw, logn, ls[p], ks[p], batch,
                     ntt8_rounds(ks[p]), post, scale);
    else
      CS_LAUNCH_SYNC(k_ntt_pass8<FrP COMMA false>, blocks, NTT8_THREADS, smem, st, d_data, d_tw, logn, ls[p], ks[p], batch,
                     ntt8_rounds(ks[p]), post, scale);
  }
  CS_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cs
