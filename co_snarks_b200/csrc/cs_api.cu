// C-ABI entry points: context, device memory, MSM, NTT, vector kernels, host helpers.
// (Groth16 entry points live in cs_groth16.cu.)  See include/cosnarks_gpu.h for the contract.
#include <stdarg.h>
#include "cs_lib.cuh"

namespace cs {

std::string& last_error() {
  static thread_local std::string e;
  return e;
}
int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  last_error() = buf;
  return code;
}
#if !defined(CS_EMU)
// The prover keeps up to 12 streams busy at once (five MSMs x {sort/fold/reduce, accumulation}, witness map, caller's
// stream).  The driver multiplexes streams onto CUDA_DEVICE_MAX_CONNECTIONS hardware queues (default 8); streams that
// share a queue serialise (the L MSM would not start until the unrelated H MSM had drained).  The variable is read when the CUDA context is created, so it is set when this library is
// loaded, unless the application chose a value itself.
__attribute__((constructor)) static void cs_more_hw_queues() { setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0); }
#endif

std::atomic<uint64_t>& launch_counter() {
  static std::atomic<uint64_t> c{0};
  return c;
}

int ctx_fork(cs_ctx* ctx, int nside) {
  if (ctx->msm_ws[0].profile) {
    if (!ctx->ev_t0) CS_CUDA(cudaEventCreateWithFlags(&ctx->ev_t0, 0));
    CS_CUDA(cudaEventRecord(ctx->ev_t0, ctx->stream));
  }
  CS_CUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));
  for (int i = 0; i < nside; i++) CS_CUDA(cudaStreamWaitEvent(ctx->side[i], ctx->ev_fork, 0));
  return 0;
}
int ctx_join(cs_ctx* ctx, int nside) {
  for (int i = 0; i < nside; i++) {
    CS_CUDA(cudaEventRecord(ctx->ev_side[i], ctx->side[i]));
    CS_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_side[i], 0));
  }
  return 0;
}

template <class FrP>
static int ntt_smem_optin() {
#if !defined(CS_EMU)
#define CS_NTT_ATTR(D, S, KB) \
  CS_CUDA(cudaFuncSetAttribute(k_ntt_pass<FrP, D, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, KB * 1024))
  CS_NTT_ATTR(true, false, (NTT_SMEM_PLAIN >> 10)); CS_NTT_ATTR(false, false, (NTT_SMEM_PLAIN >> 10));
  CS_NTT_ATTR(true, true, (NTT_SMEM_TWS >> 10)); CS_NTT_ATTR(false, true, (NTT_SMEM_TWS >> 10));
#undef CS_NTT_ATTR
#endif
  return 0;
}

}  // namespace cs

using namespace cs;

extern "C" {

const char* cs_last_error(void) { return last_error().c_str(); }

const char* cs_version(void) {
#if defined(CS_EMU)
  return "cosnarks-b200 0.1 (CPU emulation build -- tests only)";
#else
  return "cosnarks-b200 0.1 (sm_90a)";
#endif
}

int cs_ctx_create(int device, void* stream, cs_ctx** out) {
  if (!out) return fail(CS_ERR_ARG, "cs_ctx_create: out is NULL");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(CS_ERR_CUDA, "cs_ctx_create: no CUDA device available (%s); this library has no CPU path",
                e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
  if (device < 0 || device >= ndev) return fail(CS_ERR_ARG, "cs_ctx_create: device %d out of range (%d devices)", device, ndev);
  CS_CUDA(cudaSetDevice(device));
  cs_ctx* ctx = new cs_ctx();
  ctx->device = device;
  // Stream priorities (CUDA: lower number = served first).  The short, latency-bound kernels (digit sort, folds,
  // bucket reduction, NTT passes) run on higher-priority streams than the full-GPU MSM accumulation grids, so that
  // they are not queued behind every accumulation launched before them.  CS_PRIO="side,acc,wm" overrides
  // (default "-2,0,-2"); CS_MSM_SPLIT=0 keeps each MSM on a single stream.  The proof is bound by the sum of its
  // integer-pipe work; the layout only decides which MSM finishes first.
  int prio_side = -2, prio_acc = 0, prio_wm = -2;
  if (const char* e = getenv("CS_PRIO")) sscanf(e, "%d,%d,%d", &prio_side, &prio_acc, &prio_wm);
  const char* split_env = getenv("CS_MSM_SPLIT");
  const bool split = !(split_env && atoi(split_env) == 0);
  if (stream) {
    ctx->stream = (cudaStream_t)stream;
  } else {
    CS_CUDA(cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, prio_side));
    ctx->own_stream = true;
  }
  for (int i = 0; i < CS_NSIDE; i++) {
    CS_CUDA(cudaStreamCreateWithPriority(&ctx->side[i], cudaStreamNonBlocking, prio_side));
    if (split) CS_CUDA(cudaStreamCreateWithPriority(&ctx->acc[i], cudaStreamNonBlocking, prio_acc));
    CS_CUDA(cudaEventCreateWithFlags(&ctx->ev_side[i], cudaEventDisableTiming));
  }
  CS_CUDA(cudaStreamCreateWithPriority(&ctx->wm, cudaStreamNonBlocking, prio_wm));
  CS_CUDA(cudaEventCreateWithFlags(&ctx->ev_wm, cudaEventDisableTiming));
  CS_CUDA(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
  CS_TRY(ntt_smem_optin<Bn254Fr>());
  CS_TRY(msm_smem_optin<Bn254Fr>());
#if defined(CS_ENABLE_BLS12_381)
  CS_TRY(ntt_smem_optin<Bls381Fr>());
  CS_TRY(msm_smem_optin<Bls381Fr>());
#endif
  *out = ctx;
  return 0;
}

void cs_ctx_destroy(cs_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  ctx->msm_ws[CS_WIT_SORT].release();
  for (int i = 0; i < CS_NSIDE; i++) {
    ctx->msm_ws[i].release();
    if (ctx->side[i]) cudaStreamDestroy(ctx->side[i]);
    if (ctx->acc[i]) cudaStreamDestroy(ctx->acc[i]);
    if (ctx->ev_side[i]) cudaEventDestroy(ctx->ev_side[i]);
  }
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  if (ctx->wm) cudaStreamDestroy(ctx->wm);
  if (ctx->ev_wm) cudaEventDestroy(ctx->ev_wm);
  if (ctx->ev_t0) cudaEventDestroy(ctx->ev_t0);
  ctx->io.release();
  ctx->prf_keys.release();
  ctx->sc_part.release();
  ctx->sc_res.release();
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

int cs_ctx_synchronize(cs_ctx* ctx) {
  if (!ctx) return fail(CS_ERR_ARG, "ctx is NULL");
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return 0;
}

uint64_t cs_ctx_launch_count(const cs_ctx*) { return launch_counter().load(); }

int cs_dev_alloc(cs_ctx* ctx, size_t bytes, void** d_out) {
  if (!ctx || !d_out) return fail(CS_ERR_ARG, "cs_dev_alloc: bad argument");
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_CUDA(cudaMalloc(d_out, bytes ? bytes : 1));
  return 0;
}
int cs_dev_free(cs_ctx* ctx, void* d_ptr) {
  if (!ctx) return fail(CS_ERR_ARG, "ctx is NULL");
  CS_CUDA(cudaFree(d_ptr));
  return 0;
}
int cs_host_alloc_pinned(size_t bytes, void** h_out) {
  if (!h_out) return fail(CS_ERR_ARG, "h_out is NULL");
  CS_CUDA(cudaMallocHost(h_out, bytes ? bytes : 1));
  return 0;
}
int cs_host_free_pinned(void* h_ptr) {
  CS_CUDA(cudaFreeHost(h_ptr));
  return 0;
}
int cs_memcpy_h2d(cs_ctx* ctx, void* d_dst, const void* h_src, size_t bytes) {
  if (!ctx) return fail(CS_ERR_ARG, "ctx is NULL");
  CS_CUDA(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return 0;
}
int cs_memcpy_d2h(cs_ctx* ctx, void* h_dst, const void* d_src, size_t bytes) {
  if (!ctx) return fail(CS_ERR_ARG, "ctx is NULL");
  CS_CUDA(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------- MSM
namespace cs {

int table_budget(cs_ctx* ctx, size_t* out, size_t reusable) {
  size_t avail = 0, total = 0;
#if defined(CS_EMU)
  avail = total = 80ull << 30;  // the CPU emulation has no device: an 80 GB H100's, so full tables are picked as there
#else
  CS_CUDA(cudaMemGetInfo(&avail, &total));
#endif
  avail += reusable;
  avail = avail > TABLE_MARGIN ? avail - TABLE_MARGIN : 0;
  *out = ctx->table_budget && ctx->table_budget < avail ? ctx->table_budget : avail;
  return 0;
}

int pick_table_rows(cs_ctx* ctx, unsigned c, unsigned W, const std::function<size_t(unsigned)>& need, const char* who,
                    unsigned* k_out) {
  size_t budget = 0, least = SIZE_MAX;
  CS_TRY(table_budget(ctx, &budget));
  for (unsigned k = 1; k <= W; k++) {
    if ((size_t)k * (1u << (c - 1)) + 1 > (size_t)MSM_SCAN_MAX_BLOCKS * MSM_SCAN_T) break;  // k B buckets: msm_scan's limit
    const size_t b = need(k);  // not monotone in k: k B buckets of scratch can outweigh the rows saved on tiny tables
    if (b <= budget) {
      *k_out = k;
      return 0;
    }
    least = b < least ? b : least;
  }
  return fail(CS_ERR_LIMIT, "%s: the MSM tables need at least %zu bytes of device memory, %zu are available", who, least,
              budget);
}

template <class Cfg, int G>
int bases_upload_t(cs_ctx* ctx, const uint64_t* h_points, size_t n, int window_bits, unsigned k, cs_bases* b) {
  typedef typename GroupOf<Cfg, G>::F F;
  unsigned c = window_bits ? (unsigned)window_bits : msm_auto_window(n, Cfg::FR_BITS);
  // a window wider than msm_scan takes would build the table and then fail every MSM
  if (c < 2 || c > MSM_MAX_WINDOW)
    return fail(CS_ERR_ARG, "cs_bases_upload: window_bits %d out of range [2,%u] (0 = automatic)", window_bits, MSM_MAX_WINDOW);
  if (!k) {
    const unsigned W = msm_shape(Cfg::FR_BITS, c).W;
    CS_TRY(pick_table_rows(ctx, c, W, [&](unsigned kk) { return bases_bytes<Cfg, G>(n, msm_shape(Cfg::FR_BITS, c, kk)); },
                           "cs_bases_upload", &k));
  }
  b->sh = msm_shape(Cfg::FR_BITS, c, k);
  b->n = n;
  size_t total = (size_t)b->sh.T * n;
  if (total >= (1ull << 31)) return fail(CS_ERR_LIMIT, "cs_bases_upload: T*n = %zu table slots exceed 2^31", total);
  CS_TRY(b->table.reserve(total * sizeof(Affine<F>)));
  CS_CUDA(cudaMemcpyAsync(b->table.p, h_points, n * sizeof(Affine<F>), cudaMemcpyHostToDevice, ctx->stream));
  CS_TRY(b->infmask.reserve(((n + 31) / 32) * 4));
  CS_LAUNCH(k_msm_infmask<F>, ceil_div((n + 31) / 32, 128), 128, 0, ctx->stream, b->table.as<Affine<F>>(), (uint32_t)n,
            b->infmask.as<uint32_t>());
  // row j = 2^(c k j) P_i: the full-table precomputation with a window of c k bits
  CS_LAUNCH(k_msm_precompute<F>, ceil_div(n, 128), 128, 0, ctx->stream, b->table.as<Affine<F>>(), (uint32_t)n,
            b->sh.c * b->sh.k, b->sh.T);
  // BN254 G1, opt-in (CS_MSM_F52=1): bucket accumulation on the FP64 pipe (cs_msm52.cuh); its table holds the
  // coordinates in the radix-2^260 Montgomery form.  Bit-exact, but the FP64 and integer pipes do not overlap, so
  // trading IMAD.WIDE for DFMA buys nothing: the integer kernel stays the default.
  if (G == 0 && std::is_same<Cfg, Bn254Cfg>::value) {
    static int f52_env = -1;
    if (f52_env < 0) { const char* e = getenv("CS_MSM_F52"); f52_env = e ? atoi(e) : 0; }
    if (f52_env) {
      const size_t ncoords = total * 2;
      CS_LAUNCH(k_msm_table_to_m260<Bn254Fq52 COMMA Bn254Fq>, ceil_div(ncoords, 128), 128, 0, ctx->stream,
                b->table.as<uint32_t>(), ncoords);
      b->m260 = true;
    }
  }
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return 0;
}

template <class Cfg, int G>
int msm_enqueue_t(cs_ctx* ctx, int slot, cudaStream_t st, const cs_bases* b, size_t offset,
                  const uint32_t* d_scalars, unsigned sstride, size_t n, int mont, int sort_slot, bool view, unsigned K,
                  size_t pstride) {
  typedef typename GroupOf<Cfg, G>::F F;
  return msm_enqueue<F, typename Cfg::FrP>(ctx->msm_ws[slot], b->table.as<Affine<F>>(), b->infmask.as<uint32_t>(), (uint32_t)b->n, b->sh,
                                           (uint32_t)offset, d_scalars, sstride, (uint32_t)n, mont, st,
                                           sort_slot >= 0 ? &ctx->msm_ws[sort_slot] : nullptr, view, b->m260, ctx->acc[slot],
                                           K, (uint32_t)pstride);
}

// After the stream has drained: XYZZ (pinned) -> affine on the host.
template <class Cfg, int G>
void msm_finish_t(cs_ctx* ctx, int slot, uint64_t* out_affine, int* out_inf) {
  typedef typename GroupOf<Cfg, G>::HF HF;
  const host::HXyzz<HF>* r = reinterpret_cast<const host::HXyzz<HF>*>(ctx->msm_ws[slot].h_result);
  host::HAffine<HF> a = host::haffine(*r);
  memcpy(out_affine, &a, sizeof(a));
  if (out_inf) *out_inf = a.is_inf() ? 1 : 0;
}

int msm_enqueue_dyn(cs_ctx* ctx, int slot, cudaStream_t st, const cs_bases* b, size_t offset,
                    const uint32_t* d_scalars, unsigned sstride, size_t n, int mont, int sort_slot, bool view, unsigned K,
                    size_t pstride) {
  CS_DISPATCH_CURVE(b->curve, {
    if (b->group == CS_G1)
      return msm_enqueue_t<Cfg, 0>(ctx, slot, st, b, offset, d_scalars, sstride, n, mont, sort_slot, view, K, pstride);
    return msm_enqueue_t<Cfg, 1>(ctx, slot, st, b, offset, d_scalars, sstride, n, mont, sort_slot, view, K, pstride);
  });
  return 0;
}
int msm_sort_shared_dyn(cs_ctx* ctx, int slot, cudaStream_t st, const cs_bases* b, const uint32_t* d_scalars,
                        unsigned sstride, size_t n, int mont, unsigned K, size_t pstride) {
  CS_DISPATCH_CURVE(b->curve, {
    return msm_sort<typename Cfg::FrP>(ctx->msm_ws[slot], nullptr, (uint32_t)n, b->sh, 0, d_scalars, sstride, (uint32_t)n,
                                       mont, st, K, (uint32_t)pstride);
  });
  return 0;
}

int bases_upload(cs_ctx* ctx, cs_curve curve, cs_group group, const uint64_t* h_points_mont, size_t n, int window_bits,
                 unsigned k, cs_bases** out) {
  if (!ctx || !h_points_mont || !out) return fail(CS_ERR_ARG, "cs_bases_upload: NULL argument");
  if (n == 0) return fail(CS_ERR_ARG, "cs_bases_upload: empty base set");
  if (group != CS_G1 && group != CS_G2) return fail(CS_ERR_ARG, "cs_bases_upload: bad group %d", (int)group);
  CS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<cs_bases, void (*)(cs_bases*)> b(new cs_bases(), cs_bases_free);  // a failed upload frees its buffers
  b->curve = curve;
  b->group = group;
  CS_DISPATCH_CURVE(curve, {
    if (group == CS_G1) CS_TRY((bases_upload_t<Cfg, 0>(ctx, h_points_mont, n, window_bits, k, b.get())));
    else CS_TRY((bases_upload_t<Cfg, 1>(ctx, h_points_mont, n, window_bits, k, b.get())));
  });
  *out = b.release();
  return 0;
}

int msm_finish_dyn(cs_ctx* ctx, int slot, const cs_bases* b, uint64_t* out_affine, int* out_inf) {
  CS_DISPATCH_CURVE(b->curve, {
    if (b->group == CS_G1) msm_finish_t<Cfg, 0>(ctx, slot, out_affine, out_inf);
    else msm_finish_t<Cfg, 1>(ctx, slot, out_affine, out_inf);
  });
  return 0;
}

}  // namespace cs

extern "C" {

int cs_ctx_set_table_budget(cs_ctx* ctx, size_t bytes) {
  if (!ctx) return fail(CS_ERR_ARG, "ctx is NULL");
  ctx->table_budget = bytes;
  return 0;
}

int cs_bases_upload(cs_ctx* ctx, cs_curve curve, cs_group group, const uint64_t* h_points_mont, size_t n,
                    int window_bits, cs_bases** out) {
  return bases_upload(ctx, curve, group, h_points_mont, n, window_bits, 0, out);
}

void cs_bases_free(cs_bases* b) {
  if (!b) return;
  b->table.release();
  b->infmask.release();
  delete b;
}

size_t cs_bases_len(const cs_bases* b) { return b ? b->n : 0; }

int cs_bases_info(const cs_bases* b, unsigned* window_bits, unsigned* windows, unsigned* table_rows, size_t* device_bytes) {
  if (!b) return fail(CS_ERR_ARG, "cs_bases_info: bases is NULL");
  if (window_bits) *window_bits = b->sh.c;
  if (windows) *windows = b->sh.W;
  if (table_rows) *table_rows = b->sh.T;
  if (device_bytes) *device_bytes = b->table.cap + b->infmask.cap;
  return 0;
}

int cs_msm_device(cs_ctx* ctx, const cs_bases* b, size_t offset, const uint64_t* d_scalars, size_t n,
                  int scalars_montgomery, uint64_t* h_out, int* out_inf) {
  if (!ctx || !b || !h_out) return fail(CS_ERR_ARG, "cs_msm: NULL argument");
  if (offset + n > b->n) return fail(CS_ERR_ARG, "cs_msm: offset %zu + n %zu exceeds the %zu uploaded bases", offset, n, b->n);
  size_t plimbs = point_limbs64(b->curve, b->group);
  if (n == 0) {
    memset(h_out, 0, plimbs * 8);
    if (out_inf) *out_inf = 1;
    return 0;
  }
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_TRY(msm_enqueue_dyn(ctx, 0, ctx->stream, b, offset, reinterpret_cast<const uint32_t*>(d_scalars), 1, n,
                         scalars_montgomery));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return msm_finish_dyn(ctx, 0, b, h_out, out_inf);
}

int cs_msm(cs_ctx* ctx, const cs_bases* b, size_t offset, const uint64_t* h_scalars, size_t n,
           int scalars_montgomery, uint64_t* h_out, int* out_inf) {
  if (!ctx || !b || !h_out) return fail(CS_ERR_ARG, "cs_msm: NULL argument");
  if (n && !h_scalars) return fail(CS_ERR_ARG, "cs_msm: scalars is NULL");
  if (n == 0) return cs_msm_device(ctx, b, offset, nullptr, 0, scalars_montgomery, h_out, out_inf);
  CS_CUDA(cudaSetDevice(ctx->device));
  MsmWorkspace& ws = ctx->msm_ws[0];
  CS_TRY(ws.scal.reserve(n * 32));
  CS_CUDA(cudaMemcpyAsync(ws.scal.p, h_scalars, n * 32, cudaMemcpyHostToDevice, ctx->stream));
  return cs_msm_device(ctx, b, offset, ws.scal.as<uint64_t>(), n, scalars_montgomery, h_out, out_inf);
}

// rep3::pointshare::msm_public_points (pointshare.rs:201-222): two MSMs over the a and b components of
// replicated shares, run concurrently on two streams straight from the interleaved share array.
int cs_msm_rep3_shares(cs_ctx* ctx, const cs_bases* b, size_t offset, const uint64_t* h_shares, size_t n,
                       uint64_t* h_out_a, uint64_t* h_out_b) {
  if (!ctx || !b || !h_out_a || !h_out_b || (n && !h_shares)) return fail(CS_ERR_ARG, "cs_msm_rep3_shares: NULL argument");
  if (offset + n > b->n) return fail(CS_ERR_ARG, "cs_msm_rep3_shares: slice exceeds the uploaded bases");
  const size_t plimbs = point_limbs64(b->curve, b->group);
  if (n == 0) {
    memset(h_out_a, 0, plimbs * 8);
    memset(h_out_b, 0, plimbs * 8);
    return 0;
  }
  CS_CUDA(cudaSetDevice(ctx->device));
  MsmWorkspace& ws = ctx->msm_ws[0];
  CS_TRY(ws.scal.reserve(n * 64));
  CS_CUDA(cudaMemcpyAsync(ws.scal.p, h_shares, n * 64, cudaMemcpyHostToDevice, ctx->stream));
  CS_TRY(ctx_fork(ctx, 2));
  const uint32_t* sc = ws.scal.as<uint32_t>();
  CS_TRY(msm_enqueue_dyn(ctx, 1, ctx->side[0], b, offset, sc, 2, n, 1));      // component a
  CS_TRY(msm_enqueue_dyn(ctx, 2, ctx->side[1], b, offset, sc + 8, 2, n, 1));  // component b
  CS_TRY(ctx_join(ctx, 2));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  CS_TRY(msm_finish_dyn(ctx, 1, b, h_out_a, nullptr));
  return msm_finish_dyn(ctx, 2, b, h_out_b, nullptr);
}

int cs_msm_profile(cs_ctx* ctx, int enable) {
  if (!ctx) return fail(CS_ERR_ARG, "ctx is NULL");
  for (int i = 0; i < CS_NSIDE; i++) ctx->msm_ws[i].profile = enable != 0;
  return 0;
}

int cs_msm_stage_ms(cs_ctx* ctx, float* out_ms) {
  if (!ctx || !out_ms) return fail(CS_ERR_ARG, "cs_msm_stage_ms: NULL argument");
  MsmWorkspace& ws = ctx->msm_ws[0];
  if (!ws.profile || !ws.ev[MSM_NSTAGE]) return fail(CS_ERR_STATE, "cs_msm_stage_ms: no profiled MSM has run");
  for (int i = 0; i < MSM_NSTAGE; i++) {
#if defined(CS_EMU)
    out_ms[i] = 0.f;
#else
    CS_CUDA(cudaEventElapsedTime(&out_ms[i], ws.ev[i], ws.ev[i + 1]));
#endif
  }
  return 0;
}

int cs_msm_timeline_ms(cs_ctx* ctx, float* out_ms) {
  if (!ctx || !out_ms) return fail(CS_ERR_ARG, "cs_msm_timeline_ms: NULL argument");
  if (!ctx->msm_ws[0].profile || !ctx->ev_t0) return fail(CS_ERR_STATE, "cs_msm_timeline_ms: no profiled fork has run");
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_CUDA(cudaDeviceSynchronize());
  for (int w = 0; w < CS_NSIDE; w++)
    for (int i = 0; i <= MSM_NSTAGE; i++) {
      float v = -1.f;
#if !defined(CS_EMU)
      if (ctx->msm_ws[w].ev[i] && cudaEventElapsedTime(&v, ctx->ev_t0, ctx->msm_ws[w].ev[i]) != cudaSuccess) {
        v = -1.f;
        cudaGetLastError();
      }
#endif
      out_ms[w * (MSM_NSTAGE + 1) + i] = v;
    }
  return 0;
}

int cs_fixed_base_mul(cs_ctx* ctx, cs_curve curve, cs_group group, const uint64_t* h_base, const uint64_t* h_scalars,
                      size_t n, int scalars_montgomery, uint64_t* h_out) {
  if (!ctx || !h_base || !h_out || (n && !h_scalars)) return fail(CS_ERR_ARG, "cs_fixed_base_mul: NULL argument");
  if (n == 0) return 0;
  if (n >= (1ull << 31)) return fail(CS_ERR_LIMIT, "cs_fixed_base_mul: n too large");
  CS_CUDA(cudaSetDevice(ctx->device));
  const size_t pbytes = point_limbs64(curve, group) * 8;
  DevBuf dbase, dscal, dout;
  CS_TRY(dbase.reserve(pbytes));
  CS_TRY(dscal.reserve(n * 32));
  CS_TRY(dout.reserve(n * pbytes));
  CS_CUDA(cudaMemcpyAsync(dbase.p, h_base, pbytes, cudaMemcpyHostToDevice, ctx->stream));
  CS_CUDA(cudaMemcpyAsync(dscal.p, h_scalars, n * 32, cudaMemcpyHostToDevice, ctx->stream));
  CS_DISPATCH_CURVE(curve, {
    typedef typename Cfg::FrP FrP;
    if (group == CS_G1) {
      typedef typename GroupOf<Cfg, 0>::F F;
      CS_LAUNCH(k_fixed_base_mul<F COMMA FrP>, ceil_div(n, 128), 128, 0, ctx->stream, dbase.as<Affine<F>>(),
                dscal.as<uint32_t>(), (uint32_t)n, scalars_montgomery, dout.as<Affine<F>>());
    } else {
      typedef typename GroupOf<Cfg, 1>::F F;
      CS_LAUNCH(k_fixed_base_mul<F COMMA FrP>, ceil_div(n, 128), 128, 0, ctx->stream, dbase.as<Affine<F>>(),
                dscal.as<uint32_t>(), (uint32_t)n, scalars_montgomery, dout.as<Affine<F>>());
    }
  });
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(h_out, dout.p, n * pbytes, cudaMemcpyDeviceToHost, ctx->stream));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  dbase.release();
  dscal.release();
  dout.release();
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------- NTT
namespace cs {

template <class Cfg>
int domain_create_t(cs_ctx* ctx, unsigned log_n, const uint64_t* gen_mont, cs_domain* d) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HF;
  if (log_n > Cfg::TWO_ADICITY) return fail(CS_ERR_ARG, "Polynomial Degree too large");  // reduction.rs:87-89
  HF g;
  if (gen_mont) {
    memcpy(g.l, gen_mont, sizeof(g.l));
  } else {
    // Domain::new: arkworks' get_root_of_unity(n) = (GENERATOR^TRACE)^(2^(s - log_n)); GENERATOR = 5
    // (BN254 Fr) / 7 (BLS12-381 Fr).  Computed as GENERATOR^((r-1) >> log_n).
    uint64_t e[HF::N];
    for (int i = 0; i < HF::N; i++) e[i] = HF::modl(i);
    e[0] -= 1;
    for (unsigned s = 0; s < log_n; s++) {
      for (int i = 0; i < HF::N; i++) e[i] = (e[i] >> 1) | (i + 1 < HF::N ? (e[i + 1] << 63) : 0);
    }
    g = HF::from_u64(std::is_same<Cfg, Bn254Cfg>::value ? 5 : 7).pow(e, HF::N);
  }
  // sanity: g^(2^log_n) == 1 and g^(2^(log_n-1)) == -1
  {
    HF t = g;
    for (unsigned s = 0; s + 1 < log_n; s++) t = t.sqr();
    if (log_n >= 1) {
      if (t + HF::one() != HF::zero()) return fail(CS_ERR_ARG, "cs_domain_create: group_gen is not a primitive 2^%u-th root of unity", log_n);
    } else if (g != HF::one()) {
      return fail(CS_ERR_ARG, "cs_domain_create: group_gen must be 1 for a size-1 domain");
    }
  }
  d->log_n = log_n;
  d->group_gen.assign(g.l, g.l + HF::N);
  const size_t n = (size_t)1 << log_n;
  HF ninv = HF::from_u64(n).inverse();
  CS_TRY(d->inv_n.reserve(sizeof(HF)));
  CS_CUDA(cudaMemcpyAsync(d->inv_n.p, ninv.l, sizeof(HF), cudaMemcpyHostToDevice, ctx->stream));
  if (log_n >= 1) {
    const size_t half = n >> 1;
    HF ginv = g.inverse();
    std::vector<HF> pw(2 * 32);
    HF a = g, b = ginv;
    for (unsigned j = 0; j < 32; j++) {
      pw[j] = a;
      pw[32 + j] = b;
      a = a.sqr();
      b = b.sqr();
    }
    DevBuf dpw;
    CS_TRY(dpw.reserve(pw.size() * sizeof(HF)));
    CS_CUDA(cudaMemcpyAsync(dpw.p, pw.data(), pw.size() * sizeof(HF), cudaMemcpyHostToDevice, ctx->stream));
    CS_TRY(d->tw_fwd.reserve(half * sizeof(HF)));
    CS_TRY(d->tw_inv.reserve(half * sizeof(HF)));
    CS_LAUNCH(k_ntt_twiddles<FrP>, ceil_div(half, 256), 256, 0, ctx->stream, dpw.as<uint32_t>(), (uint32_t)half,
              d->tw_fwd.as<uint32_t>());
    CS_LAUNCH(k_ntt_twiddles<FrP>, ceil_div(half, 256), 256, 0, ctx->stream, dpw.as<uint32_t>() + 32 * FrP::N,
              (uint32_t)half, d->tw_inv.as<uint32_t>());
    CS_CUDA(cudaGetLastError());
    CS_CUDA(cudaStreamSynchronize(ctx->stream));
    dpw.release();
  } else {
    CS_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return 0;
}

int ntt_run(cs_ctx* ctx, const cs_domain* d, uint32_t* d_data, unsigned batch, bool inverse_in_to_out,
            const uint32_t* d_post, cudaStream_t st) {
  if (batch == 0) return fail(CS_ERR_ARG, "ntt: batch must be >= 1");
  if (d->log_n == 0) return 0;
  // CS_NTT_V2=1 selects the TMA-staged radix-8 pass (cs_ntt8.cuh).  Both passes are bound by the instruction mix of a
  // butterfly (one product + add + sub), not by the copies, and the TMA pass pays a tile set-up at small sizes, so the
  // bulk-copy staging buys nothing and the default stays the radix-2 pass.
  static int v2_env = -1;
  if (v2_env < 0) { const char* e = getenv("CS_NTT_V2"); v2_env = e ? atoi(e) : 0; }
  CS_DISPATCH_CURVE(d->curve, {
    typedef typename Cfg::FrP FrP;
    const uint32_t* twp = inverse_in_to_out ? d->tw_inv.as<uint32_t>() : d->tw_fwd.as<uint32_t>();
    const uint32_t* scale = (inverse_in_to_out && !d_post) ? d->inv_n.as<uint32_t>() : nullptr;
    if (v2_env && batch <= 2) {  // TMA-staged tiles + register radix-8 (cs_ntt8.cuh) from 2^12 on
      bool used = false;
      CS_TRY((ntt_enqueue8<FrP>(d_data, twp, d->log_n, batch, !inverse_in_to_out, d_post, scale, st, &used)));
      if (used) return 0;
    }
    return ntt_enqueue<FrP>(d_data, twp, d->log_n, batch, !inverse_in_to_out, d_post, scale, st);
  });
  return 0;
}

}  // namespace cs

extern "C" {

int cs_domain_create(cs_ctx* ctx, cs_curve curve, unsigned log_n, const uint64_t* group_gen_mont, cs_domain** out) {
  if (!ctx || !out) return fail(CS_ERR_ARG, "cs_domain_create: NULL argument");
  CS_CUDA(cudaSetDevice(ctx->device));
  std::unique_ptr<cs_domain> d(new cs_domain());
  d->curve = curve;
  CS_DISPATCH_CURVE(curve, { CS_TRY(domain_create_t<Cfg>(ctx, log_n, group_gen_mont, d.get())); });
  *out = d.release();
  return 0;
}

void cs_domain_free(cs_domain* d) {
  if (!d) return;
  d->tw_fwd.release();
  d->tw_inv.release();
  d->inv_n.release();
  delete d;
}

size_t cs_domain_size(const cs_domain* d) { return d ? ((size_t)1 << d->log_n) : 0; }

int cs_ifft_in_to_out(cs_ctx* ctx, const cs_domain* d, uint64_t* d_data, unsigned batch) {
  if (!ctx || !d || !d_data) return fail(CS_ERR_ARG, "cs_ifft_in_to_out: NULL argument");
  return ntt_run(ctx, d, reinterpret_cast<uint32_t*>(d_data), batch, true, nullptr, ctx->stream);
}
int cs_fft_out_to_in(cs_ctx* ctx, const cs_domain* d, uint64_t* d_data, unsigned batch) {
  if (!ctx || !d || !d_data) return fail(CS_ERR_ARG, "cs_fft_out_to_in: NULL argument");
  return ntt_run(ctx, d, reinterpret_cast<uint32_t*>(d_data), batch, false, nullptr, ctx->stream);
}

int cs_bit_reverse(cs_ctx* ctx, cs_curve curve, uint64_t* d_data, unsigned log_n, unsigned batch) {
  if (!ctx || !d_data) return fail(CS_ERR_ARG, "cs_bit_reverse: NULL argument");
  if (log_n > 31) return fail(CS_ERR_ARG, "cs_bit_reverse: log_n too large");
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_bit_reverse<typename Cfg::FrP>, ceil_div((size_t)1 << log_n, 256), 256, 0, ctx->stream,
              reinterpret_cast<uint32_t*>(d_data), log_n, batch);
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}

// natural-order transforms of co-plonk (`domain.fft / domain.ifft` on a Radix2EvaluationDomain with the
// snarkjs generator, co-plonk/src/mpc/rep3.rs:140-152, types.rs:76-100): the bit reversal the Groth16 path
// elides is applied explicitly.
int cs_fft(cs_ctx* ctx, const cs_domain* d, uint64_t* d_data, unsigned batch) {
  if (!ctx || !d || !d_data) return fail(CS_ERR_ARG, "cs_fft: NULL argument");
  CS_TRY(cs_bit_reverse(ctx, (cs_curve)d->curve, d_data, d->log_n, batch));
  return cs_fft_out_to_in(ctx, d, d_data, batch);
}
int cs_ifft(cs_ctx* ctx, const cs_domain* d, uint64_t* d_data, unsigned batch) {
  if (!ctx || !d || !d_data) return fail(CS_ERR_ARG, "cs_ifft: NULL argument");
  CS_TRY(cs_ifft_in_to_out(ctx, d, d_data, batch));
  return cs_bit_reverse(ctx, (cs_curve)d->curve, d_data, d->log_n, batch);
}

static int ntt_host(cs_ctx* ctx, const cs_domain* d, uint64_t* h_data, unsigned batch, bool inv) {
  if (!ctx || !d || !h_data) return fail(CS_ERR_ARG, "ntt host wrapper: NULL argument");
  size_t bytes = ((size_t)1 << d->log_n) * batch * 32;
  CS_TRY(ctx->io.reserve(bytes));
  CS_CUDA(cudaMemcpyAsync(ctx->io.p, h_data, bytes, cudaMemcpyHostToDevice, ctx->stream));
  CS_TRY(ntt_run(ctx, d, ctx->io.as<uint32_t>(), batch, inv, nullptr, ctx->stream));
  CS_CUDA(cudaMemcpyAsync(h_data, ctx->io.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return 0;
}
int cs_ifft_in_to_out_host(cs_ctx* ctx, const cs_domain* d, uint64_t* h_data, unsigned batch) {
  return ntt_host(ctx, d, h_data, batch, true);
}
int cs_fft_out_to_in_host(cs_ctx* ctx, const cs_domain* d, uint64_t* h_data, unsigned batch) {
  return ntt_host(ctx, d, h_data, batch, false);
}

// ------------------------------------------------------------------------------------------- vec
static int vec_binop(cs_ctx* ctx, cs_curve curve, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n, int op) {
  if (!ctx || !a || !b || !out) return fail(CS_ERR_ARG, "vec op: NULL argument");
  if (n == 0) return 0;
  unsigned blocks = ceil_div(n, 256);
  if (blocks > CS_NUM_SMS * 16) blocks = CS_NUM_SMS * 16;
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_vec_binop<typename Cfg::FrP>, blocks, 256, 0, ctx->stream, reinterpret_cast<const uint32_t*>(a),
              reinterpret_cast<const uint32_t*>(b), reinterpret_cast<uint32_t*>(out), n, op);
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}
int cs_vec_mul(cs_ctx* ctx, cs_curve curve, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
  return vec_binop(ctx, curve, a, b, out, n, VEC_MUL);
}
int cs_vec_add(cs_ctx* ctx, cs_curve curve, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
  return vec_binop(ctx, curve, a, b, out, n, VEC_ADD);
}
int cs_vec_sub(cs_ctx* ctx, cs_curve curve, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
  return vec_binop(ctx, curve, a, b, out, n, VEC_SUB);
}

int cs_vec_scale_table(cs_ctx* ctx, cs_curve curve, uint64_t* x, const uint64_t* table, size_t n, unsigned batch) {
  if (!ctx || !x || !table) return fail(CS_ERR_ARG, "cs_vec_scale_table: NULL argument");
  if (batch != 1 && batch != 2) return fail(CS_ERR_ARG, "cs_vec_scale_table: batch must be 1 or 2");
  if (n == 0) return 0;
  unsigned blocks = ceil_div(n * batch, 256);
  if (blocks > CS_NUM_SMS * 16) blocks = CS_NUM_SMS * 16;
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_vec_scale_table<typename Cfg::FrP>, blocks, 256, 0, ctx->stream, reinterpret_cast<uint32_t*>(x),
              reinterpret_cast<const uint32_t*>(table), n, batch);
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}

int cs_rep3_local_mul_vec(cs_ctx* ctx, cs_curve curve, const uint64_t* a, const uint64_t* b, const uint64_t* mask,
                          uint64_t* out, size_t n) {
  if (!ctx || !a || !b || !out) return fail(CS_ERR_ARG, "cs_rep3_local_mul_vec: NULL argument");
  if (n == 0) return 0;
  unsigned blocks = ceil_div(n, 256);
  if (blocks > CS_NUM_SMS * 16) blocks = CS_NUM_SMS * 16;
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_rep3_local_mul<typename Cfg::FrP>, blocks, 256, 0, ctx->stream, reinterpret_cast<const uint32_t*>(a),
              reinterpret_cast<const uint32_t*>(b), reinterpret_cast<const uint32_t*>(mask),
              (const uint32_t*)nullptr, reinterpret_cast<uint32_t*>(out), n);
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}

int cs_vec_lincomb(cs_ctx* ctx, cs_curve curve, const uint64_t* const* d_inputs, const uint64_t* h_weights_mont, unsigned k,
                   size_t n, uint64_t* d_out) {
  if (!ctx || !d_inputs || !h_weights_mont || !d_out) return fail(CS_ERR_ARG, "cs_vec_lincomb: NULL argument");
  if (k == 0 || k > LINCOMB_MAX) return fail(CS_ERR_ARG, "cs_vec_lincomb: k must be in [1, %u]", LINCOMB_MAX);
  if (n == 0) return 0;
  LincombArgs a;
  memset(&a, 0, sizeof(a));
  for (unsigned j = 0; j < k; j++) {
    if (!d_inputs[j]) return fail(CS_ERR_ARG, "cs_vec_lincomb: input %u is NULL", j);
    a.in[j] = reinterpret_cast<const uint32_t*>(d_inputs[j]);
    memcpy(a.w[j], h_weights_mont + 4 * j, 32);
  }
  unsigned blocks = ceil_div(n, 256);
  if (blocks > CS_NUM_SMS * 16) blocks = CS_NUM_SMS * 16;
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_vec_lincomb<typename Cfg::FrP>, blocks, 256, 0, ctx->stream, a, k, reinterpret_cast<uint32_t*>(d_out), n);
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}

// Rep3Rand::masking_field_elements_vec on the device (rngs.rs:137-156)
int cs_rep3_masks_device(cs_ctx* ctx, cs_curve curve, const uint8_t* h_seed1, uint64_t word_pos1, const uint8_t* h_seed2,
                         uint64_t word_pos2, unsigned rounds, size_t n, uint64_t* d_out) {
  if (!ctx || !h_seed1 || !h_seed2 || (n && !d_out)) return fail(CS_ERR_ARG, "cs_rep3_masks_device: NULL argument");
  if (rounds == 0 || (rounds & 1) || rounds > 20) return fail(CS_ERR_ARG, "cs_rep3_masks_device: rounds must be even, <= 20");
  if (n == 0) return 0;
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_TRY(ctx->prf_keys.reserve(64));
  uint8_t keys[64];
  memcpy(keys, h_seed1, 32);
  memcpy(keys + 32, h_seed2, 32);
  CS_CUDA(cudaMemcpyAsync(ctx->prf_keys.p, keys, 64, cudaMemcpyHostToDevice, ctx->stream));
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_rep3_masks<typename Cfg::FrP>, ceil_div(n, 128), 128, 0, ctx->stream, ctx->prf_keys.as<uint32_t>(),
              word_pos1, word_pos2, rounds, n, reinterpret_cast<uint32_t*>(d_out));
  });
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaStreamSynchronize(ctx->stream));  // `keys` is a stack buffer
  return 0;
}

// mul_vec = local_mul_vec + reshare_vec in one kernel over peer memory (arithmetic.rs:132-160)
int cs_rep3_mul_vec_reshare(cs_ctx* ctx, cs_curve curve, const uint64_t* d_a, const uint64_t* d_b, size_t n,
                            const cs_rep3_prf* prf, uint64_t* d_out, uint64_t* d_next_out) {
  if (!ctx || (n && (!d_a || !d_b || !d_out))) return fail(CS_ERR_ARG, "cs_rep3_mul_vec_reshare: NULL argument");
  if (prf && (prf->rounds == 0 || (prf->rounds & 1) || prf->rounds > 20))
    return fail(CS_ERR_ARG, "cs_rep3_mul_vec_reshare: rounds must be even, <= 20");
  if (n == 0) return 0;
  CS_CUDA(cudaSetDevice(ctx->device));
  PrfKeys keys;
  memset(&keys, 0, sizeof(keys));
  if (prf) {
    memcpy(keys.k, prf->seed1, 32);
    memcpy(keys.k + 8, prf->seed2, 32);
  }
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_rep3_mul_vec_reshare<typename Cfg::FrP>, ceil_div(n, 128), 128, 0, ctx->stream,
              reinterpret_cast<const uint32_t*>(d_a), reinterpret_cast<const uint32_t*>(d_b), keys,
              prf ? prf->word_pos1 : 0, prf ? prf->word_pos2 : 0, prf ? prf->rounds : 0u, n,
              reinterpret_cast<uint32_t*>(d_out), reinterpret_cast<uint32_t*>(d_next_out));
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}

int cs_rep3_set_b(cs_ctx* ctx, cs_curve curve, const uint64_t* d_recv, size_t n, uint64_t* d_out) {
  if (!ctx || (n && (!d_recv || !d_out))) return fail(CS_ERR_ARG, "cs_rep3_set_b: NULL argument");
  if (n == 0) return 0;
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_rep3_set_b<typename Cfg::FrP>, ceil_div(n, 256), 256, 0, ctx->stream,
              reinterpret_cast<const uint32_t*>(d_recv), n, reinterpret_cast<uint32_t*>(d_out));
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}

int cs_share_rep3_device(cs_ctx* ctx, cs_curve curve, const uint64_t* d_witness, size_t n, const uint8_t* h_seed32,
                         uint64_t* d_share0, uint64_t* d_share1, uint64_t* d_share2) {
  if (!ctx || (n && (!d_witness || !d_share0 || !d_share1 || !d_share2))) return fail(CS_ERR_ARG, "cs_share_rep3_device: NULL argument");
  if (n == 0) return 0;
  CS_CUDA(cudaSetDevice(ctx->device));
  uint8_t seed[32];
  if (h_seed32) memcpy(seed, h_seed32, 32); else CS_TRY(cs_os_random(seed, 32));
  PrfKey1 key;
  for (int i = 0; i < 8; i++) key.k[i] = (uint32_t)seed[4 * i] | ((uint32_t)seed[4 * i + 1] << 8) | ((uint32_t)seed[4 * i + 2] << 16) | ((uint32_t)seed[4 * i + 3] << 24);
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_share_rep3<typename Cfg::FrP>, ceil_div(n, 128), 128, 0, ctx->stream, key, 12u, Cfg::FR_BITS,
              reinterpret_cast<const uint32_t*>(d_witness), n, reinterpret_cast<uint32_t*>(d_share0),
              reinterpret_cast<uint32_t*>(d_share1), reinterpret_cast<uint32_t*>(d_share2));
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}

int cs_fr_rand_device(cs_ctx* ctx, cs_curve curve, const uint8_t* h_seed32, uint64_t stream_base, uint64_t* d_out, size_t n) {
  if (!ctx || (n && !d_out)) return fail(CS_ERR_ARG, "cs_fr_rand_device: NULL argument");
  if (n == 0) return 0;
  CS_CUDA(cudaSetDevice(ctx->device));
  uint8_t seed[32];
  if (h_seed32) memcpy(seed, h_seed32, 32); else CS_TRY(cs_os_random(seed, 32));
  PrfKey1 key;
  for (int i = 0; i < 8; i++) key.k[i] = (uint32_t)seed[4 * i] | ((uint32_t)seed[4 * i + 1] << 8) | ((uint32_t)seed[4 * i + 2] << 16) | ((uint32_t)seed[4 * i + 3] << 24);
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_fr_rand<typename Cfg::FrP>, ceil_div(n, 128), 128, 0, ctx->stream, key, stream_base, 12u, Cfg::FR_BITS, n,
              reinterpret_cast<uint32_t*>(d_out));
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}

int cs_rep3_batch(cs_ctx* ctx, cs_curve curve, cs_rep3_batch_op op, int party, const uint64_t* d_x, const uint64_t* d_y,
                  uint64_t* d_out, size_t n) {
  if (!ctx || (n && !d_out)) return fail(CS_ERR_ARG, "cs_rep3_batch: NULL argument");
  if ((int)op < 0 || (int)op > CS_R3B_PROMOTE) return fail(CS_ERR_ARG, "cs_rep3_batch: unknown op %d", (int)op);
  if (party < 0 || party > 2) return fail(CS_ERR_ARG, "cs_rep3_batch: party must be 0..2");
  if (n && op != CS_R3B_PROMOTE && !d_x) return fail(CS_ERR_ARG, "cs_rep3_batch: d_x is NULL");
  if (n && op != CS_R3B_NEG && !d_y) return fail(CS_ERR_ARG, "cs_rep3_batch: d_y is NULL");
  if (n == 0) return 0;
  CS_CUDA(cudaSetDevice(ctx->device));
  unsigned blocks = ceil_div(n, 256);
  if (blocks > CS_NUM_SMS * 16) blocks = CS_NUM_SMS * 16;
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_rep3_batch<typename Cfg::FrP>, blocks, 256, 0, ctx->stream, (int)op, party, reinterpret_cast<const uint32_t*>(d_x),
              reinterpret_cast<const uint32_t*>(d_y), reinterpret_cast<uint32_t*>(d_out), n);
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}

int cs_rep3_batch_open_send(cs_ctx* ctx, cs_curve curve, const uint64_t* d_shares, size_t n, uint64_t* d_next_recv) {
  if (!ctx || (n && (!d_shares || !d_next_recv))) return fail(CS_ERR_ARG, "cs_rep3_batch_open_send: NULL argument");
  if (n == 0) return 0;
  CS_CUDA(cudaSetDevice(ctx->device));
  unsigned blocks = ceil_div(n, 256);
  if (blocks > CS_NUM_SMS * 16) blocks = CS_NUM_SMS * 16;
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_rep3_take_b<typename Cfg::FrP>, blocks, 256, 0, ctx->stream, reinterpret_cast<const uint32_t*>(d_shares),
              reinterpret_cast<uint32_t*>(d_next_recv), n);
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}

int cs_rep3_batch_open_finish(cs_ctx* ctx, cs_curve curve, const uint64_t* d_shares, const uint64_t* d_recv,
                              uint64_t* d_out_public, size_t n) {
  if (!ctx || (n && (!d_shares || !d_recv || !d_out_public))) return fail(CS_ERR_ARG, "cs_rep3_batch_open_finish: NULL argument");
  if (n == 0) return 0;
  CS_CUDA(cudaSetDevice(ctx->device));
  unsigned blocks = ceil_div(n, 256);
  if (blocks > CS_NUM_SMS * 16) blocks = CS_NUM_SMS * 16;
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_rep3_batch<typename Cfg::FrP>, blocks, 256, 0, ctx->stream, (int)R3B_OPEN_FINISH, 0,
              reinterpret_cast<const uint32_t*>(d_shares), reinterpret_cast<const uint32_t*>(d_recv),
              reinterpret_cast<uint32_t*>(d_out_public), n);
  });
  CS_CUDA(cudaGetLastError());
  return 0;
}

// CoUtils::commit for a round of polynomials (co-noir-common/src/lib.rs:88-101 -> msm_public_points -> fast_msm)
int cs_honk_commit_batch(cs_ctx* ctx, const cs_bases* crs, cs_share_kind kind, const uint64_t* const* d_polys,
                         const size_t* lens, unsigned k, uint64_t* h_out) {
  if (!ctx || !crs || !d_polys || !lens || !h_out) return fail(CS_ERR_ARG, "cs_honk_commit_batch: NULL argument");
  if (kind != CS_PLAIN && kind != CS_REP3) return fail(CS_ERR_ARG, "cs_honk_commit_batch: bad share kind");
  const unsigned per = kind == CS_REP3 ? 2 : 1;
  if (k == 0 || k * per > (unsigned)CS_NSIDE) return fail(CS_ERR_ARG, "cs_honk_commit_batch: %u polynomials do not fit %d streams", k, CS_NSIDE);
  const size_t plimbs = point_limbs64(crs->curve, crs->group);
  for (unsigned j = 0; j < k; j++) {
    if (lens[j] > crs->n) return fail(CS_ERR_ARG, "cs_honk_commit_batch: polynomial %u has %zu coefficients, the CRS holds %zu points", j, lens[j], crs->n);
    if (lens[j] && !d_polys[j]) return fail(CS_ERR_ARG, "cs_honk_commit_batch: polynomial %u is NULL", j);
  }
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_TRY(ctx_fork(ctx, (int)(k * per)));
  for (unsigned j = 0; j < k; j++)
    for (unsigned c = 0; c < per; c++) {
      const unsigned slot = j * per + c;
      if (lens[j] == 0) continue;
      const uint32_t* sc = reinterpret_cast<const uint32_t*>(d_polys[j]) + c * 8;
      CS_TRY(msm_enqueue_dyn(ctx, (int)slot, ctx->side[slot], crs, 0, sc, per, lens[j], 1));
    }
  CS_TRY(ctx_join(ctx, (int)(k * per)));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  for (unsigned j = 0; j < k; j++)
    for (unsigned c = 0; c < per; c++) {
      const unsigned slot = j * per + c;
      uint64_t* dst = h_out + (size_t)slot * plimbs;
      if (lens[j] == 0) { memset(dst, 0, plimbs * 8); continue; }
      CS_TRY(msm_finish_dyn(ctx, (int)slot, crs, dst, nullptr));
    }
  return 0;
}

// peer mapping of another process's device buffer (one process per GPU): cudaIpc handles are 64 opaque bytes
int cs_ipc_export(cs_ctx* ctx, const void* d_ptr, uint8_t* out_handle64) {
  if (!ctx || !d_ptr || !out_handle64) return fail(CS_ERR_ARG, "cs_ipc_export: NULL argument");
  CS_CUDA(cudaSetDevice(ctx->device));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t h;
  CS_CUDA(cudaIpcGetMemHandle(&h, const_cast<void*>(d_ptr)));
  memcpy(out_handle64, &h, 64);
  return 0;
}
int cs_ipc_open(cs_ctx* ctx, const uint8_t* handle64, void** out_peer_ptr) {
  if (!ctx || !handle64 || !out_peer_ptr) return fail(CS_ERR_ARG, "cs_ipc_open: NULL argument");
  CS_CUDA(cudaSetDevice(ctx->device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  CS_CUDA(cudaIpcOpenMemHandle(out_peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}
int cs_ipc_close(cs_ctx* ctx, void* peer_ptr) {
  if (!ctx || !peer_ptr) return fail(CS_ERR_ARG, "cs_ipc_close: NULL argument");
  CS_CUDA(cudaSetDevice(ctx->device));
  CS_CUDA(cudaIpcCloseMemHandle(peer_ptr));
  return 0;
}

int cs_chacha_keystream(cs_ctx* ctx, const uint8_t* h_key, uint64_t first_block, unsigned rounds, unsigned nblocks,
                        uint32_t* h_out_words) {
  if (!ctx || !h_key || !h_out_words) return fail(CS_ERR_ARG, "cs_chacha_keystream: NULL argument");
  if (nblocks == 0) return 0;
  CS_TRY(ctx->io.reserve(32 + (size_t)nblocks * 64));
  CS_CUDA(cudaMemcpyAsync(ctx->io.p, h_key, 32, cudaMemcpyHostToDevice, ctx->stream));
  uint32_t* d_out = ctx->io.as<uint32_t>() + 8;
  CS_LAUNCH(k_chacha_keystream, ceil_div(nblocks, 64), 64, 0, ctx->stream, ctx->io.as<uint32_t>(), first_block, rounds,
            nblocks, d_out);
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaMemcpyAsync(h_out_words, d_out, (size_t)nblocks * 64, cudaMemcpyDeviceToHost, ctx->stream));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  return 0;
}

int cs_rep3_to_shamir(cs_ctx* ctx, cs_curve curve, const uint64_t* x, const uint64_t* h_ca, const uint64_t* h_cb,
                      uint64_t* out, size_t n) {
  if (!ctx || !x || !h_ca || !h_cb || !out) return fail(CS_ERR_ARG, "cs_rep3_to_shamir: NULL argument");
  if (n == 0) return 0;
  CS_TRY(ctx->io.reserve(64));
  CS_CUDA(cudaMemcpyAsync(ctx->io.p, h_ca, 32, cudaMemcpyHostToDevice, ctx->stream));
  CS_CUDA(cudaMemcpyAsync((char*)ctx->io.p + 32, h_cb, 32, cudaMemcpyHostToDevice, ctx->stream));
  unsigned blocks = ceil_div(n, 256);
  if (blocks > CS_NUM_SMS * 16) blocks = CS_NUM_SMS * 16;
  CS_DISPATCH_CURVE(curve, {
    CS_LAUNCH(k_rep3_to_shamir<typename Cfg::FrP>, blocks, 256, 0, ctx->stream, reinterpret_cast<const uint32_t*>(x),
              ctx->io.as<uint32_t>(), ctx->io.as<uint32_t>() + 8, reinterpret_cast<uint32_t*>(out), n);
  });
  CS_CUDA(cudaGetLastError());
  CS_CUDA(cudaStreamSynchronize(ctx->stream));  // io staging is reused by later calls
  return 0;
}

}  // extern "C"

namespace cs {
template <class Cfg>
int eval_poly_t(cs_ctx* ctx, const uint64_t* d_coeffs, size_t n, unsigned batch, const uint64_t* h_point, uint64_t* h_out) {
  typedef typename Cfg::FrP FrP;
  typedef host::HFp<FrP> HF;
  HF x;
  memcpy(x.l, h_point, sizeof(x.l));
  for (unsigned c = 0; c < batch; c++) memset(h_out + c * HF::N, 0, sizeof(x.l));
  if (n == 0) return 0;
  // table: point, then (point^POLY_CHUNK)^(2^j)
  std::vector<HF> tab(1 + 48);
  tab[0] = x;
  HF pc = x;
  for (unsigned k = 1; k < POLY_CHUNK; k <<= 1) pc = pc.sqr();  // POLY_CHUNK is a power of two
  for (int j = 0; j < 48; j++) { tab[1 + j] = pc; pc = pc.sqr(); }
  const unsigned threads = 128;
  const size_t nchunks = (n + POLY_CHUNK - 1) / POLY_CHUNK;
  const unsigned blocks = ceil_div(nchunks, threads);
  CS_TRY(ctx->io.reserve(tab.size() * sizeof(HF) + (size_t)blocks * batch * sizeof(HF)));
  uint32_t* d_tab = ctx->io.as<uint32_t>();
  uint32_t* d_sums = d_tab + tab.size() * FrP::N;
  CS_CUDA(cudaMemcpyAsync(d_tab, tab.data(), tab.size() * sizeof(HF), cudaMemcpyHostToDevice, ctx->stream));
  CS_LAUNCH_SYNC(k_poly_eval<FrP>, blocks, threads, (size_t)threads * batch * sizeof(HF), ctx->stream,
                 reinterpret_cast<const uint32_t*>(d_coeffs), n, batch, d_tab, d_tab + FrP::N, d_sums);
  CS_CUDA(cudaGetLastError());
  std::vector<HF> sums((size_t)blocks * batch);
  CS_CUDA(cudaMemcpyAsync(sums.data(), d_sums, sums.size() * sizeof(HF), cudaMemcpyDeviceToHost, ctx->stream));
  CS_CUDA(cudaStreamSynchronize(ctx->stream));
  for (unsigned c = 0; c < batch; c++) {
    HF acc = HF::zero();
    for (unsigned b = 0; b < blocks; b++) acc = acc + sums[(size_t)b * batch + c];
    memcpy(h_out + c * HF::N, acc.l, sizeof(acc.l));
  }
  return 0;
}
}  // namespace cs

extern "C" {
int cs_eval_poly(cs_ctx* ctx, cs_curve curve, const uint64_t* d_coeffs, size_t n, unsigned batch,
                 const uint64_t* h_point_mont, uint64_t* h_out) {
  if (!ctx || !h_point_mont || !h_out || (n && !d_coeffs)) return fail(CS_ERR_ARG, "cs_eval_poly: NULL argument");
  if (batch != 1 && batch != 2) return fail(CS_ERR_ARG, "cs_eval_poly: batch must be 1 or 2");
  CS_DISPATCH_CURVE(curve, { return eval_poly_t<Cfg>(ctx, d_coeffs, n, batch, h_point_mont, h_out); });
  return 0;
}

// ---------------------------------------------------------------------------- host-side helpers
}  // extern "C"

namespace cs {

template <class Cfg, int G>
int point_scalar_mul_t(const uint64_t* p, const uint64_t* s_mont, uint64_t* out) {
  typedef typename GroupOf<Cfg, G>::HF HF;
  typedef host::HFp<typename Cfg::FrP> HR;
  host::HAffine<HF> a;
  memcpy(&a, p, sizeof(a));
  HR s;
  memcpy(s.l, s_mont, sizeof(s.l));
  HR sc = s.from_mont();
  host::HAffine<HF> r = host::haffine(host::hmul(host::HXyzz<HF>::from_affine(a), sc.l, HR::N));
  memcpy(out, &r, sizeof(r));
  return 0;
}
template <class Cfg, int G>
int point_add_t(const uint64_t* p, const uint64_t* q, uint64_t* out) {
  typedef typename GroupOf<Cfg, G>::HF HF;
  host::HAffine<HF> a, b;
  memcpy(&a, p, sizeof(a));
  memcpy(&b, q, sizeof(b));
  host::HAffine<HF> r = host::haffine(host::hadd(host::HXyzz<HF>::from_affine(a), host::HXyzz<HF>::from_affine(b)));
  memcpy(out, &r, sizeof(r));
  return 0;
}
template <class Cfg, int G>
int point_neg_t(const uint64_t* p, uint64_t* out) {
  typedef typename GroupOf<Cfg, G>::HF HF;
  host::HAffine<HF> a;
  memcpy(&a, p, sizeof(a));
  a.y = a.y.neg();
  memcpy(out, &a, sizeof(a));
  return 0;
}
template <class P>
int field_conv(const uint64_t* in, uint64_t* out, size_t n, bool to_mont) {
  typedef host::HFp<P> HF;
  for (size_t i = 0; i < n; i++) {
    HF v;
    memcpy(v.l, in + i * HF::N, sizeof(v.l));
    HF r = to_mont ? v.to_mont() : v.from_mont();
    memcpy(out + i * HF::N, r.l, sizeof(r.l));
  }
  return 0;
}

// co-groth16/src/groth16.rs:60-100
template <class Cfg>
int roots_of_unity_t(unsigned pow, uint64_t* out_gen, uint64_t* out_shift) {
  typedef host::HFp<typename Cfg::FrP> HF;
  if (pow > Cfg::TWO_ADICITY) return fail(CS_ERR_ARG, "Polynomial Degree too large");
  // smallest quadratic non-residue: q^((r-1)/2) == -1
  uint64_t half[HF::N], trace[HF::N];
  for (int i = 0; i < HF::N; i++) half[i] = HF::modl(i);
  half[0] -= 1;
  memcpy(trace, half, sizeof(half));
  for (int i = 0; i < HF::N; i++) half[i] = (half[i] >> 1) | (i + 1 < HF::N ? (half[i + 1] << 63) : 0);
  for (unsigned s = 0; s < Cfg::TWO_ADICITY; s++)
    for (int i = 0; i < HF::N; i++) trace[i] = (trace[i] >> 1) | (i + 1 < HF::N ? (trace[i + 1] << 63) : 0);
  HF minus_one = HF::zero() - HF::one();
  uint64_t qv = 1;
  HF q = HF::from_u64(qv);
  while (q.pow(half, HF::N) != minus_one) q = HF::from_u64(++qv);
  // roots[k] = z^(2^(s-k)), z = q^TRACE
  HF z = q.pow(trace, HF::N);
  HF gen = z, shift;
  for (unsigned k = 0; k < Cfg::TWO_ADICITY - pow; k++) gen = gen.sqr();  // roots[pow]
  if (pow == Cfg::TWO_ADICITY) {
    shift = q.sqr();
  } else {
    shift = z;
    for (unsigned k = 0; k < Cfg::TWO_ADICITY - pow - 1; k++) shift = shift.sqr();  // roots[pow + 1]
  }
  memcpy(out_gen, gen.l, sizeof(gen.l));
  memcpy(out_shift, shift.l, sizeof(shift.l));
  return 0;
}

}  // namespace cs

extern "C" {

int cs_point_scalar_mul(cs_curve curve, cs_group group, const uint64_t* p, const uint64_t* s, uint64_t* out) {
  if (!p || !s || !out) return fail(CS_ERR_ARG, "cs_point_scalar_mul: NULL argument");
  CS_DISPATCH_CURVE(curve, {
    if (group == CS_G1) return point_scalar_mul_t<Cfg, 0>(p, s, out);
    return point_scalar_mul_t<Cfg, 1>(p, s, out);
  });
  return 0;
}
int cs_point_add(cs_curve curve, cs_group group, const uint64_t* p, const uint64_t* q, uint64_t* out) {
  if (!p || !q || !out) return fail(CS_ERR_ARG, "cs_point_add: NULL argument");
  CS_DISPATCH_CURVE(curve, {
    if (group == CS_G1) return point_add_t<Cfg, 0>(p, q, out);
    return point_add_t<Cfg, 1>(p, q, out);
  });
  return 0;
}
int cs_point_neg(cs_curve curve, cs_group group, const uint64_t* p, uint64_t* out) {
  if (!p || !out) return fail(CS_ERR_ARG, "cs_point_neg: NULL argument");
  CS_DISPATCH_CURVE(curve, {
    if (group == CS_G1) return point_neg_t<Cfg, 0>(p, out);
    return point_neg_t<Cfg, 1>(p, out);
  });
  return 0;
}
int cs_fr_to_mont(cs_curve curve, const uint64_t* in, uint64_t* out, size_t n) {
  CS_DISPATCH_CURVE(curve, { return field_conv<typename Cfg::FrP>(in, out, n, true); });
  return 0;
}
int cs_fr_from_mont(cs_curve curve, const uint64_t* in, uint64_t* out, size_t n) {
  CS_DISPATCH_CURVE(curve, { return field_conv<typename Cfg::FrP>(in, out, n, false); });
  return 0;
}
int cs_fq_to_mont(cs_curve curve, const uint64_t* in, uint64_t* out, size_t n) {
  CS_DISPATCH_CURVE(curve, { return field_conv<typename Cfg::FqP>(in, out, n, true); });
  return 0;
}
int cs_fq_from_mont(cs_curve curve, const uint64_t* in, uint64_t* out, size_t n) {
  CS_DISPATCH_CURVE(curve, { return field_conv<typename Cfg::FqP>(in, out, n, false); });
  return 0;
}
int cs_fr_mul(cs_curve curve, const uint64_t* a_mont, const uint64_t* b_mont, uint64_t* out_mont) {
  if (!a_mont || !b_mont || !out_mont) return fail(CS_ERR_ARG, "cs_fr_mul: NULL argument");
  CS_DISPATCH_CURVE(curve, {
    typedef host::HFp<typename Cfg::FrP> HF;
    HF a; HF b;
    memcpy(a.l, a_mont, sizeof(a.l));
    memcpy(b.l, b_mont, sizeof(b.l));
    HF r = a * b;
    memcpy(out_mont, r.l, sizeof(r.l));
  });
  return 0;
}
int cs_fr_inv(cs_curve curve, const uint64_t* a_mont, uint64_t* out_mont) {
  if (!a_mont || !out_mont) return fail(CS_ERR_ARG, "cs_fr_inv: NULL argument");
  CS_DISPATCH_CURVE(curve, {
    typedef host::HFp<typename Cfg::FrP> HF;
    HF a;
    memcpy(a.l, a_mont, sizeof(a.l));
    if (a.is_zero()) return fail(CS_ERR_ARG, "Cannot invert zero");
    HF r = a.inverse();
    memcpy(out_mont, r.l, sizeof(r.l));
  });
  return 0;
}
int cs_fr_add(cs_curve curve, const uint64_t* a_mont, const uint64_t* b_mont, uint64_t* out_mont) {
  if (!a_mont || !b_mont || !out_mont) return fail(CS_ERR_ARG, "cs_fr_add: NULL argument");
  CS_DISPATCH_CURVE(curve, {
    typedef host::HFp<typename Cfg::FrP> HF;
    HF a; HF b;
    memcpy(a.l, a_mont, sizeof(a.l));
    memcpy(b.l, b_mont, sizeof(b.l));
    HF r = a + b;
    memcpy(out_mont, r.l, sizeof(r.l));
  });
  return 0;
}
int cs_fr_sub(cs_curve curve, const uint64_t* a_mont, const uint64_t* b_mont, uint64_t* out_mont) {
  if (!a_mont || !b_mont || !out_mont) return fail(CS_ERR_ARG, "cs_fr_sub: NULL argument");
  CS_DISPATCH_CURVE(curve, {
    typedef host::HFp<typename Cfg::FrP> HF;
    HF a; HF b;
    memcpy(a.l, a_mont, sizeof(a.l));
    memcpy(b.l, b_mont, sizeof(b.l));
    HF r = a - b;
    memcpy(out_mont, r.l, sizeof(r.l));
  });
  return 0;
}
int cs_groth16_roots_of_unity(cs_curve curve, unsigned pow, uint64_t* out_gen, uint64_t* out_shift) {
  if (!out_gen || !out_shift) return fail(CS_ERR_ARG, "cs_groth16_roots_of_unity: NULL argument");
  CS_DISPATCH_CURVE(curve, { return roots_of_unity_t<Cfg>(pow, out_gen, out_shift); });
  return 0;
}

}  // extern "C"
