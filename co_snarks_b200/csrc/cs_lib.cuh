// Library internals shared by the C-ABI translation units: curve configs, context, handles.
#pragma once
#include <atomic>
#include <functional>
#include <map>
#include <memory>
#include "cs_common.cuh"
#include "cs_params.cuh"
#include "cs_curve.cuh"
#include "cs_msm.cuh"
#include "cs_msm52.cuh"
#include "cs_ntt.cuh"
#include "cs_ntt8.cuh"
#include "cs_vec.cuh"
#include "cs_prf.cuh"
#include "cs_host_field.h"
#include "../../include/cosnarks_gpu.h"

namespace cs {

struct Bn254Cfg {
  typedef Bn254Fq FqP;
  typedef Bn254Fr FrP;
  static constexpr unsigned FR_BITS = 254;
  static constexpr unsigned TWO_ADICITY = 28;
};
struct Bls381Cfg {
  typedef Bls381Fq FqP;
  typedef Bls381Fr FrP;
  static constexpr unsigned FR_BITS = 255;
  static constexpr unsigned TWO_ADICITY = 32;
};

template <class Cfg, int G> struct GroupOf;
template <class Cfg> struct GroupOf<Cfg, 0> {
  typedef Fp<typename Cfg::FqP> F;
  typedef host::HFp<typename Cfg::FqP> HF;
};
template <class Cfg> struct GroupOf<Cfg, 1> {
  typedef Fp2<typename Cfg::FqP> F;
  typedef host::HFp2<typename Cfg::FqP> HF;
};

static inline size_t fq_limbs64(int curve) { return curve == CS_BN254 ? 4 : 6; }
static inline size_t point_limbs64(int curve, int group) { return fq_limbs64(curve) * (group == CS_G1 ? 2 : 4); }

constexpr int CS_NSIDE = 5;
constexpr int CS_WIT_SORT = CS_NSIDE;  // msm_ws slot of the witness sort shared by Groth16's A, B1, B2 and L MSMs

}  // namespace cs

struct cs_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cudaStream_t side[cs::CS_NSIDE] = {};
  cudaStream_t acc[cs::CS_NSIDE] = {};   // lower priority: the MSM accumulation kernels (see msm_enqueue's st_acc)
  cudaStream_t wm = nullptr;             // highest priority: witness map -> H MSM chain of the Groth16 prover
  cudaEvent_t ev_wm = nullptr;
  cudaEvent_t ev_fork = nullptr;
  cudaEvent_t ev_t0 = nullptr;  // timing event at the last fork, recorded only while MSM profiling is on (cs_msm_timeline_ms)
  cudaEvent_t ev_side[cs::CS_NSIDE] = {};
  cs::MsmWorkspace msm_ws[cs::CS_NSIDE + 1];  // one per side stream, + the shared witness sort (CS_WIT_SORT)
  cs::DevBuf io;  // staging for host-buffer convenience calls
  cs::DevBuf prf_keys;
  cs::DevBuf sc_part, sc_res;  // sumcheck round: per-block partial sums and the 16 results (reused across rounds)
  size_t table_budget = 0;     // cs_ctx_set_table_budget: cap on the device bytes a new key's tables may take, 0 = none
};

struct cs_bases {
  int curve = 0, group = 0;
  size_t n = 0;
  cs::MsmShape sh{};
  cs::DevBuf table;    // T * n affine points: T = sh.T rows of one per sh.k windows
  cs::DevBuf infmask;  // 1 bit per base: point at infinity
  bool m260 = false;   // table coordinates are in the radix-2^260 Montgomery form: accumulate on the FP64 pipe (cs_msm52.cuh)
};

struct cs_domain {
  int curve = 0;
  unsigned log_n = 0;
  cs::DevBuf tw_fwd, tw_inv;  // n/2 twiddles each
  cs::DevBuf inv_n;           // 1/n (one element)
  std::vector<uint64_t> group_gen;  // Montgomery
};

#if defined(CS_ENABLE_BLS12_381)
#define CS_CASE_BLS(...)   \
  case CS_BLS12_381: {     \
    typedef Bls381Cfg Cfg; \
    __VA_ARGS__;           \
  } break;
#else
#define CS_CASE_BLS(...)
#endif

#define CS_DISPATCH_CURVE(curve, ...)                                        \
  switch ((int)(curve)) {                                                    \
    case CS_BN254: {                                                         \
      typedef Bn254Cfg Cfg;                                                  \
      __VA_ARGS__;                                                           \
    } break;                                                                 \
      CS_CASE_BLS(__VA_ARGS__)                                               \
    default:                                                                 \
      return cs::fail(CS_ERR_ARG, "unsupported curve id %d", (int)(curve));      \
  }


namespace cs {
std::atomic<uint64_t>& launch_counter();
int ctx_fork(cs_ctx* ctx, int nside);
int ctx_join(cs_ctx* ctx, int nside);
// sort_slot >= 0: the MSM reads the sort last enqueued in that workspace slot over the same scalars -- as it is, or
// (view) through a filtered view of the shared witness sort; see msm_enqueue.  K > 1: a batch of K MSMs, proof p's
// scalar i at (i sstride + p pstride) elements; K results in the workspace.
int msm_enqueue_dyn(cs_ctx* ctx, int slot, cudaStream_t st, const cs_bases* b, size_t offset,
                    const uint32_t* d_scalars, unsigned sstride, size_t n, int mont, int sort_slot = -1, bool view = false,
                    unsigned K = 1, size_t pstride = 0);
// Sort of n scalars (K vectors of them) into workspace `slot` without an infinity mask, entries w * n + i, in the
// window shape of b
int msm_sort_shared_dyn(cs_ctx* ctx, int slot, cudaStream_t st, const cs_bases* b, const uint32_t* d_scalars,
                        unsigned sstride, size_t n, int mont, unsigned K = 1, size_t pstride = 0);
int msm_finish_dyn(cs_ctx* ctx, int slot, const cs_bases* b, uint64_t* out_affine, int* out_inf);

// widest window an MSM can run: msm_scan takes 2^20 bucket slots, 2^(c-1) buckets plus bucket 0
constexpr unsigned MSM_MAX_WINDOW = 20;
static_assert((1u << (MSM_MAX_WINDOW - 1)) + 1 <= MSM_SCAN_MAX_BLOCKS * MSM_SCAN_T, "MSM_MAX_WINDOW exceeds the scan");

// Table rows.  A key's MSM tables keep one row per k windows (MsmShape); k is the smallest whose device bytes fit the
// budget: what cudaMemGetInfo reports free less TABLE_MARGIN (the CUDA runtime's own allocations), capped by
// cs_ctx_set_table_budget.  k = 1 (full tables) whenever they fit.
constexpr size_t TABLE_MARGIN = 256ull << 20;
// reusable: bytes the caller holds and would free before allocating (a batch's scratch as it grows)
int table_budget(cs_ctx* ctx, size_t* out, size_t reusable = 0);
// smallest k in 1..W with need(k) <= budget, or CS_ERR_LIMIT stating the bytes needed at k = W and the budget
int pick_table_rows(cs_ctx* ctx, unsigned c, unsigned W, const std::function<size_t(unsigned)>& need, const char* who,
                    unsigned* k_out);
// device bytes of an uploaded base set of n points in shape sh
template <class Cfg, int G>
size_t bases_bytes(size_t n, const MsmShape& sh) {
  return DevBuf::alloc_size((size_t)sh.T * n * sizeof(Affine<typename GroupOf<Cfg, G>::F>)) + DevBuf::alloc_size(((n + 31) / 32) * 4);
}
// cs_bases_upload with k windows per table row, or k = 0: chosen by pick_table_rows for this base set alone
int bases_upload(cs_ctx* ctx, cs_curve curve, cs_group group, const uint64_t* h_points_mont, size_t n, int window_bits,
                 unsigned k, cs_bases** out);
// cs_groth16_pk_create with k windows per table row for all five tables, or k = 0: chosen by pick_table_rows
int groth16_pk_create(cs_ctx* ctx, const cs_groth16_key_desc* d, unsigned k, cs_groth16_pk** out);
int ntt_run(cs_ctx* ctx, const cs_domain* d, uint32_t* d_data, unsigned batch, bool inverse_in_to_out,
            const uint32_t* d_post, cudaStream_t st);
}  // namespace cs
