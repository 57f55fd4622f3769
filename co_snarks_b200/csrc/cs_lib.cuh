// Library internals shared by the C-ABI translation units: curve configs, context, handles.
#pragma once
#include <atomic>
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
};

struct cs_bases {
  int curve = 0, group = 0;
  size_t n = 0;
  cs::MsmShape sh{};
  cs::DevBuf table;    // W * n affine points
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
// (view) through a filtered view of the shared witness sort; see msm_enqueue
int msm_enqueue_dyn(cs_ctx* ctx, int slot, cudaStream_t st, const cs_bases* b, size_t offset,
                    const uint32_t* d_scalars, unsigned sstride, size_t n, int mont, int sort_slot = -1, bool view = false);
// Sort of n scalars into workspace `slot` without an infinity mask, entries w * n + i, in the window shape of b
int msm_sort_shared_dyn(cs_ctx* ctx, int slot, cudaStream_t st, const cs_bases* b, const uint32_t* d_scalars,
                        unsigned sstride, size_t n, int mont);
int msm_finish_dyn(cs_ctx* ctx, int slot, const cs_bases* b, uint64_t* out_affine, int* out_inf);
int ntt_run(cs_ctx* ctx, const cs_domain* d, uint32_t* d_data, unsigned batch, bool inverse_in_to_out,
            const uint32_t* d_post, cudaStream_t st);
}  // namespace cs
