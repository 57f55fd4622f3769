// Host-side test shim for the MSM bucket sort (TEST INFRASTRUCTURE): runs msm_sort of cs_msm.cuh on BN254 scalars and
// exports count[], start[] and the bucket-sorted entries for ctypes.  Built twice by tests/test_msm_bucket_sort.py: with
// g++ -DCS_EMU against the emulation library (tests/emu/build_emu.py), and with nvcc -x cu for sm_90a.
#include "cs_msm.cuh"  // first: the standard headers it pulls in precede cs_emu.h's macros
#include "cs_params.cuh"
#include <stdarg.h>
using namespace cs;

#if !defined(CS_EMU)
// the stand-alone device build links no library: the three host helpers cs_common.cuh declares
namespace cs {
std::atomic<uint64_t>& launch_counter() { static std::atomic<uint64_t> c{0}; return c; }
std::string& last_error() { static thread_local std::string e; return e; }
int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  last_error() = buf;
  return code;
}
}  // namespace cs
#endif

// scalars: n scalars of sstride x 8 u32 each (the first 8 words of each are sorted); infmask: bits of nbases bases
// or null; window c.  out_count[B + 1], out_start[B + 2], out_sorted: room for W n entries.  0, or -1 on an error.
extern "C" int bucket_sort(uint32_t n, const uint32_t* scalars, uint32_t sstride, int mont, uint32_t c, uint32_t nbases,
                           uint32_t offset, const uint32_t* infmask, uint32_t* out_count, uint32_t* out_start,
                           uint32_t* out_sorted) {
  const MsmShape sh = msm_shape(254, c);
  const MsmSizes z(sh, n);
  MsmWorkspace ws;
  DevBuf d_scal, d_mask;
  const size_t mask_bytes = ((size_t)(nbases + 31) / 32) * 4;
  if (d_scal.reserve((size_t)n * sstride * 32) || d_mask.reserve(mask_bytes)) return -1;
  if (cudaMemcpy(d_scal.p, scalars, (size_t)n * sstride * 32, cudaMemcpyHostToDevice) != cudaSuccess) return -1;
  if (infmask && cudaMemcpy(d_mask.p, infmask, mask_bytes, cudaMemcpyHostToDevice) != cudaSuccess) return -1;
  if (msm_smem_optin<Bn254Fr>()) return -1;
  int rc = msm_sort<Bn254Fr>(ws, infmask ? d_mask.as<uint32_t>() : nullptr, nbases, sh, offset, d_scal.as<uint32_t>(),
                             sstride, n, mont, nullptr);
  if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = -1;
  if (!rc) {
    const MsmSortBufs q(ws, z);
    uint32_t total = 0;
    if (cudaMemcpy(out_count, q.count, z.nb1 * 4, cudaMemcpyDeviceToHost) ||
        cudaMemcpy(out_start, q.start, (z.nb1 + 1) * 4, cudaMemcpyDeviceToHost) ||
        cudaMemcpy(&total, q.start + z.nb1, 4, cudaMemcpyDeviceToHost) ||
        cudaMemcpy(out_sorted, ws.sorted.p, (size_t)total * 4, cudaMemcpyDeviceToHost))
      rc = -1;
  }
  ws.release();
  d_scal.release();
  d_mask.release();
  return rc;
}
