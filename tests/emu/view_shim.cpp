// Host-side test shim for the filtered view of the shared witness sort (TEST INFRASTRUCTURE): runs, on the emulated
// kernels of cs_msm.cuh, the per-table masked sort and msm_view over the unmasked sort of the same BN254 scalars, and
// exports both bucket-sorted entry lists for ctypes.  Linked against the emulation library (tests/emu/build_emu.py).
#include "cs_msm.cuh"  // first: the standard headers it pulls in precede cs_emu.h's macros
#include "cs_params.cuh"
using namespace cs;

// scalars: n x 8 u32 (canonical); infmask: bits of the table's nbases bases; window c.
// out_*: count[B + 1] then the entries (table slot | sign) grouped by bucket, room for W n entries; 0, or -1 on an
// error.  masked = the table's own sort, view = msm_view of the unmasked sort.
extern "C" int view_vs_masked(uint32_t n, const uint32_t* scalars, uint32_t c, uint32_t nbases, uint32_t offset,
                               const uint32_t* infmask, uint32_t* out_masked, uint32_t* out_view) {
  const MsmShape sh = msm_shape(254, c);
  const MsmSizes z(sh, n);
  MsmWorkspace shared, masked, view;
  DevBuf d_scal, d_mask;
  if (d_scal.reserve((size_t)n * 32) || d_mask.reserve(((nbases + 31) / 32) * 4)) return -1;
  memcpy(d_scal.p, scalars, (size_t)n * 32);
  memcpy(d_mask.p, infmask, ((nbases + 31) / 32) * 4);
  if (msm_sort<Bn254Fr>(shared, nullptr, n, sh, 0, d_scal.as<uint32_t>(), 1, n, 0, nullptr)) return -1;
  if (msm_sort<Bn254Fr>(masked, d_mask.as<uint32_t>(), nbases, sh, offset, d_scal.as<uint32_t>(), 1, n, 0, nullptr)) return -1;
  if (msm_view(view, shared, d_mask.as<uint32_t>(), nbases, sh, offset, n, nullptr)) return -1;
  MsmWorkspace* ws[2] = {&masked, &view};
  uint32_t* out[2] = {out_masked, out_view};
  for (int k = 0; k < 2; k++) {
    const MsmSortBufs q(*ws[k], z);
    memcpy(out[k], q.count, z.nb1 * 4);
    memcpy(out[k] + z.nb1, ws[k]->sorted.p, (size_t)q.start[z.nb1] * 4);
  }
  shared.release(); masked.release(); view.release();
  d_scal.release(); d_mask.release();
  return 0;
}
