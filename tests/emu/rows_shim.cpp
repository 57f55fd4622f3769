// Test shim (TEST INFRASTRUCTURE): uploads a base set or creates a Groth16 key with exactly k windows per table row
// (cs::bases_upload, cs::groth16_pk_create), where the public entry points pick k from the table budget.  The budget
// reaches only the smallest k of each row count, and on tiny keys, whose scratch grows with k faster than their tables
// shrink, only k = 1; this reaches every k.  Built by tests/test_strided_tables.py with g++ -DCS_EMU against the
// emulation library; the handles it returns are ordinary handles of that library.  heap_bytes_in_use: the emulation's
// "device" memory is the process heap, so a leaked device buffer shows there.
#include "cs_lib.cuh"
#include <malloc.h>

extern "C" int bases_upload_rows(cs_ctx* ctx, int curve, int group, const uint64_t* h_points_mont, size_t n, int window_bits,
                                 unsigned k, cs_bases** out) {
  return cs::bases_upload(ctx, (cs_curve)curve, (cs_group)group, h_points_mont, n, window_bits, k, out);
}

extern "C" int groth16_pk_create_rows(cs_ctx* ctx, const cs_groth16_key_desc* d, unsigned k, cs_groth16_pk** out) {
  return cs::groth16_pk_create(ctx, d, k, out);
}

extern "C" size_t heap_bytes_in_use() {
  const struct mallinfo2 m = mallinfo2();
  return m.uordblks + m.hblkhd;
}
