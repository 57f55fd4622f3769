// Shamir(n, t) routines on device vectors, shared by the translation units that run Shamir provers (definitions in
// cs_shamir.cu).  All vectors are Montgomery Fr, one element per share.
#pragma once
#include "cs_lib.cuh"

namespace cs {

// A DevBuf released when it goes out of scope (DevBuf itself is a plain handle), so early returns cannot leak it.
struct ScopedBuf : DevBuf {
  ScopedBuf() = default;
  ScopedBuf(const ScopedBuf&) = delete;
  ScopedBuf& operator=(const ScopedBuf&) = delete;
  ~ScopedBuf() { release(); }
};

// Device and host staging of the vector routines below, owned by a cs_shamir_state and reused from call to call (no
// per-call cudaMalloc / zeroed host vectors of the reduced vectors' size); it only grows.  A copy starts empty, so a
// forked state never shares or frees its parent's buffers.
struct ShamirWorkspace {
  ScopedBuf coef, rcv, msg;            // double sharings: dealing coefficients, received shares, one outgoing dealing
  ScopedBuf acc, stage[LINCOMB_MAX];   // degree reduction (king) and openings: Lagrange sum, received vectors
  std::vector<uint64_t> h0, h1;        // host staging for cs_net
  ShamirWorkspace() = default;
  ShamirWorkspace(const ShamirWorkspace&) {}
  ShamirWorkspace& operator=(const ShamirWorkspace&) { return *this; }
  uint64_t* host0(size_t words) { if (h0.size() < words) h0.resize(words); return h0.data(); }
  uint64_t* host1(size_t words) { if (h1.size() < words) h1.resize(words); return h1.data(); }
  size_t device_bytes() const {
    size_t b = coef.cap + rcv.cap + msg.cap + acc.cap;
    for (const ScopedBuf& s : stage) b += s.cap;
    return b;
  }
};

// device memory a state's workspace holds
size_t shamir_state_device_bytes(const cs_shamir_state* st);

// `count` fresh DN07 double sharings (r_t, r_2t) straight into the device vectors d_rt, d_r2t (count elements each).
// Dealing coefficients come from k_fr_rand under a fresh 32-byte seed from the state's ChaCha stream per dealing round.
int shamir_double_sharings(cs_ctx* ctx, cs_shamir_state* st, cs_net* net, size_t count, uint64_t* d_rt, uint64_t* d_r2t);
// degree_reduce_many with the pairs d_rt, d_r2t (len elements each); d_r2t is overwritten, d_in may equal d_out
int shamir_degree_reduce(cs_ctx* ctx, cs_shamir_state* st, cs_net* net, const uint64_t* d_in, size_t len, uint64_t* d_out,
                         const uint64_t* d_rt, uint64_t* d_r2t);
// open_vec of a degree-t (degree_2t = 0) or degree-2t sharing: send to the next d parties, then the Lagrange sum on
// the device; d_in may equal d_out
int shamir_open_vec(cs_ctx* ctx, cs_shamir_state* st, cs_net* net, int degree_2t, const uint64_t* d_in, size_t len, uint64_t* d_out);
// open_vec on `k` host scalars, in place
int shamir_open_scalars(cs_shamir_state* st, cs_net* net, int degree_2t, uint64_t* v, size_t k);
// open_point_many on `k` affine points (Montgomery), in place
int shamir_open_points(cs_shamir_state* st, cs_net* net, cs_group group, int degree_2t, uint64_t* pts, size_t k);

}  // namespace cs
