// Shared host-side plumbing: error handling, launch macros, context and device buffers.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>
#include "cs_prims.cuh"

#if !defined(CS_EMU)
#define CS_LAUNCH(kernel, grid, block, smem, stream, ...)          \
  do {                                                             \
    cs::launch_counter()++;                                        \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);    \
  } while (0)
#define CS_LAUNCH_SYNC CS_LAUNCH
#define CS_DYN_SMEM(type, name)                                  \
  extern __shared__ __align__(16) unsigned char name##_raw_[];   \
  type* name = reinterpret_cast<type*>(name##_raw_)
#endif

#define COMMA ,

// SMs of an H100 SXM; grid-stride kernels cap their grids at a small multiple of it.
#define CS_NUM_SMS 132

// NVTX ranges named after the reference's `tracing` spans (co-groth16/src/groth16.rs:230-313,
// groth16/reduction.rs:98-184), so an nsys / ncu --nvtx timeline of a proof reads like the reference's
// trace output.  No-ops in the emulation build; near-free when no tool is attached.
#if defined(CS_EMU)
struct CsNvtxRange { explicit CsNvtxRange(const char*) {} };
#else
#include <nvtx3/nvToolsExt.h>
struct CsNvtxRange {
  explicit CsNvtxRange(const char* name) { nvtxRangePushA(name); }
  ~CsNvtxRange() { nvtxRangePop(); }
  CsNvtxRange(const CsNvtxRange&) = delete;
};
#endif
#define CS_NVTX_CAT2(a, b) a##b
#define CS_NVTX_CAT(a, b) CS_NVTX_CAT2(a, b)
#define CS_SPAN(name) CsNvtxRange CS_NVTX_CAT(cs_span_, __LINE__)(name)

namespace cs {

std::atomic<uint64_t>& launch_counter();

// thread-local last error (returned by cs_last_error())
std::string& last_error();
int fail(int code, const char* fmt, ...);

#define CS_CUDA(expr)                                                                         \
  do {                                                                                        \
    cudaError_t e_ = (expr);                                                                  \
    if (e_ != cudaSuccess)                                                                    \
      return cs::fail(-2, "CUDA error %d (%s) at %s:%d: %s", (int)e_, cudaGetErrorString(e_), \
                      __FILE__, __LINE__, #expr);                                             \
  } while (0)

#define CS_TRY(expr)          \
  do {                        \
    int rc_ = (expr);         \
    if (rc_ != 0) return rc_; \
  } while (0)

static inline unsigned ceil_div(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }

// Growable device buffer (never shrinks; reused across calls so the proof loop does no cudaMalloc).
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + (bytes >> 3) + 256;
    CS_CUDA(cudaMalloc(&p, want));
    cap = want;
    return 0;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

}  // namespace cs
