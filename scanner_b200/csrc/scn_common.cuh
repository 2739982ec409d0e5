// scn_common.cuh -- shared helpers for the sm_90a kernels behind include/scn_kernels.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "scn_kernels.h"

#define SCN_MAX_PTRS 64  // frames per launch; larger batches are chunked by the launcher

namespace scn {

// Frame pointers travel in the kernel parameter block (constant bank): no H2D copy, no
// allocation, and the host array can be freed as soon as the C call returns.
struct PtrBatch {
  const uint8_t* p[SCN_MAX_PTRS];
};
struct MutPtrBatch {
  uint8_t* p[SCN_MAX_PTRS];
};

extern std::atomic<uint64_t> g_launches;
inline void count_launch(uint64_t n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// RAII scope around one kernel launch: bumps the launch counter and, when profiling is enabled,
// brackets the launch with CUDA events on the launch stream (see scn_prof_* in cabi.cu).
void prof_begin(const char* name, cudaStream_t st, void** token);
void prof_end(void* token, cudaStream_t st);
extern std::atomic<int> g_prof_on;
struct LaunchScope {
  void* token = nullptr;
  cudaStream_t st;
  LaunchScope(const char* name, cudaStream_t s) : st(s) {
    count_launch();
    if (g_prof_on.load(std::memory_order_relaxed)) prof_begin(name, st, &token);
  }
  ~LaunchScope() {
    if (token) prof_end(token, st);
  }
};

inline int sm_count() {
  static int sms = [] {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0)
      return 132;
    return v;
  }();
  return sms;
}

inline int launch_status() {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    cudaGetLastError();  // clear the sticky launch error so later calls report their own
    return (int)e;
  }
  return 0;
}

// 128-bit streaming load: read-only path, do not allocate in L1 (each byte is used once).
__device__ __forceinline__ uint4 ld_stream_u4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t ld_stream_u32(const void* p) {
  uint32_t r;
  asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t r;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
  return r;
}

}  // namespace scn
