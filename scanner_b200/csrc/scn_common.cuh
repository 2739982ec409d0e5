// scn_common.cuh -- shared helpers for the sm_90a kernels behind include/scn_kernels.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <vector>

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

// ---- the host side every batched entry point shares ----

// Calls launch(i0, cnt) for each run [i0, i0 + cnt) of at most SCN_MAX_PTRS frames of a batch of n, in order, and
// returns the first nonzero status; the runs after it are not enqueued.
template <class F>
inline int for_each_chunk(int n, F&& launch) {
  for (int i0 = 0; i0 < n; i0 += SCN_MAX_PTRS) {
    const int rc = launch(i0, n - i0 < SCN_MAX_PTRS ? n - i0 : SCN_MAX_PTRS);
    if (rc) return rc;
  }
  return 0;
}

// Pointers [i0, i0 + cnt) of a host array (cnt <= SCN_MAX_PTRS) as a PtrBatch or MutPtrBatch.
template <class Batch, class P>
inline Batch gather(const P* ptrs, int i0, int cnt) {
  Batch b;
  for (int i = 0; i < cnt; ++i) b.p[i] = ptrs[i0 + i];
  return b;
}

// Whether pointers [i0, i0 + cnt) of every host array are multiples of `align` (a power of two) bytes.
template <class... P>
inline bool aligned(uintptr_t align, int i0, int cnt, const P*... arrays) {
  uintptr_t bits = 0;
  for (int i = i0; i < i0 + cnt; ++i) bits |= (reinterpret_cast<uintptr_t>(arrays[i]) | ...);
  return (bits & (align - 1)) == 0;
}

// base, base + stride, ... : n frames of a dense batch as a host pointer array.
template <class T>
inline std::vector<T*> strided(T* base, size_t stride, int n) {
  std::vector<T*> p((size_t)n);
  for (int i = 0; i < n; ++i) p[i] = base + (size_t)i * stride;
  return p;
}

// Enqueues one launch under `name` (the launch counter and scn_prof_* see it by that name) and returns its status.
template <class F>
inline int launch_kernel(const char* name, cudaStream_t st, F&& enqueue) {
  {
    LaunchScope ls(name, st);
    enqueue();
  }
  return launch_status();
}

// Raises `kernel`'s dynamic shared-memory limit to `bytes` on the current device.  Function attributes belong to a
// device's context, so this is done once per (kernel, device); safe to call from any thread.  Each kernel is given
// one limit.
int raise_smem_limit(const void* kernel, size_t bytes);

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
