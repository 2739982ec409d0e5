// scn_common.cuh -- shared helpers for the sm_90a kernels behind include/scn_kernels.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <map>
#include <mutex>
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

// ---- entropy coders' shared pieces (jpeg.cu, h264_enc.cu) ----

// Appends bits MSB first to a frame's bit stream of big-endian 32-bit words.  The first and the last word a
// writer touches may be shared with the neighbouring writers (MCUs, macroblocks) and are ORed in; the words between
// are its own.
struct BitWriter {
  uint32_t* words;
  uint64_t word;  // index of the word being filled
  uint64_t acc;   // the low n bits are pending
  int n;
  bool first;
  __device__ BitWriter(uint32_t* w, uint64_t bit) : words(w), word(bit >> 5), acc(0), n((int)(bit & 31)), first(true) {}
  __device__ __forceinline__ void put(uint32_t bits, int len) {  // len <= 27
    acc = (acc << len) | bits;
    n += len;
    if (n >= 32) {
      n -= 32;
      const uint32_t v = __byte_perm((uint32_t)(acc >> n), 0, 0x0123);
      if (first) atomicOr(words + word, v);
      else words[word] = v;
      first = false;
      ++word;
    }
  }
  __device__ __forceinline__ void finish() {
    if (n) atomicOr(words + word, __byte_perm((uint32_t)(acc << (32 - n)), 0, 0x0123));
  }
};

// block-wide exclusive scan of one value per thread (blockDim.x a multiple of 32, at most 1024); returns the
// exclusive prefix, *total the block's sum.  Every thread of the block calls it.
template <class T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* total) {
  __shared__ T warp_sums[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xFFFFFFFFu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    T s = lane < nw ? warp_sums[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T y = __shfl_up_sync(0xFFFFFFFFu, s, o);
      if (lane >= o) s += y;
    }
    warp_sums[lane] = s;  // inclusive
  }
  __syncthreads();
  const T before = wid ? warp_sums[wid - 1] : 0;
  *total = warp_sums[nw - 1];
  __syncthreads();  // warp_sums is reused by the next call
  return before + x - v;
}

// ---- the encoders' device scratch: a stream-ordered pool per device, kept by the library ----
inline cudaMemPool_t scratch_pool() {
  static std::mutex mu;
  static std::map<int, cudaMemPool_t> pools;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  auto it = pools.find(dev);
  if (it != pools.end()) return it->second;
  cudaMemPoolProps props = {};
  props.allocType = cudaMemAllocationTypePinned;
  props.location.type = cudaMemLocationTypeDevice;
  props.location.id = dev;
  cudaMemPool_t pool = nullptr;
  if (cudaMemPoolCreate(&pool, &props) != cudaSuccess) return nullptr;
  uint64_t keep = ~0ull;  // keep freed scratch for the next call instead of returning it at every synchronisation
  cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  pools[dev] = pool;
  return pool;
}

struct Scratch {
  cudaStream_t st;
  std::vector<void*> held;
  ~Scratch() {
    for (void* p : held) cudaFreeAsync(p, st);
  }
  template <class T>
  T* get(size_t count, cudaMemPool_t pool) {
    void* p = nullptr;
    if (cudaMallocFromPoolAsync(&p, count * sizeof(T) + 16, pool, st) != cudaSuccess) return nullptr;
    held.push_back(p);
    return static_cast<T*>(p);
  }
};

}  // namespace scn
