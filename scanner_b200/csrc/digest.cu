// digest.cu -- scn_frame_digest: 16-byte integer fingerprint of device buffers (include/scn_kernels.h).
// Streaming read with 128-bit loads, 64-bit accumulators per thread, one warp-shuffle reduction and two
// atomics per warp; grid = 4 CTAs per SM striding over the words of all buffers.
#include "scn_common.cuh"

namespace scn {
namespace {

__global__ void __launch_bounds__(256)
frame_digest_kernel(PtrBatch bufs, int n, uint64_t words, unsigned long long* __restrict__ out) {
  for (int f = blockIdx.y; f < n; f += gridDim.y) {
    const uint32_t* __restrict__ w = reinterpret_cast<const uint32_t*>(bufs.p[f]);
    // words before the first 16-byte boundary, then 16-byte groups, then the tail
    const uint64_t head = min(words, (uint64_t)(((16u - (uint32_t)(reinterpret_cast<uintptr_t>(w) & 15u)) & 15u) / 4u));
    const uint64_t quads = (words - head) / 4;
    const uint4* __restrict__ q = reinterpret_cast<const uint4*>(w + head);
    unsigned long long s1 = 0, s2 = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < quads; i += (uint64_t)gridDim.x * blockDim.x) {
      const uint4 v = ld_stream_u4(q + i);
      const uint64_t k = head + 4 * i;
      s1 += (unsigned long long)v.x + v.y + v.z + v.w;
      s2 += (unsigned long long)v.x * ((k + 0) % 65521u + 1) + (unsigned long long)v.y * ((k + 1) % 65521u + 1) +
            (unsigned long long)v.z * ((k + 2) % 65521u + 1) + (unsigned long long)v.w * ((k + 3) % 65521u + 1);
    }
    if (blockIdx.x == 0) {  // at most 3 head and 3 tail words
      const uint64_t tail0 = head + 4 * quads;
      uint64_t k = words;
      if (threadIdx.x < head) k = threadIdx.x;
      else if (threadIdx.x >= 32 && tail0 + (threadIdx.x - 32) < words) k = tail0 + (threadIdx.x - 32);
      if (k < words) {
        s1 += w[k];
        s2 += (unsigned long long)w[k] * (k % 65521u + 1);
      }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, d);
      s2 += __shfl_xor_sync(0xffffffffu, s2, d);
    }
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(&out[2 * f], s1);
      atomicAdd(&out[2 * f + 1], s2);
    }
  }
}

}  // namespace
}  // namespace scn

extern "C" int scn_frame_digest(const uint8_t* const* host_ptrs, int n, size_t bytes, uint64_t* out, void* stream) {
  using namespace scn;
  if (n < 0 || (bytes & 3) || (n > 0 && (!host_ptrs || !out))) return SCN_E_BADARG;
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(out, 0, (size_t)n * 16, st);
  if (e != cudaSuccess) return (int)e;
  for (int i0 = 0; i0 < n; i0 += SCN_MAX_PTRS) {
    const int cnt = (n - i0 < SCN_MAX_PTRS) ? (n - i0) : SCN_MAX_PTRS;
    PtrBatch b;
    for (int i = 0; i < cnt; ++i) {
      b.p[i] = host_ptrs[i0 + i];
      if (reinterpret_cast<uintptr_t>(b.p[i]) & 3) return SCN_E_BADARG;
    }
    dim3 grid((unsigned)(sm_count() * 4 / (cnt < 4 ? cnt : 4) + 1), (unsigned)(cnt < 4 ? cnt : 4));
    {
      LaunchScope ls("frame_digest_kernel", st);
      frame_digest_kernel<<<grid, 256, 0, st>>>(b, cnt, bytes / 4, reinterpret_cast<unsigned long long*>(out) + 2 * i0);
    }
    const int rc = launch_status();
    if (rc) return rc;
  }
  return 0;
}
