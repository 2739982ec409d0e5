// hist.cu -- 16-bin x 3-channel histogram of u8 HWC frames (sm_90a).
// Replaces HistogramKernelCPU::execute (reference tests/test_ops.cpp:19-49): bin = v >> 4 per
// channel, int32[3][16] channel-major per frame.  Integer, bit-exact.
//
// Two kernels share the entry points:
//   hist16_generic_kernel  any pointer alignment / any size; per-warp privatised shared-memory
//                          bins.  Used for small or oddly aligned frames.
//   (the bit-sliced streaming kernel for large frames lives in hist_csa.cuh)
#include "scn_common.cuh"
#include "hist_csa.cuh"

namespace scn {

namespace {

constexpr int kGenThreads = 256;
constexpr int kGenWarps = kGenThreads / 32;

template <int PHASE>
__device__ __forceinline__ void bump16(int* h, uint4 v) {
  // byte b of the vector belongs to channel (PHASE + b) % 3
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int ch = (PHASE + 4 * j + k) % 3;
      const uint32_t bin = (w[j] >> (8 * k + 4)) & 0xF;
      atomicAdd(&h[ch * 16 + bin], 1);
    }
  }
}

__global__ void __launch_bounds__(kGenThreads)
hist16_generic_kernel(PtrBatch frames, size_t nbytes, int32_t* __restrict__ out) {
  __shared__ int sh[kGenWarps][48];
  const int warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < kGenWarps * 48; i += kGenThreads) (&sh[0][0])[i] = 0;
  __syncthreads();

  const uint8_t* base = frames.p[blockIdx.y];
  int* h = sh[warp];
  const size_t mis = (size_t)(reinterpret_cast<uintptr_t>(base) & 15);
  size_t head = (16 - mis) & 15;
  if (head > nbytes) head = nbytes;
  const size_t nvec = (nbytes - head) / 16;
  const size_t tail0 = head + nvec * 16;

  const size_t gtid = (size_t)blockIdx.x * kGenThreads + threadIdx.x;
  const size_t gstride = (size_t)gridDim.x * kGenThreads;

  // head + tail bytes (at most 30) -- first block only
  if (blockIdx.x == 0) {
    const size_t nscalar = head + (nbytes - tail0);
    for (size_t i = threadIdx.x; i < nscalar; i += kGenThreads) {
      const size_t o = i < head ? i : tail0 + (i - head);
      atomicAdd(&h[(int)(o % 3) * 16 + (base[o] >> 4)], 1);
    }
  }
  const uint8_t* vbase = base + head;
  for (size_t v = gtid; v < nvec; v += gstride) {
    const uint4 d = ld_stream_u4(vbase + v * 16);
    const int phase = (int)((head + v * 16) % 3);
    if (phase == 0) bump16<0>(h, d);
    else if (phase == 1) bump16<1>(h, d);
    else bump16<2>(h, d);
  }
  __syncthreads();
  if (threadIdx.x < 48) {
    int s = 0;
#pragma unroll
    for (int w = 0; w < kGenWarps; ++w) s += sh[w][threadIdx.x];
    if (s) atomicAdd(&out[(size_t)blockIdx.y * 48 + threadIdx.x], s);
  }
}

int launch_hist(const uint8_t* const* ptrs, int n, int width, int height, int32_t* out,
                cudaStream_t st) {
  if (n < 0 || width < 0 || height < 0 || (n > 0 && (!ptrs || !out))) return SCN_E_BADARG;
  if (n == 0) return 0;
  const size_t nbytes = (size_t)width * height * 3;
  cudaError_t e = cudaMemsetAsync(out, 0, (size_t)n * 48 * sizeof(int32_t), st);
  if (e != cudaSuccess) return (int)e;
  if (nbytes == 0) return 0;

  return for_each_chunk(n, [&](int i0, int cnt) {
    const PtrBatch pb = gather<PtrBatch>(ptrs, i0, cnt);
    int32_t* o = out + (size_t)i0 * 48;
    if (csa::eligible(ptrs, i0, cnt, nbytes)) return csa::launch(pb, cnt, nbytes, o, st);
    // grid.x: enough 256-thread blocks to give every thread ~8 vectors, capped so the whole
    // launch is a few waves of the SM array.
    size_t want = (nbytes / 16 + (size_t)kGenThreads * 8 - 1) / ((size_t)kGenThreads * 8);
    if (want < 1) want = 1;
    size_t cap = (size_t)(sm_count() * 8 + cnt - 1) / cnt;
    if (cap < 1) cap = 1;
    dim3 grid((unsigned)(want < cap ? want : cap), (unsigned)cnt);
    return launch_kernel("hist16_generic_kernel", st,
                         [&] { hist16_generic_kernel<<<grid, kGenThreads, 0, st>>>(pb, nbytes, o); });
  });
}

}  // namespace
}  // namespace scn

extern "C" int scn_hist16_u8c3(const uint8_t* const* host_frame_ptrs, int n, int width,
                               int height, int32_t* out, void* stream) {
  return scn::launch_hist(host_frame_ptrs, n, width, height, out, (cudaStream_t)stream);
}

extern "C" int scn_hist16_u8c3_strided(const uint8_t* base, size_t stride_bytes, int n,
                                       int width, int height, int32_t* out, void* stream) {
  if (n < 0) return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!base) return SCN_E_BADARG;
  return scn::launch_hist(scn::strided(base, stride_bytes, n).data(), n, width, height, out, (cudaStream_t)stream);
}
