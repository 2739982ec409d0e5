// fused.cu -- BASELINE.json configs[1] on decoder surfaces, without the RGB24 intermediate:
//     NV12 -> RGB -> { Histogram (test_ops.cpp:19-49), Resize (test_ops.cpp:124-162) }
// The reference runs three passes over HBM (image.cu NV12_to_RGB writes 3WH bytes, the two ops
// read them back).  Here the surface (1.5 WH bytes) is the only large read: the histogram is
// taken from RGB values converted in registers, and the resize converts just the 4 taps of each
// destination pixel.  Results are bit-identical to the three-pass composition.
#include "nv12_stream.cuh"

#ifndef SCN_NV12_RESIZE_DEFAULT
#define SCN_NV12_RESIZE_DEFAULT kOverlap
#endif
#include "nv12_math.cuh"
#include "scn_common.cuh"

namespace scn {

struct Tap {
  int32_t i0, i1, w0, w1;
};
constexpr size_t kPlanHeaderBytes = 32;

namespace {

constexpr int HT = 256;
constexpr int HW = HT / 32;

// One thread converts 4 horizontally adjacent pixels of one row (32-bit luma + chroma loads) and
// bumps its warp's private bins.  grid = (x-chunks, row-groups, frames); each thread walks rows
// y = blockIdx.y, blockIdx.y + gridDim.y, ...
__global__ void __launch_bounds__(HT)
nv12_hist_kernel(PtrBatch lumas, PtrBatch chromas, size_t pitch, int width, int height,
                 int quads_per_row, int vec_ok, int32_t* __restrict__ out) {
  __shared__ int sh[HW][48];
  for (int i = threadIdx.x; i < HW * 48; i += HT) (&sh[0][0])[i] = 0;
  __syncthreads();
  int* h = sh[threadIdx.x >> 5];
  const uint8_t* __restrict__ luma = lumas.p[blockIdx.z];
  const uint8_t* __restrict__ chroma = chromas.p[blockIdx.z];
  const int q = blockIdx.x * HT + threadIdx.x;
  if (q < quads_per_row) {
    const int x0 = q * 4;
    for (int y = blockIdx.y; y < height; y += gridDim.y) {
      uint32_t yy[4], cb[2], cr[2];
      const int yc = y >> 1;
      const bool avg = (y & 1) && yc < ((height >> 1) - 1);
      if (vec_ok) {
        const uint32_t yw = ld_stream_u32(luma + (size_t)y * pitch + x0);
        const uint32_t cw = __ldg(reinterpret_cast<const uint32_t*>(chroma + (size_t)yc * pitch + x0));
        yy[0] = yw & 0xFF; yy[1] = (yw >> 8) & 0xFF; yy[2] = (yw >> 16) & 0xFF; yy[3] = yw >> 24;
        cb[0] = cw & 0xFF; cr[0] = (cw >> 8) & 0xFF; cb[1] = (cw >> 16) & 0xFF; cr[1] = cw >> 24;
        if (avg) {
          const uint32_t c2 =
              __ldg(reinterpret_cast<const uint32_t*>(chroma + (size_t)(yc + 1) * pitch + x0));
          cb[0] = (cb[0] + (c2 & 0xFF) + 1) >> 1;
          cr[0] = (cr[0] + ((c2 >> 8) & 0xFF) + 1) >> 1;
          cb[1] = (cb[1] + ((c2 >> 16) & 0xFF) + 1) >> 1;
          cr[1] = (cr[1] + (c2 >> 24) + 1) >> 1;
        }
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
          yy[i] = (x0 + i < width) ? luma[(size_t)y * pitch + x0 + i] : 0;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          cb[i] = cr[i] = 0;
          if (x0 + 2 * i < width) chroma_at(chroma, pitch, height, y, x0 + 2 * i, cb[i], cr[i]);
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (x0 + i < width) {
          const Rgb8 c = yuv_to_rgb(yy[i], cb[i >> 1], cr[i >> 1]);
          atomicAdd(&h[0 * 16 + (c.r >> 4)], 1);
          atomicAdd(&h[1 * 16 + (c.g >> 4)], 1);
          atomicAdd(&h[2 * 16 + (c.b >> 4)], 1);
        }
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < 48) {
    int s = 0;
#pragma unroll
    for (int w = 0; w < HW; ++w) s += sh[w][threadIdx.x];
    if (s) atomicAdd(&out[(size_t)blockIdx.z * 48 + threadIdx.x], s);
  }
}

__global__ void __launch_bounds__(256)
nv12_resize_kernel(PtrBatch lumas, PtrBatch chromas, size_t pitch, int width, int height,
                   MutPtrBatch dst, const uint8_t* __restrict__ plan, int dw, int dh,
                   int area2x) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= dw * dh) return;
  const int dy = idx / dw, dx = idx - dy * dw;
  const uint8_t* __restrict__ luma = lumas.p[blockIdx.y];
  const uint8_t* __restrict__ chroma = chromas.p[blockIdx.y];
  uint8_t* o = dst.p[blockIdx.y] + (size_t)idx * 3;
  if (area2x) {
    const Rgb8 a = nv12_pixel(luma, chroma, pitch, height, 2 * dx, 2 * dy);
    const Rgb8 b = nv12_pixel(luma, chroma, pitch, height, 2 * dx + 1, 2 * dy);
    const Rgb8 c = nv12_pixel(luma, chroma, pitch, height, 2 * dx, 2 * dy + 1);
    const Rgb8 d = nv12_pixel(luma, chroma, pitch, height, 2 * dx + 1, 2 * dy + 1);
    o[0] = (uint8_t)((a.r + b.r + c.r + d.r + 2) >> 2);
    o[1] = (uint8_t)((a.g + b.g + c.g + d.g + 2) >> 2);
    o[2] = (uint8_t)((a.b + b.b + c.b + d.b + 2) >> 2);
    return;
  }
  // Instruction-bound: four exact NV12 -> RGB conversions per destination pixel.  Two leaner-looking forms were measured and were not faster: the XU-converting tap chain of
  // nv12_stream.cuh (46 us instead of 37 us per 64 frames) and a row-organised kernel (a CTA per destination row,
  // uniform row addresses, u16 chroma loads, chroma terms computed once per sample, mulhi blend: 312 static
  // instructions, the same 37 us).
  const Tap* __restrict__ xt = reinterpret_cast<const Tap*>(plan + kPlanHeaderBytes);
  const Tap* __restrict__ yt = xt + dw;
  const int4 tx = __ldg(reinterpret_cast<const int4*>(xt + dx));
  const int4 ty = __ldg(reinterpret_cast<const int4*>(yt + dy));
  const Rgb8 p00 = nv12_pixel(luma, chroma, pitch, height, tx.x, ty.x);
  const Rgb8 p01 = nv12_pixel(luma, chroma, pitch, height, tx.y, ty.x);
  const Rgb8 p10 = nv12_pixel(luma, chroma, pitch, height, tx.x, ty.y);
  const Rgb8 p11 = nv12_pixel(luma, chroma, pitch, height, tx.y, ty.y);
  const int a0 = tx.z, a1 = tx.w, b0 = ty.z, b1 = ty.w;
  auto blend = [&](uint32_t v00, uint32_t v01, uint32_t v10, uint32_t v11) {
    const int h0 = (int)v00 * a0 + (int)v01 * a1, h1 = (int)v10 * a0 + (int)v11 * a1;
    return (uint8_t)((((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2);
  };
  o[0] = blend(p00.r, p01.r, p10.r, p11.r);
  o[1] = blend(p00.g, p01.g, p10.g, p11.g);
  o[2] = blend(p00.b, p01.b, p10.b, p11.b);
}

// Histogram and Resize of the configs[1] DAG are independent readers of the same surfaces: the
// histogram kernel is bound by instruction issue (one persistent CTA per SM, most registers), the
// resize kernel too, at far fewer registers per thread.  When both are requested the resize runs on a
// side stream forked from / joined to the caller's stream with events, so its CTAs share the SMs
// with the histogram CTAs instead of queueing behind them.  One side stream per calling thread
// and device (pipeline instances call from their own threads).
struct SideStream {
  int dev = -1;
  cudaStream_t stream = nullptr;
  cudaEvent_t fork = nullptr, join = nullptr;
  ~SideStream() {
    // the owning thread is going away; the context may already be gone at process exit
    if (stream) {
      cudaEventDestroy(fork);
      cudaEventDestroy(join);
      cudaStreamDestroy(stream);
      cudaGetLastError();
    }
  }
};

SideStream* side_stream() {
  static thread_local SideStream side[16];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return nullptr;
  SideStream& s = side[dev];
  if (!s.stream) {
    if (cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&s.join, cudaEventDisableTiming) != cudaSuccess) {
      cudaGetLastError();
      s.stream = nullptr;
      return nullptr;
    }
    s.dev = dev;
  }
  return &s;
}

}  // namespace
}  // namespace scn

extern "C" int scn_nv12_hist_resize(const uint8_t* const* host_luma_ptrs,
                                    const uint8_t* const* host_chroma_ptrs, size_t pitch, int n,
                                    int width, int height, int32_t* hist_out,
                                    uint8_t* const* host_dst_ptrs, int dst_w, int dst_h,
                                    const void* plan, void* stream) {
  using namespace scn;
  if (n < 0 || width <= 0 || height <= 0 || (width & 1) || (height & 1) || pitch < (size_t)width)
    return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!host_luma_ptrs || !host_chroma_ptrs) return SCN_E_BADARG;
  const bool do_hist = hist_out != nullptr;
  const bool do_resize = host_dst_ptrs != nullptr;
  if (!do_hist && !do_resize) return SCN_E_BADARG;
  const bool area2x = do_resize && (width == 2 * dst_w && height == 2 * dst_h);
  if (do_resize && (dst_w <= 0 || dst_h <= 0)) return SCN_E_BADARG;
  if (do_resize && !area2x && !plan) return SCN_E_PLAN;
  cudaStream_t st = (cudaStream_t)stream;
  if (do_hist) {
    cudaError_t e = cudaMemsetAsync(hist_out, 0, (size_t)n * 48 * sizeof(int32_t), st);
    if (e != cudaSuccess) return (int)e;
  }
  const int quads = (width + 3) / 4;
  // Large aligned surfaces take the one-pass streaming kernel (nv12_stream.cuh): histogram and, when
  // both are wanted, the Resize rows of every span right behind it.  Everything else (tiny, ragged or
  // unaligned surfaces; Resize alone) runs the generic kernels below.
  bool stream_ok = do_hist;
  for (int i0 = 0; i0 < n && stream_ok; i0 += SCN_MAX_PTRS) {
    const int cnt = (n - i0 < SCN_MAX_PTRS) ? (n - i0) : SCN_MAX_PTRS;
    stream_ok = nvs::eligible(host_luma_ptrs + i0, host_chroma_ptrs + i0, cnt, pitch, width, height);
  }
  // How Histogram + Resize of the same surfaces run (SCN_NV12_RESIZE):
  //   fused    the Resize rows are produced inside the streaming pass (one HBM read of the surface);
  //   split    streaming histogram kernel, then nv12_resize_kernel behind it on the same stream;
  //   overlap  nv12_resize_kernel on a side stream next to the streaming kernel.
  enum { kFused, kSplit, kOverlap };
  static const int resize_mode = [] {
    const char* e = getenv("SCN_NV12_RESIZE");
    if (e && e[0] == 'f') return (int)kFused;
    if (e && e[0] == 'o') return (int)kOverlap;
    if (e && e[0] == 's') return (int)kSplit;
    return (int)SCN_NV12_RESIZE_DEFAULT;
  }();
  // (the exact-2x Resize, an INTER_AREA average, is not produced inside the streaming pass)
  if (stream_ok && !(do_resize && (resize_mode != kFused || area2x)))
    return nvs::launch(host_luma_ptrs, host_chroma_ptrs, n, pitch, width, height, hist_out, do_resize ? host_dst_ptrs : nullptr,
                       (do_resize && !area2x) ? (const uint8_t*)plan + kPlanHeaderBytes : nullptr, dst_w, dst_h, area2x ? 1 : 0, st);
  SideStream* side = nullptr;
  cudaStream_t rst = st;
  if (stream_ok && do_resize && resize_mode == kOverlap && (side = side_stream()) != nullptr) {
    // fork before the histogram kernel is enqueued so both kernels can be resident together
    if (cudaEventRecord(side->fork, st) != cudaSuccess || cudaStreamWaitEvent(side->stream, side->fork, 0) != cudaSuccess) {
      cudaGetLastError();
      side = nullptr;
    } else {
      rst = side->stream;
    }
  }
  if (stream_ok) {
    const int rc0 = nvs::launch(host_luma_ptrs, host_chroma_ptrs, n, pitch, width, height, hist_out, nullptr, nullptr, 0, 0, 0, st);
    if (rc0) return rc0;
  }
  const bool hist_done = stream_ok;
  // generic path: the resize kernels of this call go to the side stream (see SideStream)
  if (!hist_done && do_hist && do_resize && (side = side_stream()) != nullptr) {
    if (cudaEventRecord(side->fork, st) != cudaSuccess || cudaStreamWaitEvent(side->stream, side->fork, 0) != cudaSuccess) {
      cudaGetLastError();
      side = nullptr;
    } else {
      rst = side->stream;
    }
  }
  int rc = 0;
  for (int i0 = 0; i0 < n && rc == 0; i0 += SCN_MAX_PTRS) {
    const int cnt = (n - i0 < SCN_MAX_PTRS) ? (n - i0) : SCN_MAX_PTRS;
    PtrBatch l, c;
    MutPtrBatch d;
    int vec_ok = ((pitch & 3) == 0);
    for (int i = 0; i < cnt; ++i) {
      l.p[i] = host_luma_ptrs[i0 + i];
      c.p[i] = host_chroma_ptrs[i0 + i];
      d.p[i] = do_resize ? host_dst_ptrs[i0 + i] : nullptr;
      if (((uintptr_t)l.p[i] | (uintptr_t)c.p[i]) & 3) vec_ok = 0;
    }
    if (do_hist && !hist_done) {
      const int gx = (quads + HT - 1) / HT;
      int gy = (sm_count() * 8 + gx * cnt - 1) / (gx * cnt);
      if (gy < 1) gy = 1;
      if (gy > height) gy = height;
      dim3 grid((unsigned)gx, (unsigned)gy, (unsigned)cnt);
      {
        LaunchScope ls("nv12_hist_kernel", st);
        nv12_hist_kernel<<<grid, HT, 0, st>>>(l, c, pitch, width, height, quads, vec_ok, hist_out + (size_t)i0 * 48);
      }
      rc = launch_status();
      if (rc) break;
    }
    if (do_resize) {
      dim3 g2((unsigned)((dst_w * dst_h + 255) / 256), (unsigned)cnt);
      {
        LaunchScope ls("nv12_resize_kernel", rst);
        nv12_resize_kernel<<<g2, 256, 0, rst>>>(l, c, pitch, width, height, d, (const uint8_t*)plan, dst_w, dst_h,
                                              area2x ? 1 : 0);
      }
      rc = launch_status();
    }
  }
  // join, also on the error path: the caller's stream must not run ahead of the side stream
  if (side) {
    if (cudaEventRecord(side->join, side->stream) != cudaSuccess || cudaStreamWaitEvent(st, side->join, 0) != cudaSuccess) {
      cudaGetLastError();
      cudaStreamSynchronize(side->stream);
    }
  }
  return rc;
}
