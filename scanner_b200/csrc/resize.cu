// resize.cu -- bilinear resize of u8 HWC 3-channel frames with OpenCV's fixed-point semantics.
// Replaces ResizeKernel::execute (reference tests/test_ops.cpp:124-162), whose arithmetic is
// cv::resize(..., INTER_LINEAR) on CV_8UC3 (OpenCV modules/imgproc/src/resize.cpp):
//   horizontal: H = S[sx]*a0 + S[sx+1]*a1              (a = rint(w * 2048), int accum)
//   vertical:   D = (((b0*(H0>>4))>>16) + ((b1*(H1>>4))>>16) + 2) >> 2
//   exact 2x downscale in both axes is re-routed to the 2x2 box average (INTER_AREA fast path).
// The coefficient tables ("plan") are computed on the host with the same float expressions
// OpenCV uses and handed to the kernel, so host and device cannot round differently.
#include <limits.h>
#include <math.h>
#include <string.h>

#include "resize_plan.cuh"
#include "scn_common.cuh"

namespace scn {
namespace {

constexpr int32_t kPlanMagic = 0x5243504c;  // "LPCR"

// cv::resize's INTER_LINEAR table for one axis; with `area`, the taps INTER_AREA uses when a scale is below 1.
void fill_taps(int ssz, int dsz, bool zero_weight_clamp, bool area, Tap* t) {
  const double inv_scale = (double)dsz / (double)ssz;
  const double scale = 1.0 / inv_scale;
  for (int d = 0; d < dsz; ++d) {
    float f;
    int s;
    if (area) {
      s = (int)floor(d * scale);
      f = (float)((d + 1) - (s + 1) * inv_scale);
      f = f <= 0 ? 0.f : f - floorf(f);
    } else {
      f = (float)((d + 0.5) * scale - 0.5);
      s = (int)floorf(f);
      f -= (float)s;
    }
    if (zero_weight_clamp) {
      // x axis: out-of-range taps collapse onto the edge pixel with weight (2048, 0)
      if (s < 0) { f = 0.f; s = 0; }
      if (s >= ssz - 1) { f = 0.f; s = ssz - 1; }
    }
    const float c0 = (1.f - f) * 2048.f;
    const float c1 = f * 2048.f;
    t[d].w0 = (int32_t)(short)lrintf(c0);
    t[d].w1 = (int32_t)(short)lrintf(c1);
    // y axis keeps its fractional weights and clamps the two ROW indices instead
    int i0 = s, i1 = s + 1;
    i0 = i0 < 0 ? 0 : (i0 > ssz - 1 ? ssz - 1 : i0);
    i1 = i1 < 0 ? 0 : (i1 > ssz - 1 ? ssz - 1 : i1);
    t[d].i0 = i0;
    t[d].i1 = i1;
  }
}

// One thread per destination pixel (3 channels); grid.y = frame.
__global__ void __launch_bounds__(256)
resize_linear_kernel(PtrBatch src, MutPtrBatch dst, const uint8_t* __restrict__ plan, int sw,
                     int dw, int dh) {
  const Tap* __restrict__ xt = reinterpret_cast<const Tap*>(plan + sizeof(PlanHeader));
  const Tap* __restrict__ yt = xt + dw;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= dw * dh) return;
  const int dy = idx / dw, dx = idx - dy * dw;
  const int4 tx = __ldg(reinterpret_cast<const int4*>(xt + dx));
  const int4 ty = __ldg(reinterpret_cast<const int4*>(yt + dy));
  const uint8_t* __restrict__ s = src.p[blockIdx.y];
  const uint8_t* r0 = s + (size_t)ty.x * sw * 3;
  const uint8_t* r1 = s + (size_t)ty.y * sw * 3;
  uint8_t* o = dst.p[blockIdx.y] + (size_t)idx * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int h0 = (int)__ldg(r0 + tx.x * 3 + c) * tx.z + (int)__ldg(r0 + tx.y * 3 + c) * tx.w;
    const int h1 = (int)__ldg(r1 + tx.x * 3 + c) * tx.z + (int)__ldg(r1 + tx.y * 3 + c) * tx.w;
    o[c] = (uint8_t)((((ty.z * (h0 >> 4)) >> 16) + ((ty.w * (h1 >> 4)) >> 16) + 2) >> 2);
  }
}

__global__ void __launch_bounds__(256)
resize_area2x_kernel(PtrBatch src, MutPtrBatch dst, int sw, int dw, int dh) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= dw * dh) return;
  const int dy = idx / dw, dx = idx - dy * dw;
  const uint8_t* __restrict__ r0 = src.p[blockIdx.y] + ((size_t)(2 * dy) * sw + 2 * dx) * 3;
  const uint8_t* __restrict__ r1 = r0 + (size_t)sw * 3;
  uint8_t* o = dst.p[blockIdx.y] + (size_t)idx * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int v = (int)__ldg(r0 + c) + (int)__ldg(r0 + 3 + c) + (int)__ldg(r1 + c) +
                  (int)__ldg(r1 + 3 + c);
    o[c] = (uint8_t)((v + 2) >> 2);
  }
}

}  // namespace

// Shared with fused.cu: validate a device plan's geometry cannot be done without a D2H copy, so
// the launchers trust `plan` to be the device copy of a buffer filled for exactly these sizes.
int launch_resize(const uint8_t* const* sp, int n, int sw, int sh, uint8_t* const* dp, int dw,
                  int dh, const void* plan, cudaStream_t st) {
  if (n < 0 || sw <= 0 || sh <= 0 || dw <= 0 || dh <= 0) return SCN_E_BADARG;
  // the kernels index destination pixels with an int
  if ((int64_t)dw * dh > INT_MAX) return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!sp || !dp) return SCN_E_BADARG;
  const bool area2x = (sw == 2 * dw && sh == 2 * dh);
  if (!area2x && !plan) return SCN_E_PLAN;
  return for_each_chunk(n, [&](int i0, int cnt) {
    const PtrBatch s = gather<PtrBatch>(sp, i0, cnt);
    const MutPtrBatch d = gather<MutPtrBatch>(dp, i0, cnt);
    dim3 grid((unsigned)(((int64_t)dw * dh + 255) / 256), (unsigned)cnt);
    if (area2x)
      return launch_kernel("resize_area2x_kernel", st,
                           [&] { resize_area2x_kernel<<<grid, 256, 0, st>>>(s, d, sw, dw, dh); });
    return launch_kernel("resize_linear_kernel", st, [&] {
      resize_linear_kernel<<<grid, 256, 0, st>>>(s, d, (const uint8_t*)plan, sw, dw, dh);
    });
  });
}

}  // namespace scn

extern "C" void scn_resize_target(int src_w, int src_h, int arg_w, int arg_h, int arg_min,
                                  int arg_preserve_aspect, int* out_w, int* out_h) {
  // reference tests/test_ops.cpp:126-147
  int tw = arg_w, th = arg_h;
  if (arg_preserve_aspect) {
    if (tw == 0)
      tw = src_h ? src_w * th / src_h : 0;
    else
      th = src_w ? src_h * tw / src_w : 0;
  }
  if (arg_min && src_w <= tw && src_h <= th) {
    tw = src_w;
    th = src_h;
  }
  if (out_w) *out_w = tw;
  if (out_h) *out_h = th;
}

extern "C" size_t scn_resize_plan_bytes(int dst_w, int dst_h) {
  if (dst_w <= 0 || dst_h <= 0) return 0;
  return sizeof(scn::PlanHeader) + sizeof(scn::Tap) * ((size_t)dst_w + (size_t)dst_h);
}

void scn::fill_linear_plan(int src_w, int src_h, int dst_w, int dst_h, bool area, void* host_plan) {
  scn::PlanHeader h;
  memset(&h, 0, sizeof(h));
  h.magic = scn::kPlanMagic;
  h.src_w = src_w;
  h.src_h = src_h;
  h.dst_w = dst_w;
  h.dst_h = dst_h;
  h.area2x = (src_w == 2 * dst_w && src_h == 2 * dst_h) ? 1 : 0;
  h.kind = scn::kPlanLinearTaps;
  memcpy(host_plan, &h, sizeof(h));
  scn::Tap* t = reinterpret_cast<scn::Tap*>((uint8_t*)host_plan + sizeof(h));
  scn::fill_taps(src_w, dst_w, true, area, t);
  scn::fill_taps(src_h, dst_h, false, area, t + dst_w);
}

extern "C" int scn_resize_plan_fill(int src_w, int src_h, int dst_w, int dst_h,
                                    void* host_plan) {
  if (src_w <= 0 || src_h <= 0 || dst_w <= 0 || dst_h <= 0 || !host_plan) return SCN_E_BADARG;
  scn::fill_linear_plan(src_w, src_h, dst_w, dst_h, false, host_plan);
  return 0;
}

extern "C" int scn_resize_bilinear_u8c3(const uint8_t* const* host_src_ptrs, int n, int src_w,
                                        int src_h, uint8_t* const* host_dst_ptrs, int dst_w,
                                        int dst_h, const void* plan, void* stream) {
  return scn::launch_resize(host_src_ptrs, n, src_w, src_h, host_dst_ptrs, dst_w, dst_h, plan,
                            (cudaStream_t)stream);
}

extern "C" int scn_resize_bilinear_u8c3_strided(const uint8_t* src, size_t src_stride, int n,
                                                int src_w, int src_h, uint8_t* dst,
                                                size_t dst_stride, int dst_w, int dst_h,
                                                const void* plan, void* stream) {
  if (n < 0) return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!src || !dst) return SCN_E_BADARG;
  return scn::launch_resize(scn::strided(src, src_stride, n).data(), n, src_w, src_h,
                            scn::strided(dst, dst_stride, n).data(), dst_w, dst_h, plan, (cudaStream_t)stream);
}
