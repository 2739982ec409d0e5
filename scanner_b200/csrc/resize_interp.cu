// resize_interp.cu -- cv::resize's INTER_NEAREST and INTER_AREA on u8 HWC 3-channel frames and on NV12 decoder
// surfaces (sm_90a), bit-exact against cv2.resize.  The rules (oracle/resize_interp.c restates them in C):
//   INTER_NEAREST  s = min(floor(d * scale), ssz - 1) per axis, scale = 1.0 / ((double)dsz / ssz): a gather.
//   INTER_AREA     both scales integers (kx, ky): int box sums; 2 x 2 rounds half up (resize_area2x_kernel, as
//                  INTER_LINEAR's exact-2x re-route), every other factor rint((float)sum * (float)(1.0 / (kx ky))).
//                  both scales >= 1, not both integers: OpenCV's float tables (computeResizeAreaTab) and its order,
//                  buf = buf + S * alpha over a row's column entries, sum = beta * buf, then sum = sum + beta * buf
//                  over the cell's rows, rint.  Every product and sum is __fmul_rn / __fadd_rn, so the result does
//                  not depend on -fmad.
//                  a scale below 1: INTER_LINEAR's fixed point with area taps -- resize_linear_kernel and
//                  nv12_resize_kernel with another plan.
// The tables ("plans", resize_plan.cuh) are filled on the host with OpenCV's double and float expressions.
//
// area_kernel: one CTA per (destination row, tile of up to 256 destination columns, frame).  The CTA stages the source
// rows of its destination row through shared memory -- RGB24 rows with 16-byte loads wherever a 16-byte chunk lies
// inside the row, NV12 rows converted pixel by pixel with nv12_math.cuh -- and each thread then walks one destination
// column's table for its three channels.  Every source row is read by the CTAs of the one or two destination rows
// whose cells it overlaps.
#include <limits.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "nv12_math.cuh"
#include "resize_plan.cuh"
#include "scn_common.cuh"

namespace scn {
int launch_resize(const uint8_t* const* sp, int n, int sw, int sh, uint8_t* const* dp, int dw, int dh,
                  const void* plan, cudaStream_t st);

namespace {

constexpr int32_t kPlanMagic = 0x5243504c;  // "LPCR", as resize.cu's
constexpr int kNearest = 0, kLinear = 1, kArea = 3;  // cv::InterpolationFlags
constexpr int kAreaThreads = 256;
constexpr int kCachedTaps = 20;  // table entries per destination column kept in registers
constexpr size_t kStageBudget = 48 * 1024;       // shared memory a CTA stages rows in, when one row fits
constexpr size_t kStageMax = 227 * 1024;         // the most a CTA may have on sm_90

// ---- host: tables ----

// computeResizeAreaTab for one axis: the entries of destination index d are tab[ofs[d] .. ofs[d + 1]).
void area_tab(int ssz, int dsz, std::vector<int32_t>& ofs, std::vector<AreaTap>& tab) {
  const double scale = 1.0 / ((double)dsz / ssz);
  ofs.assign((size_t)dsz + 1, 0);
  tab.clear();
  for (int d = 0; d < dsz; ++d) {
    ofs[d] = (int32_t)tab.size();
    const double fs1 = d * scale, fs2 = fs1 + scale;
    const double cell = std::min(scale, ssz - fs1);
    int s1 = (int)ceil(fs1), s2 = (int)floor(fs2);
    s2 = std::min(s2, ssz - 1);
    s1 = std::min(s1, s2);
    if (s1 - fs1 > 1e-3) tab.push_back({s1 - 1, (float)((s1 - fs1) / cell)});
    for (int s = s1; s < s2; ++s) tab.push_back({s, (float)(1.0 / cell)});
    if (fs2 - s2 > 1e-3) tab.push_back({s2, (float)(std::min(std::min(fs2 - s2, 1.), cell) / cell)});
  }
  ofs[dsz] = (int32_t)tab.size();
}

enum Regime { kUp, kInt2x2, kInt, kFloat };
Regime area_regime(int sw, int sh, int dw, int dh) {
  const double sx = 1.0 / ((double)dw / sw), sy = 1.0 / ((double)dh / sh);
  if (sx < 1 || sy < 1) return kUp;
  if (sw % dw == 0 && sh % dh == 0) return sw == 2 * dw && sh == 2 * dh ? kInt2x2 : kInt;
  return kFloat;
}

// Byte layout of a kPlanArea plan
struct AreaLayout {
  std::vector<int32_t> xofs, yofs;
  std::vector<AreaTap> xtab, ytab;
  size_t yofs_at, xtab_at, ytab_at, bytes;
};
AreaLayout area_layout(int sw, int sh, int dw, int dh) {
  AreaLayout l;
  area_tab(sw, dw, l.xofs, l.xtab);
  area_tab(sh, dh, l.yofs, l.ytab);
  l.yofs_at = sizeof(PlanHeader) + sizeof(int32_t) * ((size_t)dw + 1);
  l.xtab_at = (l.yofs_at + sizeof(int32_t) * ((size_t)dh + 1) + 7) & ~(size_t)7;
  l.ytab_at = l.xtab_at + sizeof(AreaTap) * l.xtab.size();
  l.bytes = l.ytab_at + sizeof(AreaTap) * l.ytab.size();
  return l;
}

PlanHeader header(int sw, int sh, int dw, int dh, int kind) {
  PlanHeader h;
  memset(&h, 0, sizeof(h));
  h.magic = kPlanMagic;
  h.src_w = sw;
  h.src_h = sh;
  h.dst_w = dw;
  h.dst_h = dh;
  h.area2x = (sw == 2 * dw && sh == 2 * dh) ? 1 : 0;
  h.kind = kind;
  return h;
}

bool uses_linear_taps(int mode, int sw, int sh, int dw, int dh) {
  return mode == kLinear || (mode == kArea && area_regime(sw, sh, dw, dh) == kUp);
}

// ---- device ----

// A frame's source: RGB24 frames (a = frame, pitch = 3 * width) or NV12 surfaces (a = luma, b = chroma).
struct Source {
  PtrBatch a, b;
  size_t pitch;
  int height;
};

__device__ __forceinline__ float u8_to_float(uint32_t v) {
  return __fsub_rn(__uint_as_float(0x4B000000u | v), 8388608.0f);  // exact, without the conversion unit
}

// Offset of the staged byte of column c0 in its staged row: the RGB24 rows keep their 16-byte phase.
template <bool NV12>
__device__ __forceinline__ int stage_lead(const Source& src, int f, int sy, int c0) {
  if constexpr (NV12) return 0;
  return (int)(reinterpret_cast<uintptr_t>(src.a.p[f] + (size_t)sy * src.pitch + 3 * (size_t)c0) & 15u);
}

// Stages source columns [c0, c0 + span) of the rows ytab[j0 .. j0 + nr) into sm (row r at r * stride) as RGB bytes.
template <bool NV12>
__device__ __forceinline__ void stage_rows(const Source& src, int f, const AreaTap* __restrict__ ytab, int j0, int nr,
                                           int c0, int span, uint8_t* sm, int stride) {
  if constexpr (NV12) {
    const uint8_t* __restrict__ luma = src.a.p[f];
    const uint8_t* __restrict__ chroma = src.b.p[f];
    for (int k = threadIdx.x; k < nr * span; k += blockDim.x) {
      const int r = k / span, x = k - r * span;
      const Rgb8 c = nv12_pixel(luma, chroma, src.pitch, src.height, c0 + x, __ldg(&ytab[j0 + r].s));
      uint8_t* d = sm + r * stride + 3 * x;
      d[0] = (uint8_t)c.r;
      d[1] = (uint8_t)c.g;
      d[2] = (uint8_t)c.b;
    }
  } else {
    const int bytes = 3 * span;
    const int chunks = (15 + bytes + 15) >> 4;  // the most a row can take at any 16-byte phase
    for (int k = threadIdx.x; k < nr * chunks; k += blockDim.x) {
      const int r = k / chunks, q = k - r * chunks;
      const uint8_t* p = src.a.p[f] + (size_t)__ldg(&ytab[j0 + r].s) * src.pitch + 3 * (size_t)c0;
      const int lead = (int)(reinterpret_cast<uintptr_t>(p) & 15u);
      const int b0 = 16 * q - lead;  // the chunk's first byte, relative to p
      if (b0 >= bytes) continue;
      uint8_t* d = sm + r * stride + 16 * q;
      if (b0 >= 0 && b0 + 16 <= bytes) {
        *reinterpret_cast<uint4*>(d) = ld_stream_u4(p + b0);
      } else {
        for (int i = 0; i < 16; ++i)
          if (b0 + i >= 0 && b0 + i < bytes) d[i] = p[b0 + i];
      }
    }
  }
}

// INT: integer factors (box sums in int); otherwise OpenCV's float tables.  rows: rows staged per step; stride:
// bytes per staged row.
template <bool INT, bool NV12>
__global__ void __launch_bounds__(kAreaThreads)
area_kernel(Source src, MutPtrBatch dst, const int32_t* __restrict__ xofs, const int32_t* __restrict__ yofs,
            const AreaTap* __restrict__ xtab, const AreaTap* __restrict__ ytab, int dw, float inv_area, int rows,
            int stride) {
  extern __shared__ uint4 stage_u4[];
  uint8_t* sm = reinterpret_cast<uint8_t*>(stage_u4);
  const int dy = blockIdx.x, f = blockIdx.z;
  const int dx0 = blockIdx.y * blockDim.x, dx1 = min(dw, dx0 + (int)blockDim.x);
  const int dx = dx0 + threadIdx.x;
  const bool active = dx < dx1;
  // the source columns of this tile: from its first entry to its last
  const int c0 = __ldg(&xtab[__ldg(&xofs[dx0])].s);
  const int span = __ldg(&xtab[__ldg(&xofs[dx1]) - 1].s) - c0 + 1;
  const int e0 = active ? __ldg(&xofs[dx]) : 0, e1 = active ? __ldg(&xofs[dx + 1]) : 0;
  const int j_begin = __ldg(&yofs[dy]), j_end = __ldg(&yofs[dy + 1]);
  // a column's entries (at most kCachedTaps, 1080p and 4K to 224 included) stay in registers for all its rows, so
  // that the shared-memory loads of a row are independent of each other and of any global load
  const int ne = e1 - e0;
  const bool cached = ne <= kCachedTaps;
  int xs[kCachedTaps];
  float xw[kCachedTaps];
#pragma unroll
  for (int k = 0; k < kCachedTaps; ++k) {
    const AreaTap t = cached && k < ne ? xtab[e0 + k] : AreaTap{0, 0.f};
    xs[k] = 3 * t.s;
    xw[k] = t.w;
  }
  int isum[3] = {0, 0, 0};
  float fsum[3] = {0.f, 0.f, 0.f};
  for (int j0 = j_begin; j0 < j_end; j0 += rows) {
    const int nr = min(rows, j_end - j0);
    __syncthreads();  // the previous step's rows are consumed
    stage_rows<NV12>(src, f, ytab, j0, nr, c0, span, sm, stride);
    __syncthreads();
    if (!active) continue;
    for (int r = 0; r < nr; ++r) {
      const AreaTap yt = ytab[j0 + r];
      const uint8_t* row = sm + r * stride + stage_lead<NV12>(src, f, yt.s, c0) - 3 * c0;
      if constexpr (INT) {
        if (cached) {
#pragma unroll
          for (int k = 0; k < kCachedTaps; ++k) {
            if (k < ne) {
              const uint8_t* px = row + xs[k];
              isum[0] += px[0];
              isum[1] += px[1];
              isum[2] += px[2];
            }
          }
          continue;
        }
        for (int e = e0; e < e1; ++e) {
          const uint8_t* px = row + 3 * __ldg(&xtab[e].s);
          isum[0] += px[0];
          isum[1] += px[1];
          isum[2] += px[2];
        }
      } else {
        float buf[3] = {0.f, 0.f, 0.f};
        if (cached) {
#pragma unroll
          for (int k = 0; k < kCachedTaps; ++k) {
            if (k < ne) {
              const uint8_t* px = row + xs[k];
#pragma unroll
              for (int c = 0; c < 3; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn(u8_to_float(px[c]), xw[k]));
            }
          }
        } else {
          for (int e = e0; e < e1; ++e) {
            const AreaTap xt = xtab[e];
            const uint8_t* px = row + 3 * xt.s;
#pragma unroll
            for (int c = 0; c < 3; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn(u8_to_float(px[c]), xt.w));
          }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c)
          fsum[c] = j0 + r == j_begin ? __fmul_rn(yt.w, buf[c]) : __fadd_rn(fsum[c], __fmul_rn(yt.w, buf[c]));
      }
    }
  }
  if (!active) return;
  uint8_t* o = dst.p[f] + ((size_t)dy * dw + dx) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int v = INT ? __float2int_rn(__fmul_rn(__int2float_rn(isum[c]), inv_area)) : __float2int_rn(fsum[c]);
    o[c] = (uint8_t)min(max(v, 0), 255);
  }
}

// One thread per destination pixel.
template <bool NV12>
__global__ void __launch_bounds__(256)
nearest_kernel(Source src, MutPtrBatch dst, const int32_t* __restrict__ xs, const int32_t* __restrict__ ys, int dw,
               int dh) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= dw * dh) return;
  const int dy = idx / dw, dx = idx - dy * dw;
  const int sx = __ldg(&xs[dx]), sy = __ldg(&ys[dy]);
  uint8_t* o = dst.p[blockIdx.y] + (size_t)idx * 3;
  if constexpr (NV12) {
    const Rgb8 c = nv12_pixel(src.a.p[blockIdx.y], src.b.p[blockIdx.y], src.pitch, src.height, sx, sy);
    o[0] = (uint8_t)c.r;
    o[1] = (uint8_t)c.g;
    o[2] = (uint8_t)c.b;
  } else {
    const uint8_t* s = src.a.p[blockIdx.y] + (size_t)sy * src.pitch + 3 * (size_t)sx;
    o[0] = __ldg(s);
    o[1] = __ldg(s + 1);
    o[2] = __ldg(s + 2);
  }
}

// ---- host: launches ----

// n frames: src / chroma pointer lists (chroma null for RGB24), rows of `pitch` bytes.
template <bool NV12>
int launch_nearest(const uint8_t* const* a, const uint8_t* const* b, size_t pitch, int n, int sh, uint8_t* const* dp,
                   int dw, int dh, const void* plan, cudaStream_t st) {
  const int32_t* xs = reinterpret_cast<const int32_t*>((const uint8_t*)plan + sizeof(PlanHeader));
  const int32_t* ys = xs + dw;
  return for_each_chunk(n, [&](int i0, int cnt) {
    Source s{gather<PtrBatch>(a, i0, cnt), NV12 ? gather<PtrBatch>(b, i0, cnt) : PtrBatch{}, pitch, sh};
    const MutPtrBatch d = gather<MutPtrBatch>(dp, i0, cnt);
    dim3 grid((unsigned)(((int64_t)dw * dh + 255) / 256), (unsigned)cnt);
    return launch_kernel(NV12 ? "resize_nearest_nv12_kernel" : "resize_nearest_kernel", st,
                         [&] { nearest_kernel<NV12><<<grid, 256, 0, st>>>(s, d, xs, ys, dw, dh); });
  });
}

template <bool INT, bool NV12>
int launch_area(const uint8_t* const* a, const uint8_t* const* b, size_t pitch, int n, int sw, int sh,
                uint8_t* const* dp, int dw, int dh, const void* plan, cudaStream_t st) {
  // the launch geometry comes from the host copy of the tables the plan holds
  const AreaLayout l = area_layout(sw, sh, dw, dh);
  const int threads = std::min(kAreaThreads, (dw + 31) / 32 * 32);
  const int tiles = (dw + threads - 1) / threads;
  int span = 1, cell_rows = 1;
  for (int t = 0; t < tiles; ++t) {
    const int d0 = t * threads, d1 = std::min(dw, d0 + threads);
    span = std::max(span, l.xtab[l.xofs[d1] - 1].s - l.xtab[l.xofs[d0]].s + 1);
  }
  for (int d = 0; d < dh; ++d) cell_rows = std::max(cell_rows, l.yofs[d + 1] - l.yofs[d]);
  const size_t stride = ((size_t)3 * span + 15 + 15) & ~(size_t)15;
  if (stride > kStageMax) return SCN_E_UNSUPPORTED;
  const int rows = (int)std::max<size_t>(1, std::min<size_t>(cell_rows, kStageBudget / stride));
  const size_t smem = stride * rows;
  auto* kernel = area_kernel<INT, NV12>;
  if (smem > kStageBudget) {
    const int rc = raise_smem_limit((const void*)kernel, kStageMax);
    if (rc) return rc;
  }
  const uint8_t* p = (const uint8_t*)plan;
  const int32_t* xofs = reinterpret_cast<const int32_t*>(p + sizeof(PlanHeader));
  const int32_t* yofs = reinterpret_cast<const int32_t*>(p + l.yofs_at);
  const AreaTap* xtab = reinterpret_cast<const AreaTap*>(p + l.xtab_at);
  const AreaTap* ytab = reinterpret_cast<const AreaTap*>(p + l.ytab_at);
  const float inv_area = (float)(1.0 / ((double)(sw / dw) * (sh / dh)));
  return for_each_chunk(n, [&](int i0, int cnt) {
    Source s{gather<PtrBatch>(a, i0, cnt), NV12 ? gather<PtrBatch>(b, i0, cnt) : PtrBatch{}, pitch, sh};
    const MutPtrBatch d = gather<MutPtrBatch>(dp, i0, cnt);
    dim3 grid((unsigned)dh, (unsigned)tiles, (unsigned)cnt);
    return launch_kernel(NV12 ? "resize_area_nv12_kernel" : "resize_area_kernel", st, [&] {
      kernel<<<grid, threads, smem, st>>>(s, d, xofs, yofs, xtab, ytab, dw, inv_area, rows, (int)stride);
    });
  });
}

// SCN_E_UNSUPPORTED for a mode OpenCV has and this library does not build, SCN_E_BADARG for any other unknown one
int check_mode(int mode) {
  if (mode == kNearest || mode == kLinear || mode == kArea) return 0;
  return mode == 2 || mode == 4 || mode == 5 || mode == 6 ? SCN_E_UNSUPPORTED : SCN_E_BADARG;
}

bool bad_sizes(int sw, int sh, int dw, int dh) {
  // the kernels index destination pixels with an int
  return sw <= 0 || sh <= 0 || dw <= 0 || dh <= 0 || (int64_t)dw * dh > INT_MAX;
}

}  // namespace
}  // namespace scn

extern "C" int scn_resize_interp_code(const char* name) {
  if (!name) return SCN_E_BADARG;
  static const struct {
    const char* name;
    int code;
  } kNames[] = {{"", 1},
                {"INTER_NEAREST", 0},
                {"INTER_LINEAR", 1},
                {"INTER_AREA", 3},
                {"INTER_CUBIC", SCN_E_UNSUPPORTED},
                {"INTER_LANCZOS4", SCN_E_UNSUPPORTED},
                {"INTER_LINEAR_EXACT", SCN_E_UNSUPPORTED},
                {"INTER_NEAREST_EXACT", SCN_E_UNSUPPORTED}};
  for (const auto& e : kNames)
    if (strcmp(name, e.name) == 0) return e.code;
  return SCN_E_BADARG;
}

extern "C" const char* scn_resize_interp_supported(void) { return "INTER_NEAREST, INTER_LINEAR, INTER_AREA"; }

extern "C" size_t scn_resize_interp_plan_bytes(int mode, int src_w, int src_h, int dst_w, int dst_h) {
  using namespace scn;
  if (check_mode(mode) || bad_sizes(src_w, src_h, dst_w, dst_h)) return 0;
  if (uses_linear_taps(mode, src_w, src_h, dst_w, dst_h)) return scn_resize_plan_bytes(dst_w, dst_h);
  if (mode == kNearest) return sizeof(PlanHeader) + sizeof(int32_t) * ((size_t)dst_w + dst_h);
  return area_layout(src_w, src_h, dst_w, dst_h).bytes;
}

extern "C" int scn_resize_interp_plan_fill(int mode, int src_w, int src_h, int dst_w, int dst_h, void* host_plan) {
  using namespace scn;
  if (const int rc = check_mode(mode)) return rc;
  if (bad_sizes(src_w, src_h, dst_w, dst_h) || !host_plan) return SCN_E_BADARG;
  uint8_t* p = (uint8_t*)host_plan;
  if (uses_linear_taps(mode, src_w, src_h, dst_w, dst_h)) {
    fill_linear_plan(src_w, src_h, dst_w, dst_h, mode == kArea, host_plan);
  } else if (mode == kNearest) {
    const PlanHeader h = header(src_w, src_h, dst_w, dst_h, kPlanNearest);
    memcpy(p, &h, sizeof(h));
    int32_t* t = reinterpret_cast<int32_t*>(p + sizeof(h));
    const double fx = 1.0 / ((double)dst_w / src_w), fy = 1.0 / ((double)dst_h / src_h);
    for (int x = 0; x < dst_w; ++x) t[x] = std::min((int)floor(x * fx), src_w - 1);
    for (int y = 0; y < dst_h; ++y) t[dst_w + y] = std::min((int)floor(y * fy), src_h - 1);
  } else {
    const AreaLayout l = area_layout(src_w, src_h, dst_w, dst_h);
    memset(p, 0, l.bytes);
    const PlanHeader h = header(src_w, src_h, dst_w, dst_h, kPlanArea);
    memcpy(p, &h, sizeof(h));
    memcpy(p + sizeof(h), l.xofs.data(), sizeof(int32_t) * l.xofs.size());
    memcpy(p + l.yofs_at, l.yofs.data(), sizeof(int32_t) * l.yofs.size());
    memcpy(p + l.xtab_at, l.xtab.data(), sizeof(AreaTap) * l.xtab.size());
    memcpy(p + l.ytab_at, l.ytab.data(), sizeof(AreaTap) * l.ytab.size());
  }
  return 0;
}

extern "C" int scn_resize_interp_u8c3(int mode, const uint8_t* const* host_src_ptrs, int n, int src_w, int src_h,
                                      uint8_t* const* host_dst_ptrs, int dst_w, int dst_h, const void* plan,
                                      void* stream) {
  using namespace scn;
  if (const int rc = check_mode(mode)) return rc;
  if (n < 0 || bad_sizes(src_w, src_h, dst_w, dst_h)) return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!host_src_ptrs || !host_dst_ptrs) return SCN_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  const Regime rg = area_regime(src_w, src_h, dst_w, dst_h);
  if (uses_linear_taps(mode, src_w, src_h, dst_w, dst_h) || (mode == kArea && rg == kInt2x2))
    return launch_resize(host_src_ptrs, n, src_w, src_h, host_dst_ptrs, dst_w, dst_h, plan, st);
  if (!plan) return SCN_E_PLAN;
  const size_t pitch = 3 * (size_t)src_w;
  if (mode == kNearest)
    return launch_nearest<false>(host_src_ptrs, nullptr, pitch, n, src_h, host_dst_ptrs, dst_w, dst_h, plan, st);
  return rg == kInt ? launch_area<true, false>(host_src_ptrs, nullptr, pitch, n, src_w, src_h, host_dst_ptrs, dst_w,
                                               dst_h, plan, st)
                    : launch_area<false, false>(host_src_ptrs, nullptr, pitch, n, src_w, src_h, host_dst_ptrs, dst_w,
                                                dst_h, plan, st);
}

extern "C" int scn_resize_interp_nv12(int mode, const uint8_t* const* host_luma_ptrs,
                                      const uint8_t* const* host_chroma_ptrs, size_t pitch, int n, int width,
                                      int height, uint8_t* const* host_dst_ptrs, int dst_w, int dst_h,
                                      const void* plan, void* stream) {
  using namespace scn;
  if (const int rc = check_mode(mode)) return rc;
  if (n < 0 || bad_sizes(width, height, dst_w, dst_h) || (width & 1) || (height & 1) || pitch < (size_t)width)
    return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!host_luma_ptrs || !host_chroma_ptrs || !host_dst_ptrs) return SCN_E_BADARG;
  const Regime rg = area_regime(width, height, dst_w, dst_h);
  if (uses_linear_taps(mode, width, height, dst_w, dst_h) || (mode == kArea && rg == kInt2x2))
    return scn_nv12_hist_resize(host_luma_ptrs, host_chroma_ptrs, pitch, n, width, height, nullptr, host_dst_ptrs,
                                dst_w, dst_h, plan, stream);
  if (!plan) return SCN_E_PLAN;
  cudaStream_t st = (cudaStream_t)stream;
  if (mode == kNearest)
    return launch_nearest<true>(host_luma_ptrs, host_chroma_ptrs, pitch, n, height, host_dst_ptrs, dst_w, dst_h,
                                plan, st);
  return rg == kInt ? launch_area<true, true>(host_luma_ptrs, host_chroma_ptrs, pitch, n, width, height,
                                              host_dst_ptrs, dst_w, dst_h, plan, st)
                    : launch_area<false, true>(host_luma_ptrs, host_chroma_ptrs, pitch, n, width, height,
                                               host_dst_ptrs, dst_w, dst_h, plan, st);
}
