// convert_color.cu -- cv::cvtColor on u8 frames and on NV12 decoder surfaces (sm_90a).
// Replaces scannertools' ConvertColor kernel (cv::cvtColor with the named code).  For 8-bit input OpenCV's
// conversions are integer fixed point; each code below is restated exactly (oracle/convert_color.py holds the
// same formulas against cv2.cvtColor on all 2^24 RGB triples).  D(x, n) = (x + 2^(n-1)) >> n.
//   GRAY    Y = D(9798 R + 19235 G + 3735 B, 15)
//   YCrCb   Y = D(4899 R + 9617 G + 1868 B, 14), Cr = sat(D((R - Y) 11682 + (128 << 14), 14)),
//           Cb = sat(D((B - Y) 9241 + (128 << 14), 14))
//   HSV     OpenCV's RGB2HSV_b with its division tables (hue range 180, or 256 for _FULL, stored mod 256)
//   swap    RGB <-> BGR;  GRAY2RGB replicates the gray channel.
// Two kernels:
//   convert_color_kernel       dense HWC u8 frames.  16 pixels per thread with 128-bit loads and stores over the
//                              part of the frame where source and destination are both 16-byte aligned (stores
//                              of three-channel output staged per warp, see store_groups); the few pixels before
//                              and after it (or the whole frame, when the two alignments never meet) go pixel by
//                              pixel.
//   convert_color_nv12_kernel  packed NV12 elements: each pixel through the reference's NV12 -> RGB chain
//                              (nv12_math.cuh), then the conversion in registers; the RGB24 frame is never written.
#include <cmath>
#include <cstring>

#include "nv12_math.cuh"
#include "scn_common.cuh"

namespace scn {
namespace {

enum Algo { kGray, kYCrCb, kHsv, kSwap, kGray2Rgb };

struct Code {
  const char* name;
  Algo algo;
  bool bgr;    // the first input channel is blue
  int hrange;  // HSV hue range
};
// The order is the code numbering of scn_kernels.h.  The swap and replicate codes do the same thing either way.
constexpr Code kCodes[] = {
    {"COLOR_RGB2GRAY", kGray, false, 0},      {"COLOR_BGR2GRAY", kGray, true, 0},
    {"COLOR_RGB2YCrCb", kYCrCb, false, 0},    {"COLOR_BGR2YCrCb", kYCrCb, true, 0},
    {"COLOR_RGB2HSV", kHsv, false, 180},      {"COLOR_BGR2HSV", kHsv, true, 180},
    {"COLOR_RGB2HSV_FULL", kHsv, false, 256}, {"COLOR_BGR2HSV_FULL", kHsv, true, 256},
    {"COLOR_RGB2BGR", kSwap, false, 0},       {"COLOR_BGR2RGB", kSwap, false, 0},
    {"COLOR_GRAY2RGB", kGray2Rgb, false, 0},  {"COLOR_GRAY2BGR", kGray2Rgb, false, 0},
};
constexpr int kNumCodes = (int)(sizeof(kCodes) / sizeof(kCodes[0]));

__host__ __device__ constexpr int in_channels(Algo a) { return a == kGray2Rgb ? 1 : 3; }
__host__ __device__ constexpr int out_channels(Algo a) { return a == kGray ? 1 : 3; }

constexpr int kHsvShift = 12;
// RGB2HSV_b's tables, built on the host as OpenCV builds them; they travel in the parameter block and each block
// copies them to shared memory (the lookups diverge, which the constant bank would serialise).
struct HsvTables {
  int32_t sdiv[256];  // round((255 << 12) / v)
  int32_t hdiv[256];  // round((hrange << 12) / (6 diff))
};

HsvTables hsv_tables(int hrange) {
  HsvTables t;
  t.sdiv[0] = t.hdiv[0] = 0;
  for (int i = 1; i < 256; ++i) {
    t.sdiv[i] = (int32_t)std::lrint((255 << kHsvShift) / (1.0 * i));
    t.hdiv[i] = (int32_t)std::lrint((hrange << kHsvShift) / (6.0 * i));
  }
  return t;
}

template <Algo A>
__device__ __forceinline__ void load_tables(const HsvTables& t, int32_t* sdiv, int32_t* hdiv) {
  if constexpr (A == kHsv) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
      sdiv[i] = t.sdiv[i];
      hdiv[i] = t.hdiv[i];
    }
    __syncthreads();
  }
}

// One pixel.  (c0, c1, c2) are the input channels in memory order (c0 alone for GRAY2RGB); o receives the
// output channels.
template <Algo A, bool BGR>
__device__ __forceinline__ void convert_px(uint32_t c0, uint32_t c1, uint32_t c2, const int32_t* sdiv,
                                           const int32_t* hdiv, int hrange, uint32_t (&o)[3]) {
  const int r = (int)(BGR ? c2 : c0), g = (int)c1, b = (int)(BGR ? c0 : c2);
  if constexpr (A == kGray) {
    o[0] = (uint32_t)(9798 * r + 19235 * g + 3735 * b + (1 << 14)) >> 15;
  } else if constexpr (A == kYCrCb) {
    const int y = (4899 * r + 9617 * g + 1868 * b + (1 << 13)) >> 14;
    const int cr = ((r - y) * 11682 + (128 << 14) + (1 << 13)) >> 14;
    const int cb = ((b - y) * 9241 + (128 << 14) + (1 << 13)) >> 14;
    o[0] = (uint32_t)y;
    o[1] = (uint32_t)min(max(cr, 0), 255);
    o[2] = (uint32_t)min(max(cb, 0), 255);
  } else if constexpr (A == kHsv) {
    const int v = max(max(r, g), b);
    const int diff = v - min(min(r, g), b);
    const int s = (diff * sdiv[v] + (1 << (kHsvShift - 1))) >> kHsvShift;
    int h = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
    h = (h * hdiv[diff] + (1 << (kHsvShift - 1))) >> kHsvShift;
    h += h < 0 ? hrange : 0;
    o[0] = (uint32_t)h & 0xFFu;
    o[1] = (uint32_t)s;
    o[2] = (uint32_t)v;
  } else if constexpr (A == kSwap) {
    o[0] = c2;
    o[1] = c1;
    o[2] = c0;
  } else {
    o[0] = o[1] = o[2] = c0;
  }
}

template <int N>
__device__ __forceinline__ uint32_t byte_at(const uint32_t (&w)[N], int k) {
  return (w[k >> 2] >> (8 * (k & 3))) & 0xFFu;
}

// First pixel index at which ptr + c * p is 16-byte aligned (c odd, so it is a unit mod 16: 3^-1 = 11).
__device__ __forceinline__ uint32_t aligned_from(const void* ptr, int c) {
  const uint32_t mis = (uint32_t)reinterpret_cast<uintptr_t>(ptr) & 15u;
  return ((16u - mis) * (c == 1 ? 1u : 11u)) & 15u;
}

// Store the 16 output pixels of every lane of a warp; lane l's go to span + 16 CO l.  Three-channel output goes
// through shared memory so that each store instruction writes 512 contiguous bytes: stored straight from
// registers, each instruction would leave every 32-byte sector it touches half written, which measured about
// 1.5x slower at 1080p (GRAY2RGB, and RGB<->BGR from NV12, on an H100).  The whole warp calls this; lanes with !valid store nothing.
template <int CO>
__device__ __forceinline__ void store_groups(uint4* stage, uint8_t* span, const uint32_t (&o)[4 * CO], bool valid) {
  const int lane = threadIdx.x & 31;
  uint4* d = reinterpret_cast<uint4*>(span);
  if constexpr (CO == 1) {
    if (valid) d[lane] = make_uint4(o[0], o[1], o[2], o[3]);
  } else {
    const unsigned live = __ballot_sync(0xFFFFFFFFu, valid);
#pragma unroll
    for (int k = 0; k < 3; ++k) stage[3 * lane + k] = make_uint4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]);
    __syncwarp();
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int j = lane + 32 * k;
      if ((live >> (j / 3)) & 1u) d[j] = stage[j];
    }
    __syncwarp();
  }
}

constexpr int kThreads = 256;

template <Algo A, bool BGR>
__global__ void __launch_bounds__(kThreads)
convert_color_kernel(PtrBatch srcs, MutPtrBatch dsts, uint32_t npix, int hrange, HsvTables tables) {
  constexpr int CI = in_channels(A), CO = out_channels(A);
  __shared__ int32_t sdiv[A == kHsv ? 256 : 1], hdiv[A == kHsv ? 256 : 1];
  __shared__ uint4 stage[kThreads / 32][CO == 3 ? 96 : 1];
  load_tables<A>(tables, sdiv, hdiv);
  const uint8_t* __restrict__ src = srcs.p[blockIdx.y];
  uint8_t* __restrict__ dst = dsts.p[blockIdx.y];
  // 16-pixel groups start where both pointers are 16-byte aligned; if that never happens, nothing is vectorised
  const uint32_t hs = aligned_from(src, CI), hd = aligned_from(dst, CO);
  const uint32_t head = hs == hd ? min(hs, npix) : npix;
  const uint32_t groups = (npix - head) / 16;
  const uint32_t tail0 = head + groups * 16;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gtid = blockIdx.x * kThreads + threadIdx.x, gstride = gridDim.x * kThreads;

  // a warp walks 32 consecutive groups per step (the loop condition is the same for all its lanes)
  for (uint32_t g0 = gtid - lane; g0 < groups; g0 += gstride) {
    const bool valid = g0 + lane < groups;
    const size_t p0 = head + (size_t)(g0 + lane) * 16;
    uint32_t w[4 * CI];
#pragma unroll
    for (int k = 0; k < CI; ++k) {
      // through L1: a lane's three 16-byte loads share 32-byte sectors with its neighbours'
      const uint4 v = valid ? __ldg(reinterpret_cast<const uint4*>(src + p0 * CI) + k) : make_uint4(0, 0, 0, 0);
      w[4 * k + 0] = v.x, w[4 * k + 1] = v.y, w[4 * k + 2] = v.z, w[4 * k + 3] = v.w;
    }
    uint32_t o[4 * CO];
#pragma unroll
    for (int k = 0; k < 4 * CO; ++k) o[k] = 0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      uint32_t px[3];
      if constexpr (CI == 3)
        convert_px<A, BGR>(byte_at(w, 3 * j), byte_at(w, 3 * j + 1), byte_at(w, 3 * j + 2), sdiv, hdiv, hrange, px);
      else
        convert_px<A, BGR>(byte_at(w, j), 0, 0, sdiv, hdiv, hrange, px);
#pragma unroll
      for (int c = 0; c < CO; ++c) o[(CO * j + c) >> 2] |= px[c] << (8 * ((CO * j + c) & 3));
    }
    store_groups<CO>(stage[threadIdx.x >> 5], dst + (head + (size_t)g0 * 16) * CO, o, valid);
  }

  // the pixels before and after the groups
  const uint32_t nscalar = head + (npix - tail0);
  for (uint32_t i = gtid; i < nscalar; i += gstride) {
    const size_t p = i < head ? i : tail0 + (i - head);
    const uint8_t* s = src + p * CI;
    uint32_t px[3];
    convert_px<A, BGR>(s[0], CI == 3 ? s[1] : 0, CI == 3 ? s[2] : 0, sdiv, hdiv, hrange, px);
#pragma unroll
    for (int c = 0; c < CO; ++c) dst[p * CO + c] = (uint8_t)px[c];
  }
}

// One thread: 16 pixels of one row.  vec: width % 16 == 0 and every plane and output 16-byte aligned.
template <Algo A, bool BGR>
__global__ void __launch_bounds__(128)
convert_color_nv12_kernel(PtrBatch lumas, PtrBatch chromas, MutPtrBatch dsts, size_t pitch, int width, int height,
                          int units_per_row, int vec, int hrange, HsvTables tables) {
  constexpr int CO = out_channels(A);
  __shared__ int32_t sdiv[A == kHsv ? 256 : 1], hdiv[A == kHsv ? 256 : 1];
  __shared__ uint4 stage[4][CO == 3 ? 96 : 1];
  load_tables<A>(tables, sdiv, hdiv);
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  const bool valid = u < units_per_row;
  const uint8_t* __restrict__ luma = lumas.p[blockIdx.z];
  const uint8_t* __restrict__ chroma = chromas.p[blockIdx.z];
  uint8_t* __restrict__ out = dsts.p[blockIdx.z] + ((size_t)y * width + (size_t)u * 16) * CO;
  if (vec) {  // the same for the whole launch: every lane of the warp is here
    const int yc = y >> 1;
    uint4 yw = make_uint4(0, 0, 0, 0), cw = yw;
    if (valid) {
      yw = ld_stream_u4(luma + (size_t)y * pitch + (size_t)u * 16);
      cw = ld_stream_u4(chroma + (size_t)yc * pitch + (size_t)u * 16);
    }
    if (valid && (y & 1) && yc < (height >> 1) - 1) {  // odd luma row: rounded mean of the two chroma rows
      const uint4 c2 = ld_stream_u4(chroma + (size_t)(yc + 1) * pitch + (size_t)u * 16);
      cw = make_uint4(__vavgu4(cw.x, c2.x), __vavgu4(cw.y, c2.y), __vavgu4(cw.z, c2.z), __vavgu4(cw.w, c2.w));
    }
    const uint32_t ys[4] = {yw.x, yw.y, yw.z, yw.w}, cs[4] = {cw.x, cw.y, cw.z, cw.w};
    uint32_t o[4 * CO];
#pragma unroll
    for (int k = 0; k < 4 * CO; ++k) o[k] = 0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const Rgb8 rgb = yuv_to_rgb(byte_at(ys, j), byte_at(cs, j & ~1), byte_at(cs, j | 1));
      uint32_t px[3];
      convert_px<A, BGR>(rgb.r, rgb.g, rgb.b, sdiv, hdiv, hrange, px);
#pragma unroll
      for (int c = 0; c < CO; ++c) o[(CO * j + c) >> 2] |= px[c] << (8 * ((CO * j + c) & 3));
    }
    store_groups<CO>(stage[threadIdx.x >> 5], out - (size_t)(threadIdx.x & 31) * 16 * CO, o, valid);
    return;
  }
  if (!valid) return;
  for (int j = 0; j < 16 && u * 16 + j < width; ++j) {
    const Rgb8 rgb = nv12_pixel(luma, chroma, pitch, height, u * 16 + j, y);
    uint32_t px[3];
    convert_px<A, BGR>(rgb.r, rgb.g, rgb.b, sdiv, hdiv, hrange, px);
#pragma unroll
    for (int c = 0; c < CO; ++c) out[CO * j + c] = (uint8_t)px[c];
  }
}

template <Algo A, bool BGR>
int launch_u8(const uint8_t* const* src, uint8_t* const* dst, int n, uint32_t npix, const Code& code,
              cudaStream_t st) {
  const HsvTables tables = A == kHsv ? hsv_tables(code.hrange) : HsvTables{};
  // about two 16-pixel groups per thread
  const uint32_t want = (npix + 32u * kThreads - 1) / (32u * kThreads);
  return for_each_chunk(n, [&](int i0, int cnt) {
    const PtrBatch s = gather<PtrBatch>(src, i0, cnt);
    const MutPtrBatch d = gather<MutPtrBatch>(dst, i0, cnt);
    dim3 grid(want < 1 ? 1 : want, (unsigned)cnt);
    return launch_kernel("convert_color_kernel", st, [&] {
      convert_color_kernel<A, BGR><<<grid, kThreads, 0, st>>>(s, d, npix, code.hrange, tables);
    });
  });
}

template <Algo A, bool BGR>
int launch_nv12(const uint8_t* const* luma, const uint8_t* const* chroma, size_t pitch, int n, int width, int height,
                uint8_t* const* dst, const Code& code, cudaStream_t st) {
  const HsvTables tables = A == kHsv ? hsv_tables(code.hrange) : HsvTables{};
  const int units = (width + 15) / 16;
  return for_each_chunk(n, [&](int i0, int cnt) {
    const PtrBatch l = gather<PtrBatch>(luma, i0, cnt), c = gather<PtrBatch>(chroma, i0, cnt);
    const MutPtrBatch d = gather<MutPtrBatch>(dst, i0, cnt);
    const int vec = (width & 15) == 0 && (pitch & 15) == 0 && aligned(16, i0, cnt, luma, chroma, dst);
    dim3 grid((unsigned)((units + 127) / 128), (unsigned)height, (unsigned)cnt);
    return launch_kernel("convert_color_nv12_kernel", st, [&] {
      convert_color_nv12_kernel<A, BGR>
          <<<grid, 128, 0, st>>>(l, c, d, pitch, width, height, units, vec, code.hrange, tables);
    });
  });
}

}  // namespace
}  // namespace scn

extern "C" int scn_convert_color_code(const char* name) {
  if (!name) return SCN_E_BADARG;
  for (int i = 0; i < scn::kNumCodes; ++i)
    if (std::strcmp(name, scn::kCodes[i].name) == 0) return i;
  return SCN_E_UNSUPPORTED;
}

extern "C" const char* scn_convert_color_name(int code) {
  return code >= 0 && code < scn::kNumCodes ? scn::kCodes[code].name : nullptr;
}

extern "C" int scn_convert_color_channels(int code, int* in_channels, int* out_channels) {
  if (code < 0 || code >= scn::kNumCodes || !in_channels || !out_channels) return SCN_E_BADARG;
  *in_channels = scn::in_channels(scn::kCodes[code].algo);
  *out_channels = scn::out_channels(scn::kCodes[code].algo);
  return 0;
}

extern "C" int scn_convert_color_u8(const uint8_t* const* host_src_ptrs, int n, int width, int height, int code,
                                    uint8_t* const* host_dst_ptrs, void* stream) {
  using namespace scn;
  if (n < 0 || width < 0 || height < 0 || code < 0 || code >= kNumCodes) return SCN_E_BADARG;
  if (n == 0 || width == 0 || height == 0) return 0;
  if (!host_src_ptrs || !host_dst_ptrs) return SCN_E_BADARG;
  if ((uint64_t)width * (uint64_t)height > 0xFFFFFFF0ull) return SCN_E_UNSUPPORTED;
  const uint32_t npix = (uint32_t)width * (uint32_t)height;
  const Code& c = kCodes[code];
  cudaStream_t st = (cudaStream_t)stream;
  switch (c.algo) {
    case kGray: return c.bgr ? launch_u8<kGray, true>(host_src_ptrs, host_dst_ptrs, n, npix, c, st)
                             : launch_u8<kGray, false>(host_src_ptrs, host_dst_ptrs, n, npix, c, st);
    case kYCrCb: return c.bgr ? launch_u8<kYCrCb, true>(host_src_ptrs, host_dst_ptrs, n, npix, c, st)
                              : launch_u8<kYCrCb, false>(host_src_ptrs, host_dst_ptrs, n, npix, c, st);
    case kHsv: return c.bgr ? launch_u8<kHsv, true>(host_src_ptrs, host_dst_ptrs, n, npix, c, st)
                            : launch_u8<kHsv, false>(host_src_ptrs, host_dst_ptrs, n, npix, c, st);
    case kSwap: return launch_u8<kSwap, false>(host_src_ptrs, host_dst_ptrs, n, npix, c, st);
    case kGray2Rgb: return launch_u8<kGray2Rgb, false>(host_src_ptrs, host_dst_ptrs, n, npix, c, st);
  }
  return SCN_E_BADARG;
}

extern "C" int scn_convert_color_nv12(const uint8_t* const* host_luma_ptrs, const uint8_t* const* host_chroma_ptrs,
                                      size_t pitch, int n, int width, int height, int code,
                                      uint8_t* const* host_dst_ptrs, void* stream) {
  using namespace scn;
  if (n < 0 || width <= 0 || height <= 0 || (width & 1) || (height & 1) || pitch < (size_t)width || code < 0 ||
      code >= kNumCodes)
    return SCN_E_BADARG;
  const Code& c = kCodes[code];
  if (in_channels(c.algo) != 3) return SCN_E_BADARG;  // a decoded picture has three channels
  if (n == 0) return 0;
  if (!host_luma_ptrs || !host_chroma_ptrs || !host_dst_ptrs) return SCN_E_BADARG;
  if (height > 65535) return SCN_E_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const uint8_t* const* l = host_luma_ptrs;
  const uint8_t* const* ch = host_chroma_ptrs;
  uint8_t* const* d = host_dst_ptrs;
  switch (c.algo) {
    case kGray: return c.bgr ? launch_nv12<kGray, true>(l, ch, pitch, n, width, height, d, c, st)
                             : launch_nv12<kGray, false>(l, ch, pitch, n, width, height, d, c, st);
    case kYCrCb: return c.bgr ? launch_nv12<kYCrCb, true>(l, ch, pitch, n, width, height, d, c, st)
                              : launch_nv12<kYCrCb, false>(l, ch, pitch, n, width, height, d, c, st);
    case kHsv: return c.bgr ? launch_nv12<kHsv, true>(l, ch, pitch, n, width, height, d, c, st)
                            : launch_nv12<kHsv, false>(l, ch, pitch, n, width, height, d, c, st);
    case kSwap: return launch_nv12<kSwap, false>(l, ch, pitch, n, width, height, d, c, st);
    case kGray2Rgb: break;
  }
  return SCN_E_BADARG;
}
