// nv12.cu -- NV12 decoder surface -> dense RGB24 (sm_90a).
// Replaces convertNV12toRGBA / NV12_to_RGB (reference scanner/util/image.cu:109-200,229-239).
// The reference kernel does scalar byte loads and six scalar byte stores per thread; here one
// thread converts 4 horizontally adjacent pixels: one 32-bit luma load, one 32-bit chroma load
// per contributing chroma row, and three 32-bit stores (12 bytes = 4 RGB pixels), so every
// warp-level access is a contiguous 128-byte (loads) / 384-byte (stores) span.
#include "nv12_math.cuh"
#include "scn_common.cuh"

namespace scn {
namespace {

// ---- FMA-pipe colour math (same scheme as nv12_stream.cuh, here down to the 8-bit value) -----------
//   byte -> float : PRMT builds the bits of 2^23 + byte (no I2F: the conversion unit runs at a quarter
//                   of the FMA rate and made the first version of this kernel XU-bound)
//   x  = value * 2^-11 computed with fma.sat (lower clamp), min(x, 1023 * 2^-11) (upper clamp)
//   u8 = floor(512 * x) == ((unsigned)v) >> 2, taken from the mantissa of fma.rm(x, 512, 2^23) (no F2I)
// Power-of-two scaling commutes with IEEE rounding, so the bits equal yuv_to_rgb()'s.
constexpr float kS = 1.0f / 2048.0f;
constexpr float kCY = 4.0f * 1.1644f * kS, kKR = 4.0f * 1.596f * kS, kKG1 = 4.0f * -0.3918f * kS;
constexpr float kKG2 = 4.0f * -0.813f * kS, kKB = 4.0f * 2.0172f * kS;
constexpr float kMagic = 8388608.0f, kTop = 1023.0f * kS;

__device__ __forceinline__ float byte_magic(uint32_t word, uint32_t sel) {
  return __uint_as_float(prmt(word, 0x4B000000u, sel));
}
__device__ __forceinline__ float fma_sat(float a, float b, float c) {
  float r;
  asm("fma.rn.sat.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c));
  return r;
}
__device__ __forceinline__ uint32_t to_u8_bits(float x) {  // 0x4B0000vv
  float r;
  asm("fma.rm.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(fminf(x, kTop)), "f"(512.0f), "f"(kMagic));
  return __float_as_uint(r);
}
struct RgbBits {
  uint32_t r, g, b;
};
// image.cu's `y*k0 + cb*k1 + cr*k2` as nvcc contracts it (see nv12_math.cuh): fma(cr,k2, fma(y,k0, fl(cb*k1)))
__device__ __forceinline__ RgbBits convert(float ym, float cb, float cr) {  // ym = 2^23 + Y, cb/cr centred
  const float yf = ym - kMagic;                          // exact
  const float ly = __fmaf_rn(ym, kCY, -kMagic * kCY);    // == fl(yf * kCY): R's middle product is +-0
  RgbBits o;
  o.r = to_u8_bits(fma_sat(cr, kKR, ly));
  o.g = to_u8_bits(fma_sat(cr, kKG2, __fmaf_rn(yf, kCY, __fmul_rn(cb, kKG1))));
  o.b = to_u8_bits(fma_sat(yf, kCY, __fmul_rn(cb, kKB)));
  return o;
}
__device__ __forceinline__ uint32_t avg4(uint32_t a, uint32_t b) {  // per byte (a + b + 1) >> 1
  return (a | b) - (((a ^ b) & 0xFEFEFEFEu) >> 1);
}
// low bytes of four registers -> one word
__device__ __forceinline__ uint32_t pack4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  return prmt(prmt(a, b, 0x0040u), prmt(c, d, 0x0040u), 0x5410u);
}

__global__ void __launch_bounds__(256)
nv12_to_rgb_kernel(PtrBatch lumas, PtrBatch chromas, MutPtrBatch rgbs, size_t pitch, int width,
                   int height, size_t rgb_pitch, int quads_per_row, int vec_ok) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  if (q >= quads_per_row) return;
  const uint8_t* __restrict__ luma = lumas.p[blockIdx.z];
  const uint8_t* __restrict__ chroma = chromas.p[blockIdx.z];
  uint8_t* __restrict__ rgb = rgbs.p[blockIdx.z];
  const int x0 = q * 4;
  const int yc = y >> 1;
  const bool avg = (y & 1) && yc < ((height >> 1) - 1);
  uint8_t* o = rgb + (size_t)y * rgb_pitch + (size_t)x0 * 3;
  if (vec_ok && x0 + 4 <= width) {
    const uint32_t yw = ld_stream_u32(luma + (size_t)y * pitch + x0);
    uint32_t cw = __ldg(reinterpret_cast<const uint32_t*>(chroma + (size_t)yc * pitch + x0));
    if (avg) cw = avg4(cw, __ldg(reinterpret_cast<const uint32_t*>(chroma + (size_t)(yc + 1) * pitch + x0)));
    const float bias = -(kMagic + 128.0f);
    const float cb0 = byte_magic(cw, 0x7440u) + bias, cr0 = byte_magic(cw, 0x7441u) + bias;
    const float cb1 = byte_magic(cw, 0x7442u) + bias, cr1 = byte_magic(cw, 0x7443u) + bias;
    const RgbBits p0 = convert(byte_magic(yw, 0x7440u), cb0, cr0), p1 = convert(byte_magic(yw, 0x7441u), cb0, cr0);
    const RgbBits p2 = convert(byte_magic(yw, 0x7442u), cb1, cr1), p3 = convert(byte_magic(yw, 0x7443u), cb1, cr1);
    uint32_t* o32 = reinterpret_cast<uint32_t*>(o);
    o32[0] = pack4(p0.r, p0.g, p0.b, p1.r);
    o32[1] = pack4(p1.g, p1.b, p2.r, p2.g);
    o32[2] = pack4(p2.b, p3.r, p3.g, p3.b);
    return;
  }
  // ragged / unaligned tail: scalar reference arithmetic
  for (int i = 0; i < 4 && x0 + i < width; ++i) {
    const Rgb8 c = nv12_pixel(luma, chroma, pitch, height, x0 + i, y);
    o[3 * i + 0] = (uint8_t)c.r;
    o[3 * i + 1] = (uint8_t)c.g;
    o[3 * i + 2] = (uint8_t)c.b;
  }
}

// 16 pixels per thread: one 128-bit luma load, one 128-bit chroma load per contributing chroma row,
// three 128-bit stores (48 bytes of RGB).  Needs width % 16 == 0 and 16-byte aligned rows.
__global__ void __launch_bounds__(128)
nv12_to_rgb16_kernel(PtrBatch lumas, PtrBatch chromas, MutPtrBatch rgbs, size_t pitch, int height, size_t rgb_pitch,
                     int units_per_row) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  if (u >= units_per_row) return;
  const uint8_t* __restrict__ luma = lumas.p[blockIdx.z];
  const uint8_t* __restrict__ chroma = chromas.p[blockIdx.z];
  const int yc = y >> 1;
  const bool avg = (y & 1) && yc < ((height >> 1) - 1);
  const uint4 yw = ld_stream_u4(luma + (size_t)y * pitch + (size_t)u * 16);
  uint4 cw = ld_stream_u4(chroma + (size_t)yc * pitch + (size_t)u * 16);
  if (avg) {
    const uint4 c2 = ld_stream_u4(chroma + (size_t)(yc + 1) * pitch + (size_t)u * 16);
    cw = make_uint4(avg4(cw.x, c2.x), avg4(cw.y, c2.y), avg4(cw.z, c2.z), avg4(cw.w, c2.w));
  }
  const uint32_t ys[4] = {yw.x, yw.y, yw.z, yw.w}, cs[4] = {cw.x, cw.y, cw.z, cw.w};
  uint32_t out[12];
  const float bias = -(kMagic + 128.0f);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float cb0 = byte_magic(cs[k], 0x7440u) + bias, cr0 = byte_magic(cs[k], 0x7441u) + bias;
    const float cb1 = byte_magic(cs[k], 0x7442u) + bias, cr1 = byte_magic(cs[k], 0x7443u) + bias;
    const RgbBits p0 = convert(byte_magic(ys[k], 0x7440u), cb0, cr0), p1 = convert(byte_magic(ys[k], 0x7441u), cb0, cr0);
    const RgbBits p2 = convert(byte_magic(ys[k], 0x7442u), cb1, cr1), p3 = convert(byte_magic(ys[k], 0x7443u), cb1, cr1);
    out[3 * k + 0] = pack4(p0.r, p0.g, p0.b, p1.r);
    out[3 * k + 1] = pack4(p1.g, p1.b, p2.r, p2.g);
    out[3 * k + 2] = pack4(p2.b, p3.r, p3.g, p3.b);
  }
  uint4* o = reinterpret_cast<uint4*>(rgbs.p[blockIdx.z] + (size_t)y * rgb_pitch + (size_t)u * 48);
  o[0] = make_uint4(out[0], out[1], out[2], out[3]);
  o[1] = make_uint4(out[4], out[5], out[6], out[7]);
  o[2] = make_uint4(out[8], out[9], out[10], out[11]);
}

// Pitched decoder surface -> packed NV12 element (W x H luma rows, then W x H/2 CbCr rows).
// Row r of the packed image comes from the luma plane for r < H, from the chroma plane after.
// 16 bytes per thread when everything is 16-byte aligned, else bytes.
__global__ void __launch_bounds__(256)
nv12_pack_kernel(PtrBatch lumas, PtrBatch chromas, MutPtrBatch dsts, size_t pitch, int width, int height,
                 int vec16) {
  const uint8_t* __restrict__ luma = lumas.p[blockIdx.z];
  const uint8_t* __restrict__ chroma = chromas.p[blockIdx.z];
  uint8_t* __restrict__ dst = dsts.p[blockIdx.z];
  const int rows = height + (height >> 1);
  if (vec16) {
    const int vpr = width >> 4;  // 16-byte vectors per row
    const long total = (long)vpr * rows;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
      const int r = (int)(i / vpr), v = (int)(i - (long)r * vpr);
      const uint8_t* src = (r < height ? luma + (size_t)r * pitch : chroma + (size_t)(r - height) * pitch) + v * 16;
      *reinterpret_cast<uint4*>(dst + (size_t)r * width + v * 16) = ld_stream_u4(src);
    }
  } else {
    const long total = (long)width * rows;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
      const int r = (int)(i / width), x = (int)(i - (long)r * width);
      dst[i] = r < height ? luma[(size_t)r * pitch + x] : chroma[(size_t)(r - height) * pitch + x];
    }
  }
}

}  // namespace
}  // namespace scn

extern "C" int scn_nv12_pack(const uint8_t* const* host_luma_ptrs, const uint8_t* const* host_chroma_ptrs,
                             size_t pitch, int n, int width, int height, uint8_t* const* host_dst_ptrs,
                             void* stream) {
  using namespace scn;
  if (n < 0 || width <= 0 || height <= 0 || (width & 1) || (height & 1) || pitch < (size_t)width)
    return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!host_luma_ptrs || !host_chroma_ptrs || !host_dst_ptrs) return SCN_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  for (int i0 = 0; i0 < n; i0 += SCN_MAX_PTRS) {
    const int cnt = (n - i0 < SCN_MAX_PTRS) ? (n - i0) : SCN_MAX_PTRS;
    PtrBatch l, c;
    MutPtrBatch d;
    int vec16 = ((pitch & 15) == 0) && ((width & 15) == 0);
    for (int i = 0; i < cnt; ++i) {
      l.p[i] = host_luma_ptrs[i0 + i];
      c.p[i] = host_chroma_ptrs[i0 + i];
      d.p[i] = host_dst_ptrs[i0 + i];
      if (((uintptr_t)l.p[i] | (uintptr_t)c.p[i] | (uintptr_t)d.p[i]) & 15) vec16 = 0;
    }
    const long work = vec16 ? (long)(width >> 4) * (height + height / 2) : (long)width * (height + height / 2);
    long gx = (work + 255) / 256;
    const long cap = (long)sm_count() * 8 / cnt + 1;
    if (gx > cap) gx = cap;
    dim3 grid((unsigned)gx, 1, (unsigned)cnt);
    {
      LaunchScope ls("nv12_pack_kernel", st);
      nv12_pack_kernel<<<grid, 256, 0, st>>>(l, c, d, pitch, width, height, vec16);
    }
    int rc = launch_status();
    if (rc) return rc;
  }
  return 0;
}

extern "C" int scn_nv12_to_rgb24(const uint8_t* const* host_luma_ptrs,
                                 const uint8_t* const* host_chroma_ptrs, size_t pitch, int n,
                                 int width, int height, uint8_t* const* host_rgb_ptrs,
                                 size_t rgb_pitch, void* stream) {
  using namespace scn;
  if (n < 0 || width <= 0 || height <= 0 || (width & 1) || (height & 1) ||
      pitch < (size_t)width || rgb_pitch < (size_t)width * 3)
    return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!host_luma_ptrs || !host_chroma_ptrs || !host_rgb_ptrs) return SCN_E_BADARG;
  if (height > 65535) return SCN_E_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const int quads = (width + 3) / 4;
  for (int i0 = 0; i0 < n; i0 += SCN_MAX_PTRS) {
    const int cnt = (n - i0 < SCN_MAX_PTRS) ? (n - i0) : SCN_MAX_PTRS;
    PtrBatch l, c;
    MutPtrBatch r;
    int vec_ok = ((pitch & 3) == 0) && ((rgb_pitch & 3) == 0);
    for (int i = 0; i < cnt; ++i) {
      l.p[i] = host_luma_ptrs[i0 + i];
      c.p[i] = host_chroma_ptrs[i0 + i];
      r.p[i] = host_rgb_ptrs[i0 + i];
      if (((uintptr_t)l.p[i] | (uintptr_t)c.p[i] | (uintptr_t)r.p[i]) & 3) vec_ok = 0;
    }
    int vec16 = ((width & 15) == 0) && ((pitch & 15) == 0) && ((rgb_pitch & 15) == 0);
    for (int i = 0; i < cnt; ++i)
      if (((uintptr_t)l.p[i] | (uintptr_t)c.p[i] | (uintptr_t)r.p[i]) & 15) vec16 = 0;
    if (vec16) {
      const int units = width / 16;
      dim3 grid((unsigned)((units + 127) / 128), (unsigned)height, (unsigned)cnt);
      LaunchScope ls("nv12_to_rgb_kernel", st);
      nv12_to_rgb16_kernel<<<grid, 128, 0, st>>>(l, c, r, pitch, height, rgb_pitch, units);
    } else {
      dim3 grid((unsigned)((quads + 255) / 256), (unsigned)height, (unsigned)cnt);
      LaunchScope ls("nv12_to_rgb_kernel", st);
      nv12_to_rgb_kernel<<<grid, 256, 0, st>>>(l, c, r, pitch, width, height, rgb_pitch, quads,
                                             vec_ok);
    }
    int rc = launch_status();
    if (rc) return rc;
  }
  return 0;
}
