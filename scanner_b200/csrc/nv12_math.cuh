// nv12_math.cuh -- the reference's NV12 -> RGB arithmetic (scanner/util/image.cu:67-102,
// :109-200), written once for every kernel that consumes decoder surfaces.
//   Y' = Y<<2, C' = (C<<2)-512 (10-bit widen), float matrix {1.1644,0,1.596; 1.1644,-.3918,
//   -.813; 1.1644,2.0172,0}, clamp [0,1023], truncate, >>2.  On odd luma rows (except the last
//   chroma row) chroma is the rounded average of the two neighbouring chroma rows (:133-151).
// The products are contracted the way nvcc (12.9, default -fmad) contracts the reference
// source `y*k0 + cb*k1 + cr*k2` -- read off the SASS of the unmodified image.cu (oracle/_ref):
//     fma(cr, k2, fma(y, k0, fl(cb * k1)))          the MIDDLE product is rounded on its own.
// Terms with a zero coefficient are dropped (x + (+-0) == x, and fl(y*k0 + (+-0)) == fl(y*k0)).
// tests/test_ref_pin_gpu.py holds every kernel built on this to the reference kernel's own output
// over all 2^24 (Y,Cb,Cr) triples.
#pragma once
#include <stdint.h>

namespace scn {

struct Rgb8 {
  uint32_t r, g, b;
};

__device__ __forceinline__ uint32_t pack10(float v) {
  v = fminf(fmaxf(v, 0.0f), 1023.f);
  return ((uint32_t)v) >> 2;
}

// The arithmetic as the reference writes it (int -> float conversions, clamp, float -> int):
// kept as the readable statement of what yuv_to_rgb() below must equal.
__device__ __forceinline__ Rgb8 yuv_to_rgb_plain(uint32_t y, uint32_t cb, uint32_t cr) {
  const float l = (float)(y << 2);
  const float fcb = (float)((int)(cb << 2) - 512);
  const float fcr = (float)((int)(cr << 2) - 512);
  Rgb8 o;
  o.r = pack10(__fmaf_rn(fcr, 1.596f, __fmul_rn(l, 1.1644f)));
  o.g = pack10(__fmaf_rn(fcr, -0.813f, __fmaf_rn(l, 1.1644f, __fmul_rn(fcb, -0.3918f))));
  o.b = pack10(__fmaf_rn(l, 1.1644f, __fmul_rn(fcb, 2.0172f)));
  return o;
}

// Same values without the conversion unit (I2F / F2I issue at a quarter of the FMA rate): the
// operands enter as 2^23 + byte bit patterns, the matrix runs in a 2^-11 scaled domain (exact:
// power-of-two scaling commutes with IEEE rounding), fma.sat is the lower clamp, and the 8-bit
// result is read from the mantissa of fma.rm(x, 512, 2^23).  Bit-identical to yuv_to_rgb_plain for
// all 2^24 inputs (tests compare every kernel built on it with the oracle).
__device__ __forceinline__ Rgb8 yuv_to_rgb(uint32_t y, uint32_t cb, uint32_t cr) {
  constexpr float s = 1.0f / 2048.0f, magic = 8388608.0f, top = 1023.0f * s;
  constexpr float cy = 4.0f * 1.1644f * s, kr = 4.0f * 1.596f * s, kg1 = 4.0f * -0.3918f * s;
  constexpr float kg2 = 4.0f * -0.813f * s, kb = 4.0f * 2.0172f * s;
  const float yf = __uint_as_float(0x4B000000u | y) - magic;
  const float fcb = __uint_as_float(0x4B000000u | cb) - (magic + 128.0f);
  const float fcr = __uint_as_float(0x4B000000u | cr) - (magic + 128.0f);
  float r, g, b;
  asm("fma.rn.sat.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(fcr), "f"(kr), "f"(__fmul_rn(yf, cy)));
  asm("fma.rn.sat.f32 %0, %1, %2, %3;" : "=f"(g) : "f"(fcr), "f"(kg2), "f"(__fmaf_rn(yf, cy, __fmul_rn(fcb, kg1))));
  asm("fma.rn.sat.f32 %0, %1, %2, %3;" : "=f"(b) : "f"(yf), "f"(cy), "f"(__fmul_rn(fcb, kb)));
  auto u8bits = [&](float x) {
    float q;
    asm("fma.rm.f32 %0, %1, %2, %3;" : "=f"(q) : "f"(fminf(x, top)), "f"(512.0f), "f"(magic));
    return __float_as_uint(q) & 0xFFu;
  };
  Rgb8 o;
  o.r = u8bits(r);
  o.g = u8bits(g);
  o.b = u8bits(b);
  return o;
}

// chroma sample pair for luma row y at (even) column xc
__device__ __forceinline__ void chroma_at(const uint8_t* __restrict__ chroma, size_t pitch,
                                          int height, int y, int xc, uint32_t& cb,
                                          uint32_t& cr) {
  const int yc = y >> 1;
  const uint8_t* c0 = chroma + (size_t)yc * pitch + xc;
  cb = c0[0];
  cr = c0[1];
  if ((y & 1) && yc < ((height >> 1) - 1)) {
    cb = (cb + c0[pitch] + 1) >> 1;
    cr = (cr + c0[pitch + 1] + 1) >> 1;
  }
}

__device__ __forceinline__ Rgb8 nv12_pixel(const uint8_t* __restrict__ luma,
                                           const uint8_t* __restrict__ chroma, size_t pitch,
                                           int height, int x, int y) {
  uint32_t cb, cr;
  chroma_at(chroma, pitch, height, y, x & ~1, cb, cr);
  return yuv_to_rgb(luma[(size_t)y * pitch + x], cb, cr);
}

}  // namespace scn
