// jpeg.cu -- baseline JPEG encoding of u8 frames (sm_90a), byte for byte what cv2.imencode('.jpg') writes.
// cv2 encodes through libjpeg(-turbo) with its defaults; each step below is libjpeg's integer arithmetic
// (oracle/jpeg.py restates the same steps in numpy and is held to cv2.imencode):
//   colour     rgb_ycc_convert, 16-bit fixed point; gray frames are coded as they are
//   edges      the last pixel column / row replicated out to the block grid; for 4:2:0 chroma the last pixel row
//              is duplicated only when H is odd, ceil(H/2) rows are downsampled, then the last chroma row is
//              replicated down to the block height
//   4:2:0      (a + b + c + d + bias) >> 2, bias 1, 2, 1, 2, ... along each chroma row
//   FDCT       jpeg_fdct_islow (CONST_BITS 13, PASS1_BITS 2) on samples - 128
//   quantise   rounded division of |coef| by 8 q, sign restored; q from the Annex K tables scaled by quality
//   entropy    Annex K Huffman tables, one DC predictor per component, MCUs in row-major order; colour MCUs are
//              Y0 Y1 Y2 Y3 Cb Cr, and Y blocks outside the ceil(W/8) x ceil(H/8) grid are dummy blocks (AC zero,
//              the DC of the block coded before them); 1-bits pad the last byte, 0x00 follows every 0xFF.
// Five kernels per launch of at most 64 frames, every stage parallel:
//   jpeg_mcu_kernel<C, false>  one thread per MCU: colour, downsampling, FDCT, quantisation; records every
//                              block's quantised DC and the bit count of the MCU's AC symbols
//   jpeg_scan_kernel           one CTA per frame: adds the DC-difference bits, scans MCU bit counts into offsets
//   jpeg_mcu_kernel<C, true>   recomputes each MCU from the pixels and writes its bits at its offset (the words
//                              an MCU shares with its neighbours with atomicOr)
//   jpeg_count_ff_kernel       0xFF bytes per 4 KiB chunk of each frame's bit stream
//   jpeg_stuff_kernel          copies each chunk with a 0x00 after every 0xFF, and places the header and EOI
// The last two are the output stage of bitstream.cuh with the escape rule FfStuffing; the stage also reads back
// each frame's bit count (to size the bit streams) and its 0xFF count (to size the output).
#include <cuda_runtime.h>

#include <vector>

#include "bitstream.cuh"

namespace scn {
namespace {

constexpr int kMaxDim = 65500;  // libjpeg's JPEG_MAX_DIMENSION
constexpr int kThreads = 128;   // MCU kernels

// ---- tables (Annex K) ----
constexpr uint8_t kLumaQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
constexpr uint8_t kChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
                                  24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
                                  99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                  99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
struct HuffSpec {
  uint8_t bits[16];  // number of codes of length 1..16
  uint8_t vals[162];
  int nvals;
};
const HuffSpec kDcLuma = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}, 12};
const HuffSpec kDcChroma = {{0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}, 12};
const HuffSpec kAcLuma = {
    {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125},
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71,
     0x14, 0x32, 0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0, 0x24, 0x33, 0x62, 0x72,
     0x82, 0x09, 0x0A, 0x16, 0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x34, 0x35, 0x36, 0x37,
     0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59,
     0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x83,
     0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3,
     0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3,
     0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA, 0xE1, 0xE2,
     0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8, 0xF9, 0xFA},
    162};
const HuffSpec kAcChroma = {
    {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22,
     0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0, 0x15, 0x62, 0x72, 0xD1,
     0x0A, 0x16, 0x24, 0x34, 0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x35, 0x36,
     0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58,
     0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A,
     0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A,
     0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA,
     0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA,
     0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8, 0xF9, 0xFA},
    162};

// Zig-zag position of natural (row-major) coefficient i; folds to a constant in unrolled code.
__host__ __device__ constexpr int zz_pos(int i) {
  const int r = i >> 3, c = i & 7, s = r + c;
  const int along = (s & 1) ? r : c;
  return s <= 7 ? s * (s + 1) / 2 + along : 64 - (14 - s) * (15 - s) / 2 - (15 - s) + along - (s - 7);
}

// What the MCU kernels read, built on the host per quality; it travels in the parameter block and each CTA copies
// it to shared memory (the Huffman lookups diverge, which the constant bank would serialise).
struct Tables {
  uint32_t qmag[2][64];  // natural order: ceil(2^32 / 8q); (x * qmag) >> 32 == x / 8q for every x < 2^17
  uint16_t qdiv[2][64];  // natural order: 8q
  uint32_t dc[2][12];    // category -> code << 8 | length
  uint32_t ac[2][256];   // (run << 4 | size) -> code << 8 | length
};

void huff_table(const HuffSpec& s, uint32_t* out, int entries) {
  for (int i = 0; i < entries; ++i) out[i] = 0;
  uint32_t code = 0;
  int k = 0;
  for (int len = 1; len <= 16; ++len) {
    for (int j = 0; j < s.bits[len - 1]; ++j) out[s.vals[k++]] = code++ << 8 | (uint32_t)len;
    code <<= 1;
  }
}

int quant(int base, int quality) {  // jpeg_set_quality with force_baseline
  const int s = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  const int q = (base * s + 50) / 100;
  return q < 1 ? 1 : (q > 255 ? 255 : q);
}

Tables make_tables(int quality) {
  Tables t;
  for (int c = 0; c < 2; ++c)
    for (int i = 0; i < 64; ++i) {
      const uint32_t d = 8u * (uint32_t)quant(c ? kChromaQ[i] : kLumaQ[i], quality);
      t.qdiv[c][i] = (uint16_t)d;
      t.qmag[c][i] = (uint32_t)(((1ull << 32) + d - 1) / d);
    }
  huff_table(kDcLuma, t.dc[0], 12);
  huff_table(kDcChroma, t.dc[1], 12);
  huff_table(kAcLuma, t.ac[0], 256);
  huff_table(kAcChroma, t.ac[1], 256);
  return t;
}

// SOI, APP0 (JFIF 1.01, no units, density 1 x 1), DQT per table, SOF0, DHT per table (DC0 AC0 DC1 AC1), SOS:
// 623 bytes in colour, within the output stage's kMaxPrefix.
std::vector<uint8_t> make_header(int w, int h, int channels, int quality) {
  std::vector<uint8_t> o = {0xFF, 0xD8};
  auto marker = [&](uint8_t m, const std::vector<uint8_t>& p) {
    const size_t len = p.size() + 2;
    o.insert(o.end(), {0xFF, m, (uint8_t)(len >> 8), (uint8_t)len});
    o.insert(o.end(), p.begin(), p.end());
  };
  marker(0xE0, {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0});
  const int ntab = channels == 3 ? 2 : 1;
  for (int t = 0; t < ntab; ++t) {
    std::vector<uint8_t> p(65);
    p[0] = (uint8_t)t;
    for (int i = 0; i < 64; ++i) p[1 + zz_pos(i)] = (uint8_t)quant(t ? kChromaQ[i] : kLumaQ[i], quality);
    marker(0xDB, p);
  }
  std::vector<uint8_t> sof = {8, (uint8_t)(h >> 8), (uint8_t)h, (uint8_t)(w >> 8), (uint8_t)w, (uint8_t)channels};
  if (channels == 3)
    sof.insert(sof.end(), {1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1});
  else
    sof.insert(sof.end(), {1, 0x11, 0});
  marker(0xC0, sof);
  const HuffSpec* specs[2][2] = {{&kDcLuma, &kAcLuma}, {&kDcChroma, &kAcChroma}};
  for (int t = 0; t < ntab; ++t)
    for (int ac = 0; ac < 2; ++ac) {
      const HuffSpec& s = *specs[t][ac];
      std::vector<uint8_t> p = {(uint8_t)(ac << 4 | t)};
      p.insert(p.end(), s.bits, s.bits + 16);
      p.insert(p.end(), s.vals, s.vals + s.nvals);
      marker(0xC4, p);
    }
  if (channels == 3)
    marker(0xDA, {3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0});
  else
    marker(0xDA, {1, 1, 0x00, 0, 63, 0});
  return o;
}

// ---- geometry ----
struct Geom {
  int w, h, c;
  int mw, mh;  // MCUs per row / column (16 x 16 for colour, 8 x 8 for gray)
  int bpm;     // blocks per MCU
  int bw, bh;  // real Y blocks per row / column
  int ch_rows; // rows of the downsampled chroma planes before replication (ceil(H / 2))
  __host__ __device__ uint32_t mcus() const { return (uint32_t)mw * (uint32_t)mh; }
};

Geom make_geom(int w, int h, int c) {
  Geom g;
  g.w = w, g.h = h, g.c = c;
  const int m = c == 3 ? 16 : 8;
  g.mw = (w + m - 1) / m, g.mh = (h + m - 1) / m;
  g.bpm = c == 3 ? 6 : 1;
  g.bw = (w + 7) / 8, g.bh = (h + 7) / 8;
  g.ch_rows = (h + 1) / 2;
  return g;
}

// ---- one block: samples -> FDCT -> quantised coefficients in zig-zag order (shared memory) ----

// Y of pixel (x, y) of a frame with C channels.
template <int C>
__device__ __forceinline__ int luma(const uint8_t* __restrict__ p) {
  if constexpr (C == 1) {
    return __ldg(p);
  } else {
    const int r = __ldg(p), g = __ldg(p + 1), b = __ldg(p + 2);
    return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
  }
}
// Cb (K == 1) or Cr (K == 2) of one pixel
template <int K>
__device__ __forceinline__ int chroma(const uint8_t* __restrict__ p) {
  const int r = __ldg(p), g = __ldg(p + 1), b = __ldg(p + 2);
  constexpr int bias = (128 << 16) + 32767;
  if constexpr (K == 1)
    return (-11059 * r - 21709 * g + 32768 * b + bias) >> 16;
  else
    return (32768 * r - 27439 * g - 5329 * b + bias) >> 16;
}

// The loaders write a block's samples - 128 to zz[i * kThreads] (natural order), where fdct_quant picks them up: one
// call site of the FDCT for every kind of block keeps it in registers.

// the Y block at block column bx, block row by, edges replicated
template <int C>
__device__ __forceinline__ void load_luma(const uint8_t* __restrict__ src, const Geom& g, int bx, int by,
                                          int16_t* zz) {
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const uint8_t* row = src + (size_t)min(8 * by + r, g.h - 1) * g.w * C;
#pragma unroll
    for (int c = 0; c < 8; ++c)
      zz[(8 * r + c) * kThreads] = (int16_t)(luma<C>(row + (size_t)min(8 * bx + c, g.w - 1) * C) - 128);
  }
}

// the Cb or Cr block of MCU (mx, my): h2v2 downsampling with libjpeg's edge handling
template <int K>
__device__ __forceinline__ void load_chroma(const uint8_t* __restrict__ src, const Geom& g, int mx, int my,
                                            int16_t* zz) {
#pragma unroll 1
  for (int r = 0; r < 8; ++r) {
    const int cy = min(8 * my + r, g.ch_rows - 1);
    const uint8_t* r0 = src + (size_t)(2 * cy) * g.w * 3;
    const uint8_t* r1 = src + (size_t)min(2 * cy + 1, g.h - 1) * g.w * 3;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const size_t x0 = (size_t)min(16 * mx + 2 * c, g.w - 1) * 3, x1 = (size_t)min(16 * mx + 2 * c + 1, g.w - 1) * 3;
      const int s = chroma<K>(r0 + x0) + chroma<K>(r0 + x1) + chroma<K>(r1 + x0) + chroma<K>(r1 + x1);
      zz[(8 * r + c) * kThreads] = (int16_t)(((s + 1 + (c & 1)) >> 2) - 128);
    }
  }
}

constexpr int kConstBits = 13, kPass1Bits = 2;

// one pass of jpeg_fdct_islow over the 8 values d[o], d[o + s], ..., d[o + 7 s]
template <bool Pass1>
__device__ __forceinline__ void fdct8(int (&d)[64], int o, int s) {
  constexpr int sh = Pass1 ? kConstBits - kPass1Bits : kConstBits + kPass1Bits;
  auto descale = [](int x, int n) { return (x + (1 << (n - 1))) >> n; };
  int t0 = d[o] + d[o + 7 * s], t7 = d[o] - d[o + 7 * s];
  int t1 = d[o + s] + d[o + 6 * s], t6 = d[o + s] - d[o + 6 * s];
  int t2 = d[o + 2 * s] + d[o + 5 * s], t5 = d[o + 2 * s] - d[o + 5 * s];
  int t3 = d[o + 3 * s] + d[o + 4 * s], t4 = d[o + 3 * s] - d[o + 4 * s];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  if (Pass1) {
    d[o] = (t10 + t11) << kPass1Bits;
    d[o + 4 * s] = (t10 - t11) << kPass1Bits;
  } else {
    d[o] = descale(t10 + t11, kPass1Bits);
    d[o + 4 * s] = descale(t10 - t11, kPass1Bits);
  }
  int z1 = (t12 + t13) * 4433;
  d[o + 2 * s] = descale(z1 + t13 * 6270, sh);
  d[o + 6 * s] = descale(z1 - t12 * 15137, sh);
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * 9633;
  t4 *= 2446, t5 *= 16819, t6 *= 25172, t7 *= 12299;
  z1 *= -7373, z2 *= -20995, z3 = z3 * -16069 + z5, z4 = z4 * -3196 + z5;
  d[o + 7 * s] = descale(t4 + z1 + z3, sh);
  d[o + 5 * s] = descale(t5 + z2 + z4, sh);
  d[o + 3 * s] = descale(t6 + z2 + z3, sh);
  d[o + s] = descale(t7 + z1 + z4, sh);
}

// FDCT and quantisation of the samples a loader left in zz; writes the coefficients back to zz[k * kThreads]
// (zig-zag position k) and returns the mask of nonzero AC positions (bit k).
__device__ __forceinline__ uint64_t fdct_quant(const uint32_t* qmag, const uint16_t* qdiv, int16_t* zz) {
  int d[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = zz[i * kThreads];
#pragma unroll
  for (int r = 0; r < 8; ++r) fdct8<true>(d, 8 * r, 1);
#pragma unroll
  for (int c = 0; c < 8; ++c) fdct8<false>(d, c, 8);
  uint64_t nz = 0;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int v = d[i];
    const uint32_t a = (uint32_t)abs(v);
    const int q = (int)__umulhi(a + (qdiv[i] >> 1), qmag[i]);
    const int k = zz_pos(i);  // a constant once the loop is unrolled
    zz[k * kThreads] = (int16_t)(v < 0 ? -q : q);
    if (k && q) nz |= 1ull << k;
  }
  return nz;
}

__device__ __forceinline__ int bit_length(int v) { return 32 - __clz(abs(v)); }

// bits of the AC symbols of one block (zz in shared memory, nz its nonzero AC mask); with W, also writes them
template <bool Emit>
__device__ __forceinline__ uint32_t code_ac(const int16_t* zz, uint64_t nz, const uint32_t* ac, BitWriter* bw) {
  uint32_t bits = 0;
  int prev = 0;
  while (nz) {
    const int k = __ffsll((long long)nz) - 1;
    nz &= nz - 1;
    int run = k - prev - 1;
    const int v = zz[k * kThreads];
    const int nb = bit_length(v);
    for (; run > 15; run -= 16) {
      if (Emit) bw->put(ac[0xF0] >> 8, ac[0xF0] & 0xFF);
      bits += ac[0xF0] & 0xFF;
    }
    const uint32_t sym = ac[(run << 4) | nb];
    if (Emit) bw->put(((sym >> 8) << nb) | ((uint32_t)(v < 0 ? v - 1 : v) & ((1u << nb) - 1)), (int)(sym & 0xFF) + nb);
    bits += (sym & 0xFF) + nb;
    prev = k;
  }
  if (prev != 63) {
    if (Emit) bw->put(ac[0] >> 8, ac[0] & 0xFF);
    bits += ac[0] & 0xFF;
  }
  return bits;
}

__device__ __forceinline__ void code_dc(int diff, const uint32_t* dc, BitWriter& bw) {
  const int nb = bit_length(diff);
  const uint32_t sym = dc[nb];
  bw.put(((sym >> 8) << nb) | ((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << nb) - 1)), (int)(sym & 0xFF) + nb);
}

// block b of MCU m: table (0 luma, 1 chroma) and the index in dcs of the DC its difference is taken against (-1: 0)
__device__ __forceinline__ int64_t prev_dc_index(int bpm, uint32_t m, int b) {
  if (bpm == 1) return (int64_t)m - 1;
  if (b >= 1 && b <= 3) return (int64_t)m * 6 + b - 1;
  if (m == 0) return -1;
  return (int64_t)(m - 1) * 6 + (b == 0 ? 3 : b);
}

struct MeasureOut {
  int16_t* dc;      // [frame][mcu][bpm] quantised DC (a dummy block holds its predecessor's)
  uint32_t* acbits; // [frame][mcu] bits of the MCU's AC symbols
};
struct EmitIn {
  const int16_t* dc;
  const uint64_t* mcu_bit;  // [frame][mcu] bit offset of the MCU within its frame's stream
  const uint64_t* total;    // [frame] bits of each frame's stream
  uint8_t* streams;
  uint64_t stream_off[SCN_MAX_PTRS];  // byte offset of each frame's stream in `streams` (a multiple of 16)
};

// One thread per MCU.  !Emit: records DCs and AC bit counts.  Emit: writes the MCU's bits.
template <int C, bool Emit>
__global__ void __launch_bounds__(kThreads)
jpeg_mcu_kernel(PtrBatch srcs, int i0, Geom g, const __grid_constant__ Tables tables, MeasureOut mo,
                const __grid_constant__ EmitIn ei) {
  __shared__ Tables t;
  __shared__ int16_t zzs[64 * kThreads];
  for (int i = threadIdx.x; i < (int)(sizeof(Tables) / 4); i += kThreads)
    reinterpret_cast<uint32_t*>(&t)[i] = reinterpret_cast<const uint32_t*>(&tables)[i];
  __syncthreads();
  const uint32_t m = blockIdx.x * kThreads + threadIdx.x;
  const uint32_t nm = g.mcus();
  if (m >= nm) return;
  const int f = i0 + (int)blockIdx.y;
  const uint8_t* __restrict__ src = srcs.p[blockIdx.y];
  const int mx = (int)(m % (uint32_t)g.mw), my = (int)(m / (uint32_t)g.mw);
  int16_t* zz = zzs + threadIdx.x;
  const size_t rec = (size_t)f * nm + m;
  constexpr int bpm = C == 3 ? 6 : 1;
  int16_t* dcs = Emit ? nullptr : mo.dc + (size_t)f * nm * bpm;
  const int16_t* dcr = Emit ? ei.dc + (size_t)f * nm * bpm : nullptr;

  BitWriter bw(Emit ? reinterpret_cast<uint32_t*>(ei.streams + ei.stream_off[blockIdx.y]) : nullptr,
               Emit ? ei.mcu_bit[rec] : 0);
  uint32_t acbits = 0;
  int16_t last_dc = 0;
#pragma unroll 1
  for (int b = 0; b < bpm; ++b) {
    const int tab = b < 4 ? 0 : 1;
    bool real = true;
    if constexpr (C == 1) {
      load_luma<1>(src, g, mx, my, zz);
    } else if (b < 4) {
      const int bx = 2 * mx + (b & 1), by = 2 * my + (b >> 1);
      real = bx < g.bw && by < g.bh;
      if (real) load_luma<3>(src, g, bx, by, zz);
    } else if (b == 4) {
      load_chroma<1>(src, g, mx, my, zz);
    } else {
      load_chroma<2>(src, g, mx, my, zz);
    }
    uint64_t nz = 0;
    int16_t dc = last_dc;  // a dummy block's DC is its predecessor's
    if (real) {
      nz = fdct_quant(t.qmag[tab], t.qdiv[tab], zz);
      dc = zz[0];
    }
    if constexpr (Emit) {
      const int64_t p = prev_dc_index(bpm, m, b);
      code_dc(dc - (p < 0 ? 0 : dcr[p]), t.dc[tab], bw);
    } else {
      dcs[(size_t)m * bpm + b] = dc;
    }
    if (real) acbits += code_ac<Emit>(zz, nz, t.ac[tab], &bw);
    else acbits += code_ac<Emit>(zz, 0, t.ac[tab], &bw);  // EOB
    last_dc = dc;
  }
  if constexpr (Emit) {
    if (m == nm - 1) {  // 1-bits pad the last byte of the frame
      const int pad = (int)((8 - (ei.total[f] & 7)) & 7);
      if (pad) bw.put((1u << pad) - 1, pad);
    }
    bw.finish();
  } else {
    mo.acbits[rec] = acbits;
  }
}

// One CTA per frame: MCU bit counts (AC bits + DC difference bits) -> bit offsets, and the frame's total.
__global__ void __launch_bounds__(1024)
jpeg_scan_kernel(int i0, uint32_t nm, int bpm, Tables tables, const int16_t* dcs_all, const uint32_t* acbits_all,
                 uint64_t* mcu_bit_all, uint64_t* total) {
  __shared__ uint32_t dclen[2][12];
  if (threadIdx.x < 24) dclen[threadIdx.x / 12][threadIdx.x % 12] = tables.dc[threadIdx.x / 12][threadIdx.x % 12] & 0xFF;
  __syncthreads();
  const int f = i0 + (int)blockIdx.x;
  const int16_t* dcs = dcs_all + (size_t)f * nm * bpm;
  const uint32_t* acbits = acbits_all + (size_t)f * nm;
  uint64_t* mcu_bit = mcu_bit_all + (size_t)f * nm;
  const uint32_t per = (nm + blockDim.x - 1) / blockDim.x;
  const uint32_t m0 = min(nm, threadIdx.x * per), m1 = min(nm, m0 + per);
  auto mcu_bits = [&](uint32_t m) {
    uint64_t bits = acbits[m];
    for (int b = 0; b < bpm; ++b) {
      const int64_t p = prev_dc_index(bpm, m, b);
      const int nb = bit_length(dcs[(size_t)m * bpm + b] - (p < 0 ? 0 : dcs[p]));
      bits += dclen[b < 4 ? 0 : 1][nb] + nb;
    }
    return bits;
  };
  uint64_t sum = 0;
  for (uint32_t m = m0; m < m1; ++m) sum += mcu_bits(m);
  uint64_t all;
  uint64_t off = block_exclusive_scan<unsigned long long>(sum, reinterpret_cast<unsigned long long*>(&all));
  for (uint32_t m = m0; m < m1; ++m) {
    mcu_bit[m] = off;
    off += mcu_bits(m);
  }
  if (threadIdx.x == 0) total[f] = all;
}

// B.1.1.5: a 0x00 after every 0xFF of the scan
struct FfStuffing {
  static constexpr const char* count_name = "jpeg_count_ff_kernel";
  static constexpr const char* copy_name = "jpeg_stuff_kernel";
  static __device__ __forceinline__ int count(const uint8_t*, uint64_t, const uint4& v, int valid) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    int c = 0;
#pragma unroll
    for (int k = 0; k < 16; ++k) c += (k < valid) && ((w[k >> 2] >> (8 * (k & 3))) & 0xFF) == 0xFF;
    return c;
  }
  static __device__ __forceinline__ uint8_t* copy(const uint8_t*, uint64_t, const uint4& v, int valid, uint8_t* o) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    for (int k = 0; k < valid; ++k) {
      const uint8_t b = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
      *o++ = b;
      if (b == 0xFF) *o++ = 0;
    }
    return o;
  }
};

size_t worst_bits_per_block() { return 11 + 11 + 63 * (16 + 10); }  // DC code + value, 63 AC codes + values

}  // namespace
}  // namespace scn

extern "C" size_t scn_jpeg_encode_bound(int width, int height, int channels) {
  using namespace scn;
  if (width <= 0 || height <= 0 || width > kMaxDim || height > kMaxDim || (channels != 1 && channels != 3)) return 0;
  const Geom g = make_geom(width, height, channels);
  const size_t blocks = (size_t)g.mcus() * g.bpm;
  const size_t bytes = (blocks * worst_bits_per_block() + 7) / 8;
  return make_header(width, height, channels, 95).size() + 2 * bytes + 2;
}

extern "C" int scn_jpeg_encode_u8(const uint8_t* const* host_src_ptrs, int n, int width, int height, int channels,
                                  int quality, scn_alloc_fn alloc_out, void* alloc_ctx, size_t* host_sizes,
                                  void* stream) {
  using namespace scn;
  if (n < 0 || width <= 0 || height <= 0 || quality < 1 || quality > 100) return SCN_E_BADARG;
  if (channels != 1 && channels != 3) return SCN_E_UNSUPPORTED;
  if (width > kMaxDim || height > kMaxDim) return SCN_E_UNSUPPORTED;
  if (n == 0) return 0;
  if (!host_src_ptrs || !alloc_out || !host_sizes) return SCN_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemPool_t pool = scratch_pool();
  if (!pool) return (int)cudaErrorMemoryAllocation;
  const Geom g = make_geom(width, height, channels);
  const uint32_t nm = g.mcus();
  const Tables tables = make_tables(quality);
  Affixes ax;
  if (!make_affixes(&ax, make_header(width, height, channels, quality), {}, {0xFF, 0xD9})) return SCN_E_UNSUPPORTED;

  Scratch s{st, {}};
  int16_t* dcs = s.get<int16_t>((size_t)n * nm * g.bpm, pool);
  uint32_t* acbits = s.get<uint32_t>((size_t)n * nm, pool);
  uint64_t* mcu_bit = s.get<uint64_t>((size_t)n * nm, pool);
  uint64_t* bits = s.get<uint64_t>((size_t)n, pool);
  if (!dcs || !acbits || !mcu_bit || !bits) return (int)cudaErrorMemoryAllocation;
  const dim3 mcu_grid((nm + kThreads - 1) / kThreads);

  // DCs and AC bit counts, then per-frame scans into bit offsets
  auto measure = [&] {
    return for_each_chunk(n, [&](int i0, int cnt) {
      const PtrBatch src = gather<PtrBatch>(host_src_ptrs, i0, cnt);
      const MeasureOut mo = {dcs, acbits};
      const dim3 grid(mcu_grid.x, (unsigned)cnt);
      const int e = launch_kernel("jpeg_mcu_kernel<measure>", st, [&] {
        if (channels == 3)
          jpeg_mcu_kernel<3, false><<<grid, kThreads, 0, st>>>(src, i0, g, tables, mo, EmitIn{});
        else
          jpeg_mcu_kernel<1, false><<<grid, kThreads, 0, st>>>(src, i0, g, tables, mo, EmitIn{});
      });
      if (e) return e;
      return launch_kernel("jpeg_scan_kernel", st, [&] {
        jpeg_scan_kernel<<<cnt, 1024, 0, st>>>(i0, nm, g.bpm, tables, dcs, acbits, mcu_bit, bits);
      });
    });
  };
  // each MCU's bits at its offset in its frame's stream
  auto emit = [&](int i0, int cnt, uint8_t* streams, const uint64_t* stream_off) {
    const PtrBatch src = gather<PtrBatch>(host_src_ptrs, i0, cnt);
    EmitIn ei = {dcs, mcu_bit, bits, streams, {}};
    for (int j = 0; j < cnt; ++j) ei.stream_off[j] = stream_off[j];
    const dim3 grid(mcu_grid.x, (unsigned)cnt);
    return launch_kernel("jpeg_mcu_kernel<emit>", st, [&] {
      if (channels == 3)
        jpeg_mcu_kernel<3, true><<<grid, kThreads, 0, st>>>(src, i0, g, tables, MeasureOut{}, ei);
      else
        jpeg_mcu_kernel<1, true><<<grid, kThreads, 0, st>>>(src, i0, g, tables, MeasureOut{}, ei);
    });
  };
  return run_output_stage<FfStuffing>(n, st, pool, s, bits, nullptr, ax, measure, emit, alloc_out, alloc_ctx,
                                      host_sizes);
}
