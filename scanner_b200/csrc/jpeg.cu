// jpeg.cu -- baseline JPEG encoding of u8 frames (sm_90a), byte for byte what cv2.imencode('.jpg') writes.
// cv2 encodes through libjpeg(-turbo) with its defaults; each step below is libjpeg's integer arithmetic
// (oracle/jpeg.py restates the same steps in numpy and is held to cv2.imencode):
//   colour     rgb_ycc_convert, 16-bit fixed point; gray frames are coded as they are
//   sampling   luma factors (h, v), chroma at (1, 1): 4:2:0 (2, 2) by default, or 4:4:4 (1, 1), 4:2:2 (2, 1),
//              4:4:0 (1, 2), 4:1:1 (4, 1) (cv2's IMWRITE_JPEG_SAMPLING_FACTOR); an MCU is 8h x 8v pixels
//   edges      the last pixel column / row replicated out to the block grid; for chroma the last pixel row is
//              replicated out to a multiple of v, ceil(H/v) rows are downsampled, then the last chroma row is
//              replicated down to the block height (jcprepct.c)
//   downsample jcsample.c: 4:2:0 (a + b + c + d + bias) >> 2, bias 1, 2, 1, 2, ... along each chroma row; 4:2:2
//              (a + b + bias) >> 1, bias 0, 1, 0, 1, ...; 4:4:0 and 4:1:1 int_downsample, (sum + 2 or 1) / 4 or 2
//   FDCT       jpeg_fdct_islow (CONST_BITS 13, PASS1_BITS 2) on samples - 128
//   quantise   rounded division of |coef| by 8 q, sign restored; q from the Annex K tables scaled by quality, or
//              each table by its own quality as cv2 does with IMWRITE_JPEG_LUMA_QUALITY / _CHROMA_QUALITY
//   entropy    Annex K Huffman tables, one DC predictor per component, MCUs in row-major order; colour MCUs are
//              Y0 .. Y(hv-1) Cb Cr (Y in row-major order within the MCU), and Y blocks outside the
//              ceil(W/8) x ceil(H/8) grid are dummy blocks (AC zero, the DC of the block coded before them);
//              1-bits pad the last byte, 0x00 follows every 0xFF.
// Five kernels per launch of at most 64 frames, every stage parallel:
//   jpeg_mcu_kernel<C, H, V, false>  one thread per MCU: colour, downsampling, FDCT, quantisation; records
//                                    every block's quantised DC and the bit count of the MCU's AC symbols
//   jpeg_scan_kernel                 one CTA per frame: adds the DC-difference bits, scans MCU bit counts into
//                                    offsets
//   jpeg_mcu_kernel<C, H, V, true>   recomputes each MCU from the pixels and writes its bits at its offset (the
//                                    words an MCU shares with its neighbours with atomicOr)
//   jpeg_count_ff_kernel             0xFF bytes per 4 KiB chunk of each frame's bit stream
//   jpeg_stuff_kernel                copies each chunk with a 0x00 after every 0xFF, and places the header and EOI
// The last two are the output stage of bitstream.cuh with the escape rule FfStuffing; the stage also reads back
// each frame's bit count (to size the bit streams) and its 0xFF count (to size the output).  H, V are the luma
// sampling factors (1, 1 for gray frames, which have no chroma and ignore the sampling option).
#include <cuda_runtime.h>

#include <type_traits>
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

Tables make_tables(const int (&quality)[2]) {
  Tables t;
  for (int c = 0; c < 2; ++c)
    for (int i = 0; i < 64; ++i) {
      const uint32_t d = 8u * (uint32_t)quant(c ? kChromaQ[i] : kLumaQ[i], quality[c]);
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
// 623 bytes in colour, within the output stage's kMaxPrefix.  hv: the luma sampling factors h << 4 | v.
std::vector<uint8_t> make_header(int w, int h, int channels, const int (&quality)[2], int hv) {
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
    for (int i = 0; i < 64; ++i) p[1 + zz_pos(i)] = (uint8_t)quant(t ? kChromaQ[i] : kLumaQ[i], quality[t]);
    marker(0xDB, p);
  }
  std::vector<uint8_t> sof = {8, (uint8_t)(h >> 8), (uint8_t)h, (uint8_t)(w >> 8), (uint8_t)w, (uint8_t)channels};
  if (channels == 3)
    sof.insert(sof.end(), {1, (uint8_t)hv, 0, 2, 0x11, 1, 3, 0x11, 1});
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
  int mw, mh;  // MCUs per row / column (8 H x 8 V for colour, 8 x 8 for gray)
  int bpm;     // blocks per MCU
  int ny;      // Y blocks per MCU (H V)
  int bw, bh;  // real Y blocks per row / column
  int ch_rows; // rows of the downsampled chroma planes before replication (ceil(H / V))
  __host__ __device__ uint32_t mcus() const { return (uint32_t)mw * (uint32_t)mh; }
};

// hv: the luma sampling factors h << 4 | v (0x11 for gray frames)
Geom make_geom(int w, int h, int c, int hv) {
  Geom g;
  g.w = w, g.h = h, g.c = c;
  const int sh = hv >> 4, sv = hv & 15;
  g.mw = (w + 8 * sh - 1) / (8 * sh), g.mh = (h + 8 * sv - 1) / (8 * sv);
  g.ny = sh * sv;
  g.bpm = c == 3 ? g.ny + 2 : 1;
  g.bw = (w + 7) / 8, g.bh = (h + 7) / 8;
  g.ch_rows = (h + sv - 1) / sv;
  return g;
}

// The encoder's settings after cv2's rules (grfmt_jpeg.cpp, probed on cv2 4.13): a luma quality alone sets both
// tables, a chroma quality alone is ignored, both together scale each table by its own, and two different ones
// force 4:4:4 whatever the sampling option says.  Gray frames have one table and no chroma: luma quality (or
// quality) and 1 x 1.  False for an unknown sampling or a quality outside 1-100.
struct Settings {
  int quality[2];  // luma, chroma table
  int hv;          // luma sampling factors h << 4 | v
};

bool settings(int channels, int quality, const scn_jpeg_options* o, Settings* s) {
  const scn_jpeg_options none = {0, 0, 0, 0};
  if (!o) o = &none;
  const int hv = o->sampling ? o->sampling : 0x22;
  if (hv != 0x11 && hv != 0x21 && hv != 0x22 && hv != 0x12 && hv != 0x41) return false;
  for (int q : {quality, o->luma_quality, o->chroma_quality})
    if (q < 0 || q > 100) return false;
  if (quality < 1 || o->optimize < 0 || o->optimize > 1) return false;
  const int lq = o->luma_quality ? o->luma_quality : quality;
  const int cq = o->luma_quality && o->chroma_quality ? o->chroma_quality : lq;
  s->quality[0] = lq, s->quality[1] = cq;
  s->hv = channels != 3 ? 0x11 : (lq != cq ? 0x11 : hv);
  return true;
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

// the Cb or Cr block of MCU (mx, my) with luma factors H, V: jcsample.c's downsampling with libjpeg's edge
// handling (the sum of the H x V pixels under each chroma sample, then h2v2, h2v1 or int_downsample's rounding)
template <int K, int H, int V>
__device__ __forceinline__ void load_chroma(const uint8_t* __restrict__ src, const Geom& g, int mx, int my,
                                            int16_t* zz) {
  if constexpr (H == 2 && V == 2) {  // the default, written out
#pragma unroll 1
    for (int r = 0; r < 8; ++r) {
      const int cy = min(8 * my + r, g.ch_rows - 1);
      const uint8_t* r0 = src + (size_t)(2 * cy) * g.w * 3;
      const uint8_t* r1 = src + (size_t)min(2 * cy + 1, g.h - 1) * g.w * 3;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const size_t x0 = (size_t)min(16 * mx + 2 * c, g.w - 1) * 3;
        const size_t x1 = (size_t)min(16 * mx + 2 * c + 1, g.w - 1) * 3;
        const int s = chroma<K>(r0 + x0) + chroma<K>(r0 + x1) + chroma<K>(r1 + x0) + chroma<K>(r1 + x1);
        zz[(8 * r + c) * kThreads] = (int16_t)(((s + 1 + (c & 1)) >> 2) - 128);
      }
    }
    return;
  }
#pragma unroll 1
  for (int r = 0; r < 8; ++r) {
    const int cy = min(8 * my + r, g.ch_rows - 1);
    const uint8_t* rows[V];
    rows[0] = src + (size_t)(V * cy) * g.w * 3;  // V cy <= H - 1 as cy < ceil(H / V)
#pragma unroll
    for (int dy = 1; dy < V; ++dy) rows[dy] = src + (size_t)min(V * cy + dy, g.h - 1) * g.w * 3;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      int s = 0;
#pragma unroll
      for (int dx = 0; dx < H; ++dx) {
        const size_t x = (size_t)min(8 * H * mx + H * c + dx, g.w - 1) * 3;
#pragma unroll
        for (int dy = 0; dy < V; ++dy) s += chroma<K>(rows[dy] + x);
      }
      int v;
      if constexpr (H == 1 && V == 1) v = s;                              // fullsize_downsample
      else if constexpr (H == 2 && V == 1) v = (s + (c & 1)) >> 1;        // h2v1_downsample
      else v = (s + H * V / 2) / (H * V);                                 // int_downsample
      zz[(8 * r + c) * kThreads] = (int16_t)(v - 128);
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

// bits of the AC symbols of one block (zz in shared memory, nz its nonzero AC mask); with Emit, also writes them;
// with Count, also adds each symbol to hist (shared memory)
template <bool Emit, bool Count = false>
__device__ __forceinline__ uint32_t code_ac(const int16_t* zz, uint64_t nz, const uint32_t* ac, BitWriter* bw,
                                            uint32_t* hist = nullptr) {
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
      if (Count) atomicAdd(hist + 0xF0, 1u);
      bits += ac[0xF0] & 0xFF;
    }
    if (Count) atomicAdd(hist + ((run << 4) | nb), 1u);
    const uint32_t sym = ac[(run << 4) | nb];
    if (Emit) bw->put(((sym >> 8) << nb) | ((uint32_t)(v < 0 ? v - 1 : v) & ((1u << nb) - 1)), (int)(sym & 0xFF) + nb);
    bits += (sym & 0xFF) + nb;
    prev = k;
  }
  if (prev != 63) {
    if (Emit) bw->put(ac[0] >> 8, ac[0] & 0xFF);
    if (Count) atomicAdd(hist, 1u);
    bits += ac[0] & 0xFF;
  }
  return bits;
}

__device__ __forceinline__ void code_dc(int diff, const uint32_t* dc, BitWriter& bw) {
  const int nb = bit_length(diff);
  const uint32_t sym = dc[nb];
  bw.put(((sym >> 8) << nb) | ((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << nb) - 1)), (int)(sym & 0xFF) + nb);
}

// block b of MCU m (bpm blocks, the first ny of them Y): the index in dcs of the DC its difference is taken against
// (-1: 0)
__device__ __forceinline__ int64_t prev_dc_index(int bpm, int ny, uint32_t m, int b) {
  if (b >= 1 && b < ny) return (int64_t)m * bpm + b - 1;
  if (m == 0) return -1;
  return (int64_t)(m - 1) * bpm + (b == 0 ? ny - 1 : b);
}

struct MeasureOut {
  int16_t* dc;      // [frame][mcu][bpm] quantised DC (a dummy block holds its predecessor's)
  uint32_t* acbits; // [frame][mcu] bits of the MCU's AC symbols
};
// Optimised Huffman tables: the symbol counts the statistics pass gathers and the codes built from them, per frame
constexpr int kCodeWords = 2 * 12 + 2 * 256;  // Tables::dc and Tables::ac
constexpr int kCodeWord0 = (int)(offsetof(Tables, dc) / 4);
struct FrameTables {
  const uint32_t* codes;  // [frame][kCodeWords] in Tables' dc, ac layout; null: the Annex K tables of `tables`
  uint32_t* ac_hist;      // [frame][table][256] AC symbol counts (the statistics pass adds to them)
};
struct EmitIn {
  const int16_t* dc;
  const uint64_t* mcu_bit;  // [frame][mcu] bit offset of the MCU within its frame's stream
  const uint64_t* total;    // [frame] bits of each frame's stream
  uint8_t* streams;
  uint64_t stream_off[SCN_MAX_PTRS];  // byte offset of each frame's stream in `streams` (a multiple of 16)
};

enum { kMeasure, kEmit, kStats };

// The work of the thread of MCU m (see jpeg_mcu_kernel).
template <int C, int H, int V, int Mode>
__device__ __forceinline__ void mcu_body(const PtrBatch& srcs, const Geom& g, uint32_t m, int f, const Tables& t,
                                         int16_t* zzs, const MeasureOut& mo, const EmitIn& ei, uint32_t* hist) {
  constexpr bool Emit = Mode == kEmit, Stats = Mode == kStats;
  const uint32_t nm = g.mcus();
  const uint8_t* __restrict__ src = srcs.p[blockIdx.y];
  const int mx = (int)(m % (uint32_t)g.mw), my = (int)(m / (uint32_t)g.mw);
  int16_t* zz = zzs + threadIdx.x;
  const size_t rec = (size_t)f * nm + m;
  constexpr int ny = H * V, bpm = C == 3 ? ny + 2 : 1;
  int16_t* dcs = Emit ? nullptr : mo.dc + (size_t)f * nm * bpm;
  const int16_t* dcr = Emit ? ei.dc + (size_t)f * nm * bpm : nullptr;

  BitWriter bw(Emit ? reinterpret_cast<uint32_t*>(ei.streams + ei.stream_off[blockIdx.y]) : nullptr,
               Emit ? ei.mcu_bit[rec] : 0);
  uint32_t acbits = 0;
  int16_t last_dc = 0;
#pragma unroll 1
  for (int b = 0; b < bpm; ++b) {
    const int tab = b < ny ? 0 : 1;
    bool real = true;
    if constexpr (C == 1) {
      load_luma<1>(src, g, mx, my, zz);
    } else if (b < ny) {
      const int bx = H * mx + b % H, by = V * my + b / H;
      real = bx < g.bw && by < g.bh;
      if (real) load_luma<3>(src, g, bx, by, zz);
    } else if (b == ny) {
      load_chroma<1, H, V>(src, g, mx, my, zz);
    } else {
      load_chroma<2, H, V>(src, g, mx, my, zz);
    }
    uint64_t nz = 0;
    int16_t dc = last_dc;  // a dummy block's DC is its predecessor's
    if (real) {
      nz = fdct_quant(t.qmag[tab], t.qdiv[tab], zz);
      dc = zz[0];
    }
    if constexpr (Emit) {
      const int64_t p = prev_dc_index(bpm, ny, m, b);
      code_dc(dc - (p < 0 ? 0 : dcr[p]), t.dc[tab], bw);
    } else {
      dcs[(size_t)m * bpm + b] = dc;
    }
    if (real) acbits += code_ac<Emit, Stats>(zz, nz, t.ac[tab], &bw, hist + 256 * tab);
    else acbits += code_ac<Emit, Stats>(zz, 0, t.ac[tab], &bw, hist + 256 * tab);  // EOB
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

// One thread per MCU.  kMeasure: records DCs and AC bit counts.  kEmit: writes the MCU's bits.  kStats: records
// DCs and counts the AC symbols of each table, in shared memory per CTA and then into ft.ac_hist.  PerFrame: the
// Huffman codes are this frame's (ft.codes) instead of those of `tables` (a separate instance, so that the Annex K
// kernels carry nothing of it).
template <int C, int H, int V, int Mode, bool PerFrame>
__global__ void __launch_bounds__(kThreads)
jpeg_mcu_kernel(PtrBatch srcs, int i0, Geom g, const __grid_constant__ Tables tables, MeasureOut mo,
                const __grid_constant__ EmitIn ei, FrameTables ft) {
  constexpr bool Stats = Mode == kStats;
  __shared__ Tables t;
  __shared__ int16_t zzs[64 * kThreads];
  __shared__ uint32_t hist[Stats ? 2 * 256 : 1];
  const int f = i0 + (int)blockIdx.y;
  for (int i = threadIdx.x; i < (int)(sizeof(Tables) / 4); i += kThreads)
    reinterpret_cast<uint32_t*>(&t)[i] = reinterpret_cast<const uint32_t*>(&tables)[i];
  if constexpr (Stats)
    for (int i = threadIdx.x; i < 2 * 256; i += kThreads) hist[i] = 0;
  __syncthreads();
  if constexpr (PerFrame) {  // this frame's codes over the Annex K ones
    for (int i = threadIdx.x; i < kCodeWords; i += kThreads)
      reinterpret_cast<uint32_t*>(&t)[kCodeWord0 + i] = ft.codes[(size_t)f * kCodeWords + i];
    __syncthreads();
  }
  const uint32_t m = blockIdx.x * kThreads + threadIdx.x;
  const uint32_t nm = g.mcus();
  if constexpr (Stats) {
    if (m < nm) mcu_body<C, H, V, Mode>(srcs, g, m, f, t, zzs, mo, ei, hist);
    __syncthreads();
    uint32_t* out = ft.ac_hist + (size_t)f * 2 * 256;
    for (int i = threadIdx.x; i < 2 * 256; i += kThreads)
      if (hist[i]) atomicAdd(out + i, hist[i]);
  } else {
    if (m >= nm) return;
    mcu_body<C, H, V, Mode>(srcs, g, m, f, t, zzs, mo, ei, hist);
  }
}

// One CTA per frame: MCU bit counts (AC bits + DC difference bits) -> bit offsets, and the frame's total.  codes:
// per-frame tables (FrameTables::codes), or null for those of `tables`.
__global__ void __launch_bounds__(1024)
jpeg_scan_kernel(int i0, uint32_t nm, int bpm, int ny, Tables tables, const uint32_t* codes, const int16_t* dcs_all,
                 const uint32_t* acbits_all, uint64_t* mcu_bit_all, uint64_t* total) {
  __shared__ uint32_t dclen[2][12];
  const int f = i0 + (int)blockIdx.x;
  if (threadIdx.x < 24)
    dclen[threadIdx.x / 12][threadIdx.x % 12] =
        (codes ? codes[(size_t)f * kCodeWords + threadIdx.x] : tables.dc[threadIdx.x / 12][threadIdx.x % 12]) & 0xFF;
  __syncthreads();
  const int16_t* dcs = dcs_all + (size_t)f * nm * bpm;
  const uint32_t* acbits = acbits_all + (size_t)f * nm;
  uint64_t* mcu_bit = mcu_bit_all + (size_t)f * nm;
  const uint32_t per = (nm + blockDim.x - 1) / blockDim.x;
  const uint32_t m0 = min(nm, threadIdx.x * per), m1 = min(nm, m0 + per);
  auto mcu_bits = [&](uint32_t m) {
    uint64_t bits = acbits[m];
    for (int b = 0; b < bpm; ++b) {
      const int64_t p = prev_dc_index(bpm, ny, m, b);
      const int nb = bit_length(dcs[(size_t)m * bpm + b] - (p < 0 ? 0 : dcs[p]));
      bits += dclen[b < ny ? 0 : 1][nb] + nb;
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

// ---- optimised Huffman tables ----
// Per frame and table, what the header's DHT segments carry: BITS[1..16] and HUFFVAL, for the DC and the AC table.
struct HuffOut {
  uint8_t bits[2][16];    // [class: 0 DC, 1 AC]
  uint8_t vals[2][256];
  int nvals[2];
};

// jpeg_gen_optimal_table (jchuff.c) on one warp: freq[0..256] (freq[256] is set to 1 here: the reserved code point
// that keeps any code from being all 1-bits) -> o's bits and vals for class cls, and code[symbol] = code << 8 | length
// (0 for a symbol that does not occur).  The two smallest nonzero frequencies are merged until one is left; ties go to
// the larger index (libjpeg's "<=" scan), the second pick excludes the first.  Lengths over 16 are folded back by the
// K.3 adjust loop; HUFFVAL lists the symbols by their unadjusted length, then by value.  Lane 0 does the list walks,
// the warp the minimum searches.  freq, codesize and others are this warp's shared scratch.
__device__ void gen_optimal_table(uint64_t* freq, int* codesize, int* others, HuffOut* o, int cls, uint32_t* code,
                                  int ncode) {
  const int lane = threadIdx.x & 31;
  for (int i = lane; i < 257; i += 32) codesize[i] = 0, others[i] = -1;
  if (lane == 0) freq[256] = 1;
  __syncwarp();
  auto pick = [&](int exclude) {  // the smallest nonzero frequency, the largest index among equals; -1: none
    unsigned long long best = ~0ull;
    for (int i = lane; i < 257; i += 32)
      if (freq[i] && i != exclude) {
        const unsigned long long key = (unsigned long long)freq[i] << 9 | (unsigned)(511 - i);
        best = key < best ? key : best;
      }
#pragma unroll
    for (int d = 16; d; d >>= 1) {
      const unsigned long long y = __shfl_xor_sync(0xFFFFFFFFu, best, d);
      best = y < best ? y : best;
    }
    return best == ~0ull ? -1 : 511 - (int)(best & 511);
  };
  for (;;) {
    int c1 = pick(-1);
    int c2 = pick(c1);
    if (c2 < 0) break;
    if (lane == 0) {
      freq[c1] += freq[c2];
      freq[c2] = 0;
      ++codesize[c1];
      while (others[c1] >= 0) c1 = others[c1], ++codesize[c1];
      others[c1] = c2;
      ++codesize[c2];
      while (others[c2] >= 0) c2 = others[c2], ++codesize[c2];
    }
    __syncwarp();
  }
  if (lane == 0) {
    int bits[33] = {0};
    for (int i = 0; i < 257; ++i)  // libjpeg refuses lengths over 32 (Fibonacci-like counts of over 9 M)
      if (codesize[i]) ++bits[min(codesize[i], 32)];
    for (int i = 32; i > 16; --i)
      while (bits[i] > 0) {
        int j = i - 2;
        while (bits[j] == 0) --j;
        bits[i] -= 2;
        ++bits[i - 1];
        bits[j + 1] += 2;
        --bits[j];
      }
    int i = 16;
    while (i > 0 && bits[i] == 0) --i;
    if (i > 0) --bits[i];  // the reserved code point
    int n = 0;
    for (int len = 1; len <= 32; ++len)
      for (int j = 0; j < 256; ++j)
        if (codesize[j] == len) o->vals[cls][n++] = (uint8_t)j;
    o->nvals[cls] = n;
    for (int k = 0; k < ncode; ++k) code[k] = 0;
    uint32_t c = 0;
    int k = 0;
    for (int len = 1; len <= 16; ++len) {
      o->bits[cls][len - 1] = (uint8_t)bits[len];
      for (int j = 0; j < bits[len]; ++j) code[o->vals[cls][k++]] = c++ << 8 | (uint32_t)len;
      c <<= 1;
    }
  }
  __syncwarp();
}

// The bytes of each frame's header: SOI, APP0, DQT and SOF0 (head), the four DHT segments of its tables, SOS.
struct HeaderParts {
  uint8_t head[kMaxPrefix];
  uint8_t sos[16];
  int head_len, sos_len, ntab;
};

// One CTA of two warps per frame: warp t counts the DC categories of table t's blocks from the recorded DCs, then
// builds table t's DC and AC codes from those counts and the statistics pass's AC counts (gen_optimal_table).  Then
// thread 0 writes the frame's header to prefix[frame] (kMaxPrefix bytes per frame) and its length to prefix_len.
__global__ void __launch_bounds__(64)
jpeg_table_kernel(int i0, uint32_t nm, int bpm, int ny, const int16_t* dcs_all, const uint32_t* ac_hist,
                  uint32_t* codes, uint8_t* prefix, uint32_t* prefix_len, const __grid_constant__ HeaderParts hp) {
  __shared__ uint64_t freq[2][257];
  __shared__ int codesize[2][257], others[2][257];
  __shared__ uint32_t dccount[2][12];
  __shared__ HuffOut out[2];
  const int f = i0 + (int)blockIdx.x, t = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t* code = codes + (size_t)f * kCodeWords;
  if (lane < 12) dccount[t][lane] = 0;
  __syncwarp();
  if (t < hp.ntab) {
    const int16_t* dcs = dcs_all + (size_t)f * nm * bpm;
    const uint64_t blocks = (uint64_t)nm * bpm;
    for (uint64_t i = lane; i < blocks; i += 32) {
      const uint32_t m = (uint32_t)(i / bpm);
      const int b = (int)(i - (uint64_t)m * bpm);
      if ((b < ny ? 0 : 1) != t) continue;
      const int64_t p = prev_dc_index(bpm, ny, m, b);
      atomicAdd(&dccount[t][bit_length(dcs[i] - (p < 0 ? 0 : dcs[p]))], 1u);
    }
    __syncwarp();
    for (int i = lane; i < 257; i += 32) freq[t][i] = i < 12 ? dccount[t][i] : 0;
    __syncwarp();
    gen_optimal_table(freq[t], codesize[t], others[t], &out[t], 0, code + 12 * t, 12);
    const uint32_t* h = ac_hist + ((size_t)f * 2 + t) * 256;
    for (int i = lane; i < 257; i += 32) freq[t][i] = i < 256 ? h[i] : 0;
    __syncwarp();
    gen_optimal_table(freq[t], codesize[t], others[t], &out[t], 1, code + 24 + 256 * t, 256);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint8_t* o = prefix + (size_t)f * kMaxPrefix;
    int n = 0;
    for (int k = 0; k < hp.head_len; ++k) o[n++] = hp.head[k];
    for (int tab = 0; tab < hp.ntab; ++tab)
      for (int cls = 0; cls < 2; ++cls) {
        const int len = 2 + 1 + 16 + out[tab].nvals[cls];
        o[n++] = 0xFF, o[n++] = 0xC4, o[n++] = (uint8_t)(len >> 8), o[n++] = (uint8_t)len;
        o[n++] = (uint8_t)(cls << 4 | tab);
        for (int k = 0; k < 16; ++k) o[n++] = out[tab].bits[cls][k];
        for (int k = 0; k < out[tab].nvals[cls]; ++k) o[n++] = out[tab].vals[cls][k];
      }
    for (int k = 0; k < hp.sos_len; ++k) o[n++] = hp.sos[k];
    prefix_len[f] = (uint32_t)n;
  }
}

// One warp: gen_optimal_table of 257 given frequencies (freq[256] ignored) -> bits, vals, nvals (test entry point)
__global__ void jpeg_gen_table_kernel(const uint64_t* freq_in, uint8_t* bits, uint8_t* vals, int* nvals) {
  __shared__ uint64_t freq[257];
  __shared__ int codesize[257], others[257];
  __shared__ HuffOut out;
  __shared__ uint32_t code[256];
  for (int i = threadIdx.x; i < 257; i += 32) freq[i] = i < 256 ? freq_in[i] : 0;
  __syncwarp();
  gen_optimal_table(freq, codesize, others, &out, 0, code, 256);
  for (int i = threadIdx.x; i < 256; i += 32) vals[i] = out.vals[0][i];
  if (threadIdx.x < 16) bits[threadIdx.x] = out.bits[0][threadIdx.x];
  if (threadIdx.x == 0) *nvals = out.nvals[0];
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

// DC code + value, 63 AC codes + values: Annex K codes are at most 11 (DC) and 16 (AC) bits, optimised ones 16
size_t worst_bits_per_block(bool optimize) { return (optimize ? 16 : 11) + 11 + 63 * (16 + 10); }

// jpeg_mcu_kernel for the channels and luma sampling factors of one call
template <int Mode>
void launch_mcu(int channels, int hv, dim3 grid, cudaStream_t st, const PtrBatch& src, int i0, const Geom& g,
                const Tables& tables, const MeasureOut& mo, const EmitIn& ei, const FrameTables& ft) {
  constexpr bool kOpt = Mode != kStats;  // the statistics pass codes nothing, so it needs no per-frame codes
  auto pick = [&](auto per_frame) {
    constexpr bool P = decltype(per_frame)::value;
    auto k = jpeg_mcu_kernel<1, 1, 1, Mode, P>;
    if (channels == 3) {
      switch (hv) {
        case 0x11: k = jpeg_mcu_kernel<3, 1, 1, Mode, P>; break;
        case 0x21: k = jpeg_mcu_kernel<3, 2, 1, Mode, P>; break;
        case 0x12: k = jpeg_mcu_kernel<3, 1, 2, Mode, P>; break;
        case 0x41: k = jpeg_mcu_kernel<3, 4, 1, Mode, P>; break;
        default: k = jpeg_mcu_kernel<3, 2, 2, Mode, P>; break;
      }
    }
    k<<<grid, kThreads, 0, st>>>(src, i0, g, tables, mo, ei, ft);
  };
  if constexpr (kOpt) {
    if (ft.codes) return pick(std::true_type{});
  }
  pick(std::false_type{});
}

}  // namespace
}  // namespace scn

extern "C" size_t scn_jpeg_encode_bound(int width, int height, int channels) {
  return scn_jpeg_encode_bound_opts(width, height, channels, nullptr);
}

extern "C" size_t scn_jpeg_encode_bound_opts(int width, int height, int channels, const scn_jpeg_options* opts) {
  using namespace scn;
  if (width <= 0 || height <= 0 || width > kMaxDim || height > kMaxDim || (channels != 1 && channels != 3)) return 0;
  Settings set;
  if (!settings(channels, 95, opts, &set)) return 0;
  const Geom g = make_geom(width, height, channels, set.hv);
  const size_t blocks = (size_t)g.mcus() * g.bpm;
  const size_t bytes = (blocks * worst_bits_per_block(opts && opts->optimize) + 7) / 8;
  // the Annex K tables list every DC and AC symbol, so no optimised header is longer
  return make_header(width, height, channels, set.quality, set.hv).size() + 2 * bytes + 2;
}

extern "C" int scn_jpeg_encode_u8(const uint8_t* const* host_src_ptrs, int n, int width, int height, int channels,
                                  int quality, scn_alloc_fn alloc_out, void* alloc_ctx, size_t* host_sizes,
                                  void* stream) {
  return scn_jpeg_encode_u8_opts(host_src_ptrs, n, width, height, channels, quality, nullptr, alloc_out, alloc_ctx,
                                 host_sizes, stream);
}

extern "C" int scn_jpeg_encode_u8_opts(const uint8_t* const* host_src_ptrs, int n, int width, int height,
                                       int channels, int quality, const scn_jpeg_options* opts, scn_alloc_fn alloc_out,
                                       void* alloc_ctx, size_t* host_sizes, void* stream) {
  using namespace scn;
  Settings set;
  if (n < 0 || width <= 0 || height <= 0 || !settings(channels, quality, opts, &set)) return SCN_E_BADARG;
  if (channels != 1 && channels != 3) return SCN_E_UNSUPPORTED;
  if (width > kMaxDim || height > kMaxDim) return SCN_E_UNSUPPORTED;
  if (n == 0) return 0;
  if (!host_src_ptrs || !alloc_out || !host_sizes) return SCN_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemPool_t pool = scratch_pool();
  if (!pool) return (int)cudaErrorMemoryAllocation;
  const Geom g = make_geom(width, height, channels, set.hv);
  const uint32_t nm = g.mcus();
  const Tables tables = make_tables(set.quality);
  Affixes ax;
  if (!make_affixes(&ax, make_header(width, height, channels, set.quality, set.hv), {}, {0xFF, 0xD9}))
    return SCN_E_UNSUPPORTED;

  Scratch s{st, {}};
  int16_t* dcs = s.get<int16_t>((size_t)n * nm * g.bpm, pool);
  uint32_t* acbits = s.get<uint32_t>((size_t)n * nm, pool);
  uint64_t* mcu_bit = s.get<uint64_t>((size_t)n * nm, pool);
  uint64_t* bits = s.get<uint64_t>((size_t)n, pool);
  if (!dcs || !acbits || !mcu_bit || !bits) return (int)cudaErrorMemoryAllocation;
  const dim3 mcu_grid((nm + kThreads - 1) / kThreads);

  // optimised tables: per-frame AC counts, codes and headers in scratch
  const bool optimize = opts && opts->optimize;
  FrameTables ft = {nullptr, nullptr};
  FramePrefixes fp = {nullptr, nullptr};
  HeaderParts hp = {};
  if (optimize) {
    uint32_t* ac_hist = s.get<uint32_t>((size_t)n * 2 * 256, pool);
    uint32_t* codes = s.get<uint32_t>((size_t)n * kCodeWords, pool);
    uint8_t* prefix = s.get<uint8_t>((size_t)n * kMaxPrefix, pool);
    uint32_t* prefix_len = s.get<uint32_t>((size_t)n, pool);
    if (!ac_hist || !codes || !prefix || !prefix_len) return (int)cudaErrorMemoryAllocation;
    const int rc = (int)cudaMemsetAsync(ac_hist, 0, (size_t)n * 2 * 256 * 4, st);
    if (rc) return rc;
    ft = {codes, ac_hist};
    fp = {prefix, prefix_len};
    // the Annex K header's parts around its DHT segments
    const std::vector<uint8_t> full = make_header(width, height, channels, set.quality, set.hv);
    size_t at = 2, dht = 0, sos = 0;
    while (at + 4 <= full.size()) {
      if (full[at + 1] == 0xC4 && !dht) dht = at;
      if (full[at + 1] == 0xDA) sos = at;
      at += 2 + ((size_t)full[at + 2] << 8 | full[at + 3]);
    }
    std::copy(full.begin(), full.begin() + dht, hp.head);
    std::copy(full.begin() + sos, full.end(), hp.sos);
    hp.head_len = (int)dht, hp.sos_len = (int)(full.size() - sos), hp.ntab = channels == 3 ? 2 : 1;
  }

  // DCs and AC bit counts, then per-frame scans into bit offsets; with optimised tables, first the symbol counts and
  // the tables built from them
  auto measure = [&] {
    return for_each_chunk(n, [&](int i0, int cnt) {
      const PtrBatch src = gather<PtrBatch>(host_src_ptrs, i0, cnt);
      const MeasureOut mo = {dcs, acbits};
      const dim3 grid(mcu_grid.x, (unsigned)cnt);
      int e = 0;
      if (optimize) {
        e = launch_kernel("jpeg_mcu_kernel<stats>", st, [&] {
          launch_mcu<kStats>(channels, set.hv, grid, st, src, i0, g, tables, mo, EmitIn{}, FrameTables{nullptr,
                                                                                                         ft.ac_hist});
        });
        if (!e)
          e = launch_kernel("jpeg_table_kernel", st, [&] {
            jpeg_table_kernel<<<cnt, 64, 0, st>>>(i0, nm, g.bpm, g.ny, dcs, ft.ac_hist, const_cast<uint32_t*>(ft.codes),
                                                  const_cast<uint8_t*>(fp.bytes), const_cast<uint32_t*>(fp.len), hp);
          });
        if (e) return e;
      }
      e = launch_kernel("jpeg_mcu_kernel<measure>", st, [&] {
        launch_mcu<kMeasure>(channels, set.hv, grid, st, src, i0, g, tables, mo, EmitIn{}, ft);
      });
      if (e) return e;
      return launch_kernel("jpeg_scan_kernel", st, [&] {
        jpeg_scan_kernel<<<cnt, 1024, 0, st>>>(i0, nm, g.bpm, g.ny, tables, ft.codes, dcs, acbits, mcu_bit, bits);
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
      launch_mcu<kEmit>(channels, set.hv, grid, st, src, i0, g, tables, MeasureOut{}, ei, ft);
    });
  };
  return run_output_stage<FfStuffing>(n, st, pool, s, bits, nullptr, ax, measure, emit, alloc_out, alloc_ctx,
                                      host_sizes, fp);
}

extern "C" int scn_jpeg_optimal_table(const uint64_t* host_freq, uint8_t* host_bits, uint8_t* host_vals) {
  using namespace scn;
  if (!host_freq || !host_bits || !host_vals) return SCN_E_BADARG;
  uint64_t* d_freq = nullptr;
  uint8_t* d_out = nullptr;
  int rc = (int)cudaMalloc(&d_freq, 256 * 8);
  if (!rc) rc = (int)cudaMalloc(&d_out, 16 + 256 + 4);
  if (!rc) rc = (int)cudaMemcpy(d_freq, host_freq, 256 * 8, cudaMemcpyHostToDevice);
  if (!rc)
    rc = launch_kernel("jpeg_gen_table_kernel", nullptr, [&] {
      jpeg_gen_table_kernel<<<1, 32>>>(d_freq, d_out, d_out + 16, reinterpret_cast<int*>(d_out + 272));
    });
  uint8_t out[16 + 256 + 4];
  if (!rc) rc = (int)cudaMemcpy(out, d_out, sizeof(out), cudaMemcpyDeviceToHost);
  cudaFree(d_freq);
  cudaFree(d_out);
  if (rc) return rc;
  std::copy(out, out + 16, host_bits);
  std::copy(out + 16, out + 272, host_vals);
  return 0;
}
