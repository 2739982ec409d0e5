// h264_enc.cu -- intra-only H.264 (Baseline, CAVLC) encoding of RGB24 frames (sm_90a).
// oracle/h264_enc.py restates every step in integer numpy and is held to FFmpeg's decoder; this file is held to
// the oracle byte for byte.  The bitstream (H.264 (04/2017) clause numbers):
//   colour      integer BT.601 studio range; chroma from each 2x2 block's channel sums; planes padded to the
//               macroblock grid by repeating their last column and row, SPS cropping gives the display size
//   pictures    one slice each, deblocking off (a decoder then outputs exactly the reconstruction below); an
//               IDR with SPS + PPS at every multiple of keyframe_distance within the item, non-IDR I pictures
//               between; every macroblock Intra16x16, mb_qp_delta 0
//   modes       luma V/H/DC/Plane, chroma DC/H/V/Plane: the least SAD among the available ones, ties to the
//               lower mode number
//   residual    4x4 core transform, luma DC 4x4 Hadamard ((H W H) >> 1), chroma DC 2x2 Hadamard; deadzone
//               quantisation (f = 2^qbits / 3, doubled with qbits + 1 for DC), levels clamped to +-2063; luma AC
//               coded for all 16 blocks or none, chroma cbp 0 / 1 / 2 from the levels
//   entropy     CAVLC (9.2): coeff_token for every nC class, level_prefix escapes 14 and 15, total_zeros,
//               run_before; emulation prevention over the whole slice payload
// Kernels per launch of at most 64 frames:
//   h264_mb_kernel         one CTA per frame, one warp per macroblock: the reconstruction wavefront, one
//                          anti-diagonal of macroblocks per step (a macroblock needs its left, top and top-left
//                          neighbours, all on earlier diagonals), __syncthreads between steps.  Writes each
//                          macroblock's modes, cbp, levels and per-4x4 TotalCoeff.
//   h264_bits_kernel<E>    one thread per macroblock: E false counts the macroblock's bits (nC from the
//                          neighbours' TotalCoeff); E true writes them at the macroblock's offset
//   h264_scan_kernel       one CTA per frame: macroblock bit counts -> bit offsets after the slice header
//   h264_count_epb_kernel  emulation-prevention bytes per 4 KiB chunk of each frame's payload
//   h264_stuff_kernel      copies each chunk with its 0x03 bytes after the NAL prefix (SPS + PPS for an IDR)
// The last two are the output stage of bitstream.cuh with the escape rule EmulationPrevention, as in jpeg.cu.
// Lane roles in h264_mb_kernel: lanes 0-15 are the 16 luma 4x4 blocks (raster order), lanes 16-19 the Cb and
// 20-23 the Cr 4x4 blocks; lanes 24-31 only help load neighbours.
#include <cuda_runtime.h>

#include <vector>

#include "bitstream.cuh"

namespace scn {
namespace {

constexpr int kMaxSide = 4096;
constexpr int kMaxMbs = 36864;  // MaxFS of level 5.1
constexpr int kWarps = 16;      // macroblocks in flight per frame
constexpr int kThreads = 128;   // h264_bits_kernel
constexpr int kMaxNalPrefix = 96;  // at most this many bytes (SPS, PPS, the slice's NAL header) precede a payload
constexpr int kLevelMax = 2063;  // the largest |level| a level_prefix <= 15 codes at suffixLength 0
constexpr uint32_t kFull = 0xFFFFFFFFu;

struct Geom {
  int w, h, wmb, hmb;
  __host__ __device__ int mbs() const { return wmb * hmb; }
  __host__ __device__ size_t rec_bytes() const { return (size_t)mbs() * 384; }  // padded Y, Cb, Cr
};

// What h264_mb_kernel leaves for the entropy passes, per macroblock.
struct MbRec {
  uint8_t lmode, cmode, cbpl, cbpc;
  uint8_t ltc[16];      // TotalCoeff of each luma 4x4 block's AC levels (raster), 0 when not coded
  uint8_t ctc[8];       // the same for the chroma blocks, Cb 0-3 then Cr 0-3
  int16_t ldc[16];      // Intra16x16DCLevel, scan order
  int16_t lac[16][16];  // Intra16x16ACLevel of each luma block (raster), scan order, [0] unused
  int16_t cdc[8];       // ChromaDCLevel, Cb then Cr
  int16_t cac[8][16];   // ChromaACLevel, scan order, [0] unused
};

// ---- tables ----
__host__ __device__ constexpr int zigzag(int s) {  // scan index -> raster index (row * 4 + column)
  constexpr int z[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
  return z[s];
}
__host__ __device__ constexpr int pos_class(int k) {  // raster index -> 0 (even, even), 1 (odd, odd), 2 otherwise
  return ((k >> 2) & 1) == (k & 1) ? ((k & 1) ? 1 : 0) : 2;
}
__host__ __device__ constexpr int hsign(int u, int i) {  // 4x4 Hadamard [[1,1,1,1],[1,1,-1,-1],[1,-1,-1,1],[1,-1,1,-1]]
  constexpr int h[4] = {0x0, 0xC, 0x6, 0xA};           // bit i set: entry -1
  return (h[u] >> i) & 1 ? -1 : 1;
}
__constant__ int kMF[6][3] = {{13107, 5243, 8066}, {11916, 4660, 7490}, {10082, 4194, 6554},
                              {9362, 3647, 5825},  {8192, 3355, 5243},  {7282, 2893, 4559}};
__constant__ int kV[6][3] = {{10, 16, 13}, {11, 18, 14}, {13, 20, 16}, {14, 23, 18}, {16, 25, 20}, {18, 29, 23}};

int chroma_qp(int qp) {
  static const int t[22] = {29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39};
  return qp < 30 ? qp : t[qp - 30];
}

// Table 9-5 as code << 5 | length, [nC class][TotalCoeff * 4 + TrailingOnes]: nC 0-1, 2-3, 4-7, 8+; then nC -1
__device__ const uint16_t kCoeffToken[5][68] = {
    {1 << 5 | 1,   0,           0,           0,           5 << 5 | 6,  1 << 5 | 2,  0,           0,
     7 << 5 | 8,   4 << 5 | 6,  1 << 5 | 3,  0,           7 << 5 | 9,  6 << 5 | 8,  5 << 5 | 7,  3 << 5 | 5,
     7 << 5 | 10,  6 << 5 | 9,  5 << 5 | 8,  3 << 5 | 6,  7 << 5 | 11, 6 << 5 | 10, 5 << 5 | 9,  4 << 5 | 7,
     15 << 5 | 13, 6 << 5 | 11, 5 << 5 | 10, 4 << 5 | 8,  11 << 5 | 13, 14 << 5 | 13, 5 << 5 | 11, 4 << 5 | 9,
     8 << 5 | 13,  10 << 5 | 13, 13 << 5 | 13, 4 << 5 | 10, 15 << 5 | 14, 14 << 5 | 14, 9 << 5 | 13, 4 << 5 | 11,
     11 << 5 | 14, 10 << 5 | 14, 13 << 5 | 14, 12 << 5 | 13, 15 << 5 | 15, 14 << 5 | 15, 9 << 5 | 14, 12 << 5 | 14,
     11 << 5 | 15, 10 << 5 | 15, 13 << 5 | 15, 8 << 5 | 14, 15 << 5 | 16, 1 << 5 | 15, 9 << 5 | 15, 12 << 5 | 15,
     11 << 5 | 16, 14 << 5 | 16, 13 << 5 | 16, 8 << 5 | 15, 7 << 5 | 16, 10 << 5 | 16, 9 << 5 | 16, 12 << 5 | 16,
     4 << 5 | 16,  6 << 5 | 16,  5 << 5 | 16,  8 << 5 | 16},
    {3 << 5 | 2,   0,           0,           0,           11 << 5 | 6, 2 << 5 | 2,  0,           0,
     7 << 5 | 6,   7 << 5 | 5,  3 << 5 | 3,  0,           7 << 5 | 7,  10 << 5 | 6, 9 << 5 | 6,  5 << 5 | 4,
     7 << 5 | 8,   6 << 5 | 6,  5 << 5 | 6,  4 << 5 | 4,  4 << 5 | 8,  6 << 5 | 7,  5 << 5 | 7,  6 << 5 | 5,
     7 << 5 | 9,   6 << 5 | 8,  5 << 5 | 8,  8 << 5 | 6,  15 << 5 | 11, 6 << 5 | 9,  5 << 5 | 9,  4 << 5 | 6,
     11 << 5 | 11, 14 << 5 | 11, 13 << 5 | 11, 4 << 5 | 7, 15 << 5 | 12, 10 << 5 | 11, 9 << 5 | 11, 4 << 5 | 9,
     11 << 5 | 12, 14 << 5 | 12, 13 << 5 | 12, 12 << 5 | 11, 8 << 5 | 12, 10 << 5 | 12, 9 << 5 | 12, 8 << 5 | 11,
     15 << 5 | 13, 14 << 5 | 13, 13 << 5 | 13, 12 << 5 | 12, 11 << 5 | 13, 10 << 5 | 13, 9 << 5 | 13, 12 << 5 | 13,
     7 << 5 | 13,  11 << 5 | 14, 6 << 5 | 13, 8 << 5 | 13, 9 << 5 | 14, 8 << 5 | 14, 10 << 5 | 14, 1 << 5 | 13,
     7 << 5 | 14,  6 << 5 | 14,  5 << 5 | 14,  4 << 5 | 14},
    {15 << 5 | 4,  0,           0,           0,           15 << 5 | 6, 14 << 5 | 4, 0,           0,
     11 << 5 | 6,  15 << 5 | 5, 13 << 5 | 4, 0,           8 << 5 | 6,  12 << 5 | 5, 14 << 5 | 5, 12 << 5 | 4,
     15 << 5 | 7,  10 << 5 | 5, 11 << 5 | 5, 11 << 5 | 4, 11 << 5 | 7, 8 << 5 | 5,  9 << 5 | 5,  10 << 5 | 4,
     9 << 5 | 7,   14 << 5 | 6, 13 << 5 | 6, 9 << 5 | 4,  8 << 5 | 7,  10 << 5 | 6, 9 << 5 | 6,  8 << 5 | 4,
     15 << 5 | 8,  14 << 5 | 7, 13 << 5 | 7, 13 << 5 | 5, 11 << 5 | 8, 14 << 5 | 8, 10 << 5 | 7, 12 << 5 | 6,
     15 << 5 | 9,  10 << 5 | 8, 13 << 5 | 8, 12 << 5 | 7, 11 << 5 | 9, 14 << 5 | 9, 9 << 5 | 8,  12 << 5 | 8,
     8 << 5 | 9,   10 << 5 | 9, 13 << 5 | 9, 8 << 5 | 8,  13 << 5 | 10, 7 << 5 | 9, 9 << 5 | 9,  12 << 5 | 9,
     9 << 5 | 10,  12 << 5 | 10, 11 << 5 | 10, 10 << 5 | 10, 5 << 5 | 10, 8 << 5 | 10, 7 << 5 | 10, 6 << 5 | 10,
     1 << 5 | 10,  4 << 5 | 10,  3 << 5 | 10,  2 << 5 | 10},
    {},  // nC >= 8: a 6-bit code, built in coeff_token()
    {1 << 5 | 2, 0, 0, 0, 7 << 5 | 6, 1 << 5 | 1, 0, 0, 4 << 5 | 6, 6 << 5 | 6, 1 << 5 | 3, 0,
     3 << 5 | 6, 3 << 5 | 7, 2 << 5 | 7, 5 << 5 | 6, 2 << 5 | 6, 3 << 5 | 8, 2 << 5 | 8, 0 << 5 | 7}};

// Tables 9-7 / 9-8, [TotalCoeff - 1][total_zeros], code << 4 | length
#define TZ(b, l) (uint8_t)((b) << 4 | (l))
__device__ const uint8_t kTotalZeros[15][16] = {
    {TZ(1, 1), TZ(3, 3), TZ(2, 3), TZ(3, 4), TZ(2, 4), TZ(3, 5), TZ(2, 5), TZ(3, 6), TZ(2, 6), TZ(3, 7), TZ(2, 7),
     TZ(3, 8), TZ(2, 8), TZ(3, 9), TZ(2, 9), TZ(1, 9)},
    {TZ(7, 3), TZ(6, 3), TZ(5, 3), TZ(4, 3), TZ(3, 3), TZ(5, 4), TZ(4, 4), TZ(3, 4), TZ(2, 4), TZ(3, 5), TZ(2, 5),
     TZ(3, 6), TZ(2, 6), TZ(1, 6), TZ(0, 6)},
    {TZ(5, 4), TZ(7, 3), TZ(6, 3), TZ(5, 3), TZ(4, 4), TZ(3, 4), TZ(4, 3), TZ(3, 3), TZ(2, 4), TZ(3, 5), TZ(2, 5),
     TZ(1, 6), TZ(1, 5), TZ(0, 6)},
    {TZ(3, 5), TZ(7, 3), TZ(5, 4), TZ(4, 4), TZ(6, 3), TZ(5, 3), TZ(4, 3), TZ(3, 4), TZ(3, 3), TZ(2, 4), TZ(2, 5),
     TZ(1, 5), TZ(0, 5)},
    {TZ(5, 4), TZ(4, 4), TZ(3, 4), TZ(7, 3), TZ(6, 3), TZ(5, 3), TZ(4, 3), TZ(3, 3), TZ(2, 4), TZ(1, 5), TZ(1, 4),
     TZ(0, 5)},
    {TZ(1, 6), TZ(1, 5), TZ(7, 3), TZ(6, 3), TZ(5, 3), TZ(4, 3), TZ(3, 3), TZ(2, 3), TZ(1, 4), TZ(1, 3), TZ(0, 6)},
    {TZ(1, 6), TZ(1, 5), TZ(5, 3), TZ(4, 3), TZ(3, 3), TZ(3, 2), TZ(2, 3), TZ(1, 4), TZ(1, 3), TZ(0, 6)},
    {TZ(1, 6), TZ(1, 4), TZ(1, 5), TZ(3, 3), TZ(3, 2), TZ(2, 2), TZ(2, 3), TZ(1, 3), TZ(0, 6)},
    {TZ(1, 6), TZ(0, 6), TZ(1, 4), TZ(3, 2), TZ(2, 2), TZ(1, 3), TZ(1, 2), TZ(1, 5)},
    {TZ(1, 5), TZ(0, 5), TZ(1, 3), TZ(3, 2), TZ(2, 2), TZ(1, 2), TZ(1, 4)},
    {TZ(0, 4), TZ(1, 4), TZ(1, 3), TZ(2, 3), TZ(1, 1), TZ(3, 3)},
    {TZ(0, 4), TZ(1, 4), TZ(1, 2), TZ(1, 1), TZ(1, 3)},
    {TZ(0, 3), TZ(1, 3), TZ(1, 1), TZ(1, 2)},
    {TZ(0, 2), TZ(1, 2), TZ(1, 1)},
    {TZ(0, 1), TZ(1, 1)}};
// Table 9-9a (chroma DC), [TotalCoeff - 1][total_zeros]
__device__ const uint8_t kTotalZerosDc[3][4] = {
    {TZ(1, 1), TZ(1, 2), TZ(1, 3), TZ(0, 3)}, {TZ(1, 1), TZ(1, 2), TZ(0, 2)}, {TZ(1, 1), TZ(0, 1)}};
// Table 9-10, [min(zerosLeft, 7) - 1][run_before]
__device__ const uint8_t kRunBefore[7][15] = {
    {TZ(1, 1), TZ(0, 1)},
    {TZ(1, 1), TZ(1, 2), TZ(0, 2)},
    {TZ(3, 2), TZ(2, 2), TZ(1, 2), TZ(0, 2)},
    {TZ(3, 2), TZ(2, 2), TZ(1, 2), TZ(1, 3), TZ(0, 3)},
    {TZ(3, 2), TZ(2, 2), TZ(3, 3), TZ(2, 3), TZ(1, 3), TZ(0, 3)},
    {TZ(3, 2), TZ(0, 3), TZ(1, 3), TZ(3, 3), TZ(2, 3), TZ(5, 3), TZ(4, 3)},
    {TZ(7, 3), TZ(6, 3), TZ(5, 3), TZ(4, 3), TZ(3, 3), TZ(2, 3), TZ(1, 3), TZ(1, 4), TZ(1, 5), TZ(1, 6), TZ(1, 7),
     TZ(1, 8), TZ(1, 9), TZ(1, 10), TZ(1, 11)}};
#undef TZ

// ---- colour: Y of pixel (x, y), chroma of chroma sample (x, y); coordinates clamped to the picture ----
__device__ __forceinline__ int luma_at(const uint8_t* __restrict__ src, const Geom& g, int x, int y) {
  const uint8_t* p = src + ((size_t)min(y, g.h - 1) * g.w + min(x, g.w - 1)) * 3;
  return ((66 * __ldg(p) + 129 * __ldg(p + 1) + 25 * __ldg(p + 2) + 128) >> 8) + 16;
}
__device__ __forceinline__ int chroma_at(const uint8_t* __restrict__ src, const Geom& g, int comp, int x, int y) {
  x = min(x, g.w / 2 - 1), y = min(y, g.h / 2 - 1);
  int sr = 0, sg = 0, sb = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint8_t* p = src + ((size_t)(2 * y + (k >> 1)) * g.w + 2 * x + (k & 1)) * 3;
    sr += __ldg(p), sg += __ldg(p + 1), sb += __ldg(p + 2);
  }
  return comp == 0 ? ((-38 * sr - 74 * sg + 112 * sb + 512) >> 10) + 128
                   : ((112 * sr - 94 * sg - 18 * sb + 512) >> 10) + 128;
}

// forward core transform of one row / column: [1 1 1 1; 2 1 -1 -2; 1 -1 -1 1; 1 -2 2 -1]
__device__ __forceinline__ void fwd4(int& a, int& b, int& c, int& d) {
  const int s03 = a + d, d03 = a - d, s12 = b + c, d12 = b - c;
  a = s03 + s12, b = 2 * d03 + d12, c = s03 - s12, d = d03 - 2 * d12;
}
// inverse (8.5.12.2) of one row / column
__device__ __forceinline__ void inv4(int& a, int& b, int& c, int& d) {
  const int e0 = a + c, e1 = a - c, e2 = (b >> 1) - d, e3 = b + (d >> 1);
  a = e0 + e3, b = e1 + e2, c = e1 - e2, d = e0 - e3;
}

__device__ __forceinline__ int quant(int w, int mf, int f, int qbits) {
  const int q = min((abs(w) * mf + f) >> qbits, kLevelMax);
  return w < 0 ? -q : q;
}

// The 2-D (4x4 luma or 2x2 chroma) Hadamard of the values v held by a lane group: lane (u, v) of the group gets
// sum_ij H[u][i] v(i, j) H[j][v].  Every lane of the warp calls it.
__device__ __forceinline__ int group_hadamard(int v, bool luma, int base, int u, int w) {
  int acc = 0;
#pragma unroll
  for (int t = 0; t < 16; ++t) {
    const int x = __shfl_sync(kFull, v, luma ? t : base + (t & 3));
    if (luma) {
      acc += hsign(u, t >> 2) * hsign(t & 3, w) * x;
    } else if (t < 4) {
      const int su = (u & (t >> 1)) ? -1 : 1, sw = ((t & 1) & w) ? -1 : 1;
      acc += su * sw * x;
    }
  }
  return acc;
}

// One CTA per frame.  recon: the chunk's padded planes, frame blockIdx.x at blockIdx.x * rec_bytes.
__global__ void __launch_bounds__(kWarps * 32)
h264_mb_kernel(PtrBatch srcs, int i0, Geom g, int qp, int qpc, MbRec* __restrict__ recs, uint8_t* recon) {
  __shared__ int nbs[kWarps][68];  // luma top 0-15, left 16-31, corner 32; then Cb and Cr: top 8, left 8, corner
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint8_t* __restrict__ src = srcs.p[blockIdx.x];
  const int yp = 16 * g.wmb, cp = 8 * g.wmb;
  uint8_t* ry = recon + (size_t)blockIdx.x * g.rec_bytes();
  auto rc = [&](int c) { return ry + (size_t)(256 + 64 * c) * g.mbs(); };  // Cb, Cr
  MbRec* frame_recs = recs + (size_t)(i0 + blockIdx.x) * g.mbs();
  int* nb = nbs[warp];

  const bool is_luma = lane < 16, is_chroma = lane >= 16 && lane < 24;
  const int comp = (lane - 16) >> 2;  // chroma lanes: 0 Cb, 1 Cr
  const int bx = is_luma ? (lane & 3) : ((lane - 16) & 1), by = is_luma ? (lane >> 2) : (((lane - 16) >> 1) & 1);
  const int q = is_luma ? qp : qpc;
  const int qbits = 15 + q / 6, qf = (1 << qbits) / 3;
  const int n = is_luma ? 16 : 8;  // prediction block side
  const int* top = is_luma ? nb : nb + 33 + 17 * (comp & 1);
  const int* left = top + n;
  const int corner_i = n * 2;

#pragma unroll 1
  for (int d = 0; d < g.wmb + g.hmb - 1; ++d) {
    const int my1 = min(g.hmb - 1, d);
#pragma unroll 1
    for (int my = max(0, d - g.wmb + 1) + warp; my <= my1; my += kWarps) {
      const int mx = d - my;
      const bool ht = my > 0, hl = mx > 0;
      // neighbours from the reconstruction
      __syncwarp();
      if (lane < 16) {
        nb[lane] = ht ? ry[(size_t)(16 * my - 1) * yp + 16 * mx + lane] : 0;
        nb[16 + lane] = hl ? ry[(size_t)(16 * my + lane) * yp + 16 * mx - 1] : 0;
      } else {
        const int c = (lane - 16) >> 3, k = lane & 7;
        int* cn = nb + 33 + 17 * c;
        cn[k] = ht ? rc(c)[(size_t)(8 * my - 1) * cp + 8 * mx + k] : 0;
        cn[8 + k] = hl ? rc(c)[(size_t)(8 * my + k) * cp + 8 * mx - 1] : 0;
        if (k == 0) cn[16] = ht && hl ? rc(c)[(size_t)(8 * my - 1) * cp + 8 * mx - 1] : 0;
      }
      if (lane == 0) nb[32] = ht && hl ? ry[(size_t)(16 * my - 1) * yp + 16 * mx - 1] : 0;
      __syncwarp();

      // source samples of the lane's 4x4 block
      int s[16];
      const int x0 = 4 * bx, y0 = 4 * by;  // within the macroblock (component samples)
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        if (is_luma) s[k] = luma_at(src, g, 16 * mx + x0 + (k & 3), 16 * my + y0 + (k >> 2));
        else if (is_chroma) s[k] = chroma_at(src, g, comp, 8 * mx + x0 + (k & 3), 8 * my + y0 + (k >> 2));
        else s[k] = 0;
      }

      // prediction parameters: DC of the lane's block, plane a, b, c
      int dcv = 128;
      int pa = 0, pb = 0, pc = 0;
      if (lane < 24) {
        const int corner = top[corner_i];
        if (is_luma) {
          int st = 0, sl = 0;
#pragma unroll
          for (int k = 0; k < 16; ++k) st += top[k], sl += left[k];
          dcv = ht && hl ? (st + sl + 16) >> 5 : ht ? (st + 8) >> 4 : hl ? (sl + 8) >> 4 : 128;
        } else {
          int st = 0, sl = 0;
#pragma unroll
          for (int k = 0; k < 4; ++k) st += top[x0 + k], sl += left[y0 + k];
          const int both = (st + sl + 4) >> 3, t_only = (st + 2) >> 2, l_only = (sl + 2) >> 2;
          if (bx == 1 && by == 0) dcv = ht ? t_only : hl ? l_only : 128;
          else if (bx == 0 && by == 1) dcv = hl ? l_only : ht ? t_only : 128;
          else dcv = ht && hl ? both : hl ? l_only : ht ? t_only : 128;
        }
        const int half = n / 2 - 1;
        int hh = -(half + 1) * corner, vv = -(half + 1) * corner;
        for (int k = 0; k < n; ++k) hh += (k - half) * top[k], vv += (k - half) * left[k];
        const int mul = is_luma ? 5 : 34;
        pa = 16 * (left[n - 1] + top[n - 1]);
        pb = (mul * hh + 32) >> 6;
        pc = (mul * vv + 32) >> 6;
        pa += 16 - half * (pb + pc);  // folds the centre offsets and the rounding term
      }
      // kind of prediction: 0 V, 1 H, 2 DC, 3 Plane; luma mode numbers are the kinds, chroma's are DC H V Plane
      auto kind_of = [&](int m) { return is_luma ? m : (m == 0 ? 2 : m == 2 ? 0 : m); };
      auto pred = [&](int kind, int k) {
        const int x = x0 + (k & 3), y = y0 + (k >> 2);
        if (kind == 0) return top[x];
        if (kind == 1) return left[y];
        if (kind == 2) return dcv;
        return min(max((pa + pb * x + pc * y) >> 5, 0), 255);
      };
      int best = 0, best_sad = 0x7FFFFFFF;
#pragma unroll 1
      for (int m = 0; m < 4; ++m) {
        const int kind = kind_of(m);
        int sad = 0;
        if (lane < 24) {
#pragma unroll
          for (int k = 0; k < 16; ++k) sad += abs(s[k] - pred(kind, k));
        }
        sad += __shfl_xor_sync(kFull, sad, 1);
        sad += __shfl_xor_sync(kFull, sad, 2);
        sad += __shfl_xor_sync(kFull, sad, 4);
        const int other = __shfl_xor_sync(kFull, sad, 8);
        if (is_luma) sad += other;
        const bool ok = kind == 2 || (kind == 0 && ht) || (kind == 1 && hl) || (kind == 3 && ht && hl);
        if (ok && sad < best_sad) best_sad = sad, best = m;
      }
      const int kind = kind_of(best);

      // residual, forward transform, AC quantisation
      int w[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) w[k] = s[k] - pred(kind, k);
#pragma unroll
      for (int r = 0; r < 4; ++r) fwd4(w[4 * r], w[4 * r + 1], w[4 * r + 2], w[4 * r + 3]);
#pragma unroll
      for (int c = 0; c < 4; ++c) fwd4(w[c], w[4 + c], w[8 + c], w[12 + c]);
      const int qm = q % 6;
      bool acnz = false;
#pragma unroll
      for (int k = 1; k < 16; ++k) {
        w[k] = quant(w[k], kMF[qm][pos_class(k)], qf, qbits);
        acnz |= w[k] != 0;
      }
      // DC: Hadamard over the lane group, quantised with qbits + 1
      const int u = by, v = bx;
      const int gbase = 16 + 4 * (comp & 1);
      int dcw = group_hadamard(w[0], is_luma, gbase, u, v);
      if (is_luma) dcw >>= 1;
      int dl = quant(dcw, kMF[qm][0], 2 * qf, qbits + 1);
      if (lane >= 24) dl = 0, acnz = false;
      const uint32_t bal_ac = __ballot_sync(kFull, acnz), bal_dc = __ballot_sync(kFull, dl != 0);
      const int cbpl = (bal_ac & 0xFFFFu) ? 15 : 0;
      const int cbpc = (bal_ac & 0xFF0000u) ? 2 : (bal_dc & 0xFF0000u) ? 1 : 0;
      const bool ac_coded = is_luma ? cbpl != 0 : cbpc == 2;
      int tc = 0;
#pragma unroll
      for (int k = 1; k < 16; ++k) {
        if (!ac_coded) w[k] = 0;
        tc += w[k] != 0;
      }

      // record the levels
      MbRec& rec = frame_recs[my * g.wmb + mx];
      if (is_luma) {
        rec.ltc[lane] = (uint8_t)tc;
        rec.lac[lane][0] = 0;
#pragma unroll
        for (int sidx = 1; sidx < 16; ++sidx) rec.lac[lane][sidx] = (int16_t)w[zigzag(sidx)];
#pragma unroll
        for (int sidx = 0; sidx < 16; ++sidx)
          if (zigzag(sidx) == lane) rec.ldc[sidx] = (int16_t)dl;
      } else if (is_chroma) {
        const int b = lane - 16;
        rec.ctc[b] = (uint8_t)tc;
        rec.cdc[b] = (int16_t)dl;
        rec.cac[b][0] = 0;
#pragma unroll
        for (int sidx = 1; sidx < 16; ++sidx) rec.cac[b][sidx] = (int16_t)w[zigzag(sidx)];
      }
      const int cmode = __shfl_sync(kFull, best, 16);
      if (lane == 0) {
        rec.lmode = (uint8_t)best;
        rec.cmode = (uint8_t)cmode;
        rec.cbpl = (uint8_t)cbpl;
        rec.cbpc = (uint8_t)cbpc;
      }

      // reconstruction: dequantise, inverse DC Hadamard, inverse transform, add the prediction
      const int f = group_hadamard(dl, is_luma, gbase, u, v);
      const int ls = 16 * kV[qm][0], sh = q / 6;
      if (is_luma) w[0] = q >= 36 ? (f * ls) << (sh - 6) : (f * ls + (1 << (5 - sh))) >> (6 - sh);
      else w[0] = ((f * ls) << sh) >> 5;
#pragma unroll
      for (int k = 1; k < 16; ++k) w[k] = (w[k] * kV[qm][pos_class(k)]) << sh;
#pragma unroll
      for (int r = 0; r < 4; ++r) inv4(w[4 * r], w[4 * r + 1], w[4 * r + 2], w[4 * r + 3]);
#pragma unroll
      for (int c = 0; c < 4; ++c) inv4(w[c], w[4 + c], w[8 + c], w[12 + c]);
      if (lane < 24) {
        uint8_t* plane = is_luma ? ry : rc(comp);
        const int pitch = is_luma ? yp : cp;
        const int px = (is_luma ? 16 : 8) * mx + x0, py = (is_luma ? 16 : 8) * my + y0;
#pragma unroll
        for (int k = 0; k < 16; ++k)
          plane[(size_t)(py + (k >> 2)) * pitch + px + (k & 3)] =
              (uint8_t)min(max(pred(kind, k) + ((w[k] + 32) >> 6), 0), 255);
      }
    }
    __syncthreads();
  }
}

// ---- CAVLC ----
__device__ __forceinline__ int nc_of(int a, int b) {  // -1: unavailable
  return a >= 0 && b >= 0 ? (a + b + 1) >> 1 : a >= 0 ? a : b >= 0 ? b : 0;
}

template <bool Emit>
struct Sink {
  BitWriter* bw;
  uint32_t bits = 0;
  __device__ __forceinline__ void put(uint32_t v, int len) {
    if (Emit) bw->put(v, len);
    bits += len;
  }
  __device__ __forceinline__ void ue(uint32_t v) {  // v < 2^13
    const int b = 32 - __clz(v + 1);
    put(v + 1, 2 * b - 1);
  }
};

// residual_block_cavlc of coef[0 .. max_num) (scan order); nc -1 for chroma DC
template <bool Emit>
__device__ void cavlc(Sink<Emit>& o, const int16_t* __restrict__ coef, int max_num, int nc) {
  uint32_t mask = 0;
  for (int i = 0; i < max_num; ++i)
    if (coef[i]) mask |= 1u << i;
  const int tc = __popc(mask);
  int t1 = 0;
  for (uint32_t m = mask; m && t1 < 3; ++t1) {
    const int i = 31 - __clz(m);
    if (abs(coef[i]) != 1) break;
    m &= ~(1u << i);
  }
  const int cls = nc < 0 ? 4 : nc < 2 ? 0 : nc < 4 ? 1 : nc < 8 ? 2 : 3;
  if (cls == 3) {
    o.put(tc ? (uint32_t)((tc - 1) << 2 | t1) : 3u, 6);
  } else {
    const uint16_t e = kCoeffToken[cls][tc * 4 + t1];
    o.put(e >> 5, e & 31);
  }
  if (!tc) return;
  int sl = tc > 10 && t1 < 3 ? 1 : 0;
  int i = 0;
  for (uint32_t m = mask; m; ++i) {
    const int k = 31 - __clz(m);
    m &= ~(1u << k);
    const int lv = coef[k];
    if (i < t1) {
      o.put(lv < 0, 1);
      continue;
    }
    int code = lv > 0 ? 2 * lv - 2 : -2 * lv - 1;
    if (i == t1 && t1 < 3) code -= 2;
    if (sl == 0 && code < 14) {
      o.put(1, code + 1);
    } else if (sl == 0 && code < 30) {
      o.put(1, 15);
      o.put(code - 14, 4);
    } else if (sl > 0 && (code >> sl) < 15) {
      o.put(1, (code >> sl) + 1);
      o.put(code & ((1 << sl) - 1), sl);
    } else {
      o.put(1, 16);
      o.put(code - (sl == 0 ? 30 : 15 << sl), 12);
    }
    if (sl == 0) sl = 1;
    if (abs(lv) > (3 << (sl - 1)) && sl < 6) ++sl;
  }
  if (tc < max_num) {
    const int top = 31 - __clz(mask);
    const int tz = top + 1 - tc;
    const uint8_t e = max_num == 4 ? kTotalZerosDc[tc - 1][tz] : kTotalZeros[tc - 1][tz];
    o.put(e >> 4, e & 15);
    int zl = tz, prev = top;
    for (uint32_t m = mask & ~(1u << top); m && zl > 0;) {
      const int k = 31 - __clz(m);
      m &= ~(1u << k);
      const int run = prev - k - 1;
      const uint8_t r = kRunBefore[min(zl, 7) - 1][run];
      o.put(r >> 4, r & 15);
      zl -= run;
      prev = k;
    }
  }
}

// macroblock_layer of one Intra16x16 macroblock; left / top null when unavailable
template <bool Emit>
__device__ void code_mb(Sink<Emit>& o, const MbRec& r, const MbRec* left, const MbRec* top) {
  o.ue(1 + r.lmode + 4 * r.cbpc + (r.cbpl ? 12 : 0));  // mb_type I_16x16_<mode>_<cbpc>_<cbpl>
  o.ue(r.cmode);                                      // intra_chroma_pred_mode
  o.put(1, 1);                                        // mb_qp_delta se(0)
  auto ltc = [&](int x, int y) -> int {               // TotalCoeff of luma block (x, y), x, y in -1..3
    if (x < 0) return left ? left->ltc[y * 4 + 3] : -1;
    if (y < 0) return top ? top->ltc[12 + x] : -1;
    return r.ltc[y * 4 + x];
  };
  cavlc(o, r.ldc, 16, nc_of(ltc(-1, 0), ltc(0, -1)));
  if (r.cbpl)
    for (int blk = 0; blk < 16; ++blk) {
      const int x = ((blk >> 2) & 1) * 2 + (blk & 1), y = ((blk >> 3) & 1) * 2 + ((blk >> 1) & 1);
      cavlc(o, r.lac[y * 4 + x] + 1, 15, nc_of(ltc(x - 1, y), ltc(x, y - 1)));
    }
  if (r.cbpc)
    for (int c = 0; c < 2; ++c) cavlc(o, r.cdc + 4 * c, 4, -1);
  if (r.cbpc == 2)
    for (int c = 0; c < 2; ++c)
      for (int blk = 0; blk < 4; ++blk) {
        const int x = blk & 1, y = blk >> 1;
        const int a = x ? r.ctc[4 * c + 2 * y] : left ? left->ctc[4 * c + 2 * y + 1] : -1;
        const int b = y ? r.ctc[4 * c + x] : top ? top->ctc[4 * c + 2 + x] : -1;
        cavlc(o, r.cac[4 * c + blk] + 1, 15, nc_of(a, b));
      }
}

struct SliceHeads {
  uint64_t bits[SCN_MAX_PTRS];  // slice header of each frame, right-aligned
  int len[SCN_MAX_PTRS];
};
struct EmitIn {
  uint8_t* streams;
  uint64_t stream_off[SCN_MAX_PTRS];  // byte offset of each frame's payload in `streams` (a multiple of 16)
};

// One thread per macroblock.  !Emit: its bit count to mb_bit.  Emit: its bits at the offset mb_bit now holds
// (macroblock 0 also writes the slice header, the last one the rbsp stop bit).
template <bool Emit>
__global__ void __launch_bounds__(kThreads)
h264_bits_kernel(int i0, Geom g, const MbRec* __restrict__ recs, uint32_t* mb_bit,
                 const __grid_constant__ SliceHeads heads, const __grid_constant__ EmitIn ei) {
  const int m = blockIdx.x * kThreads + threadIdx.x;
  if (m >= g.mbs()) return;
  const int f = i0 + (int)blockIdx.y;
  const MbRec* fr = recs + (size_t)f * g.mbs();
  const int mx = m % g.wmb, my = m / g.wmb;
  const size_t at = (size_t)f * g.mbs() + m;
  BitWriter bw(Emit ? reinterpret_cast<uint32_t*>(ei.streams + ei.stream_off[blockIdx.y]) : nullptr,
               Emit ? (m ? mb_bit[at] : 0) : 0);
  Sink<Emit> o{&bw};
  if (Emit && m == 0) {
    const uint64_t hb = heads.bits[blockIdx.y];
    const int hl = heads.len[blockIdx.y];
    if (hl > 24) o.put((uint32_t)(hb >> 24), hl - 24);
    o.put((uint32_t)(hb & 0xFFFFFF), hl > 24 ? 24 : hl);
  }
  code_mb(o, fr[m], mx ? &fr[m - 1] : nullptr, my ? &fr[m - g.wmb] : nullptr);
  if constexpr (Emit) {
    if (m == g.mbs() - 1) o.put(1, 1);  // rbsp_stop_one_bit; the alignment zeros are already there
    bw.finish();
  } else {
    mb_bit[at] = o.bits;
  }
}

// One CTA per frame: macroblock bit counts -> bit offsets (after the slice header), and the payload's total bits
// (stop bit and alignment included).
__global__ void __launch_bounds__(1024)
h264_scan_kernel(int i0, int nm, const __grid_constant__ SliceHeads heads, uint32_t* mb_bit_all, uint64_t* total) {
  const int f = i0 + (int)blockIdx.x;
  uint32_t* mb_bit = mb_bit_all + (size_t)f * nm;
  const int per = (nm + blockDim.x - 1) / blockDim.x;
  const int m0 = min(nm, (int)threadIdx.x * per), m1 = min(nm, m0 + per);
  unsigned long long sum = 0;
  for (int m = m0; m < m1; ++m) sum += mb_bit[m];
  unsigned long long all;
  unsigned long long off = block_exclusive_scan<unsigned long long>(sum, &all) + heads.len[blockIdx.x];
  for (int m = m0; m < m1; ++m) {
    const uint32_t b = mb_bit[m];
    mb_bit[m] = (uint32_t)off;
    off += b;
  }
  if (threadIdx.x == 0) total[f] = (heads.len[blockIdx.x] + all + 1 + 7) / 8 * 8;
}

// Emulation prevention (7.4.1): 0x03 goes before payload byte i when it is <= 3 and follows z >= 2 zero bytes with z
// even (counting the payload's own zeros, not inserted bytes).
struct EmulationPrevention {
  static constexpr const char* count_name = "h264_count_epb_kernel";
  static constexpr const char* copy_name = "h264_stuff_kernel";
  static __device__ __forceinline__ int zeros_before(const uint8_t* p, uint64_t at) {
    int z = 0;
    while (at > 0 && p[at - 1] == 0) --at, ++z;
    return z;
  }
  static __device__ __forceinline__ int count(const uint8_t* p, uint64_t at, const uint4& v, int valid) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    int z = zeros_before(p, at), c = 0;
    for (int k = 0; k < valid; ++k) {
      const uint32_t b = (w[k >> 2] >> (8 * (k & 3))) & 0xFF;
      c += b <= 3 && z >= 2 && !(z & 1);
      z = b ? 0 : z + 1;
    }
    return c;
  }
  static __device__ __forceinline__ uint8_t* copy(const uint8_t* p, uint64_t at, const uint4& v, int valid,
                                                  uint8_t* o) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    int z = zeros_before(p, at);
    for (int k = 0; k < valid; ++k) {
      const uint8_t b = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
      if (b <= 3 && z >= 2 && !(z & 1)) *o++ = 3;
      *o++ = b;
      z = b ? 0 : z + 1;
    }
    return o;
  }
};

// ---- host: parameter sets and slice headers ----
struct Bits {
  std::vector<uint8_t> bits;
  void u(int n, uint32_t v) {
    for (int k = n - 1; k >= 0; --k) bits.push_back((v >> k) & 1);
  }
  void ue(uint32_t v) {
    const int b = 32 - __builtin_clz(v + 1);
    u(2 * b - 1, v + 1);
  }
  void se(int v) { ue(v > 0 ? 2 * v - 1 : -2 * v); }
  std::vector<uint8_t> rbsp() {  // with rbsp_trailing_bits
    u(1, 1);
    while (bits.size() % 8) bits.push_back(0);
    std::vector<uint8_t> o(bits.size() / 8, 0);
    for (size_t k = 0; k < bits.size(); ++k) o[k / 8] |= bits[k] << (7 - k % 8);
    return o;
  }
};

void append_nal(std::vector<uint8_t>& o, int ref_idc, int type, const std::vector<uint8_t>& rbsp) {
  o.insert(o.end(), {0, 0, 0, 1, (uint8_t)(ref_idc << 5 | type)});
  int z = 0;
  for (uint8_t b : rbsp) {
    if (z >= 2 && b <= 3) o.push_back(3), z = 0;
    o.push_back(b);
    z = b ? 0 : z + 1;
  }
}

int level_idc(const Geom& g) { return g.mbs() <= 8192 ? 41 : 51; }

std::vector<uint8_t> sps(const Geom& g) {
  Bits b;
  b.u(8, 66);    // profile_idc Baseline
  b.u(8, 0xC0);  // constraint_set0_flag, constraint_set1_flag
  b.u(8, level_idc(g));
  b.ue(0);  // seq_parameter_set_id
  b.ue(0);  // log2_max_frame_num_minus4
  b.ue(2);  // pic_order_cnt_type
  b.ue(1);  // max_num_ref_frames
  b.u(1, 0);
  b.ue(g.wmb - 1);
  b.ue(g.hmb - 1);
  b.u(1, 1);  // frame_mbs_only_flag
  b.u(1, 1);  // direct_8x8_inference_flag
  const bool crop = g.wmb * 16 != g.w || g.hmb * 16 != g.h;
  b.u(1, crop);
  if (crop) {
    b.ue(0);
    b.ue((g.wmb * 16 - g.w) / 2);
    b.ue(0);
    b.ue((g.hmb * 16 - g.h) / 2);
  }
  b.u(1, 1);  // vui_parameters_present_flag
  b.u(1, 0);  // aspect_ratio_info_present_flag
  b.u(1, 0);  // overscan_info_present_flag
  b.u(1, 1);  // video_signal_type_present_flag
  b.u(3, 5);  // video_format unspecified
  b.u(1, 0);  // video_full_range_flag: studio range
  b.u(1, 1);  // colour_description_present_flag
  b.u(8, 6);  // colour_primaries, transfer_characteristics, matrix_coefficients: BT.601
  b.u(8, 6);
  b.u(8, 6);
  b.u(1, 0);  // chroma_loc_info_present_flag
  b.u(1, 0);  // timing_info_present_flag
  b.u(1, 0);  // nal_hrd_parameters_present_flag
  b.u(1, 0);  // vcl_hrd_parameters_present_flag
  b.u(1, 0);  // pic_struct_present_flag
  b.u(1, 1);  // bitstream_restriction_flag
  b.u(1, 1);  // motion_vectors_over_pic_boundaries_flag
  b.ue(0);    // max_bytes_per_pic_denom
  b.ue(0);    // max_bits_per_mb_denom
  b.ue(16);   // log2_max_mv_length_horizontal
  b.ue(16);   // log2_max_mv_length_vertical
  b.ue(0);    // max_num_reorder_frames
  b.ue(1);    // max_dec_frame_buffering
  return b.rbsp();
}

std::vector<uint8_t> pps(int qp) {
  Bits b;
  b.ue(0);
  b.ue(0);
  b.u(1, 0);  // entropy_coding_mode_flag: CAVLC
  b.u(1, 0);
  b.ue(0);
  b.ue(0);
  b.ue(0);
  b.u(1, 0);
  b.u(2, 0);
  b.se(qp - 26);  // pic_init_qp_minus26
  b.se(0);
  b.se(0);    // chroma_qp_index_offset
  b.u(1, 1);  // deblocking_filter_control_present_flag
  b.u(1, 0);
  b.u(1, 0);
  return b.rbsp();
}

void slice_header(int pos, int keyframe_distance, uint64_t* bits, int* len, bool* idr) {
  const int k = pos % keyframe_distance;
  *idr = k == 0;
  Bits b;
  b.ue(0);  // first_mb_in_slice
  b.ue(7);  // slice_type I
  b.ue(0);  // pic_parameter_set_id
  b.u(4, k % 16);  // frame_num
  if (*idr) {
    b.ue((pos / keyframe_distance) & 1);  // idr_pic_id
    b.u(1, 0);                            // no_output_of_prior_pics_flag
    b.u(1, 0);                            // long_term_reference_flag
  } else {
    b.u(1, 0);  // adaptive_ref_pic_marking_mode_flag
  }
  b.se(0);  // slice_qp_delta
  b.ue(1);  // disable_deblocking_filter_idc
  uint64_t v = 0;
  for (uint8_t x : b.bits) v = v << 1 | x;
  *bits = v;
  *len = (int)b.bits.size();
}

Geom make_geom(int w, int h) { return Geom{w, h, (w + 15) / 16, (h + 15) / 16}; }

// the longest a macroblock can code: mb_type, chroma mode and qp delta, then 27 blocks with every coefficient at
// the longest level code (28 bits), the longest coeff_token, total_zeros and runs
constexpr size_t kWorstMbBits = 32 + 27 * (16 + 16 * 28 + 9 + 15 * 11);

}  // namespace
}  // namespace scn

extern "C" size_t scn_h264_encode_bound(int width, int height) {
  using namespace scn;
  if (width <= 0 || height <= 0 || (width | height) & 1 || width > kMaxSide || height > kMaxSide) return 0;
  const Geom g = make_geom(width, height);
  if (g.mbs() > kMaxMbs) return 0;
  const size_t payload = ((size_t)g.mbs() * kWorstMbBits + 64) / 8 + 1;
  return (size_t)kMaxNalPrefix + payload + payload / 2 + 1;  // at most one 0x03 per two payload bytes
}

extern "C" int scn_h264_encode_u8(const uint8_t* const* host_src_ptrs, int n, int width, int height, int qp,
                                  const int* host_positions, int keyframe_distance, scn_alloc_fn alloc_out,
                                  void* alloc_ctx, size_t* host_sizes, void* stream) {
  using namespace scn;
  if (n < 0 || width <= 0 || height <= 0 || qp < 0 || qp > 51 || keyframe_distance < 1) return SCN_E_BADARG;
  if ((width | height) & 1 || width > kMaxSide || height > kMaxSide) return SCN_E_UNSUPPORTED;
  const Geom g = make_geom(width, height);
  if (g.mbs() > kMaxMbs) return SCN_E_UNSUPPORTED;
  if (n == 0) return 0;
  if (!host_src_ptrs || !alloc_out || !host_sizes) return SCN_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemPool_t pool = scratch_pool();
  if (!pool) return (int)cudaErrorMemoryAllocation;
  const int nm = g.mbs();

  std::vector<uint64_t> head_bits((size_t)n);
  std::vector<int> head_len((size_t)n);
  std::vector<uint8_t> idr((size_t)n);
  for (int i = 0; i < n; ++i) {
    const int pos = host_positions ? host_positions[i] : i;
    if (pos < 0) return SCN_E_BADARG;
    bool key;
    slice_header(pos, keyframe_distance, &head_bits[i], &head_len[i], &key);
    idr[i] = key;
  }
  // prefix 0 starts a non-IDR picture's access unit, prefix 1 (SPS, PPS, then the slice NAL) an IDR picture's
  std::vector<uint8_t> key;
  append_nal(key, 3, 7, sps(g));
  append_nal(key, 3, 8, pps(qp));
  key.insert(key.end(), {0, 0, 0, 1, 3 << 5 | 5});
  Affixes ax;
  if (!make_affixes(&ax, {0, 0, 0, 1, 2 << 5 | 1}, key, {})) return SCN_E_UNSUPPORTED;
  auto heads = [&](int i0, int cnt) {
    SliceHeads h = {};
    for (int j = 0; j < cnt; ++j) h.bits[j] = head_bits[i0 + j], h.len[j] = head_len[i0 + j];
    return h;
  };

  Scratch s{st, {}};
  MbRec* recs = s.get<MbRec>((size_t)n * nm, pool);
  uint8_t* recon = s.get<uint8_t>((size_t)(n < SCN_MAX_PTRS ? n : SCN_MAX_PTRS) * g.rec_bytes(), pool);
  uint32_t* mb_bit = s.get<uint32_t>((size_t)n * nm, pool);
  uint64_t* bits = s.get<uint64_t>((size_t)n, pool);
  if (!recs || !recon || !mb_bit || !bits) return (int)cudaErrorMemoryAllocation;
  const int qpc = chroma_qp(qp);
  const unsigned mb_blocks = (unsigned)((nm + kThreads - 1) / kThreads);

  // the wavefront, macroblock bit counts, per-frame scans into bit offsets
  auto measure = [&] {
    return for_each_chunk(n, [&](int i0, int cnt) {
      const PtrBatch src = gather<PtrBatch>(host_src_ptrs, i0, cnt);
      int e = launch_kernel("h264_mb_kernel", st, [&] {
        h264_mb_kernel<<<cnt, kWarps * 32, 0, st>>>(src, i0, g, qp, qpc, recs, recon);
      });
      if (e) return e;
      const SliceHeads h = heads(i0, cnt);
      e = launch_kernel("h264_bits_kernel<count>", st, [&] {
        h264_bits_kernel<false><<<dim3(mb_blocks, (unsigned)cnt), kThreads, 0, st>>>(i0, g, recs, mb_bit, h, EmitIn{});
      });
      if (e) return e;
      return launch_kernel("h264_scan_kernel", st, [&] {
        h264_scan_kernel<<<cnt, 1024, 0, st>>>(i0, nm, h, mb_bit, bits);
      });
    });
  };
  // each macroblock's bits at its offset in its frame's payload
  auto emit = [&](int i0, int cnt, uint8_t* streams, const uint64_t* stream_off) {
    EmitIn ei = {streams, {}};
    for (int j = 0; j < cnt; ++j) ei.stream_off[j] = stream_off[j];
    const SliceHeads h = heads(i0, cnt);
    return launch_kernel("h264_bits_kernel<emit>", st, [&] {
      h264_bits_kernel<true><<<dim3(mb_blocks, (unsigned)cnt), kThreads, 0, st>>>(i0, g, recs, mb_bit, h, ei);
    });
  };
  return run_output_stage<EmulationPrevention>(n, st, pool, s, bits, idr.data(), ax, measure, emit, alloc_out,
                                               alloc_ctx, host_sizes);
}
