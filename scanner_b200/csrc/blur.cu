// blur.cu -- integer box filter on u8 HWC 3-channel frames (sm_90a).
// Replaces BlurKernel::execute (reference tests/test_ops.cpp:265-294): for interior pixels
// out = (sum of the (fl+fr+1)^2 window) / (fl+fr+1)^2 with fl = ceil(k/2)-1, fr = k/2; the
// reference never writes the border of its freshly allocated frame -- here it is written as 0.
// Integer, bit-exact on the interior.
//
//   box3_kernel   kernel_size 3 (BASELINE configs[2]).  A thread owns one 32-bit column of the byte
//                 image (4 bytes = 1 1/3 pixels) and walks down a strip of rows.  The three taps of
//                 the horizontal pass are byte-shifted views of three neighbouring words (funnel
//                 shifts), summed as packed u16x2 lanes; the vertical pass is a 3-row sliding sum
//                 held in registers; /9 is an exact multiply-shift; four results are stored as one
//                 32-bit word.  No shared memory: neighbouring threads' loads overlap in L1.
//   box_packed_kernel<K> kernel_size 2..31 on 16-byte aligned rows (every BASELINE frame size): u16x2 lanes, running
//                 vertical sums, 128-bit loads two rows ahead; 3.9 TB/s at K = 3 (60 % of the copy peak), > 3 TB/s to K = 9.
//   box_stream_kernel    SCN_BLUR_PATH=stream only (r02 first kernel): bulk-async (cp.async.bulk + mbarrier) row
//                 ring, sliding horizontal sums, running vertical sums: O(1) work per sample.
//   box_generic_kernel   the rest (unaligned or tiny frames, kernel_size 1): shared-memory tile, direct sums.
#include <string.h>

#include "scn_common.cuh"

namespace scn {
namespace {

// ---------------------------------------------------------------------------------------------
constexpr int B3_THREADS = 256;
constexpr int B3_ROWS = 64;  // output rows per CTA strip

// packed u16x2 horizontal sums of the 4 bytes of a word column: even = bytes 0,2 ; odd = bytes 1,3
struct H3 {
  uint32_t even, odd;
};

__device__ __forceinline__ H3 hsum3(uint32_t wm, uint32_t w0, uint32_t wp) {
  // byte views: A = bytes [x-3 .. x], B = [x .. x+3], C = [x+3 .. x+6]
  const uint32_t A = __funnelshift_r(wm, w0, 8);
  const uint32_t C = __funnelshift_r(w0, wp, 24);
  H3 h;
  h.even = (A & 0x00FF00FFu) + (w0 & 0x00FF00FFu) + (C & 0x00FF00FFu);
  h.odd = prmt(A, 0u, 0x4341u) + prmt(w0, 0u, 0x4341u) + prmt(C, 0u, 0x4341u);
  return h;
}

// floor(v / 9) for v <= 2295 (3*3*255): (v * 7282) >> 16, exact (checked exhaustively in the tests)
__device__ __forceinline__ uint32_t div9_pack(uint32_t even, uint32_t odd) {
  const uint32_t e0 = ((even & 0xFFFFu) * 7282u) >> 16, e1 = __umulhi(even & 0xFFFF0000u, 7282u);
  const uint32_t o0 = ((odd & 0xFFFFu) * 7282u) >> 16, o1 = __umulhi(odd & 0xFFFF0000u, 7282u);
  return e0 | (o0 << 8) | (e1 << 16) | (o1 << 24);
}

// words_per_row = width*3/4 (requires width % 4 == 0 and 4-byte aligned frames)
__global__ void __launch_bounds__(B3_THREADS)
box3_kernel(PtrBatch src, MutPtrBatch dst, int width, int height, int words_per_row) {
  const int wx = blockIdx.x * B3_THREADS + threadIdx.x;
  if (wx >= words_per_row) return;
  const uint32_t* __restrict__ s = reinterpret_cast<const uint32_t*>(src.p[blockIdx.z]);
  uint32_t* __restrict__ d = reinterpret_cast<uint32_t*>(dst.p[blockIdx.z]);
  const int y0 = blockIdx.y * B3_ROWS;
  const int y1 = min(height, y0 + B3_ROWS);

  // bytes of this word that are interior in x: pixel = byte / 3 must be in [1, width-2]
  uint32_t xmask = 0;
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    const int px = (wx * 4 + b) / 3;
    if (px >= 1 && px <= width - 2) xmask |= 0xFFu << (8 * b);
  }
  // Loads never branch: a word left of the row / right of it / a row above or below the frame only ever feeds
  // outputs that are border samples (masked to 0 below), so the index is clamped instead of the value zeroed.
  const int wm_off = wx > 0 ? -1 : 0, wp_off = wx + 1 < words_per_row ? 1 : 0;
  struct Raw {
    uint32_t m, c, p;
  };
  auto load_raw = [&](int y) -> Raw {
    const uint32_t* row = s + (size_t)min(max(y, 0), height - 1) * words_per_row + wx;
    return Raw{__ldg(row + wm_off), __ldg(row), __ldg(row + wp_off)};
  };
  auto emit = [&](int y, const H3& a, const H3& b, const H3& c) {
    uint32_t out = 0;
    if (y >= 1 && y <= height - 2) out = div9_pack(a.even + b.even + c.even, a.odd + b.odd + c.odd) & xmask;
    d[(size_t)y * words_per_row + wx] = out;
  };

  // The kernel is latency-bound when a thread has one row (3 words) in flight: 64 warps x 128 B = 8 KB per SM
  // against the ~35 KB that 6.5 TB/s x ~0.8 us need (r01: 43 % of the copy peak).  Four rows are requested before
  // the first is consumed.
  Raw ra = load_raw(y0 - 1), rb = load_raw(y0);
  H3 a = hsum3(ra.m, ra.c, ra.p), b = hsum3(rb.m, rb.c, rb.p);
  int y = y0;
  for (; y + 4 <= y1; y += 4) {
    const Raw r0 = load_raw(y + 1), r1 = load_raw(y + 2), r2 = load_raw(y + 3), r3 = load_raw(y + 4);
    const H3 c0 = hsum3(r0.m, r0.c, r0.p);
    emit(y, a, b, c0);
    const H3 c1 = hsum3(r1.m, r1.c, r1.p);
    emit(y + 1, b, c0, c1);
    const H3 c2 = hsum3(r2.m, r2.c, r2.p);
    emit(y + 2, c0, c1, c2);
    const H3 c3 = hsum3(r3.m, r3.c, r3.p);
    emit(y + 3, c1, c2, c3);
    a = c2;
    b = c3;
  }
  for (; y < y1; ++y) {
    const Raw r = load_raw(y + 1);
    const H3 c = hsum3(r.m, r.c, r.p);
    emit(y, a, b, c);
    a = b;
    b = c;
  }
}

// ---------------------------------------------------------------------------------------------
constexpr int TW = 64;   // tile width in pixels
constexpr int TH = 32;   // tile height in pixels
constexpr int KMAX = 31;
constexpr int BT = 256;  // 8 warps: warp <-> row, lane <-> byte

__global__ void __launch_bounds__(BT)
box_generic_kernel(PtrBatch src, MutPtrBatch dst, int width, int height, int fl, int fr) {
  extern __shared__ uint8_t smem_raw[];
  const int k = fl + fr + 1;
  const int in_w = TW + k - 1, in_h = TH + k - 1;
  const int in_wb = in_w * 3, out_wb = TW * 3;
  uint8_t* tile = smem_raw;                                                              // in_h x in_wb
  uint16_t* hsum = reinterpret_cast<uint16_t*>(smem_raw + ((in_h * in_wb + 15) & ~15));  // in_h x out_wb
  const uint8_t* __restrict__ s = src.p[blockIdx.z];
  uint8_t* __restrict__ d = dst.p[blockIdx.z];
  const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row_bytes = width * 3;

  for (int r = warp; r < in_h; r += BT / 32) {
    const int sy = y0 - fl + r;
    const bool row_ok = sy >= 0 && sy < height;
    const uint8_t* srow = s + (size_t)(row_ok ? sy : 0) * row_bytes;
    const int xb0 = (x0 - fl) * 3;
    for (int c = lane; c < in_wb; c += 32) {
      const int sxb = xb0 + c;
      tile[r * in_wb + c] = (row_ok && sxb >= 0 && sxb < row_bytes) ? __ldg(srow + sxb) : (uint8_t)0;
    }
  }
  __syncthreads();
  for (int r = warp; r < in_h; r += BT / 32) {
    const uint8_t* trow = tile + r * in_wb;
    for (int c = lane; c < out_wb; c += 32) {
      uint32_t acc = 0;
      for (int j = 0; j < k; ++j) acc += trow[c + j * 3];
      hsum[r * out_wb + c] = (uint16_t)acc;  // <= 31 * 255
    }
  }
  __syncthreads();
  const uint32_t div = (uint32_t)(k * k);
  for (int r = warp; r < TH; r += BT / 32) {
    const int y = y0 + r;
    if (y >= height) break;
    const bool row_in = y >= fl && y < height - fr;
    for (int c = lane; c < out_wb; c += 32) {
      const int xb = x0 * 3 + c;
      if (xb >= row_bytes) break;
      uint32_t acc = 0;
      for (int j = 0; j < k; ++j) acc += hsum[(r + j) * out_wb + c];
      const int x = xb / 3;
      const bool interior = row_in && x >= fl && x < width - fr;
      d[(size_t)y * row_bytes + xb] = interior ? (uint8_t)(acc / div) : (uint8_t)0;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// box_stream_kernel: any kernel_size, O(1) work per sample.  A CTA owns a strip of kStripBytes byte
// columns and walks down kStripRows output rows:
//   * each input row segment arrives by ONE bulk-async copy (cp.async.bulk global -> shared, completion on
//     an mbarrier) into a ring of kRowSlots slots, issued kRowSlots - 1 rows ahead by one thread;
//   * horizontal pass: a thread owns 4 pixels (12 bytes); the first pixel's window is summed directly, the
//     next three slide (add the entering sample, drop the leaving one);
//   * vertical pass: running column sums in registers: + this row's horizontal sums, - those of the row
//     that leaves the window (kept in a shared-memory ring of k rows of u16);
//   * out = sum / k^2 by an exact multiply-shift, 12 bytes stored per thread (a warp writes 384 contiguous
//     bytes).  Border samples (window not inside the frame) are written as 0, so whatever a row segment
//     holds beyond the frame never reaches an output.
// Needs 16-byte aligned rows (width % 16 == 0, 16-byte aligned frames).
constexpr int kStripBytes = 3072;  // 1024 pixels: 256 threads x 12 bytes
constexpr int kStripRows = 128;
constexpr int kRowSlots = 4;
constexpr int BS = 256;

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nWAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

__global__ void __launch_bounds__(BS)
box_stream_kernel(PtrBatch src, MutPtrBatch dst, int width, int height, int fl, int fr, uint32_t div_magic) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  __shared__ __align__(8) unsigned long long bars[kRowSlots];
  const int k = fl + fr + 1;
  const int row_bytes = width * 3;
  const int x0b = blockIdx.x * kStripBytes;                       // first output byte column of the strip
  const int out_wb = min(kStripBytes, row_bytes - x0b);
  // bytes of a row this strip reads: [c0, c1), widened to 16-byte boundaries, clipped to the row
  const int c0 = max(0, (x0b - 3 * fl) & ~15);
  const int c1 = min(row_bytes, (x0b + out_wb + 3 * fr + 15) & ~15);
  const int seg = c1 - c0;
  const int lead = x0b - c0;                                      // strip byte 0 sits at segment byte `lead`
  // a slot: kLeftPad bytes nobody writes (reads of a border pixel's window may fall before the segment),
  // then the segment: at most kStripBytes + 2 * (45 + 15) bytes (KMAX = 31: fl, fr <= 15)
  constexpr int kLeftPad = 48;
  constexpr int kSegMax = kLeftPad + kStripBytes + 128;
  uint8_t* rows = smem_raw;                                       // kRowSlots x kSegMax
  uint16_t* hring = reinterpret_cast<uint16_t*>(smem_raw + kRowSlots * kSegMax);  // k x kStripBytes
  const uint8_t* __restrict__ s = src.p[blockIdx.z];
  uint8_t* __restrict__ d = dst.p[blockIdx.z];
  const int y_out0 = blockIdx.y * kStripRows, y_out1 = min(height, y_out0 + kStripRows);
  // input rows needed: [y_out0 - fl, y_out1 + fr), clipped; rows outside the frame only feed border outputs
  const int r_first = max(0, y_out0 - fl), r_last = min(height, y_out1 + fr);
  const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(bars);
  const uint32_t rows_s = (uint32_t)__cvta_generic_to_shared(rows);
  const int t = threadIdx.x;
  if (t == 0) {
    for (int i = 0; i < kRowSlots; ++i) mbar_init(bar0 + 8 * i, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int r) {  // thread 0: bulk copy of input row r into its slot
    const int slot = (r - r_first) % kRowSlots;
    mbar_expect_tx(bar0 + 8 * slot, (uint32_t)seg);
    bulk_g2s(rows_s + slot * kSegMax + kLeftPad, s + (size_t)r * row_bytes + c0, (uint32_t)seg, bar0 + 8 * slot);
  };
  if (t == 0)
    for (int r = r_first; r < min(r_last, r_first + kRowSlots - 1); ++r) issue(r);

  const int b0 = 12 * t;                       // this thread's first output byte in the strip
  const bool active = b0 < out_wb;             // out_wb is a multiple of 12 (row_bytes % 48 == 0, strips of 3072)
  uint32_t vsum[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) vsum[i] = 0;
  // x-interior flags of the 4 pixels
  bool xin[4];
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int px = (x0b + b0) / 3 + p;
    xin[p] = px >= fl && px < width - fr;
  }

  for (int r = r_first; r < r_last; ++r) {
    const int idx = r - r_first, slot = idx % kRowSlots;
    if (t == 0 && r + kRowSlots - 1 < r_last) issue(r + kRowSlots - 1);   // its slot was released by the last barrier
    mbar_wait(bar0 + 8 * slot, (uint32_t)((idx / kRowSlots) & 1));
    uint16_t h[12];
    if (active) {
      const uint8_t* row = rows + slot * kSegMax + kLeftPad + lead + b0;
      // window of pixel 0 summed directly: samples at byte offsets 3 * (j - fl) + ch (a border pixel's window
      // may start in the pad or end in stale bytes: its output is masked); pixels 1..3 slide
      uint32_t a0 = 0, a1 = 0, a2 = 0;
      const int lo = -3 * fl;
      for (int j = 0; j < k; ++j) {
        a0 += row[lo + 3 * j + 0];
        a1 += row[lo + 3 * j + 1];
        a2 += row[lo + 3 * j + 2];
      }
      h[0] = (uint16_t)a0;
      h[1] = (uint16_t)a1;
      h[2] = (uint16_t)a2;
#pragma unroll
      for (int p = 1; p < 4; ++p) {
        a0 += row[3 * (p + fr) + 0] - row[3 * (p - 1 - fl) + 0];
        a1 += row[3 * (p + fr) + 1] - row[3 * (p - 1 - fl) + 1];
        a2 += row[3 * (p + fr) + 2] - row[3 * (p - 1 - fl) + 2];
        h[3 * p + 0] = (uint16_t)a0;
        h[3 * p + 1] = (uint16_t)a1;
        h[3 * p + 2] = (uint16_t)a2;
      }
      // vertical running sums: + this row, - the row leaving the window (input row r - k, if it was fed);
      // the ring holds 12 u16 per thread = three 8-byte words
      uint2* hslot = reinterpret_cast<uint2*>(hring + (size_t)(idx % k) * kStripBytes + b0);
      if (idx >= k) {
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          const uint2 o = hslot[q];
          vsum[4 * q + 0] -= o.x & 0xFFFFu;
          vsum[4 * q + 1] -= o.x >> 16;
          vsum[4 * q + 2] -= o.y & 0xFFFFu;
          vsum[4 * q + 3] -= o.y >> 16;
        }
      }
#pragma unroll
      for (int i = 0; i < 12; ++i) vsum[i] += h[i];
#pragma unroll
      for (int q = 0; q < 3; ++q)
        hslot[q] = make_uint2((uint32_t)h[4 * q] | ((uint32_t)h[4 * q + 1] << 16), (uint32_t)h[4 * q + 2] | ((uint32_t)h[4 * q + 3] << 16));
      // output row y = r - fr is complete once input row r is in (its window is rows y-fl .. y+fr)
      const int y = r - fr;
      if (y >= y_out0 && y < y_out1) {
        const bool yin = y >= fl && y < height - fr;
        uint32_t o[12];
#pragma unroll
        for (int i = 0; i < 12; ++i) o[i] = (yin && xin[i / 3]) ? __umulhi(vsum[i], div_magic) : 0u;
        uint32_t* dp = reinterpret_cast<uint32_t*>(d + (size_t)y * row_bytes + x0b + b0);
        dp[0] = o[0] | (o[1] << 8) | (o[2] << 16) | (o[3] << 24);
        dp[1] = o[4] | (o[5] << 8) | (o[6] << 16) | (o[7] << 24);
        dp[2] = o[8] | (o[9] << 8) | (o[10] << 16) | (o[11] << 24);
      }
    }
    __syncthreads();  // everyone is done with this row's slot: thread 0 may refill it next iteration
  }
  // output rows whose window reaches below the frame are border rows: written as 0 (their input rows never came)
  for (int y = max(y_out0, r_last - fr); y < y_out1; ++y) {
    if (active && y >= 0) {
      uint32_t* dp = reinterpret_cast<uint32_t*>(d + (size_t)y * row_bytes + x0b + b0);
      dp[0] = dp[1] = dp[2] = 0u;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// box_packed_kernel<K>: kernel_size 2..31 on 16-byte aligned rows, all arithmetic on packed u16x2 lanes.
//   * a thread owns one 16-byte column (a "quad": 4 words) and walks down a strip of rows; a warp owns 32
//     neighbouring quads of which the R on each side are halo (R = 1 for K <= 11, 2 up to K = 21, else 3);
//   * vertical first: running column sums  acc += row(r) - row(r - K)  with the bytes of a word split into its even
//     (0, 2) and odd (1, 3) bytes as u16 lanes -- one IADD3 adds the entering and subtracts the leaving row for two
//     byte columns (lanes cannot borrow: the true lane values stay in [0, 255 K]).  Both rows come by 128-bit loads
//     (the leaving row from L2), requested one iteration ahead;
//   * the warp publishes its 32 x 8 lane-words to its own shared-memory row (double-buffered, __syncwarp only) and
//     every thread reads its neighbours' (2R + 1) quads back with 128-bit loads;
//   * horizontal: the window of the byte pair (b, b + 2) is K terms 3 bytes apart; a term is, depending on its byte
//     offset mod 4, an even-lane word, an odd-lane word, or one of those shifted by one lane into the next word
//     (funnel shift, computed once per word and shared by all outputs): (K - 1) / 2 IADD3 per pair, every index a
//     compile-time constant.  Lane sums stay below 255 K^2 <= 65280 for K <= 16; above, the terms are summed in
//     groups of 8 (8 x 255 x 31 fits a lane) and the groups unpacked into 32-bit sums;
//   * out = sum / K^2 by the exact multiply-shift, border samples masked to 0, one 128-bit store per thread.
// ~6-12 instructions per byte (K = 3..15) where box_stream_kernel spends 15 and more on byte loads.
constexpr int BP_WARPS = 4;
template <int K>
struct PackedGeom {
  static constexpr int fl = (K + 1) / 2 - 1, fr = K / 2;
  static constexpr int R = (3 * fr + 15) / 16;       // halo quads on each side of a thread's quad
  static constexpr int NW = 4 * (2 * R + 1);         // lane-words a thread reads back
  static constexpr int OUT_QUADS = 32 - 2 * R;       // output quads per warp
  static constexpr int kGroup = K <= 16 ? K : 8;     // terms whose packed sum still fits a u16 lane (255 K per term)
  static_assert(255 * K * kGroup <= 65535, "a group of packed terms must not carry into the next lane");
  static_assert(3 * fr <= 16 * R && 3 * fl <= 16 * R, "the halo must cover the window");
};

template <int K>
__global__ void __launch_bounds__(BP_WARPS * 32)
box_packed_kernel(PtrBatch src, MutPtrBatch dst, int width, int height, int rows_per_strip, uint32_t div_magic) {
  using G = PackedGeom<K>;
  constexpr int fl = G::fl, fr = G::fr, R = G::R, NW = G::NW;
  __shared__ __align__(16) uint4 vbuf[BP_WARPS][2][2][32];  // [warp][parity][even / odd lanes][quad]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int quads = width * 3 / 16;
  const int q_out = (blockIdx.x * BP_WARPS + warp) * G::OUT_QUADS + lane - R;  // the quad this lane would output
  if ((blockIdx.x * BP_WARPS + warp) * G::OUT_QUADS >= quads) return;           // whole warp beyond the row
  const int q_ld = min(max(q_out, 0), quads - 1);   // clamped: a duplicate only ever feeds border samples
  const bool writes = lane >= R && lane < 32 - R && q_out < quads;
  const uint4* __restrict__ s = reinterpret_cast<const uint4*>(src.p[blockIdx.z]) + q_ld;
  uint4* __restrict__ d = reinterpret_cast<uint4*>(dst.p[blockIdx.z]) + q_ld;
  const int y0 = blockIdx.y * rows_per_strip, y1 = min(height, y0 + rows_per_strip);
  // byte masks of the x-interior samples of this quad
  uint32_t xmask[4];
#pragma unroll
  for (int w = 0; w < 4; ++w) {
    xmask[w] = 0;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int px = (q_ld * 16 + w * 4 + b) / 3;
      if (px >= fl && px < width - fr) xmask[w] |= 0xFFu << (8 * b);
    }
  }
  uint32_t accE[4] = {0, 0, 0, 0}, accO[4] = {0, 0, 0, 0};
  const int r_first = y0 - fl, r_last = y1 + fr;  // input rows [r_first, r_last)
  // Rows outside the frame count as zero (they only reach border outputs), so the row pointer simply advances by one
  // row per step and the loads are predicated on the (warp-uniform) row number; the leaving row is K rows behind.
  // running pointers: pn = the row the next load_rows() call reads, po = K rows behind it, pd = the next output row
  const uint4* pn = s + (ptrdiff_t)r_first * quads;
  const uint4* po = pn - (ptrdiff_t)K * quads;
  uint4* pd = d + (ptrdiff_t)y0 * quads;
  int r_ld = r_first;
  auto load_rows = [&](uint4& nw, uint4& od) {  // rows r_ld and r_ld - K (the latter once the window is full)
    const int ro = r_ld - K;
    nw = r_ld < r_last && r_ld >= 0 && r_ld < height ? __ldg(pn) : make_uint4(0, 0, 0, 0);
    od = r_ld < r_last && ro >= r_first && ro >= 0 && ro < height ? __ldg(po) : make_uint4(0, 0, 0, 0);
    pn += quads;
    po += quads;
    ++r_ld;
  };
  uint4* const my_e = &vbuf[warp][0][0][lane];  // + 64 uint4 for the odd lanes, + 128 for the other parity
  const uint4* const nb = my_e - R;

  auto process = [&](int r, const uint4& nw, const uint4& od) {
    const uint32_t n4[4] = {nw.x, nw.y, nw.z, nw.w}, o4[4] = {od.x, od.y, od.z, od.w};
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      accE[w] = accE[w] + (n4[w] & 0x00FF00FFu) - (o4[w] & 0x00FF00FFu);
      accO[w] = accO[w] + prmt(n4[w], 0u, 0x4341u) - prmt(o4[w], 0u, 0x4341u);
    }
    const int y = r - fr;
    if (y < y0) return;  // warp-uniform
    const int par = (y & 1) * 64;
    my_e[par] = make_uint4(accE[0], accE[1], accE[2], accE[3]);
    my_e[par + 32] = make_uint4(accO[0], accO[1], accO[2], accO[3]);
    __syncwarp();
    if (writes) {
      uint4 out = make_uint4(0, 0, 0, 0);
      if (y >= fl && y < height - fr) {
        // lane-words of quads lane - R .. lane + R: index 4 * R + i = word i of the own quad
        uint32_t VE[NW], VO[NW];
#pragma unroll
        for (int k = 0; k < 2 * R + 1; ++k) {
          const uint4 e = nb[par + k], o = nb[par + 32 + k];
          VE[4 * k] = e.x, VE[4 * k + 1] = e.y, VE[4 * k + 2] = e.z, VE[4 * k + 3] = e.w;
          VO[4 * k] = o.x, VO[4 * k + 1] = o.y, VO[4 * k + 2] = o.z, VO[4 * k + 3] = o.w;
        }
        // streams shifted by one lane: (hi of word i, lo of word i + 1)
        uint32_t SE[NW - 1], SO[NW - 1];
#pragma unroll
        for (int i = 0; i < NW - 1; ++i) {
          SE[i] = __funnelshift_r(VE[i], VE[i + 1], 16);
          SO[i] = __funnelshift_r(VO[i], VO[i + 1], 16);
        }
        uint32_t ow[4];
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          // window sums of the byte pairs (0, 2) and (1, 3) of word w, as four 32-bit values.  A u16 lane holds at
          // most 65535 = 8 terms of 255 * 31: the K terms are summed packed in groups of kGroup and the groups
          // unpacked (K <= 16: one group, exactly the code there was before kernel sizes above 16 came here)
          uint32_t e_lo = 0, e_hi = 0, o_lo = 0, o_hi = 0;
#pragma unroll
          for (int j0 = 0; j0 < K; j0 += G::kGroup) {
            uint32_t he = 0, ho = 0;
#pragma unroll
            for (int j = j0; j < (j0 + G::kGroup < K ? j0 + G::kGroup : K); ++j) {
              // first byte of the pair's term j, relative to the own quad's byte 0, offset so that it is >= 0
              const int te = 16 * R + 4 * w + 3 * (j - fl), to = te + 1;
              const int we = te >> 2, wo = to >> 2;
              he += (te & 3) == 0 ? VE[we] : (te & 3) == 1 ? VO[we] : (te & 3) == 2 ? SE[we] : SO[we];
              ho += (to & 3) == 0 ? VE[wo] : (to & 3) == 1 ? VO[wo] : (to & 3) == 2 ? SE[wo] : SO[wo];
            }
            e_lo += he & 0xFFFFu;
            e_hi += he >> 16;
            o_lo += ho & 0xFFFFu;
            o_hi += ho >> 16;
          }
          const uint32_t e0 = __umulhi(e_lo, div_magic), e1 = __umulhi(e_hi, div_magic);
          const uint32_t o0 = __umulhi(o_lo, div_magic), o1 = __umulhi(o_hi, div_magic);
          // quotients are < 256: byte 1 of each is zero and serves as the zero source of the packing
          ow[w] = prmt(prmt(e0, o0, 0x1140u), prmt(e1, o1, 0x1140u), 0x5410u) & xmask[w];
        }
        out = make_uint4(ow[0], ow[1], ow[2], ow[3]);
      }
      *pd = out;
    }
    pd += quads;
  };

  // two rows per iteration, each row's loads requested one step ahead (no register rotation)
  // three rows per iteration, every row's two loads requested two rows ahead of their use (three register sets, no
  // rotation): with one row ahead the kernel sat at ~53 % of the copy peak for every K <= 9 -- latency, not issue
  uint4 nA, oA, nB, oB, nC, oC;
  load_rows(nA, oA);
  load_rows(nB, oB);
  for (int r = r_first; r < r_last; r += 3) {
    load_rows(nC, oC);
    process(r, nA, oA);
    load_rows(nA, oA);
    if (r + 1 < r_last) process(r + 1, nB, oB);
    load_rows(nB, oB);
    if (r + 2 < r_last) process(r + 2, nC, oC);
  }
}

int launch_blur(const uint8_t* const* sp, int n, int width, int height, int ksize,
                uint8_t* const* dp, cudaStream_t st) {
  if (n < 0 || width <= 0 || height <= 0 || ksize < 1 || ksize > KMAX) return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!sp || !dp) return SCN_E_BADARG;
  const int fl = (ksize + 1) / 2 - 1;  // ceil(k/2.0) - 1
  const int fr = ksize / 2;
  const int k = fl + fr + 1;
  const int in_w = TW + k - 1, in_h = TH + k - 1;
  const size_t smem = (((size_t)in_h * in_w * 3 + 15) & ~(size_t)15) + (size_t)in_h * TW * 3 * 2;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(box_generic_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         100 * 1024);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  if (((height + TH - 1) / TH) > 65535) return SCN_E_UNSUPPORTED;
  for (int i0 = 0; i0 < n; i0 += SCN_MAX_PTRS) {
    const int cnt = (n - i0 < SCN_MAX_PTRS) ? (n - i0) : SCN_MAX_PTRS;
    PtrBatch s;
    MutPtrBatch d;
    bool aligned = (width % 4) == 0 && width >= 4 && height >= 3;
    for (int i = 0; i < cnt; ++i) {
      s.p[i] = sp[i0 + i];
      d.p[i] = dp[i0 + i];
      if (((uintptr_t)s.p[i] | (uintptr_t)d.p[i]) & 3) aligned = false;
    }
    bool aligned16 = (width % 16) == 0 && height >= k;
    for (int i = 0; i < cnt; ++i)
      if (((uintptr_t)s.p[i] | (uintptr_t)d.p[i]) & 15) aligned16 = false;
    static const bool stream3 = [] {
      const char* e = getenv("SCN_BLUR3");
      return e && e[0] == 's';  // SCN_BLUR3=stream: kernel_size 3 through the streaming kernel too (measurement switch)
    }();
    // SCN_BLUR_PATH=stream keeps kernel sizes 2..16 on the byte-wise streaming kernel; =box3 keeps kernel_size 3 on
    // box3_kernel even when the rows are 16-byte aligned (measurement switches)
    static const int path = [] {
      const char* e = getenv("SCN_BLUR_PATH");
      return !e ? 0 : strcmp(e, "stream") == 0 ? 1 : strcmp(e, "box3") == 0 ? 2 : 0;
    }();
    if (aligned16 && k >= 2 && k <= 31 && path != 1 && (ksize != 3 || path != 2)) {
      const unsigned d2 = (unsigned)(k * k);
      const uint32_t magic = (uint32_t)((1ull << 32) / d2) + 1u;
      const int quads = width * 3 / 16;
      const int out_quads = 32 - 2 * ((3 * fr + 15) / 16);
      const unsigned gx = (unsigned)((quads + out_quads * BP_WARPS - 1) / (out_quads * BP_WARPS));
      // rows per strip: a strip re-reads k - 1 rows of its neighbour; shorter strips when the grid would not fill the GPU
      int rows = 128;
      while (rows > 32 && (size_t)gx * ((height + rows - 1) / rows) * cnt < 2 * (size_t)sm_count()) rows >>= 1;
      dim3 grid(gx, (unsigned)((height + rows - 1) / rows), (unsigned)cnt);
      LaunchScope ls("box_packed_kernel", st);
      switch (k) {
#define SCN_BP_CASE(KK) \
  case KK: box_packed_kernel<KK><<<grid, BP_WARPS * 32, 0, st>>>(s, d, width, height, rows, magic); break;
        SCN_BP_CASE(2) SCN_BP_CASE(3) SCN_BP_CASE(4) SCN_BP_CASE(5) SCN_BP_CASE(6) SCN_BP_CASE(7) SCN_BP_CASE(8)
        SCN_BP_CASE(9) SCN_BP_CASE(10) SCN_BP_CASE(11) SCN_BP_CASE(12) SCN_BP_CASE(13) SCN_BP_CASE(14)
        SCN_BP_CASE(15) SCN_BP_CASE(16) SCN_BP_CASE(17) SCN_BP_CASE(18) SCN_BP_CASE(19) SCN_BP_CASE(20) SCN_BP_CASE(21)
        SCN_BP_CASE(22) SCN_BP_CASE(23) SCN_BP_CASE(24) SCN_BP_CASE(25) SCN_BP_CASE(26) SCN_BP_CASE(27) SCN_BP_CASE(28)
        SCN_BP_CASE(29) SCN_BP_CASE(30) SCN_BP_CASE(31)
#undef SCN_BP_CASE
      }
    } else if (aligned16 && k >= 2 && (ksize != 3 || stream3)) {
      const size_t smem_s = (size_t)kRowSlots * (48 + kStripBytes + 128) + (size_t)k * kStripBytes * 2;
      static bool attr2 = false;
      if (!attr2) {
        cudaError_t e = cudaFuncSetAttribute(box_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 210 * 1024);
        if (e != cudaSuccess) return (int)e;
        attr2 = true;
      }
      const unsigned d2 = (unsigned)(k * k);
      const uint32_t magic = (uint32_t)((1ull << 32) / d2) + 1u;  // floor(v * magic / 2^32) == v / d2 for v <= 255 * d2
      dim3 grid((unsigned)((width * 3 + kStripBytes - 1) / kStripBytes), (unsigned)((height + kStripRows - 1) / kStripRows),
                (unsigned)cnt);
      LaunchScope ls("box_stream_kernel", st);
      box_stream_kernel<<<grid, BS, smem_s, st>>>(s, d, width, height, fl, fr, magic);
    } else if (ksize == 3 && aligned) {
      const int wpr = width * 3 / 4;
      dim3 grid((unsigned)((wpr + B3_THREADS - 1) / B3_THREADS), (unsigned)((height + B3_ROWS - 1) / B3_ROWS),
                (unsigned)cnt);
      LaunchScope ls("box3_kernel", st);
      box3_kernel<<<grid, B3_THREADS, 0, st>>>(s, d, width, height, wpr);
    } else {
      dim3 grid((unsigned)((width + TW - 1) / TW), (unsigned)((height + TH - 1) / TH), (unsigned)cnt);
      LaunchScope ls("box_generic_kernel", st);
      box_generic_kernel<<<grid, BT, smem, st>>>(s, d, width, height, fl, fr);
    }
    int rc = launch_status();
    if (rc) return rc;
  }
  return 0;
}

}  // namespace
}  // namespace scn

extern "C" int scn_box_blur_u8c3(const uint8_t* const* host_src_ptrs, int n, int width,
                                 int height, int kernel_size, uint8_t* const* host_dst_ptrs,
                                 void* stream) {
  return scn::launch_blur(host_src_ptrs, n, width, height, kernel_size, host_dst_ptrs,
                          (cudaStream_t)stream);
}

extern "C" int scn_box_blur_u8c3_strided(const uint8_t* src, size_t stride_bytes, int n,
                                         int width, int height, int kernel_size, uint8_t* dst,
                                         void* stream) {
  if (n < 0) return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!src || !dst) return SCN_E_BADARG;
  const uint8_t* sp[SCN_MAX_PTRS];
  uint8_t* dp[SCN_MAX_PTRS];
  for (int i0 = 0; i0 < n; i0 += SCN_MAX_PTRS) {
    const int cnt = (n - i0 < SCN_MAX_PTRS) ? (n - i0) : SCN_MAX_PTRS;
    for (int i = 0; i < cnt; ++i) {
      sp[i] = src + (size_t)(i0 + i) * stride_bytes;
      dp[i] = dst + (size_t)(i0 + i) * stride_bytes;
    }
    int rc = scn::launch_blur(sp, cnt, width, height, kernel_size, dp, (cudaStream_t)stream);
    if (rc) return rc;
  }
  return 0;
}
