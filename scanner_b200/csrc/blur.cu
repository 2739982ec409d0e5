// blur.cu -- integer box filter on u8 HWC 3-channel frames (sm_90a).
// Replaces BlurKernel::execute (reference tests/test_ops.cpp:265-294): for interior pixels
// out = (sum of the (fl+fr+1)^2 window) / (fl+fr+1)^2 with fl = ceil(k/2)-1, fr = k/2; the
// reference never writes the border of its freshly allocated frame -- here it is written as 0.
// Integer, bit-exact on the interior.
//
// The launcher takes the first kernel that fits the batch:
//   box_packed_kernel<K> kernel_size 2..31 on 16-byte aligned rows (every BASELINE frame size): u16x2 lanes, running
//                 vertical sums, 128-bit loads two rows ahead; 3.9 TB/s at K = 3 (60 % of the copy peak), > 3 TB/s to K = 9.
//   box3_kernel   kernel_size 3 on 4-byte aligned rows.  A thread owns one 32-bit column of the byte
//                 image (4 bytes = 1 1/3 pixels) and walks down a strip of rows.  The three taps of
//                 the horizontal pass are byte-shifted views of three neighbouring words (funnel
//                 shifts), summed as packed u16x2 lanes; the vertical pass is a 3-row sliding sum
//                 held in registers; /9 is an exact multiply-shift; four results are stored as one
//                 32-bit word.  No shared memory: neighbouring threads' loads overlap in L1.
//   box_generic_kernel   the rest (unaligned or tiny frames, kernel_size 1): shared-memory tile, direct sums.
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
// ~6-12 instructions per byte (K = 3..15).
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
  // byte offsets within a row reach width * 3 plus a tile's halo in int arithmetic: 2^29 pixels keep them far
  // from INT_MAX
  if (n < 0 || width <= 0 || width > (1 << 29) || height <= 0 || ksize < 1 || ksize > KMAX) return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!sp || !dp) return SCN_E_BADARG;
  const int fl = (ksize + 1) / 2 - 1;  // ceil(k/2.0) - 1
  const int fr = ksize / 2;
  const int k = fl + fr + 1;
  const int in_w = TW + k - 1, in_h = TH + k - 1;
  const size_t smem = (((size_t)in_h * in_w * 3 + 15) & ~(size_t)15) + (size_t)in_h * TW * 3 * 2;
  // box_generic_kernel's grid has one y block per TH rows (at most 65535); past this bound no row count is
  // rounded up in int arithmetic either
  if (height > 65535 * TH) return SCN_E_UNSUPPORTED;
  return for_each_chunk(n, [&](int i0, int cnt) {
    const PtrBatch s = gather<PtrBatch>(sp, i0, cnt);
    const MutPtrBatch d = gather<MutPtrBatch>(dp, i0, cnt);
    if ((width % 16) == 0 && height >= k && k >= 2 && aligned(16, i0, cnt, sp, dp)) {
      const unsigned d2 = (unsigned)(k * k);
      const uint32_t magic = (uint32_t)((1ull << 32) / d2) + 1u;  // floor(v * magic / 2^32) == v / d2 for v <= 255 * d2
      const int quads = width * 3 / 16;
      const int out_quads = 32 - 2 * ((3 * fr + 15) / 16);
      const unsigned gx = (unsigned)((quads + out_quads * BP_WARPS - 1) / (out_quads * BP_WARPS));
      // rows per strip: a strip re-reads k - 1 rows of its neighbour; shorter strips when the grid would not fill the GPU
      int rows = 128;
      while (rows > 32 && (size_t)gx * ((height + rows - 1) / rows) * cnt < 2 * (size_t)sm_count()) rows >>= 1;
      dim3 grid(gx, (unsigned)((height + rows - 1) / rows), (unsigned)cnt);
      return launch_kernel("box_packed_kernel", st, [&] {
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
      });
    }
    if (ksize == 3 && (width % 4) == 0 && width >= 4 && height >= 3 && aligned(4, i0, cnt, sp, dp)) {
      const int wpr = width * 3 / 4;
      dim3 grid((unsigned)((wpr + B3_THREADS - 1) / B3_THREADS), (unsigned)((height + B3_ROWS - 1) / B3_ROWS),
                (unsigned)cnt);
      return launch_kernel("box3_kernel", st, [&] { box3_kernel<<<grid, B3_THREADS, 0, st>>>(s, d, width, height, wpr); });
    }
    // at most 41,296 bytes of dynamic shared memory (k = 31): under the default limit
    dim3 grid((unsigned)((width + TW - 1) / TW), (unsigned)((height + TH - 1) / TH), (unsigned)cnt);
    return launch_kernel("box_generic_kernel", st,
                         [&] { box_generic_kernel<<<grid, BT, smem, st>>>(s, d, width, height, fl, fr); });
  });
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
  // n <= 0: the same argument checks as the pointer-list entry, no launch
  if (n <= 0) return scn::launch_blur(nullptr, n, width, height, kernel_size, nullptr, (cudaStream_t)stream);
  if (!src || !dst) return SCN_E_BADARG;
  return scn::launch_blur(scn::strided(src, stride_bytes, n).data(), n, width, height, kernel_size,
                          scn::strided(dst, stride_bytes, n).data(), (cudaStream_t)stream);
}
