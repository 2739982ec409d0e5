// nv12_stream.cuh -- ONE pass over NV12 decoder surfaces for the Histogram of BASELINE configs[1]:
//     NV12 -> RGB -> Histogram (tests/test_ops.cpp:19-49)
// with the reference's NV12->RGB arithmetic (scanner/util/image.cu:67-200 as nvcc contracts it, see
// nv12_math.cuh) and no RGB frame in HBM.
//
// Design (the kernel is bound by instruction issue, not by HBM: every choice below trades ALU, FMA and
// XU (conversion) pipe work against each other so that no pipe is the only busy one):
//   * surfaces are streamed with cp.async into a per-warp shared-memory ring (no load registers, the
//     prefetch runs kStages-1 steps ahead across span and frame boundaries); a lane owns a "unit" of
//     16 pixels x 2 rows per step (two luma rows, the chroma row and the next chroma row);
//   * steps run in blocks of 4, so the fold of the carry-save carries has no run-time branches; the last steps
//     of a frame and of a span run one at a time (see the span loop);
//   * byte -> float on the XU pipe: `(float)((w >> 8k) & 0xff)` is I2F.U8 Rd, Rs.Bk -- no ALU work;
//   * colour math on the FMA pipe.  Only the 4-bit bin reaches the histogram, so any arithmetic that
//     yields the reference's bin for every input is exact by exhaustion (tests/test_ref_pin_gpu.py
//     runs the reference's own kernel on all 2^24 (Y,Cb,Cr) triples):
//       R, B (depend on 2^16 inputs each; reference values never come closer than 1.6e-3 to a bin
//             edge):  x = fma.sat(Y, a, c(chroma)),  bin = floor(15.5 x)   -- v/992 domain, both
//             clamps from .sat (v >= 992 is bin 15 anyway), ONE FMA per pixel, the chroma term per
//             chroma sample;
//       G    (2^24 inputs, values DO land on bin edges): the exact chain in a 2^-11 scaled domain
//             (power-of-two scaling commutes with IEEE rounding): gi = fma(Y, cy, fl(cb*k1)),
//             x = fma.sat(cr, k2, gi), m = floor(32 x) in 0..31, upper clamp by a second .sat;
//   * floor: fma.rm(x, k, 2^23) leaves the integer in the mantissa; four bins are packed into the
//     16-bit selector of a PRMT with IMADs on the float's bits (R, B) / an FMA accumulate (G);
//   * counting: PRMT as an 8-entry one-hot LUT + bit-sliced carry-save adders (csa_core.cuh).
// Resize of the same surfaces is nv12_resize_kernel (fused.cu), run beside this kernel on a side stream.
#pragma once
#include "csa_core.cuh"
#include "nv12_math.cuh"
#include "scn_common.cuh"

namespace scn {
namespace nvs {

constexpr int kWarps = 12;
constexpr int kThreads = kWarps * 32;
constexpr int kStages = 4;
static_assert((kStages & (kStages - 1)) == 0, "the ring index is a mask");
constexpr int kPlanes = 10;
constexpr int kHi = kPlanes - 3;   // planes 3..9
constexpr int kMaxSteps = 127;     // 127 * 8 words per accumulator <= 1023
constexpr size_t kSmemBytes = (size_t)kWarps * kStages * 4 * 32 * 16;

using Acc = csa::Acc8<kHi>;
using csa::acc_clear;
using csa::finish_span;
using csa::fold_step;
using csa::push8;

// ---- constants -----------------------------------------------------------------------------------
constexpr float kMagic = 8388608.0f;                    // 2^23
// R, B: v / 992 domain (bins only; verified exhaustively)
constexpr float kA = 4.0f * 1.1644f / 992.0f;
constexpr float kRC = 4.0f * 1.596f / 992.0f;
constexpr float kBC = 4.0f * 2.0172f / 992.0f;
// G: exact, 2^-11 scaled
constexpr float kS = 1.0f / 2048.0f;
constexpr float kCY = 4.0f * 1.1644f * kS;
constexpr float kKG1 = 4.0f * -0.3918f * kS;
constexpr float kKG2 = 4.0f * -0.813f * kS;
constexpr float kQScale = 0.0625f;
constexpr float kQBias = 0.0625f - 524288.0f;           // 1/16 - 2^19
constexpr float kSInit = kMagic - 4369.0f;              // 2^23 - 0x1111

// Two floats that take the same operation.  sm_90 has no packed f32x2 arithmetic: each helper is two
// scalar instructions with the rounding of the packed form, so the results are bit-identical to it.
struct f2 {
  float lo, hi;
};
__device__ __forceinline__ f2 pack2(float lo, float hi) { return f2{lo, hi}; }
__device__ __forceinline__ void unpack2(f2 v, float& lo, float& hi) {
  lo = v.lo;
  hi = v.hi;
}
__device__ __forceinline__ f2 splat(float v) { return pack2(v, v); }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return f2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)}; }
__device__ __forceinline__ f2 fma2_rm(f2 a, f2 b, f2 c) { return f2{__fmaf_rd(a.lo, b.lo, c.lo), __fmaf_rd(a.hi, b.hi, c.hi)}; }
__device__ __forceinline__ float fma_sat(float a, float b, float c) {
  float r;
  asm("fma.rn.sat.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c));
  return r;
}
__device__ __forceinline__ uint32_t imad(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t r;
  asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
  return r;
}
template <int K>
__device__ __forceinline__ float byte_f(uint32_t w) {  // I2F.U8 Rd, Rs.BK (XU pipe)
  return (float)((w >> (8 * K)) & 0xFFu);
}
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return f2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return f2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }

// The two (Cb,Cr) samples of a chroma word, everything that does not depend on luma, as register
// pairs (sample 0, sample 1) so that one packed instruction serves both
struct Chroma2 {
  f2 tb;      // B: fl((cb-128) * kBC)
  f2 cr;      // R: fl((cr-128) * kRC)
  f2 tg;      // G: fl((cb-128) * kKG1)      (the product image.cu rounds on its own)
  f2 crc;     // G: cr - 128
};
__device__ __forceinline__ Chroma2 chroma_terms(uint32_t cw) {
  Chroma2 c;
  // ALU pipe: PRMT builds the bits of 2^23 + byte; one exact FADD removes the bias and centres
  const f2 cbc = add2(pack2(__uint_as_float(prmt(cw, 0x4B000000u, 0x7440u)), __uint_as_float(prmt(cw, 0x4B000000u, 0x7442u))),
                      splat(-(kMagic + 128.0f)));
  c.crc = add2(pack2(__uint_as_float(prmt(cw, 0x4B000000u, 0x7441u)), __uint_as_float(prmt(cw, 0x4B000000u, 0x7443u))),
               splat(-(kMagic + 128.0f)));
  c.tb = mul2(cbc, splat(kBC));
  c.cr = mul2(c.crc, splat(kRC));
  c.tg = mul2(cbc, splat(kKG1));
  return c;
}

struct Sel {  // nibble selectors of one 4-pixel word being built
  uint32_t r, b;
  float g;
};

// one luma word: pixels 0,1 share chroma sample 0, pixels 2,3 sample 1.  Pixel j is paired with
// pixel j+2 wherever an operation has a packed form: their chroma terms already sit in one pair.
__device__ __forceinline__ void four_pixels(Sel& s, uint32_t yw, const Chroma2& c) {
  const float y0 = byte_f<0>(yw), y1 = byte_f<1>(yw), y2 = byte_f<2>(yw), y3 = byte_f<3>(yw);
  float cr0, cr1, tb0, tb1, crc0, crc1;
  unpack2(c.cr, cr0, cr1);
  unpack2(c.tb, tb0, tb1);
  unpack2(c.crc, crc0, crc1);
  const float xr0 = fma_sat(y0, kA, cr0), xr1 = fma_sat(y1, kA, cr0), xr2 = fma_sat(y2, kA, cr1), xr3 = fma_sat(y3, kA, cr1);
  const float xb0 = fma_sat(y0, kA, tb0), xb1 = fma_sat(y1, kA, tb0), xb2 = fma_sat(y2, kA, tb1), xb3 = fma_sat(y3, kA, tb1);
  float gi0, gi1, gi2, gi3;
  unpack2(fma2(pack2(y0, y2), splat(kCY), c.tg), gi0, gi2);
  unpack2(fma2(pack2(y1, y3), splat(kCY), c.tg), gi1, gi3);
  const float xg0 = fma_sat(crc0, kKG2, gi0), xg1 = fma_sat(crc0, kKG2, gi1);
  const float xg2 = fma_sat(crc1, kKG2, gi2), xg3 = fma_sat(crc1, kKG2, gi3);
  float r0, b0, r1, b1, r2, b2, r3, b3, g0, g1, g2, g3;
  unpack2(fma2_rm(pack2(xr0, xb0), splat(15.5f), splat(kMagic)), r0, b0);   // 2^23 + bin
  unpack2(fma2_rm(pack2(xr1, xb1), splat(15.5f), splat(kMagic)), r1, b1);
  unpack2(fma2_rm(pack2(xr2, xb2), splat(15.5f), splat(kMagic)), r2, b2);
  unpack2(fma2_rm(pack2(xr3, xb3), splat(15.5f), splat(kMagic)), r3, b3);
  unpack2(fma2_rm(pack2(xg0, xg1), splat(32.0f), splat(kMagic)), g0, g1);   // 2^23 + m, m in 0..31
  unpack2(fma2_rm(pack2(xg2, xg3), splat(32.0f), splat(kMagic)), g2, g3);
  // (min(m,15)+1)/16, accumulated as nibbles: G starts at 2^23 - 0x1111
  s.g = __fmaf_rn(fma_sat(g0, kQScale, kQBias), 16.0f, kSInit);
  s.g = __fmaf_rn(fma_sat(g1, kQScale, kQBias), 256.0f, s.g);
  s.g = __fmaf_rn(fma_sat(g2, kQScale, kQBias), 4096.0f, s.g);
  s.g = __fmaf_rn(fma_sat(g3, kQScale, kQBias), 65536.0f, s.g);
  // (0x4B000000 | bin) * 16^j: the low 16 bits PRMT reads hold only the nibbles
  s.r = imad(__float_as_uint(r1), 16u, __float_as_uint(r0));
  s.b = imad(__float_as_uint(b1), 16u, __float_as_uint(b0));
  s.r = imad(__float_as_uint(r2), 256u, s.r);
  s.b = imad(__float_as_uint(b2), 256u, s.b);
  s.r = imad(__float_as_uint(r3), 4096u, s.r);
  s.b = imad(__float_as_uint(b3), 4096u, s.b);
}

// `lut_lo` is csa::kLutLo held in a vector register: PRMT takes only one immediate, and as a literal
// (or any value ptxas can prove uniform) the low LUT word sits in a uniform register and is copied
// with an IMAD before every PRMT
template <int K>
__device__ __forceinline__ void count4(Acc& A, Acc& B, uint32_t z, uint32_t& cA, uint32_t& cB, uint32_t lut_lo) {
  push8<K>(A, prmt(lut_lo, csa::kLutHiA, z), cA);
  push8<K>(B, prmt(lut_lo, csa::kLutHiB, z ^ 0x8888u), cB);
}

// one luma word (4 pixels) with its chroma word (2 Cb,Cr samples): push K of every accumulator
template <int K>
__device__ __forceinline__ void quad(Acc (&A)[3], Acc (&B)[3], uint32_t (&cyA)[3], uint32_t (&cyB)[3], uint32_t yw,
                                     uint32_t cw, uint32_t lut_lo) {
  Sel s;
  four_pixels(s, yw, chroma_terms(cw));
  count4<K>(A[0], B[0], s.r, cyA[0], cyB[0], lut_lo);
  count4<K>(A[1], B[1], __float_as_uint(s.g), cyA[1], cyB[1], lut_lo);
  count4<K>(A[2], B[2], s.b, cyA[2], cyB[2], lut_lo);
}

__device__ __forceinline__ uint32_t avg4(uint32_t a, uint32_t b) {  // per byte (a + b + 1) >> 1
  return (a | b) - (((a ^ b) & 0xFEFEFEFEu) >> 1);
}

// csa::kLutLo once per lane: loaded with a per-lane index so the value is not provably uniform
__device__ const uint32_t g_lut_lo[32] = {
    csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo,
    csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo,
    csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo,
    csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo, csa::kLutLo};

struct Params {
  PtrBatch luma, chroma;
  size_t pitch;
  int width, height;
  uint32_t units_per_row;     // width / 16
  uint64_t upr_recip;         // floor(2^32 / units_per_row) + 1: 33 bits when units_per_row == 1
  uint32_t units_per_frame;   // units_per_row * height / 2
  uint32_t steps_per_frame;   // ceil(units_per_frame / 32)
  uint64_t total_steps;
  // a step moves a lane 32 units on: q = 32 / units_per_row row pairs and xs_step = 32 % units_per_row columns, plus
  // one row pair more where the column wraps.  Its pointers move by 512 + (q + wrap) * (2 * pitch - width) bytes in
  // the luma plane, 512 + (q + wrap) * (pitch - width) in the chroma plane (32 bits: see kMaxPitch)
  uint32_t xs_step;
  uint32_t inc_l, inc_l_wrap, inc_c, inc_c_wrap;
  uint32_t fast_steps;        // leading steps of a frame whose 32 units all lie above the last chroma row
};

// bounds the per-step pointer increments above (< 512 + 33 * 2 * pitch) to 32 bits
constexpr size_t kMaxPitch = (size_t)1 << 25;

__device__ __forceinline__ uint32_t lane_count(const Acc& a, int lane) {
  uint32_t pl[kPlanes + 5];
  csa::planes_of(a, pl);
  csa::warp_sum<kPlanes>(pl);
  uint32_t v = csa::extract_lane<kPlanes>(pl, lane);
  // the four byte slots of a word carry the same channel: fold them onto lanes 0..7
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  return v;
}

__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gptr, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr), "l"(gptr), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gptr) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr), "l"(gptr) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t smem_addr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(smem_addr));
  return r;
}

template <int J>
struct Phase {
  static constexpr int value = J;
};

static __global__ void __launch_bounds__(kThreads, 1)
nv12_stream_kernel(const Params prm, int32_t* __restrict__ out) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ int sh[kWarps][48];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* h = sh[warp];
  const uint64_t gwarp = (uint64_t)blockIdx.x * kWarps + warp;
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  const uint64_t g_begin = prm.total_steps * gwarp / nwarps;
  const uint64_t g_end = prm.total_steps * (gwarp + 1) / nwarps;
  const int last_crow = (prm.height >> 1) - 1;
  const uint32_t lut_lo = g_lut_lo[lane];
  // this lane's 16-byte slot in stage s, row k:  ring + ((s * 4 + k) * 32 + lane) * 16
  const uint32_t ring = (uint32_t)__cvta_generic_to_shared(smem_raw) + (uint32_t)warp * (kStages * 4 * 32 * 16) + lane * 16;

  // ring stage of global step g: g mod kStages, for the consumer and for the prefetch kStages - 1 steps ahead of it
  auto slot_of = [&](uint32_t g) { return ring + (g & (kStages - 1)) * (4 * 32 * 16); };

  // ---- prefetch side.  Two paths: fast_prefetch() serves the steps whose 32 lanes all read a unit of the frame
  // above its last chroma row (all but the last few steps of a frame) with per-lane pointers it moves on by one
  // select each; prefetch() serves any step (frame ends, padding lanes, the last chroma row, the range's end),
  // locating the lane's unit from scratch.  The consumer picks the fast path a block of 4 steps at a time.
  uint32_t pf_left = (uint32_t)(g_end - g_begin);         // steps still to prefetch
  uint32_t pf_frame = (uint32_t)(g_begin / prm.steps_per_frame);
  uint32_t pf_s = (uint32_t)(g_begin - (uint64_t)pf_frame * prm.steps_per_frame);
  uint32_t pf_fast = 0;                                    // steps from (pf_frame, pf_s) on that the fast path may take
  uint32_t pf_xs;                                          // this lane's column unit in step (pf_frame, pf_s)
  const uint8_t *pf_l, *pf_c;                              // its luma / chroma 16-byte groups
  auto locate = [&](uint32_t& yp) {                        // returns whether the lane's unit lies in the frame
    const uint32_t unit = pf_s * 32u + (uint32_t)lane;
    yp = (uint32_t)(((uint64_t)unit * prm.upr_recip) >> 32);   // == unit / units_per_row
    pf_xs = unit - yp * prm.units_per_row;
    const bool active = unit < prm.units_per_frame;        // lanes past the frame's last unit: any valid address
    pf_l = prm.luma.p[pf_frame] + (active ? (size_t)(2 * yp) * prm.pitch + (size_t)pf_xs * 16 : 0);
    pf_c = prm.chroma.p[pf_frame] + (active ? (size_t)yp * prm.pitch + (size_t)pf_xs * 16 : 0);
    return active;
  };
  auto prefetch = [&](uint32_t slot) {
    if (pf_left) {
      uint32_t yp;
      const uint32_t nbytes = locate(yp) ? 16u : 0u;     // 0: the slot is zero-filled, nothing is read
      const size_t cnext = ((int)yp < last_crow) ? prm.pitch : 0;
      cp_async16(slot, pf_l, nbytes);
      cp_async16(slot + 512, pf_l + prm.pitch, nbytes);
      cp_async16(slot + 1024, pf_c, nbytes);
      cp_async16(slot + 1536, pf_c + cnext, nbytes);
      --pf_left;
      if (++pf_s == prm.steps_per_frame) {                 // next frame (warp-uniform, once per frame)
        pf_s = 0;
        ++pf_frame;
      }
      pf_fast = pf_s < prm.fast_steps ? min(prm.fast_steps - pf_s, pf_left) : 0u;
    }
    cp_async_commit();
  };
  auto fast_prefetch = [&](uint32_t slot) {                // pointers valid (locate() at the start of a fast run)
    cp_async16(slot, pf_l);
    cp_async16(slot + 512, pf_l + prm.pitch);
    cp_async16(slot + 1024, pf_c);
    cp_async16(slot + 1536, pf_c + prm.pitch);
    cp_async_commit();
    pf_xs += prm.xs_step;                                  // < 2 * units_per_row: at most one wrap
    const bool wrap = pf_xs >= prm.units_per_row;
    pf_xs -= wrap ? prm.units_per_row : 0u;
    pf_l += wrap ? prm.inc_l_wrap : prm.inc_l;
    pf_c += wrap ? prm.inc_c_wrap : prm.inc_c;
  };
#pragma unroll
  for (int i = 0; i < kStages - 1; ++i) prefetch(slot_of((uint32_t)g_begin + i));

  uint64_t g0 = g_begin;
  while (g0 < g_end) {
    const uint32_t frame = (uint32_t)(g0 / prm.steps_per_frame);
    const uint32_t s0 = (uint32_t)(g0 - (uint64_t)frame * prm.steps_per_frame);
    uint32_t ns = prm.steps_per_frame - s0;
    if ((uint64_t)ns > g_end - g0) ns = (uint32_t)(g_end - g0);
    if (ns > (uint32_t)kMaxSteps) ns = kMaxSteps;

    for (int i = lane; i < 48; i += 32) h[i] = 0;
    __syncwarp();
    Acc A[3], B[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      acc_clear(A[c]);
      acc_clear(B[c]);
    }
    const uint32_t gs = (uint32_t)g0;   // step j of the span is global step gs + j

    // one step's 32 pixels x 2 rows per lane (its group is the oldest in flight: wait for it, own bytes only, no
    // barrier), counted into the accumulators; cA / cB get the weight-8 carries for the fold
    auto count_step = [&](uint32_t slot, uint32_t (&cA)[3], uint32_t (&cB)[3]) {
      cp_async_wait<kStages - 1>();
      const uint4 ya = lds128(slot), c0 = lds128(slot + 1024);
      quad<0>(A, B, cA, cB, ya.x, c0.x, lut_lo);
      quad<1>(A, B, cA, cB, ya.y, c0.y, lut_lo);
      quad<2>(A, B, cA, cB, ya.z, c0.z, lut_lo);
      quad<3>(A, B, cA, cB, ya.w, c0.w, lut_lo);
      // odd luma row: rounded average of the two neighbouring chroma rows (image.cu:133-151)
      const uint4 yb = lds128(slot + 512), c1 = lds128(slot + 1536);
      quad<4>(A, B, cA, cB, yb.x, avg4(c0.x, c1.x), lut_lo);
      quad<5>(A, B, cA, cB, yb.y, avg4(c0.y, c1.y), lut_lo);
      quad<6>(A, B, cA, cB, yb.z, avg4(c0.z, c1.z), lut_lo);
      quad<7>(A, B, cA, cB, yb.w, avg4(c0.w, c1.w), lut_lo);
    };
    // step j of a block of 4.  Blocks start at span steps that are multiples of 4, so j is the fold's phase, and
    // gs + j is the step's ring stage mod kStages
    auto block_step = [&](auto phase) {
      constexpr int j = decltype(phase)::value;
      fast_prefetch(slot_of(gs + j + kStages - 1));
      uint32_t cA[3], cB[3];
      count_step(slot_of(gs + j), cA, cB);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        fold_step<j>(A[c], cA[c]);
        fold_step<j>(B[c], cB[c]);
      }
    };

    uint32_t step = 0;
    while (step < ns) {
      if (ns - step >= 4 && pf_fast >= 4) {   // step is a multiple of 4 here
        uint32_t yp;
        locate(yp);
        do {
          block_step(Phase<0>{});
          block_step(Phase<1>{});
          block_step(Phase<2>{});
          block_step(Phase<3>{});
          step += 4;
          pf_s += 4;
          pf_left -= 4;
          pf_fast -= 4;
        } while (ns - step >= 4 && pf_fast >= 4);
      } else {                                // single steps up to the next multiple of 4 or the span's end
        do {
          prefetch(slot_of(gs + step + kStages - 1));
          uint32_t cA[3], cB[3];
          count_step(slot_of(gs + step), cA, cB);
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            fold_step(A[c], cA[c], (int)step);
            fold_step(B[c], cB[c], (int)step);
          }
          ++step;
        } while (step < ns && (step & 3));
      }
    }

    // ---- flush the span
    const uint32_t values = ns * 32u * 32u;  // pixels (per channel) this warp fed, padding included
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      finish_span(A[c], (int)ns);
      finish_span(B[c], (int)ns);
      uint32_t ca = lane_count(A[c], lane);  // lanes 0..7: bins 0..7 (+ n15 each)
      uint32_t cb = lane_count(B[c], lane);  // lanes 0..6: bins 8..14
      uint32_t sum = (lane < 8) ? ca + cb : 0u;
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      sum += __shfl_xor_sync(0xffffffffu, sum, 4);
      const uint32_t n15 = (sum - values) / 7u;
      if (lane < 8) {
        ca -= n15;
        if (lane == 7) cb = n15;
        if (ca) atomicAdd(&h[c * 16 + lane], (int)ca);
        if (cb) atomicAdd(&h[c * 16 + 8 + lane], (int)cb);
      }
    }
    // padding units (the lanes past the frame's last unit in its last step) were fed as all-zero bytes: remove
    // what 32 such pixels each contributed
    const uint32_t pad_total = (s0 + ns == prm.steps_per_frame) ? prm.steps_per_frame * 32u - prm.units_per_frame : 0u;
    __syncwarp();
    if (pad_total && lane == 0) {
      const Rgb8 z = yuv_to_rgb(0, 0, 0);
      atomicSub(&h[0 * 16 + (z.r >> 4)], (int)(pad_total * 32u));
      atomicSub(&h[1 * 16 + (z.g >> 4)], (int)(pad_total * 32u));
      atomicSub(&h[2 * 16 + (z.b >> 4)], (int)(pad_total * 32u));
    }
    __syncwarp();
    for (int i = lane; i < 48; i += 32)
      if (h[i]) atomicAdd(&out[(size_t)frame * 48 + i], h[i]);
    __syncwarp();

    g0 += ns;
  }
  cp_async_wait<0>();
}

// Whether surfaces [i0, i0 + cnt) of `lp` / `cp` can take nv12_stream_kernel.
inline bool eligible(const uint8_t* const* lp, const uint8_t* const* cp, int i0, int cnt, size_t pitch, int width,
                     int height) {
  if ((width & 15) || (pitch & 15) || (height & 1)) return false;
  if ((size_t)width * height < 64 * 1024 || pitch > kMaxPitch) return false;
  return aligned(16, i0, cnt, lp, cp);
}

// One launch over the `n` surfaces of `luma` / `chroma`.  `out` must already be zeroed.
inline int launch(const PtrBatch& luma, const PtrBatch& chroma, int n, size_t pitch, int width, int height,
                  int32_t* out, cudaStream_t st) {
  const int e = raise_smem_limit((const void*)nv12_stream_kernel, kSmemBytes);
  if (e) return e;
  Params p;
  p.luma = luma;
  p.chroma = chroma;
  p.pitch = pitch;
  p.width = width;
  p.height = height;
  p.units_per_row = (uint32_t)(width / 16);
  p.upr_recip = (1ull << 32) / p.units_per_row + 1u;
  p.units_per_frame = p.units_per_row * (uint32_t)(height / 2);
  p.steps_per_frame = (p.units_per_frame + 31) / 32;
  p.total_steps = (uint64_t)n * p.steps_per_frame;
  const uint32_t wrap_l = (uint32_t)(2 * pitch) - (uint32_t)width, wrap_c = (uint32_t)pitch - (uint32_t)width;
  const uint32_t q = 32u / p.units_per_row;
  p.xs_step = 32u % p.units_per_row;
  p.inc_l = 512u + q * wrap_l;
  p.inc_l_wrap = p.inc_l + wrap_l;
  p.inc_c = 512u + q * wrap_c;
  p.inc_c_wrap = p.inc_c + wrap_c;
  p.fast_steps = (uint32_t)((uint64_t)(height / 2 - 1) * p.units_per_row / 32);
  uint64_t ctas = (p.total_steps + kWarps * 8 - 1) / (kWarps * 8);
  if (ctas > (uint64_t)sm_count()) ctas = sm_count();
  if (ctas < 1) ctas = 1;
  return launch_kernel("nv12_stream_kernel", st,
                       [&] { nv12_stream_kernel<<<(unsigned)ctas, kThreads, kSmemBytes, st>>>(p, out); });
}

}  // namespace nvs
}  // namespace scn
