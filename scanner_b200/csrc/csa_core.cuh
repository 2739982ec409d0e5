// csa_core.cuh -- bit-sliced counting primitives shared by the histogram kernels (sm_90a).
//   * PRMT as an 8-entry byte LUT: four 4-bit bins (the nibbles of a 16-bit selector) -> four
//     one-hot bytes.  Word A carries bins 0..7 (bin 15 shows up as 0xFF through PRMT's
//     sign-replicate mode), word B (selector ^ 0x8888) bins 8..14; bin 15 is recovered from the
//     known total:  n15 = (sum(A) + sum(B) - N) / 7.
//   * Harley-Seal carry-save adders sum one-hot words into bit planes: plane p holds bit p of 32
//     independent counters (one per bit position), 2 LOP3 per CSA.
//   * 8 words per accumulator per step give a weight-8 carry that is folded into the high planes
//     with two more pending levels, so the amortised cost above plane 2 is < 1 LOP3 per word.
#pragma once
#include "scn_common.cuh"

namespace scn {
namespace csa {

constexpr uint32_t kLutLo = 0x08040201u;   // one-hot bytes for index 0..3
constexpr uint32_t kLutHiA = 0x80402010u;  // index 4..7 (A: bin 7 -> 0x80; bin 15 reads it in sign mode -> 0xFF)
constexpr uint32_t kLutHiB = 0x00402010u;  // B: index 7 (bin 15) -> 0

__device__ __forceinline__ void csa3(uint32_t& h, uint32_t& l, uint32_t a, uint32_t b, uint32_t c) {
  const uint32_t u = a ^ b;
  h = (a & b) | (u & c);
  l = u ^ c;
}

// planes 0..2 + HI high planes (3 .. 2+HI); counters hold up to 2^(3+HI) - 1
template <int HI>
struct Acc8 {
  uint32_t p0, p1, p2;
  uint32_t t0, t1, t2;   // tree temporaries, dead between steps
  uint32_t hi[HI];
  uint32_t pend3, pend4;
};

template <int HI>
__device__ __forceinline__ void acc_clear(Acc8<HI>& a) {
  a.p0 = a.p1 = a.p2 = a.t0 = a.t1 = a.t2 = 0;
#pragma unroll
  for (int i = 0; i < HI; ++i) a.hi[i] = 0;
  a.pend3 = a.pend4 = 0;
}

template <int K, int HI>  // K-th (0..7) word of a step; K == 7 yields the weight-8 carry
__device__ __forceinline__ void push8(Acc8<HI>& a, uint32_t x, uint32_t& c8) {
  if constexpr ((K & 1) == 0) {
    a.t0 = x;
  } else {
    uint32_t tw;
    csa3(tw, a.p0, a.p0, a.t0, x);
    if constexpr (((K >> 1) & 1) == 0) {
      a.t1 = tw;
    } else {
      uint32_t fo;
      csa3(fo, a.p1, a.p1, a.t1, tw);
      if constexpr (((K >> 2) & 1) == 0) {
        a.t2 = fo;
      } else {
        csa3(c8, a.p2, a.p2, a.t2, fo);
      }
    }
  }
}

// planes 0..3 + HI high planes (4 .. 3+HI): 16 words per accumulator per step
template <int HI>
struct Acc16 {
  uint32_t p0, p1, p2, p3;
  uint32_t t0, t1, t2, t3;   // tree temporaries, dead between steps
  uint32_t hi[HI];
  uint32_t pend3, pend4;     // pending weight-16 / weight-32 carries (names shared with Acc8's code)
};

template <int HI>
__device__ __forceinline__ void acc_clear(Acc16<HI>& a) {
  a.p0 = a.p1 = a.p2 = a.p3 = a.t0 = a.t1 = a.t2 = a.t3 = 0;
#pragma unroll
  for (int i = 0; i < HI; ++i) a.hi[i] = 0;
  a.pend3 = a.pend4 = 0;
}

template <int K, int HI>  // K-th (0..15) word of a step; K == 15 yields the weight-16 carry
__device__ __forceinline__ void push16(Acc16<HI>& a, uint32_t x, uint32_t& c16) {
  if constexpr ((K & 1) == 0) {
    a.t0 = x;
  } else {
    uint32_t tw;
    csa3(tw, a.p0, a.p0, a.t0, x);
    if constexpr (((K >> 1) & 1) == 0) {
      a.t1 = tw;
    } else {
      uint32_t fo;
      csa3(fo, a.p1, a.p1, a.t1, tw);
      if constexpr (((K >> 2) & 1) == 0) {
        a.t2 = fo;
      } else {
        uint32_t ei;
        csa3(ei, a.p2, a.p2, a.t2, fo);
        if constexpr (((K >> 3) & 1) == 0) {
          a.t3 = ei;
        } else {
          csa3(c16, a.p3, a.p3, a.t3, ei);
        }
      }
    }
  }
}

template <int HI>
__device__ __forceinline__ void planes_of(const Acc16<HI>& a, uint32_t (&pl)[4 + HI + 5]) {
  pl[0] = a.p0;
  pl[1] = a.p1;
  pl[2] = a.p2;
  pl[3] = a.p3;
#pragma unroll
  for (int q = 0; q < HI; ++q) pl[4 + q] = a.hi[q];
#pragma unroll
  for (int q = 4 + HI; q < 4 + HI + 5; ++q) pl[q] = 0;
}

template <int FROM, int HI>
__device__ __forceinline__ void ripple(Acc16<HI>& a, uint32_t c) {
#pragma unroll
  for (int q = FROM; q < HI; ++q) {
    const uint32_t t = a.hi[q] & c;
    a.hi[q] ^= c;
    c = t;
  }
}

template <int HI>
__device__ __forceinline__ void fold_step(Acc16<HI>& a, uint32_t c16, int step) {
  if (step & 1) {
    uint32_t c32;
    csa3(c32, a.hi[0], a.hi[0], a.pend3, c16);
    if (step & 2) {
      uint32_t c64;
      csa3(c64, a.hi[1], a.hi[1], a.pend4, c32);
      ripple<2>(a, c64);
    } else {
      a.pend4 = c32;
    }
  } else {
    a.pend3 = c16;
  }
}

template <int HI>
__device__ __forceinline__ void finish_span(Acc16<HI>& a, int nsteps) {
  if (nsteps & 2) ripple<1>(a, a.pend4);
  if (nsteps & 1) ripple<0>(a, a.pend3);
}

template <int FROM, int HI>
__device__ __forceinline__ void ripple(Acc8<HI>& a, uint32_t c) {
#pragma unroll
  for (int q = FROM; q < HI; ++q) {
    const uint32_t t = a.hi[q] & c;
    a.hi[q] ^= c;
    c = t;
  }
}

template <int HI>
__device__ __forceinline__ void fold_step(Acc8<HI>& a, uint32_t c8, int step) {
  if (step & 1) {
    uint32_t c16;
    csa3(c16, a.hi[0], a.hi[0], a.pend3, c8);
    if (step & 2) {
      uint32_t c32;
      csa3(c32, a.hi[1], a.hi[1], a.pend4, c16);
      ripple<2>(a, c32);
    } else {
      a.pend4 = c16;
    }
  } else {
    a.pend3 = c8;
  }
}

template <int HI>
__device__ __forceinline__ void finish_span(Acc8<HI>& a, int nsteps) {
  if (nsteps & 2) ripple<1>(a, a.pend4);
  if (nsteps & 1) ripple<0>(a, a.pend3);
}

// cross-lane sum of a bit-sliced counter set of P planes: afterwards every lane holds the warp
// total in pl[0 .. P+4]
template <int P>
__device__ __forceinline__ void warp_sum(uint32_t (&pl)[P + 5]) {
#pragma unroll
  for (int d = 0; d < 5; ++d) {
    uint32_t carry = 0;
#pragma unroll
    for (int p = 0; p < P + 5; ++p) {
      if (p < P + d) {
        const uint32_t o = __shfl_xor_sync(0xffffffffu, pl[p], 1 << d);
        const uint32_t u = pl[p] ^ o;
        const uint32_t nc = (pl[p] & o) | (u & carry);
        pl[p] = u ^ carry;
        carry = nc;
      } else if (p == P + d) {
        pl[p] = carry;
      }
    }
  }
}

template <int P>
__device__ __forceinline__ uint32_t extract_lane(const uint32_t (&pl)[P + 5], int lane) {
  uint32_t v = 0;
#pragma unroll
  for (int p = 0; p < P + 5; ++p) v |= ((pl[p] >> lane) & 1u) << p;
  return v;
}

template <int HI>
__device__ __forceinline__ void planes_of(const Acc8<HI>& a, uint32_t (&pl)[3 + HI + 5]) {
  pl[0] = a.p0;
  pl[1] = a.p1;
  pl[2] = a.p2;
#pragma unroll
  for (int q = 0; q < HI; ++q) pl[3 + q] = a.hi[q];
#pragma unroll
  for (int q = 3 + HI; q < 3 + HI + 5; ++q) pl[q] = 0;
}

// 16-bit selector halves of z (8 nibbles = 8 bins) -> one-hot words for bins 0-7 (A) and 8-14 (B)
__device__ __forceinline__ void decode8(uint32_t z, uint32_t& a_lo, uint32_t& a_hi, uint32_t& b_lo, uint32_t& b_hi) {
  const uint32_t zx = z ^ 0x88888888u;
  a_lo = prmt(kLutLo, kLutHiA, z);
  a_hi = prmt(kLutLo, kLutHiA, z >> 16);
  b_lo = prmt(kLutLo, kLutHiB, zx);
  b_hi = prmt(kLutLo, kLutHiB, zx >> 16);
}

}  // namespace csa
}  // namespace scn
