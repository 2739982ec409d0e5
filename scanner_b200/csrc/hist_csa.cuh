// hist_csa.cuh -- bit-sliced streaming histogram for large u8 HWC 3-channel frames (sm_90a).
//
// Why: a 16-bin histogram at HBM speed needs ~25 bytes/clk/SM; shared-memory atomics manage ~1 and
// per-byte register counters ~8 (integer pipe: 64 lanes/clk/SM).  Here (csa_core.cuh) PRMT turns
// high nibbles into one-hot bytes and carry-save adders count them 32 counters per LOP3.
//
// v3 layout: a warp streams blocks of 12 x 512 B (lane l owns 16 B of every 512 B round).  Words
// three rounds apart start at the same byte offset mod 3, i.e. have the same byte->channel phase,
// so they are PAIRED: the high nibbles of x go to the even nibbles and those of y stay in the odd
// nibbles of one selector word  z = ((x >> 4) & 0x0F0F0F0F) | (y & 0xF0F0F0F0)  (SHF + LOP3), and
// every PRMT lookup then decodes four useful bins instead of two (v1 decoded each word alone and
// needed a third PRMT to compact): 9 integer ops per 8 bytes.
// The low selector half of a pair of phase p covers channels (p, p, p+1, p+1) in its four byte
// slots, the high half (p+2, p+2, p, p) -- which is exactly the low-half layout of phase p+2.  So
// the high-half words of phase set s are added into the accumulator of set (s+2)%3 and six
// accumulators suffice (3 layouts x bins 0-7 / 8-14), each fed 16 words per block through a
// 4-level carry-save tree.  Two register buffers hold alternate blocks and prefetch each other
// (loop unrolled by two: no register moves, no conditional loads).
// Main loop ~2.3 integer ops per byte.  Bit-exact.
#pragma once
#include "csa_core.cuh"
#include "scn_common.cuh"

namespace scn {
namespace csa {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kHi = 6;                 // planes 4..9 -> counters up to 1023
constexpr int kPlanes = 4 + kHi;
constexpr int kWarpBlock = 6144;       // bytes per warp per block: 12 rounds x 32 lanes x 16 B
constexpr int kMaxBlocks = 63;         // 63 * 16 words per accumulator <= 1023

using Acc = Acc16<kHi>;

// pair sequence index q = half*12 + r*4 + j (half block, round within the half, word of the uint4).
// Its phase set; the low selector half is counted by accumulator set(q), the high half by
// (set(q)+2)%3.  rank_* = how many words that accumulator has already received in the block.
__host__ __device__ constexpr int pair_set(int q) { return (2 * ((q % 12) / 4) + (q % 4)) % 3; }
__host__ __device__ constexpr int pushes_before(int q, int acc) {
  int c = 0;
  for (int i = 0; i < q; ++i) {
    if (pair_set(i) == acc) ++c;
    if ((pair_set(i) + 2) % 3 == acc) ++c;
  }
  return c;
}

struct Sets {
  Acc a[3], b[3];  // [channel layout]: bins 0-7(+15) / bins 8-14
};
struct Carries {
  uint32_t a[3], b[3];
};

template <int Q>
__device__ __forceinline__ void eat_pair(Sets& S, Carries& C, uint32_t x, uint32_t y) {
  constexpr int lo = pair_set(Q), hi = (pair_set(Q) + 2) % 3;
  constexpr int klo = pushes_before(Q, lo), khi = pushes_before(Q, hi);
  const uint32_t z = ((x >> 4) & 0x0F0F0F0Fu) | (y & 0xF0F0F0F0u);
  uint32_t a_lo, a_hi, b_lo, b_hi;
  decode8(z, a_lo, a_hi, b_lo, b_hi);
  push16<klo>(S.a[lo], a_lo, C.a[lo]);
  push16<klo>(S.b[lo], b_lo, C.b[lo]);
  push16<khi>(S.a[hi], a_hi, C.a[hi]);
  push16<khi>(S.b[hi], b_hi, C.b[hi]);
}

template <int HALF>
__device__ __forceinline__ void eat_half(Sets& S, Carries& C, const uint4* v /* 6 rounds */) {
  eat_pair<HALF * 12 + 0>(S, C, v[0].x, v[3].x);
  eat_pair<HALF * 12 + 1>(S, C, v[0].y, v[3].y);
  eat_pair<HALF * 12 + 2>(S, C, v[0].z, v[3].z);
  eat_pair<HALF * 12 + 3>(S, C, v[0].w, v[3].w);
  eat_pair<HALF * 12 + 4>(S, C, v[1].x, v[4].x);
  eat_pair<HALF * 12 + 5>(S, C, v[1].y, v[4].y);
  eat_pair<HALF * 12 + 6>(S, C, v[1].z, v[4].z);
  eat_pair<HALF * 12 + 7>(S, C, v[1].w, v[4].w);
  eat_pair<HALF * 12 + 8>(S, C, v[2].x, v[5].x);
  eat_pair<HALF * 12 + 9>(S, C, v[2].y, v[5].y);
  eat_pair<HALF * 12 + 10>(S, C, v[2].z, v[5].z);
  eat_pair<HALF * 12 + 11>(S, C, v[2].w, v[5].w);
}

__device__ __forceinline__ void eat_block(Sets& S, const uint4 (&v)[12], int blk) {
  Carries C;
  eat_half<0>(S, C, v);
  eat_half<1>(S, C, v + 6);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    fold_step(S.a[c], C.a[c], blk);
    fold_step(S.b[c], C.b[c], blk);
  }
}

__device__ __forceinline__ uint32_t sel3(int rot, uint32_t x0, uint32_t x1, uint32_t x2) {
  return rot == 0 ? x0 : (rot == 1 ? x1 : x2);
}

// Flush one span: add this warp's counts of `nblk` blocks into hist48.
// On lane l (rot = l % 3) accumulator c holds the layout of true phase (c + rot) % 3: byte slot k
// of its words belongs to channel (phase + k/2) % 3.
__device__ __forceinline__ void flush_span(Sets& S, int nblk, int lane, int* hist48) {
  const int rot = lane % 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    finish_span(S.a[c], nblk);
    finish_span(S.b[c], nblk);
  }
  const uint32_t words_per_slot = (uint32_t)nblk * 16u * 32u;  // per accumulator, whole warp
#pragma unroll
  for (int phase = 0; phase < 3; ++phase) {
    const int pick = (phase + 3 - rot) % 3;
    uint32_t pa[kPlanes + 5], pb[kPlanes + 5], x0[kPlanes + 5], x1[kPlanes + 5], x2[kPlanes + 5];
    planes_of(S.a[0], x0);
    planes_of(S.a[1], x1);
    planes_of(S.a[2], x2);
#pragma unroll
    for (int p = 0; p < kPlanes + 5; ++p) pa[p] = sel3(pick, x0[p], x1[p], x2[p]);
    planes_of(S.b[0], x0);
    planes_of(S.b[1], x1);
    planes_of(S.b[2], x2);
#pragma unroll
    for (int p = 0; p < kPlanes + 5; ++p) pb[p] = sel3(pick, x0[p], x1[p], x2[p]);
    warp_sum<kPlanes>(pa);
    warp_sum<kPlanes>(pb);
    uint32_t ca = extract_lane<kPlanes>(pa, lane);  // A counter of (slot lane/8, bit lane%8), + n15 of the slot
    uint32_t cb = extract_lane<kPlanes>(pb, lane);  // B counter: bins 8..14 (bit 7 stays 0)
    uint32_t sum = ca + cb;
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    sum += __shfl_xor_sync(0xffffffffu, sum, 4);
    const uint32_t n15 = (sum - words_per_slot) / 7u;
    ca -= n15;
    const int bit = lane & 7, slot = lane >> 3;
    if (bit == 7) cb = n15;
    const int ch = (phase + (slot >> 1)) % 3;
    if (ca) atomicAdd(&hist48[ch * 16 + bit], (int)ca);
    if (cb) atomicAdd(&hist48[ch * 16 + 8 + bit], (int)cb);
  }
}

struct Params {
  PtrBatch frames;
  int n;                      // frames in this launch
  uint32_t blocks_per_frame;  // whole warp blocks per frame
  uint32_t tail_bytes;        // bytes after the last whole block of a frame
  uint64_t total_blocks;      // n * blocks_per_frame
};

// One warp owns a contiguous range of the global warp-block index space and walks it frame by
// frame; at most kMaxBlocks blocks between flushes.
static __global__ void __launch_bounds__(kThreads, 1)
hist16_csa_kernel(const Params prm, int32_t* __restrict__ out) {
  __shared__ int sh[kWarps][48];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* h = sh[warp];
  const uint64_t gwarp = (uint64_t)blockIdx.x * kWarps + warp;
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  uint64_t g0 = prm.total_blocks * gwarp / nwarps;
  const uint64_t g1 = prm.total_blocks * (gwarp + 1) / nwarps;

  while (g0 < g1) {
    const uint32_t frame = (uint32_t)(g0 / prm.blocks_per_frame);
    const uint32_t b0 = (uint32_t)(g0 - (uint64_t)frame * prm.blocks_per_frame);
    uint32_t nb = prm.blocks_per_frame - b0;
    if ((uint64_t)nb > g1 - g0) nb = (uint32_t)(g1 - g0);
    if (nb > (uint32_t)kMaxBlocks) nb = kMaxBlocks;
    const uint8_t* __restrict__ src = prm.frames.p[frame] + (size_t)b0 * kWarpBlock + (size_t)lane * 16;

    for (int i = lane; i < 48; i += 32) h[i] = 0;
    __syncwarp();

    Sets S;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      acc_clear(S.a[c]);
      acc_clear(S.b[c]);
    }
    // two register buffers hold alternate blocks; every load is unconditional (indices clamp to
    // the last block) so no load sits in a divergent region
    auto load_block = [&](uint4 (&v)[12], uint32_t blk) {
      const uint8_t* p = src + (size_t)(blk < nb ? blk : nb - 1) * kWarpBlock;
#pragma unroll
      for (int r = 0; r < 12; ++r) v[r] = ld_stream_u4(p + r * 512);
    };
    uint4 va[12], vb[12];
    uint32_t blk = 0;
    load_block(va, 0);
    if (nb & 1) {  // odd count: peel one block so the unrolled loop below always runs pairs
      load_block(vb, 1);
      eat_block(S, va, 0);
#pragma unroll
      for (int r = 0; r < 12; ++r) va[r] = vb[r];
      blk = 1;
    }
    for (; blk < nb; blk += 2) {
      load_block(vb, blk + 1);
      eat_block(S, va, (int)blk);
      load_block(va, blk + 2);
      eat_block(S, vb, (int)blk + 1);
    }
    flush_span(S, (int)nb, lane, h);

    // the warp that finishes a frame's last block also counts the frame's tail bytes
    if (b0 + nb == prm.blocks_per_frame && prm.tail_bytes) {
      const uint8_t* t = prm.frames.p[frame] + (size_t)prm.blocks_per_frame * kWarpBlock;
      for (uint32_t o = lane; o < prm.tail_bytes; o += 32) atomicAdd(&h[(o % 3) * 16 + (t[o] >> 4)], 1);
    }
    __syncwarp();
    for (int i = lane; i < 48; i += 32)
      if (h[i]) atomicAdd(&out[(size_t)frame * 48 + i], h[i]);
    __syncwarp();
    g0 += nb;
  }
}

inline bool eligible(const uint8_t* const* ptrs, int n, size_t nbytes) {
  if (nbytes < (size_t)kWarpBlock * 8) return false;
  if (nbytes / kWarpBlock > 0xFFFFFFFFull) return false;
  for (int i = 0; i < n; ++i)
    if (reinterpret_cast<uintptr_t>(ptrs[i]) & 15) return false;
  return true;
}

// `out` must already be zeroed (launch_hist memsets it).
inline int launch(const uint8_t* const* ptrs, int n, size_t nbytes, int32_t* out, cudaStream_t st) {
  for (int i0 = 0; i0 < n; i0 += SCN_MAX_PTRS) {
    const int cnt = (n - i0 < SCN_MAX_PTRS) ? (n - i0) : SCN_MAX_PTRS;
    Params p;
    for (int i = 0; i < cnt; ++i) p.frames.p[i] = ptrs[i0 + i];
    p.n = cnt;
    p.blocks_per_frame = (uint32_t)(nbytes / kWarpBlock);
    p.tail_bytes = (uint32_t)(nbytes - (size_t)p.blocks_per_frame * kWarpBlock);
    p.total_blocks = (uint64_t)cnt * p.blocks_per_frame;
    // persistent: one CTA per SM; with little work use fewer CTAs so every warp gets >= 4 blocks
    uint64_t ctas = (p.total_blocks + kWarps * 4 - 1) / (kWarps * 4);
    if (ctas > (uint64_t)sm_count()) ctas = sm_count();
    if (ctas < 1) ctas = 1;
    {
      LaunchScope ls("hist16_csa_kernel", st);
      hist16_csa_kernel<<<(unsigned)ctas, kThreads, 0, st>>>(p, out + (size_t)i0 * 48);
    }
    int rc = launch_status();
    if (rc) return rc;
  }
  return 0;
}

}  // namespace csa
}  // namespace scn
