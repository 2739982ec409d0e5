// bitstream.cuh -- what the entropy coders (jpeg.cu, h264_enc.cu) share: the bit writer and block scan of their
// passes, their device scratch, and the output stage that turns each frame's bit stream into the caller's bytes.
//
// The output stage (run_output_stage), after an encoder's measure passes have counted each frame's bits:
//   the streams are laid out at 16-byte multiples, zeroed and emitted by the encoder;
//   escape_count_kernel   escape bytes per 4 KiB chunk of each frame's stream
//   escape_copy_kernel    copies each chunk with its escapes behind the frame's prefix; the suffix follows the last
// The host reads back each frame's bit count (to size the streams) and its escape count (to size the output): two
// small copies, each behind a stream synchronisation.  An encoder gives the stage an escape rule, a type with
//   count(p, at, v, valid)     the escape bytes among the `valid` (1-16) bytes v at offset `at` of the stream p
//   copy(p, at, v, valid, o)   writes those bytes with their escapes from o on and returns the end
//   count_name, copy_name      the two launches' names (for the launch counter and scn_prof_*)
// and the bytes around each stream: two prefixes, one chosen per frame, and a suffix.  Or, instead of the two
// prefixes, one prefix per frame that the measure passes leave in device memory (FramePrefixes); the host reads their
// lengths back with the bit counts.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <vector>

#include "scn_common.cuh"

namespace scn {

// Appends bits MSB first to a frame's bit stream of big-endian 32-bit words.  The first and the last word a
// writer touches may be shared with the neighbouring writers (MCUs, macroblocks) and are ORed in; the words between
// are its own.
struct BitWriter {
  uint32_t* words;
  uint64_t word;  // index of the word being filled
  uint64_t acc;   // the low n bits are pending
  int n;
  bool first;
  __device__ BitWriter(uint32_t* w, uint64_t bit) : words(w), word(bit >> 5), acc(0), n((int)(bit & 31)), first(true) {}
  __device__ __forceinline__ void put(uint32_t bits, int len) {  // len <= 27
    acc = (acc << len) | bits;
    n += len;
    if (n >= 32) {
      n -= 32;
      const uint32_t v = __byte_perm((uint32_t)(acc >> n), 0, 0x0123);
      if (first) atomicOr(words + word, v);
      else words[word] = v;
      first = false;
      ++word;
    }
  }
  __device__ __forceinline__ void finish() {
    if (n) atomicOr(words + word, __byte_perm((uint32_t)(acc << (32 - n)), 0, 0x0123));
  }
};

// block-wide exclusive scan of one value per thread (blockDim.x a multiple of 32, at most 1024); returns the
// exclusive prefix, *total the block's sum.  Every thread of the block calls it.
template <class T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* total) {
  __shared__ T warp_sums[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xFFFFFFFFu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    T s = lane < nw ? warp_sums[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T y = __shfl_up_sync(0xFFFFFFFFu, s, o);
      if (lane >= o) s += y;
    }
    warp_sums[lane] = s;  // inclusive
  }
  __syncthreads();
  const T before = wid ? warp_sums[wid - 1] : 0;
  *total = warp_sums[nw - 1];
  __syncthreads();  // warp_sums is reused by the next call
  return before + x - v;
}

// ---- the encoders' device scratch: a stream-ordered pool per device, kept by the library ----
inline cudaMemPool_t scratch_pool() {
  static std::mutex mu;
  static std::map<int, cudaMemPool_t> pools;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  auto it = pools.find(dev);
  if (it != pools.end()) return it->second;
  cudaMemPoolProps props = {};
  props.allocType = cudaMemAllocationTypePinned;
  props.location.type = cudaMemLocationTypeDevice;
  props.location.id = dev;
  cudaMemPool_t pool = nullptr;
  if (cudaMemPoolCreate(&pool, &props) != cudaSuccess) return nullptr;
  uint64_t keep = ~0ull;  // keep freed scratch for the next call instead of returning it at every synchronisation
  cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  pools[dev] = pool;
  return pool;
}

struct Scratch {
  cudaStream_t st;
  std::vector<void*> held;
  ~Scratch() {
    for (void* p : held) cudaFreeAsync(p, st);
  }
  template <class T>
  T* get(size_t count, cudaMemPool_t pool) {
    void* p = nullptr;
    if (cudaMallocFromPoolAsync(&p, count * sizeof(T) + 16, pool, st) != cudaSuccess) return nullptr;
    held.push_back(p);
    return static_cast<T*>(p);
  }
};

// ---- the output stage ----
constexpr int kLane = 16;                       // bytes of stream per thread of the escape passes (one 16-byte load)
constexpr int kChunk = 4096;                    // bytes of stream per CTA of the escape passes
constexpr int kChunkThreads = kChunk / kLane;
constexpr int kMaxPrefix = 640;                 // bytes; JPEG's header is the longest prefix
constexpr int kMaxSuffix = 2;

struct StreamSlots {
  uint64_t stream_off[SCN_MAX_PTRS];  // byte offset of each frame's bit stream
  uint64_t bytes[SCN_MAX_PTRS];       // bytes of each frame's bit stream (before escapes)
  uint64_t chunk_off[SCN_MAX_PTRS];   // index of each frame's first chunk count
  uint64_t out_off[SCN_MAX_PTRS];     // byte offset of each frame's output
  uint8_t prefix[SCN_MAX_PTRS];       // which of the two prefixes each frame gets
  uint16_t prefix_len[SCN_MAX_PTRS];  // with per-frame prefixes: each frame's prefix length
};

// Per-frame prefixes in device memory: frame i's at bytes + i * kMaxPrefix, len[i] bytes long (at most kMaxPrefix).
struct FramePrefixes {
  const uint8_t* bytes;
  const uint32_t* len;
};

// The bytes around each frame's stream in the output.
struct Affixes {
  uint8_t prefix[2][kMaxPrefix];
  uint8_t suffix[kMaxSuffix];
  int prefix_len[2];
  int suffix_len;
};

// Fills *a; false (and *a untouched) when a prefix or the suffix does not fit.
inline bool make_affixes(Affixes* a, const std::vector<uint8_t>& prefix0, const std::vector<uint8_t>& prefix1,
                         const std::vector<uint8_t>& suffix) {
  if (prefix0.size() > kMaxPrefix || prefix1.size() > kMaxPrefix || suffix.size() > kMaxSuffix) return false;
  *a = {};
  std::copy(prefix0.begin(), prefix0.end(), a->prefix[0]);
  std::copy(prefix1.begin(), prefix1.end(), a->prefix[1]);
  std::copy(suffix.begin(), suffix.end(), a->suffix);
  a->prefix_len[0] = (int)prefix0.size();
  a->prefix_len[1] = (int)prefix1.size();
  a->suffix_len = (int)suffix.size();
  return true;
}

template <class Rule>
__global__ void __launch_bounds__(kChunkThreads)
escape_count_kernel(int i0, const __grid_constant__ StreamSlots s, const uint8_t* streams, uint32_t* chunk_esc,
                    unsigned long long* esc) {
  const int j = blockIdx.y;
  const uint64_t bytes = s.bytes[j];
  const uint64_t at = (uint64_t)blockIdx.x * kChunk;
  if (at >= bytes) return;
  const uint8_t* p = streams + s.stream_off[j];
  const uint64_t i = at + threadIdx.x * kLane;
  int c = 0;
  if (i < bytes)
    c = Rule::count(p, i, *reinterpret_cast<const uint4*>(p + i), (int)min(bytes - i, (uint64_t)kLane));
  unsigned long long total;
  block_exclusive_scan<unsigned long long>((unsigned long long)c, &total);
  if (threadIdx.x == 0) {
    chunk_esc[s.chunk_off[j] + blockIdx.x] = (uint32_t)total;
    atomicAdd(esc + i0 + j, total);
  }
}

// PerFrame: each frame's prefix is at frame_prefix + j * kMaxPrefix (FramePrefixes), else one of ax's two
template <class Rule, bool PerFrame>
__global__ void __launch_bounds__(kChunkThreads)
escape_copy_kernel(const __grid_constant__ StreamSlots s, const __grid_constant__ Affixes ax, const uint8_t* streams,
                   const uint32_t* chunk_esc, uint8_t* out, const uint8_t* frame_prefix) {
  const int j = blockIdx.y;
  const uint64_t bytes = s.bytes[j];
  const uint64_t at = (uint64_t)blockIdx.x * kChunk;
  if (at >= bytes) return;
  const int pre = s.prefix[j];
  const int pre_len = PerFrame ? s.prefix_len[j] : ax.prefix_len[pre];
  uint8_t* dst = out + s.out_off[j];
  if (blockIdx.x == 0) {
    if constexpr (PerFrame) {
      const uint8_t* pre_bytes = frame_prefix + (size_t)j * kMaxPrefix;
      for (int k = threadIdx.x; k < pre_len; k += blockDim.x) dst[k] = pre_bytes[k];
    } else {
      for (int k = threadIdx.x; k < pre_len; k += blockDim.x) dst[k] = ax.prefix[pre][k];
    }
  }
  // escapes of the chunks before this one
  unsigned long long before = 0;
  for (uint32_t c = threadIdx.x; c < blockIdx.x; c += blockDim.x) before += chunk_esc[s.chunk_off[j] + c];
  unsigned long long chunk_before;
  block_exclusive_scan<unsigned long long>(before, &chunk_before);
  const uint8_t* p = streams + s.stream_off[j];
  const uint64_t i = at + threadIdx.x * kLane;
  uint4 v = make_uint4(0, 0, 0, 0);
  const int valid = i < bytes ? (int)min(bytes - i, (uint64_t)kLane) : 0;
  if (valid) v = *reinterpret_cast<const uint4*>(p + i);
  unsigned long long total;
  const unsigned long long mine =
      block_exclusive_scan<unsigned long long>((unsigned long long)(valid ? Rule::count(p, i, v, valid) : 0), &total);
  if (!valid) return;
  uint8_t* o = Rule::copy(p, i, v, valid, dst + pre_len + i + chunk_before + mine);
  if (i + valid == bytes)
    for (int k = 0; k < ax.suffix_len; ++k) o[k] = ax.suffix[k];
}

// Runs the output stage of one call of n frames.  measure() enqueues the passes that leave each frame's bit count
// in bits[0, n) (device); emit(i0, cnt, streams, stream_off) enqueues the pass that writes frames [i0, i0 + cnt)
// into the zeroed `streams`, frame i0 + j at byte stream_off[j].  prefix[i] picks frame i's prefix in ax; a null
// prefix gives every frame prefix 0; frame_prefixes, when given, replace both (measure() leaves them).  The outputs
// go back to back into one buffer from alloc_out, their sizes to host_sizes.  Returns the first nonzero status.
template <class Rule, class Measure, class Emit>
int run_output_stage(int n, cudaStream_t st, cudaMemPool_t pool, Scratch& s, const uint64_t* bits,
                     const uint8_t* prefix, const Affixes& ax, Measure&& measure, Emit&& emit, scn_alloc_fn alloc_out,
                     void* alloc_ctx, size_t* host_sizes, FramePrefixes frame_prefixes = {nullptr, nullptr}) {
  unsigned long long* escs = s.get<unsigned long long>((size_t)n, pool);
  if (!escs) return (int)cudaErrorMemoryAllocation;
  int rc = measure();
  if (rc) return rc;
  std::vector<uint64_t> host_bits((size_t)n);
  std::vector<uint32_t> pre_len((size_t)n);
  if ((rc = (int)cudaMemcpyAsync(host_bits.data(), bits, (size_t)n * 8, cudaMemcpyDeviceToHost, st))) return rc;
  if (frame_prefixes.bytes &&
      (rc = (int)cudaMemcpyAsync(pre_len.data(), frame_prefixes.len, (size_t)n * 4, cudaMemcpyDeviceToHost, st)))
    return rc;
  if ((rc = (int)cudaStreamSynchronize(st))) return rc;
  for (int i = 0; i < n; ++i) {
    if (!frame_prefixes.bytes) pre_len[i] = (uint32_t)ax.prefix_len[prefix ? prefix[i] : 0];
    if (pre_len[i] > kMaxPrefix) return SCN_E_UNSUPPORTED;
  }

  // the streams, 16-byte aligned, and their chunks
  std::vector<uint64_t> bytes((size_t)n), stream_off((size_t)n), chunk_off((size_t)n), out_off((size_t)n);
  uint64_t stream_total = 0, chunks = 0, max_chunks = 0;
  for (int i = 0; i < n; ++i) {
    bytes[i] = (host_bits[i] + 7) / 8;
    stream_off[i] = stream_total;
    stream_total += (bytes[i] + kLane - 1) / kLane * kLane;
    chunk_off[i] = chunks;
    const uint64_t c = (bytes[i] + kChunk - 1) / kChunk;
    chunks += c;
    max_chunks = c > max_chunks ? c : max_chunks;
  }
  uint8_t* streams = s.get<uint8_t>(stream_total, pool);
  uint32_t* chunk_esc = s.get<uint32_t>(chunks, pool);
  if (!streams || !chunk_esc) return (int)cudaErrorMemoryAllocation;
  if ((rc = (int)cudaMemsetAsync(streams, 0, stream_total, st))) return rc;
  if ((rc = (int)cudaMemsetAsync(escs, 0, (size_t)n * 8, st))) return rc;
  auto slots = [&](int i0, int cnt) {  // out_off is all zero until the escapes are known
    StreamSlots sl = {};
    for (int j = 0; j < cnt; ++j) {
      sl.stream_off[j] = stream_off[i0 + j];
      sl.bytes[j] = bytes[i0 + j];
      sl.chunk_off[j] = chunk_off[i0 + j];
      sl.out_off[j] = out_off[i0 + j];
      sl.prefix[j] = prefix ? prefix[i0 + j] : 0;
      sl.prefix_len[j] = (uint16_t)pre_len[i0 + j];
    }
    return sl;
  };

  // emit each launch's streams and count their escapes
  rc = for_each_chunk(n, [&](int i0, int cnt) {
    const int e = emit(i0, cnt, streams, stream_off.data() + i0);
    if (e) return e;
    const StreamSlots sl = slots(i0, cnt);
    return launch_kernel(Rule::count_name, st, [&] {
      escape_count_kernel<Rule>
          <<<dim3((unsigned)max_chunks, (unsigned)cnt), kChunkThreads, 0, st>>>(i0, sl, streams, chunk_esc, escs);
    });
  });
  if (rc) return rc;
  std::vector<uint64_t> esc((size_t)n);
  if ((rc = (int)cudaMemcpyAsync(esc.data(), escs, (size_t)n * 8, cudaMemcpyDeviceToHost, st))) return rc;
  if ((rc = (int)cudaStreamSynchronize(st))) return rc;

  // the outputs, back to back in the caller's buffer
  size_t out_total = 0;
  for (int i = 0; i < n; ++i) {
    host_sizes[i] = (size_t)pre_len[i] + bytes[i] + esc[i] + ax.suffix_len;
    out_off[i] = out_total;
    out_total += host_sizes[i];
  }
  uint8_t* out = static_cast<uint8_t*>(alloc_out(alloc_ctx, out_total));
  if (!out) return SCN_E_ALLOC;
  return for_each_chunk(n, [&](int i0, int cnt) {
    const StreamSlots sl = slots(i0, cnt);
    const uint8_t* fp = frame_prefixes.bytes ? frame_prefixes.bytes + (size_t)i0 * kMaxPrefix : nullptr;
    const dim3 grid((unsigned)max_chunks, (unsigned)cnt);
    return launch_kernel(Rule::copy_name, st, [&] {
      if (fp)
        escape_copy_kernel<Rule, true><<<grid, kChunkThreads, 0, st>>>(sl, ax, streams, chunk_esc, out, fp);
      else
        escape_copy_kernel<Rule, false><<<grid, kChunkThreads, 0, st>>>(sl, ax, streams, chunk_esc, out, fp);
    });
  });
}

}  // namespace scn
