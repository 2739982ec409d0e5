// tvl1.cu -- TV-L1 dense optical flow on the GPU (sm_90a).  The specification is DESIGN.md's "TV-L1" section;
// oracle/tvl1.c (orc_tvl1_u8) is the same algorithm in sequential C, and every per-pixel expression here is
// written in the same order.  This file is compiled with -fmad=false (csrc/Makefile), so apart from the error sum
// that decides when a warp step stops, the kernels round exactly as the oracle does.
//
// Shape of a call (n pairs of one geometry, in chunks of up to 64):
//   once:       u8 -> float level 0 of both frames (1 launch), each coarser level from the one above (1 launch
//               per level)
//   per level:  Ix, Iy of I1, zero p (and u at the coarsest level) or upsample u from the coarser level (1-2)
//   per warp:   bicubic warp of I1, Ix, Iy -> (I1wx, I1wy, rho_c)                              (1 launch)
//               all iterations of the warp for all pairs: one cooperative kernel            (1 launch)
//               median of u1, u2                                                             (1 launch, if on)
//   at the end: (u1, u2) -> the caller's interleaved flows                                   (1 launch)
// Every launch serves all pairs of the chunk, so the launch count of a call does not grow with n.
//
// The iteration kernel keeps a pair's work on a fixed tiling: tile t of a pair is pixels [1024 t, 1024 t + 1024),
// and its error partial is summed in a fixed order whatever block runs it.  After the v/u phase a grid-wide sync,
// then the p phase, during which one block per pair sums that pair's tile partials (fixed order, double) and
// decides whether the pair runs another iteration; a second grid-wide sync publishes the decision.  No float
// atomics anywhere: a pair's flow is bit-identical run to run and alone or inside any batch.
#include <cooperative_groups.h>
#include <math.h>
#include <string.h>

#include "scn_common.cuh"

namespace cg = cooperative_groups;

namespace scn {
namespace {

constexpr int kT = 256;                 // threads per block in every kernel here
constexpr int kPxPerThread = 4;
constexpr int kTile = kT * kPxPerThread;  // pixels of one error tile
constexpr int kMaxLevels = 10;
constexpr int kMaxWarps = 20;

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Per-pair planes.  Every plane holds up to the full-resolution level; a pair's planes are pair_stride floats
// apart.  The pyramids of both frames take kMaxLevels planes each (the worst case: scale_step near 1).
enum Plane { kU1 = 0, kU2, kU1b, kU2b, kIx, kIy, kWx, kWy, kRho, kP11, kP12, kP21, kP22, kPart, kPyr0, kNumFixed = kPyr0 };

struct Layout {
  size_t ps;           // floats per plane
  size_t pair_stride;  // floats per pair
  __host__ __device__ size_t plane(int k) const { return (size_t)k * ps; }
  __host__ __device__ size_t pyr(int frame, size_t level_off) const { return (size_t)(kPyr0 + frame * kMaxLevels) * ps + level_off; }
};

Layout layout(int width, int height) {
  Layout L;
  L.ps = ((size_t)width * height + 63) & ~(size_t)63;
  L.pair_stride = (size_t)(kNumFixed + 2 * kMaxLevels) * L.ps;
  return L;
}
constexpr size_t kHeadBytes = 256 + sizeof(int) * 2 * SCN_MAX_PTRS + sizeof(int) * SCN_MAX_PTRS * kMaxLevels * kMaxWarps;

int plan_levels(int width, int height, int nscales, float scale_step, int* lw, int* lh) {
  int n = 1;
  lw[0] = width;
  lh[0] = height;
  while (n < nscales) {
    const int w = (int)floor((double)lw[n - 1] * scale_step + 0.5), h = (int)floor((double)lh[n - 1] * scale_step + 0.5);
    if (w < 16 || h < 16) break;
    lw[n] = w;
    lh[n] = h;
    ++n;
  }
  return n;
}

// ---- pyramid, gradients, upsampling ----
// blockIdx.y = pair * 2 + frame
__global__ void __launch_bounds__(kT) tvl1_gray_kernel(PtrBatch prev, PtrBatch next, int npx, float* __restrict__ ws,
                                                       size_t pair_stride, size_t off0, size_t off1) {
  const int i = blockIdx.x * kT + threadIdx.x;
  if (i >= npx) return;
  const int pair = blockIdx.y >> 1, f = blockIdx.y & 1;
  const uint8_t* src = f ? next.p[pair] : prev.p[pair];
  ws[pair * pair_stride + (f ? off1 : off0) + i] = (float)src[i];
}

struct Pair2 {
  size_t src[2], dst[2];
};
// cv2.resize(INTER_LINEAR) of float planes with an explicit dsize (orc_tvl1_resize_f32), times `mul`;
// blockIdx.y = pair * 2 + job, each job its own (src, dst) plane offset
__global__ void __launch_bounds__(kT) tvl1_resize_kernel(float* __restrict__ ws, size_t pair_stride, Pair2 jobs,
                                                         int sw, int sh, int dw, int dh, double sx, double sy,
                                                         float mul, int apply_mul) {
  const int i = blockIdx.x * kT + threadIdx.x;
  if (i >= dw * dh) return;
  const int pair = blockIdx.y >> 1, j = blockIdx.y & 1;
  const float* src = ws + pair * pair_stride + jobs.src[j];
  float* dst = ws + pair * pair_stride + jobs.dst[j];
  const int y = i / dw, x = i - y * dw;
  float fy = (float)((y + 0.5) * sy - 0.5);
  int iy = (int)floorf(fy);
  fy -= (float)iy;
  if (iy < 0) { fy = 0.f; iy = 0; }
  if (iy >= sh - 1) { fy = 0.f; iy = sh - 1; }
  const int iy1 = iy + 1 < sh ? iy + 1 : sh - 1;
  float fx = (float)((x + 0.5) * sx - 0.5);
  int ix = (int)floorf(fx);
  fx -= (float)ix;
  if (ix < 0) { fx = 0.f; ix = 0; }
  if (ix >= sw - 1) { fx = 0.f; ix = sw - 1; }
  const int ix1 = ix + 1 < sw ? ix + 1 : sw - 1;
  const float a = src[(size_t)iy * sw + ix], b = src[(size_t)iy * sw + ix1];
  const float d = src[(size_t)iy1 * sw + ix], e = src[(size_t)iy1 * sw + ix1];
  const float top = a * (1.f - fx) + b * fx, bot = d * (1.f - fx) + e * fx;
  const float v = top * (1.f - fy) + bot * fy;
  dst[(size_t)y * dw + x] = apply_mul ? v * mul : v;
}

// centred differences of I1 (one-sided at the edges); p = 0; at the coarsest level also u = 0.  blockIdx.y = pair
__global__ void __launch_bounds__(kT) tvl1_grad_kernel(float* __restrict__ ws, size_t pair_stride, Layout L,
                                                       size_t i1_off, int w, int h, int zero_u, int ucur) {
  const int i = blockIdx.x * kT + threadIdx.x;
  if (i >= w * h) return;
  float* base = ws + blockIdx.y * pair_stride;
  const float* J = base + i1_off;
  const int y = i / w, x = i - y * w;
  const float xl = J[(size_t)y * w + (x > 0 ? x - 1 : 0)], xr = J[(size_t)y * w + (x < w - 1 ? x + 1 : w - 1)];
  const float yu = J[(size_t)(y > 0 ? y - 1 : 0) * w + x], yd = J[(size_t)(y < h - 1 ? y + 1 : h - 1) * w + x];
  base[L.plane(kIx) + i] = 0.5f * (x == 0 ? J[i + 1] - J[i] : (x == w - 1 ? J[i] - J[i - 1] : xr - xl));
  base[L.plane(kIy) + i] = 0.5f * (y == 0 ? J[i + w] - J[i] : (y == h - 1 ? J[i] - J[i - w] : yd - yu));
  base[L.plane(kP11) + i] = 0.f;
  base[L.plane(kP12) + i] = 0.f;
  base[L.plane(kP21) + i] = 0.f;
  base[L.plane(kP22) + i] = 0.f;
  if (zero_u) {
    base[L.plane(ucur ? kU1b : kU1) + i] = 0.f;
    base[L.plane(ucur ? kU2b : kU2) + i] = 0.f;
  }
}

// ---- warp ----
__device__ __forceinline__ float cubic(float v0, float v1, float v2, float v3, float t) {
  return v1 + 0.5f * t * (v2 - v0 + t * (2.f * v0 - 5.f * v1 + 4.f * v2 - v3 + t * (3.f * (v1 - v2) + v3 - v0)));
}

// I1, Ix, Iy at (x + u1, y + u2) -> wx, wy, rho_c = I1w - wx u1 - wy u2 - I0.  Each of the three planes is sampled
// with the same 4 x 4 taps.  blockIdx.y = pair
__global__ void __launch_bounds__(kT) tvl1_warp_kernel(float* __restrict__ ws, size_t pair_stride, Layout L,
                                                       size_t i0_off, size_t i1_off, int w, int h, int ucur) {
  const int i = blockIdx.x * kT + threadIdx.x;
  if (i >= w * h) return;
  float* base = ws + blockIdx.y * pair_stride;
  const float* J[3] = {base + i1_off, base + L.plane(kIx), base + L.plane(kIy)};
  const float u1 = base[L.plane(ucur ? kU1b : kU1) + i], u2 = base[L.plane(ucur ? kU2b : kU2) + i];
  const int y = i / w, x = i - y * w;
  float px = (float)x + u1, py = (float)y + u2;
  // clamp to [-2, w + 1] x [-2, h + 1]: moves no finite sample (all taps already clamp there), keeps NaN in range
  if (!(px >= -2.f)) px = -2.f;
  if (!(px <= (float)(w + 1))) px = (float)(w + 1);
  if (!(py >= -2.f)) py = -2.f;
  if (!(py <= (float)(h + 1))) py = (float)(h + 1);
  const int ix = (int)floorf(px), iy = (int)floorf(py);
  const float tx = px - (float)ix, ty = py - (float)iy;
  int cx[4], ry[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    cx[k] = clampi(ix - 1 + k, 0, w - 1);
    ry[k] = clampi(iy - 1 + k, 0, h - 1) * w;
  }
  float r[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    float col[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float* row = J[q] + ry[j];
      col[j] = cubic(row[cx[0]], row[cx[1]], row[cx[2]], row[cx[3]], tx);
    }
    r[q] = cubic(col[0], col[1], col[2], col[3], ty);
  }
  base[L.plane(kWx) + i] = r[1];
  base[L.plane(kWy) + i] = r[2];
  base[L.plane(kRho) + i] = r[0] - r[1] * u1 - r[2] * u2 - base[i0_off + i];
}

// ---- the iterations of one warp step, all pairs, one cooperative launch ----
struct IterArgs {
  float* ws;
  size_t pair_stride;
  Layout L;
  int ucur, w, h, npx, tiles, npairs;
  float l_t, theta, taut;
  double eps2;
  int iterations;
  int* flags;   // [2][SCN_MAX_PTRS]: pair still iterating, double-buffered by iteration parity
  int* counts;  // [pair][nscales][warps]
  int count_idx, count_stride;
};

// fixed-order block sum (shuffle tree, then the 8 warp sums in order); every thread of the block calls it
template <class T>
__device__ __forceinline__ T block_sum(T v, T* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  T s = 0;
  if (threadIdx.x == 0)
    for (int k = 0; k < kT / 32; ++k) s += sh[k];
  __syncthreads();
  return s;  // valid in thread 0
}

__global__ void __launch_bounds__(kT) tvl1_iterate_kernel(IterArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ float shf[kT / 32];
  __shared__ double shd[kT / 32];
  const Layout& L = a.L;
  const int w = a.w, h = a.h, npx = a.npx;
  const int work = a.npairs * a.tiles;
  const size_t o_u1 = L.plane(a.ucur ? kU1b : kU1), o_u2 = L.plane(a.ucur ? kU2b : kU2);
  for (int k = 0; k < a.iterations; ++k) {
    const int* act = a.flags + (k & 1) * SCN_MAX_PTRS;
    if (k > 0) {  // every block reads the same flags (published by the last grid sync): a uniform exit
      int any = 0;
      for (int p = 0; p < a.npairs; ++p) any |= act[p];
      if (!any) break;
    }
    // phase 1: v and the new u; the squared change summed per tile
    for (int t = blockIdx.x; t < work; t += gridDim.x) {
      const int pair = t / a.tiles, tile = t - pair * a.tiles;
      if (k > 0 && !act[pair]) continue;
      float* base = a.ws + pair * a.pair_stride;
      float* u1 = base + o_u1;
      float* u2 = base + o_u2;
      const float *wxp = base + L.plane(kWx), *wyp = base + L.plane(kWy), *rhop = base + L.plane(kRho);
      const float *p11 = base + L.plane(kP11), *p12 = base + L.plane(kP12), *p21 = base + L.plane(kP21),
                  *p22 = base + L.plane(kP22);
      float e = 0.f;
#pragma unroll
      for (int j = 0; j < kPxPerThread; ++j) {
        const int i = tile * kTile + j * kT + threadIdx.x;
        if (i >= npx) break;
        const int y = i / w, x = i - y * w;
        const float gx = wxp[i], gy = wyp[i], grad = gx * gx + gy * gy;
        const float uo1 = u1[i], uo2 = u2[i];
        const float rho = rhop[i] + gx * uo1 + gy * uo2;
        float d1, d2;
        if (rho < -a.l_t * grad) {
          d1 = a.l_t * gx;
          d2 = a.l_t * gy;
        } else if (rho > a.l_t * grad) {
          d1 = -a.l_t * gx;
          d2 = -a.l_t * gy;
        } else if (grad < 1e-10f) {
          d1 = d2 = 0.f;
        } else {
          const float fi = -rho / grad;
          d1 = fi * gx;
          d2 = fi * gy;
        }
        const float v1 = uo1 + d1, v2 = uo2 + d2;
        const float div1 = (p11[i] - (x > 0 ? p11[i - 1] : 0.f)) + (p12[i] - (y > 0 ? p12[i - w] : 0.f));
        const float div2 = (p21[i] - (x > 0 ? p21[i - 1] : 0.f)) + (p22[i] - (y > 0 ? p22[i - w] : 0.f));
        const float n1 = v1 + a.theta * div1, n2 = v2 + a.theta * div2;
        const float e1 = n1 - uo1, e2 = n2 - uo2;
        e += e1 * e1 + e2 * e2;
        u1[i] = n1;
        u2[i] = n2;
      }
      const float s = block_sum(e, shf);
      if (threadIdx.x == 0) base[L.plane(kPart) + tile] = s;
    }
    grid.sync();
    // phase 2: the dual variables from the new u
    for (int t = blockIdx.x; t < work; t += gridDim.x) {
      const int pair = t / a.tiles, tile = t - pair * a.tiles;
      if (k > 0 && !act[pair]) continue;
      float* base = a.ws + pair * a.pair_stride;
      const float* u1 = base + o_u1;
      const float* u2 = base + o_u2;
      float *p11 = base + L.plane(kP11), *p12 = base + L.plane(kP12), *p21 = base + L.plane(kP21),
            *p22 = base + L.plane(kP22);
#pragma unroll
      for (int j = 0; j < kPxPerThread; ++j) {
        const int i = tile * kTile + j * kT + threadIdx.x;
        if (i >= npx) break;
        const int y = i / w, x = i - y * w;
        const float c1 = u1[i], c2 = u2[i];
        const float a1 = x < w - 1 ? u1[i + 1] - c1 : 0.f, b1 = y < h - 1 ? u1[i + w] - c1 : 0.f;
        const float a2 = x < w - 1 ? u2[i + 1] - c2 : 0.f, b2 = y < h - 1 ? u2[i + w] - c2 : 0.f;
        const float ng1 = 1.f + a.taut * sqrtf(a1 * a1 + b1 * b1), ng2 = 1.f + a.taut * sqrtf(a2 * a2 + b2 * b2);
        p11[i] = (p11[i] + a.taut * a1) / ng1;
        p12[i] = (p12[i] + a.taut * b1) / ng1;
        p21[i] = (p21[i] + a.taut * a2) / ng2;
        p22[i] = (p22[i] + a.taut * b2) / ng2;
      }
    }
    // the stop decision of each pair, by one block per pair, from the tile partials of phase 1
    int* next = a.flags + ((k + 1) & 1) * SCN_MAX_PTRS;
    for (int pair = blockIdx.x; pair < a.npairs; pair += gridDim.x) {
      if (k > 0 && !act[pair]) {
        if (threadIdx.x == 0) next[pair] = 0;
        continue;
      }
      const float* part = a.ws + pair * a.pair_stride + L.plane(kPart);
      double s = 0.0;
      for (int t = threadIdx.x; t < a.tiles; t += kT) s += (double)part[t];
      s = block_sum(s, shd);
      if (threadIdx.x == 0) {
        const double err = s / (double)npx;
        next[pair] = err > a.eps2 && k + 1 < a.iterations;
        a.counts[pair * a.count_stride + a.count_idx] = k + 1;
      }
    }
    grid.sync();
  }
}

// ---- median (cv2.medianBlur, float, replicate borders) of u1 and u2 into the other u planes ----
template <int K>
__global__ void __launch_bounds__(kT) tvl1_median_kernel(float* __restrict__ ws, size_t pair_stride, Layout L, int w,
                                                         int h, int ucur) {
  const int i = blockIdx.x * kT + threadIdx.x;
  if (i >= w * h) return;
  const int pair = blockIdx.y >> 1, c = blockIdx.y & 1;
  float* base = ws + pair * pair_stride;
  const float* src = base + L.plane(c ? (ucur ? kU2b : kU2) : (ucur ? kU1b : kU1));
  float* dst = base + L.plane(c ? (ucur ? kU2 : kU2b) : (ucur ? kU1 : kU1b));
  const int y = i / w, x = i - y * w;
  constexpr int R = K / 2, N = K * K;
  float v[N];
#pragma unroll
  for (int dy = -R; dy <= R; ++dy) {
    const float* row = src + (size_t)clampi(y + dy, 0, h - 1) * w;
#pragma unroll
    for (int dx = -R; dx <= R; ++dx) v[(dy + R) * K + dx + R] = row[clampi(x + dx, 0, w - 1)];
  }
  // partial bubble sort: after pass m, v[m] holds the (m + 1)-th smallest; the median is settled after N / 2 + 1
#pragma unroll
  for (int m = 0; m <= N / 2; ++m)
#pragma unroll
    for (int j = N - 1; j > m; --j) {
      const float lo = fminf(v[j - 1], v[j]), hi = fmaxf(v[j - 1], v[j]);
      v[j - 1] = lo;
      v[j] = hi;
    }
  dst[i] = v[N / 2];
}

// (u1, u2) -> the caller's interleaved flow.  blockIdx.y = pair
__global__ void __launch_bounds__(kT) tvl1_store_kernel(const float* __restrict__ ws, size_t pair_stride, Layout L,
                                                        int npx, int ucur, MutPtrBatch out) {
  const int i = blockIdx.x * kT + threadIdx.x;
  if (i >= npx) return;
  const float* base = ws + blockIdx.y * pair_stride;
  float2* f = reinterpret_cast<float2*>(out.p[blockIdx.y]);
  f[i] = make_float2(base[L.plane(ucur ? kU1b : kU1) + i], base[L.plane(ucur ? kU2b : kU2) + i]);
}

int iterate_grid() {
  static int blocks = [] {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, tvl1_iterate_kernel, kT, 0) != cudaSuccess ||
        per_sm <= 0)
      return 0;
    return per_sm * sm_count();
  }();
  return blocks;
}

bool finite(float v) { return isfinite(v); }

}  // namespace
}  // namespace scn

extern "C" size_t scn_tvl1_workspace_bytes(int width, int height, int n) {
  if (width < 2 || height < 2 || n < 0) return 0;
  const int chunk = n < SCN_MAX_PTRS ? n : SCN_MAX_PTRS;
  return scn::kHeadBytes + scn::layout(width, height).pair_stride * sizeof(float) * (size_t)(chunk > 0 ? chunk : 1);
}

extern "C" int scn_tvl1_u8(const uint8_t* const* host_prev_ptrs, const uint8_t* const* host_next_ptrs, int n,
                           int width, int height, float* const* host_flow_ptrs, float tau, float lambda, float theta,
                           int nscales, int warps, float epsilon, int iterations, float scale_step,
                           int median_filtering, int* host_iterations, void* workspace, size_t workspace_bytes,
                           void* stream) {
  using namespace scn;
  if (n < 0 || width < 2 || height < 2 || !finite(tau) || !finite(lambda) || !finite(theta) || !finite(epsilon) ||
      !finite(scale_step) || !(tau > 0.f) || !(lambda > 0.f) || !(theta > 0.f) || nscales < 1 ||
      nscales > kMaxLevels || warps < 1 || warps > kMaxWarps || iterations < 1 || iterations > 10000 ||
      !(scale_step > 0.f) || !(scale_step < 1.f) ||
      (median_filtering != 1 && median_filtering != 3 && median_filtering != 5))
    return SCN_E_BADARG;
  if ((size_t)width * height > (size_t)1 << 30) return SCN_E_BADARG;  // pixel indices are int
  if (n == 0) return 0;
  if (!host_prev_ptrs || !host_next_ptrs || !host_flow_ptrs || !workspace) return SCN_E_BADARG;
  if (workspace_bytes < scn_tvl1_workspace_bytes(width, height, n)) return SCN_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid_max = iterate_grid();
  if (grid_max <= 0) return launch_status() ? launch_status() : (int)cudaErrorNoDevice;

  int lw[kMaxLevels], lh[kMaxLevels];
  const int levels = plan_levels(width, height, nscales, scale_step, lw, lh);
  size_t level_off[kMaxLevels];
  for (int s = 0, off = 0; s < levels; ++s) {  // a frame's levels packed into its kMaxLevels planes
    level_off[s] = (size_t)off;
    off += (int)(((size_t)lw[s] * lh[s] + 63) & ~(size_t)63);
  }
  const Layout L = layout(width, height);
  int* flags = (int*)workspace;
  int* counts = flags + 2 * SCN_MAX_PTRS;
  float* ws = (float*)((uint8_t*)workspace + kHeadBytes);
  const size_t pair_stride = L.pair_stride;
  const int npx0 = width * height;
  const float l_t = lambda * theta, taut = tau / theta;
  const double eps2 = epsilon > 0.f ? (double)epsilon * epsilon : -1.0;
  const float up = (float)(1.0 / scale_step);
  const int count_stride = nscales * warps;
  auto blocks = [](int px) { return (unsigned)((px + kT - 1) / kT); };

  return for_each_chunk(n, [&](int i0, int cnt) -> int {
    int rc;
    if (host_iterations && (rc = (int)cudaMemsetAsync(counts, 0, sizeof(int) * (size_t)cnt * count_stride, st)))
      return rc;
    const PtrBatch prev = gather<PtrBatch>(host_prev_ptrs, i0, cnt), next = gather<PtrBatch>(host_next_ptrs, i0, cnt);
    rc = launch_kernel("tvl1_gray_kernel", st, [&] {
      tvl1_gray_kernel<<<dim3(blocks(npx0), (unsigned)cnt * 2), kT, 0, st>>>(prev, next, npx0, ws, pair_stride,
                                                                           L.pyr(0, 0), L.pyr(1, 0));
    });
    if (rc) return rc;
    for (int s = 1; s < levels; ++s) {
      const Pair2 jobs = {{L.pyr(0, level_off[s - 1]), L.pyr(1, level_off[s - 1])},
                          {L.pyr(0, level_off[s]), L.pyr(1, level_off[s])}};
      rc = launch_kernel("tvl1_resize_kernel", st, [&] {
        tvl1_resize_kernel<<<dim3(blocks(lw[s] * lh[s]), (unsigned)cnt * 2), kT, 0, st>>>(
            ws, pair_stride, jobs, lw[s - 1], lh[s - 1], lw[s], lh[s], 1.0 / ((double)lw[s] / lw[s - 1]),
            1.0 / ((double)lh[s] / lh[s - 1]), 1.f, 0);
      });
      if (rc) return rc;
    }
    int ucur = 0;
    for (int s = levels - 1; s >= 0; --s) {
      const int w = lw[s], h = lh[s], npx = w * h;
      if (s < levels - 1) {  // u of the coarser level, upsampled into the other u planes and scaled
        const Pair2 jobs = {{L.plane(ucur ? kU1b : kU1), L.plane(ucur ? kU2b : kU2)},
                            {L.plane(ucur ? kU1 : kU1b), L.plane(ucur ? kU2 : kU2b)}};
        rc = launch_kernel("tvl1_resize_kernel", st, [&] {
          tvl1_resize_kernel<<<dim3(blocks(npx), (unsigned)cnt * 2), kT, 0, st>>>(
              ws, pair_stride, jobs, lw[s + 1], lh[s + 1], w, h, 1.0 / ((double)w / lw[s + 1]),
              1.0 / ((double)h / lh[s + 1]), up, 1);
        });
        if (rc) return rc;
        ucur ^= 1;
      }
      rc = launch_kernel("tvl1_grad_kernel", st, [&] {
        tvl1_grad_kernel<<<dim3(blocks(npx), (unsigned)cnt), kT, 0, st>>>(ws, pair_stride, L, L.pyr(1, level_off[s]),
                                                                          w, h, s == levels - 1, ucur);
      });
      if (rc) return rc;
      const int tiles = (npx + kTile - 1) / kTile;
      for (int wi = 0; wi < warps; ++wi) {
        rc = launch_kernel("tvl1_warp_kernel", st, [&] {
          tvl1_warp_kernel<<<dim3(blocks(npx), (unsigned)cnt), kT, 0, st>>>(ws, pair_stride, L, L.pyr(0, level_off[s]),
                                                                            L.pyr(1, level_off[s]), w, h, ucur);
        });
        if (rc) return rc;
        IterArgs a;
        a.ws = ws;
        a.pair_stride = pair_stride;
        a.L = L;
        a.ucur = ucur;
        a.w = w;
        a.h = h;
        a.npx = npx;
        a.tiles = tiles;
        a.npairs = cnt;
        a.l_t = l_t;
        a.theta = theta;
        a.taut = taut;
        a.eps2 = eps2;
        a.iterations = iterations;
        a.flags = flags;
        a.counts = counts;
        a.count_idx = s * warps + wi;
        a.count_stride = count_stride;
        const int grid = grid_max < cnt * tiles ? grid_max : cnt * tiles;
        void* params[] = {&a};
        cudaError_t ce = cudaSuccess;
        rc = launch_kernel("tvl1_iterate_kernel", st, [&] {
          ce = cudaLaunchCooperativeKernel((const void*)tvl1_iterate_kernel, dim3((unsigned)grid), dim3(kT), params, 0,
                                           st);
        });
        if (ce != cudaSuccess) return (int)ce;
        if (rc) return rc;
        if (median_filtering > 1) {
          rc = launch_kernel("tvl1_median_kernel", st, [&] {
            if (median_filtering == 3)
              tvl1_median_kernel<3><<<dim3(blocks(npx), (unsigned)cnt * 2), kT, 0, st>>>(ws, pair_stride, L, w, h, ucur);
            else
              tvl1_median_kernel<5><<<dim3(blocks(npx), (unsigned)cnt * 2), kT, 0, st>>>(ws, pair_stride, L, w, h, ucur);
          });
          if (rc) return rc;
          ucur ^= 1;
        }
      }
    }
    const MutPtrBatch out = gather<MutPtrBatch>((uint8_t* const*)host_flow_ptrs, i0, cnt);
    rc = launch_kernel("tvl1_store_kernel", st, [&] {
      tvl1_store_kernel<<<dim3(blocks(npx0), (unsigned)cnt), kT, 0, st>>>(ws, pair_stride, L, npx0, ucur, out);
    });
    if (rc) return rc;
    if (host_iterations) {
      cudaError_t e = cudaMemcpyAsync(host_iterations + (size_t)i0 * count_stride, counts,
                                      sizeof(int) * (size_t)cnt * count_stride, cudaMemcpyDeviceToHost, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
      if (e != cudaSuccess) return (int)e;
    }
    return 0;
  });
}
