// flow.cu -- dense optical flow of the reference's OpticalFlow op on the GPU (sm_90a).
// Replaces OpticalFlowKernelCPU::execute (reference tests/test_ops.cpp:63-111):
//   gray = cvtColor(frame, COLOR_BGR2GRAY)                           (15-bit fixed point)
//   flow = cv::FarnebackOpticalFlow(3, 0.5, false, 15, 3, 5, 1.2, 0)->calc(gray0, gray1)
// The Farneback arithmetic is OpenCV's (modules/video/src/optflowgf.cpp): per pyramid level
//   I_i   = resize(GaussianBlur(gray_i as f32, smooth_sz, sigma), level size)   (fastPyramids=false)
//   R_i   = polynomial expansion (separable (2n+1)-tap Gaussian-weighted basis, 5 coefficients)
//   M     = UpdateMatrices(R0, R1 warped by the current flow)        (5 floats per pixel)
//   flow  = solve 2x2 from the winSize x winSize box average of M,   numIters times
// Floating point: sums are taken in a different order than OpenCV's SIMD code, so parity is within
// a tolerance (tests/test_flow_gpu.py), not bit-exact.  The 2x2 solve runs in double like OpenCV's (the
// determinant cancels catastrophically in float); the window sums in float (box_solve_f32_kernel) or double.
// All kernels are plain per-pixel / separable memory-bound passes (no tensor cores).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "scn_common.cuh"

namespace scn {
namespace {

constexpr int kMaxTaps = 32;   // Gaussian half-width limit (ksize <= 63)
constexpr int kMaxPolyN = 7;

struct GaussK {
  int radius;
  float k[2 * kMaxTaps + 1];
};
struct PolyK {
  int n;
  float g[kMaxPolyN + 1], xg[kMaxPolyN + 1], xxg[kMaxPolyN + 1];
  float ig11, ig03, ig33, ig55;
};

__device__ __forceinline__ int reflect101(int p, int len) {
  if (len == 1) return 0;
  while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - 2 - p;
  return p;
}
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// RGB24 -> gray (as float) with OpenCV's BGR2GRAY weights applied to channel order as stored
__global__ void gray_kernel(const uint8_t* __restrict__ src, int n, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* p = src + (size_t)i * 3;
  dst[i] = (float)((p[0] * 3735 + p[1] * 19235 + p[2] * 9798 + 16384) >> 15);
}

__global__ void gauss_h_kernel(const float* __restrict__ src, int w, int h, GaussK gk, float* __restrict__ dst) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const float* row = src + (size_t)y * w;
  float s = 0.f;
  for (int i = -gk.radius; i <= gk.radius; ++i) s = __fmaf_rn(gk.k[i + gk.radius], row[reflect101(x + i, w)], s);
  dst[(size_t)y * w + x] = s;
}

__global__ void gauss_v_kernel(const float* __restrict__ src, int w, int h, GaussK gk, float* __restrict__ dst) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  float s = 0.f;
  for (int i = -gk.radius; i <= gk.radius; ++i) s = __fmaf_rn(gk.k[i + gk.radius], src[(size_t)reflect101(y + i, h) * w + x], s);
  dst[(size_t)y * w + x] = s;
}

// cv::resize INTER_LINEAR on float images with CN channels; `mul` scales the result (flow upsample)
template <int CN>
__global__ void resize_f32_kernel(const float* __restrict__ src, int sw, int sh, float* __restrict__ dst, int dw,
                                  int dh, double sx, double sy, float mul) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= dw) return;
  float fy = (float)__dsub_rn(__dmul_rn((double)y + 0.5, sy), 0.5);
  int iy = (int)floorf(fy);
  fy -= (float)iy;
  if (iy < 0) { fy = 0.f; iy = 0; }
  if (iy >= sh - 1) { fy = 0.f; iy = sh - 1; }
  const int iy1 = min(iy + 1, sh - 1);
  float fx = (float)__dsub_rn(__dmul_rn((double)x + 0.5, sx), 0.5);
  int ix = (int)floorf(fx);
  fx -= (float)ix;
  if (ix < 0) { fx = 0.f; ix = 0; }
  if (ix >= sw - 1) { fx = 0.f; ix = sw - 1; }
  const int ix1 = min(ix + 1, sw - 1);
#pragma unroll
  for (int c = 0; c < CN; ++c) {
    const float a = src[((size_t)iy * sw + ix) * CN + c], b = src[((size_t)iy * sw + ix1) * CN + c];
    const float d = src[((size_t)iy1 * sw + ix) * CN + c], e = src[((size_t)iy1 * sw + ix1) * CN + c];
    const float top = __fadd_rn(__fmul_rn(a, 1.f - fx), __fmul_rn(b, fx));
    const float bot = __fadd_rn(__fmul_rn(d, 1.f - fx), __fmul_rn(e, fx));
    dst[((size_t)y * dw + x) * CN + c] = __fadd_rn(__fmul_rn(top, 1.f - fy), __fmul_rn(bot, fy)) * mul;
  }
}

// polynomial expansion, vertical pass: (t0,t1,t2) per pixel, rows clamped at the border
__global__ void poly_v_kernel(const float* __restrict__ src, int w, int h, PolyK pk, float* __restrict__ dst3) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  float t0 = src[(size_t)y * w + x] * pk.g[0], t1 = 0.f, t2 = 0.f;
  for (int k = 1; k <= pk.n; ++k) {
    const float sp = src[(size_t)clampi(y + k, 0, h - 1) * w + x], sm = src[(size_t)clampi(y - k, 0, h - 1) * w + x];
    t0 = __fmaf_rn(pk.g[k], sp + sm, t0);
    t1 = __fmaf_rn(pk.xg[k], sp - sm, t1);
    t2 = __fmaf_rn(pk.xxg[k], sp + sm, t2);
  }
  float* d = dst3 + ((size_t)y * w + x) * 3;
  d[0] = t0;
  d[1] = t1;
  d[2] = t2;
}

// horizontal pass: columns clamped (OpenCV replicates the edge triple into its row padding)
__global__ void poly_h_kernel(const float* __restrict__ src3, int w, int h, PolyK pk, float* __restrict__ dst5) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const float* row = src3 + (size_t)y * w * 3;
  const float* c0 = row + (size_t)x * 3;
  float b1 = c0[0] * pk.g[0], b2 = 0.f, b3 = c0[1] * pk.g[0], b4 = 0.f, b5 = c0[2] * pk.g[0], b6 = 0.f;
  for (int k = 1; k <= pk.n; ++k) {
    const float* p = row + (size_t)clampi(x + k, 0, w - 1) * 3;
    const float* m = row + (size_t)clampi(x - k, 0, w - 1) * 3;
    const float tg = p[0] + m[0];
    b1 = __fmaf_rn(tg, pk.g[k], b1);
    b2 = __fmaf_rn(p[0] - m[0], pk.xg[k], b2);
    b4 = __fmaf_rn(tg, pk.xxg[k], b4);
    b3 = __fmaf_rn(p[1] + m[1], pk.g[k], b3);
    b6 = __fmaf_rn(p[1] - m[1], pk.xg[k], b6);
    b5 = __fmaf_rn(p[2] + m[2], pk.g[k], b5);
  }
  float* d = dst5 + (size_t)y * w + x;  // coefficient planes (see "layout" above update_matrices_kernel)
  const size_t ps = (size_t)w * h;
  d[1 * ps] = b2 * pk.ig11;
  d[0] = b3 * pk.ig11;
  d[3 * ps] = __fmaf_rn(b4, pk.ig33, __fmul_rn(b1, pk.ig03));
  d[2 * ps] = __fmaf_rn(b5, pk.ig33, __fmul_rn(b1, pk.ig03));
  d[4 * ps] = b6 * pk.ig55;
}

constexpr int UMW = 32, UMH = 8;
// Layout: the 5 expansion coefficients (R0, R1) and the 5 matrix elements (M) of a level are PLANES of w x h floats,
// coefficient c of pixel (x, y) at [c * w * h + y * w + x].  With the 5 values of a pixel adjacent (20 bytes: no
// 128-bit access possible) every one of the 30 loads / stores of a pixel here touched 5-6 cache lines per warp and the
// kernel ran against the L1 wavefront rate; planes make each a
// contiguous 128-byte row segment.
__global__ void update_matrices_kernel(const float* __restrict__ R0, const float* __restrict__ R1,
                                       const float* __restrict__ flow, int w, int h, float* __restrict__ M) {
  // a CTA is a UMW x UMH pixel tile (a warp = 32 pixels of a row): the bilinear taps of row y + 1 are mostly the
  // lower taps of row y, and with eight rows in one CTA they meet in L1 instead of L2
  const int x = blockIdx.x * UMW + (threadIdx.x & (UMW - 1)), y = blockIdx.y * UMH + threadIdx.x / UMW;
  if (x >= w || y >= h) return;
  const float border[5] = {0.14f, 0.14f, 0.4472f, 0.4472f, 0.4472f};
  const int BORDER = 5;
  const size_t ps = (size_t)w * h;
  const float* r0p = R0 + (size_t)y * w + x;
  const float r0[5] = {r0p[0], r0p[ps], r0p[2 * ps], r0p[3 * ps], r0p[4 * ps]};
  const float dx = flow[((size_t)y * w + x) * 2], dy = flow[((size_t)y * w + x) * 2 + 1];
  float fx = (float)x + dx, fy = (float)y + dy;
  const int x1 = (int)floorf(fx), y1 = (int)floorf(fy);
  fx -= (float)x1;
  fy -= (float)y1;
  float r2, r3, r4, r5, r6;
  if ((unsigned)x1 < (unsigned)(w - 1) && (unsigned)y1 < (unsigned)(h - 1)) {
    const float a00 = (1.f - fx) * (1.f - fy), a01 = fx * (1.f - fy), a10 = (1.f - fx) * fy, a11 = fx * fy;
    const float* p = R1 + (size_t)y1 * w + x1;
    const float* q = p + w;
    r2 = a00 * p[0] + a01 * p[1] + a10 * q[0] + a11 * q[1];
    r3 = a00 * p[ps] + a01 * p[ps + 1] + a10 * q[ps] + a11 * q[ps + 1];
    r4 = a00 * p[2 * ps] + a01 * p[2 * ps + 1] + a10 * q[2 * ps] + a11 * q[2 * ps + 1];
    r5 = a00 * p[3 * ps] + a01 * p[3 * ps + 1] + a10 * q[3 * ps] + a11 * q[3 * ps + 1];
    r6 = a00 * p[4 * ps] + a01 * p[4 * ps + 1] + a10 * q[4 * ps] + a11 * q[4 * ps + 1];
    r4 = (r0[2] + r4) * 0.5f;
    r5 = (r0[3] + r5) * 0.5f;
    r6 = (r0[4] + r6) * 0.25f;
  } else {
    r2 = r3 = 0.f;
    r4 = r0[2];
    r5 = r0[3];
    r6 = r0[4] * 0.5f;
  }
  r2 = (r0[0] - r2) * 0.5f;
  r3 = (r0[1] - r3) * 0.5f;
  r2 += r4 * dy + r6 * dx;
  r3 += r6 * dy + r5 * dx;
  if ((unsigned)(x - BORDER) >= (unsigned)(w - BORDER * 2) || (unsigned)(y - BORDER) >= (unsigned)(h - BORDER * 2)) {
    const float scale = (x < BORDER ? border[x] : 1.f) * (x >= w - BORDER ? border[w - x - 1] : 1.f) *
                        (y < BORDER ? border[y] : 1.f) * (y >= h - BORDER ? border[h - y - 1] : 1.f);
    r2 *= scale;
    r3 *= scale;
    r4 *= scale;
    r5 *= scale;
    r6 *= scale;
  }
  float* m = M + (size_t)y * w + x;
  m[0] = r4 * r4 + r6 * r6;
  m[ps] = (r4 + r5) * r6;
  m[2 * ps] = r5 * r5 + r6 * r6;
  m[3 * ps] = r4 * r2 + r6 * r3;
  m[4 * ps] = r6 * r2 + r5 * r3;
}

// box filter, vertical pass in double (rows clamped); one thread per (x, channel)
__global__ void box_v_kernel(const float* __restrict__ M, int w, int h, int m, double* __restrict__ V) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (i >= w * 5) return;
  const int c = i / w, x = i - c * w;
  const size_t ps = (size_t)w * h;
  double s = 0.0;
  for (int k = -m; k <= m; ++k) s += (double)M[c * ps + (size_t)clampi(y + k, 0, h - 1) * w + x];
  V[c * ps + (size_t)y * w + x] = s;
}

// horizontal pass (columns clamped) + the 2x2 solve of FarnebackUpdateFlow_Blur
__global__ void box_h_solve_kernel(const double* __restrict__ V, int w, int h, int m, double scale,
                                   float* __restrict__ flow) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const double* row = V + (size_t)y * w;
  const size_t ps = (size_t)w * h;
  double hs[5] = {0, 0, 0, 0, 0};
  for (int k = -m; k <= m; ++k) {
    const double* p = row + clampi(x + k, 0, w - 1);
#pragma unroll
    for (int c = 0; c < 5; ++c) hs[c] += p[c * ps];
  }
  const double g11 = hs[0] * scale, g12 = hs[1] * scale, g22 = hs[2] * scale, h1 = hs[3] * scale, h2 = hs[4] * scale;
  const double idet = 1. / (g11 * g22 - g12 * g12 + 1e-3);
  flow[((size_t)y * w + x) * 2] = (float)((g11 * h2 - g12 * h1) * idet);
  flow[((size_t)y * w + x) * 2 + 1] = (float)((g22 * h1 - g12 * h2) * idet);
}


// ---- fused, shared-memory tiled forms of the three separable stages -------------------------------
// The per-row kernels above make two global round trips per stage (h pass, v pass) with one pixel
// per thread and a clamp/reflect per tap.  The fused kernels load a tile with its halo once
// (border handling happens while loading), run both passes out of shared memory and keep the
// summation order of the two-pass kernels, so their results are bit-identical to them
// (tests/test_flow_gpu.py compares the two paths).  256 threads per CTA.
constexpr int FT = 256;

// GaussianBlur: tile (TH + 2r) x (TW + 2r) in, h pass into hbuf, v pass out.  Threads are laid out
// 64 x 4 (column, row phase) so no index needs a division.
constexpr int GTW = 64, GTH = 32;
template <int R>  // R > 0: radius known at compile time (taps unrolled, coefficients read in place); 0: generic
__global__ void __launch_bounds__(FT)
gauss_fused_kernel(const float* __restrict__ src, int w, int h, GaussK gk, float* __restrict__ dst) {
  extern __shared__ float fsm[];
  const int r = R > 0 ? R : gk.radius, iw = GTW + 2 * r, ih = GTH + 2 * r;
  float* in = fsm;             // ih x iw
  float* hb = fsm + ih * iw;   // ih x GTW
  const int x0 = blockIdx.x * GTW, y0 = blockIdx.y * GTH;
  const int tx = threadIdx.x & 63, tq = threadIdx.x >> 6;
  // tile load, 8 independent global loads in flight per thread before the first shared store (a
  // plain load->store loop serialises on the load latency: r01 ncu long_scoreboard 3-9 per issue)
  for (int i = tx; i < iw; i += 64) {
    const int sx = reflect101(x0 - r + i, w);
    for (int j0 = tq; j0 < ih; j0 += 32) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int j = j0 + 4 * u;
        v[u] = j < ih ? src[(size_t)reflect101(y0 - r + j, h) * w + sx] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int j = j0 + 4 * u;
        if (j < ih) in[j * iw + i] = v[u];
      }
    }
  }
  __syncthreads();
  for (int j = tq; j < ih; j += 4) {
    const float* row = in + j * iw + tx;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i <= 2 * r; ++i) s = __fmaf_rn(gk.k[i], row[i], s);
    hb[j * GTW + tx] = s;
  }
  __syncthreads();
  const int x = x0 + tx;
  if (x >= w) return;
  for (int ty = tq; ty < GTH; ty += 4) {
    const int y = y0 + ty;
    if (y >= h) break;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i <= 2 * r; ++i) s = __fmaf_rn(gk.k[i], hb[(ty + i) * GTW + tx], s);
    dst[(size_t)y * w + x] = s;
  }
}

// Polynomial expansion: v pass (3 values per pixel) into shared memory, h pass to 5 coefficients.
constexpr int PTW = 64, PTH = 32;
template <int N>  // N > 0: polyN known at compile time; 0: generic
__global__ void __launch_bounds__(FT)
poly_fused_kernel(const float* __restrict__ src, int w, int h, PolyK pk, float* __restrict__ dst5) {
  extern __shared__ float fsm[];
  const int n = N > 0 ? N : pk.n, iw = PTW + 2 * n, ih = PTH + 2 * n;
  float* in = fsm;            // ih x iw
  float* t3 = fsm + ih * iw;  // PTH x iw x 3
  const int x0 = blockIdx.x * PTW, y0 = blockIdx.y * PTH;
  const int tx = threadIdx.x & 63, tq = threadIdx.x >> 6;
  for (int i = tx; i < iw; i += 64) {
    const int sx = clampi(x0 - n + i, 0, w - 1);
    for (int j0 = tq; j0 < ih; j0 += 32) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int j = j0 + 4 * u;
        v[u] = j < ih ? src[(size_t)clampi(y0 - n + j, 0, h - 1) * w + sx] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int j = j0 + 4 * u;
        if (j < ih) in[j * iw + i] = v[u];
      }
    }
  }
  __syncthreads();
  for (int jy = tq; jy < PTH; jy += 4)
    for (int i = tx; i < iw; i += 64) {
      const float* c = in + (jy + n) * iw + i;
      float t0 = c[0] * pk.g[0], t1 = 0.f, t2 = 0.f;
#pragma unroll
      for (int k = 1; k <= n; ++k) {
        const float sp = c[k * iw], sm = c[-k * iw];
        t0 = __fmaf_rn(pk.g[k], sp + sm, t0);
        t1 = __fmaf_rn(pk.xg[k], sp - sm, t1);
        t2 = __fmaf_rn(pk.xxg[k], sp + sm, t2);
      }
      float* d = t3 + ((size_t)jy * iw + i) * 3;
      d[0] = t0;
      d[1] = t1;
      d[2] = t2;
    }
  __syncthreads();
  const int x = x0 + tx;
  if (x >= w) return;
  for (int ty = tq; ty < PTH; ty += 4) {
    const int y = y0 + ty;
    if (y >= h) break;
    const float* c0 = t3 + ((size_t)ty * iw + tx + n) * 3;
    float b1 = c0[0] * pk.g[0], b2 = 0.f, b3 = c0[1] * pk.g[0], b4 = 0.f, b5 = c0[2] * pk.g[0], b6 = 0.f;
#pragma unroll
    for (int k = 1; k <= n; ++k) {
      const float* p = c0 + k * 3;
      const float* m = c0 - k * 3;
      const float tg = p[0] + m[0];
      b1 = __fmaf_rn(tg, pk.g[k], b1);
      b2 = __fmaf_rn(p[0] - m[0], pk.xg[k], b2);
      b4 = __fmaf_rn(tg, pk.xxg[k], b4);
      b3 = __fmaf_rn(p[1] + m[1], pk.g[k], b3);
      b6 = __fmaf_rn(p[1] - m[1], pk.xg[k], b6);
      b5 = __fmaf_rn(p[2] + m[2], pk.g[k], b5);
    }
    float* d = dst5 + (size_t)y * w + x;
    const size_t ps = (size_t)w * h;
    d[1 * ps] = b2 * pk.ig11;
    d[0] = b3 * pk.ig11;
    d[3 * ps] = __fmaf_rn(b4, pk.ig33, __fmul_rn(b1, pk.ig03));
    d[2 * ps] = __fmaf_rn(b5, pk.ig33, __fmul_rn(b1, pk.ig03));
    d[4 * ps] = b6 * pk.ig55;
  }
}

// winSize x winSize box average of M (double sums, clamped borders) + the 2x2 solve.  MW = window
// half-width at compile time (winSize 15 -> 7).  Both passes are register-blocked by 4: a thread
// converts 2 MW + 4 inputs once and forms four overlapping (2 MW + 1)-term sums from them, each in the
// two-pass kernels' order.  The vertical pass reads M straight from global memory (no input tile:
// 50 KB of shared memory per CTA instead of 97 KB, 4 CTAs per SM); its sums are kept with an odd row
// stride so that the 16 rows a half-warp reads in the horizontal pass fall into distinct banks.
constexpr int BTW = 64, BTH = 16;
template <int MW>
__global__ void __launch_bounds__(FT)
box_solve_fused_kernel(const float* __restrict__ M, int w, int h, double scale, float* __restrict__ flow) {
  extern __shared__ double dsm[];
  constexpr int iw = BTW + 2 * MW, rowf = iw * 5, vstride = rowf | 1, taps = 2 * MW + 1;
  double* V = dsm;  // BTH x vstride doubles: the vertical sums of this tile (with the horizontal halo)
  const int x0 = blockIdx.x * BTW, y0 = blockIdx.y * BTH;
  // vertical: item = (group of 4 rows, column-channel q); the 2 MW + 4 inputs come straight from
  // global memory (neighbouring groups and CTAs re-read them from L1/L2), all loads issued before
  // the first conversion
  for (int e = threadIdx.x; e < (BTH / 4) * rowf; e += FT) {
    const int g4 = e / rowf, qq = e - g4 * rowf;
    const int c = qq / iw, i = qq - c * iw;  // consecutive threads: consecutive columns of one plane
    const int q = i * 5 + c;                 // shared-memory slot (pixel-major, as the horizontal pass reads it)
    // 32-bit element indices (the launcher checks w * h * 5 < 2^31); rows away from the top and
    // bottom edge need no clamp, which was most of this kernel's instructions (r01 ncu: 45 %
    // IMAD / SHF / VIADDMNMX / SEL index arithmetic)
    const int stride = w;
    const int idx0 = c * (w * h) + clampi(x0 - MW + i, 0, w - 1);
    const int ytop = y0 + g4 * 4 - MW;
    float f[taps + 3];
    if (ytop >= 0 && ytop + taps + 2 < h) {
      const float* col = M + idx0 + ytop * stride;
#pragma unroll
      for (int k = 0; k < taps + 3; ++k) f[k] = col[k * stride];
    } else {
#pragma unroll
      for (int k = 0; k < taps + 3; ++k) f[k] = M[idx0 + clampi(ytop + k, 0, h - 1) * stride];
    }
    double v[taps + 3];
#pragma unroll
    for (int k = 0; k < taps + 3; ++k) v[k] = (double)f[k];
    // first window summed directly, the next three slide (+ new - old).  Every addend is a float
    // held in a double, so the partial sums are exact -- and the sliding results identical to direct
    // sums -- unless the 2 MW + 4 values span more than ~2^28 in magnitude (OpenCV's own
    // FarnebackUpdateFlow_Blur slides the same way).
    double sum = 0.0;
#pragma unroll
    for (int k = 0; k < taps; ++k) sum += v[k];
    V[(size_t)(g4 * 4) * vstride + q] = sum;
#pragma unroll
    for (int o = 1; o < 4; ++o) {
      sum = (sum + v[o + taps - 1]) - v[o - 1];
      V[(size_t)(g4 * 4 + o) * vstride + q] = sum;
    }
  }
  __syncthreads();
  // horizontal + solve: thread = (row ty, group of 4 columns)
  const int ty = threadIdx.x & (BTH - 1), gx = threadIdx.x / BTH;  // 16 rows x 16 groups = 256 threads
  const int y = y0 + ty;
  if (y >= h) return;
  const double* p = V + (size_t)ty * vstride + (gx * 4) * 5;
  double hs[4][5];
#pragma unroll
  for (int c = 0; c < 5; ++c) {
    double s0 = 0.0;
#pragma unroll
    for (int k = 0; k < taps; ++k) s0 += p[k * 5 + c];
    hs[0][c] = s0;
#pragma unroll
    for (int o = 1; o < 4; ++o) {  // slide: + entering column - leaving column
      s0 = (s0 + p[(o + taps - 1) * 5 + c]) - p[(o - 1) * 5 + c];
      hs[o][c] = s0;
    }
  }
#pragma unroll
  for (int o = 0; o < 4; ++o) {
    const int x = x0 + gx * 4 + o;
    if (x >= w) break;
    const double g11 = hs[o][0] * scale, g12 = hs[o][1] * scale, g22 = hs[o][2] * scale, h1 = hs[o][3] * scale,
                 h2 = hs[o][4] * scale;
    const double idet = 1. / (g11 * g22 - g12 * g12 + 1e-3);
    flow[((size_t)y * w + x) * 2] = (float)((g11 * h2 - g12 * h1) * idet);
    flow[((size_t)y * w + x) * 2 + 1] = (float)((g22 * h1 - g12 * h2) * idet);
  }
}

// The same stage with FLOAT window sums (the default): the 225 addends of a window are float32 values; summed in
// float32 in a fixed tree (12 shared core rows/columns, then the 3 edge terms of each of 4 overlapping windows -- no
// subtraction, so no cancellation beyond the data's own) the relative error of a sum is ~1e-6 of sum|m|, and only the
// 2x2 solve -- where g11 g22 - g12^2 cancels -- is done in double, from those sums.  Against the double sums this
// moves the flow by <= 2e-4 px on the test pairs (tests/test_flow_gpu.py keeps the 2e-3 / 1e-4 px bounds against
// cv2), removes the f32->f64 conversions (XU pipe, 4.5 per sum) and halves the shared-memory traffic.
// SCN_FLOW_BOX=f64 selects the double kernel above.
// Tile 88 x 32 outputs: 5 * (88 + 14) = 510 column-channels ~ 2 x 256 threads.  A thread takes a column-channel
// and loads its 32 + 14 input rows ONCE into registers (coalesced: consecutive threads, consecutive floats), then
// forms the 32 vertical window sums from them -- the first version re-read 18 rows for every 4 outputs through an
// L1 squeezed by the shared-memory carve-out and was L2-bound (about 12x the input in L2 traffic per launch).
constexpr int B32W = 88, B32H = 32;
template <int MW>
struct Box32Geom {
  static constexpr int iw = B32W + 2 * MW;          // columns of a tile with its halo
  static constexpr int cp = (iw + 3) & ~3;          // pitch of one channel's row segment: 16-byte aligned
  static constexpr int vstride = 5 * cp + 4;        // floats per tile row; (vstride / 4) odd: a quarter-warp's
                                                    // eight 128-bit reads (8 rows) cover all 32 banks
  static_assert(((5 * cp + 4) / 4) % 2 == 1, "row stride must be 4 x odd floats");
};
template <int MW>
__global__ void __launch_bounds__(FT)  // 128 registers, 2 CTAs / SM: capping at 80 (3 CTAs) serialises the 46 loads: slower
box_solve_f32_kernel(const float* __restrict__ M, int w, int h, double scale, float* __restrict__ flow) {
  extern __shared__ __align__(16) float bsm[];
  using G = Box32Geom<MW>;
  constexpr int iw = G::iw, cp = G::cp, vstride = G::vstride, taps = 2 * MW + 1, in_rows = B32H + 2 * MW;
  static_assert(taps >= 7, "the 4-window tree needs at least 3 edge terms on each side");
  float* V = bsm;  // B32H x vstride: row r, channel c, column i at [r * vstride + c * cp + i]
  const int x0 = blockIdx.x * B32W, y0 = blockIdx.y * B32H;
  const int stride = w, ps = w * h;
  for (int q = threadIdx.x; q < 5 * iw; q += FT) {
    const int c = q / iw, i = q - c * iw;  // consecutive threads: consecutive columns of one plane
    const int idx0 = c * ps + clampi(x0 - MW + i, 0, w - 1);
    const int ytop = y0 - MW;
    float f[in_rows];
    if (ytop >= 0 && ytop + in_rows <= h) {
      const float* col = M + idx0 + ytop * stride;
#pragma unroll
      for (int k = 0; k < in_rows; ++k) f[k] = col[k * stride];
    } else {
#pragma unroll
      for (int k = 0; k < in_rows; ++k) f[k] = M[idx0 + clampi(ytop + k, 0, h - 1) * stride];
    }
    // rows 4g .. 4g+3: windows f[4g + o .. 4g + o + taps - 1], o = 0..3; f[4g + 3 .. 4g + taps - 1] is common
    float* vo = V + c * cp + i;
#pragma unroll
    for (int g = 0; g < B32H / 4; ++g) {
      const float* e = f + 4 * g;
      float core = e[3];
#pragma unroll
      for (int k = 4; k < taps; ++k) core += e[k];
      vo[(4 * g) * vstride] = core + ((e[0] + e[1]) + e[2]);
      vo[(4 * g + 1) * vstride] = core + ((e[1] + e[2]) + e[taps]);
      vo[(4 * g + 2) * vstride] = core + ((e[2] + e[taps]) + e[taps + 1]);
      vo[(4 * g + 3) * vstride] = core + ((e[taps] + e[taps + 1]) + e[taps + 2]);
    }
  }
  __syncthreads();
  // horizontal + solve: item = (row, group of 4 columns); a warp's lanes are 32 rows.  The taps + 3 = 18 values of a
  // channel are contiguous: four 128-bit reads and one 64-bit read instead of 18 scalar ones.
  static_assert(taps + 3 == 18, "the vector reads below are laid out for winSize 15");
  for (int e = threadIdx.x; e < B32H * (B32W / 4); e += FT) {
    const int ty = e & (B32H - 1), gx = e / B32H;
    const int y = y0 + ty;
    if (y >= h || x0 + gx * 4 >= w) continue;
    const float* p = V + (size_t)ty * vstride + gx * 4;
    float hs[4][5];
#pragma unroll
    for (int c = 0; c < 5; ++c) {
      float v[20];
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {
        const float4 t = *reinterpret_cast<const float4*>(p + c * cp + 4 * k4);
        v[4 * k4] = t.x, v[4 * k4 + 1] = t.y, v[4 * k4 + 2] = t.z, v[4 * k4 + 3] = t.w;
      }
      const float2 t2 = *reinterpret_cast<const float2*>(p + c * cp + 16);
      v[16] = t2.x, v[17] = t2.y;
      float core = v[3];
#pragma unroll
      for (int k = 4; k < taps; ++k) core += v[k];
      hs[0][c] = core + ((v[0] + v[1]) + v[2]);
      hs[1][c] = core + ((v[1] + v[2]) + v[taps]);
      hs[2][c] = core + ((v[2] + v[taps]) + v[taps + 1]);
      hs[3][c] = core + ((v[taps] + v[taps + 1]) + v[taps + 2]);
    }
    float2 out[4];
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      const double g11 = hs[o][0] * scale, g12 = hs[o][1] * scale, g22 = hs[o][2] * scale, h1 = hs[o][3] * scale,
                   h2 = hs[o][4] * scale;
      const double idet = 1. / (g11 * g22 - g12 * g12 + 1e-3);
      out[o] = make_float2((float)((g11 * h2 - g12 * h1) * idet), (float)((g22 * h1 - g12 * h2) * idet));
    }
    float2* dst = reinterpret_cast<float2*>(flow) + (size_t)y * w + x0 + gx * 4;
#pragma unroll
    for (int o = 0; o < 4; ++o)
      if (x0 + gx * 4 + o < w) dst[o] = out[o];
  }
}
inline size_t box32_smem(int) { return (size_t)B32H * Box32Geom<7>::vstride * 4; }  // kBoxMW
inline bool box_in_f64() {
  static const bool v = [] {
    const char* e = getenv("SCN_FLOW_BOX");
    return e && strcmp(e, "f64") == 0;
  }();
  return v;
}

constexpr size_t kFusedSmemCap = 160 * 1024;
inline size_t gauss_smem(int r) { return ((size_t)(GTH + 2 * r) * (GTW + 2 * r) + (size_t)(GTH + 2 * r) * GTW) * 4; }
inline size_t poly_smem(int n) { return ((size_t)(PTH + 2 * n) * (PTW + 2 * n) + (size_t)PTH * (PTW + 2 * n) * 3) * 4; }
constexpr int kBoxMW = 7;  // the fused box kernel is instantiated for winSize 15 (the reference's)
inline size_t box_smem(int m) { return (size_t)BTH * (((BTW + 2 * m) * 5) | 1) * 8; }
// SCN_FLOW_UNFUSED=1 selects the two-pass kernels (kept as the reference the fused ones are tested against); they
// also run on a device that refuses the fused kernels' shared-memory limit
inline bool use_fused() {
  static const bool off = [] {
    const char* e = getenv("SCN_FLOW_UNFUSED");
    return e && e[0] == '1';
  }();
  if (off) return false;
  for (const void* f : {(const void*)gauss_fused_kernel<0>, (const void*)gauss_fused_kernel<1>,
                        (const void*)gauss_fused_kernel<4>, (const void*)gauss_fused_kernel<9>,
                        (const void*)poly_fused_kernel<0>, (const void*)poly_fused_kernel<5>,
                        (const void*)box_solve_fused_kernel<kBoxMW>, (const void*)box_solve_f32_kernel<kBoxMW>})
    if (raise_smem_limit(f, kFusedSmemCap)) return false;
  return true;
}

// ---- host-side constants --------------------------------------------------------------------
void make_gauss(int ksize, double sigma, GaussK& gk) {
  static const float small_tab[4][7] = {{1.f},
                                        {0.25f, 0.5f, 0.25f},
                                        {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f},
                                        {0.03125f, 0.109375f, 0.21875f, 0.28125f, 0.21875f, 0.109375f, 0.03125f}};
  gk.radius = ksize / 2;
  if (sigma <= 0 && (ksize & 1) && ksize <= 7) {
    for (int i = 0; i < ksize; ++i) gk.k[i] = small_tab[ksize >> 1][i];
    return;
  }
  if (sigma <= 0) sigma = ((ksize - 1) * 0.5 - 1) * 0.3 + 0.8;
  const double scale2x = -0.5 / (sigma * sigma);
  double tmp[2 * kMaxTaps + 1], sum = 0;
  for (int i = 0; i < ksize; ++i) {
    const double x = i - (ksize - 1) * 0.5;
    tmp[i] = exp(scale2x * x * x);
    sum += tmp[i];
  }
  for (int i = 0; i < ksize; ++i) gk.k[i] = (float)(tmp[i] / sum);
}

void make_poly(int n, double sigma, PolyK& pk) {
  float g[2 * kMaxPolyN + 1];
  double s = 0;
  for (int x = -n; x <= n; ++x) {
    g[x + n] = (float)exp(-x * x / (2 * sigma * sigma));
    s += g[x + n];
  }
  s = 1. / s;
  for (int x = -n; x <= n; ++x) g[x + n] = (float)(g[x + n] * s);
  pk.n = n;
  for (int x = 0; x <= n; ++x) {
    pk.g[x] = g[x + n];
    pk.xg[x] = (float)(x * g[x + n]);
    pk.xxg[x] = (float)(x * x * g[x + n]);
  }
  double G[6][6];
  memset(G, 0, sizeof(G));
  for (int y = -n; y <= n; ++y)
    for (int x = -n; x <= n; ++x) {
      G[0][0] += g[y + n] * g[x + n];
      G[1][1] += g[y + n] * g[x + n] * x * x;
      G[3][3] += g[y + n] * g[x + n] * x * x * x * x;
      G[5][5] += g[y + n] * g[x + n] * x * x * y * y;
    }
  G[2][2] = G[0][3] = G[0][4] = G[3][0] = G[4][0] = G[1][1];
  G[4][4] = G[3][3];
  G[3][4] = G[4][3] = G[5][5];
  double A[6][12];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 12; ++j) A[i][j] = j < 6 ? G[i][j] : (j - 6 == i ? 1.0 : 0.0);
  for (int c = 0; c < 6; ++c) {
    int p = c;
    for (int r = c + 1; r < 6; ++r)
      if (fabs(A[r][c]) > fabs(A[p][c])) p = r;
    if (p != c)
      for (int j = 0; j < 12; ++j) {
        const double t = A[c][j];
        A[c][j] = A[p][j];
        A[p][j] = t;
      }
    const double d = A[c][c];
    for (int j = 0; j < 12; ++j) A[c][j] /= d;
    for (int r = 0; r < 6; ++r)
      if (r != c) {
        const double f = A[r][c];
        for (int j = 0; j < 12; ++j) A[r][j] -= f * A[c][j];
      }
  }
  pk.ig11 = (float)A[1][7];
  pk.ig03 = (float)A[0][9];
  pk.ig33 = (float)A[3][9];
  pk.ig55 = (float)A[5][11];
}

struct Level {
  int w, h, smooth;
  double sigma;
};

int plan_levels(int width, int height, int num_levels, double pyr_scale, Level* lv /* [num_levels+1] */) {
  int levels = num_levels, k;
  double scale = 1;
  for (k = 0; k < levels; ++k) {
    scale *= pyr_scale;
    if (width * scale < 32 || height * scale < 32) break;
  }
  levels = k;
  for (k = 0; k <= levels; ++k) {
    scale = 1;
    for (int i = 0; i < k; ++i) scale *= pyr_scale;
    lv[k].sigma = (1. / scale - 1) * 0.5;
    int sm = (int)lrint(lv[k].sigma * 5) | 1;
    lv[k].smooth = sm < 3 ? 3 : sm;
    lv[k].w = (int)lrint(width * scale);
    lv[k].h = (int)lrint(height * scale);
  }
  return levels;
}

// workspace layout (floats unless noted), all sized for the full-resolution level
constexpr int kPyramidRoom = 2;
struct Workspace {
  float *gray[2], *tmp, *blur, *I, *poly3, *R[2], *M, *flow_a, *flow_b;
  double* V;
};

size_t carve(void* base, int w, int h, Workspace* ws) {
  const size_t px = (size_t)w * h;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    void* p = base ? (void*)((uint8_t*)base + off) : nullptr;
    off += (bytes + 255) & ~(size_t)255;
    return p;
  };
  Workspace tmpws;
  Workspace& o = ws ? *ws : tmpws;
  o.gray[0] = (float*)take(px * 4);
  o.gray[1] = (float*)take(px * 4);
  o.tmp = (float*)take(px * 4);
  o.blur = (float*)take(px * 4);
  o.I = (float*)take(px * 4);
  o.poly3 = (float*)take(px * 12);
  o.R[0] = (float*)take(px * 20 * kPyramidRoom);  // all levels of a frame's expansion when they fit (pyr_scale <= 0.7)
  o.R[1] = (float*)take(px * 20 * kPyramidRoom);
  o.M = (float*)take(px * 20);
  o.flow_a = (float*)take(px * 8);
  o.flow_b = (float*)take(px * 8);
  o.V = (double*)take(px * 40);
  return off;
}

}  // namespace
}  // namespace scn

extern "C" size_t scn_farneback_workspace_bytes(int width, int height) {
  if (width <= 0 || height <= 0) return 0;
  return scn::carve(nullptr, width, height, nullptr);
}

extern "C" int scn_farneback_u8c3(const uint8_t* const* host_prev_ptrs, const uint8_t* const* host_next_ptrs, int n,
                                  int width, int height, float* const* host_flow_ptrs, int num_levels,
                                  double pyr_scale, int win_size, int num_iters, int poly_n, double poly_sigma,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  return scn_farneback_u8c3_chain(host_prev_ptrs, host_next_ptrs, n, width, height, host_flow_ptrs, num_levels,
                                  pyr_scale, win_size, num_iters, poly_n, poly_sigma, workspace, workspace_bytes, 0,
                                  nullptr, stream);
}

extern "C" int scn_farneback_u8c3_chain(const uint8_t* const* host_prev_ptrs, const uint8_t* const* host_next_ptrs,
                                        int n, int width, int height, float* const* host_flow_ptrs, int num_levels,
                                        double pyr_scale, int win_size, int num_iters, int poly_n, double poly_sigma,
                                        void* workspace, size_t workspace_bytes, int reuse_prev, int* chain,
                                        void* stream) {
  using namespace scn;
  if (chain && (*chain < 0 || *chain > 2)) return SCN_E_BADARG;
  // win_size 1 is refused: at window half-width 0 OpenCV's FarnebackUpdateFlow_Blur does not compute a 1 x 1 box
  // (its running sums appear to start one row too many), so the plain box here would not match cv2 there
  if (n < 0 || width <= 0 || height <= 0 || num_levels < 0 || num_levels > 15 || pyr_scale <= 0 || pyr_scale >= 1 ||
      win_size < 2 || num_iters < 1 || poly_n < 1 || poly_n > kMaxPolyN || poly_sigma <= 0)
    return SCN_E_BADARG;
  if (n == 0) return 0;
  if (!host_prev_ptrs || !host_next_ptrs || !host_flow_ptrs || !workspace) return SCN_E_BADARG;
  if (workspace_bytes < scn_farneback_workspace_bytes(width, height)) return SCN_E_BADARG;
  if (height > 65535) return SCN_E_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const bool fused = use_fused();
  Workspace ws;
  carve(workspace, width, height, &ws);
  Level lv[16];
  const int levels = plan_levels(width, height, num_levels, pyr_scale, lv);
  for (int k = 0; k <= levels; ++k)
    if (lv[k].smooth / 2 > kMaxTaps) return SCN_E_UNSUPPORTED;
  PolyK pk;
  make_poly(poly_n, poly_sigma, pk);
  const int T = 128;
  auto grid2 = [&](int w, int h) { return dim3((unsigned)((w + T - 1) / T), (unsigned)h); };

  // Polynomial expansion of one frame at one level: GaussianBlur of the full-resolution gray image with the level's
  // sigma, resize to the level, expansion -> 5 coefficients per pixel at dstR.
  auto expand = [&](const float* gray, int k, float* dstR) {
    const int w = lv[k].w, h = lv[k].h;
    GaussK gk;
    make_gauss(lv[k].smooth, lv[k].sigma, gk);
    if (fused && gauss_smem(gk.radius) <= kFusedSmemCap) {
      LaunchScope ls("flow_gauss_fused_kernel", st);
      const dim3 gg((unsigned)((width + GTW - 1) / GTW), (unsigned)((height + GTH - 1) / GTH));
      const size_t sm = gauss_smem(gk.radius);
      // the radii of the reference's pyramid are instantiated: pyrScale 0.5 gives sigma 0, 0.5, 1.5, 3.5 and
      // ksize = max(3, lrint(5 sigma) | 1) = 3, 3, 9, 19 (lrint rounds 7.5 and 17.5 to even)
      switch (gk.radius) {
        case 1: gauss_fused_kernel<1><<<gg, FT, sm, st>>>(gray, width, height, gk, ws.blur); break;
        case 4: gauss_fused_kernel<4><<<gg, FT, sm, st>>>(gray, width, height, gk, ws.blur); break;
        case 9: gauss_fused_kernel<9><<<gg, FT, sm, st>>>(gray, width, height, gk, ws.blur); break;
        default: gauss_fused_kernel<0><<<gg, FT, sm, st>>>(gray, width, height, gk, ws.blur); break;
      }
    } else {
      {
        LaunchScope ls("flow_gauss_h_kernel", st);
        gauss_h_kernel<<<grid2(width, height), T, 0, st>>>(gray, width, height, gk, ws.tmp);
      }
      {
        LaunchScope ls("flow_gauss_v_kernel", st);
        gauss_v_kernel<<<grid2(width, height), T, 0, st>>>(ws.tmp, width, height, gk, ws.blur);
      }
    }
    const float* I = ws.blur;
    if (w != width || h != height) {
      LaunchScope ls("flow_resize_kernel", st);
      resize_f32_kernel<1><<<grid2(w, h), T, 0, st>>>(ws.blur, width, height, ws.I, w, h, (double)width / w,
                                                      (double)height / h, 1.f);
      I = ws.I;
    }
    if (fused && poly_smem(pk.n) <= kFusedSmemCap) {
      LaunchScope ls("flow_poly_fused_kernel", st);
      const dim3 pg((unsigned)((w + PTW - 1) / PTW), (unsigned)((h + PTH - 1) / PTH));
      if (pk.n == 5) poly_fused_kernel<5><<<pg, FT, poly_smem(pk.n), st>>>(I, w, h, pk, dstR);
      else poly_fused_kernel<0><<<pg, FT, poly_smem(pk.n), st>>>(I, w, h, pk, dstR);
    } else {
      {
        LaunchScope ls("flow_poly_v_kernel", st);
        poly_v_kernel<<<grid2(w, h), T, 0, st>>>(I, w, h, pk, ws.poly3);
      }
      {
        LaunchScope ls("flow_poly_h_kernel", st);
        poly_h_kernel<<<grid2(w, h), T, 0, st>>>(ws.poly3, w, h, pk, dstR);
      }
    }
  };
  // When every level of a frame's expansion fits its R buffer (pyr_scale <= ~0.7: the reference's 0.5 does), the
  // whole pyramid of a frame is built once and kept: in a run of consecutive pairs (next[p] == prev[p + 1], what the
  // OpticalFlow op's stencil [0, 1] produces) the second frame of a pair is the first of the next, and its gray
  // conversion, 4 full-resolution Gaussians, resizes and expansions are not repeated (1 frame per pair instead of 2).
  size_t level_off[16], pyr_px = 0;
  for (int k = 0; k <= levels; ++k) {
    level_off[k] = pyr_px * 5;
    pyr_px += ((size_t)lv[k].w * lv[k].h + 63) & ~(size_t)63;
  }
  const bool whole_pyramid = pyr_px <= (size_t)kPyramidRoom * width * height && !getenv("SCN_FLOW_NO_PYRAMID_CACHE");
  float* Rbuf[2] = {ws.R[0], ws.R[1]};
  // a caller that keeps the workspace between calls (the OpticalFlow op: one pair per call) says so through `chain`
  const bool chained = whole_pyramid && reuse_prev && chain && *chain != 0;
  if (chained) {  // *chain: 1 = the last call's `next` expansion is in ws.R[0], 2 = in ws.R[1]; it is pair 0's `prev`
    Rbuf[0] = ws.R[*chain - 1];
    Rbuf[1] = ws.R[2 - *chain];
  }
  const int npx = width * height;
  auto to_gray = [&](const uint8_t* src, float* dst) {
    LaunchScope ls("flow_gray_kernel", st);
    gray_kernel<<<(npx + 255) / 256, 256, 0, st>>>(src, npx, dst);
  };
  auto build_pyramid = [&](const uint8_t* src, float* R) {
    to_gray(src, ws.gray[0]);
    for (int k = levels; k >= 0; --k) expand(ws.gray[0], k, R + level_off[k]);
  };

  for (int pair = 0; pair < n; ++pair) {
    if (whole_pyramid) {
      if (pair > 0 && host_prev_ptrs[pair] == host_next_ptrs[pair - 1]) {
        float* t = Rbuf[0];
        Rbuf[0] = Rbuf[1];
        Rbuf[1] = t;
      } else if (pair > 0 || !chained) {
        build_pyramid(host_prev_ptrs[pair], Rbuf[0]);
      }
      build_pyramid(host_next_ptrs[pair], Rbuf[1]);
    } else {
      to_gray(host_prev_ptrs[pair], ws.gray[0]);
      to_gray(host_next_ptrs[pair], ws.gray[1]);
    }
    float* prev_flow = nullptr;
    int pw = 0, ph = 0;
    for (int k = levels; k >= 0; --k) {
      const int w = lv[k].w, h = lv[k].h;
      // the coarser levels ping-pong between two scratch flows; level 0 writes the caller's frame
      float* flow = k == 0 ? host_flow_ptrs[pair] : (prev_flow == ws.flow_a ? ws.flow_b : ws.flow_a);
      if (!prev_flow) {
        cudaError_t e = cudaMemsetAsync(flow, 0, (size_t)w * h * 8, st);
        if (e != cudaSuccess) return (int)e;
      } else {
        LaunchScope ls("flow_resize_kernel", st);
        resize_f32_kernel<2><<<grid2(w, h), T, 0, st>>>(prev_flow, pw, ph, flow, w, h, (double)pw / w,
                                                        (double)ph / h, (float)(1. / pyr_scale));
      }
      const float *R0 = Rbuf[0], *R1 = Rbuf[1];
      if (whole_pyramid) {
        R0 += level_off[k];
        R1 += level_off[k];
      } else {
        expand(ws.gray[0], k, Rbuf[0]);
        expand(ws.gray[1], k, Rbuf[1]);
      }
      {
        LaunchScope ls("flow_update_matrices_kernel", st);
        update_matrices_kernel<<<dim3((unsigned)((w + UMW - 1) / UMW), (unsigned)((h + UMH - 1) / UMH)), UMW * UMH, 0, st>>>(R0, R1, flow, w, h, ws.M);
      }
      const int m = win_size / 2;
      for (int it = 0; it < num_iters; ++it) {
        if (fused && !box_in_f64() && m == kBoxMW && (size_t)w * h * 5 < ((size_t)1 << 31)) {
          LaunchScope ls("flow_box_solve_f32_kernel", st);
          box_solve_f32_kernel<kBoxMW><<<dim3((unsigned)((w + B32W - 1) / B32W), (unsigned)((h + B32H - 1) / B32H)), FT,
                                         box32_smem(m), st>>>(ws.M, w, h, 1.0 / ((double)win_size * win_size), flow);
        } else if (fused && m == kBoxMW && (size_t)w * h * 5 < ((size_t)1 << 31)) {
          LaunchScope ls("flow_box_solve_fused_kernel", st);
          box_solve_fused_kernel<kBoxMW><<<dim3((unsigned)((w + BTW - 1) / BTW), (unsigned)((h + BTH - 1) / BTH)), FT,
                                           box_smem(m), st>>>(ws.M, w, h, 1.0 / ((double)win_size * win_size), flow);
        } else {
          {
            LaunchScope ls("flow_box_v_kernel", st);
            box_v_kernel<<<grid2(w * 5, h), T, 0, st>>>(ws.M, w, h, m, ws.V);
          }
          {
            LaunchScope ls("flow_box_h_solve_kernel", st);
            box_h_solve_kernel<<<grid2(w, h), T, 0, st>>>(ws.V, w, h, m, 1.0 / ((double)win_size * win_size), flow);
          }
        }
        if (it < num_iters - 1) {
          LaunchScope ls("flow_update_matrices_kernel", st);
          update_matrices_kernel<<<dim3((unsigned)((w + UMW - 1) / UMW), (unsigned)((h + UMH - 1) / UMH)), UMW * UMH, 0, st>>>(R0, R1, flow, w, h, ws.M);
        }
      }
      prev_flow = flow;
      pw = w;
      ph = h;
    }
    int rc = launch_status();
    if (rc) {
      if (chain) *chain = 0;
      return rc;
    }
  }
  if (chain) *chain = whole_pyramid ? (Rbuf[1] == ws.R[0] ? 1 : 2) : 0;
  return 0;
}
