/*
 * farneback_k.c -- Farneback dense optical flow in the order of scanner_b200/csrc/flow.cu.  TEST INFRASTRUCTURE ONLY
 * (like scn_oracle.c): nothing in the product path may link, import or call this file.
 *
 * orc_farneback_u8 (scn_oracle.c) is the specification held to cv2: it follows OpenCV's optflowgf.cpp, sums the
 * polynomial expansion in double and slides its box sums.  This file restates what the CUDA kernels compute instead,
 * expression for expression: the same float32 / float64 operations in the same order, a fused multiply-add (C fmaf /
 * fma) exactly where flow.cu writes __fmaf_rn / __fma_rn, every other expression rounded as written.  The kernels
 * must equal it bit for bit (tests/test_flow_exact_gpu.py); against cv2 it is within the tolerance of
 * orc_farneback_u8 (tests/test_flow_exact_cpu.py).
 *
 * The tile geometry of a kernel matters only where it fixes an order: the box kernels sum their windows in groups of
 * 4 outputs that start at multiples of 4 (both tile widths and heights are multiples of 4), so the group of a pixel
 * is (x & ~3, y & ~3).  The three box variants are chosen by `box`:
 *   0  "f32"       box_solve_f32_kernel: float sums, a shared core of taps - 3 terms plus 3 edge terms per window
 *   1  "f64_slide" box_solve_fused_kernel: double sums, the first window of a group direct, the next three slid
 *   2  "f64"       box_v_kernel + box_h_solve_kernel: double sums, every window direct
 *
 * Build: oracle/farneback_k.py compiles it into oracle/libfarneback_k.so with gcc -O2 -ffp-contract=off
 * -fno-fast-math, the flags of liborc.so (__graft_entry__.build() does so up front).
 */
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define FK_MAX_TAPS 32 /* flow.cu kMaxTaps: Gaussian half-width limit */
#define FK_MAX_POLY_N 7

typedef struct {
  int radius;
  float k[2 * FK_MAX_TAPS + 1];
} fk_gauss;
typedef struct {
  int n;
  float g[FK_MAX_POLY_N + 1], xg[FK_MAX_POLY_N + 1], xxg[FK_MAX_POLY_N + 1];
  float ig11, ig03, ig33, ig55;
} fk_poly;
typedef struct {
  int w, h, smooth;
  double sigma;
} fk_level;

static int fk_clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
static int fk_reflect101(int p, int len) {
  if (len == 1) return 0;
  while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - 2 - p;
  return p;
}
/* (int)floorf(v) as the GPU converts it (cvt.rmi.s32.f32): saturating, NaN -> 0 */
static int fk_floor_i(float v) {
  if (v != v) return 0;
  v = floorf(v);
  if (v >= 2147483648.f) return INT_MAX;
  if (v <= -2147483648.f) return INT_MIN;
  return (int)v;
}

/* ---- host-side constants: flow.cu make_gauss / make_poly / plan_levels, verbatim ---------------------------- */
static void fk_make_gauss(int ksize, double sigma, fk_gauss* gk) {
  static const float small_tab[4][7] = {{1.f},
                                        {0.25f, 0.5f, 0.25f},
                                        {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f},
                                        {0.03125f, 0.109375f, 0.21875f, 0.28125f, 0.21875f, 0.109375f, 0.03125f}};
  gk->radius = ksize / 2;
  if (sigma <= 0 && (ksize & 1) && ksize <= 7) {
    for (int i = 0; i < ksize; ++i) gk->k[i] = small_tab[ksize >> 1][i];
    return;
  }
  if (sigma <= 0) sigma = ((ksize - 1) * 0.5 - 1) * 0.3 + 0.8;
  const double scale2x = -0.5 / (sigma * sigma);
  double tmp[2 * FK_MAX_TAPS + 1], sum = 0;
  for (int i = 0; i < ksize; ++i) {
    const double x = i - (ksize - 1) * 0.5;
    tmp[i] = exp(scale2x * x * x);
    sum += tmp[i];
  }
  for (int i = 0; i < ksize; ++i) gk->k[i] = (float)(tmp[i] / sum);
}

static void fk_make_poly(int n, double sigma, fk_poly* pk) {
  float g[2 * FK_MAX_POLY_N + 1];
  double s = 0;
  for (int x = -n; x <= n; ++x) {
    g[x + n] = (float)exp(-x * x / (2 * sigma * sigma));
    s += g[x + n];
  }
  s = 1. / s;
  for (int x = -n; x <= n; ++x) g[x + n] = (float)(g[x + n] * s);
  pk->n = n;
  for (int x = 0; x <= n; ++x) {
    pk->g[x] = g[x + n];
    pk->xg[x] = (float)(x * g[x + n]);
    pk->xxg[x] = (float)(x * x * g[x + n]);
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
  pk->ig11 = (float)A[1][7];
  pk->ig03 = (float)A[0][9];
  pk->ig33 = (float)A[3][9];
  pk->ig55 = (float)A[5][11];
}

static int fk_plan_levels(int width, int height, int num_levels, double pyr_scale, fk_level* lv) {
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

/* [w0, h0, w1, h1, ...] of the levels scn_farneback_u8c3 runs, level 0 first; returns the number of levels */
int fbk_levels(int width, int height, int num_levels, double pyr_scale, int* wh) {
  fk_level lv[16];
  const int levels = fk_plan_levels(width, height, num_levels, pyr_scale, lv);
  for (int k = 0; k <= levels; ++k) wh[2 * k] = lv[k].w, wh[2 * k + 1] = lv[k].h;
  return levels + 1;
}

/* ---- the per-pixel stages -------------------------------------------------------------------------------------- */
static void fk_gray(const uint8_t* src, int n, float* dst) { /* gray_kernel */
  for (int i = 0; i < n; ++i) {
    const uint8_t* p = src + (size_t)i * 3;
    dst[i] = (float)((p[0] * 3735 + p[1] * 19235 + p[2] * 9798 + 16384) >> 15);
  }
}

/* gauss_h_kernel then gauss_v_kernel (gauss_fused_kernel: the same taps, 0 .. 2r from 0, on reflected rows) */
static void fk_gauss_blur(const float* src, int w, int h, const fk_gauss* gk, float* tmp, float* dst) {
  const int r = gk->radius;
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      float s = 0.f;
      for (int i = -r; i <= r; ++i) s = fmaf(gk->k[i + r], src[(size_t)y * w + fk_reflect101(x + i, w)], s);
      tmp[(size_t)y * w + x] = s;
    }
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      float s = 0.f;
      for (int i = -r; i <= r; ++i) s = fmaf(gk->k[i + r], tmp[(size_t)fk_reflect101(y + i, h) * w + x], s);
      dst[(size_t)y * w + x] = s;
    }
}

/* resize_f32_kernel<CN> */
static void fk_resize(const float* src, int sw, int sh, float* dst, int dw, int dh, double sx, double sy, float mul,
                      int cn) {
  for (int y = 0; y < dh; ++y) {
    float fy = (float)(((double)y + 0.5) * sy - 0.5);
    int iy = fk_floor_i(fy);
    fy -= (float)iy;
    if (iy < 0) { fy = 0.f; iy = 0; }
    if (iy >= sh - 1) { fy = 0.f; iy = sh - 1; }
    const int iy1 = iy + 1 < sh - 1 ? iy + 1 : sh - 1;
    for (int x = 0; x < dw; ++x) {
      float fx = (float)(((double)x + 0.5) * sx - 0.5);
      int ix = fk_floor_i(fx);
      fx -= (float)ix;
      if (ix < 0) { fx = 0.f; ix = 0; }
      if (ix >= sw - 1) { fx = 0.f; ix = sw - 1; }
      const int ix1 = ix + 1 < sw - 1 ? ix + 1 : sw - 1;
      for (int c = 0; c < cn; ++c) {
        const float a = src[((size_t)iy * sw + ix) * cn + c], b = src[((size_t)iy * sw + ix1) * cn + c];
        const float d = src[((size_t)iy1 * sw + ix) * cn + c], e = src[((size_t)iy1 * sw + ix1) * cn + c];
        const float top = a * (1.f - fx) + b * fx;
        const float bot = d * (1.f - fx) + e * fx;
        dst[((size_t)y * dw + x) * cn + c] = (top * (1.f - fy) + bot * fy) * mul;
      }
    }
  }
}

/* poly_v_kernel + poly_h_kernel (poly_fused_kernel: the same, on a tile of clamped rows and columns); dst5 = 5
 * coefficient planes of w x h */
static void fk_poly_expand(const float* src, int w, int h, const fk_poly* pk, float* t3, float* dst5) {
  const int n = pk->n;
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      float t0 = src[(size_t)y * w + x] * pk->g[0], t1 = 0.f, t2 = 0.f;
      for (int k = 1; k <= n; ++k) {
        const float sp = src[(size_t)fk_clampi(y + k, 0, h - 1) * w + x];
        const float sm = src[(size_t)fk_clampi(y - k, 0, h - 1) * w + x];
        t0 = fmaf(pk->g[k], sp + sm, t0);
        t1 = fmaf(pk->xg[k], sp - sm, t1);
        t2 = fmaf(pk->xxg[k], sp + sm, t2);
      }
      float* d = t3 + ((size_t)y * w + x) * 3;
      d[0] = t0, d[1] = t1, d[2] = t2;
    }
  const size_t ps = (size_t)w * h;
  for (int y = 0; y < h; ++y) {
    const float* row = t3 + (size_t)y * w * 3;
    for (int x = 0; x < w; ++x) {
      const float* c0 = row + (size_t)x * 3;
      float b1 = c0[0] * pk->g[0], b2 = 0.f, b3 = c0[1] * pk->g[0], b4 = 0.f, b5 = c0[2] * pk->g[0], b6 = 0.f;
      for (int k = 1; k <= n; ++k) {
        const float* p = row + (size_t)fk_clampi(x + k, 0, w - 1) * 3;
        const float* m = row + (size_t)fk_clampi(x - k, 0, w - 1) * 3;
        const float tg = p[0] + m[0];
        b1 = fmaf(tg, pk->g[k], b1);
        b2 = fmaf(p[0] - m[0], pk->xg[k], b2);
        b4 = fmaf(tg, pk->xxg[k], b4);
        b3 = fmaf(p[1] + m[1], pk->g[k], b3);
        b6 = fmaf(p[1] - m[1], pk->xg[k], b6);
        b5 = fmaf(p[2] + m[2], pk->g[k], b5);
      }
      float* d = dst5 + (size_t)y * w + x;
      d[1 * ps] = b2 * pk->ig11;
      d[0] = b3 * pk->ig11;
      d[3 * ps] = fmaf(b4, pk->ig33, b1 * pk->ig03);
      d[2 * ps] = fmaf(b5, pk->ig33, b1 * pk->ig03);
      d[4 * ps] = b6 * pk->ig55;
    }
  }
}

/* update_matrices_kernel: R0, R1, M are 5 planes of w x h; flow is (dx, dy) interleaved */
static void fk_update_matrices(const float* R0, const float* R1, const float* flow, int w, int h, float* M) {
  static const float border[5] = {0.14f, 0.14f, 0.4472f, 0.4472f, 0.4472f};
  const int BORDER = 5;
  const size_t ps = (size_t)w * h;
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      const float* r0p = R0 + (size_t)y * w + x;
      const float r0[5] = {r0p[0], r0p[ps], r0p[2 * ps], r0p[3 * ps], r0p[4 * ps]};
      const float dx = flow[((size_t)y * w + x) * 2], dy = flow[((size_t)y * w + x) * 2 + 1];
      float fx = (float)x + dx, fy = (float)y + dy;
      const int x1 = fk_floor_i(fx), y1 = fk_floor_i(fy);
      fx -= (float)x1;
      fy -= (float)y1;
      float r2, r3, r4, r5, r6;
      if ((unsigned)x1 < (unsigned)(w - 1) && (unsigned)y1 < (unsigned)(h - 1)) {
        const float a00 = (1.f - fx) * (1.f - fy), a01 = fx * (1.f - fy), a10 = (1.f - fx) * fy, a11 = fx * fy;
        const float* p = R1 + (size_t)y1 * w + x1;
        const float* q = p + w;
        float rr[5];
        for (int c = 0; c < 5; ++c) {
          float t = fmaf(a00, p[c * ps], a01 * p[c * ps + 1]);
          t = fmaf(a10, q[c * ps], t);
          rr[c] = fmaf(a11, q[c * ps + 1], t);
        }
        r2 = rr[0], r3 = rr[1], r4 = rr[2], r5 = rr[3], r6 = rr[4];
        r4 = (r0[2] + r4) * 0.5f;
        r5 = (r0[3] + r5) * 0.5f;
        r6 = (r0[4] + r6) * 0.25f;
      } else {
        r2 = r3 = 0.f;
        r4 = r0[2];
        r5 = r0[3];
        r6 = r0[4] * 0.5f;
      }
      r2 = r0[0] - r2;
      r3 = r0[1] - r3;
      r2 = fmaf(r2, 0.5f, fmaf(dy, r4, dx * r6));
      r3 = fmaf(r3, 0.5f, fmaf(dx, r5, dy * r6));
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
      m[0] = fmaf(r4, r4, r6 * r6);
      m[ps] = (r4 + r5) * r6;
      m[2 * ps] = fmaf(r5, r5, r6 * r6);
      m[3 * ps] = fmaf(r2, r4, r3 * r6);
      m[4 * ps] = fmaf(r3, r5, r2 * r6);
    }
}

/* solve2x2 */
static void fk_solve(double g11, double g12, double g22, double h1, double h2, float* out) {
  const double idet = 1. / (fma(g11, g22, -(g12 * g12)) + 1e-3);
  out[0] = (float)(fma(g11, h2, -(g12 * h1)) * idet);
  out[1] = (float)(fma(g22, h1, -(g12 * h2)) * idet);
}

/* the window sums of the f32 kernel: e[0 .. taps + 2] are the taps + 3 inputs of a group, o the output in it */
static float fk_tree(const float* e, int taps, int o) {
  float core = e[3];
  for (int k = 4; k < taps; ++k) core += e[k];
  switch (o) {
    case 0: return core + ((e[0] + e[1]) + e[2]);
    case 1: return core + ((e[1] + e[2]) + e[taps]);
    case 2: return core + ((e[2] + e[taps]) + e[taps + 1]);
    default: return core + ((e[taps] + e[taps + 1]) + e[taps + 2]);
  }
}
/* the double sums of the fused kernel: first window of a group direct, then (s + entering) - leaving */
static double fk_slide(const double* v, int taps, int o) {
  double s = 0.0;
  for (int k = 0; k < taps; ++k) s += v[k];
  for (int i = 1; i <= o; ++i) s = (s + v[i + taps - 1]) - v[i - 1];
  return s;
}

/* box average of M (win_size = 2 m + 1 ... or 2 m for even sizes, m = win_size / 2) + the 2x2 solve -> flow */
static void fk_box_solve(const float* M, int w, int h, int win_size, int box, void* scratch, float* flow) {
  const int m = win_size / 2, taps = 2 * m + 1;
  const size_t ps = (size_t)w * h;
  const double scale = 1.0 / ((double)win_size * win_size);
  if (box == 0) { /* box_solve_f32_kernel (m == 7) */
    float* V = (float*)scratch;
    float e[64], hs[5];
    for (int c = 0; c < 5; ++c)
      for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
          const int yb = y & ~3;
          for (int k = 0; k < taps + 3; ++k) e[k] = M[c * ps + (size_t)fk_clampi(yb - m + k, 0, h - 1) * w + x];
          V[c * ps + (size_t)y * w + x] = fk_tree(e, taps, y & 3);
        }
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) {
        const int xb = x & ~3;
        for (int c = 0; c < 5; ++c) {
          for (int k = 0; k < taps + 3; ++k) e[k] = V[c * ps + (size_t)y * w + fk_clampi(xb - m + k, 0, w - 1)];
          hs[c] = fk_tree(e, taps, x & 3);
        }
        fk_solve(hs[0] * scale, hs[1] * scale, hs[2] * scale, hs[3] * scale, hs[4] * scale, flow + ((size_t)y * w + x) * 2);
      }
  } else if (box == 1) { /* box_solve_fused_kernel (m == 7) */
    double* V = (double*)scratch;
    double v[64], hs[5];
    for (int c = 0; c < 5; ++c)
      for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
          const int yb = y & ~3;
          for (int k = 0; k < taps + 3; ++k) v[k] = (double)M[c * ps + (size_t)fk_clampi(yb - m + k, 0, h - 1) * w + x];
          V[c * ps + (size_t)y * w + x] = fk_slide(v, taps, y & 3);
        }
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) {
        const int xb = x & ~3;
        for (int c = 0; c < 5; ++c) {
          for (int k = 0; k < taps + 3; ++k) v[k] = V[c * ps + (size_t)y * w + fk_clampi(xb - m + k, 0, w - 1)];
          hs[c] = fk_slide(v, taps, x & 3);
        }
        fk_solve(hs[0] * scale, hs[1] * scale, hs[2] * scale, hs[3] * scale, hs[4] * scale, flow + ((size_t)y * w + x) * 2);
      }
  } else { /* box_v_kernel + box_h_solve_kernel */
    double* V = (double*)scratch;
    for (int c = 0; c < 5; ++c)
      for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
          double s = 0.0;
          for (int k = -m; k <= m; ++k) s += (double)M[c * ps + (size_t)fk_clampi(y + k, 0, h - 1) * w + x];
          V[c * ps + (size_t)y * w + x] = s;
        }
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) {
        double hs[5] = {0, 0, 0, 0, 0};
        for (int k = -m; k <= m; ++k) {
          const size_t xi = (size_t)fk_clampi(x + k, 0, w - 1);
          for (int c = 0; c < 5; ++c) hs[c] += V[c * ps + (size_t)y * w + xi];
        }
        fk_solve(hs[0] * scale, hs[1] * scale, hs[2] * scale, hs[3] * scale, hs[4] * scale, flow + ((size_t)y * w + x) * 2);
      }
  }
}

/* ---- scn_farneback_u8c3 for one pair ------------------------------------------------------------------------------
 * f0, f1: RGB24 frames (the channel order gray_kernel weighs); out: (h, w, 2) float.  Returns 0, -1 for arguments
 * scn_farneback_u8c3 refuses (SCN_E_BADARG), -2 for a Gaussian over FK_MAX_TAPS (SCN_E_UNSUPPORTED), -3 for a box
 * variant its launcher would not pick (f32 / f64_slide need win_size 15 or 14), -4 out of memory. */
int fbk_flow_u8c3(const uint8_t* f0, const uint8_t* f1, int width, int height, int num_levels, double pyr_scale,
                  int win_size, int num_iters, int poly_n, double poly_sigma, int box, float* out) {
  if (width <= 0 || height <= 0 || num_levels < 0 || num_levels > 15 || pyr_scale <= 0 || pyr_scale >= 1 ||
      win_size < 2 || num_iters < 1 || poly_n < 1 || poly_n > FK_MAX_POLY_N || poly_sigma <= 0)
    return -1;
  if (box < 0 || box > 2 || (box != 2 && win_size / 2 != 7)) return -3;
  fk_level lv[16];
  const int levels = fk_plan_levels(width, height, num_levels, pyr_scale, lv);
  for (int k = 0; k <= levels; ++k)
    if (lv[k].smooth / 2 > FK_MAX_TAPS) return -2;
  fk_poly pk;
  fk_make_poly(poly_n, poly_sigma, &pk);
  const size_t px = (size_t)width * height;
  float* gray[2] = {malloc(px * 4), malloc(px * 4)};
  float *tmp = malloc(px * 4), *blur = malloc(px * 4), *I = malloc(px * 4), *t3 = malloc(px * 12);
  float *R[2] = {malloc(px * 20), malloc(px * 20)}, *M = malloc(px * 20);
  float* fl[2] = {malloc(px * 8), malloc(px * 8)};
  void* scratch = malloc(px * 40);
  int rc = 0;
  if (!gray[0] || !gray[1] || !tmp || !blur || !I || !t3 || !R[0] || !R[1] || !M || !fl[0] || !fl[1] || !scratch) {
    rc = -4;
    goto done;
  }
  fk_gray(f0, (int)px, gray[0]);
  fk_gray(f1, (int)px, gray[1]);
  float* prev = NULL;
  int pw = 0, ph = 0;
  for (int k = levels; k >= 0; --k) {
    const int w = lv[k].w, h = lv[k].h;
    float* flow = k == 0 ? out : (prev == fl[0] ? fl[1] : fl[0]);
    if (!prev)
      memset(flow, 0, (size_t)w * h * 8);
    else
      fk_resize(prev, pw, ph, flow, w, h, (double)pw / w, (double)ph / h, (float)(1. / pyr_scale), 2);
    fk_gauss gk;
    fk_make_gauss(lv[k].smooth, lv[k].sigma, &gk);
    for (int f = 0; f < 2; ++f) {
      fk_gauss_blur(gray[f], width, height, &gk, tmp, blur);
      const float* src = blur;
      if (w != width || h != height) {
        fk_resize(blur, width, height, I, w, h, (double)width / w, (double)height / h, 1.f, 1);
        src = I;
      }
      fk_poly_expand(src, w, h, &pk, t3, R[f]);
    }
    fk_update_matrices(R[0], R[1], flow, w, h, M);
    for (int it = 0; it < num_iters; ++it) {
      fk_box_solve(M, w, h, win_size, box, scratch, flow);
      if (it < num_iters - 1) fk_update_matrices(R[0], R[1], flow, w, h, M);
    }
    prev = flow;
    pw = w;
    ph = h;
  }
done:
  free(gray[0]), free(gray[1]), free(tmp), free(blur), free(I), free(t3), free(R[0]), free(R[1]), free(M);
  free(fl[0]), free(fl[1]), free(scratch);
  return rc;
}
