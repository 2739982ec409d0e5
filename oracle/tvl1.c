/*
 * tvl1.c -- CPU restatement of TV-L1 dense optical flow.  TEST INFRASTRUCTURE ONLY (like scn_oracle.c): nothing in
 * the product path may link, import or call this file.
 *
 * The Zach-Pock-Bischof duality scheme as written out in Sanchez Perez, Meinhardt-Llopis and Facciolo, "TV-L1
 * Optical Flow Estimation" (IPOL 2013), with OpenCV DualTVL1OpticalFlow's parameter names and defaults, gamma = 0.
 * DESIGN.md section 11 is the specification; this is it in plain sequential float32, every expression rounded as
 * written.  scanner_b200/csrc/tvl1.cu evaluates the same expressions in the same order.
 *
 * Build: oracle/tvl1.py compiles it into oracle/libtvl1.so with gcc -O2 -ffp-contract=off -fno-fast-math, the
 * flags of liborc.so (__graft_entry__.build() does so up front).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int tv_clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* cv2.resize(INTER_LINEAR) of a float32 image with an explicit dsize: the map uses OpenCV's
 * scale = 1 / (dsize / ssize) and (d + 0.5) * scale - 0.5, edge taps clamped */
void orc_tvl1_resize_f32(const float* src, int sw, int sh, float* dst, int dw, int dh) {
  const double sx = 1.0 / ((double)dw / sw), sy = 1.0 / ((double)dh / sh);
  for (int y = 0; y < dh; ++y) {
    float fy = (float)((y + 0.5) * sy - 0.5);
    int iy = (int)floorf(fy);
    fy -= (float)iy;
    if (iy < 0) { fy = 0.f; iy = 0; }
    if (iy >= sh - 1) { fy = 0.f; iy = sh - 1; }
    const int iy1 = iy + 1 < sh ? iy + 1 : sh - 1;
    for (int x = 0; x < dw; ++x) {
      float fx = (float)((x + 0.5) * sx - 0.5);
      int ix = (int)floorf(fx);
      fx -= (float)ix;
      if (ix < 0) { fx = 0.f; ix = 0; }
      if (ix >= sw - 1) { fx = 0.f; ix = sw - 1; }
      const int ix1 = ix + 1 < sw ? ix + 1 : sw - 1;
      const float a = src[(size_t)iy * sw + ix], b = src[(size_t)iy * sw + ix1];
      const float d = src[(size_t)iy1 * sw + ix], e = src[(size_t)iy1 * sw + ix1];
      const float top = a * (1.f - fx) + b * fx, bot = d * (1.f - fx) + e * fx;
      dst[(size_t)y * dw + x] = top * (1.f - fy) + bot * fy;
    }
  }
}

/* cv2.medianBlur(float32, k), k = 3 or 5: the median of the k x k window, borders replicated */
void orc_tvl1_median_f32(const float* src, int w, int h, int k, float* dst) {
  const int r = k / 2;
  float win[25];
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      int m = 0;
      for (int dy = -r; dy <= r; ++dy)
        for (int dx = -r; dx <= r; ++dx) {
          const float v = src[(size_t)tv_clampi(y + dy, 0, h - 1) * w + tv_clampi(x + dx, 0, w - 1)];
          int j = m++;
          while (j > 0 && win[j - 1] > v) {
            win[j] = win[j - 1];
            --j;
          }
          win[j] = v;
        }
      dst[(size_t)y * w + x] = win[m / 2];
    }
}

/* Catmull-Rom (Keys, a = -0.5) through v[0..3] at t in [0, 1) between v[1] and v[2] */
static float orc_cubic(const float* v, float t) {
  return v[1] + 0.5f * t * (v[2] - v[0] + t * (2.f * v[0] - 5.f * v[1] + 4.f * v[2] - v[3] +
                                                t * (3.f * (v[1] - v[2]) + v[3] - v[0])));
}

/* separable bicubic of img at (px, py): each of the 4 rows interpolated along x, then the 4 results along y;
 * every tap index clamped into the image.  Positions are first clamped to [-2, w + 1] x [-2, h + 1] (this moves no
 * finite sample: outside that range all taps already clamp to the edge) so NaN and huge values index safely. */
static float orc_bicubic(const float* img, int w, int h, float px, float py) {
  if (!(px >= -2.f)) px = -2.f;
  if (!(px <= (float)(w + 1))) px = (float)(w + 1);
  if (!(py >= -2.f)) py = -2.f;
  if (!(py <= (float)(h + 1))) py = (float)(h + 1);
  const int ix = (int)floorf(px), iy = (int)floorf(py);
  const float tx = px - (float)ix, ty = py - (float)iy;
  float col[4];
  for (int j = 0; j < 4; ++j) {
    const float* row = img + (size_t)tv_clampi(iy - 1 + j, 0, h - 1) * w;
    float v[4];
    for (int i = 0; i < 4; ++i) v[i] = row[tv_clampi(ix - 1 + i, 0, w - 1)];
    col[j] = orc_cubic(v, tx);
  }
  return orc_cubic(col, ty);
}

/* The pyramid of a TV-L1 call: level sizes and count.  Returns the number of levels (>= 1). */
int orc_tvl1_levels(int width, int height, int nscales, float scale_step, int* ws, int* hs) {
  int n = 1;
  ws[0] = width;
  hs[0] = height;
  while (n < nscales) {
    const int w = (int)floor((double)ws[n - 1] * scale_step + 0.5), h = (int)floor((double)hs[n - 1] * scale_step + 0.5);
    if (w < 16 || h < 16) break;
    ws[n] = w;
    hs[n] = h;
    ++n;
  }
  return n;
}

/* lane 0 of a 32-lane __shfl_down_sync tree at offsets 16, 8, 4, 2, 1 (v is overwritten) */
static float tv_lane_tree_f(float* v) {
  for (int o = 16; o > 0; o >>= 1)
    for (int l = 0; l < o; ++l) v[l] += v[l + o];
  return v[0];
}
static double tv_lane_tree_d(double* v) {
  for (int o = 16; o > 0; o >>= 1)
    for (int l = 0; l < o; ++l) v[l] += v[l + o];
  return v[0];
}

/* sum of term[0 .. npx) in tvl1_iterate_kernel's order.  Tile t is pixels [1024 t, 1024 t + 1024); thread x of
 * 256 adds, in float from 0, the terms of pixels 1024 t + 256 j + x (j = 0..3, below npx); each warp of 32 threads
 * is reduced by the lane tree, and the 8 warp sums are added in order from 0 in float.  The tile sums of one pair
 * are then summed in double: thread x adds tiles x, x + 256, ... in order from 0, and the same lane tree and warp
 * order reduce the 256 thread sums. */
double orc_tvl1_tile_sum(const float* term, int npx) {
  const int tiles = (npx + 1023) / 1024;
  double acc[256];
  for (int x = 0; x < 256; ++x) acc[x] = 0.0;
  for (int t = 0; t < tiles; ++t) {
    float e[256];
    for (int x = 0; x < 256; ++x) {
      e[x] = 0.f;
      for (int j = 0; j < 4; ++j) {
        const long i = 1024L * t + 256L * j + x;
        if (i >= npx) break;
        e[x] += term[i];
      }
    }
    float s = 0.f;
    for (int k = 0; k < 8; ++k) s += tv_lane_tree_f(e + 32 * k);
    acc[t % 256] += (double)s;
  }
  double s = 0.0;
  for (int k = 0; k < 8; ++k) s += tv_lane_tree_d(acc + 32 * k);
  return s;
}

/* gray0, gray1: u8 [height][width] -> flow float32 [height][width][2] = (dx, dy).  iters (nullable):
 * int [nscales][warps], level 0 (finest) first, the iterations each (level, warp) ran; 0 for levels the pyramid
 * does not have.  tile_error = 0 sums the stop error sequentially in double (the specification); 1 sums the same
 * float terms as tvl1_iterate_kernel does (orc_tvl1_tile_sum), so that the stop decisions match the kernel's.
 * Arguments are assumed valid (kernels.py / tests check them). */
void orc_tvl1_u8(const uint8_t* gray0, const uint8_t* gray1, int width, int height, float tau, float lambda,
                 float theta, int nscales, int warps, float epsilon, int iterations, float scale_step,
                 int median_filtering, int tile_error, float* flow, int* iters) {
  int lw[16], lh[16];
  const int L = orc_tvl1_levels(width, height, nscales, scale_step, lw, lh);
  if (iters) memset(iters, 0, sizeof(int) * (size_t)nscales * warps);
  const size_t px0 = (size_t)width * height;
  float *I0[16], *I1[16];
  for (int s = 0; s < L; ++s) {
    I0[s] = (float*)malloc(sizeof(float) * (size_t)lw[s] * lh[s]);
    I1[s] = (float*)malloc(sizeof(float) * (size_t)lw[s] * lh[s]);
  }
  for (size_t i = 0; i < px0; ++i) {
    I0[0][i] = (float)gray0[i];
    I1[0][i] = (float)gray1[i];
  }
  for (int s = 1; s < L; ++s) {
    orc_tvl1_resize_f32(I0[s - 1], lw[s - 1], lh[s - 1], I0[s], lw[s], lh[s]);
    orc_tvl1_resize_f32(I1[s - 1], lw[s - 1], lh[s - 1], I1[s], lw[s], lh[s]);
  }
  float* buf[13];
  for (int b = 0; b < 13; ++b) buf[b] = (float*)calloc(px0, sizeof(float));
  float *u1 = buf[0], *u2 = buf[1], *c1 = buf[2], *c2 = buf[3], *Ix = buf[4], *Iy = buf[5], *wx = buf[6],
        *wy = buf[7], *rho_c = buf[8], *p11 = buf[9], *p12 = buf[10], *p21 = buf[11], *p22 = buf[12];
  float* tmp = (float*)malloc(sizeof(float) * px0);
  float* term = tile_error ? (float*)malloc(sizeof(float) * px0) : NULL;
  const float l_t = lambda * theta, taut = tau / theta;
  const double eps2 = epsilon > 0.f ? (double)epsilon * epsilon : -1.0;
  const float up = (float)(1.0 / scale_step);
  for (int s = L - 1; s >= 0; --s) {
    const int w = lw[s], h = lh[s];
    const size_t npx = (size_t)w * h;
    if (s == L - 1) {
      memset(u1, 0, sizeof(float) * npx);
      memset(u2, 0, sizeof(float) * npx);
    } else {  /* c1, c2 hold the coarser level's flow */
      orc_tvl1_resize_f32(c1, lw[s + 1], lh[s + 1], u1, w, h);
      orc_tvl1_resize_f32(c2, lw[s + 1], lh[s + 1], u2, w, h);
      for (size_t i = 0; i < npx; ++i) {
        u1[i] = u1[i] * up;
        u2[i] = u2[i] * up;
      }
    }
    memset(p11, 0, sizeof(float) * npx);
    memset(p12, 0, sizeof(float) * npx);
    memset(p21, 0, sizeof(float) * npx);
    memset(p22, 0, sizeof(float) * npx);
    const float* J = I1[s];
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) {
        const size_t i = (size_t)y * w + x;
        const float xl = J[(size_t)y * w + (x > 0 ? x - 1 : 0)], xr = J[(size_t)y * w + (x < w - 1 ? x + 1 : w - 1)];
        const float yu = J[(size_t)(y > 0 ? y - 1 : 0) * w + x], yd = J[(size_t)(y < h - 1 ? y + 1 : h - 1) * w + x];
        Ix[i] = 0.5f * (x == 0 ? J[i + 1] - J[i] : (x == w - 1 ? J[i] - J[i - 1] : xr - xl));
        Iy[i] = 0.5f * (y == 0 ? J[i + w] - J[i] : (y == h - 1 ? J[i] - J[i - w] : yd - yu));
      }
    for (int wi = 0; wi < warps; ++wi) {
      for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
          const size_t i = (size_t)y * w + x;
          const float px = (float)x + u1[i], py = (float)y + u2[i];
          const float a = orc_bicubic(J, w, h, px, py), gx = orc_bicubic(Ix, w, h, px, py),
                      gy = orc_bicubic(Iy, w, h, px, py);
          wx[i] = gx;
          wy[i] = gy;
          rho_c[i] = a - gx * u1[i] - gy * u2[i] - I0[s][i];
        }
      int n = 0;
      double error = INFINITY;
      while (error > eps2 && n < iterations) {
        ++n;
        double acc = 0.0;
        for (int y = 0; y < h; ++y)
          for (int x = 0; x < w; ++x) {
            const size_t i = (size_t)y * w + x;
            const float gx = wx[i], gy = wy[i], grad = gx * gx + gy * gy;
            const float rho = rho_c[i] + gx * u1[i] + gy * u2[i];
            float d1, d2;
            if (rho < -l_t * grad) {
              d1 = l_t * gx;
              d2 = l_t * gy;
            } else if (rho > l_t * grad) {
              d1 = -l_t * gx;
              d2 = -l_t * gy;
            } else if (grad < 1e-10f) {
              d1 = d2 = 0.f;
            } else {
              const float fi = -rho / grad;
              d1 = fi * gx;
              d2 = fi * gy;
            }
            const float v1 = u1[i] + d1, v2 = u2[i] + d2;
            const float div1 = (p11[i] - (x > 0 ? p11[i - 1] : 0.f)) + (p12[i] - (y > 0 ? p12[i - w] : 0.f));
            const float div2 = (p21[i] - (x > 0 ? p21[i - 1] : 0.f)) + (p22[i] - (y > 0 ? p22[i - w] : 0.f));
            const float n1 = v1 + theta * div1, n2 = v2 + theta * div2;
            const float e1 = n1 - u1[i], e2 = n2 - u2[i];
            const float e = e1 * e1 + e2 * e2;
            if (term)
              term[i] = e;
            else
              acc += (double)e;
            u1[i] = n1;
            u2[i] = n2;
          }
        if (term) acc = orc_tvl1_tile_sum(term, (int)npx);
        error = acc / (double)npx;
        for (int y = 0; y < h; ++y)
          for (int x = 0; x < w; ++x) {
            const size_t i = (size_t)y * w + x;
            const float a1 = x < w - 1 ? u1[i + 1] - u1[i] : 0.f, b1 = y < h - 1 ? u1[i + w] - u1[i] : 0.f;
            const float a2 = x < w - 1 ? u2[i + 1] - u2[i] : 0.f, b2 = y < h - 1 ? u2[i + w] - u2[i] : 0.f;
            const float ng1 = 1.f + taut * sqrtf(a1 * a1 + b1 * b1), ng2 = 1.f + taut * sqrtf(a2 * a2 + b2 * b2);
            p11[i] = (p11[i] + taut * a1) / ng1;
            p12[i] = (p12[i] + taut * b1) / ng1;
            p21[i] = (p21[i] + taut * a2) / ng2;
            p22[i] = (p22[i] + taut * b2) / ng2;
          }
      }
      if (iters) iters[s * warps + wi] = n;
      if (median_filtering > 1) {
        orc_tvl1_median_f32(u1, w, h, median_filtering, tmp);
        memcpy(u1, tmp, sizeof(float) * npx);
        orc_tvl1_median_f32(u2, w, h, median_filtering, tmp);
        memcpy(u2, tmp, sizeof(float) * npx);
      }
    }
    memcpy(c1, u1, sizeof(float) * npx);
    memcpy(c2, u2, sizeof(float) * npx);
  }
  for (size_t i = 0; i < px0; ++i) {
    flow[2 * i] = u1[i];
    flow[2 * i + 1] = u2[i];
  }
  free(tmp);
  free(term);
  for (int b = 0; b < 13; ++b) free(buf[b]);
  for (int s = 0; s < L; ++s) {
    free(I0[s]);
    free(I1[s]);
  }
}
