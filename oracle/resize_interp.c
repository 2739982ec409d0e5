/*
 * resize_interp.c -- CPU restatement of cv::resize's INTER_NEAREST and INTER_AREA on u8 frames.
 *
 * TEST INFRASTRUCTURE ONLY (see scn_oracle.c).  OpenCV (modules/imgproc/src/resize.cpp, 4.x) is restated from its
 * published algorithm, in its order of operations; tests/test_resize_interp_cpu.py holds every function here to live
 * cv2.resize and to SHA-256 hashes of cv2 4.13's output (tests/golden/resize_interp_cv2.json).
 *
 * Scales are OpenCV's: inv_scale = (double)dsz / ssz, scale = 1.0 / inv_scale.
 *
 * INTER_NEAREST: s = min(floor(d * scale), ssz - 1) per axis; a gather.
 *
 * INTER_AREA, three regimes:
 *   1. both scales integers kx, ky >= 1 (resizeAreaFast): int box sums.  kx = ky = 2 rounds half up,
 *      (a + b + c + d + 2) >> 2; every other factor is rint((float)sum * (float)(1.0 / (kx * ky))).
 *   2. both scales >= 1, not both integers (resizeArea): per axis a table of (source index, float alpha) entries
 *      (computeResizeAreaTab).  For each source row of a destination row, in order: buf = 0,
 *      buf = buf + (float)S * alpha over the column entries in order; then sum = beta * buf on the row's first
 *      source row and sum = sum + beta * buf on each later one.  Output rint(sum), saturated.  float32 throughout,
 *      nothing contracted (this file is built with -ffp-contract=off).
 *   3. either scale < 1: INTER_LINEAR's 11-bit fixed point (scn_oracle.c orc_resize_bilinear_u8) with area taps:
 *      s = floor(d * scale), f = (float)((d + 1) - (s + 1) * inv_scale), f = f <= 0 ? 0 : f - floor(f), then the
 *      x axis's zero-weight clamp and the y axis's row clamp as for INTER_LINEAR.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

static uint8_t sat_u8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

ORC_API void orc_resize_nearest_u8(const uint8_t* src, int sw, int sh, int cn, uint8_t* dst, int dw, int dh) {
  const double fx = 1.0 / ((double)dw / sw), fy = 1.0 / ((double)dh / sh);
  for (int y = 0; y < dh; ++y) {
    int sy = (int)floor(y * fy);
    if (sy > sh - 1) sy = sh - 1;
    for (int x = 0; x < dw; ++x) {
      int sx = (int)floor(x * fx);
      if (sx > sw - 1) sx = sw - 1;
      memcpy(dst + ((size_t)y * dw + x) * cn, src + ((size_t)sy * sw + sx) * cn, (size_t)cn);
    }
  }
}

/* computeResizeAreaTab: the entries of destination index d go to idx/alpha[ofs[d] .. ofs[d+1]).  Returns the entry
 * count; with idx == NULL only counts. */
static int area_tab(int ssz, int dsz, double scale, int* ofs, int* idx, float* alpha) {
  int k = 0;
  for (int d = 0; d < dsz; ++d) {
    if (ofs) ofs[d] = k;
    const double fs1 = d * scale, fs2 = fs1 + scale;
    const double cell = scale < ssz - fs1 ? scale : ssz - fs1;
    int s1 = (int)ceil(fs1), s2 = (int)floor(fs2);
    if (s2 > ssz - 1) s2 = ssz - 1;
    if (s1 > s2) s1 = s2;
    if (s1 - fs1 > 1e-3) {
      if (idx) idx[k] = s1 - 1, alpha[k] = (float)((s1 - fs1) / cell);
      ++k;
    }
    for (int s = s1; s < s2; ++s) {
      if (idx) idx[k] = s, alpha[k] = (float)(1.0 / cell);
      ++k;
    }
    if (fs2 - s2 > 1e-3) {
      double w = fs2 - s2 < 1.0 ? fs2 - s2 : 1.0;
      if (cell < w) w = cell;
      if (idx) idx[k] = s2, alpha[k] = (float)(w / cell);
      ++k;
    }
  }
  if (ofs) ofs[dsz] = k;
  return k;
}

static void area_float(const uint8_t* src, int sw, int sh, int cn, uint8_t* dst, int dw, int dh, double sx,
                       double sy) {
  const int nx = area_tab(sw, dw, sx, NULL, NULL, NULL), ny = area_tab(sh, dh, sy, NULL, NULL, NULL);
  int* xo = (int*)malloc(sizeof(int) * (dw + 1));
  int* yo = (int*)malloc(sizeof(int) * (dh + 1));
  int* xi = (int*)malloc(sizeof(int) * (nx + 1));
  int* yi = (int*)malloc(sizeof(int) * (ny + 1));
  float* xa = (float*)malloc(sizeof(float) * (nx + 1));
  float* ya = (float*)malloc(sizeof(float) * (ny + 1));
  float* buf = (float*)malloc(sizeof(float) * dw * cn);
  float* sum = (float*)malloc(sizeof(float) * dw * cn);
  area_tab(sw, dw, sx, xo, xi, xa);
  area_tab(sh, dh, sy, yo, yi, ya);
  for (int y = 0; y < dh; ++y) {
    for (int j = yo[y]; j < yo[y + 1]; ++j) {
      const uint8_t* S = src + (size_t)yi[j] * sw * cn;
      const float beta = ya[j];
      for (int x = 0; x < dw; ++x)
        for (int c = 0; c < cn; ++c) {
          float b = 0.f;
          for (int k = xo[x]; k < xo[x + 1]; ++k) b = b + (float)S[(size_t)xi[k] * cn + c] * xa[k];
          buf[x * cn + c] = b;
        }
      for (int i = 0; i < dw * cn; ++i) sum[i] = j == yo[y] ? beta * buf[i] : sum[i] + beta * buf[i];
    }
    for (int i = 0; i < dw * cn; ++i)
      dst[(size_t)y * dw * cn + i] = yo[y] == yo[y + 1] ? 0 : sat_u8((int)lrintf(sum[i]));
  }
  free(xo), free(yo), free(xi), free(yi), free(xa), free(ya), free(buf), free(sum);
}

static void area_int(const uint8_t* src, int sw, int cn, uint8_t* dst, int dw, int dh, int kx, int ky) {
  const float scale = (float)(1.0 / ((double)kx * ky));
  for (int y = 0; y < dh; ++y)
    for (int x = 0; x < dw; ++x)
      for (int c = 0; c < cn; ++c) {
        int64_t s = 0;
        for (int j = 0; j < ky; ++j)
          for (int i = 0; i < kx; ++i) s += src[((size_t)(y * ky + j) * sw + (size_t)x * kx + i) * cn + c];
        dst[((size_t)y * dw + x) * cn + c] =
            kx == 2 && ky == 2 ? (uint8_t)((s + 2) >> 2) : sat_u8((int)lrintf((float)(int)s * scale));
      }
}

static void area_up_tab(int ssz, int dsz, int clamp_zero, int* ofs, short* coef) {
  const double inv_scale = (double)dsz / ssz, scale = 1.0 / inv_scale;
  for (int d = 0; d < dsz; ++d) {
    int s = (int)floor(d * scale);
    float f = (float)((d + 1) - (s + 1) * inv_scale);
    f = f <= 0 ? 0.f : f - floorf(f);
    if (clamp_zero) {
      if (s < 0) f = 0.f, s = 0;
      if (s >= ssz - 1) f = 0.f, s = ssz - 1;
    }
    ofs[d] = s;
    coef[2 * d] = (short)lrintf((1.f - f) * 2048.f);
    coef[2 * d + 1] = (short)lrintf(f * 2048.f);
  }
}

static void area_up(const uint8_t* src, int sw, int sh, int cn, uint8_t* dst, int dw, int dh) {
  int* xo = (int*)malloc(sizeof(int) * dw);
  int* yo = (int*)malloc(sizeof(int) * dh);
  short* xa = (short*)malloc(sizeof(short) * 2 * dw);
  short* yb = (short*)malloc(sizeof(short) * 2 * dh);
  area_up_tab(sw, dw, 1, xo, xa);
  area_up_tab(sh, dh, 0, yo, yb);
  for (int y = 0; y < dh; ++y) {
    int r0 = yo[y], r1 = yo[y] + 1;
    r0 = r0 < 0 ? 0 : (r0 > sh - 1 ? sh - 1 : r0);
    r1 = r1 < 0 ? 0 : (r1 > sh - 1 ? sh - 1 : r1);
    const uint8_t* s0 = src + (size_t)r0 * sw * cn;
    const uint8_t* s1 = src + (size_t)r1 * sw * cn;
    for (int x = 0; x < dw; ++x) {
      const int x0 = xo[x], x1 = x0 + 1 < sw ? x0 + 1 : sw - 1;
      for (int c = 0; c < cn; ++c) {
        const int h0 = s0[x0 * cn + c] * xa[2 * x] + s0[x1 * cn + c] * xa[2 * x + 1];
        const int h1 = s1[x0 * cn + c] * xa[2 * x] + s1[x1 * cn + c] * xa[2 * x + 1];
        const int v = (((yb[2 * y] * (h0 >> 4)) >> 16) + ((yb[2 * y + 1] * (h1 >> 4)) >> 16) + 2) >> 2;
        dst[((size_t)y * dw + x) * cn + c] = sat_u8(v);
      }
    }
  }
  free(xo), free(yo), free(xa), free(yb);
}

ORC_API void orc_resize_area_u8(const uint8_t* src, int sw, int sh, int cn, uint8_t* dst, int dw, int dh) {
  const double sx = 1.0 / ((double)dw / sw), sy = 1.0 / ((double)dh / sh);
  if (sx < 1 || sy < 1)
    area_up(src, sw, sh, cn, dst, dw, dh);
  else if (sw % dw == 0 && sh % dh == 0)
    area_int(src, sw, cn, dst, dw, dh, sw / dw, sh / dh);
  else
    area_float(src, sw, sh, cn, dst, dw, dh, sx, sy);
}
