/*
 * scn_oracle.c -- CPU restatement of the reference's per-frame pixel ops.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (scanner_b200/, the
 * C-ABI in include/) may link, import or call this file.  It exists so that
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg can check the
 * CUDA path against an independent scalar implementation.
 *
 * Every function cites the reference file:line it follows (paths relative to
 * the scanner-research/scanner tree).  The pixel arithmetic of Histogram and
 * Resize lives in OpenCV (pinned 4.2.0 by the reference's deps.sh:643), which
 * is not vendored: those two functions restate OpenCV's published algorithm and
 * are pinned against cv2 outputs committed under tests/golden/ (see
 * oracle/make_golden.py).  Blur and NV12->RGB are fully open-coded in the
 * reference and are restated from its source directly.
 *
 * Build: see oracle/Makefile (plain gcc, -ffp-contract=off so that float
 * expressions round exactly as written).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------- */
/* Histogram -- tests/test_ops.cpp:13-59.
 * cv::calcHist(&img,1,{j},Mat(),hist,1,&BINS(16),range [0,256)) per channel j,
 * converted to CV_32S.  With 16 uniform bins over [0,256) the bin of an 8-bit
 * value v is floor(v * 16 / 256) == v >> 4.  Output layout: int32[3][16],
 * channel-major (test_ops.cpp:40-42: output_buf + j*BINS*sizeof(int)). */
ORC_API void orc_hist16_u8c3(const uint8_t* frame, int width, int height,
                             int32_t* out48) {
  memset(out48, 0, 48 * sizeof(int32_t));
  size_t npix = (size_t)width * (size_t)height;
  for (size_t p = 0; p < npix; ++p) {
    out48[0 * 16 + (frame[3 * p + 0] >> 4)]++;
    out48[1 * 16 + (frame[3 * p + 1] >> 4)]++;
    out48[2 * 16 + (frame[3 * p + 2] >> 4)]++;
  }
}

/* ------------------------------------------------------------------------- */
/* Resize target size -- tests/test_ops.cpp:126-147 (ResizeKernel::execute).
 * width/height/min/preserve_aspect are the ResizeArgs fields
 * (tests/test_ops.proto:8-14); the interpolation string is ignored by the
 * reference (test_ops.cpp:156 calls cv::resize with the default). */
ORC_API void orc_resize_target(int src_w, int src_h, int arg_w, int arg_h,
                               int arg_min, int arg_preserve_aspect,
                               int* out_w, int* out_h) {
  int tw = arg_w, th = arg_h;
  if (arg_preserve_aspect) {
    if (tw == 0) {
      tw = src_w * th / src_h;
    } else {
      th = src_h * tw / src_w;
    }
  }
  if (arg_min) {
    if (src_w <= tw && src_h <= th) {
      tw = src_w;
      th = src_h;
    }
  }
  *out_w = tw;
  *out_h = th;
}

/* ------------------------------------------------------------------------- */
/* Resize -- tests/test_ops.cpp:156: cv::resize(img, out, Size(w,h)) i.e.
 * INTER_LINEAR on CV_8UC3.  OpenCV (modules/imgproc/src/resize.cpp, 4.x):
 *   - if both scale factors are exactly 2 the call is re-routed to the
 *     INTER_AREA fast path: (a+b+c+d+2)>>2 over each 2x2 block;
 *   - otherwise: per destination column dx
 *        fx = (float)((dx+0.5)*scale_x - 0.5); sx = floor(fx); fx -= sx;
 *        sx<0 -> (sx,fx)=(0,0); sx>=sw-1 -> (sx,fx)=(sw-1,0)
 *        alpha = { rint((1.f-fx)*2048), rint(fx*2048) }   (saturate_cast<short>)
 *     per destination row dy the same WITHOUT the clamp-with-zeroed-weight:
 *        sy = floor(fy), beta from fy, and the two source rows are
 *        clip(sy,0,sh-1), clip(sy+1,0,sh-1);
 *     horizontal pass in int:  H = S[sx]*a0 + S[sx+1]*a1      (scale 2^11)
 *     vertical pass (u8 specialisation, identical in the SIMD and scalar tails):
 *        D = ( ((b0*(H0>>4))>>16) + ((b1*(H1>>4))>>16) + 2 ) >> 2
 * Pinned bit-exact against cv2.resize 4.13.0 for up- and down-scales
 * (tests/golden/resize_*.npz). */
static void orc_linear_tab(int ssz, int dsz, int clamp_zero, int* ofs,
                           short* coef /* 2 per entry */) {
  double inv_scale = (double)dsz / (double)ssz;
  double scale = 1.0 / inv_scale;
  for (int d = 0; d < dsz; ++d) {
    float f = (float)((d + 0.5) * scale - 0.5);
    int s = (int)floorf(f);
    f -= (float)s;
    if (clamp_zero) {
      if (s < 0) {
        f = 0.f;
        s = 0;
      }
      if (s >= ssz - 1) {
        f = 0.f;
        s = ssz - 1;
      }
    }
    ofs[d] = s;
    float c0 = (1.f - f) * 2048.f;
    float c1 = f * 2048.f;
    coef[2 * d + 0] = (short)lrintf(c0);
    coef[2 * d + 1] = (short)lrintf(c1);
  }
}

ORC_API void orc_resize_bilinear_u8(const uint8_t* src, int sw, int sh, int cn,
                                    uint8_t* dst, int dw, int dh) {
  if (dw <= 0 || dh <= 0) return;
  if (sw == 2 * dw && sh == 2 * dh) {
    for (int y = 0; y < dh; ++y) {
      const uint8_t* r0 = src + (size_t)(2 * y) * sw * cn;
      const uint8_t* r1 = r0 + (size_t)sw * cn;
      for (int x = 0; x < dw; ++x)
        for (int c = 0; c < cn; ++c) {
          int v = r0[(2 * x) * cn + c] + r0[(2 * x + 1) * cn + c] +
                  r1[(2 * x) * cn + c] + r1[(2 * x + 1) * cn + c];
          dst[((size_t)y * dw + x) * cn + c] = (uint8_t)((v + 2) >> 2);
        }
    }
    return;
  }
  int* xofs = (int*)malloc(sizeof(int) * dw);
  int* yofs = (int*)malloc(sizeof(int) * dh);
  short* xa = (short*)malloc(sizeof(short) * 2 * dw);
  short* yb = (short*)malloc(sizeof(short) * 2 * dh);
  int* row0 = (int*)malloc(sizeof(int) * dw * cn);
  int* row1 = (int*)malloc(sizeof(int) * dw * cn);
  orc_linear_tab(sw, dw, 1, xofs, xa);
  orc_linear_tab(sh, dh, 0, yofs, yb);
  for (int y = 0; y < dh; ++y) {
    int sy0 = yofs[y], sy1 = yofs[y] + 1;
    if (sy0 < 0) sy0 = 0;
    if (sy0 > sh - 1) sy0 = sh - 1;
    if (sy1 < 0) sy1 = 0;
    if (sy1 > sh - 1) sy1 = sh - 1;
    const uint8_t* s0 = src + (size_t)sy0 * sw * cn;
    const uint8_t* s1 = src + (size_t)sy1 * sw * cn;
    for (int x = 0; x < dw; ++x) {
      int sx0 = xofs[x];
      int sx1 = sx0 + 1 < sw ? sx0 + 1 : sw - 1;
      int a0 = xa[2 * x], a1 = xa[2 * x + 1];
      for (int c = 0; c < cn; ++c) {
        row0[x * cn + c] = s0[sx0 * cn + c] * a0 + s0[sx1 * cn + c] * a1;
        row1[x * cn + c] = s1[sx0 * cn + c] * a0 + s1[sx1 * cn + c] * a1;
      }
    }
    int b0 = yb[2 * y], b1 = yb[2 * y + 1];
    uint8_t* d = dst + (size_t)y * dw * cn;
    for (int i = 0; i < dw * cn; ++i) {
      d[i] = (uint8_t)((((b0 * (row0[i] >> 4)) >> 16) +
                        ((b1 * (row1[i] >> 4)) >> 16) + 2) >>
                       2);
    }
  }
  free(xofs);
  free(yofs);
  free(xa);
  free(yb);
  free(row0);
  free(row1);
}

/* ------------------------------------------------------------------------- */
/* Blur -- tests/test_ops.cpp:239-310.  A box filter (sigma is parsed and never
 * used): filter_left = ceil(k/2.0)-1, filter_right = k/2 (:252-253); only
 * interior pixels y in [fl, H-fr), x in [fl, W-fr) are written (:278-279) with
 * value = (sum over the (fl+fr+1)^2 window as u32) / ((fl+fr+1)^2) (integer
 * division, :288-290).  The reference leaves the border of its freshly
 * allocated output frame UNINITIALISED; this restatement (and the CUDA path)
 * defines the border as 0 -- parity is claimed on the interior only. */
ORC_API void orc_blur_u8c3(const uint8_t* src, int width, int height,
                           int kernel_size, uint8_t* dst) {
  int fl = (int)ceil(kernel_size / 2.0) - 1;
  int fr = kernel_size / 2;
  memset(dst, 0, (size_t)width * height * 3);
  uint32_t div = (uint32_t)((fr + fl + 1) * (fr + fl + 1));
  for (int y = fl; y < height - fr; ++y)
    for (int x = fl; x < width - fr; ++x)
      for (int c = 0; c < 3; ++c) {
        uint32_t value = 0;
        for (int ry = -fl; ry < fr + 1; ++ry)
          for (int rx = -fl; rx < fr + 1; ++rx)
            value += src[((size_t)(y + ry) * width + (x + rx)) * 3 + c];
        dst[((size_t)y * width + x) * 3 + c] = (uint8_t)(value / div);
      }
}

/* ------------------------------------------------------------------------- */
/* NV12 -> RGB24 -- scanner/util/image.cu:67-102 (matrix, clamp, pack) and
 * :109-200 (pixel fetch, odd-row chroma averaging).
 *   Y' = Y<<2;  C' = (C<<2) - 512 with, on odd luma rows that are not in the
 *   last chroma row, C = (C[r] + C[r+1] + 1) >> 1   (:133-151)
 *   R = Y'*1.1644 + Cb'*0      + Cr'*1.596
 *   G = Y'*1.1644 + Cb'*-.3918 + Cr'*-.813
 *   B = Y'*1.1644 + Cb'*2.0172 + Cr'*0
 *   clamp to [0,1023], truncate to uint, >>2   (:92-102)
 * The reference is CUDA source compiled by nvcc with its default -fmad=true.
 * oracle/_ref builds that source UNMODIFIED (oracle/Makefile, nvcc 12.9, sm_90a);
 * its SASS evaluates `a*b + c*d + e*f` as  fma(e,f, fma(a,b, fl(c*d)))  -- the
 * MIDDLE product is the one rounded on its own (FMUL cb*k1; FFMA luma,k0; FFMA
 * cr,k2).  That order is written out explicitly here, and
 * tests/golden/nv12_ref.npz holds that kernel's output over all 2^24 (Y,Cb,Cr)
 * triples (run on an H100), and tests/test_oracle_golden.py asserts equality with this function.
 * (There is no -16 luma offset in the reference, :74.) */
static inline uint8_t orc_pack10(float v) {
  v = fminf(fmaxf(v, 0.0f), 1023.f);
  return (uint8_t)(((uint32_t)v) >> 2);
}

ORC_API void orc_nv12_to_rgb24(const uint8_t* luma, const uint8_t* chroma,
                               size_t pitch, int width, int height,
                               uint8_t* rgb, size_t rgb_pitch) {
  for (int y = 0; y < height; ++y) {
    int yc = y >> 1;
    for (int x = 0; x < width; ++x) {
      int xc = x & ~1;
      uint32_t cb = chroma[(size_t)yc * pitch + xc];
      uint32_t cr = chroma[(size_t)yc * pitch + xc + 1];
      if ((y & 1) && yc < ((height >> 1) - 1)) {
        cb = (cb + chroma[(size_t)(yc + 1) * pitch + xc] + 1) >> 1;
        cr = (cr + chroma[(size_t)(yc + 1) * pitch + xc + 1] + 1) >> 1;
      }
      float l = (float)((uint32_t)luma[(size_t)y * pitch + x] << 2);
      float fcb = (float)((int)(cb << 2) - 512);
      float fcr = (float)((int)(cr << 2) - 512);
      float r = fmaf(fcr, 1.596f, fmaf(l, 1.1644f, fcb * 0.0f));
      float g = fmaf(fcr, -0.813f, fmaf(l, 1.1644f, fcb * -0.3918f));
      float b = fmaf(fcr, 0.0f, fmaf(l, 1.1644f, fcb * 2.0172f));
      uint8_t* o = rgb + (size_t)y * rgb_pitch + (size_t)x * 3;
      o[0] = orc_pack10(r);
      o[1] = orc_pack10(g);
      o[2] = orc_pack10(b);
    }
  }
}

/* ------------------------------------------------------------------------- */
/* The C2 DAG of BASELINE.json configs[1] on one decoded surface:
 * NV12 -> RGB24 -> { Histogram, Resize(dw,dh) }.  Restated as the plain
 * composition of the three functions above (that is what the reference's
 * pipeline does: decoder output column feeds both ops,
 * scanner/engine/evaluate_worker.cpp:710-1261). */
ORC_API void orc_nv12_hist_resize(const uint8_t* luma, const uint8_t* chroma,
                                  size_t pitch, int width, int height,
                                  int32_t* out48, uint8_t* resized, int dw,
                                  int dh, uint8_t* scratch_rgb) {
  orc_nv12_to_rgb24(luma, chroma, pitch, width, height, scratch_rgb,
                    (size_t)width * 3);
  orc_hist16_u8c3(scratch_rgb, width, height, out48);
  if (resized) orc_resize_bilinear_u8(scratch_rgb, width, height, 3, resized, dw, dh);
}

/* Index column -- scanner/engine/ingest.cpp:337-345: row i is the
 * little-endian int64 i. */
ORC_API void orc_index_column(int64_t start, int64_t n, uint8_t* out) {
  for (int64_t i = 0; i < n; ++i) {
    uint64_t v = (uint64_t)(start + i);
    for (int b = 0; b < 8; ++b) out[i * 8 + b] = (uint8_t)(v >> (8 * b));
  }
}

/* ------------------------------------------------------------------------- */
/* OpticalFlow -- tests/test_ops.cpp:63-111: stencil {0,1};
 *   cvtColor(frame, gray, COLOR_BGR2GRAY) applied to the decoder's RGB data (:91-92), so
 *     gray = (ch0*3735 + ch1*19235 + ch2*9798 + 16384) >> 15       (OpenCV's 15-bit fixed point)
 *   cv::FarnebackOpticalFlow::create(numLevels=3, pyrScale=0.5, fastPyramids=false, winSize=15,
 *     numIters=3, polyN=5, polySigma=1.2, flags=0)->calc(gray0, gray1, flow)   (:68-69, :94)
 * The Farneback arithmetic lives in OpenCV (modules/video/src/optflowgf.cpp); this is a
 * restatement of that published algorithm in float, pinned against cv2.calcOpticalFlowFarneback
 * within a tolerance (tests/golden/flow_cv2.npz): float summation order differs from OpenCV's
 * SIMD code, so parity is NOT bit-exact (stated tolerance: see tests/test_oracle_golden.py). */
ORC_API void orc_bgr2gray_u8c3(const uint8_t* src, int width, int height, uint8_t* gray) {
  size_t n = (size_t)width * height;
  for (size_t i = 0; i < n; ++i)
    gray[i] = (uint8_t)((src[3 * i] * 3735 + src[3 * i + 1] * 19235 + src[3 * i + 2] * 9798 + 16384) >> 15);
}

static int orc_round(double v) { return (int)lrint(v); }
static int orc_clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
/* OpenCV BORDER_REFLECT_101 index */
static int orc_reflect101(int p, int len) {
  if (len == 1) return 0;
  while (p < 0 || p >= len) {
    if (p < 0) p = -p;
    else p = 2 * len - 2 - p;
  }
  return p;
}

/* cv::getGaussianKernel(ksize, sigma, CV_32F) (imgproc/smooth: sigma<=0 -> 0.3*((ksize-1)*0.5-1)+0.8) */
static void orc_gauss_kernel(int ksize, double sigma, float* k) {
  /* cv::getGaussianKernel: odd ksize <= 7 with sigma <= 0 uses a fixed table */
  static const float small_tab[4][7] = {{1.f},
                                        {0.25f, 0.5f, 0.25f},
                                        {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f},
                                        {0.03125f, 0.109375f, 0.21875f, 0.28125f, 0.21875f, 0.109375f, 0.03125f}};
  if (sigma <= 0 && (ksize & 1) && ksize <= 7) {
    for (int i = 0; i < ksize; ++i) k[i] = small_tab[ksize >> 1][i];
    return;
  }
  if (sigma <= 0) sigma = ((ksize - 1) * 0.5 - 1) * 0.3 + 0.8;
  double scale2x = -0.5 / (sigma * sigma), sum = 0;
  double* tmp = (double*)malloc(sizeof(double) * (size_t)ksize);
  for (int i = 0; i < ksize; ++i) {
    double x = i - (ksize - 1) * 0.5;
    tmp[i] = exp(scale2x * x * x);
    sum += tmp[i];
  }
  for (int i = 0; i < ksize; ++i) k[i] = (float)(tmp[i] / sum);
  free(tmp);
}

/* GaussianBlur on float, separable, BORDER_REFLECT_101 (OpenCV default) */
/* (ksize grows with the pyramid depth: 79 taps at level 5 of pyr_scale 0.5, so the taps are sized to it) */
static void orc_gaussian_blur_f32(const float* src, int w, int h, int ksize, double sigma, float* dst) {
  float* k = (float*)malloc(sizeof(float) * (size_t)ksize);
  orc_gauss_kernel(ksize, sigma, k);
  int r = ksize / 2;
  float* tmp = (float*)malloc(sizeof(float) * (size_t)w * h);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      float s = 0;
      for (int i = -r; i <= r; ++i) s += k[i + r] * src[(size_t)y * w + orc_reflect101(x + i, w)];
      tmp[(size_t)y * w + x] = s;
    }
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      float s = 0;
      for (int i = -r; i <= r; ++i) s += k[i + r] * tmp[(size_t)orc_reflect101(y + i, h) * w + x];
      dst[(size_t)y * w + x] = s;
    }
  free(tmp);
  free(k);
}

/* cv::resize INTER_LINEAR for float images, cn channels (half-pixel centres, edge clamp) */
static void orc_resize_linear_f32(const float* src, int sw, int sh, int cn, float* dst, int dw, int dh) {
  double sx = (double)sw / dw, sy = (double)sh / dh;
  for (int y = 0; y < dh; ++y) {
    float fy = (float)((y + 0.5) * sy - 0.5);
    int iy = (int)floorf(fy);
    fy -= iy;
    if (iy < 0) { fy = 0; iy = 0; }
    if (iy >= sh - 1) { fy = 0; iy = sh - 1; }
    int iy1 = iy + 1 < sh ? iy + 1 : sh - 1;
    for (int x = 0; x < dw; ++x) {
      float fx = (float)((x + 0.5) * sx - 0.5);
      int ix = (int)floorf(fx);
      fx -= ix;
      if (ix < 0) { fx = 0; ix = 0; }
      if (ix >= sw - 1) { fx = 0; ix = sw - 1; }
      int ix1 = ix + 1 < sw ? ix + 1 : sw - 1;
      for (int c = 0; c < cn; ++c) {
        float a = src[((size_t)iy * sw + ix) * cn + c], b = src[((size_t)iy * sw + ix1) * cn + c];
        float d = src[((size_t)iy1 * sw + ix) * cn + c], e = src[((size_t)iy1 * sw + ix1) * cn + c];
        float top = a * (1.f - fx) + b * fx, bot = d * (1.f - fx) + e * fx;
        dst[((size_t)y * dw + x) * cn + c] = top * (1.f - fy) + bot * fy;
      }
    }
  }
}

/* FarnebackPrepareGaussian + FarnebackPolyExp: per pixel 5 coefficients
 * [0]=b3*ig11 (d/dy), [1]=b2*ig11 (d/dx), [2]=b1*ig03+b5*ig33 (yy), [3]=b1*ig03+b4*ig33 (xx), [4]=b6*ig55 (xy) */
static void orc_poly_exp(const float* src, int w, int h, int n, double sigma, float* dst) {
  float g[16], xg[16], xxg[16];
  double s = 0;
  for (int x = -n; x <= n; ++x) {
    g[x + n] = (float)exp(-x * x / (2 * sigma * sigma));
    s += g[x + n];
  }
  s = 1. / s;
  for (int x = -n; x <= n; ++x) {
    g[x + n] = (float)(g[x + n] * s);
    xg[x + n] = (float)(x * g[x + n]);
    xxg[x + n] = (float)(x * x * g[x + n]);
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
  /* invert the 6x6 (Gauss-Jordan; the matrix is SPD) */
  double A[6][12];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 12; ++j) A[i][j] = j < 6 ? G[i][j] : (j - 6 == i ? 1.0 : 0.0);
  for (int c = 0; c < 6; ++c) {
    int p = c;
    for (int r2 = c + 1; r2 < 6; ++r2)
      if (fabs(A[r2][c]) > fabs(A[p][c])) p = r2;
    if (p != c)
      for (int j = 0; j < 12; ++j) { double t = A[c][j]; A[c][j] = A[p][j]; A[p][j] = t; }
    double d = A[c][c];
    for (int j = 0; j < 12; ++j) A[c][j] /= d;
    for (int r2 = 0; r2 < 6; ++r2)
      if (r2 != c) {
        double f = A[r2][c];
        for (int j = 0; j < 12; ++j) A[r2][j] -= f * A[c][j];
      }
  }
  double ig11 = A[1][7], ig03 = A[0][9], ig33 = A[3][9], ig55 = A[5][11];

  float* row = (float*)malloc(sizeof(float) * (size_t)(w + 2 * n) * 3);
  float* rc = row + n * 3;
  for (int y = 0; y < h; ++y) {
    const float* s0 = src + (size_t)y * w;
    for (int x = 0; x < w; ++x) {
      float g0 = g[n];
      float t0 = s0[x] * g0, t1 = 0, t2 = 0;
      for (int k = 1; k <= n; ++k) {
        const float* sp = src + (size_t)orc_clampi(y + k, 0, h - 1) * w;
        const float* sm = src + (size_t)orc_clampi(y - k, 0, h - 1) * w;
        float gk = g[n + k], xgk = xg[n + k], xxgk = xxg[n + k];
        t0 += gk * (sp[x] + sm[x]);
        t1 += xgk * (sp[x] - sm[x]);
        t2 += xxgk * (sp[x] + sm[x]);
      }
      rc[x * 3] = t0;
      rc[x * 3 + 1] = t1;
      rc[x * 3 + 2] = t2;
    }
    for (int x = 0; x < n * 3; ++x) {
      rc[-1 - x] = rc[2 - (x % 3)];
      rc[w * 3 + x] = rc[(w - 1) * 3 + (x % 3)];
    }
    float* d = dst + (size_t)y * w * 5;
    for (int x = 0; x < w; ++x) {
      float g0 = g[n];
      double b1 = rc[x * 3] * g0, b2 = 0, b3 = rc[x * 3 + 1] * g0, b4 = 0, b5 = rc[x * 3 + 2] * g0, b6 = 0;
      for (int k = 1; k <= n; ++k) {
        double tg = rc[(x + k) * 3] + rc[(x - k) * 3];
        b1 += tg * g[n + k];
        b2 += (rc[(x + k) * 3] - rc[(x - k) * 3]) * xg[n + k];
        b4 += tg * xxg[n + k];
        b3 += (rc[(x + k) * 3 + 1] + rc[(x - k) * 3 + 1]) * g[n + k];
        b6 += (rc[(x + k) * 3 + 1] - rc[(x - k) * 3 + 1]) * xg[n + k];
        b5 += (rc[(x + k) * 3 + 2] + rc[(x - k) * 3 + 2]) * g[n + k];
      }
      d[x * 5 + 1] = (float)(b2 * ig11);
      d[x * 5] = (float)(b3 * ig11);
      d[x * 5 + 3] = (float)(b1 * ig03 + b4 * ig33);
      d[x * 5 + 2] = (float)(b1 * ig03 + b5 * ig33);
      d[x * 5 + 4] = (float)(b6 * ig55);
    }
  }
  free(row);
}

static void orc_update_matrices(const float* R0, const float* R1, const float* flow, int w, int h, float* M) {
  static const float border[5] = {0.14f, 0.14f, 0.4472f, 0.4472f, 0.4472f};
  const int BORDER = 5;
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      const float* r0 = R0 + ((size_t)y * w + x) * 5;
      float dx = flow[((size_t)y * w + x) * 2], dy = flow[((size_t)y * w + x) * 2 + 1];
      float fx = x + dx, fy = y + dy;
      int x1 = (int)floorf(fx), y1 = (int)floorf(fy);
      float r2, r3, r4, r5, r6;
      fx -= x1;
      fy -= y1;
      if ((unsigned)x1 < (unsigned)(w - 1) && (unsigned)y1 < (unsigned)(h - 1)) {
        float a00 = (1.f - fx) * (1.f - fy), a01 = fx * (1.f - fy), a10 = (1.f - fx) * fy, a11 = fx * fy;
        const float* p = R1 + ((size_t)y1 * w + x1) * 5;
        const float* q = p + (size_t)w * 5;
        r2 = a00 * p[0] + a01 * p[5] + a10 * q[0] + a11 * q[5];
        r3 = a00 * p[1] + a01 * p[6] + a10 * q[1] + a11 * q[6];
        r4 = a00 * p[2] + a01 * p[7] + a10 * q[2] + a11 * q[7];
        r5 = a00 * p[3] + a01 * p[8] + a10 * q[3] + a11 * q[8];
        r6 = a00 * p[4] + a01 * p[9] + a10 * q[4] + a11 * q[9];
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
        float scale = (x < BORDER ? border[x] : 1.f) * (x >= w - BORDER ? border[w - x - 1] : 1.f) *
                      (y < BORDER ? border[y] : 1.f) * (y >= h - BORDER ? border[h - y - 1] : 1.f);
        r2 *= scale; r3 *= scale; r4 *= scale; r5 *= scale; r6 *= scale;
      }
      float* m = M + ((size_t)y * w + x) * 5;
      m[0] = r4 * r4 + r6 * r6;
      m[1] = (r4 + r5) * r6;
      m[2] = r5 * r5 + r6 * r6;
      m[3] = r4 * r2 + r6 * r3;
      m[4] = r6 * r2 + r5 * r3;
    }
}

/* FarnebackUpdateFlow_Blur: box filter of M (window block_size, replicated borders), 2x2 solve */
static void orc_update_flow_blur(const float* M, int w, int h, int block_size, float* flow) {
  int m = block_size / 2;
  double scale = 1.0 / (block_size * block_size);
  double* vsum = (double*)malloc(sizeof(double) * (size_t)(w + 2 * m + 2) * 5);
  for (int y = 0; y < h; ++y) {
    double* vs = vsum + (m + 1) * 5;
    for (int x = 0; x < w * 5; ++x) {
      double s = 0;
      for (int k = -m; k <= m; ++k) s += M[(size_t)orc_clampi(y + k, 0, h - 1) * w * 5 + x];
      vs[x] = s;
    }
    for (int x = 0; x < (m + 1) * 5; ++x) {
      vs[-1 - x] = vs[4 - (x % 5)];
      vs[w * 5 + x] = vs[(w - 1) * 5 + (x % 5)];
    }
    for (int x = 0; x < w; ++x) {
      double hs[5] = {0, 0, 0, 0, 0};
      for (int k = -m; k <= m; ++k)
        for (int c = 0; c < 5; ++c) hs[c] += vs[(x + k) * 5 + c];
      double g11 = hs[0] * scale, g12 = hs[1] * scale, g22 = hs[2] * scale, h1 = hs[3] * scale, h2 = hs[4] * scale;
      double idet = 1. / (g11 * g22 - g12 * g12 + 1e-3);
      flow[((size_t)y * w + x) * 2] = (float)((g11 * h2 - g12 * h1) * idet);
      flow[((size_t)y * w + x) * 2 + 1] = (float)((g22 * h1 - g12 * h2) * idet);
    }
  }
  free(vsum);
}

ORC_API void orc_farneback_u8(const uint8_t* prev, const uint8_t* next, int width, int height, int num_levels,
                              double pyr_scale, int win_size, int num_iters, int poly_n, double poly_sigma,
                              float* flow_out) {
  const int min_size = 32;
  int levels = num_levels, k;
  double scale = 1;
  for (k = 0; k < levels; ++k) {
    scale *= pyr_scale;
    if (width * scale < min_size || height * scale < min_size) break;
  }
  levels = k;
  float* prev_flow = NULL;
  int pw = 0, ph = 0;
  size_t full = (size_t)width * height;
  float* fimg = (float*)malloc(sizeof(float) * full);
  float* blurred = (float*)malloc(sizeof(float) * full);
  for (k = levels; k >= 0; --k) {
    scale = 1;
    for (int i = 0; i < k; ++i) scale *= pyr_scale;
    double sigma = (1. / scale - 1) * 0.5;
    int smooth_sz = orc_round(sigma * 5) | 1;
    if (smooth_sz < 3) smooth_sz = 3;
    int w = orc_round(width * scale), h = orc_round(height * scale);
    float* flow = k > 0 ? (float*)malloc(sizeof(float) * (size_t)w * h * 2) : flow_out;
    if (!prev_flow) {
      memset(flow, 0, sizeof(float) * (size_t)w * h * 2);
    } else {
      orc_resize_linear_f32(prev_flow, pw, ph, 2, flow, w, h);
      float mul = (float)(1. / pyr_scale);
      for (size_t i = 0; i < (size_t)w * h * 2; ++i) flow[i] *= mul;
    }
    float* R[2];
    float* I = (float*)malloc(sizeof(float) * (size_t)w * h);
    for (int i = 0; i < 2; ++i) {
      const uint8_t* img = i == 0 ? prev : next;
      for (size_t p = 0; p < full; ++p) fimg[p] = (float)img[p];
      orc_gaussian_blur_f32(fimg, width, height, smooth_sz, sigma, blurred);
      orc_resize_linear_f32(blurred, width, height, 1, I, w, h);
      R[i] = (float*)malloc(sizeof(float) * (size_t)w * h * 5);
      orc_poly_exp(I, w, h, poly_n, poly_sigma, R[i]);
    }
    float* M = (float*)malloc(sizeof(float) * (size_t)w * h * 5);
    orc_update_matrices(R[0], R[1], flow, w, h, M);
    for (int i = 0; i < num_iters; ++i) {
      orc_update_flow_blur(M, w, h, win_size, flow);
      if (i < num_iters - 1) orc_update_matrices(R[0], R[1], flow, w, h, M);
    }
    free(M);
    free(R[0]);
    free(R[1]);
    free(I);
    if (prev_flow) free(prev_flow);
    prev_flow = flow;
    pw = w;
    ph = h;
  }
  free(fimg);
  free(blurred);
}
