/* cv2.GaussianBlur on CV_8U frames, restated in plain C -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
 *
 * OpenCV >= 4 runs 8-bit input through a fixed-point path whose every step is exact integer arithmetic once the taps
 * are known, so this file can match cv2 byte for byte on any host.  Each rule is written next to its code; the rules
 * were settled against live cv2 4.13 (tests/test_gaussian_blur_cpu.py).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MAXK 31

/* Kernel size from sigma (createGaussianKernels, 8U rule): ksize 0 -> cvRound(sigma * 3 * 2 + 1) | 1.  Returns 0 or
 * -1 (even or negative size, size 0 with sigma <= 0) or -2 (a size above MAXK). */
static int ksize_of(int k, double sigma, int* out) {
    if (k < 0 || (k > 0 && !(k & 1))) return -1;
    if (k == 0) {
        if (!(sigma > 0)) return -1;
        double d = sigma * 3 * 2 + 1;
        if (!(d < 2.0 * MAXK)) return -2;
        k = (int)nearbyint(d) | 1;
    }
    if (k > MAXK) return -2;
    *out = k;
    return 0;
}

/* getGaussianKernel in double.  sigma <= 0 and n <= 9: fixed tables (n = 9 is 4 13 30 51 60 51 30 13 4 / 256).
 * Otherwise sigma <= 0 becomes 0.15 n + 0.35 with one rounding (softfloat mulAdd), and
 *   t_i = exp((2x)^2 * (-0.125 / sigma^2)), x = i - (n-1)/2, for the left half; sum = 2 * sum(t_i) + 1;
 *   k_i = t_i * (1 / sum), centre = 1 / sum.
 * cv2 evaluates exp in soft-float; libm's exp differs from it in the last bits of the double kernel for many
 * sigmas, which changes no 8-bit tap below (the CPU test checks the taps against cv2's own on a sweep). */
static void gaussian_double(int n, double sigma, double* k) {
    static const double t9[9] = {4, 13, 30, 51, 60, 51, 30, 13, 4};
    static const double t7[7] = {8, 28, 56, 72, 56, 28, 8};
    static const double t5[5] = {16, 64, 96, 64, 16};
    static const double t3[3] = {64, 128, 64};
    if (n == 1) { k[0] = 1.0; return; }
    if (sigma <= 0 && n <= 9) {
        const double* t = n == 3 ? t3 : n == 5 ? t5 : n == 7 ? t7 : t9;
        for (int i = 0; i < n; i++) k[i] = t[i] / 256.0;
        return;
    }
    double s = sigma > 0 ? sigma : fma((double)n, 0.15, 0.35);
    double scale2 = -0.125 / (s * s);
    int half = (n - 1) / 2;
    double t[MAXK], sum = 0.0;
    for (int i = 0, x = 1 - n; i < half; i++, x += 2) {
        t[i] = exp((double)(x * x) * scale2);
        sum += t[i];
    }
    sum = sum * 2.0 + 1.0;
    double mul = 1.0 / sum;
    for (int i = 0; i < half; i++) k[i] = k[n - 1 - i] = t[i] * mul;
    k[half] = mul;
}

/* getGaussianKernelFixedPoint_ED with 8 fraction bits (ufixedpoint16): left to right over the left half,
 * v = cvRound(k_i * 256 + err) (half to even), err = (k_i * 256 + err) - v; mirrored; centre = 256 - 2 * sum. */
static void fixed_taps(int n, double sigma, int32_t* taps) {
    double k[MAXK], err = 0.0;
    int32_t sum = 0;
    gaussian_double(n, sigma, k);
    for (int i = 0; i < n / 2; i++) {
        double adj = k[i] * 256.0 + err;
        int32_t v = (int32_t)nearbyint(adj);
        err = adj - (double)v;
        taps[i] = taps[n - 1 - i] = v;
        sum += v;
    }
    taps[n / 2] = 256 - 2 * sum;
}

/* The taps of (kw, kh, sigma_x, sigma_y) -> 0, or -1 / -2 as ksize_of.  sigma_y <= 0 means sigma_x; a negative
 * sigma is 0 (ksize-derived); equal sizes with |sigma_x - sigma_y| < DBL_EPSILON share the x kernel. */
int orc_gaussian_taps(int kw, int kh, double sx, double sy, int32_t* kx, int* kw_out, int32_t* ky, int* kh_out) {
    if (!isfinite(sx) || !isfinite(sy)) return -1;
    if (sy <= 0) sy = sx;
    int rx = ksize_of(kw, sx, &kw), ry = ksize_of(kh, sy, &kh);
    if (rx == -1 || ry == -1) return -1;
    if (rx || ry) return -2;
    sx = sx > 0 ? sx : 0.0;
    sy = sy > 0 ? sy : 0.0;
    fixed_taps(kw, sx, kx);
    if (kh == kw && fabs(sx - sy) < DBL_EPSILON)
        memcpy(ky, kx, sizeof(int32_t) * kw);
    else
        fixed_taps(kh, sy, ky);
    *kw_out = kw;
    *kh_out = kh;
    return 0;
}

/* cv::borderInterpolate: 1 BORDER_REPLICATE (clamp), 2 BORDER_REFLECT (fedcba|abcdefgh|hgfedcb),
 * 4 BORDER_REFLECT_101 (gfedcb|abcdefgh|gfedcba), reflected as many times as a side shorter than the kernel needs;
 * a side of 1 maps everything to 0. */
static int border_at(int p, int len, int border) {
    if (p >= 0 && p < len) return p;
    if (border == 1) return p < 0 ? 0 : len - 1;
    if (len == 1) return 0;
    int delta = border == 4;
    do {
        p = p < 0 ? -p - 1 + delta : len - 1 - (p - len) - delta;
    } while (p < 0 || p >= len);
    return p;
}

/* The passes (fixedSmoothInvoker<uint8_t, ufixedpoint16>): a horizontal pass into 8.8 fixed-point row sums,
 * row[x] = sum_j kx[j] * src[border(x + j - kw/2)] (never above 255 * 256), then a vertical pass
 * out = (sum_i ky[i] * row[border(y + i - kh/2)] + 2^15) >> 16.  cv2's special forms for symmetric 3- and 5-tap
 * kernels ([1 2 1], [1 4 6 4 1], a b a, a b c b a) and for a 1-tap axis compute the same integers.  A 1-row or
 * 1-column frame makes cv2 use a 1-tap kernel on that axis, which every border above already gives.
 * Returns 0, or -1 / -2 for refused arguments. */
int orc_gaussian_blur_u8(const uint8_t* src, int w, int h, int c, uint8_t* dst, int kw, int kh, double sx, double sy,
                         int border) {
    int32_t kx[MAXK], ky[MAXK];
    if (border != 1 && border != 2 && border != 4) return -1;
    int rc = orc_gaussian_taps(kw, kh, sx, sy, kx, &kw, ky, &kh);
    if (rc) return rc;
    int rw = w * c;
    uint32_t* rows = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)rw * h);
    if (!rows) return -3;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++)
            for (int ch = 0; ch < c; ch++) {
                uint32_t s = 0;
                for (int j = 0; j < kw; j++) s += (uint32_t)kx[j] * src[(size_t)y * rw + border_at(x + j - kw / 2, w, border) * c + ch];
                rows[(size_t)y * rw + x * c + ch] = s;
            }
    for (int y = 0; y < h; y++)
        for (int i = 0; i < rw; i++) {
            uint32_t s = 0;
            for (int j = 0; j < kh; j++) s += (uint32_t)ky[j] * rows[(size_t)border_at(y + j - kh / 2, h, border) * rw + i];
            dst[(size_t)y * rw + i] = (uint8_t)((s + (1u << 15)) >> 16);
        }
    free(rows);
    return 0;
}
