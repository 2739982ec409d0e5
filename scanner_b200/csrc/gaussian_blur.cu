// gaussian_blur.cu -- cv2.GaussianBlur on u8 frames (HxWx1, HxWx3) and on NV12 surfaces, bit-exact.
//
// cv2 runs CV_8U input through a fixed-point path (OpenCV >= 4): the Gaussian is built in double, normalised, and
// turned into taps with 8 fractional bits that sum to exactly 256; a horizontal pass keeps 8.8 fixed-point row sums,
// and a vertical pass rounds the 16.16 total back to u8 with (s + 2^15) >> 16.  Every product and sum is an exact
// integer, so the passes may run in any order: the kernel runs the vertical pass first on staged u8 rows (two 16-bit
// lanes per 32-bit multiply, since a tap times a pixel and any partial column sum fit 16 bits), then the horizontal
// pass on those sums in fp32, where every product and partial sum is an integer below 2^24 and so exact.
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>

#include "nv12_math.cuh"
#include "scn_common.cuh"

namespace scn {
namespace {

constexpr int kMaxK = 31;          // per axis
constexpr int kTileW = 384;        // output bytes per tile row (a multiple of 3 and of 16)
constexpr int kTileH = 16;         // output rows per tile
constexpr int kThreads = 192;      // kTileW / 16 * kTileH / 2 items of the horizontal pass: two per thread
constexpr uint32_t kPlanMagic = 0x47534231u;  // "GSB1"

enum Border { kReplicate = 1, kReflect = 2, kReflect101 = 4 };  // cv2's BorderTypes numbers

struct Plan {  // what scn_gaussian_blur_plan_fill writes; scn_gaussian_blur_plan_bytes() == sizeof(Plan)
  uint32_t magic;
  int32_t kw, kh, border;
  int32_t kx[32], ky[32];  // taps, 8 fractional bits, each axis sums to 256
};

// The taps as the kernels take them, in the parameter block: kx as floats for the unrolled horizontal pass.
struct Taps {
  float kx[32];
  int32_t ky[32];
  int32_t kh, border;
};

// ---- the host plan: cv2's kernel construction (smooth.dispatch.cpp, createGaussianKernels) ----

// getGaussianKernel's double kernel.  sigma <= 0 with n <= 9 takes fixed binomial-like tables; otherwise
// exp(-x^2 / (2 sigma^2)) for x = i - (n-1)/2 (written as exp((2x)^2 * (-0.125 / sigma^2))), normalised by 1/sum with
// the centre taken as 1 and the sum as 2 * (left half) + 1.  A sigma <= 0 becomes fma(n, 0.15, 0.35), i.e.
// 0.3 * ((n-1) * 0.5 - 1) + 0.8 with one rounding.  cv2 computes this in soft-float with its own exp; the double
// values here may differ from it in the last bits, which moves no fixed-point tap (tests/test_gaussian_blur_cpu.py checks the taps against cv2's own on a
// sweep of sigmas).
void gaussian_double(int n, double sigma, double* out) {
  static const double t3[] = {0.25, 0.5, 0.25};
  static const double t5[] = {0.0625, 0.25, 0.375, 0.25, 0.0625};
  static const double t7[] = {0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125};
  static const double t9[] = {4 / 256., 13 / 256., 30 / 256., 51 / 256., 60 / 256.,
                              51 / 256., 30 / 256., 13 / 256., 4 / 256.};
  if (n == 1) {
    out[0] = 1.0;
    return;
  }
  if (sigma <= 0 && n <= 9) {
    const double* t = n == 3 ? t3 : n == 5 ? t5 : n == 7 ? t7 : t9;
    for (int i = 0; i < n; ++i) out[i] = t[i];
    return;
  }
  const double s = sigma > 0 ? sigma : std::fma((double)n, 0.15, 0.35);
  const double scale2 = -0.125 / (s * s);
  const int half = (n - 1) / 2;
  double vals[kMaxK], sum = 0.0;
  for (int i = 0, x = 1 - n; i < half; ++i, x += 2) {
    vals[i] = std::exp((double)(x * x) * scale2);
    sum += vals[i];
  }
  sum = sum * 2.0 + 1.0;
  const double mul = 1.0 / sum;
  for (int i = 0; i < half; ++i) out[i] = out[n - 1 - i] = vals[i] * mul;
  out[half] = mul;
}

// getGaussianKernelFixedPoint_ED: the left half rounded (half to even) with the rounding error carried to the next
// tap, mirrored, and the centre set so that the taps sum to exactly 1 << 8.
void fixed_taps(int n, double sigma, int32_t* taps) {
  double k[kMaxK];
  gaussian_double(n, sigma, k);
  double err = 0.0;
  int32_t sum = 0;
  for (int i = 0; i < n / 2; ++i) {
    const double adj = k[i] * 256.0 + err;
    const int32_t v = (int32_t)std::nearbyint(adj);
    err = adj - (double)v;
    taps[i] = taps[n - 1 - i] = v;
    sum += v;
  }
  taps[n / 2] = 256 - 2 * sum;
}

// ksize 0 comes from sigma: cvRound(sigma * 3 * 2 + 1) | 1 (the 8U rule).  Returns 0 or an SCN_E_*.
int derive_ksize(int& k, double sigma) {
  if (k < 0 || (k > 0 && !(k & 1))) return SCN_E_BADARG;
  if (k == 0) {
    if (!(sigma > 0)) return SCN_E_BADARG;
    const double d = sigma * 3 * 2 + 1;
    if (!(d < 2.0 * kMaxK)) return SCN_E_UNSUPPORTED;
    k = (int)std::nearbyint(d) | 1;
  }
  return k > kMaxK ? SCN_E_UNSUPPORTED : 0;
}

bool plan_ok(const Plan* p) {
  if (!p || p->magic != kPlanMagic) return false;
  if (p->border != kReplicate && p->border != kReflect && p->border != kReflect101) return false;
  for (int a = 0; a < 2; ++a) {
    const int k = a ? p->kh : p->kw;
    const int32_t* t = a ? p->ky : p->kx;
    if (k < 1 || k > kMaxK || !(k & 1)) return false;
    int32_t s = 0;
    for (int i = 0; i < k; ++i) {
      if (t[i] < 0 || t[i] > 256) return false;
      s += t[i];
    }
    if (s != 256) return false;
  }
  return true;
}

// ---- device side ----

// cv::borderInterpolate for the three supported borders; p may lie any distance outside [0, len).
__host__ __device__ __forceinline__ int border_at(int p, int len, int border) {
  if ((unsigned)p < (unsigned)len) return p;
  if (border == kReplicate) return p < 0 ? 0 : len - 1;
  if (len == 1) return 0;
  const int delta = border == kReflect101;
  do {
    p = p < 0 ? -p - 1 + delta : len - 1 - (p - len) - delta;
  } while ((unsigned)p >= (unsigned)len);
  return p;
}

__device__ __forceinline__ int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// Stages source rows y0 - kh/2 .. y0 + kTileH + kh/2 - 1 (border-mapped) of one tile into smem, row r at
// src_s + r * sp, byte j holding row byte x0 - R + j (columns border-mapped per pixel).  From u8 frames: each thread
// fills 16 bytes with two aligned 16-byte loads and funnel shifts where those lie inside the row, else byte by byte.
template <int C>
__device__ __forceinline__ void stage_u8(const uint8_t* __restrict__ frame, int width, int height, int x0, int y0,
                                         int R, int rows, int sp, int border, uint8_t* src_s) {
  const int rowbytes = width * C;
  const int slots = sp >> 4;
  const int ry = (rows - kTileH) >> 1;
  for (int it = threadIdx.x; it < rows * slots; it += kThreads) {
    const int r = it / slots, u = it - r * slots;
    const int y = border_at(y0 - ry + r, height, border);
    const uint8_t* row = frame + (size_t)y * rowbytes;
    const int xb = x0 - R + 16 * u;  // row byte of smem byte 16u
    uint32_t o[4];
    const uintptr_t a = reinterpret_cast<uintptr_t>(row) + xb;  // meaningful when xb >= 0
    const uintptr_t al = a & ~(uintptr_t)15;
    const int sh = (int)(a & 15);
    if (xb >= 0 && al >= reinterpret_cast<uintptr_t>(row) &&
        al + 32 <= reinterpret_cast<uintptr_t>(row) + (uintptr_t)rowbytes) {
      const uint4 c0 = __ldg(reinterpret_cast<const uint4*>(al));
      const uint4 c1 = __ldg(reinterpret_cast<const uint4*>(al + 16));
      const uint32_t w[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      const int q = sh >> 2, b = (sh & 3) * 8;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t lo = q == 0 ? w[i] : q == 1 ? w[i + 1] : q == 2 ? w[i + 2] : w[i + 3];
        const uint32_t hi = q == 0 ? w[i + 1] : q == 1 ? w[i + 2] : q == 2 ? w[i + 3] : w[i + 4];
        o[i] = __funnelshift_r(lo, hi, b);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) o[i] = 0;
#pragma unroll 4
      for (int j = 0; j < 16; ++j) {
        const int x = xb + j;
        int m = x;
        if ((unsigned)x >= (unsigned)rowbytes) {
          const int px = floor_div(x, C);
          m = border_at(px, width, border) * C + (x - px * C);
        }
        o[j >> 2] |= (uint32_t)row[m] << (8 * (j & 3));
      }
    }
    *reinterpret_cast<uint4*>(src_s + r * sp + 16 * u) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// The same from an NV12 surface: each staged pixel is the reference's NV12 -> RGB24 conversion of the border-mapped
// source pixel, so the result equals scn_nv12_to_rgb24 followed by the u8 kernel.
__device__ __forceinline__ void stage_nv12(const uint8_t* __restrict__ luma, const uint8_t* __restrict__ chroma,
                                           size_t pitch, int width, int height, int x0, int y0, int R, int rows,
                                           int sp, int border, uint8_t* src_s) {
  const int pix = sp / 3;
  const int ry = (rows - kTileH) >> 1;
  const int px0 = (x0 - R) / 3;  // x0 and R are multiples of 3
  for (int it = threadIdx.x; it < rows * pix; it += kThreads) {
    const int r = it / pix, p = it - r * pix;
    const int y = border_at(y0 - ry + r, height, border);
    const int x = border_at(px0 + p, width, border);
    const Rgb8 c = nv12_pixel(luma, chroma, pitch, height, x, y);
    uint8_t* d = src_s + r * sp + 3 * p;
    d[0] = c.r;
    d[1] = c.g;
    d[2] = c.b;
  }
}

// u16 column sum -> float, exactly (v < 2^23)
__device__ __forceinline__ float u2f(uint32_t v) { return __uint_as_float(0x4B000000u | v) - 8388608.0f; }

// One CTA: output rows [y0, y0 + kTileH) x row bytes [x0, x0 + kTileW) of one frame.
template <int KW, int C, bool NV12>
__global__ void __launch_bounds__(kThreads)
gaussian_blur_kernel(PtrBatch srcs, PtrBatch chromas, MutPtrBatch dsts, size_t pitch, int width, int height,
                     Taps taps) {
  extern __shared__ __align__(16) uint8_t smem[];
  constexpr int R = (KW / 2) * C;
  constexpr int VW = kTileW + 2 * R;             // bytes of column sums a tile row needs
  constexpr int SP = (VW + 15) & ~15;            // staged row pitch (bytes) and column-sum row pitch (floats)
  const int kh = taps.kh;
  const int rows = kTileH + kh - 1;
  uint8_t* src_s = smem;
  float* col_s = reinterpret_cast<float*>(smem + (size_t)rows * SP);
  __shared__ int32_t ky[32];
  if (threadIdx.x < 32) ky[threadIdx.x] = taps.ky[threadIdx.x];

  const int f = blockIdx.z;
  const int x0 = blockIdx.x * kTileW, y0 = blockIdx.y * kTileH;
  const int rowbytes = width * C;
  if (NV12)
    stage_nv12(srcs.p[f], chromas.p[f], pitch, width, height, x0, y0, R, rows, SP, taps.border, src_s);
  else
    stage_u8<C>(srcs.p[f], width, height, x0, y0, R, rows, SP, taps.border, src_s);
  __syncthreads();

  // vertical pass: two output rows x four bytes per item, two 16-bit lanes per multiply
  constexpr int words = SP / 4;
  for (int it = threadIdx.x; it < (kTileH / 2) * words; it += kThreads) {
    const int t = 2 * (it / words), wd = it - (t / 2) * words;
    const uint32_t* s = reinterpret_cast<const uint32_t*>(src_s + t * SP) + wd;
    // staged row t + i carries tap i for output row t and tap i - 1 for output row t + 1
    uint32_t a0 = 0, a1 = 0, b0 = 0, b1 = 0;  // row t: even / odd bytes; row t + 1: even / odd bytes
    uint32_t kprev = 0;
    for (int i = 0; i <= kh; ++i) {
      const uint32_t w = s[i * (SP / 4)];
      const uint32_t e = w & 0x00FF00FFu, o = (w >> 8) & 0x00FF00FFu;
      const uint32_t k = i < kh ? (uint32_t)ky[i] : 0u;
      a0 += e * k;
      a1 += o * k;
      b0 += e * kprev;
      b1 += o * kprev;
      kprev = k;
    }
    float4* d = reinterpret_cast<float4*>(col_s + t * SP) + wd;
    d[0] = make_float4(u2f(a0 & 0xFFFF), u2f(a1 & 0xFFFF), u2f(a0 >> 16), u2f(a1 >> 16));
    d[SP / 4] = make_float4(u2f(b0 & 0xFFFF), u2f(b1 & 0xFFFF), u2f(b0 >> 16), u2f(b1 >> 16));
  }
  __syncthreads();

  // horizontal pass: 16 output bytes per item from a register window of column sums, taps at compile-time offsets
  constexpr int L = 16 + (KW - 1) * C;
  constexpr int L4 = (L + 3) / 4;
  for (int it = threadIdx.x; it < kTileH * (kTileW / 16); it += kThreads) {
    const int t = it / (kTileW / 16), m0 = 16 * (it - t * (kTileW / 16));
    const int y = y0 + t;
    if (y >= height || x0 + m0 >= rowbytes) continue;
    const float4* v = reinterpret_cast<const float4*>(col_s + t * SP + m0);
    float acc[16];
#pragma unroll
    for (int m = 0; m < 16; ++m) acc[m] = 32768.0f;  // the rounding half of (s + 2^15) >> 16
#pragma unroll
    for (int c4 = 0; c4 < L4; ++c4) {
      const float4 q = v[c4];
      const float w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int p = 4 * c4 + e;
#pragma unroll
        for (int m = 0; m < 16; ++m) {
          const int d = p - m;
          if (d >= 0 && d % C == 0 && d / C < KW) acc[m] = __fmaf_rn(taps.kx[d / C], w[e], acc[m]);
        }
      }
    }
    uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
    for (int m = 0; m < 16; ++m) {  // floor(acc / 2^16) from the mantissa of acc * 2^-16 + 2^23, rounded down
      const uint32_t b = __float_as_uint(__fmaf_rd(acc[m], 1.0f / 65536.0f, 8388608.0f)) - 0x4B000000u;
      o[m >> 2] |= b << (8 * (m & 3));
    }
    uint8_t* out = dsts.p[f] + (size_t)y * rowbytes + x0 + m0;
    const int valid = min(16, rowbytes - (x0 + m0));
    const uintptr_t ad = reinterpret_cast<uintptr_t>(out);
    if (valid == 16 && (ad & 15) == 0) {
      *reinterpret_cast<uint4*>(out) = make_uint4(o[0], o[1], o[2], o[3]);
    } else if (valid == 16 && (ad & 3) == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i) reinterpret_cast<uint32_t*>(out)[i] = o[i];
    } else {
      for (int j = 0; j < valid; ++j) out[j] = (uint8_t)(o[j >> 2] >> (8 * (j & 3)));
    }
  }
}

size_t smem_bytes(int kw, int kh, int c) {
  const int sp = (kTileW + 2 * (kw / 2) * c + 15) & ~15;
  return (size_t)(kTileH + kh - 1) * sp + (size_t)kTileH * sp * sizeof(float);
}

template <int KW, int C, bool NV12>
int launch(const Plan& p, const uint8_t* const* src, const uint8_t* const* chroma, size_t pitch, int n, int width,
           int height, uint8_t* const* dst, cudaStream_t st) {
  auto* kern = gaussian_blur_kernel<KW, C, NV12>;
  const size_t smem = smem_bytes(KW, p.kh, C);
  if (int rc = raise_smem_limit(reinterpret_cast<const void*>(kern), smem_bytes(KW, kMaxK, C))) return rc;
  Taps taps;
  for (int i = 0; i < 32; ++i) {
    taps.kx[i] = (float)p.kx[i];
    taps.ky[i] = p.ky[i];
  }
  taps.kh = p.kh;
  taps.border = p.border;
  const long long rowbytes = (long long)width * C;
  dim3 grid((unsigned)((rowbytes + kTileW - 1) / kTileW), (unsigned)((height + kTileH - 1) / kTileH), 1);
  return for_each_chunk(n, [&](int i0, int cnt) {
    const PtrBatch s = gather<PtrBatch>(src, i0, cnt);
    const PtrBatch c = NV12 ? gather<PtrBatch>(chroma, i0, cnt) : PtrBatch{};
    const MutPtrBatch d = gather<MutPtrBatch>(dst, i0, cnt);
    grid.z = (unsigned)cnt;
    return launch_kernel(NV12 ? "gaussian_blur_nv12_kernel" : "gaussian_blur_kernel", st, [&] {
      kern<<<grid, kThreads, smem, st>>>(s, c, d, pitch, width, height, taps);
    });
  });
}

template <int C, bool NV12>
int dispatch(const Plan& p, const uint8_t* const* src, const uint8_t* const* chroma, size_t pitch, int n, int width,
             int height, uint8_t* const* dst, cudaStream_t st) {
#define SCN_GB_CASE(K) \
  case K: return launch<K, C, NV12>(p, src, chroma, pitch, n, width, height, dst, st);
  switch (p.kw) {
    SCN_GB_CASE(1) SCN_GB_CASE(3) SCN_GB_CASE(5) SCN_GB_CASE(7) SCN_GB_CASE(9) SCN_GB_CASE(11) SCN_GB_CASE(13)
    SCN_GB_CASE(15) SCN_GB_CASE(17) SCN_GB_CASE(19) SCN_GB_CASE(21) SCN_GB_CASE(23) SCN_GB_CASE(25)
    SCN_GB_CASE(27) SCN_GB_CASE(29) SCN_GB_CASE(31)
  }
#undef SCN_GB_CASE
  return SCN_E_PLAN;
}

// The checks every launch entry shares; 1 means "nothing to do".
int check_geometry(int n, int width, int height, int c) {
  if (n < 0 || width < 0 || height < 0 || (c != 1 && c != 3)) return SCN_E_BADARG;
  if ((long long)width * height > INT_MAX) return SCN_E_BADARG;
  if ((long long)width * c > INT_MAX || height > 65535 * kTileH) return SCN_E_UNSUPPORTED;
  return 0;
}

}  // namespace
}  // namespace scn

extern "C" int scn_gaussian_blur_border_code(const char* name) {
  using namespace scn;
  if (!name) return SCN_E_BADARG;
  if (!*name || !std::strcmp(name, "BORDER_DEFAULT") || !std::strcmp(name, "BORDER_REFLECT_101") ||
      !std::strcmp(name, "BORDER_REFLECT101"))
    return kReflect101;
  if (!std::strcmp(name, "BORDER_REPLICATE")) return kReplicate;
  if (!std::strcmp(name, "BORDER_REFLECT")) return kReflect;
  if (!std::strcmp(name, "BORDER_CONSTANT") || !std::strcmp(name, "BORDER_WRAP") ||
      !std::strcmp(name, "BORDER_TRANSPARENT") || !std::strcmp(name, "BORDER_ISOLATED"))
    return SCN_E_UNSUPPORTED;
  return SCN_E_BADARG;
}

extern "C" const char* scn_gaussian_blur_borders(void) {
  return "BORDER_DEFAULT (= BORDER_REFLECT_101, also \"\"), BORDER_REPLICATE, BORDER_REFLECT";
}

extern "C" size_t scn_gaussian_blur_plan_bytes(void) { return sizeof(scn::Plan); }

extern "C" int scn_gaussian_blur_plan_fill(int kw, int kh, double sigma_x, double sigma_y, int border,
                                           void* host_plan) {
  using namespace scn;
  if (!host_plan || !std::isfinite(sigma_x) || !std::isfinite(sigma_y)) return SCN_E_BADARG;
  if (border != kReplicate && border != kReflect && border != kReflect101) return SCN_E_BADARG;
  if (sigma_y <= 0) sigma_y = sigma_x;  // createGaussianKernels: sigma2 <= 0 means sigma1
  int rcx = derive_ksize(kw, sigma_x), rcy = derive_ksize(kh, sigma_y);
  if (rcx == SCN_E_BADARG || rcy == SCN_E_BADARG) return SCN_E_BADARG;
  if (rcx || rcy) return SCN_E_UNSUPPORTED;
  sigma_x = sigma_x > 0 ? sigma_x : 0.0;
  sigma_y = sigma_y > 0 ? sigma_y : 0.0;
  Plan p;
  std::memset(&p, 0, sizeof(p));
  p.magic = kPlanMagic;
  p.kw = kw;
  p.kh = kh;
  p.border = border;
  fixed_taps(kw, sigma_x, p.kx);
  if (kh == kw && std::fabs(sigma_x - sigma_y) < DBL_EPSILON)  // cv2 reuses the x kernel here
    std::memcpy(p.ky, p.kx, sizeof(p.kx));
  else
    fixed_taps(kh, sigma_y, p.ky);
  std::memcpy(host_plan, &p, sizeof(p));
  return 0;
}

extern "C" int scn_gaussian_blur_u8(const void* plan, const uint8_t* const* host_src_ptrs, int n, int width,
                                    int height, int channels, uint8_t* const* host_dst_ptrs, void* stream) {
  using namespace scn;
  Plan p;
  if (!plan) return SCN_E_PLAN;
  std::memcpy(&p, plan, sizeof(p));
  if (!plan_ok(&p)) return SCN_E_PLAN;
  if (int rc = check_geometry(n, width, height, channels)) return rc;
  if (n == 0 || width == 0 || height == 0) return 0;
  if (!host_src_ptrs || !host_dst_ptrs) return SCN_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  return channels == 1 ? dispatch<1, false>(p, host_src_ptrs, nullptr, 0, n, width, height, host_dst_ptrs, st)
                       : dispatch<3, false>(p, host_src_ptrs, nullptr, 0, n, width, height, host_dst_ptrs, st);
}

extern "C" int scn_gaussian_blur_nv12(const void* plan, const uint8_t* const* host_luma_ptrs,
                                      const uint8_t* const* host_chroma_ptrs, size_t pitch, int n, int width,
                                      int height, uint8_t* const* host_dst_ptrs, void* stream) {
  using namespace scn;
  Plan p;
  if (!plan) return SCN_E_PLAN;
  std::memcpy(&p, plan, sizeof(p));
  if (!plan_ok(&p)) return SCN_E_PLAN;
  if (width <= 0 || height <= 0 || (width & 1) || (height & 1) || pitch < (size_t)width) return SCN_E_BADARG;
  if (int rc = check_geometry(n, width, height, 3)) return rc;
  if (n == 0) return 0;
  if (!host_luma_ptrs || !host_chroma_ptrs || !host_dst_ptrs) return SCN_E_BADARG;
  return dispatch<3, true>(p, host_luma_ptrs, host_chroma_ptrs, pitch, n, width, height, host_dst_ptrs,
                           (cudaStream_t)stream);
}
