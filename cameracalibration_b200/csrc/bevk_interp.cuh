// bevk_interp.cuh -- cv2.remap's INTER_CUBIC and INTER_LANCZOS4 (OpenCV 4.13, CV_16SC2 + CV_16UC1 maps): the weight
// tables and the per-pixel tap sums, and cv2's border modes for every gather (border_window), shared by the device
// gathers and the host harnesses under tests/host/.  DESIGN.md section 2 has the arithmetic.
#pragma once
#include <float.h>
#include <math.h>
#include <string.h>

#include "bevk_device.cuh"

namespace bevk {

constexpr int INTER_TAB_SIZE2 = TAB * TAB;   // weight rows, indexed by map2 = fy * 32 + fx
constexpr int COEF_BITS = 15;                // INTER_REMAP_COEF_BITS: the weights of a row sum to 1 << 15

// ---- OpenCV's 1-D kernels (imgwarp.cpp interpolateCubic / interpolateLanczos4) at x = i / 32, i in 0..31.
// OpenCV's baseline x86-64 unit has no FMA, so every float and double operation is rounded on its own: the host forms
// of fmul / fadd / fsub / dmul / dadd / ddiv go through volatile stores, which no -ffp-contract or -march setting in
// BEVK_NVCC_FLAGS can fuse.  sin / cos are the host libm's, the library cv2 itself calls (DESIGN.md section 2).
inline void cubic_coeffs(float x, float* c) {
  const float A = -0.75f;   // 5A, 8A, 4A, A + 2, A + 3 are exact
  const float x1 = fadd(x, 1.f), xm = fsub(1.f, x);
  c[0] = fsub(fmul(fadd(fmul(fsub(fmul(A, x1), 5 * A), x1), 8 * A), x1), 4 * A);
  c[1] = fadd(fmul(fmul(fsub(fmul(A + 2, x), A + 3), x), x), 1.f);
  c[2] = fadd(fmul(fmul(fsub(fmul(A + 2, xm), A + 3), xm), xm), 1.f);
  c[3] = fsub(fsub(fsub(1.f, c[0]), c[1]), c[2]);
}

inline void lanczos4_coeffs(float x, float* c) {
  if (x < FLT_EPSILON) {
    for (int i = 0; i < 8; ++i) c[i] = 0.f;
    c[3] = 1.f;
    return;
  }
  const double s45 = 0.70710678118654752440084436210485, pi = 3.141592653589793238462643383279502884;
  static const double cs[8][2] = {{1, 0}, {-s45, -s45}, {0, 1}, {s45, -s45}, {-1, 0}, {s45, s45}, {0, -1}, {-s45, s45}};
  const double y0 = dmul(dmul((double)-fadd(x, 3.f), pi), 0.25), s0 = sin(y0), c0 = cos(y0);
  float sum = 0.f;
  for (int i = 0; i < 8; ++i) {
    const double y = dmul(dmul((double)-fsub(fadd(x, 3.f), (float)i), pi), 0.25);
    c[i] = (float)ddiv(dadd(dmul(cs[i][0], s0), dmul(cs[i][1], c0)), dmul(y, y));
    sum = fadd(sum, c[i]);
  }
  volatile float inv = 1.f / sum;
  for (int i = 0; i < 8; ++i) c[i] = fmul(c[i], inv);
}

// ---- initInterTab2D for 8-bit images: tab[(fy * 32 + fx) * KS * KS + k1 * KS + k2] = round(vy[k1] * vx[k2] * 2^15) as
// int16, then each row forced to sum to 2^15.  OpenCV looks for the row's least and greatest weight in rows and columns
// [KS/2, KS/2 + 2) -- not the central 2x2 -- starting from entry (KS/2, KS/2); a surplus comes off the least one, a
// deficit goes onto the greatest.  KS = 4: cubic, 8: Lanczos4.
template <int KS>
inline void build_interp_tab(short* tab) {
  float k1d[TAB][KS];
  for (int i = 0; i < TAB; ++i) {
    const float x = (float)i * (1.f / TAB);
    if (KS == 4) cubic_coeffs(x, k1d[i]);
    else lanczos4_coeffs(x, k1d[i]);
  }
  for (int fy = 0; fy < TAB; ++fy)
    for (int fx = 0; fx < TAB; ++fx) {
      short* t = tab + (fy * TAB + fx) * KS * KS;
      int isum = 0;
      for (int k1 = 0; k1 < KS; ++k1)
        for (int k2 = 0; k2 < KS; ++k2) {
          const float v = fmul(fmul(k1d[fy][k1], k1d[fx][k2]), (float)(1 << COEF_BITS));
          isum += t[k1 * KS + k2] = (short)max(-32768, min(32767, f2i_rn(v)));
        }
      const int diff = isum - (1 << COEF_BITS);
      if (diff == 0) continue;
      const int h = KS / 2;
      int mk1 = h, mk2 = h, Mk1 = h, Mk2 = h;
      for (int k1 = h; k1 < h + 2; ++k1)
        for (int k2 = h; k2 < h + 2; ++k2) {
          if (t[k1 * KS + k2] < t[mk1 * KS + mk2]) mk1 = k1, mk2 = k2;
          else if (t[k1 * KS + k2] > t[Mk1 * KS + Mk2]) Mk1 = k1, Mk2 = k2;
        }
      if (diff < 0) t[Mk1 * KS + Mk2] = (short)(t[Mk1 * KS + Mk2] - diff);
      else t[mk1 * KS + mk2] = (short)(t[mk1 * KS + mk2] - diff);
    }
}

// Both tables back to back, as the library uploads them: cubic (1024 rows of 16) at 0, Lanczos4 (1024 rows of 64) at
// INTERP_TAB_LANCZOS4.
constexpr int INTERP_TAB_LANCZOS4 = INTER_TAB_SIZE2 * 16;
constexpr int INTERP_TAB_SHORTS = INTERP_TAB_LANCZOS4 + INTER_TAB_SIZE2 * 64;
inline void build_interp_tabs(short* tabs) {
  build_interp_tab<4>(tabs);
  build_interp_tab<8>(tabs + INTERP_TAB_LANCZOS4);
}

__host__ __device__ __forceinline__ int tap8(const uint8_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// ---- The 16U, 16S and 32F sources: cv2 takes its float tables there (initInterTab2D without the fixed-point form),
// whose 2-D entry is vy[k1] * vx[k2] rounded to float, with no fix-up.  The 1-D rows are all the gathers keep: cubic
// (32 rows of 4) at 0, Lanczos4 (32 rows of 8) at INTERP_ROWS_LANCZOS4; each pixel forms its products from two of them.
constexpr int INTERP_ROWS_LANCZOS4 = TAB * 4;
constexpr int INTERP_ROWS_FLOATS = INTERP_ROWS_LANCZOS4 + TAB * 8;
inline void build_interp_rows(float* rows) {
  for (int i = 0; i < TAB; ++i) {
    const float x = (float)i * (1.f / TAB);
    cubic_coeffs(x, rows + i * 4);
    lanczos4_coeffs(x, rows + INTERP_ROWS_LANCZOS4 + i * 8);
  }
}

// One element of type T at byte address p (16U, 16S, 32F: element-aligned), and a float sum stored as cv2's
// Cast<float, T> stores it: cvRound (half to even) and saturation for the integer depths, the float itself for 32F.
template <class T>
__host__ __device__ __forceinline__ T ld_elem(const uint8_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(reinterpret_cast<const T*>(p));
#else
  T v;
  memcpy(&v, p, sizeof v);
  return v;
#endif
}

template <class T>
__host__ __device__ __forceinline__ void st_sum(uint8_t* p, float v) {
  T r;
  if constexpr (sizeof(T) == 4) r = v;
  else if constexpr ((T)-1 > 0) r = (T)max(0, min(65535, f2i_rn(v)));
  else r = (T)max(-32768, min(32767, f2i_rn(v)));
#ifdef __CUDA_ARCH__
  *reinterpret_cast<T*>(p) = r;
#else
  memcpy(p, &r, sizeof r);
#endif
}

// ---- Borders: what the gathers read for a tap outside the source, as cv2.remap / warpPerspective / warpAffine do.
// cv2's border modes, with cv2's values (BEVK_BORDER_* in include/bevk.h).
constexpr int BORDER_CONSTANT = 0, BORDER_REPLICATE = 1, BORDER_REFLECT = 2, BORDER_WRAP = 3, BORDER_REFLECT_101 = 4,
              BORDER_TRANSPARENT = 5;

// A gather's border mode and value.  v holds four elements of the image's depth (bytes 0..4*esize), converted from
// cv2's Scalar as cv2 converts it (make_border); channel c reads element c.
struct Border {
  int mode;
  unsigned char v[16];
};

template <class T>
__host__ __device__ __forceinline__ T border_elem(const Border& b, int c) {
  T r;
  memcpy(&r, b.v + c * sizeof(T), sizeof r);
  return r;
}

// cv2's Scalar border value at depth (0 8U, 2 16U, 3 16S, 5 32F) as cv2's scalarToRawData converts it: cvRound (half
// to even; INT_MIN for NaN, +-inf and anything beyond int) then saturation at the integer depths, (float) at 32F.
inline Border make_border(int mode, int depth, const double (&val)[4]) {
  Border b{};
  b.mode = mode;
  for (int c = 0; c < 4; ++c) {
    const double v = val[c];
    if (depth == 5) {
      const float f = (float)v;
      memcpy(b.v + 4 * c, &f, 4);
    } else if (depth == 0) {
      b.v[c] = (unsigned char)max(0, min(255, cv_round(v)));
    } else {
      const int lo = depth == 2 ? 0 : -32768, hi = depth == 2 ? 65535 : 32767;
      const unsigned short e = (unsigned short)max(lo, min(hi, cv_round(v)));
      memcpy(b.v + 2 * c, &e, 2);
    }
  }
  return b;
}

// cv2.borderInterpolate in closed form: the source index position p reads on an axis of n >= 1 pixels, or -1 for the
// border value (BORDER_CONSTANT).  cv2 walks REFLECT and REFLECT_101 back one period per loop pass (about 16k passes for
// a 2-pixel axis at the int16 floor); the remainder modulo the period gives the same index for every p.
__host__ __device__ __forceinline__ int border_index(int p, int n, int mode) {
  if ((unsigned)p < (unsigned)n) return p;
  if (mode == BORDER_REPLICATE) return p < 0 ? 0 : n - 1;
  if (mode == BORDER_WRAP) {
    const int q = p % n;
    return q < 0 ? q + n : q;
  }
  if (mode == BORDER_REFLECT || mode == BORDER_REFLECT_101) {
    if (n == 1) return 0;
    const int d = mode == BORDER_REFLECT_101, per = 2 * (n - d);   // REFLECT: ..cb|abc..; REFLECT_101: ..c|abc..
    int q = p % per;
    if (q < 0) q += per;
    return q < n ? q : per - 1 + d - q;
  }
  return -1;
}

// A K x K window (K = 1 NEAREST, 2 LINEAR, 4 CUBIC, 8 LANCZOS4) with top-left tap (sx, sy), on a source of sw x sh:
// BW_SKIP, cv2 leaves the destination pixel as it is (BORDER_TRANSPARENT with the window's anchor -- the map's own
// pixel, tap K/2 - 1 -- outside the source); BW_FILL, cv2 writes the border value (BORDER_CONSTANT, window wholly
// outside); BW_TAPS, the taps are the source's columns xs and rows ys, -1 standing for the border value.
// BORDER_TRANSPARENT reads its other windows as REPLICATE (NEAREST, LINEAR) or REFLECT_101 (CUBIC, LANCZOS4).
enum { BW_TAPS = 0, BW_FILL = 1, BW_SKIP = 2 };
template <int K>
__host__ __device__ __forceinline__ int border_window(const Border& b, int sx, int sy, int sw, int sh, int (&xs)[K],
                                                      int (&ys)[K]) {
  constexpr int A = K > 1 ? K / 2 - 1 : 0;
  int m = b.mode;
  if (m == BORDER_TRANSPARENT) {
    if ((unsigned)(sx + A) >= (unsigned)sw || (unsigned)(sy + A) >= (unsigned)sh) return BW_SKIP;
    m = K > 2 ? BORDER_REFLECT_101 : BORDER_REPLICATE;
  } else if (m == BORDER_CONSTANT && (sx >= sw || sx + K <= 0 || sy >= sh || sy + K <= 0)) {
    return BW_FILL;
  }
#pragma unroll
  for (int k = 0; k < K; ++k) {
    xs[k] = border_index(sx + k, sw, m);
    ys[k] = border_index(sy + k, sh, m);
  }
  return BW_TAPS;
}

// The border value's C elements written as the pixel at o
template <int C, class T>
__host__ __device__ __forceinline__ void st_border(uint8_t* o, const Border& b) {
#pragma unroll
  for (int c = 0; c < C; ++c) {
#ifdef __CUDA_ARCH__
    reinterpret_cast<T*>(o)[c] = border_elem<T>(b, c);
#else
    memcpy(o + c * sizeof(T), b.v + c * sizeof(T), sizeof(T));
#endif
  }
}

// ---- A window of taps_px / taps_px_f that is not wholly inside the source, under any border (border_window): OpenCV
// sums it as cv * ONE + sum (S - cv) w over the taps it reads, cv the border value in every mode.  With int16 weights
// summing to 2^15 (8U) that is the sum with cv in place of the taps outside; in float (16U, 16S, 32F) it is not, so cv
// changes such windows even under REPLICATE, where no tap is outside.  The float sum takes the taps one by one in
// row-major order.
template <int KS, int C>
__host__ __device__ __forceinline__ void taps_px_edge(const uint8_t* __restrict__ src, long long spitch, int sw, int sh, int sx,
                                                      int sy, const short (&w)[KS * KS], uint8_t* __restrict__ o,
                                                      const Border& bd) {
  int xs[KS], ys[KS];
  const int act = border_window<KS>(bd, sx, sy, sw, sh, xs, ys);
  if (act == BW_SKIP) return;
  if (act == BW_FILL) {
    st_border<C, uint8_t>(o, bd);
    return;
  }
  int sum[C];
#pragma unroll
  for (int c = 0; c < C; ++c) sum[c] = (int)bd.v[c] << COEF_BITS;
#pragma unroll
  for (int k1 = 0; k1 < KS; ++k1) {
    if (ys[k1] < 0) continue;
    const uint8_t* q = src + (long long)ys[k1] * spitch;
#pragma unroll
    for (int k2 = 0; k2 < KS; ++k2) {
      if (xs[k2] < 0) continue;
#pragma unroll
      for (int c = 0; c < C; ++c) sum[c] += (tap8(q + (long long)xs[k2] * C + c) - (int)bd.v[c]) * w[k1 * KS + k2];
    }
  }
#pragma unroll
  for (int c = 0; c < C; ++c) o[c] = (uint8_t)max(0, min(255, (sum[c] + (1 << (COEF_BITS - 1))) >> COEF_BITS));
}

template <int KS, int C, class T>
__host__ __device__ __forceinline__ void taps_px_f_edge(const uint8_t* __restrict__ src, long long spitch, int sw, int sh,
                                                        int sx, int sy, const float (&vy)[KS], const float (&vx)[KS],
                                                        uint8_t* __restrict__ o, const Border& bd) {
  constexpr int E = (int)sizeof(T);
  int xs[KS], ys[KS];
  const int act = border_window<KS>(bd, sx, sy, sw, sh, xs, ys);
  if (act == BW_SKIP) return;
  if (act == BW_FILL) {
    st_border<C, T>(o, bd);
    return;
  }
  float sum[C], cv[C];
#pragma unroll
  for (int c = 0; c < C; ++c) sum[c] = cv[c] = (float)border_elem<T>(bd, c);
#pragma unroll
  for (int k1 = 0; k1 < KS; ++k1) {
    if (ys[k1] < 0) continue;
    const uint8_t* q = src + (long long)ys[k1] * spitch;
#pragma unroll
    for (int k2 = 0; k2 < KS; ++k2) {
      if (xs[k2] < 0) continue;
      const float w = fmul(vy[k1], vx[k2]);
#pragma unroll
      for (int c = 0; c < C; ++c)
        sum[c] = fadd(sum[c], fmul(fsub((float)ld_elem<T>(q + ((long long)xs[k2] * C + c) * E), cv[c]), w));
    }
  }
#pragma unroll
  for (int c = 0; c < C; ++c) st_sum<T>(o + c * E, sum[c]);
}

// ---- one output pixel of a KS x KS kernel (remapBicubic / remapLanczos4).  (sx, sy): the window's top-left tap, map1 -
// (KS/2 - 1) in int, so the int16 extremes do not wrap; w: the fraction class's row of weights, k1 * KS + k2.
// A tap outside the source adds nothing (OpenCV's BORDER_CONSTANT sum is cval * 2^15 + sum (S - cval) w with cval 0, and
// a window wholly outside is cval); windows wholly inside take OpenCV's fast-path test and read without checks.
// BD (k_gather_taps_border): a window not wholly inside follows border_window (taps_px_edge) instead.
template <int KS, int C, bool BD = false>
__host__ __device__ __forceinline__ void taps_px(const uint8_t* __restrict__ src, long long spitch, int sw, int sh, int sx,
                                                 int sy, const short (&w)[KS * KS], uint8_t* __restrict__ o,
                                                 const Border& bd) {
  if constexpr (BD) {
    if (!((unsigned)sx < (unsigned)max(sw - (KS - 1), 0) && (unsigned)sy < (unsigned)max(sh - (KS - 1), 0))) {
      taps_px_edge<KS, C>(src, spitch, sw, sh, sx, sy, w, o, bd);
      return;
    }
  }
  int sum[C];
#pragma unroll
  for (int c = 0; c < C; ++c) sum[c] = 0;
  if ((unsigned)sx < (unsigned)max(sw - (KS - 1), 0) && (unsigned)sy < (unsigned)max(sh - (KS - 1), 0)) {
    const uint8_t* q = src + (long long)sy * spitch + (long long)sx * C;
#pragma unroll
    for (int k1 = 0; k1 < KS; ++k1, q += spitch)
#pragma unroll
      for (int k2 = 0; k2 < KS; ++k2)
#pragma unroll
        for (int c = 0; c < C; ++c) sum[c] += tap8(q + k2 * C + c) * w[k1 * KS + k2];
  } else if (sx < sw && sx + KS > 0 && sy < sh && sy + KS > 0) {
#pragma unroll
    for (int k1 = 0; k1 < KS; ++k1) {
      if ((unsigned)(sy + k1) >= (unsigned)sh) continue;
      const uint8_t* q = src + (long long)(sy + k1) * spitch;
#pragma unroll
      for (int k2 = 0; k2 < KS; ++k2) {
        if ((unsigned)(sx + k2) >= (unsigned)sw) continue;
#pragma unroll
        for (int c = 0; c < C; ++c) sum[c] += tap8(q + (long long)(sx + k2) * C + c) * w[k1 * KS + k2];
      }
    }
  }
#pragma unroll
  for (int c = 0; c < C; ++c) o[c] = (uint8_t)max(0, min(255, (sum[c] + (1 << (COEF_BITS - 1))) >> COEF_BITS));
}

// The same pixel from a 16U, 16S or 32F source, in cv2's float arithmetic: weight vy[k1] * vx[k2], each tap times its
// weight rounded on its own, no contraction.  Inside the frame (the same fast-path test) a row's KS products are summed
// left to right; cubic then adds rows 1..3 onto row 0, Lanczos4 adds rows 0..7 onto +0 (so an all -0.0 window gives -0.0
// with cubic and +0.0 with Lanczos4).  Across an edge the sum starts at +0 and takes the in-frame taps one by one in
// row-major order; a window wholly outside is +0.  A NaN or inf tap inside the frame poisons the sum whatever its weight.
template <int KS, int C, class T, bool BD = false>
__host__ __device__ __forceinline__ void taps_px_f(const uint8_t* __restrict__ src, long long spitch, int sw, int sh, int sx,
                                                   int sy, const float (&vy)[KS], const float (&vx)[KS], uint8_t* __restrict__ o,
                                                   const Border& bd) {
  if constexpr (BD) {
    if (!((unsigned)sx < (unsigned)max(sw - (KS - 1), 0) && (unsigned)sy < (unsigned)max(sh - (KS - 1), 0))) {
      taps_px_f_edge<KS, C, T>(src, spitch, sw, sh, sx, sy, vy, vx, o, bd);
      return;
    }
  }
  constexpr int E = (int)sizeof(T);
  float sum[C];
#pragma unroll
  for (int c = 0; c < C; ++c) sum[c] = 0.f;
  if ((unsigned)sx < (unsigned)max(sw - (KS - 1), 0) && (unsigned)sy < (unsigned)max(sh - (KS - 1), 0)) {
    const uint8_t* q = src + (long long)sy * spitch + (long long)sx * (C * E);
#pragma unroll
    for (int k1 = 0; k1 < KS; ++k1, q += spitch) {
      float r[C];
#pragma unroll
      for (int k2 = 0; k2 < KS; ++k2) {
        const float w = fmul(vy[k1], vx[k2]);
#pragma unroll
        for (int c = 0; c < C; ++c) {
          const float t = fmul((float)ld_elem<T>(q + (k2 * C + c) * E), w);
          r[c] = k2 ? fadd(r[c], t) : t;
        }
      }
#pragma unroll
      for (int c = 0; c < C; ++c) sum[c] = (KS == 4 && k1 == 0) ? r[c] : fadd(sum[c], r[c]);
    }
  } else if (sx < sw && sx + KS > 0 && sy < sh && sy + KS > 0) {
#pragma unroll
    for (int k1 = 0; k1 < KS; ++k1) {
      if ((unsigned)(sy + k1) >= (unsigned)sh) continue;
      const uint8_t* q = src + (long long)(sy + k1) * spitch;
#pragma unroll
      for (int k2 = 0; k2 < KS; ++k2) {
        if ((unsigned)(sx + k2) >= (unsigned)sw) continue;
        const float w = fmul(vy[k1], vx[k2]);
#pragma unroll
        for (int c = 0; c < C; ++c) sum[c] = fadd(sum[c], fmul((float)ld_elem<T>(q + ((long long)(sx + k2) * C + c) * E), w));
      }
    }
  }
#pragma unroll
  for (int c = 0; c < C; ++c) st_sum<T>(o + c * E, sum[c]);
}

}  // namespace bevk
