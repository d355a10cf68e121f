// bevk_resize.cuh -- cv2.resize for 8-bit images (OpenCV 4.13): INTER_NEAREST, INTER_LINEAR and INTER_AREA, with the
// coordinates and weights computed per pixel from cv2's own formulas (DESIGN.md section 2), so the kernel needs no tables.
// Host-capable: tests/host/resize_affine.cu runs resize_frames over the device's grid.
//
// cv2 picks one of five bodies from the flag and the scales (resize_kind):
//   NEAREST      sx = min(floor(dx * scale_x), sw - 1), in double
//   LINEAR       11-bit weights of f = (float)((dx + 0.5) * scale - 0.5); an exact 2x2 downscale goes to AREA_FAST
//   AREA_LINEAR  INTER_AREA with a scale below 1 on either axis: LINEAR's weights, fractions from the cell edges
//   AREA_FAST    INTER_AREA at integer factors: the mean of the cell (2x2: (sum + 2) >> 2)
//   AREA         INTER_AREA at other downscales: float cell weights, summed per source row, then over the rows
#pragma once
#include <float.h>
#include <math.h>

#include "bevk_device.cuh"

namespace bevk {

enum { RZ_NEAREST = 0, RZ_LINEAR = 1, RZ_AREA_LINEAR = 2, RZ_AREA_FAST = 3, RZ_AREA = 4 };

struct ResizeArgs {
  const uint8_t* src; int sw, sh; long long spitch;
  uint8_t* dst; int dw, dh; long long dpitch;
  double scale_x, scale_y;   // 1 / inv_scale, as cv::resize computes them
  double inv_x, inv_y;       // inv_scale: dw / sw, or fx (dsize (0, 0))
  int ix, iy;                // AREA_FAST: the integer factors
  int n; long long sistride, distride;
};

// cv::resize's size rule: dsize (0, 0) takes dw = saturate_cast<int>(sw * fx) and keeps fx as the inverse scale; any
// other dsize gives inv = dw / sw.  false: an empty size or a non-positive scale (cv2 asserts).
inline bool resize_geometry(int sw, int sh, int* dw, int* dh, double* inv_x, double* inv_y) {
  if (*dw == 0 && *dh == 0) {
    if (!(*inv_x > 0) || !(*inv_y > 0)) return false;
    *dw = cv_round((double)sw * *inv_x);
    *dh = cv_round((double)sh * *inv_y);
  } else {
    *inv_x = (double)*dw / sw;
    *inv_y = (double)*dh / sh;
  }
  return *dw > 0 && *dh > 0;
}

// The body cv2 runs for interp (BEVK_INTER_NEAREST / _LINEAR / _AREA); fills a's scales and integer factors.
inline int resize_kind(int interp, ResizeArgs& a) {
  a.scale_x = 1. / a.inv_x;
  a.scale_y = 1. / a.inv_y;
  if (interp == 0) return RZ_NEAREST;
  a.ix = cv_round(a.scale_x);
  a.iy = cv_round(a.scale_y);
  const bool fast = fabs(a.scale_x - a.ix) < DBL_EPSILON && fabs(a.scale_y - a.iy) < DBL_EPSILON;
  if (interp == 1 && !(fast && a.ix == 2 && a.iy == 2)) return RZ_LINEAR;
  if (a.scale_x >= 1 && a.scale_y >= 1) return fast ? RZ_AREA_FAST : RZ_AREA;
  return RZ_AREA_LINEAR;
}

__host__ __device__ __forceinline__ int floor_d(double v) { return (int)floor(v); }
__host__ __device__ __forceinline__ int floor_f(float v) { return (int)floorf(v); }

// LINEAR / AREA_LINEAR along one axis: the first source index s and the 11-bit weights of s and s + 1.  Columns clamp
// (s < 0 or s >= size - 1 take f = 0 at the clamped s); rows keep their weights, and only their indices are clamped.
__host__ __device__ __forceinline__ void resize_lin_axis(bool area, double scale, double inv, int d, int size, bool clamp,
                                                         int& s, int& w0, int& w1) {
  float f;
  if (!area) {
    f = (float)dadd(dmul(dadd((double)d, 0.5), scale), -0.5);
    s = floor_f(f);
    f = fsub(f, (float)s);
  } else {
    s = floor_d(dmul((double)d, scale));
    f = (float)dadd((double)(d + 1), -dmul((double)(s + 1), inv));
    f = f <= 0.f ? 0.f : fsub(f, (float)floor_f(f));
  }
  if (clamp) {
    if (s < 0) f = 0.f, s = 0;
    if (s >= size - 1) f = 0.f, s = size - 1;
  }
  w0 = f2i_rn(fmul(fsub(1.f, f), 2048.f));
  w1 = f2i_rn(fmul(f, 2048.f));
}

// AREA along one axis: computeResizeAreaTab's entries of destination index d -- source indices [lo, hi), weight `head`
// for lo when has_head, `tail` for hi - 1 when has_tail, `mid` for the others -- in the order cv2 sums them.
struct AreaSpan { int lo, hi; bool has_head, has_tail; float head, mid, tail; };
__host__ __device__ __forceinline__ AreaSpan resize_area_axis(double scale, int d, int size) {
  const double fs1 = dmul((double)d, scale), fs2 = dadd(fs1, scale);
  const double cell = fmin(scale, dadd((double)size, -fs1));
  int s2 = floor_d(fs2);
  s2 = min(s2, size - 1);
  const int s1 = min((int)ceil(fs1), s2);
  AreaSpan a;
  a.has_head = dadd((double)s1, -fs1) > 1e-3;
  a.has_tail = dadd(fs2, -(double)s2) > 1e-3;
  a.head = (float)ddiv(dadd((double)s1, -fs1), cell);
  a.mid = (float)ddiv(1.0, cell);
  a.tail = (float)ddiv(fmin(fmin(dadd(fs2, -(double)s2), 1.), cell), cell);
  a.lo = a.has_head ? s1 - 1 : s1;
  a.hi = a.has_tail ? s2 + 1 : s2;
  return a;
}
__host__ __device__ __forceinline__ float area_weight(const AreaSpan& a, int s) {
  return (a.has_head && s == a.lo) ? a.head : (a.has_tail && s == a.hi - 1) ? a.tail : a.mid;
}

__host__ __device__ __forceinline__ int ld8(const uint8_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
__host__ __device__ __forceinline__ uint8_t sat_u8(int v) { return (uint8_t)max(0, min(255, v)); }

// One thread of k_resize: output pixel (x, y) of frames [f0, min(n, f0 + NB)).  The coordinates and weights depend on
// the pixel only and serve every frame of the group.
template <int C, int KIND, int NB>
__host__ __device__ __forceinline__ void resize_frames(const ResizeArgs& a, int x, int y, int f0) {
  const int nf = a.n - f0 < NB ? a.n - f0 : NB;
  const uint8_t* s = a.src + (long long)f0 * a.sistride;
  uint8_t* o = a.dst + (long long)f0 * a.distride + (long long)y * a.dpitch + (long long)x * C;
  if (KIND == RZ_NEAREST) {
    const int sx = min(floor_d(dmul((double)x, a.scale_x)), a.sw - 1);
    const int sy = min(floor_d(dmul((double)y, a.scale_y)), a.sh - 1);
    const long long off = (long long)sy * a.spitch + (long long)sx * C;
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride)
#pragma unroll
      for (int c = 0; c < C; ++c) o[c] = (uint8_t)ld8(s + off + c);
  } else if (KIND == RZ_LINEAR || KIND == RZ_AREA_LINEAR) {
    int sx, sy, a0, a1, b0, b1;
    resize_lin_axis(KIND == RZ_AREA_LINEAR, a.scale_x, a.inv_x, x, a.sw, true, sx, a0, a1);
    resize_lin_axis(KIND == RZ_AREA_LINEAR, a.scale_y, a.inv_y, y, a.sh, false, sy, b0, b1);
    const bool two = sx + 1 < a.sw;
    const long long r0 = (long long)max(0, min(a.sh - 1, sy)) * a.spitch + (long long)sx * C;
    const long long r1 = (long long)max(0, min(a.sh - 1, sy + 1)) * a.spitch + (long long)sx * C;
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride)
#pragma unroll
      for (int c = 0; c < C; ++c) {
        // HResizeLinear in int, then VResizeLinear's SIMD step: int16 high-half products of (H >> 4) and the weights
        const int h0 = ld8(s + r0 + c) * a0 + (two ? ld8(s + r0 + C + c) * a1 : 0);
        const int h1 = ld8(s + r1 + c) * a0 + (two ? ld8(s + r1 + C + c) * a1 : 0);
        o[c] = sat_u8((((h0 >> 4) * b0 >> 16) + ((h1 >> 4) * b1 >> 16) + 2) >> 2);
      }
  } else if (KIND == RZ_AREA_FAST) {
    const int sx0 = x * a.ix, sy0 = y * a.iy;
    const bool full = sy0 + a.iy <= a.sh && x < a.sw / a.ix;
    const int area = a.ix * a.iy;
    const float inv_area = 1.f / (float)area;
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride)
#pragma unroll
      for (int c = 0; c < C; ++c) {
        int sum = 0, count = 0;
        for (int j = 0; j < a.iy && sy0 + j < a.sh; ++j)
          for (int i = 0; i < a.ix && sx0 + i < a.sw; ++i, ++count)
            sum += ld8(s + (long long)(sy0 + j) * a.spitch + (long long)(sx0 + i) * C + c);
        // whole cells: the 2x2 vector body rounds half up, the others cvRound(sum * (1.f / area)); the cells cut by
        // the right or bottom edge: cvRound((float)sum / count)
        o[c] = !full ? sat_u8(f2i_rn(count ? (float)sum / (float)count : 0.f))
                     : area == 4 ? (uint8_t)((sum + 2) >> 2) : sat_u8(f2i_rn(fmul((float)sum, inv_area)));
      }
  } else {   // RZ_AREA
    const AreaSpan ax = resize_area_axis(a.scale_x, x, a.sw), ay = resize_area_axis(a.scale_y, y, a.sh);
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride) {
      float sum[C];
#pragma unroll
      for (int c = 0; c < C; ++c) sum[c] = 0.f;
      for (int sy = ay.lo; sy < ay.hi; ++sy) {
        const float beta = area_weight(ay, sy);
        const uint8_t* row = s + (long long)sy * a.spitch;
        float buf[C];
#pragma unroll
        for (int c = 0; c < C; ++c) buf[c] = 0.f;
        for (int sx = ax.lo; sx < ax.hi; ++sx) {
          const float alpha = area_weight(ax, sx);
#pragma unroll
          for (int c = 0; c < C; ++c) buf[c] = fadd(buf[c], fmul((float)ld8(row + (long long)sx * C + c), alpha));
        }
#pragma unroll
        for (int c = 0; c < C; ++c) sum[c] = fadd(sum[c], fmul(beta, buf[c]));
      }
#pragma unroll
      for (int c = 0; c < C; ++c) o[c] = sat_u8(f2i_rn(sum[c]));
    }
  }
}

#ifdef __CUDACC__
// grid (ceil(dw / 32), ceil(dh / 8), ceil(n / NB)), 256 threads: one output pixel per thread, NB frames per grid-z slice
template <int C, int KIND, int NB>
__global__ void __launch_bounds__(256) k_resize(ResizeArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.dw || y >= a.dh) return;
  resize_frames<C, KIND, NB>(a, x, y, blockIdx.z * NB);
}
#endif

}  // namespace bevk
