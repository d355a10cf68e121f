// bevk_kernels.cuh -- the sm_90a kernels behind libbevk.so.
//
//   k_undistort_map   K1  cv2.fisheye.initUndistortRectifyMap / cv2.initUndistortRectifyMap
//   k_gather          K3/K4  cv2.remap, fused undistort (no map), cv2.warpPerspective / cv2.warpAffine on images
//   k_gather_taps     K3/K4  the same with INTER_CUBIC / INTER_LANCZOS4
//   k_warp_maps       K2  cv2.warpPerspective on the 16SC2/16UC1 map planes (BEV LUT build),
//                         optionally fused with K1 so the full-size undistort map never exists
//   k_blend_masks     K10 BlendMask.get_blend_mask
//   k_vsum / k_delta  K8  per-camera sum of V = max(B,G,R) and the luminance offsets
//   k_bev             K3+K5+K6+K7(+K8 per tap): the fused per-frame kernel
//   k_gain            K9  grey-world gains + car overlay
//   k_sat_sum         multi-GPU compose of per-camera partial canvases
#pragma once
#include "bevk_device.cuh"
#include "bevk_interp.cuh"

#include <type_traits>

namespace bevk {

constexpr int BEVK_MAX_CAMERAS_K = 8;   // == BEVK_MAX_CAMERAS in include/bevk.h

// ---------------------------------------------------------------------------------
// K1
// ---------------------------------------------------------------------------------
// The camera model's CV_16SC2 + CV_16UC1 map entry of pixel (x, y), as cv2.initUndistortRectifyMap stores it.  Every
// in-kernel evaluation of the model (the map build, the fused gathers' MODE 1, k_warp_maps' fused taps) goes through it.
template <int LENS>
__host__ __device__ __forceinline__ void model_entry(const CamModel& cm, const LensExt& lx, int x, int y, short& mx, short& my,
                                                     unsigned short& fr) {
  double u, v;
  undistort_point<LENS>(cm, lx, x, y, u, v);
  quantise_uv(u, v, mx, my, fr, pack_saturates(cm.model, x, cm.w));
}

// The camera model's CV_32FC1 / CV_32FC2 map entry of pixel (x, y): cv2 stores (float)u, (float)v of the very (u, v)
// the CV_16SC2 build quantises.
template <int LENS>
__host__ __device__ __forceinline__ void model_entry_f32(const CamModel& cm, const LensExt& lx, int x, int y, float& fx,
                                                         float& fy) {
  double u, v;
  undistort_point<LENS>(cm, lx, x, y, u, v);
  fx = d2f(u); fy = d2f(v);
}

template <int LENS>
__global__ void __launch_bounds__(256) k_undistort_map(CamModel cm, LensExt lx, short2* __restrict__ map1,
                                                       unsigned short* __restrict__ map2) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= cm.w || y >= cm.h) return;
  short mx, my;
  unsigned short fr;
  model_entry<LENS>(cm, lx, x, y, mx, my, fr);
  const size_t i = (size_t)y * cm.w + x;
  map1[i] = make_short2(mx, my);
  map2[i] = fr;
}

// K1 into CV_32FC1 (map2 = the y plane) or CV_32FC2 (map2 null, map1 interleaved).
template <int LENS>
__host__ __device__ __forceinline__ void undistort_map_f32_px(const CamModel& cm, const LensExt& lx, int x, int y,
                                                             float* __restrict__ map1, float* __restrict__ map2) {
  float fx, fy;
  model_entry_f32<LENS>(cm, lx, x, y, fx, fy);
  const size_t i = (size_t)y * cm.w + x;
  if (map2) { map1[i] = fx; map2[i] = fy; }
  else { map1[2 * i] = fx; map1[2 * i + 1] = fy; }
}

template <int LENS>
__global__ void __launch_bounds__(256) k_undistort_map_f32(CamModel cm, LensExt lx, float* __restrict__ map1,
                                                           float* __restrict__ map2) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= cm.w || y >= cm.h) return;
  undistort_map_f32_px<LENS>(cm, lx, x, y, map1, map2);
}

// cv2.convertMaps between CV_16SC2 (+ CV_16UC1), CV_32FC1 and CV_32FC2, one map entry per thread.  Map types are cv2's
// values (BEVK_CV_*); a float source is read as (x, y), a CV_16SC2 one as its exact float value (unquantise_xy).
constexpr int MAP_16SC2 = 11, MAP_32FC1 = 5, MAP_32FC2 = 13;
struct ConvertMapsArgs {
  const void* in1; const void* in2; int intype;   // in2: CV_16UC1 (may be null) or the y plane of CV_32FC1
  void* out1; void* out2; int outtype;            // out2: CV_16UC1 (null with nn) or the y plane of CV_32FC1
  bool nn;                                        // nninterpolation: CV_16SC2 without map2, rounded to whole pixels
  long long n;
};

__host__ __device__ __forceinline__ void convert_map_px(const ConvertMapsArgs& a, long long i) {
  float x, y;
  if (a.intype == MAP_16SC2) {
    const short2 m = static_cast<const short2*>(a.in1)[i];
    unquantise_xy(m.x, m.y, a.in2 ? static_cast<const unsigned short*>(a.in2)[i] : 0u, x, y);
  } else if (a.intype == MAP_32FC2) {
    x = static_cast<const float*>(a.in1)[2 * i]; y = static_cast<const float*>(a.in1)[2 * i + 1];
  } else {
    x = static_cast<const float*>(a.in1)[i]; y = static_cast<const float*>(a.in2)[i];
  }
  if (a.outtype == MAP_16SC2) {
    short mx, my;
    unsigned short fr;
    quantise_xy(x, y, a.nn, mx, my, fr);
    static_cast<short2*>(a.out1)[i] = make_short2(mx, my);
    if (!a.nn) static_cast<unsigned short*>(a.out2)[i] = fr;
  } else if (a.outtype == MAP_32FC2) {
    static_cast<float*>(a.out1)[2 * i] = x; static_cast<float*>(a.out1)[2 * i + 1] = y;
  } else {
    static_cast<float*>(a.out1)[i] = x; static_cast<float*>(a.out2)[i] = y;
  }
}

__global__ void __launch_bounds__(256) k_convert_maps(ConvertMapsArgs a) {
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < a.n; i += (long long)gridDim.x * 256) convert_map_px(a, i);
}

// K1 set-up of a camera whose rays depend on the row (LensExt::rays): one thread walks one row.
template <int MODEL>
__global__ void __launch_bounds__(128) k_walk_rays(CamModel cm, double* __restrict__ rays) {
  const int i = blockIdx.x * 128 + threadIdx.x;
  if (i < cm.h) walk_rays<MODEL>(cm, i, rays);
}

// ---------------------------------------------------------------------------------
// K3 / K4: generic gather.  MODE 0: maps in HBM, 1: camera model evaluated in-kernel
// (fused undistort), 2: homography (warpPerspective), 3: affine matrix (warpAffine, inverse in hm.M[0..5]),
// 4: CV_32FC1 / CV_32FC2 maps in HBM, 5: camera model rounded to float as a float map holds it.  MODE 4 and 5 resolve
// their taps as cv2.remap converts float maps (quantise_xy).
// Over a batch of n frames: the taps of an output pixel depend on the pixel only, so a thread
// resolves them once (map load or camera model) and gathers them from GATHER_NB frames of its
// grid-z slice.  Frame f is read at src + f * sistride and written at dst + f * distride.
// ---------------------------------------------------------------------------------
struct GatherArgs {
  const uint8_t* src; int sw, sh; long long spitch;
  uint8_t* dst; int dw, dh; long long dpitch;
  // MODE 0: CV_16SC2 + CV_16UC1 (map2 may be null for NEAREST); MODE 4: x and y planes (CV_32FC1), or fmap2 null and
  // (x, y) pairs in fmap1 (CV_32FC2).  Unions, so that the arguments of every other MODE keep their offsets.
  union { const short2* map1; const float* fmap1; };
  union { const unsigned short* map2; const float* fmap2; };
  CamModel cm;
  LensExt lx;                            // MODE 1 with LENS = 1 only
  Homog hm;
  int n; long long sistride, distride;   // frames, and the 64-bit image strides of source and destination
  Border bd;                             // taps outside the source (border_window); zero-initialised: BORDER_CONSTANT 0
};

// Frames per thread (grid.z = ceil(n / GATHER_NB)); DESIGN.md section 4 has the measurement that chose it.
#ifndef BEVK_GATHER_NB
#define BEVK_GATHER_NB 8
#endif
constexpr int GATHER_NB = BEVK_GATHER_NB;

// MODE 2 / 3: the fixed-point source position of destination pixel (x, y), at TAB scale or (nearest) in whole pixels.
template <int MODE>
__host__ __device__ __forceinline__ void warp_xy(const Homog& hm, int x, int y, bool nearest, int& X, int& Y) {
  if (MODE == 3) affine_point(hm, x, y, nearest, X, Y);
  else warp_point(hm, x, y, nearest ? 1.0 : (double)TAB, X, Y);
}

// A CV_16SC2 + CV_16UC1 map entry as source pixel (sx, sy) and 1/32 fractions (fx, fy).  nn_delta: INTER_NEAREST
// through an entry that has a fraction, which moves the pixel by OpenCV's NNDeltaTab_i -- inverted: frac < 16 picks the
// +1 neighbour.
__host__ __device__ __forceinline__ void split_entry(short mx, short my, unsigned short fr, bool nn_delta, int& sx, int& sy,
                                                     int& fx, int& fy) {
  sx = mx; sy = my;
  fx = fr & (TAB - 1); fy = (fr >> INTER_BITS) & (TAB - 1);
  if (nn_delta) { sx += (fx < 16); sy += (fy < 16); }
}

// The source position of output pixel (x, y) in every MODE: source pixel (sx, sy) and 1/32 fractions (fx, fy), as
// cv2.remap / cv2.warpPerspective / cv2.warpAffine pick them.  MODE 0 reads the map entry, MODE 1 evaluates the camera
// model (model_entry), MODE 4 and 5 quantise a float map entry or the model rounded to float (model_entry_f32) as
// cv2.remap converts float maps (quantise_xy), MODE 2 / 3 warp the pixel (warp_xy).  nearest (INTER_NEAREST): MODE 0 / 1
// apply NNDeltaTab when the entry has a fraction (map2 may be null only then), MODE 4 / 5 round to whole pixels with no
// fraction, MODE 2 / 3 warp in whole pixels; (fx, fy) are then 0 or unused.
template <int MODE, int LENS>
__host__ __device__ __forceinline__ void source_pos(const GatherArgs& a, int x, int y, bool nearest, int& sx, int& sy, int& fx,
                                                    int& fy) {
  if (MODE == 2 || MODE == 3) {
    int X, Y;
    warp_xy<MODE>(a.hm, x, y, nearest, X, Y);
    if (nearest) { sx = sat_i16(X); sy = sat_i16(Y); fx = fy = 0; }
    else {
      sx = sat_i16(X >> INTER_BITS); sy = sat_i16(Y >> INTER_BITS);
      fx = X & (TAB - 1); fy = Y & (TAB - 1);
    }
    return;
  }
  short mx, my;
  unsigned short fr;
  bool frac = true;
  if (MODE == 0) {
    const size_t i = (size_t)y * a.dw + x;
    const short2 m = a.map1[i];
    mx = m.x; my = m.y;
    frac = !nearest || a.map2 != nullptr;
    fr = frac ? a.map2[i] : 0;
  } else if (MODE == 1) {
    model_entry<LENS>(a.cm, a.lx, x, y, mx, my, fr);
  } else {
    float X, Y;
    if (MODE == 4) {
      const size_t i = (size_t)y * a.dw + x;
      if (a.fmap2) { X = a.fmap1[i]; Y = a.fmap2[i]; }
      else { X = a.fmap1[2 * i]; Y = a.fmap1[2 * i + 1]; }
    } else {
      model_entry_f32<LENS>(a.cm, a.lx, x, y, X, Y);
    }
    quantise_xy(X, Y, nearest, mx, my, fr);
    frac = !nearest;
  }
  split_entry(mx, my, fr, nearest && frac, sx, sy, fx, fy);
}

template <int C>
__host__ __device__ __forceinline__ void load_px(const uint8_t* __restrict__ src, long long spitch, int sw, int sh,
                                                 int x, int y, int (&p)[C]) {
  if ((unsigned)x < (unsigned)sw && (unsigned)y < (unsigned)sh) {
    const uint8_t* q = src + (long long)y * spitch + (long long)x * C;
#ifdef __CUDA_ARCH__
#pragma unroll
    for (int c = 0; c < C; ++c) p[c] = __ldg(q + c);
#else
    for (int c = 0; c < C; ++c) p[c] = q[c];
#endif
  } else {
#pragma unroll
    for (int c = 0; c < C; ++c) p[c] = 0;
  }
}

// load_px of a 16U, 16S or 32F pixel, as float; a tap outside the frame is +0 (cv2's BORDER_CONSTANT value)
template <int C, class T>
__host__ __device__ __forceinline__ void load_px_f(const uint8_t* __restrict__ src, long long spitch, int sw, int sh,
                                                   int x, int y, float (&p)[C]) {
  const bool in = (unsigned)x < (unsigned)sw && (unsigned)y < (unsigned)sh;
  const uint8_t* q = src + (long long)y * spitch + (long long)x * (C * (int)sizeof(T));
#pragma unroll
  for (int c = 0; c < C; ++c) p[c] = in ? (float)ld_elem<T>(q + c * sizeof(T)) : 0.f;
}

// One thread of k_gather: output pixel (x, y) of frames [f0, min(n, f0 + GATHER_NB)).  Host-capable, so that
// tests/host/undistort_stack.cu runs the same frame loop and addressing on a CPU.
// LENS (MODE 1): the camera model's instance, undistort_point<LENS>.  T: the source and destination element, uint8_t or
// (tests/host/remap_depth.cu) uint16_t, int16_t, float.  The taps are T-independent: cv2 quantises to 1/32 px at every
// depth.  8-bit LINEAR is the Q10 sum; the wider depths take cv2's float bilinear (gather_px_f).
template <int MODE, int C, int LINEAR, int LENS = 0, class T = uint8_t>
__host__ __device__ __forceinline__ void gather_frames(const GatherArgs& a, int x, int y, int f0) {
  int sx, sy, fx, fy;
  source_pos<MODE, LENS>(a, x, y, !LINEAR, sx, sy, fx, fy);
  constexpr int PX = C * (int)sizeof(T);   // bytes per pixel
  const int nf = a.n - f0 < GATHER_NB ? a.n - f0 : GATHER_NB;
  const uint8_t* s = a.src + (long long)f0 * a.sistride;
  uint8_t* o = a.dst + (long long)f0 * a.distride + (long long)y * a.dpitch + (long long)x * PX;
  if constexpr (sizeof(T) == 1) {
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride) {
      if (LINEAR) {
        int p00[C], p01[C], p10[C], p11[C];
        load_px<C>(s, a.spitch, a.sw, a.sh, sx, sy, p00);
        load_px<C>(s, a.spitch, a.sw, a.sh, sx + 1, sy, p01);
        load_px<C>(s, a.spitch, a.sw, a.sh, sx, sy + 1, p10);
        load_px<C>(s, a.spitch, a.sw, a.sh, sx + 1, sy + 1, p11);
#pragma unroll
        for (int c = 0; c < C; ++c) o[c] = (uint8_t)bilerp_q10(p00[c], p01[c], p10[c], p11[c], fx, fy);
      } else {
        int p[C];
        load_px<C>(s, a.spitch, a.sw, a.sh, sx, sy, p);
#pragma unroll
        for (int c = 0; c < C; ++c) o[c] = (uint8_t)p[c];
      }
    }
  } else if constexpr (LINEAR) {
    // cv2's float table: w = vy * vx with vx = {1 - fx / 32, fx / 32}, each product rounded to float
    const float ax = fmul((float)fx, 1.f / TAB), ay = fmul((float)fy, 1.f / TAB);
    const float bx = fsub(1.f, ax), by = fsub(1.f, ay);
    const float w00 = fmul(by, bx), w01 = fmul(by, ax), w10 = fmul(ay, bx), w11 = fmul(ay, ax);
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride) {
      float p00[C], p01[C], p10[C], p11[C];
      load_px_f<C, T>(s, a.spitch, a.sw, a.sh, sx, sy, p00);
      load_px_f<C, T>(s, a.spitch, a.sw, a.sh, sx + 1, sy, p01);
      load_px_f<C, T>(s, a.spitch, a.sw, a.sh, sx, sy + 1, p10);
      load_px_f<C, T>(s, a.spitch, a.sw, a.sh, sx + 1, sy + 1, p11);
#pragma unroll
      for (int c = 0; c < C; ++c)   // ((t00 w00 + t01 w01) + t10 w10) + t11 w11, taps outside the frame 0
        st_sum<T>(o + c * sizeof(T), fadd(fadd(fadd(fmul(p00[c], w00), fmul(p01[c], w01)), fmul(p10[c], w10)), fmul(p11[c], w11)));
    }
  } else {
    // NEAREST moves the element's bits: a float NaN keeps its payload, -0.0 its sign; outside the frame 0
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride) {
      const bool in = (unsigned)sx < (unsigned)a.sw && (unsigned)sy < (unsigned)a.sh;
      const uint8_t* q = s + (long long)sy * a.spitch + (long long)sx * PX;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const T v = in ? ld_elem<T>(q + c * sizeof(T)) : (T)0;
#ifdef __CUDA_ARCH__
        reinterpret_cast<T*>(o)[c] = v;
#else
        memcpy(o + c * sizeof(T), &v, sizeof v);
#endif
      }
    }
  }
}

// One tap of k_gather at source column x and row y as border_window resolves them (-1: the border value), as ints (8-bit)
// or as floats (16U, 16S, 32F)
template <int C>
__host__ __device__ __forceinline__ void load_tap(const uint8_t* __restrict__ src, long long spitch, int x, int y,
                                                 const Border& bd, int (&p)[C]) {
  if ((x | y) >= 0) {
    const uint8_t* q = src + (long long)y * spitch + (long long)x * C;
#ifdef __CUDA_ARCH__
#pragma unroll
    for (int c = 0; c < C; ++c) p[c] = __ldg(q + c);
#else
    for (int c = 0; c < C; ++c) p[c] = q[c];
#endif
  } else {
#pragma unroll
    for (int c = 0; c < C; ++c) p[c] = bd.v[c];
  }
}

template <int C, class T>
__host__ __device__ __forceinline__ void load_tap_f(const uint8_t* __restrict__ src, long long spitch, int x, int y,
                                                   const Border& bd, float (&p)[C]) {
  const bool in = (x | y) >= 0;
  const uint8_t* q = src + (long long)y * spitch + (long long)x * (C * (int)sizeof(T));
#pragma unroll
  for (int c = 0; c < C; ++c) p[c] = (float)(in ? ld_elem<T>(q + c * sizeof(T)) : border_elem<T>(bd, c));
}

// gather_frames under a border other than a zero BORDER_CONSTANT (k_gather_border): the border (a.bd) is resolved once
// per pixel for all its frames -- the taps' source columns and rows, the border value, or no write at all.  NEAREST
// through an entry with a fraction wraps NNDeltaTab's +1 to int16, as cv2's map buffer does (32767 + 1 reads -32768);
// every other position is int16 already.
template <int MODE, int C, int LINEAR, int LENS = 0, class T = uint8_t>
__host__ __device__ __forceinline__ void gather_frames_border(const GatherArgs& a, int x, int y, int f0) {
  int sx, sy, fx, fy;
  source_pos<MODE, LENS>(a, x, y, !LINEAR, sx, sy, fx, fy);
  if (!LINEAR) { sx = (short)sx; sy = (short)sy; }
  constexpr int K = LINEAR ? 2 : 1;
  int xs[K], ys[K];
  const int act = border_window<K>(a.bd, sx, sy, a.sw, a.sh, xs, ys);
  if (act == BW_SKIP) return;
  constexpr int PX = C * (int)sizeof(T);   // bytes per pixel
  const int nf = a.n - f0 < GATHER_NB ? a.n - f0 : GATHER_NB;
  const uint8_t* s = a.src + (long long)f0 * a.sistride;
  uint8_t* o = a.dst + (long long)f0 * a.distride + (long long)y * a.dpitch + (long long)x * PX;
  if (act == BW_FILL) {
    for (int f = 0; f < nf; ++f, o += a.distride) st_border<C, T>(o, a.bd);
    return;
  }
  if constexpr (sizeof(T) == 1) {
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride) {
      if (LINEAR) {
        int p00[C], p01[C], p10[C], p11[C];
        load_tap<C>(s, a.spitch, xs[0], ys[0], a.bd, p00);
        load_tap<C>(s, a.spitch, xs[K - 1], ys[0], a.bd, p01);
        load_tap<C>(s, a.spitch, xs[0], ys[K - 1], a.bd, p10);
        load_tap<C>(s, a.spitch, xs[K - 1], ys[K - 1], a.bd, p11);
#pragma unroll
        for (int c = 0; c < C; ++c) o[c] = (uint8_t)bilerp_q10(p00[c], p01[c], p10[c], p11[c], fx, fy);
      } else {
        int p[C];
        load_tap<C>(s, a.spitch, xs[0], ys[0], a.bd, p);
#pragma unroll
        for (int c = 0; c < C; ++c) o[c] = (uint8_t)p[c];
      }
    }
  } else if constexpr (LINEAR) {
    // cv2's float table: w = vy * vx with vx = {1 - fx / 32, fx / 32}, each product rounded to float
    const float ax = fmul((float)fx, 1.f / TAB), ay = fmul((float)fy, 1.f / TAB);
    const float bx = fsub(1.f, ax), by = fsub(1.f, ay);
    const float w00 = fmul(by, bx), w01 = fmul(by, ax), w10 = fmul(ay, bx), w11 = fmul(ay, ax);
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride) {
      float p00[C], p01[C], p10[C], p11[C];
      load_tap_f<C, T>(s, a.spitch, xs[0], ys[0], a.bd, p00);
      load_tap_f<C, T>(s, a.spitch, xs[K - 1], ys[0], a.bd, p01);
      load_tap_f<C, T>(s, a.spitch, xs[0], ys[K - 1], a.bd, p10);
      load_tap_f<C, T>(s, a.spitch, xs[K - 1], ys[K - 1], a.bd, p11);
#pragma unroll
      for (int c = 0; c < C; ++c)   // ((t00 w00 + t01 w01) + t10 w10) + t11 w11, taps outside the frame the border value
        st_sum<T>(o + c * sizeof(T), fadd(fadd(fadd(fmul(p00[c], w00), fmul(p01[c], w01)), fmul(p10[c], w10)), fmul(p11[c], w11)));
    }
  } else {
    // NEAREST moves the element's bits: a float NaN keeps its payload, -0.0 its sign
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride) {
      const uint8_t* q = s + (long long)ys[0] * a.spitch + (long long)xs[0] * PX;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const T v = (xs[0] | ys[0]) >= 0 ? ld_elem<T>(q + c * sizeof(T)) : border_elem<T>(a.bd, c);
#ifdef __CUDA_ARCH__
        reinterpret_cast<T*>(o)[c] = v;
#else
        memcpy(o + c * sizeof(T), &v, sizeof v);
#endif
      }
    }
  }
}

template <int MODE, int C, int LINEAR, int LENS, class T>
__global__ void __launch_bounds__(256) k_gather(GatherArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.dw || y >= a.dh) return;
  gather_frames<MODE, C, LINEAR, LENS, T>(a, x, y, blockIdx.z * GATHER_NB);
}

// k_gather under cv2's other border modes and values: a kernel of its own, so that the zero-constant instances keep
// their machine code and speed
template <int MODE, int C, int LINEAR, int LENS, class T>
__global__ void __launch_bounds__(256) k_gather_border(GatherArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.dw || y >= a.dh) return;
  gather_frames_border<MODE, C, LINEAR, LENS, T>(a, x, y, blockIdx.z * GATHER_NB);
}

// The weights k_gather_taps reads: 8-bit sources the int16 2-D rows of build_interp_tabs, wider ones the float 1-D rows
// of build_interp_rows.
template <class T>
using TapWeights = typename std::conditional<sizeof(T) == 1, short, float>::type;

// K3 / K4 with INTER_CUBIC (KS = 4) and INTER_LANCZOS4 (KS = 8): the source position is INTER_LINEAR's (map entry, camera
// model, or warp_point at TAB scale), the map2 value picks a row of KS * KS int16 weights from wtab (bevk_interp.cuh,
// 32 or 128 bytes read once per pixel through the read-only path), and the row and window serve up to GATHER_NB frames.
// A 16U, 16S or 32F source instead reads the fraction's two 1-D float rows (2 * KS floats) and forms each 2-D weight as
// cv2's float table holds it (taps_px_f): 2 * KS registers rather than KS * KS.
// Host-capable, like gather_frames (tests/host/remap_interp.cu, tests/host/remap_depth.cu).
template <int MODE, int C, int KS, int LENS = 0, class T = uint8_t, bool BD = false>
__host__ __device__ __forceinline__ void gather_taps_frames(const GatherArgs& a, const TapWeights<T>* __restrict__ wtab, int x,
                                                            int y, int f0) {
  int sx, sy, fx, fy;
  source_pos<MODE, LENS>(a, x, y, false, sx, sy, fx, fy);
  sx -= KS / 2 - 1; sy -= KS / 2 - 1;
  if constexpr (sizeof(T) == 1) {
    const unsigned fr = (unsigned)(fy * TAB + fx);
    short w[KS * KS];
#ifdef __CUDA_ARCH__
    const uint4* wr = reinterpret_cast<const uint4*>(wtab + fr * (KS * KS));
#pragma unroll
    for (int i = 0; i < KS * KS / 8; ++i) {
      const uint4 q = __ldg(wr + i);
      const unsigned u[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) { w[8 * i + 2 * k] = (short)(u[k] & 0xffffu); w[8 * i + 2 * k + 1] = (short)(u[k] >> 16); }
    }
#else
    memcpy(w, wtab + fr * (KS * KS), sizeof w);
#endif
    const int nf = a.n - f0 < GATHER_NB ? a.n - f0 : GATHER_NB;
    const uint8_t* s = a.src + (long long)f0 * a.sistride;
    uint8_t* o = a.dst + (long long)f0 * a.distride + (long long)y * a.dpitch + (long long)x * (C * (int)sizeof(T));
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride) taps_px<KS, C, BD>(s, a.spitch, a.sw, a.sh, sx, sy, w, o, a.bd);
  } else {
    float vy[KS], vx[KS];
    const float* ry = wtab + fy * KS;
    const float* rx = wtab + fx * KS;
#ifdef __CUDA_ARCH__
#pragma unroll
    for (int i = 0; i < KS / 4; ++i) {
      const float4 qy = __ldg(reinterpret_cast<const float4*>(ry) + i), qx = __ldg(reinterpret_cast<const float4*>(rx) + i);
      vy[4 * i] = qy.x; vy[4 * i + 1] = qy.y; vy[4 * i + 2] = qy.z; vy[4 * i + 3] = qy.w;
      vx[4 * i] = qx.x; vx[4 * i + 1] = qx.y; vx[4 * i + 2] = qx.z; vx[4 * i + 3] = qx.w;
    }
#else
    memcpy(vy, ry, sizeof vy);
    memcpy(vx, rx, sizeof vx);
#endif
    const int nf = a.n - f0 < GATHER_NB ? a.n - f0 : GATHER_NB;
    const uint8_t* s = a.src + (long long)f0 * a.sistride;
    uint8_t* o = a.dst + (long long)f0 * a.distride + (long long)y * a.dpitch + (long long)x * (C * (int)sizeof(T));
    for (int f = 0; f < nf; ++f, s += a.sistride, o += a.distride) taps_px_f<KS, C, T, BD>(s, a.spitch, a.sw, a.sh, sx, sy, vy, vx, o, a.bd);
  }
}

template <int MODE, int C, int KS, int LENS, class T>
__global__ void __launch_bounds__(256) k_gather_taps(GatherArgs a, const TapWeights<T>* __restrict__ wtab) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.dw || y >= a.dh) return;
  gather_taps_frames<MODE, C, KS, LENS, T>(a, wtab, x, y, blockIdx.z * GATHER_NB);
}

// k_gather_taps under cv2's other border modes and values (BD: the edge windows follow border_window)
template <int MODE, int C, int KS, int LENS, class T>
__global__ void __launch_bounds__(256) k_gather_taps_border(GatherArgs a, const TapWeights<T>* __restrict__ wtab) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.dw || y >= a.dh) return;
  gather_taps_frames<MODE, C, KS, LENS, T, true>(a, wtab, x, y, blockIdx.z * GATHER_NB);
}

// ---------------------------------------------------------------------------------
// K2: warpPerspective of the map planes.  FROM_MODEL=1 evaluates the undistort map at
// the four taps instead of reading und_w x und_h planes from HBM (fused K1+K2).
// ---------------------------------------------------------------------------------
struct WarpMapsArgs {
  const short2* in1; const unsigned short* in2; int sw, sh;   // FROM_MODEL=0
  CamModel cm;                                                // FROM_MODEL=1 (sw,sh = cm.w,cm.h)
  LensExt lx;                                                 // FROM_MODEL=1 with LENS = 1 only
  Homog hm;
  short2* out1; unsigned short* out2; int dw, dh;
};

// One destination pixel of that warp (host-capable: tests/host/kernel_math.cu runs it on a CPU against cv2).
template <int FROM_MODEL, int LENS = 0>
__host__ __device__ __forceinline__ void warp_maps_pixel(const WarpMapsArgs& a, int x, int y, short& ox, short& oy,
                                                         unsigned short& of) {
  int X, Y;
  warp_point(a.hm, x, y, (double)TAB, X, Y);
  const int sx = sat_i16(X >> INTER_BITS), sy = sat_i16(Y >> INTER_BITS);
  const float ax = fmul((float)(X & (TAB - 1)), 1.0f / TAB);
  const float ay = fmul((float)(Y & (TAB - 1)), 1.0f / TAB);
  const float w[4] = {fmul(fsub(1.f, ay), fsub(1.f, ax)), fmul(fsub(1.f, ay), ax), fmul(ay, fsub(1.f, ax)), fmul(ay, ax)};
  float accx = 0.f, accy = 0.f, accf = 0.f;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int tx = sx + (t & 1), ty = sy + (t >> 1);
    float vx = 0.f, vy = 0.f, vf = 0.f;
    if ((unsigned)tx < (unsigned)a.sw && (unsigned)ty < (unsigned)a.sh) {
      short mx, my;
      unsigned short fr;
      if (FROM_MODEL) {
        model_entry<LENS>(a.cm, a.lx, tx, ty, mx, my, fr);
      } else {
        const size_t i = (size_t)ty * a.sw + tx;
        const short2 m = a.in1[i];
        mx = m.x; my = m.y; fr = a.in2[i];
      }
      vx = (float)mx; vy = (float)my; vf = (float)fr;
    }
    // acc = ((t0*w0 + t1*w1) + t2*w2) + t3*w3, each product and sum rounded (no FMA)
    if (t == 0) { accx = fmul(vx, w[0]); accy = fmul(vy, w[0]); accf = fmul(vf, w[0]); }
    else {
      accx = fadd(accx, fmul(vx, w[t]));
      accy = fadd(accy, fmul(vy, w[t]));
      accf = fadd(accf, fmul(vf, w[t]));
    }
  }
  ox = (short)sat_i16(f2i_rn(accx));
  oy = (short)sat_i16(f2i_rn(accy));
  const int fi = f2i_rn(accf);
  of = (unsigned short)(fi < 0 ? 0 : (fi > 65535 ? 65535 : fi));
}

template <int FROM_MODEL, int LENS>
__global__ void __launch_bounds__(256) k_warp_maps(WarpMapsArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.dw || y >= a.dh) return;
  short ox, oy;
  unsigned short of;
  warp_maps_pixel<FROM_MODEL, LENS>(a, x, y, ox, oy, of);
  const size_t o = (size_t)y * a.dw + x;
  a.out1[o] = make_short2(ox, oy);
  a.out2[o] = of;
}

// ---------------------------------------------------------------------------------
// K10: blend weights.  polys/out: uint8[4][h][w]; lines: int[8][4] = (ax,ay,bx,by) for
// FL,FR,BL,BR,LF,LB,RF,RB.
// ---------------------------------------------------------------------------------
struct BlendArgs { const uint8_t* polys; uint8_t* out; int w, h; int lines[8][4]; };

__host__ __device__ __forceinline__ double seg_dist(double px, double py, const int* L) {
  const double ax = L[0], ay = L[1], bx = L[2], by = L[3];
  const double dx = bx - ax, dy = by - ay;
  const double d1x = px - ax, d1y = py - ay, d2x = px - bx, d2y = py - by;
  double sq;
  if (dadd(dmul(d1x, dx), dmul(d1y, dy)) <= 0) sq = dadd(dmul(d1x, d1x), dmul(d1y, d1y));
  else if (dadd(dmul(d2x, dx), dmul(d2y, dy)) >= 0) sq = dadd(dmul(d2x, d2x), dmul(d2y, d2y));
  else {
    const double cr = dadd(dmul(d1y, dx), -dmul(d1x, dy));
    sq = ddiv(dmul(cr, cr), dadd(dmul(dx, dx), dmul(dy, dy)));
  }
  return dsqrt(sq);
}

// One canvas pixel of the four blend masks (host-capable for tests/host/kernel_math.cu).
__host__ __device__ __forceinline__ void blend_pixel(const BlendArgs& a, int x, int y) {
  const size_t plane = (size_t)a.w * a.h, p = (size_t)y * a.w + x;
  uint8_t m[4];
#pragma unroll
  for (int n = 0; n < 4; ++n) m[n] = a.polys[n * plane + p];
  // (other, lineA, lineB) per camera, in the reference's order (surroundBEV.py:171-186)
  const int other[4][2] = {{2, 3}, {2, 3}, {0, 1}, {0, 1}};
  const int la[4][2] = {{0, 1}, {2, 3}, {4, 5}, {6, 7}};
  const int lb[4][2] = {{4, 6}, {5, 7}, {0, 2}, {1, 3}};
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    int v = m[n];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (v != 0 && m[other[n][k]] != 0) {
        const double dA = seg_dist((double)x, (double)y, a.lines[la[n][k]]);
        const double dB = seg_dist((double)x, (double)y, a.lines[lb[n][k]]);
        const double a2 = dmul(dA, dA), b2 = dmul(dB, dB);
        v = (int)dmul(ddiv(a2, dadd(dadd(a2, b2), 1e-6)), 255.0);   // C cast: truncation
      }
    }
    a.out[n * plane + p] = (uint8_t)v;
  }
}

__global__ void __launch_bounds__(256) k_blend_masks(BlendArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.w || y >= a.h) return;
  blend_pixel(a, x, y);
}

// ---------------------------------------------------------------------------------
// K8 part 1: exact integer sum of V = max(B,G,R) over every dense BGR frame.
// grid = (blocks, n_frames).  48-byte (16-pixel) steps with three 16-byte loads.
// ---------------------------------------------------------------------------------
__device__ __forceinline__ unsigned vsum_16px(const uint4 a, const uint4 b, const uint4 c) {
  const unsigned w[12] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w};
  unsigned s = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {   // 12 bytes = 4 pixels per 3 words
    const unsigned w0 = w[3 * q], w1 = w[3 * q + 1], w2 = w[3 * q + 2];
    // pixel bytes: (w0.0,w0.1,w0.2) (w0.3,w1.0,w1.1) (w1.2,w1.3,w2.0) (w2.1,w2.2,w2.3)
    s += max(max(w0 & 255u, (w0 >> 8) & 255u), (w0 >> 16) & 255u);
    s += max(max(w0 >> 24, w1 & 255u), (w1 >> 8) & 255u);
    s += max(max((w1 >> 16) & 255u, w1 >> 24), w2 & 255u);
    s += max(max((w2 >> 8) & 255u, (w2 >> 16) & 255u), w2 >> 24);
  }
  return s;
}

// The frames of cameras [lo, lo + n) of a frame-set-major stack of n_cam cameras: launch index i (grid y) -> frame
// (i / n) * n_cam + lo + i % n.  A camera-sharded rank converts only its own cameras; the whole range {0, n_cam, n_cam}
// is the identity.
struct CamRange { int lo, n, n_cam; };
__host__ __device__ __forceinline__ int range_frame(CamRange r, int i) { return (i / r.n) * r.n_cam + r.lo + i % r.n; }

// grid y = frames of the range; vsum[frame] += its V sum.  A streaming reduction: 8 CTAs (a full SM of threads) per SM.
__global__ void __launch_bounds__(256, 8) k_vsum(Frames frames, long long frame_bytes, unsigned long long* __restrict__ vsum,
                                                 CamRange cr) {
  const int fi = range_frame(cr, blockIdx.y);
  const uint8_t* f = frames.frame(fi);
  const long long n48 = frame_bytes / 48;
  unsigned long long acc = 0;
  if ((reinterpret_cast<uintptr_t>(f) & 15) == 0) {
    const uint4* f4 = reinterpret_cast<const uint4*>(f);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n48; i += (long long)gridDim.x * blockDim.x) {
      const uint4 a = __ldg(f4 + 3 * i), b = __ldg(f4 + 3 * i + 1), c = __ldg(f4 + 3 * i + 2);
      acc += vsum_16px(a, b, c);
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n48 * 16; i += (long long)gridDim.x * blockDim.x) {
      const uint8_t* q = f + 3 * i;
      acc += max(max(q[0], q[1]), q[2]);
    }
  }
  if (blockIdx.x == 0)   // tail pixels (frame_bytes % 48)
    for (long long i = n48 * 16 + threadIdx.x; i * 3 < frame_bytes; i += blockDim.x) {
      const uint8_t* q = f + 3 * i;
      acc += max(max(q[0], q[1]), q[2]);
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ unsigned long long part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int k = 0; k < 8; ++k) t += part[k];
    atomicAdd(vsum + fi, t);
  }
}

// K8 part 2: delta_c = cvRound(V_mean - V_c) per frame-set (cv2.add rounds the scalar).
// luminance offsets of one frame-set from its exact V sums (surroundBEV.py:66-74); host-capable for the CPU tests
__host__ __device__ __forceinline__ void lum_deltas(const unsigned long long* vsum, int n_cam, double npix, int* delta) {
  double tot = 0.0;
  for (int c = 0; c < n_cam; ++c) tot = dadd(tot, ddiv((double)vsum[c], npix));
  const double vmean = ddiv(tot, (double)n_cam);
  for (int c = 0; c < n_cam; ++c) delta[c] = cv_round(dadd(vmean, -ddiv((double)vsum[c], npix)));
}

// The same from `world` blocks of V sums, block w at vsum + w * block_stride: camera-sharded ranks each fill the
// columns of their own cameras and leave the others zero, so the column sums are exact and equal the single-GPU sums.
// world 1 is the single-GPU case.
__host__ __device__ __forceinline__ void gathered_deltas(const unsigned long long* vsum, long long block_stride, int world,
                                                         int n_cam, double npix, int* delta) {
  unsigned long long v[BEVK_MAX_CAMERAS_K];
  for (int c = 0; c < n_cam; ++c) {
    unsigned long long s = 0;
    for (int w = 0; w < world; ++w) s += vsum[w * block_stride + c];
    v[c] = s;
  }
  lum_deltas(v, n_cam, npix, delta);
}

// vsum: [world][batch][n_cam]
__global__ void k_delta(const unsigned long long* __restrict__ vsum, int n_cam, int batch, int world, double npix,
                        int* __restrict__ delta) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  gathered_deltas(vsum + b * n_cam, (long long)batch * n_cam, world, n_cam, npix, delta + b * n_cam);
}

// ---------------------------------------------------------------------------------
// K9: color_balance (surroundBEV.py:43-55) + car overlay.  Gains from the channel sums;
// out = sat(cvRound(double(px) * K_c)) through a 3x256 table built per CTA in shared memory.
// ---------------------------------------------------------------------------------
// grey-world gains of one canvas from its channel sums, and one entry of the 3 x 256 output table (host-capable)
__host__ __device__ __forceinline__ void gray_world_gains(const unsigned long long* csum, double npix, double* gain) {
  const double B = ddiv((double)csum[0], npix), G = ddiv((double)csum[1], npix), R = ddiv((double)csum[2], npix);
  const double K = ddiv(dadd(dadd(R, G), B), 3.0);
  gain[0] = ddiv(K, B); gain[1] = ddiv(K, G); gain[2] = ddiv(K, R);
}
__host__ __device__ __forceinline__ uint8_t gain_entry(double gain, int v) {
  const int r = cv_round(dmul((double)v, gain));   // non-finite -> INT_MIN -> saturates to 0, as on x86
  return (uint8_t)(r < 0 ? 0 : (r > 255 ? 255 : r));
}
// The 3 x 256 table of one canvas (channel sums csum[0..2]) into tab[c * 256 + v], filled by the threads of a CTA.  The
// caller synchronises before reading it.
__device__ __forceinline__ void gain_table(const unsigned long long* csum, double npix, uint8_t* tab) {
  double gain[3];
  gray_world_gains(csum, npix, gain);
  for (int i = threadIdx.x; i < 768; i += blockDim.x) tab[i] = gain_entry(gain[i >> 8], i & 255);
}

__global__ void __launch_bounds__(256) k_gain(uint8_t* __restrict__ canvas, long long canvas_bytes, double npix,
                                              const unsigned long long* __restrict__ csum,
                                              const uint8_t* __restrict__ car) {
  __shared__ uint8_t tab[3][256];
  const int b = blockIdx.y;
  gain_table(csum + b * 3, npix, &tab[0][0]);
  __syncthreads();
  uint8_t* cv = canvas + (size_t)b * canvas_bytes;
  // 12-byte (4-pixel) steps keep the channel phase fixed per byte lane
  const long long n12 = canvas_bytes / 12;
  const bool aligned = (canvas_bytes % 4 == 0) && ((reinterpret_cast<uintptr_t>(canvas) & 3) == 0) &&
                       (!car || (reinterpret_cast<uintptr_t>(car) & 3) == 0);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n12; i += (long long)gridDim.x * blockDim.x) {
    if (aligned) {
      unsigned* p = reinterpret_cast<unsigned*>(cv + i * 12);
      unsigned w[3] = {p[0], p[1], p[2]};
      unsigned o[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        unsigned r = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int byte_idx = k * 4 + j;
          r |= (unsigned)tab[byte_idx % 3][(w[k] >> (8 * j)) & 255u] << (8 * j);
        }
        o[k] = r;
      }
      if (car) {
        const unsigned* c = reinterpret_cast<const unsigned*>(car + i * 12);
        o[0] = __vaddus4(o[0], __ldg(c)); o[1] = __vaddus4(o[1], __ldg(c + 1)); o[2] = __vaddus4(o[2], __ldg(c + 2));
      }
      p[0] = o[0]; p[1] = o[1]; p[2] = o[2];
    } else {
      for (int j = 0; j < 12; ++j) {
        int v = tab[j % 3][cv[i * 12 + j]];
        if (car) v = min(255, v + car[i * 12 + j]);
        cv[i * 12 + j] = (uint8_t)v;
      }
    }
  }
  if (blockIdx.x == 0)
    for (long long i = n12 * 12 + threadIdx.x; i < canvas_bytes; i += blockDim.x) {
      int v = tab[i % 3][cv[i]];
      if (car) v = min(255, v + car[i]);
      cv[i] = (uint8_t)v;
    }
}

// ---------------------------------------------------------------------------------
// Multi-GPU compose: saturating sum of n partial canvases (+ car).  16-byte vectors.
// ---------------------------------------------------------------------------------
struct SatSumArgs { const uint8_t* parts[BEVK_MAX_CAMERAS_K]; int n; unsigned long long bytes; const uint8_t* car; uint8_t* out; };

__global__ void __launch_bounds__(256) k_sat_sum(SatSumArgs a) {
  const unsigned long long n16 = a.bytes / 16;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n16;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    uint4 s = __ldg(reinterpret_cast<const uint4*>(a.parts[0]) + i);
    for (int k = 1; k < a.n; ++k) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(a.parts[k]) + i);
      s.x = __vaddus4(s.x, v.x); s.y = __vaddus4(s.y, v.y); s.z = __vaddus4(s.z, v.z); s.w = __vaddus4(s.w, v.w);
    }
    if (a.car) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(a.car) + i);
      s.x = __vaddus4(s.x, v.x); s.y = __vaddus4(s.y, v.y); s.z = __vaddus4(s.z, v.z); s.w = __vaddus4(s.w, v.w);
    }
    reinterpret_cast<uint4*>(a.out)[i] = s;
  }
  if (blockIdx.x == 0)
    for (unsigned long long i = n16 * 16 + threadIdx.x; i < a.bytes; i += blockDim.x) {
      int s = 0;
      for (int k = 0; k < a.n; ++k) s = min(255, s + a.parts[k][i]);
      if (a.car) s = min(255, s + a.car[i]);
      a.out[i] = (uint8_t)s;
    }
}

// ---------------------------------------------------------------------------------
// Stand-alone forms of K5/K6 (Mask / BlendMask.__call__), K8 (luminance_balance on whole
// frames) and the channel sums of K9, for callers that use those reference functions
// outside BevGenerator.  Dense BGR images.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_apply_mask(const uint8_t* __restrict__ img, const uint8_t* __restrict__ mask,
                                                    uint8_t* __restrict__ out, long long npx, int blend) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += (long long)gridDim.x * blockDim.x) {
    const unsigned w = mask[i];
    int b = img[3 * i], g = img[3 * i + 1], r = img[3 * i + 2];
    if (!blend) { if (!w) b = g = r = 0; }
    else {
      const float wf = __double2float_rn(__ddiv_rn((double)w, 255.0));
      b = (int)__fmul_rn((float)b, wf); g = (int)__fmul_rn((float)g, wf); r = (int)__fmul_rn((float)r, wf);
    }
    out[3 * i] = (uint8_t)b; out[3 * i + 1] = (uint8_t)g; out[3 * i + 2] = (uint8_t)r;
  }
}

__global__ void __launch_bounds__(256) k_chan_sum(const uint8_t* __restrict__ img, long long npx,
                                                  unsigned long long* __restrict__ csum) {
  unsigned long long sb = 0, sg = 0, sr = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += (long long)gridDim.x * blockDim.x) {
    sb += img[3 * i]; sg += img[3 * i + 1]; sr += img[3 * i + 2];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sb += __shfl_xor_sync(0xffffffffu, sb, o);
    sg += __shfl_xor_sync(0xffffffffu, sg, o);
    sr += __shfl_xor_sync(0xffffffffu, sr, o);
  }
  if ((threadIdx.x & 31) == 0) { atomicAdd(csum, sb); atomicAdd(csum + 1, sg); atomicAdd(csum + 2, sr); }
}

// grid.y = frame index; frame i of the input and output stacks at in / out + i * frame_stride; delta[frame] from k_delta
__global__ void __launch_bounds__(256) k_lum_apply(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, long long frame_stride,
                                                   int w, int h, const int* __restrict__ delta,
                                                   const int* __restrict__ hsv_tab) {
  __shared__ int s_tab[512];
  for (int i = threadIdx.x; i < 512; i += 256) s_tab[i] = hsv_tab[i];
  __syncthreads();
  const uint8_t* f = in + blockIdx.y * frame_stride;
  uint8_t* o = out + blockIdx.y * frame_stride;
  const int d = delta[blockIdx.y], tail = w - (w % 32);
  const long long npx = (long long)w * h;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += (long long)gridDim.x * blockDim.x) {
    int b = f[3 * i], g = f[3 * i + 1], r = f[3 * i + 2];
    hsv_roundtrip(b, g, r, d, (int)(i % w) >= tail, s_tab, s_tab + 256);
    o[3 * i] = (uint8_t)b; o[3 * i + 1] = (uint8_t)g; o[3 * i + 2] = (uint8_t)r;
  }
}

// ---------------------------------------------------------------------------------
// K8 part 3 for the fused BEV path: luminance_balance applied ONCE to every source pixel the LUT
// can sample.  spans[cam * FH + y] = (first, last+1) source column of row y that any tap of camera
// `cam` touches (bevk_bev_finalize); everything else in the frame is never read by k_bev, so it
// is not converted (about 17 % of a frame at the fixture geometry, 4.6x fewer HSV round trips
// than converting the four taps of every output pixel).  grid = (FH / LUM_ROWS, frames of the camera range `cr`).
// ---------------------------------------------------------------------------------
constexpr int LUM_ROWS = 16;   // source rows per CTA

// One CTA converts the sampled spans of LUM_ROWS consecutive source rows of one frame.  The work items -- groups of 4
// pixels = 3 aligned words in, 3 out -- of all its rows form ONE flat list (prefix sums of the rows' group counts in shared
// memory) that the threads stride through, so that a row with a short span costs nothing and every thread has several
// independent groups in flight; the sector selection of hsv_roundtrip is branch-free.  Frame f's balanced copy goes to
// out_base + f * out_stride.
__global__ void __launch_bounds__(128) k_lum_spans(Frames in, uint8_t* __restrict__ out_base, long long out_stride,
                                                   const int2* __restrict__ spans, CamRange cr, int w, int h,
                                                   const int* __restrict__ delta, const int* __restrict__ hsv_tab) {
  const int f = range_frame(cr, blockIdx.y), y0 = blockIdx.x * LUM_ROWS, y1 = min(h, y0 + LUM_ROWS), nrows = y1 - y0;
  const int2* sp_cam = spans + (size_t)(f % cr.n_cam) * h;
  const uint8_t* const frame = in.frame(f);
  uint8_t* const out = out_base + f * out_stride;
  __shared__ int s_tab[512];
  __shared__ int s_pref[LUM_ROWS + 1], s_g0[LUM_ROWS];
  const bool words = (w & 3) == 0 && ((reinterpret_cast<uintptr_t>(frame) | reinterpret_cast<uintptr_t>(out)) & 3) == 0;
  if (threadIdx.x == 0) {
    // groups cover each span rounded out to multiples of 4 pixels: the extra pixels are converted too, which nobody samples
    int acc = 0;
    for (int r = 0; r < nrows; ++r) {
      const int2 sp = sp_cam[y0 + r];
      const int g0 = sp.x >> 2, g1 = sp.y > sp.x ? (sp.y + 3) >> 2 : g0;
      s_pref[r] = acc; s_g0[r] = g0;
      acc += g1 - g0;
    }
    for (int r = nrows; r <= LUM_ROWS; ++r) s_pref[r] = acc;
  }
  for (int i = threadIdx.x; i < 512; i += 128) s_tab[i] = hsv_tab[i];
  __syncthreads();
  const int total = s_pref[LUM_ROWS];
  if (total == 0) return;
  const int d = delta[f], tail = w - (w % 32);
  if (words) {
    const size_t row_words = (size_t)w * 3 / 4;
    const unsigned* src0 = reinterpret_cast<const unsigned*>(frame) + (size_t)y0 * row_words;
    unsigned* dst0 = reinterpret_cast<unsigned*>(out) + (size_t)y0 * row_words;
    int r = 0;
#pragma unroll 2
    for (int i = threadIdx.x; i < total; i += 128) {
      while (i >= s_pref[r + 1]) ++r;                       // the thread's items are visited in increasing order
      const int gidx = s_g0[r] + (i - s_pref[r]);
      const unsigned* q = src0 + (size_t)r * row_words + 3 * gidx;
      const unsigned w0 = __ldg(q), w1 = __ldg(q + 1), w2 = __ldg(q + 2);       // B0 G0 R0 B1 | G1 R1 B2 G2 | R2 B3 G3 R3
      int c[12];
#pragma unroll
      for (int k = 0; k < 4; ++k) { c[k] = (w0 >> (8 * k)) & 255; c[4 + k] = (w1 >> (8 * k)) & 255; c[8 + k] = (w2 >> (8 * k)) & 255; }
      const bool rt = 4 * gidx >= tail;      // tail is a multiple of 4 here: a group is entirely body or entirely row tail
#pragma unroll
      for (int px = 0; px < 4; ++px) hsv_roundtrip(c[3 * px], c[3 * px + 1], c[3 * px + 2], d, rt, s_tab, s_tab + 256);
      unsigned* o = dst0 + (size_t)r * row_words + 3 * gidx;
      o[0] = (unsigned)c[0] | ((unsigned)c[1] << 8) | ((unsigned)c[2] << 16) | ((unsigned)c[3] << 24);
      o[1] = (unsigned)c[4] | ((unsigned)c[5] << 8) | ((unsigned)c[6] << 16) | ((unsigned)c[7] << 24);
      o[2] = (unsigned)c[8] | ((unsigned)c[9] << 8) | ((unsigned)c[10] << 16) | ((unsigned)c[11] << 24);
    }
  } else {
    for (int y = y0; y < y1; ++y) {
      const int2 sp = sp_cam[y];
      const uint8_t* src = frame + (size_t)y * w * 3;
      uint8_t* dst = out + (size_t)y * w * 3;
      for (int x = sp.x + threadIdx.x; x < sp.y; x += 128) {
        int b = src[3 * x], g = src[3 * x + 1], r = src[3 * x + 2];
        hsv_roundtrip(b, g, r, d, x >= tail, s_tab, s_tab + 256);
        dst[3 * x] = (uint8_t)b; dst[3 * x + 1] = (uint8_t)g; dst[3 * x + 2] = (uint8_t)r;
      }
    }
  }
}

// ---------------------------------------------------------------------------------
// YUV 4:2:0 sources (NV12, I420), FW and FH even.  The conversion reads a frame through its planes (YuvFrame: a Y plane,
// then NV12: one plane of interleaved U,V; I420: a U and a V plane), each at its own address and row pitch, as decoder
// surfaces come.  cv2's single-buffer layout is one instance: a uint8[FH*3/2][FW] image whose first FH rows are the Y
// plane.  NV12: then FH/2 rows of interleaved U,V.  I420: then the U plane and the V plane, each FW/2 x FH/2 and packed,
// so two chroma rows share a buffer row: chroma row k (U rows 0..FH/2-1, then the V rows) starts at buffer row FH + k/2,
// column (k & 1) * FW/2 -- which is also where cv2 looks for it in a buffer with padded rows.
// YUV 4:2:2 sources (YUYV, UYVY), FW even, FH any: one plane uint8[FH][FW][2] (cv2's input of COLOR_YUV2BGR_YUY2 /
// _UYVY) whose rows hold pixel pairs of 4 bytes, YUYV: Y0 U0 Y1 V0, UYVY: U0 Y0 V0 Y1; both pixels of a pair take its U
// and V, so pixel (x, y) has the chroma sample (x/2, y).  It reads through plane 0 of a YuvFrame like the others.
// The colour conversion runs once per sampled source pixel into the same copy stack the BALANCE pre-pass fills; the
// fused render then reads BGR from there as it always does.
// ---------------------------------------------------------------------------------
enum { YUV_NV12 = 1, YUV_I420 = 2, YUV_YUYV = 3, YUV_UYVY = 4 };

// Packed 4:2:2: byte positions within a pixel pair.  Y0 at yuv_y_byte, Y1 two bytes on; U at yuv_u_byte, V two bytes on.
template <int FMT>
__host__ __device__ __forceinline__ constexpr bool yuv_packed() { return FMT == YUV_YUYV || FMT == YUV_UYVY; }
template <int FMT>
__host__ __device__ __forceinline__ constexpr int yuv_y_byte() { return FMT == YUV_YUYV ? 0 : 1; }
template <int FMT>
__host__ __device__ __forceinline__ constexpr int yuv_u_byte() { return FMT == YUV_YUYV ? 1 : 0; }
// Chroma rows of an FH-row frame: FH / 2 for 4:2:0, FH for 4:2:2.
template <int FMT>
__host__ __device__ __forceinline__ constexpr int yuv_chroma_rows_of(int FH) { return yuv_packed<FMT>() ? FH : FH / 2; }

// cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420), OpenCV 4.x's fixed-point form (20 fraction bits), with U, V the chroma
// samples of pixel (x/2, y/2).  One definition for the kernels and the CPU tests.
__host__ __device__ __forceinline__ void yuv_bgr(int Y, int U, int V, int& b, int& g, int& r) {
  const int y = max(0, Y - 16) * 1220542, u = U - 128, v = V - 128, h = 1 << 19;
  b = min(255, max(0, (y + h + 2116026 * u) >> 20));
  g = min(255, max(0, (y + h - 852492 * v - 409993 * u) >> 20));
  r = min(255, max(0, (y + h + 1673527 * v) >> 20));
}

// Byte offsets of chroma row cy of a frame whose rows are `pitch` bytes apart: the U and V samples of pixel x are at
// u + step * (x/2) and v + step * (x/2), step = yuv_chroma_step<FMT>.
template <int FMT>
__host__ __device__ __forceinline__ void yuv_chroma_rows(int FW, int FH, long long pitch, int cy, long long& u, long long& v) {
  if (FMT == YUV_NV12) {
    u = (long long)(FH + cy) * pitch;
    v = u + 1;
  } else {
    const int ku = cy, kv = FH / 2 + cy;
    u = (long long)(FH + ku / 2) * pitch + (ku & 1) * (FW / 2);
    v = (long long)(FH + kv / 2) * pitch + (kv & 1) * (FW / 2);
  }
}
template <int FMT>
__host__ __device__ __forceinline__ constexpr int yuv_chroma_step() { return FMT == YUV_NV12 ? 2 : 1; }

// The planes of one YUV frame as the conversion reads them: row r of plane p starts at plane[p] + r * pitch[p].  Plane 0
// is Y (FW bytes a row), plane 1 interleaved U,V (NV12, FW bytes) or U (I420, FW/2), plane 2 V (I420, FW/2; unused for
// NV12).  YUYV / UYVY: plane 0 is the packed frame (2 FW bytes a row); planes 1 and 2 are not read.  Rows may be padded
// to any pitch and the planes may lie anywhere, as a video decoder's surfaces do.
struct YuvFrame {
  const uint8_t* plane[3];
  long long pitch[3];
};

// The planes of every frame of a call: plane p of frame i at f[p].frame(i) (a stack or a device table per plane), rows
// pitch[p] bytes apart.  Kernels take it by value.
struct YuvPlanes {
  Frames f[3];
  long long pitch[3];
  __host__ __device__ __forceinline__ YuvFrame frame(long long i) const {
    return YuvFrame{{f[0].frame(i), f[1].frame(i), f[2].frame(i)}, {pitch[0], pitch[1], pitch[2]}};
  }
};

// cv2's single-buffer layout uint8[FH*3/2][FW] as planes: byte offsets and pitches of Y, UV / U and V in the buffer.
// NV12: {0, FH*FW}, pitches {FW, FW}; I420: {0, FH*FW, FH*FW + FH*FW/4}, pitches {FW, FW/2, FW/2} (the packed U and V
// planes, chroma row k of yuv_chroma_rows at FH*FW + k*FW/2).  YUYV / UYVY: the one plane uint8[FH][FW][2], pitch 2 FW.
template <int FMT>
__host__ __device__ __forceinline__ void yuv_dense_layout(int FW, int FH, long long (&off)[3], long long (&pitch)[3]) {
  const long long y = (long long)FW * FH;
  off[0] = 0; pitch[0] = FW;
  if (yuv_packed<FMT>()) {
    pitch[0] = 2LL * FW;
    off[1] = off[2] = 0; pitch[1] = pitch[2] = 2LL * FW;   // unused
  } else if (FMT == YUV_NV12) {
    off[1] = y; pitch[1] = FW;
    off[2] = y; pitch[2] = FW;   // unused
  } else {
    off[1] = y; pitch[1] = FW / 2;
    off[2] = y + y / 4; pitch[2] = FW / 2;
  }
}

// The dense frames at base + i * stride (cv2's layout) as planes.
template <int FMT>
__host__ __device__ __forceinline__ YuvPlanes yuv_dense_planes(const uint8_t* base, long long stride, int FW, int FH) {
  long long off[3], pitch[3];
  yuv_dense_layout<FMT>(FW, FH, off, pitch);
  YuvPlanes p;
  for (int k = 0; k < 3; ++k) { p.f[k] = Frames(base + off[k], stride); p.pitch[k] = pitch[k]; }
  return p;
}

// One dense frame at f (cv2's layout) as planes.
template <int FMT>
__host__ __device__ __forceinline__ YuvFrame yuv_dense_frame(const uint8_t* f, int FW, int FH) {
  long long off[3], pitch[3];
  yuv_dense_layout<FMT>(FW, FH, off, pitch);
  return YuvFrame{{f + off[0], f + off[1], f + off[2]}, {pitch[0], pitch[1], pitch[2]}};
}

// Chroma row cy of a frame: the U and V samples of pixel x are at u + step * (x/2) and v + step * (x/2).
template <int FMT>
__host__ __device__ __forceinline__ void yuv_chroma_ptrs(const YuvFrame& fr, int cy, const uint8_t*& u, const uint8_t*& v) {
  u = fr.plane[1] + (long long)cy * fr.pitch[1];
  v = FMT == YUV_NV12 ? u + 1 : fr.plane[2] + (long long)cy * fr.pitch[2];
}

__host__ __device__ __forceinline__ int ld_u8(const uint8_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// The 4-pixel groups [g0, g1) that cover span sp of a row (k_lum_spans' rule); a group's pixels at or past FW (the last
// group of a row when FW % 4 == 2) are not converted.
__host__ __device__ __forceinline__ void span_groups(int2 sp, int& g0, int& g1) {
  g0 = sp.x >> 2;
  g1 = sp.y > sp.x ? (sp.y + 3) >> 2 : g0;
}

// The Y, U and V samples of group g (pixels [4g, 4g + n)) of row y of a packed 4:2:2 frame: its n/2 pixel pairs, bytes
// [8g, 8g + 2n) of the row.  One 8-byte load when they are a whole 8-aligned group, word loads when 4-aligned, bytes
// otherwise (chosen per pointer).  Y[2k], Y[2k+1], U[k], V[k] come from pair k; a missing second pair reads as zero.
template <int FMT>
__host__ __device__ __forceinline__ void yuv_packed_group(const YuvFrame& fr, int y, int x0, int n, int (&Y)[4], int (&U)[2],
                                                          int (&V)[2]) {
  const uint8_t* p = fr.plane[0] + (long long)y * fr.pitch[0] + 2 * x0;
  unsigned w[2] = {0u, 0u};
#ifdef __CUDA_ARCH__
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  if (n == 4 && (a & 7) == 0) {
    const uint2 q = __ldg(reinterpret_cast<const uint2*>(p));
    w[0] = q.x; w[1] = q.y;
  } else if ((a & 3) == 0) {
    for (int k = 0; k < (n >> 1); ++k) w[k] = __ldg(reinterpret_cast<const unsigned*>(p) + k);
  } else
#endif
  {
    for (int k = 0; k < (n >> 1); ++k)
      for (int j = 0; j < 4; ++j) w[k] |= (unsigned)ld_u8(p + 4 * k + j) << (8 * j);
  }
  constexpr int yb = 8 * yuv_y_byte<FMT>(), ub = 8 * yuv_u_byte<FMT>();
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    Y[2 * k] = (w[k] >> yb) & 255; Y[2 * k + 1] = (w[k] >> (yb + 16)) & 255;
    U[k] = (w[k] >> ub) & 255; V[k] = (w[k] >> (ub + 16)) & 255;
  }
}

// One work item of k_yuv_spans: group g of row y of frame fr, converted to BGR in c[3 * px + {0,1,2}] and, with BAL,
// luminance-balanced by delta d (tab: the HSV division tables).  Returns the number of pixels (4 or 2).  The word loads
// are chosen per pointer, so an odd base or pitch only costs byte loads.
template <int FMT, bool BAL>
__host__ __device__ __forceinline__ int yuv_group(const YuvFrame& fr, int FW, int y, int g, int d, const int* __restrict__ tab,
                                                  int (&c)[12]) {
  const int x0 = 4 * g, n = min(4, FW - x0);
  if constexpr (yuv_packed<FMT>()) {
    int Y[4], U[2], V[2];
    yuv_packed_group<FMT>(fr, y, x0, n, Y, U, V);
    const bool rt = x0 >= FW - (FW % 32);   // luminance_balance's row tail (a multiple of 4: whole groups)
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      yuv_bgr(Y[px], U[px >> 1], V[px >> 1], c[3 * px], c[3 * px + 1], c[3 * px + 2]);
      if (BAL) hsv_roundtrip(c[3 * px], c[3 * px + 1], c[3 * px + 2], d, rt, tab, tab + 256);
    }
    return n;
  }
  const uint8_t *ur, *vr;
  yuv_chroma_ptrs<FMT>(fr, y >> 1, ur, vr);
  ur += yuv_chroma_step<FMT>() * (x0 >> 1);
  vr += yuv_chroma_step<FMT>() * (x0 >> 1);
  const uint8_t* yr = fr.plane[0] + (long long)y * fr.pitch[0] + x0;
  int Y[4] = {0, 0, 0, 0}, U[2] = {128, 128}, V[2] = {128, 128};
#ifdef __CUDA_ARCH__
  if (n == 4 && (reinterpret_cast<uintptr_t>(yr) & 3) == 0) {
    const unsigned w = __ldg(reinterpret_cast<const unsigned*>(yr));
#pragma unroll
    for (int k = 0; k < 4; ++k) Y[k] = (w >> (8 * k)) & 255;
  } else
#endif
  {
    for (int k = 0; k < n; ++k) Y[k] = ld_u8(yr + k);
  }
#ifdef __CUDA_ARCH__
  if (FMT == YUV_NV12 && n == 4 && (reinterpret_cast<uintptr_t>(ur) & 3) == 0) {   // U0 V0 U1 V1
    const unsigned w = __ldg(reinterpret_cast<const unsigned*>(ur));
    U[0] = w & 255; V[0] = (w >> 8) & 255; U[1] = (w >> 16) & 255; V[1] = w >> 24;
  } else
#endif
  {
    for (int k = 0; k < (n >> 1); ++k) { U[k] = ld_u8(ur + yuv_chroma_step<FMT>() * k); V[k] = ld_u8(vr + yuv_chroma_step<FMT>() * k); }
  }
  const bool rt = x0 >= FW - (FW % 32);   // luminance_balance's row tail (a multiple of 4: whole groups)
#pragma unroll
  for (int px = 0; px < 4; ++px) {
    yuv_bgr(Y[px], U[px >> 1], V[px >> 1], c[3 * px], c[3 * px + 1], c[3 * px + 2]);
    if (BAL) hsv_roundtrip(c[3 * px], c[3 * px + 1], c[3 * px + 2], d, rt, tab, tab + 256);
  }
  return n;
}

// The same on a dense frame f in cv2's layout (rows FW bytes apart).
template <int FMT, bool BAL>
__host__ __device__ __forceinline__ int yuv_group(const uint8_t* __restrict__ f, int FW, int FH, int y, int g, int d,
                                                  const int* __restrict__ tab, int (&c)[12]) {
  return yuv_group<FMT, BAL>(yuv_dense_frame<FMT>(f, FW, FH), FW, y, g, d, tab, c);
}

// The YUV source pre-pass of a fused render: k_lum_spans' work decomposition (one CTA per LUM_ROWS source rows of one
// frame, the rows' span groups as one flat list), reading Y row y and chroma row y/2 of the frame's planes (4:2:2: row y
// of the packed plane) and writing BGR
// into the copy stack (frame f at out_base + f * out_stride, rows FW * 3 bytes); with BAL each pixel then takes
// luminance_balance's HSV round trip with the frame's delta, so a balanced YUV render has no extra pass over the frames.
template <int FMT, bool BAL>
__global__ void __launch_bounds__(128) k_yuv_spans(YuvPlanes in, uint8_t* __restrict__ out_base, long long out_stride,
                                                   const int2* __restrict__ spans, CamRange cr, int w, int h,
                                                   const int* __restrict__ delta, const int* __restrict__ hsv_tab) {
  const int f = range_frame(cr, blockIdx.y), y0 = blockIdx.x * LUM_ROWS, y1 = min(h, y0 + LUM_ROWS), nrows = y1 - y0;
  const int2* sp_cam = spans + (size_t)(f % cr.n_cam) * h;
  const YuvFrame frame = in.frame(f);
  uint8_t* const out = out_base + f * out_stride;
  __shared__ int s_tab[BAL ? 512 : 1];
  __shared__ int s_pref[LUM_ROWS + 1], s_g0[LUM_ROWS];
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int r = 0; r < nrows; ++r) {
      int g0, g1;
      span_groups(sp_cam[y0 + r], g0, g1);
      s_pref[r] = acc; s_g0[r] = g0;
      acc += g1 - g0;
    }
    for (int r = nrows; r <= LUM_ROWS; ++r) s_pref[r] = acc;
  }
  if (BAL)
    for (int i = threadIdx.x; i < 512; i += 128) s_tab[i] = hsv_tab[i];
  __syncthreads();
  const int total = s_pref[LUM_ROWS];
  if (total == 0) return;
  const int d = BAL ? delta[f] : 0;
  const bool words = (w & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0;
  const size_t row_bytes = (size_t)w * 3;
  int r = 0;
#pragma unroll 2
  for (int i = threadIdx.x; i < total; i += 128) {
    while (i >= s_pref[r + 1]) ++r;                       // the thread's items are visited in increasing order
    const int gidx = s_g0[r] + (i - s_pref[r]);
    int c[12];
    const int n = yuv_group<FMT, BAL>(frame, w, y0 + r, gidx, d, s_tab, c);
    uint8_t* o = out + (size_t)(y0 + r) * row_bytes + 12 * (size_t)gidx;
    if (words) {
      unsigned* o4 = reinterpret_cast<unsigned*>(o);
      o4[0] = (unsigned)c[0] | ((unsigned)c[1] << 8) | ((unsigned)c[2] << 16) | ((unsigned)c[3] << 24);
      o4[1] = (unsigned)c[4] | ((unsigned)c[5] << 8) | ((unsigned)c[6] << 16) | ((unsigned)c[7] << 24);
      o4[2] = (unsigned)c[8] | ((unsigned)c[9] << 8) | ((unsigned)c[10] << 16) | ((unsigned)c[11] << 24);
    } else {
#pragma unroll
      for (int k = 0; k < 12; ++k)
        if (k < 3 * n) o[k] = (uint8_t)c[k];
    }
  }
}

// V = max(B, G, R) summed over the four pixels that share chroma sample (cx, cy) of frame fr.
template <int FMT>
__host__ __device__ __forceinline__ unsigned yuv_vsum_2x2(const YuvFrame& fr, int cx, int cy) {
  const uint8_t *ur, *vr;
  yuv_chroma_ptrs<FMT>(fr, cy, ur, vr);
  const int U = ld_u8(ur + yuv_chroma_step<FMT>() * cx), V = ld_u8(vr + yuv_chroma_step<FMT>() * cx);
  const long long yp = fr.pitch[0];
  const uint8_t* y = fr.plane[0] + (long long)(2 * cy) * yp + 2 * cx;
  const int Yv[4] = {ld_u8(y), ld_u8(y + 1), ld_u8(y + yp), ld_u8(y + yp + 1)};
  unsigned s = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    int b, g, r;
    yuv_bgr(Yv[k], U, V, b, g, r);
    s += (unsigned)max(b, max(g, r));
  }
  return s;
}

// The same on a dense frame f in cv2's layout (rows FW bytes apart).
template <int FMT>
__host__ __device__ __forceinline__ unsigned yuv_vsum_2x2(const uint8_t* __restrict__ f, int FW, int FH, int cx, int cy) {
  return yuv_vsum_2x2<FMT>(yuv_dense_frame<FMT>(f, FW, FH), cx, cy);
}

// V = max(B, G, R) summed over the pixel pair that shares chroma sample (cx, y) of a packed 4:2:2 frame fr.
template <int FMT>
__host__ __device__ __forceinline__ unsigned yuv_vsum_pair(const YuvFrame& fr, int cx, int y) {
  const uint8_t* p = fr.plane[0] + (long long)y * fr.pitch[0] + 4 * cx;
  const int U = ld_u8(p + yuv_u_byte<FMT>()), V = ld_u8(p + yuv_u_byte<FMT>() + 2);
  const int Yv[2] = {ld_u8(p + yuv_y_byte<FMT>()), ld_u8(p + yuv_y_byte<FMT>() + 2)};
  unsigned s = 0;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    int b, g, r;
    yuv_bgr(Yv[k], U, V, b, g, r);
    s += (unsigned)max(b, max(g, r));
  }
  return s;
}

// The sum of V over the pixels of chroma sample (cx, cy): a 2 x 2 block (4:2:0) or a pixel pair (4:2:2).
template <int FMT>
__host__ __device__ __forceinline__ unsigned yuv_vsum_sample(const YuvFrame& fr, int cx, int cy) {
  if constexpr (yuv_packed<FMT>()) return yuv_vsum_pair<FMT>(fr, cx, cy);
  else return yuv_vsum_2x2<FMT>(fr, cx, cy);
}

// The same on a dense packed frame f (rows 2 FW bytes apart).
template <int FMT>
__host__ __device__ __forceinline__ unsigned yuv_vsum_pair(const uint8_t* __restrict__ f, int FW, int FH, int cx, int y) {
  return yuv_vsum_pair<FMT>(yuv_dense_frame<FMT>(f, FW, FH), cx, y);
}

// k_vsum for YUV frames: vsum[frame] += the exact sum of V over the whole converted frame (what luminance_balance sees
// after cvtColor).  grid = (blocks over chroma rows (yuv_chroma_rows_of), frames of the range `cr`).
template <int FMT>
__global__ void __launch_bounds__(256, 8) k_vsum_yuv(YuvPlanes frames, int w, int h, unsigned long long* __restrict__ vsum,
                                                     CamRange cr) {
  const int fi = range_frame(cr, blockIdx.y);
  const YuvFrame f = frames.frame(fi);
  unsigned long long acc = 0;
  for (int cy = blockIdx.x; cy < yuv_chroma_rows_of<FMT>(h); cy += gridDim.x) {
    unsigned s = 0;   // at most 4 * 255 per sample and FW/2 <= 16384 samples per row: fits 32 bits
    for (int cx = threadIdx.x; cx < w / 2; cx += blockDim.x) s += yuv_vsum_sample<FMT>(f, cx, cy);
    acc += s;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ unsigned long long part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int k = 0; k < 8; ++k) t += part[k];
    atomicAdd(vsum + fi, t);
  }
}

// ---------------------------------------------------------------------------------
// YUV 4:2:0 canvases (BEVK_FLAG_OUT_NV12 / _I420).  Canvas b is the dense uint8[BH*3/2][BW] buffer (BW, BH even) at
// out + b * BW*BH*3/2: the Y plane, then NV12: BH/2 rows of interleaved U,V; I420: the U plane, then the V plane, each
// BW/2 x BH/2 and packed.  Its bytes are cv2.cvtColor(bgr, COLOR_BGR2YUV_I420) of the BGR canvas (NV12: the same planes
// interleaved), converted by a streaming pass over the rendered BGR canvases.
// ---------------------------------------------------------------------------------
// cv2.cvtColor(COLOR_BGR2YUV_I420) of one pixel, OpenCV 4.x's fixed-point form (20 fraction bits).  Over all 2^24 BGR
// triples Y lies in [16, 235] and U, V in [16, 240], so nothing saturates.  cv2 takes a 2 x 2 block's U and V from its
// top-left pixel alone.  One definition for the kernel and the CPU tests.
__host__ __device__ __forceinline__ void bgr_yuv(int b, int g, int r, int& Y, int& U, int& V) {
  const int hy = (16 << 20) + (1 << 19), hc = (128 << 20) + (1 << 19);
  Y = (269484 * r + 528482 * g + 102760 * b + hy) >> 20;
  U = (-155188 * r - 305135 * g + 460324 * b + hc) >> 20;
  V = (460324 * r - 385875 * g - 74448 * b + hc) >> 20;
}

struct CanvasYuvArgs {
  const uint8_t* canvas;                 // BGR canvases, canvas b at canvas + b * BW*BH*3 (library scratch, 4-byte aligned)
  uint8_t* out;                          // 4:2:0 canvases, canvas b at out + b * BW*BH*3/2 (the caller's: any alignment)
  int BW, BH;
  const unsigned long long* csum;        // GAIN: channel sums of the raw canvases, [batch][3]
  const uint8_t* car;                    // GAIN: null, or the car overlay uint8[BH][BW][3] (any alignment)
  double npix;                           // GAIN: BW * BH
};

// May the work items use 32-bit loads and stores?  The BGR rows of a 4-pixel group are then 3 aligned words (BW % 4 == 0
// and the scratch base aligned), and so are its Y words, its NV12 chroma word and its two I420 chroma halves, when the
// caller's out (and car) are 4-byte aligned.  BW % 4 == 2 (an odd chroma row width) takes the byte path.
__host__ __device__ __forceinline__ bool canvas_yuv_words(const CanvasYuvArgs& a) {
  return (a.BW & 3) == 0 && ((reinterpret_cast<uintptr_t>(a.out) | reinterpret_cast<uintptr_t>(a.car)) & 3) == 0;
}

__host__ __device__ __forceinline__ unsigned ld_u32(const uint8_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(reinterpret_cast<const unsigned*>(p));
#else
  return *reinterpret_cast<const unsigned*>(p);
#endif
}

// One work item of k_canvas_yuv: pixels [4g, 4g + 4) (2 at the end of a BW % 4 == 2 row) of canvas rows 2cy and 2cy + 1
// of canvas b.  Writes their Y bytes, and U and V of the even row's even pixels.  GAIN: the canvas is raw and each
// byte first goes through tab (gain_table: color_balance), then the car is added with saturation, as k_gain does.
template <int FMT, bool GAIN>
__host__ __device__ __forceinline__ void canvas_yuv_item(const CanvasYuvArgs& a, int b, const uint8_t* tab, int cy, int g,
                                                         bool words) {
  const int BW = a.BW, x0 = 4 * g, n = min(4, BW - x0);
  const long long plane = (long long)BW * a.BH, row3 = 3ll * BW;
  const long long src_off = (long long)(2 * cy) * row3 + 3 * x0;
  const uint8_t* src = a.canvas + b * 3 * plane + src_off;
  const uint8_t* car = GAIN && a.car ? a.car + src_off : nullptr;
  int c[2][12];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (words) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const unsigned w = ld_u32(src + r * row3 + 4 * k);
#pragma unroll
        for (int j = 0; j < 4; ++j) c[r][4 * k + j] = (w >> (8 * j)) & 255;
      }
    } else {
#pragma unroll
      for (int k = 0; k < 12; ++k) c[r][k] = k < 3 * n ? ld_u8(src + r * row3 + k) : 0;
    }
    if (GAIN) {
#pragma unroll
      for (int k = 0; k < 12; ++k) c[r][k] = tab[(k % 3) * 256 + c[r][k]];
      if (car) {
        if (words) {
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const unsigned w = ld_u32(car + r * row3 + 4 * k);
#pragma unroll
            for (int j = 0; j < 4; ++j) c[r][4 * k + j] = min(255, c[r][4 * k + j] + (int)((w >> (8 * j)) & 255));
          }
        } else {
#pragma unroll
          for (int k = 0; k < 12; ++k)
            if (k < 3 * n) c[r][k] = min(255, c[r][k] + ld_u8(car + r * row3 + k));
        }
      }
    }
  }
  int Y[2][4], U[2], V[2];
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      int u, v;
      bgr_yuv(c[r][3 * p], c[r][3 * p + 1], c[r][3 * p + 2], Y[r][p], u, v);
      if (r == 0 && !(p & 1)) { U[p >> 1] = u; V[p >> 1] = v; }   // the top-left pixel of each 2 x 2 block
    }
  uint8_t* o = a.out + b * (3 * plane / 2);
  uint8_t* y0 = o + (long long)(2 * cy) * BW + x0;
  uint8_t* u0;
  uint8_t* v0;
  if (FMT == YUV_NV12) {
    u0 = o + plane + (long long)cy * BW + x0;
    v0 = u0 + 1;
  } else {
    u0 = o + plane + (long long)cy * (BW / 2) + (x0 >> 1);
    v0 = u0 + plane / 4;
  }
  if (words) {
#pragma unroll
    for (int r = 0; r < 2; ++r)
      *reinterpret_cast<unsigned*>(y0 + r * BW) =
          (unsigned)Y[r][0] | ((unsigned)Y[r][1] << 8) | ((unsigned)Y[r][2] << 16) | ((unsigned)Y[r][3] << 24);
    if (FMT == YUV_NV12) {
      *reinterpret_cast<unsigned*>(u0) = (unsigned)U[0] | ((unsigned)V[0] << 8) | ((unsigned)U[1] << 16) | ((unsigned)V[1] << 24);
    } else {
      *reinterpret_cast<unsigned short*>(u0) = (unsigned short)(U[0] | (U[1] << 8));
      *reinterpret_cast<unsigned short*>(v0) = (unsigned short)(V[0] | (V[1] << 8));
    }
  } else {
#pragma unroll
    for (int p = 0; p < 4; ++p)
      if (p < n) { y0[p] = (uint8_t)Y[0][p]; y0[BW + p] = (uint8_t)Y[1][p]; }
#pragma unroll
    for (int k = 0; k < 2; ++k)
      if (2 * k < n) { u0[yuv_chroma_step<FMT>() * k] = (uint8_t)U[k]; v0[yuv_chroma_step<FMT>() * k] = (uint8_t)V[k]; }
  }
}

// The conversion pass: grid = (blocks, batch); the items (4-pixel groups of row pairs) of canvas blockIdx.y, row pair
// major, are strided over its blocks, so that a warp reads 32 consecutive groups of two rows and writes 32 consecutive Y
// words per row.  GAIN: the canvases are raw BALANCE renders (render of a YUV canvas) and each CTA builds the
// canvas's gain table in shared memory, so k_gain does not run and the balanced BGR canvas is never written.
template <int FMT, bool GAIN>
__global__ void __launch_bounds__(256) k_canvas_yuv(CanvasYuvArgs a) {
  __shared__ uint8_t tab[GAIN ? 768 : 1];
  const int b = blockIdx.y;
  if (GAIN) {
    gain_table(a.csum + 3 * b, a.npix, tab);
    __syncthreads();
  }
  const int ng = (a.BW + 3) >> 2, items = ng * (a.BH >> 1);   // at most 16384 x 32768: fits an int
  const bool words = canvas_yuv_words(a);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < items; i += gridDim.x * blockDim.x) {
    const int cy = i / ng;
    canvas_yuv_item<FMT, GAIN>(a, b, tab, cy, i - cy * ng, words);
  }
}

// ---------------------------------------------------------------------------------
// Host -> device ingest for page-locked (mapped) host frames: instead of DMA rectangles, the SMs
// read exactly the sampled row spans of every frame straight out of host memory (zero-copy, 16-byte
// vectors, coalesced) and write them into the device frame buffers.  Moves ~17 % of each frame
// over PCIe instead of the 23-34 % a band / bounding-box DMA needs.  grid = (FH, n_frames); frame f goes to
// dev_frames + f * dev_stride.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_fetch_spans(const uint8_t* const* __restrict__ host_frames, uint8_t* __restrict__ dev_frames,
                                                     long long dev_stride, const int2* __restrict__ spans, int n_cam, int h,
                                                     long long host_stride, int row_bytes) {
  const int y = blockIdx.x, f = blockIdx.y;
  const int2 sp = spans[(f % n_cam) * h + y];
  if (sp.y <= sp.x) return;
  // 16-byte window around the span (+4 px each side for the aligned word reads of the gather)
  const int b0 = max(0, 3 * sp.x - 12) & ~15, b1 = min(row_bytes, (3 * sp.y + 12 + 15) & ~15);
  const uint4* src = reinterpret_cast<const uint4*>(host_frames[f] + (size_t)y * host_stride + b0);
  uint4* dst = reinterpret_cast<uint4*>(dev_frames + f * dev_stride + (size_t)y * row_bytes + b0);
  for (int i = threadIdx.x; i < (b1 - b0) >> 4; i += 128) dst[i] = src[i];
}

// The same for page-locked YUV frames: buffer row y of the uint8[FH*3/2][FW] frame brings its one or two 16-byte
// windows win[camera][y] = (x0, x1, x2, x3), bytes [x0, x1) and [x2, x3) (yuv_windows in bevk_plan.cuh: everything
// k_yuv_spans reads of the row).  grid = (FH*3/2, n_frames); frame f goes to dev_frames + f * dev_stride, rows
// row_bytes (= FW) apart.  Packed 4:2:2 frames uint8[FH][FW][2] take the same kernel with FH rows of 2 FW bytes.
__global__ void __launch_bounds__(128) k_fetch_yuv(const uint8_t* const* __restrict__ host_frames, uint8_t* __restrict__ dev_frames,
                                                   long long dev_stride, const int4* __restrict__ win, int n_cam, int rows,
                                                   long long host_stride, int row_bytes) {
  const int y = blockIdx.x, f = blockIdx.y;
  const int4 wd = win[(size_t)(f % n_cam) * rows + y];
  const int n1 = (wd.y - wd.x) >> 4, n = n1 + ((wd.w - wd.z) >> 4);
  const uint8_t* src = host_frames[f] + (size_t)y * host_stride;
  uint8_t* dst = dev_frames + f * dev_stride + (size_t)y * row_bytes;
  for (int i = threadIdx.x; i < n; i += 128) {
    const int off = i < n1 ? wd.x + 16 * i : wd.z + 16 * (i - n1);
    *reinterpret_cast<uint4*>(dst + off) = *reinterpret_cast<const uint4*>(src + off);
  }
}

}  // namespace bevk
