// bevk_device.cuh -- device-side arithmetic shared by the bevk kernels (sm_90a).
//
// Everything here is a bit-exact restatement target: the coordinate math is IEEE
// FP64 with NO fused multiply-add (OpenCV's x86 baseline build has none), so every
// product/sum goes through __dmul_rn/__dadd_rn, which the compiler may not contract.
// Specs: SURVEY.md Appendix A1 (fisheye map), A11 (pinhole map), A2 (fixed-point
// bilinear), A3 (warpPerspective coordinates), A9 (8-bit HSV round trip).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

namespace bevk {

constexpr int INTER_BITS = 5;
constexpr int TAB = 32;

// Where the frames of a call live, for the host and the kernels alike: a frame STACK (frame i at base + i * stride), or a
// device table of frame pointers for frames that really are scattered.  Kernels take it by value, so a captured CUDA
// graph keeps the addresses it was captured with.
struct Frames {
  const uint8_t* const* table = nullptr;
  const uint8_t* base = nullptr;
  long long stride = 0;
  Frames() = default;
  __host__ __device__ explicit Frames(const void* d_table) : table(static_cast<const uint8_t* const*>(d_table)) {}
  __host__ __device__ Frames(const void* d_base, long long frame_stride)
      : base(static_cast<const uint8_t*>(d_base)), stride(frame_stride) {}
  __host__ __device__ __forceinline__ const uint8_t* frame(long long i) const { return table ? table[i] : base + i * stride; }
};

struct CamModel {      // cv2.fisheye / cv2 initUndistortRectifyMap inputs, pre-digested on the host
  double iR[9];        // inv(P * R)
  double k[5];         // fisheye: k1..k4 ; pinhole: k1,k2,p1,p2,k3
  double fx, fy, cx, cy;
  int model;           // BEVK_MODEL_*
  int w, h;            // size of the undistorted (destination) frame
  const double* xs;    // rays independent of the row (xs_table_applies): OpenCV's running _x of column j; else null
};

// What cv2's full lens models add to CamModel.  Only the LENS = 1 instances of the kernels receive it (lens_model), so
// that the 4-coefficient fisheye and the 5-coefficient pinhole keep the instances they always ran.
struct LensExt {
  double k[7];          // pinhole: k4 k5 k6 (rational), s1 s2 s3 s4 (thin prism); zeros when D has fewer coefficients
  double T[9];          // pinhole: computeTiltProjectionMatrix(tauX, tauY); the identity without tilt
  const double* rays;   // rays that depend on the row: cv2's running _x, _y, _w (walk_rays), or null
};

struct Homog { double M[9]; };   // inv(H), as cv2.warpPerspective computes it

// OpenCV's closed-form 3x3 inverse (cv::invert, DECOMP_LU, n == 3, CV_64F).
inline bool inv3(const double* S, double* T) {
#define M(r, c) S[(r) * 3 + (c)]
  double d = M(0, 0) * (M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) - M(0, 1) * (M(1, 0) * M(2, 2) - M(1, 2) * M(2, 0)) +
             M(0, 2) * (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0));
  if (d == 0.) return false;
  d = 1. / d;
  T[0] = (M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) * d;
  T[1] = (M(0, 2) * M(2, 1) - M(0, 1) * M(2, 2)) * d;
  T[2] = (M(0, 1) * M(1, 2) - M(0, 2) * M(1, 1)) * d;
  T[3] = (M(1, 2) * M(2, 0) - M(1, 0) * M(2, 2)) * d;
  T[4] = (M(0, 0) * M(2, 2) - M(0, 2) * M(2, 0)) * d;
  T[5] = (M(0, 2) * M(1, 0) - M(0, 0) * M(1, 2)) * d;
  T[6] = (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0)) * d;
  T[7] = (M(0, 1) * M(2, 0) - M(0, 0) * M(2, 1)) * d;
  T[8] = (M(0, 0) * M(1, 1) - M(0, 1) * M(1, 0)) * d;
#undef M
  return true;
}

// does undistorted pixel column j take the saturating (vector-body) pack?  (pinhole model only)
__host__ __device__ __forceinline__ bool pack_saturates(int model, int j, int w) { return model == 1 && j < w - (w % 8); }

// Separately rounded FP64 operations (no FMA contraction), as OpenCV's scalar C++ evaluates them.  The host
// forms let tests/host/kernel_math.cu run the very same coordinate code on a CPU (built without contraction).
#ifdef __CUDA_ARCH__
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double dsqrt(double a) { return __dsqrt_rn(a); }
__device__ __forceinline__ double dinf() { return __longlong_as_double(0x7ff0000000000000LL); }
__device__ __forceinline__ int d2i_rn(double v) { return __double2int_rn(v); }
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ int f2i_rn(float v) { return __float2int_rn(v); }
#else
inline double dmul(double a, double b) { volatile double r = a * b; return r; }
inline double dadd(double a, double b) { volatile double r = a + b; return r; }
inline double ddiv(double a, double b) { volatile double r = a / b; return r; }
inline double dsqrt(double a) { return sqrt(a); }
inline double dinf() { return HUGE_VAL; }
inline int d2i_rn(double v) { return (int)nearbyint(v); }   // default rounding mode: to nearest even
inline float fmul(float a, float b) { volatile float r = a * b; return r; }
inline float fsub(float a, float b) { volatile float r = a - b; return r; }
inline float fadd(float a, float b) { volatile float r = a + b; return r; }
inline float ffma(float a, float b, float c) { return fmaf(a, b, c); }
inline int f2i_rn(float v) { return (int)nearbyintf(v); }
#endif

// cvRound / saturate_cast<int>(double): x86 cvtsd2si returns INT_MIN ("integer
// indefinite") for NaN and out-of-range inputs.
__host__ __device__ __forceinline__ int cv_round(double v) {
  if (!(fabs(v) < 2147483648.0)) return INT_MIN;
  return d2i_rn(v);
}

// A1 / A11: cv2 builds the rays of a map row from running sums that start at _x = i*iR01 + iR02 (the same for _y, _w).
// cv2.fisheye.initUndistortRectifyMap adds iR00 column by column.  cv2.initUndistortRectifyMap (pinhole) adds 8*iR00 per
// 8-column block of its vector body and offsets column k of a block by k*iR00; its scalar tail (the last W % 8 columns)
// adds iR00 column by column from where the blocks end.  The 8 is the AVX2 build's, as in pack_saturates.
// j*iR00 + (i*iR01 + iR02) differs from those sums in the last bits, which moves cvRound ties and, where _w is near 0,
// decides between _w == 0 and a tiny _w.  row_sums writes the sums of one row and one ray component from x0 by step.
template <int MODEL>
__host__ __device__ __forceinline__ void row_sums(double x0, double step, int w, double* out) {
  int j = 0;
  if (MODEL == 1)
    for (; j < w - w % 8; j += 8, x0 = dadd(x0, dmul(8.0, step)))
      for (int k = 0; k < 8; ++k) out[j + k] = dadd(x0, dmul((double)k, step));
  for (; j < w; ++j, x0 = dadd(x0, step)) out[j] = x0;
}

// When iR has no skew and the last row (0, 0, *) -- every P of dst_camera_matrix, R = I, R = diag(-1, -1, 1) -- the
// sums of _y and _w add zeros (exact) and _x depends on the column only: the host tabulates it once per map
// (fill_xs_table), the kernels read xs[j].  Any other P without R keeps the direct form.
inline bool xs_table_applies(const CamModel& c) {
  return c.iR[1] == 0. && c.iR[3] == 0. && c.iR[6] == 0. && c.iR[7] == 0.;
}
inline void fill_xs_table(const CamModel& c, double* xs) {   // x0 = 0 * iR01 + iR02
  if (c.model == 1) row_sums<1>(c.iR[2], c.iR[0], c.w, xs);
  else row_sums<0>(c.iR[2], c.iR[0], c.w, xs);
}

// A1 / A11 with a general R, for a camera whose rays depend on the row (rays_walk): what camera_ray<1> reads of lx.rays,
// walked once per row first (k_walk_rays), since the sums are serial along the row.
//   fisheye: cv2's rays of every pixel, [3][h][w] (24 bytes per map entry);
//   pinhole: the block starts of every row, [3][h][w / 8 + 1] (3 bytes per map entry): entry b of row i is the sum at
//            column 8b, the last one where the scalar tail starts.  A pixel needs its block start and k*iR00 (or, in the
//            tail, at most 7 running adds), so a fused pinhole slot can keep the table and evaluate per pixel.
inline int ray_row_len(const CamModel& c) { return c.model == 1 ? c.w / 8 + 1 : c.w; }

template <int MODEL>
__host__ __device__ __forceinline__ void walk_rays(const CamModel& c, int i, double* rays) {
  const double di = (double)i;
  if (MODEL == 1) {
    const int nb = c.w / 8;
    const size_t n = (size_t)(nb + 1) * c.h, q = (size_t)i * (nb + 1);
    for (int k = 0; k < 3; ++k) {
      double x = dadd(dmul(di, c.iR[3 * k + 1]), c.iR[3 * k + 2]);
      const double step8 = dmul(8.0, c.iR[3 * k]);
      for (int b = 0; b <= nb; ++b, x = dadd(x, step8)) rays[k * n + q + b] = x;
    }
    return;
  }
  const size_t n = (size_t)c.w * c.h, q = (size_t)i * c.w;
  double _x = dadd(dmul(di, c.iR[1]), c.iR[2]), _y = dadd(dmul(di, c.iR[4]), c.iR[5]), _w = dadd(dmul(di, c.iR[7]), c.iR[8]);
  for (int j = 0; j < c.w; ++j) {
    rays[q + j] = _x; rays[n + q + j] = _y; rays[2 * n + q + j] = _w;
    _x = dadd(_x, c.iR[0]); _y = dadd(_y, c.iR[3]); _w = dadd(_w, c.iR[6]);
  }
}
__host__ __device__ __forceinline__ void walk_rays(const CamModel& c, int i, double* rays) {
  if (c.model == 1) walk_rays<1>(c, i, rays);
  else walk_rays<0>(c, i, rays);
}

__host__ __device__ __forceinline__ double ldd(const double* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// The ray (_x, _y, _w) of undistorted pixel (j,i) that undistort_point<LENS> projects: from the walked rays of lx when it
// has them (LENS = 1), else the column table's _x or the direct form.  tests/host/lens_models.cu reads it.
template <int LENS>
__host__ __device__ __forceinline__ void camera_ray(const CamModel& c, const LensExt& lx, int j, int i, double& _x, double& _y,
                                                    double& _w) {
  const double dj = (double)j, di = (double)i;
  if (LENS && lx.rays && c.model == 1) {   // block start, then row_sums' in-block offset or tail sum
    const int nb1 = c.w / 8 + 1, b = j >> 3, k = j & 7;
    const size_t n = (size_t)nb1 * c.h, q = (size_t)i * nb1 + b;
    double r[3];
    for (int p = 0; p < 3; ++p) {
      double x = ldd(lx.rays + p * n + q);
      if (b < nb1 - 1) x = dadd(x, dmul((double)k, c.iR[3 * p]));
      else for (int t = 0; t < k; ++t) x = dadd(x, c.iR[3 * p]);
      r[p] = x;
    }
    _x = r[0]; _y = r[1]; _w = r[2];
  } else if (LENS && lx.rays) {
    const size_t n = (size_t)c.w * c.h, q = (size_t)i * c.w + j;
    _x = ldd(lx.rays + q); _y = ldd(lx.rays + n + q); _w = ldd(lx.rays + 2 * n + q);
  } else {
    _x = c.xs ? ldd(c.xs + j) : dadd(dmul(dj, c.iR[0]), dadd(dmul(di, c.iR[1]), c.iR[2]));
    _y = dadd(dmul(dj, c.iR[3]), dadd(dmul(di, c.iR[4]), c.iR[5]));
    _w = dadd(dmul(dj, c.iR[6]), dadd(dmul(di, c.iR[7]), c.iR[8]));
  }
}

// A1 / A11: source-image position (u,v) of undistorted pixel (j,i).  LENS = 0 is the 4-coefficient fisheye and the
// 5-coefficient pinhole; LENS = 1 adds what lx holds: cv2's rational denominator, thin-prism terms and tilt, and the
// walked rays.  With lx's coefficients zero, T the identity and no rays, LENS = 1 computes LENS = 0's values
// (a division by 1, adds of 0, a multiply by 1).
template <int LENS>
__host__ __device__ __forceinline__ void undistort_point(const CamModel& c, const LensExt& lx, int j, int i, double& u, double& v) {
  double _x, _y, _w;
  camera_ray<LENS>(c, lx, j, i, _x, _y, _w);
  if (c.model == 0) {  // equidistant fisheye
    if (_w <= 0) {
      const double inf = dinf();
      u = (_x > 0) ? -inf : inf;
      v = (_y > 0) ? -inf : inf;
      return;
    }
    const double x = ddiv(_x, _w), y = ddiv(_y, _w);
    const double r = dsqrt(dadd(dmul(x, x), dmul(y, y)));
    const double th = atan(r);
    const double t2 = dmul(th, th), t4 = dmul(t2, t2), t6 = dmul(t4, t2), t8 = dmul(t4, t4);
    const double poly = dadd(dadd(dadd(dadd(1.0, dmul(c.k[0], t2)), dmul(c.k[1], t4)), dmul(c.k[2], t6)), dmul(c.k[3], t8));
    const double thd = dmul(th, poly);
    const double s = (r == 0) ? 1.0 : ddiv(thd, r);
    u = dadd(dmul(dmul(c.fx, x), s), c.cx);
    v = dadd(dmul(dmul(c.fy, y), s), c.cy);
  } else {             // pinhole, k1 k2 p1 p2 k3 (LENS: k4 k5 k6 s1 s2 s3 s4 tauX tauY)
    const double w = ddiv(1.0, _w), x = dmul(_x, w), y = dmul(_y, w);
    const double x2 = dmul(x, x), y2 = dmul(y, y);
    const double r2 = dadd(x2, y2), _2xy = dmul(dmul(2.0, x), y);
    const double k1 = c.k[0], k2 = c.k[1], p1 = c.k[2], p2 = c.k[3], k3 = c.k[4];
    double kr = dadd(1.0, dmul(dadd(dmul(dadd(dmul(k3, r2), k2), r2), k1), r2));
    if (LENS) kr = ddiv(kr, dadd(1.0, dmul(dadd(dmul(dadd(dmul(lx.k[2], r2), lx.k[1]), r2), lx.k[0]), r2)));
    double xd = dadd(dadd(dmul(x, kr), dmul(p1, _2xy)), dmul(p2, dadd(r2, dmul(2.0, x2))));
    double yd = dadd(dadd(dmul(y, kr), dmul(p1, dadd(r2, dmul(2.0, y2)))), dmul(p2, _2xy));
    if (LENS) {
      xd = dadd(dadd(xd, dmul(lx.k[3], r2)), dmul(dmul(lx.k[4], r2), r2));
      yd = dadd(dadd(yd, dmul(lx.k[5], r2)), dmul(dmul(lx.k[6], r2), r2));
      const double* T = lx.T;   // cv2: vecTilt = matTilt * (xd, yd, 1), invProj = vecTilt(2) ? 1 / vecTilt(2) : 1
      const double vx = dadd(dadd(dmul(T[0], xd), dmul(T[1], yd)), T[2]);
      const double vy = dadd(dadd(dmul(T[3], xd), dmul(T[4], yd)), T[5]);
      const double vz = dadd(dadd(dmul(T[6], xd), dmul(T[7], yd)), T[8]);
      const double ip = vz != 0. ? ddiv(1.0, vz) : 1.0;
      u = dadd(dmul(dmul(c.fx, ip), vx), c.cx);
      v = dadd(dmul(dmul(c.fy, ip), vy), c.cy);
    } else {
      u = dadd(dmul(c.fx, xd), c.cx);
      v = dadd(dmul(c.fy, yd), c.cy);
    }
  }
}

__host__ __device__ __forceinline__ void undistort_point(const CamModel& c, int j, int i, double& u, double& v) {
  const LensExt none{};
  undistort_point<0>(c, none, j, i, u, v);
}

// ---- the camera set-up of every entry point (host only; tests/host/lens_models.cu runs it against cv2)
// A 3x3 product as cv::Matx forms P * R and the tilt matrix: entry (r, c) = (a_r0 b_0c + a_r1 b_1c) + a_r2 b_2c.
inline void mul3(const double* A, const double* B, double* C) {
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 3; ++k)
      C[r * 3 + k] = dadd(dadd(dmul(A[r * 3], B[k]), dmul(A[r * 3 + 1], B[3 + k])), dmul(A[r * 3 + 2], B[6 + k]));
}
inline bool is_identity3(const double* M) {
  for (int i = 0; i < 9; ++i)
    if (M[i] != (i % 4 == 0 ? 1. : 0.)) return false;
  return true;
}
// cv::detail::computeTiltProjectionMatrix(tauX, tauY): projZ(Ry * Rx) * (Ry * Rx)
inline void tilt_matrix(double tx, double ty, double* T) {
  const double ctx = cos(tx), stx = sin(tx), cty = cos(ty), sty = sin(ty);
  const double Rx[9] = {1, 0, 0, 0, ctx, stx, 0, -stx, ctx}, Ry[9] = {cty, 0, -sty, 0, 1, 0, sty, 0, cty};
  double Rxy[9];
  mul3(Ry, Rx, Rxy);
  const double Pz[9] = {Rxy[8], 0, -Rxy[2], 0, Rxy[8], -Rxy[5], 0, 0, 1};
  mul3(Pz, Rxy, T);
}

// D lengths cv2.initUndistortRectifyMap (pinhole) and cv2.fisheye.initUndistortRectifyMap accept (an empty D is zeros)
inline bool dist_count_ok(int model, int n) {
  return model == 0 ? (n == 0 || n == 4) : (n == 0 || n == 4 || n == 5 || n == 8 || n == 12 || n == 14);
}

enum { LENS_OK = 0, LENS_BAD_COUNT = 1, LENS_SINGULAR = 2 };

// cv2.initUndistortRectifyMap / cv2.fisheye.initUndistortRectifyMap's (K, D, R, P) as the kernels take them: iR =
// inv(P * R) (R == null: inv(P)), k1..k5 in cm, the rest of a 8-, 12- or 14-coefficient D and the tilt matrix in lx.
// *lens says whether the camera's lens needs the LENS = 1 instances: a pinhole with any of k4..k6, s1..s4, tauX, tauY
// non-zero, or a fisheye whose rotated rays depend on the row (fisheye_walks).  A camera whose rays walk (rays_walk)
// needs them too.  Any other camera, R included, computes the same bytes in the LENS = 0 instances.  The caller attaches
// cm.xs and lx.rays.
inline int lens_model(int model, const double* K, const double* D, int n_dist, const double* R, const double* P, int w, int h,
                      CamModel* cm, LensExt* lx, bool* lens) {
  memset(cm, 0, sizeof *cm);
  memset(lx, 0, sizeof *lx);
  if (!dist_count_ok(model, n_dist)) return LENS_BAD_COUNT;
  const bool rotated = R && !is_identity3(R);
  double PR[9];
  if (rotated) mul3(P, R, PR);
  if (!inv3(rotated ? PR : P, cm->iR)) return LENS_SINGULAR;
  for (int i = 0; i < n_dist && i < (model == 0 ? 4 : 5); ++i) cm->k[i] = D[i];
  for (int i = 5; i < n_dist && i < 12; ++i) lx->k[i - 5] = D[i];
  tilt_matrix(n_dist == 14 ? D[12] : 0., n_dist == 14 ? D[13] : 0., lx->T);
  cm->fx = K[0]; cm->fy = K[4]; cm->cx = K[2]; cm->cy = K[5];
  cm->model = model; cm->w = w; cm->h = h;
  if (model == 0) {
    *lens = rotated && !xs_table_applies(*cm);
  } else {
    bool extra = !is_identity3(lx->T);
    for (double k : lx->k) extra = extra || k != 0.;
    *lens = extra;
  }
  return LENS_OK;
}

// Does R make the rays of cm depend on the row, so that the map builds walk them (walk_rays) and the LENS = 1 instances
// read them?  Without R (or with R = I) the rays keep the column table or the direct form.
inline bool rays_walk(const CamModel& cm, const double* R) { return R && !is_identity3(R) && !xs_table_applies(cm); }

// A fisheye whose rays walk: a fused gather cannot walk its per-pixel rays, so only a map-resident slot takes it.
inline bool fisheye_walks(const CamModel& cm, bool lens) { return lens && cm.model == 0; }

// CV_16SC2 + CV_16UC1 quantisation of (u,v): map1 = (iu>>5, iv>>5) as int16 (wrapping
// cast), map2 = (iv&31)*32 + (iu&31).
// `saturate`: cv2.initUndistortRectifyMap's (pinhole) vector body packs with signed
// saturation for columns j < W - W%8; everything else wraps like the C cast it is.
__host__ __device__ __forceinline__ void quantise_uv(double u, double v, short& mx, short& my, unsigned short& frac,
                                            bool saturate = false) {
  const int iu = cv_round(dmul(u, (double)TAB));
  const int iv = cv_round(dmul(v, (double)TAB));
  const int hx = iu >> INTER_BITS, hy = iv >> INTER_BITS;
  mx = saturate ? (short)max(-32768, min(32767, hx)) : (short)hx;
  my = saturate ? (short)max(-32768, min(32767, hy)) : (short)hy;
  frac = (unsigned short)((iv & (TAB - 1)) * TAB + (iu & (TAB - 1)));
}

// A3: fixed-point pre-image of destination pixel (x,y) under cv2.warpPerspective.
// unit = 32 for INTER_LINEAR, 1 for INTER_NEAREST.  OpenCV evaluates in 64-pixel blocks.
__host__ __device__ __forceinline__ void warp_point(const Homog& hm, int x, int y, double unit, int& X, int& Y) {
  const double* M = hm.M;
  const int bxi = (x >> 6) << 6;
  const double bx = (double)bxi, x1 = (double)(x - bxi), dy = (double)y;
  const double X0 = dadd(dadd(dmul(M[0], bx), dmul(M[1], dy)), M[2]);
  const double Y0 = dadd(dadd(dmul(M[3], bx), dmul(M[4], dy)), M[5]);
  const double W0 = dadd(dadd(dmul(M[6], bx), dmul(M[7], dy)), M[8]);
  double W = dadd(W0, dmul(M[6], x1));
  W = (W != 0.0) ? ddiv(unit, W) : 0.0;
  double fX = dmul(dadd(X0, dmul(M[0], x1)), W);
  double fY = dmul(dadd(Y0, dmul(M[3], x1)), W);
  fX = fmax(-2147483648.0, fmin(2147483647.0, fX));   // std::max(INT_MIN, std::min(INT_MAX, .))
  fY = fmax(-2147483648.0, fmin(2147483647.0, fY));
  X = cv_round(fX);
  Y = cv_round(fY);
}

// A3': cv2.warpAffine.  Unless WARP_INVERSE_MAP is set, cv2 inverts M with invertAffineTransform's closed form (a
// singular M gives D = 0 and the zero matrix's translation part); the inverse lives in Homog::M[0..5].
inline void inv_affine(const double* S, double* T) {
  double D = S[0] * S[4] - S[1] * S[3];
  D = D != 0. ? 1. / D : 0.;
  const double A11 = S[4] * D, A22 = S[0] * D, A12 = S[1] * -D, A21 = S[3] * -D;
  T[0] = A11; T[1] = A12; T[3] = A21; T[4] = A22;
  T[2] = -T[0] * S[2] - T[1] * S[5];
  T[5] = -T[3] * S[2] - T[4] * S[5];
}

// Fixed-point pre-image of destination pixel (x,y) under cv2.warpAffine (AB_BITS = 10): X = (X0(y) + adelta(x)) >> 5
// at TAB scale (every flag but NEAREST), >> 10 in whole pixels for NEAREST.  The int sum wraps as cv2's SIMD add does;
// the consumers saturate X >> 5 to int16 as cv2's pack does.
__host__ __device__ __forceinline__ void affine_point(const Homog& hm, int x, int y, bool nearest, int& X, int& Y) {
  const double* M = hm.M;
  const int round_delta = nearest ? 512 : 16, shift = nearest ? 10 : 10 - INTER_BITS;
  const double dy = (double)y, dx = (double)x;
  const unsigned X0 = (unsigned)cv_round(dmul(dadd(dmul(M[1], dy), M[2]), 1024.)) + round_delta;
  const unsigned Y0 = (unsigned)cv_round(dmul(dadd(dmul(M[4], dy), M[5]), 1024.)) + round_delta;
  X = (int)(X0 + (unsigned)cv_round(dmul(dmul(M[0], dx), 1024.))) >> shift;
  Y = (int)(Y0 + (unsigned)cv_round(dmul(dmul(M[3], dx), 1024.))) >> shift;
}

__host__ __device__ __forceinline__ int sat_i16(int v) { return max(-32768, min(32767, v)); }

// ---- CV_32FC1 / CV_32FC2 maps ------------------------------------------------
// cv2 stores a float map entry as (float)u of the double the CV_16SC2 build quantises.
__host__ __device__ __forceinline__ float d2f(double v) {
#ifdef __CUDA_ARCH__
  return __double2float_rn(v);
#else
  return (float)v;
#endif
}

// cvRound(float) / saturate_cast<int>(float) on x86 (cvtss2si): INT_MIN for NaN, +-inf and anything outside the int
// range.  PTX cvt.rni.s32.f32 saturates instead and gives 0 for NaN.
__host__ __device__ __forceinline__ int x86_round(float v) {
  if (!(fabsf(v) < 2147483648.f)) return INT_MIN;
  return f2i_rn(v);
}

// cv2.convertMaps(x, y, CV_16SC2, nninterpolation), which is what cv2.remap does to float maps before its integer
// remap.  Non-NEAREST: ix = cvRound(x * 32.f) in float, map1 = saturate_cast<short>(ix >> 5), frac = (iy & 31) * 32 +
// (ix & 31).  NEAREST: map1 = saturate_cast<short>(cvRound(x)), rounding half to even on the float itself, and no frac
// (so no NNDeltaTab rule either).
__host__ __device__ __forceinline__ void quantise_xy(float x, float y, bool nearest, short& mx, short& my, unsigned short& frac) {
  if (nearest) {
    mx = (short)sat_i16(x86_round(x));
    my = (short)sat_i16(x86_round(y));
    frac = 0;
    return;
  }
  const int ix = x86_round(fmul(x, (float)TAB)), iy = x86_round(fmul(y, (float)TAB));
  mx = (short)sat_i16(ix >> INTER_BITS);
  my = (short)sat_i16(iy >> INTER_BITS);
  frac = (unsigned short)((iy & (TAB - 1)) * TAB + (ix & (TAB - 1)));
}

// cv2.convertMaps(CV_16SC2 [+ CV_16UC1] -> CV_32F): x + (frac & 31) / 32, exact in float.  No map2 is frac 0.
__host__ __device__ __forceinline__ void unquantise_xy(short mx, short my, unsigned frac, float& x, float& y) {
  frac &= TAB * TAB - 1;
  x = fadd((float)mx, fmul((float)(frac & (TAB - 1)), 1.f / TAB));
  y = fadd((float)my, fmul((float)(frac >> INTER_BITS), 1.f / TAB));
}

// ---- byte-lane primitives with a host form ------------------------------------
// The packed integer arithmetic of the gathers (interp_fast, sat_add_bgr, the tile write-out) is built from
// these; on the device they are single SASS instructions (PRMT, SHF, IDP.2A, VADDUS4-style), on the host plain
// C, so tests/host/kernel_math.cu can check the packed forms against the scalar definitions without a GPU.
__host__ __device__ __forceinline__ unsigned lane_perm(unsigned a, unsigned b, unsigned sel) {
#ifdef __CUDA_ARCH__
  return __byte_perm(a, b, sel);
#else
  const unsigned long long v = ((unsigned long long)b << 32) | a;   // selector nibbles 0..7 only (no sign replication here)
  unsigned r = 0;
  for (int i = 0; i < 4; ++i) r |= (unsigned)((v >> (8 * ((sel >> (4 * i)) & 7u))) & 255u) << (8 * i);
  return r;
#endif
}
__host__ __device__ __forceinline__ unsigned lane_funnel_r(unsigned lo, unsigned hi, unsigned shift) {
#ifdef __CUDA_ARCH__
  return __funnelshift_r(lo, hi, shift);
#else
  shift &= 31u;
  return shift ? (lo >> shift) | (hi << (32u - shift)) : lo;
#endif
}
// two unsigned 16-bit weights (a) times the low / high byte pair of b, plus c
__host__ __device__ __forceinline__ unsigned lane_dp2a_lo(unsigned a, unsigned b, unsigned c) {
#ifdef __CUDA_ARCH__
  return __dp2a_lo(a, b, c);
#else
  return c + (a & 0xffffu) * (b & 255u) + (a >> 16) * ((b >> 8) & 255u);
#endif
}
__host__ __device__ __forceinline__ unsigned lane_dp2a_hi(unsigned a, unsigned b, unsigned c) {
#ifdef __CUDA_ARCH__
  return __dp2a_hi(a, b, c);
#else
  return c + (a & 0xffffu) * ((b >> 16) & 255u) + (a >> 16) * (b >> 24);
#endif
}
__host__ __device__ __forceinline__ unsigned lane_addus4(unsigned a, unsigned b) {   // per-byte saturating add
#ifdef __CUDA_ARCH__
  return __vaddus4(a, b);
#else
  unsigned r = 0;
  for (int i = 0; i < 4; ++i) {
    const unsigned t = ((a >> (8 * i)) & 255u) + ((b >> (8 * i)) & 255u);
    r |= (t > 255u ? 255u : t) << (8 * i);
  }
  return r;
#endif
}

// A2: (sum w*p + 512) >> 10 with integer weights.
__host__ __device__ __forceinline__ int bilerp_q10(int p00, int p01, int p10, int p11, int fx, int fy) {
  const int w11 = fx * fy, w01 = (fx << 5) - w11, w10 = (fy << 5) - w11;
  const int w00 = 1024 - (fx << 5) - (fy << 5) + w11;
  return (w00 * p00 + w01 * p01 + w10 * p10 + w11 * p11 + 512) >> 10;
}

// ---- A9: OpenCV's 8-bit BGR -> HSV -> (V + delta) -> BGR round trip ------------
// sdiv[i] = cvRound((255<<12)/i), hdiv[i] = cvRound((180<<12)/(6 i)); filled on the host.
struct HsvTables { int sdiv[256]; int hdiv[256]; };

__host__ __device__ __forceinline__ void hsv_roundtrip(int& b, int& g, int& r, int delta, bool rounding_tail,
                                              const int* __restrict__ sdiv, const int* __restrict__ hdiv) {
  const int v = max(b, max(g, r)), mn = min(b, min(g, r));
  const int d = v - mn;
  const int s = (d * sdiv[v] + 2048) >> 12;
  int hh = (v == r) ? (g - b) : ((v == g) ? (b - r + 2 * d) : (r - g + 4 * d));
  hh = (hh * hdiv[d] + 2048) >> 12;
  if (hh < 0) hh += 180;
  const int v2 = max(0, min(255, v + delta));
  // HSV2BGR, OpenCV's vector body: fp32 with these exact FMA contractions, truncation.
  const float sf = fmul((float)s, 1.0f / 255.0f);
  const float vf = fmul((float)v2, 1.0f / 255.0f);
  const float hx = fmul((float)hh, 6.0f / 180.0f);
  const float secf = truncf(hx);
  const float f = fsub(hx, secf);
  int sec = (int)secf;
  sec = sec % 6;
  const float t0 = vf;
  const float t1 = fmul(vf, fsub(1.0f, sf));
  const float t2 = fmul(vf, ffma(-sf, f, 1.0f));
  const float t3 = fmul(vf, ffma(-sf, fsub(1.0f, f), 1.0f));
  // sector table {1,3,0},{1,0,2},{3,0,1},{0,2,1},{0,1,3},{2,1,0} (b, g, r pick t[.]), anything else like sector 5 --
  // as selects, not as a switch: neighbouring pixels lie in different sectors, and a six-way divergent branch per pixel was
  // what k_lum_spans spent its time on.  Two bits per sector and channel:
  const unsigned sc = (unsigned)sec > 5u ? 10u : 2u * (unsigned)sec;
  const unsigned ib = ((1u | 1u << 2 | 3u << 4 | 0u << 6 | 0u << 8 | 2u << 10) >> sc) & 3u;
  const unsigned ig = ((3u | 0u << 2 | 0u << 4 | 2u << 6 | 1u << 8 | 1u << 10) >> sc) & 3u;
  const unsigned ir = ((0u | 2u << 2 | 1u << 4 | 1u << 6 | 3u << 8 | 0u << 10) >> sc) & 3u;
  float fb = (ib & 2u) ? ((ib & 1u) ? t3 : t2) : ((ib & 1u) ? t1 : t0);
  float fg = (ig & 2u) ? ((ig & 1u) ? t3 : t2) : ((ig & 1u) ? t1 : t0);
  float fr = (ir & 2u) ? ((ir & 1u) ? t3 : t2) : ((ir & 1u) ? t1 : t0);
  fb = fmul(fb, 255.0f); fg = fmul(fg, 255.0f); fr = fmul(fr, 255.0f);
  if (rounding_tail) {   // the < 32-pixel row tail goes through OpenCV's scalar path, which rounds
    b = max(0, min(255, f2i_rn(fb)));
    g = max(0, min(255, f2i_rn(fg)));
    r = max(0, min(255, f2i_rn(fr)));
  } else {
    b = max(0, min(255, (int)fb));
    g = max(0, min(255, (int)fg));
    r = max(0, min(255, (int)fr));
  }
}

}  // namespace bevk
