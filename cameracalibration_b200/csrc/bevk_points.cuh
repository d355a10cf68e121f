// bevk_points.cuh -- cv2's point functions on the device (sm_90a): undistortPoints / undistortPointsIter,
// fisheye.undistortPoints, projectPoints, fisheye.projectPoints, fisheye.distortPoints and perspectiveTransform (2-D points,
// 3x3 matrix).  One thread per point.  The per-point forms are __host__ __device__ so that tests/host/points.cu runs them
// on the CPU against live cv2; like the map code they are FP64 without contraction (dadd / dmul / ddiv), in the order
// OpenCV 4.13's scalar C++ evaluates them.  DESIGN.md §2 records each order and the rules below.
#pragma once
#include "bevk_device.cuh"

namespace bevk {

enum { PT_UNDISTORT = 0, PT_PROJECT = 1, PT_DISTORT = 2, PT_PERSPECTIVE = 3 };
enum { CRIT_COUNT = 1, CRIT_EPS = 2 };   // cv2.TermCriteria_COUNT / _EPS

// One camera's constants, set up on the host (points_camera) and passed to the kernel by value.
struct PointCam {
  double fx, fy, cx, cy, ifx, ify;   // ifx = 1./fx, as cv2.undistortPoints forms it
  double k[14];                      // cv2's k[0..13] (pinhole: k1 k2 p1 p2 k3 k4 k5 k6 s1 s2 s3 s4 tauX tauY; fisheye k1..k4)
  double RR[9];                      // undistort: P * R (pinhole: cvMatMul's sums; fisheye: Matx's); project: the rotation;
                                     // perspective: the matrix
  double t[3];                       // project: tvec
  double T[9], iT[9];                // pinhole: the tilt matrix and its inverse (identity without tilt)
  double alpha;                      // fisheye skew
  double eps;                        // criteria.epsilon
  int max_count, crit;               // criteria.maxCount, criteria.type
  int has_dist;                      // pinhole undistort: a D was given (cv2 skips the iteration without one)
  int has_rr;                        // undistort: an R or a P was given (without either, cv2 returns the normalised point)
};

#ifdef __CUDA_ARCH__
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dfma(double a, double b, double c) { return __fma_rn(a, b, c); }
#else
inline double dsub(double a, double b) { volatile double r = a - b; return r; }
inline double dfma(double a, double b, double c) { return fma(a, b, c); }
#endif

// a result stored as T: (float) or the double itself
template <class T> __host__ __device__ __forceinline__ T to_t(double v);
template <> __host__ __device__ __forceinline__ float to_t<float>(double v) { return d2f(v); }
template <> __host__ __device__ __forceinline__ double to_t<double>(double v) { return v; }

// cv::Matx * Vec: each entry a sum from 0 (so -0 becomes +0, as cv2's does), left to right
__host__ __device__ __forceinline__ double mrow(const double* M, int r, double a, double b, double c) {
  double s = 0.;
  s = dadd(s, dmul(M[r * 3], a));
  s = dadd(s, dmul(M[r * 3 + 1], b));
  return dadd(s, dmul(M[r * 3 + 2], c));
}

// std::min / std::max as cv2 calls them: NaN in the second argument loses, in the first it wins
__host__ __device__ __forceinline__ double std_max(double a, double b) { return (a < b) ? b : a; }
__host__ __device__ __forceinline__ double std_min(double a, double b) { return (b < a) ? b : a; }

// cvProjectPoints2Internal's distortion of a normalised point (x, y): rational, thin prism, tilt, then the pixel
__host__ __device__ __forceinline__ void pinhole_distort(const PointCam& c, double x, double y, double& u, double& v) {
  const double* k = c.k;
  const double r2 = dadd(dmul(x, x), dmul(y, y)), r4 = dmul(r2, r2), r6 = dmul(r4, r2);
  const double a1 = dmul(dmul(2., x), y), a2 = dadd(r2, dmul(dmul(2., x), x)), a3 = dadd(r2, dmul(dmul(2., y), y));
  const double cdist = dadd(dadd(dadd(1., dmul(k[0], r2)), dmul(k[1], r4)), dmul(k[4], r6));
  const double icdist2 = ddiv(1., dadd(dadd(dadd(1., dmul(k[5], r2)), dmul(k[6], r4)), dmul(k[7], r6)));
  const double xd0 = dadd(dadd(dadd(dadd(dmul(dmul(x, cdist), icdist2), dmul(k[2], a1)), dmul(k[3], a2)), dmul(k[8], r2)),
                          dmul(k[9], r4));
  const double yd0 = dadd(dadd(dadd(dadd(dmul(dmul(y, cdist), icdist2), dmul(k[2], a3)), dmul(k[3], a1)), dmul(k[10], r2)),
                          dmul(k[11], r4));
  const double vx = mrow(c.T, 0, xd0, yd0, 1.), vy = mrow(c.T, 1, xd0, yd0, 1.), vz = mrow(c.T, 2, xd0, yd0, 1.);
  const double ip = vz != 0. ? ddiv(1., vz) : 1.;
  u = dadd(dmul(dmul(ip, vx), c.fx), c.cx);
  v = dadd(dmul(dmul(ip, vy), c.fy), c.cy);
}

// cv2.undistortPoints / undistortPointsIter (cvUndistortPointsInternal) of pixel (u, v).  When icdist < 0 cv2 restarts
// from the raw normalised point and stops iterating.
__host__ __device__ __forceinline__ void undistort_pinhole(const PointCam& c, double u, double v, double& ox, double& oy) {
  double x = dmul(dsub(u, c.cx), c.ifx), y = dmul(dsub(v, c.cy), c.ify);
  if (c.has_dist) {
    const double* k = c.k;
    const double ux = mrow(c.iT, 0, x, y, 1.), uy = mrow(c.iT, 1, x, y, 1.), uz = mrow(c.iT, 2, x, y, 1.);
    const double ip = uz != 0. ? ddiv(1., uz) : 1.;
    const double x0 = dmul(ip, ux), y0 = dmul(ip, uy);
    x = x0; y = y0;
    for (int j = 0; j < c.max_count; ++j) {   // COUNT only: points_camera refuses the pinhole EPS criterion
      const double r2 = dadd(dmul(x, x), dmul(y, y));
      const double icdist = ddiv(dadd(1., dmul(dadd(dmul(dadd(dmul(k[7], r2), k[6]), r2), k[5]), r2)),
                                 dadd(1., dmul(dadd(dmul(dadd(dmul(k[4], r2), k[1]), r2), k[0]), r2)));
      if (icdist < 0) {
        x = dmul(dsub(u, c.cx), c.ifx);
        y = dmul(dsub(v, c.cy), c.ify);
        break;
      }
      const double dX = dadd(dadd(dadd(dmul(dmul(dmul(2., k[2]), x), y), dmul(k[3], dadd(r2, dmul(dmul(2., x), x)))),
                                  dmul(k[8], r2)), dmul(dmul(k[9], r2), r2));
      const double dY = dadd(dadd(dadd(dmul(k[2], dadd(r2, dmul(dmul(2., y), y))), dmul(dmul(dmul(2., k[3]), x), y)),
                                  dmul(k[10], r2)), dmul(dmul(k[11], r2), r2));
      x = dmul(dsub(x0, dX), icdist);
      y = dmul(dsub(y0, dY), icdist);
    }
  }
  if (!c.has_rr) {
    ox = x; oy = y;
    return;
  }
  const double xx = dadd(dadd(dmul(c.RR[0], x), dmul(c.RR[1], y)), c.RR[2]);
  const double yy = dadd(dadd(dmul(c.RR[3], x), dmul(c.RR[4], y)), c.RR[5]);
  const double ww = ddiv(1., dadd(dadd(dmul(c.RR[6], x), dmul(c.RR[7], y)), c.RR[8]));
  ox = dmul(xx, ww);
  oy = dmul(yy, ww);
}

// cv2.fisheye.undistortPoints of pixel (u, v): theta_d clamped to +-pi/2 (NaN becomes -pi/2, as std::max does), Newton
// steps, scale = tan(theta) / theta_d; |theta_d| < eps leaves scale 0 (the point maps to the principal ray).  A point
// that did not converge under EPS, or whose theta changed sign, is (-1e6, -1e6).
__host__ __device__ __forceinline__ void undistort_fisheye(const PointCam& c, double u, double v, double& ox, double& oy) {
  const double* k = c.k;
  const double pwx = ddiv(dsub(u, c.cx), c.fx), pwy = ddiv(dsub(v, c.cy), c.fy);
  double scale = 0.0;
  double theta_d = dsqrt(dadd(dmul(pwx, pwx), dmul(pwy, pwy)));
  theta_d = std_min(std_max(-M_PI / 2., theta_d), M_PI / 2.);
  const bool is_eps = (c.crit & CRIT_EPS) != 0;
  const int max_count = c.max_count;   // points_camera requires COUNT
  bool converged = false;
  double theta = theta_d;
  if (fabs(theta_d) >= c.eps) {
    for (int j = 0; j < max_count; ++j) {
      const double t2 = dmul(theta, theta), t4 = dmul(t2, t2), t6 = dmul(t4, t2), t8 = dmul(t6, t2);
      const double k0t2 = dmul(k[0], t2), k1t4 = dmul(k[1], t4), k2t6 = dmul(k[2], t6), k3t8 = dmul(k[3], t8);
      const double num = dsub(dmul(theta, dadd(dadd(dadd(dadd(1., k0t2), k1t4), k2t6), k3t8)), theta_d);
      const double den = dadd(dadd(dadd(dadd(1., dmul(3., k0t2)), dmul(5., k1t4)), dmul(7., k2t6)), dmul(9., k3t8));
      const double fix = ddiv(num, den);
      theta = dsub(theta, fix);
      if (is_eps && fabs(fix) < c.eps) {
        converged = true;
        break;
      }
    }
    scale = ddiv(tan(theta), theta_d);
  } else {
    converged = true;
  }
  const bool flipped = (theta_d < 0 && theta > 0) || (theta_d > 0 && theta < 0);
  if ((converged || !is_eps) && !flipped) {
    const double px = dmul(pwx, scale), py = dmul(pwy, scale);
    if (!c.has_rr) {
      ox = px; oy = py;
      return;
    }
    const double rx = mrow(c.RR, 0, px, py, 1.), ry = mrow(c.RR, 1, px, py, 1.), rz = mrow(c.RR, 2, px, py, 1.);
    ox = ddiv(rx, rz);
    oy = ddiv(ry, rz);
  } else {
    ox = oy = -1000000.0;
  }
}

// cv::fisheye::distortPoints of a normalised point, and the tail of cv::fisheye::projectPoints
__host__ __device__ __forceinline__ void fisheye_distort(const PointCam& c, double x, double y, double& u, double& v) {
  const double* k = c.k;
  const double r = dsqrt(dadd(dmul(x, x), dmul(y, y)));
  const double th = atan(r);
  const double t2 = dmul(th, th), t3 = dmul(t2, th), t4 = dmul(t2, t2), t5 = dmul(t4, th), t6 = dmul(t3, t3),
               t7 = dmul(t6, th), t8 = dmul(t4, t4), t9 = dmul(t8, th);
  const double thd = dadd(dadd(dadd(dadd(th, dmul(k[0], t3)), dmul(k[1], t5)), dmul(k[2], t7)), dmul(k[3], t9));
  const double inv_r = r > 1e-8 ? ddiv(1.0, r) : 1.;
  const double cdist = r > 1e-8 ? dmul(thd, inv_r) : 1.;
  const double x1 = dmul(x, cdist), y1 = dmul(y, cdist);
  const double x3 = dadd(x1, dmul(c.alpha, y1));
  u = dadd(dmul(x3, c.fx), c.cx);
  v = dadd(dmul(y1, c.fy), c.cy);
}

// cv2.projectPoints (cvProjectPoints2Internal) / cv2.fisheye.projectPoints of object point (X, Y, Z)
template <int MODEL>
__host__ __device__ __forceinline__ void project_point(const PointCam& c, double X, double Y, double Z, double& u, double& v) {
  const double* R = c.RR;
  const double x = dadd(dadd(dadd(dmul(R[0], X), dmul(R[1], Y)), dmul(R[2], Z)), c.t[0]);
  const double y = dadd(dadd(dadd(dmul(R[3], X), dmul(R[4], Y)), dmul(R[5], Z)), c.t[1]);
  double z = dadd(dadd(dadd(dmul(R[6], X), dmul(R[7], Y)), dmul(R[8], Z)), c.t[2]);
  if (MODEL == 0) {                       // Affine3d * Xi, then fabs(z) < DBL_MIN -> 1 and x / z
    if (fabs(z) < 2.2250738585072014e-308) z = 1.;
    fisheye_distort(c, ddiv(x, z), ddiv(y, z), u, v);
  } else {                                // z = z ? 1./z : 1, x *= z
    z = z != 0. ? ddiv(1., z) : 1.;
    pinhole_distort(c, dmul(x, z), dmul(y, z), u, v);
  }
}

// cv2.perspectiveTransform of a 2-D point by a 3x3 M; |w| <= FLT_EPSILON gives (0, 0).  The element is promoted to
// double, and cv2's body contracts each row's first product pair into one FMA: fma(x, m0, y * m1) + m2, for float32 and
// float64 alike (bit for bit on the host test's corpus; fma is correctly rounded on both sides).
template <class T>
__host__ __device__ __forceinline__ double persp_row(const double* m, int r, T x, T y) {
  return dadd(dfma((double)x, m[3 * r], dmul((double)y, m[3 * r + 1])), m[3 * r + 2]);
}
template <class T>
__host__ __device__ __forceinline__ void perspective_point(const double* m, T x, T y, T& ox, T& oy) {
  double w = persp_row<T>(m, 2, x, y);
  if (fabs(w) > 1.1920928955078125e-07) {
    w = ddiv(1., w);
    ox = to_t<T>(dmul(persp_row<T>(m, 0, x, y), w));
    oy = to_t<T>(dmul(persp_row<T>(m, 1, x, y), w));
  } else {
    ox = oy = (T)0;
  }
}

// One point of op OP (camera model MODEL where the op has one): src holds 2 (3 for PT_PROJECT) T per point, dst 2.
template <int OP, int MODEL, class T>
__host__ __device__ __forceinline__ void point_op(const PointCam& c, const T* src, T* dst, long long i) {
  double u, v;
  if (OP == PT_PERSPECTIVE) {
    T ox, oy;
    perspective_point<T>(c.RR, src[2 * i], src[2 * i + 1], ox, oy);
    dst[2 * i] = ox; dst[2 * i + 1] = oy;
    return;
  }
  if (OP == PT_PROJECT) {
    project_point<MODEL>(c, (double)src[3 * i], (double)src[3 * i + 1], (double)src[3 * i + 2], u, v);
  } else {
    const double x = (double)src[2 * i], y = (double)src[2 * i + 1];
    if (OP == PT_DISTORT) fisheye_distort(c, x, y, u, v);
    else if (MODEL == 0) undistort_fisheye(c, x, y, u, v);
    else undistort_pinhole(c, x, y, u, v);
  }
  dst[2 * i] = to_t<T>(u);
  dst[2 * i + 1] = to_t<T>(v);
}

template <int OP, int MODEL, class T>
__global__ void __launch_bounds__(256) k_points(PointCam c, const T* src, T* dst, long long n) {
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (long long)gridDim.x * 256) point_op<OP, MODEL, T>(c, src, dst, i);
}

// ---- host set-up (tests/host/points.cu runs it against cv2)

// cv::Rodrigues of an rvec (and cv::Affine3d(rvec)'s rotation, which is the same formula): R = c I + (1 - c) r r^T +
// s [r]x over theta = |rvec|, entry by entry; theta < DBL_EPSILON is the identity.
inline void rodrigues(const double* rv, double* R) {
  const double theta = sqrt(dadd(dadd(dmul(rv[0], rv[0]), dmul(rv[1], rv[1])), dmul(rv[2], rv[2])));
  if (theta < 2.220446049250313e-16) {
    for (int i = 0; i < 9; ++i) R[i] = i % 4 == 0 ? 1. : 0.;
    return;
  }
  const double c = cos(theta), s = sin(theta), c1 = 1. - c, it = theta != 0. ? 1. / theta : 0.;
  const double rx = dmul(rv[0], it), ry = dmul(rv[1], it), rz = dmul(rv[2], it);
  const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  const double rrt[9] = {dmul(rx, rx), dmul(rx, ry), dmul(rx, rz), dmul(rx, ry), dmul(ry, ry), dmul(ry, rz),
                         dmul(rx, rz), dmul(ry, rz), dmul(rz, rz)};
  const double rk[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
  for (int i = 0; i < 9; ++i) R[i] = dadd(dadd(dmul(c, I[i]), dmul(c1, rrt[i])), dmul(s, rk[i]));
}

// cv::Matx33d product A * B, sums from 0
inline void matx_mul3(const double* A, const double* B, double* C) {
  double t[9];
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 3; ++k) t[r * 3 + k] = mrow(A, r, B[k], B[3 + k], B[6 + k]);
  memcpy(C, t, sizeof t);
}

enum { PTS_OK = 0, PTS_BAD_COUNT = 1, PTS_BAD_CRITERIA = 2, PTS_EPS_UNFOLLOWED = 3, PTS_TOO_MANY_ITERATIONS = 4 };
// The most iterations one point may take: each is a few FP64 divisions, and a launch over millions of points with an
// unbounded count would hold a shared device for minutes.  cv2's defaults are 5 (pinhole) and 10 (fisheye).
constexpr int MAX_POINT_ITERATIONS = 1000;

// The PointCam of one call.  K: 3x3.  D: n_dist coefficients (D == null or n_dist == 0: none).  R: null, 9 entries
// (3x3) or, for the fisheye, 3 (an rvec: cv::Affine3d's rotation), as n_r says.  P: null or 3x3.  For PT_PROJECT, R
// is the rvec (n_r == 3) and t the tvec.  crit / max_count / eps: cv2.TermCriteria.  Refused: a criteria without COUNT
// (cv2 then iterates without bound, and a point that never converges would never finish), more than
// MAX_POINT_ITERATIONS iterations, and the pinhole EPS criterion (cv2.undistortPointsIter's reprojection-error stop is
// not restated).
inline int points_camera(int op, int model, const double* K, const double* D, int n_dist, const double* R, int n_r,
                         const double* P, const double* t, double alpha, int crit, int max_count, double eps, PointCam* c) {
  memset(c, 0, sizeof *c);
  if (D == nullptr) n_dist = 0;
  if (!dist_count_ok(model, n_dist)) return PTS_BAD_COUNT;
  if (op == PT_UNDISTORT && !(crit & CRIT_COUNT)) return PTS_BAD_CRITERIA;
  if (op == PT_UNDISTORT && max_count > MAX_POINT_ITERATIONS) return PTS_TOO_MANY_ITERATIONS;
  if (op == PT_UNDISTORT && model == 1 && (crit & CRIT_EPS)) return PTS_EPS_UNFOLLOWED;
  for (int i = 0; i < n_dist; ++i) c->k[i] = D[i];
  c->fx = K[0]; c->fy = K[4]; c->cx = K[2]; c->cy = K[5];
  c->ifx = 1. / c->fx; c->ify = 1. / c->fy;
  c->alpha = alpha; c->eps = eps; c->max_count = max_count; c->crit = crit;
  c->has_dist = n_dist > 0;
  // cv::detail::computeTiltProjectionMatrix: the matrix when tauX or tauY is non-zero, else the identity (both)
  for (int i = 0; i < 9; ++i) c->T[i] = c->iT[i] = i % 4 == 0 ? 1. : 0.;
  if (model == 1 && (c->k[12] != 0 || c->k[13] != 0)) {
    const double tx = c->k[12], ty = c->k[13];
    const double ctx = cos(tx), stx = sin(tx), cty = cos(ty), sty = sin(ty);
    const double Rx[9] = {1, 0, 0, 0, ctx, stx, 0, -stx, ctx}, Ry[9] = {cty, 0, -sty, 0, 1, 0, sty, 0, cty};
    double Rxy[9];
    matx_mul3(Ry, Rx, Rxy);
    const double Pz[9] = {Rxy[8], 0, -Rxy[2], 0, Rxy[8], -Rxy[5], 0, 0, 1};
    matx_mul3(Pz, Rxy, c->T);
    // invMatTilt = Rxy^T * invMatProjZ, invMatProjZ = (1/R22, 0, R02/R22; 0, 1/R22, R12/R22; 0, 0, 1)
    const double inv = 1. / Rxy[8];
    const double iPz[9] = {inv, 0, Rxy[2] * inv, 0, inv, Rxy[5] * inv, 0, 0, 1};
    const double RxyT[9] = {Rxy[0], Rxy[3], Rxy[6], Rxy[1], Rxy[4], Rxy[7], Rxy[2], Rxy[5], Rxy[8]};
    matx_mul3(RxyT, iPz, c->iT);
  }
  for (int i = 0; i < 9; ++i) c->RR[i] = i % 4 == 0 ? 1. : 0.;
  if (op == PT_PROJECT) {
    if (R) rodrigues(R, c->RR);
    for (int i = 0; i < 3; ++i) c->t[i] = t[i];
  } else if (op == PT_UNDISTORT) {
    c->has_rr = R || P;
    if (R && n_r == 3) rodrigues(R, c->RR);
    else if (R) memcpy(c->RR, R, sizeof c->RR);
    if (P) {
      double PR[9];
      if (model == 1) mul3(P, c->RR, PR);   // cvMatMul(PP, RR, RR)
      else matx_mul3(P, c->RR, PR);         // RR = PP * RR
      memcpy(c->RR, PR, sizeof PR);
    }
  }
  return PTS_OK;
}

}  // namespace bevk
