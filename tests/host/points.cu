// Host build of the point kernels' per-point code (point_op of k_points, after points_camera, the set-up bevk_api.cu
// does).  Built and run by tests/test_host_points.py with nvcc (host code only is executed), compared there with live
// cv2 bit for bit.
//   points run <op> <model> <depth> <n> <n_dist> <n_r> <has_P> <crit> <max_count> <in.bin> <out.bin>
//       stdin: K[9] D[n_dist] R[n_r] P[9 if has_P] t[3] alpha eps as C99 hex floats.  depth: 5 (float32) or 6 (float64).
//       in: n points of 2 (3 for PT_PROJECT) elements; out: n points of 2.  Exit 3: points_camera refused the camera.
//   points rodrigues
//       stdin: rvec[3]; stdout: the rotation's 9 entries as hex floats
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_points.cuh"

using namespace bevk;

static bool read_doubles(double* v, int n) {
  for (int i = 0; i < n; ++i) {
    char tok[64];
    if (scanf("%63s", tok) != 1) return false;
    v[i] = strtod(tok, nullptr);
  }
  return true;
}

template <int OP, int MODEL, class T>
static void run_all(const PointCam& c, const void* in, void* out, long long n) {
  for (long long i = 0; i < n; ++i) point_op<OP, MODEL, T>(c, (const T*)in, (T*)out, i);
}

template <class T>
static int dispatch(int op, int model, const PointCam& c, const void* in, void* out, long long n) {
  if (op == PT_UNDISTORT && model == 0) run_all<PT_UNDISTORT, 0, T>(c, in, out, n);
  else if (op == PT_UNDISTORT) run_all<PT_UNDISTORT, 1, T>(c, in, out, n);
  else if (op == PT_PROJECT && model == 0) run_all<PT_PROJECT, 0, T>(c, in, out, n);
  else if (op == PT_PROJECT) run_all<PT_PROJECT, 1, T>(c, in, out, n);
  else if (op == PT_DISTORT) run_all<PT_DISTORT, 0, T>(c, in, out, n);
  else if (op == PT_PERSPECTIVE) run_all<PT_PERSPECTIVE, 0, T>(c, in, out, n);
  else return 2;
  return 0;
}

static int mode_run(char** a) {
  const int op = atoi(a[0]), model = atoi(a[1]), depth = atoi(a[2]);
  const long long n = atoll(a[3]);
  const int n_dist = atoi(a[4]), n_r = atoi(a[5]), has_p = atoi(a[6]), crit = atoi(a[7]), max_count = atoi(a[8]);
  double K[9], D[16], R[9], P[9], t[3], alpha, eps;
  if (n_dist < 0 || n_dist > 16 || n_r < 0 || n_r > 9 || !read_doubles(K, 9) || !read_doubles(D, n_dist) ||
      !read_doubles(R, n_r) || (has_p && !read_doubles(P, 9)) || !read_doubles(t, 3) || !read_doubles(&alpha, 1) ||
      !read_doubles(&eps, 1))
    return 2;
  PointCam c;
  if (op == PT_PERSPECTIVE) {
    memset(&c, 0, sizeof c);
    memcpy(c.RR, K, sizeof c.RR);
  } else if (points_camera(op, model, K, n_dist ? D : nullptr, n_dist, n_r ? R : nullptr, n_r, has_p ? P : nullptr, t, alpha,
                           crit, max_count, eps, &c) != PTS_OK) {
    return 3;
  }
  const size_t es = depth == 6 ? 8 : 4, in_n = op == PT_PROJECT ? 3 : 2;
  std::vector<unsigned char> in(n * in_n * es + 8), out(n * 2 * es + 8);
  FILE* f = fopen(a[9], "rb");
  if (!f) return 4;
  if (fread(in.data(), es * in_n, n, f) != (size_t)n) return 5;
  fclose(f);
  const int r = depth == 6 ? dispatch<double>(op, model, c, in.data(), out.data(), n)
                           : dispatch<float>(op, model, c, in.data(), out.data(), n);
  if (r) return r;
  f = fopen(a[10], "wb");
  if (!f) return 4;
  fwrite(out.data(), es * 2, n, f);
  fclose(f);
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 13 && !strcmp(argv[1], "run")) return mode_run(argv + 2);
  if (argc >= 2 && !strcmp(argv[1], "rodrigues")) {
    double rv[3], R[9];
    if (!read_doubles(rv, 3)) return 2;
    rodrigues(rv, R);
    for (double v : R) printf("%a\n", v);
    return 0;
  }
  fprintf(stderr, "usage: points run ... | points rodrigues\n");
  return 2;
}
