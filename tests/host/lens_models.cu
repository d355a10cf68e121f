// Host build of the kernels' camera set-up and coordinate code for cv2's full lens models and rectification rotations:
// lens_model (P * R, the tilt matrix, the D counts cv2 takes), walk_rays, undistort_point<LENS>, warp_maps_pixel<1, LENS>.
// Built and run by tests/test_host_lens_models.py with nvcc (host code only is executed), compared there with live cv2.
//   lens_models maps <model> <w> <h> <n_dist> <has_R> <instance: -1 as the library picks, 0, 1> <out.bin>
//       stdin: K[9] D[n_dist] R[9 if has_R] P[9] as C99 hex floats; prints "lens <0|1> walks <0|1>" (the instance the
//       library picks, and whether it walks the rays) and exits 5 for a D length lens_model refuses
//   lens_models bevmaps <model> <w> <h> <n_dist> <bw> <bh> <out.bin>   stdin: K[9] D[n_dist] P[9] H[9]
//   lens_models rays <model> <w> <h> <n_dist> <has_R> <out.bin>   stdin as for maps; the rays camera_ray<LENS> hands to the
//       projection in the instance the library picks, as double[3][h][w] (_x, _y, _w planes)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_kernels.cuh"

using namespace bevk;

static bool read_doubles(double* v, int n) {
  for (int i = 0; i < n; ++i) {
    char tok[64];
    if (scanf("%63s", tok) != 1) return false;
    v[i] = strtod(tok, nullptr);
  }
  return true;
}

static int write_planes(const char* path, const short* m1, const unsigned short* m2, size_t n) {
  FILE* f = fopen(path, "wb");
  if (!f) return 4;
  fwrite(m1, 4, n, f);
  fwrite(m2, 2, n, f);
  fclose(f);
  return 0;
}

// As bevk_api.cu sets a camera up: lens_model, then the column table (xs_table_applies) and, for a camera that walks, the
// rays of every row.
struct Camera {
  CamModel cm;
  LensExt lx;
  bool lens = false, walks = false;
  std::vector<double> xs, rays;
  int setup(int model, const double* K, const double* D, int n, const double* R, const double* P, int w, int h) {
    const int r = lens_model(model, K, D, n, R, P, w, h, &cm, &lx, &lens);
    if (r != LENS_OK) return r;
    walks = rays_walk(cm, R);
    lens = lens || walks;
    xs.resize(w);
    if (xs_table_applies(cm)) { fill_xs_table(cm, xs.data()); cm.xs = xs.data(); }
    if (walks) {   // k_walk_rays
      rays.resize((size_t)ray_row_len(cm) * h * 3);
      for (int i = 0; i < h; ++i) walk_rays(cm, i, rays.data());
      lx.rays = rays.data();
    }
    return LENS_OK;
  }
};

static int mode_maps(int model, int w, int h, int n, int has_r, int instance, const char* path) {
  double K[9], D[16], R[9], P[9];
  if (n < 0 || n > 16 || !read_doubles(K, 9) || !read_doubles(D, n) || (has_r && !read_doubles(R, 9)) || !read_doubles(P, 9))
    return 2;
  Camera cam;
  const int r = cam.setup(model, K, D, n, has_r ? R : nullptr, P, w, h);
  if (r == LENS_BAD_COUNT) { printf("refused\n"); return 5; }
  if (r != LENS_OK) return 3;
  printf("lens %d walks %d\n", (int)cam.lens, (int)cam.walks);
  const bool full = instance < 0 ? cam.lens : instance == 1;
  const size_t N = (size_t)w * h;
  std::vector<short> m1(2 * N);
  std::vector<unsigned short> m2(N);
  for (int i = 0; i < h; ++i)
    for (int j = 0; j < w; ++j) {   // k_undistort_map<LENS>
      double u, v;
      if (full) undistort_point<1>(cam.cm, cam.lx, j, i, u, v);
      else undistort_point<0>(cam.cm, cam.lx, j, i, u, v);
      const size_t q = (size_t)i * w + j;
      quantise_uv(u, v, m1[2 * q], m1[2 * q + 1], m2[q], pack_saturates(model, j, w));
    }
  return write_planes(path, m1.data(), m2.data(), N);
}

static int mode_rays(int model, int w, int h, int n, int has_r, const char* path) {
  double K[9], D[16], R[9], P[9];
  if (n < 0 || n > 16 || !read_doubles(K, 9) || !read_doubles(D, n) || (has_r && !read_doubles(R, 9)) || !read_doubles(P, 9))
    return 2;
  Camera cam;
  if (cam.setup(model, K, D, n, has_r ? R : nullptr, P, w, h) != LENS_OK) return 3;
  const size_t N = (size_t)w * h;
  std::vector<double> out(3 * N);
  for (int i = 0; i < h; ++i)
    for (int j = 0; j < w; ++j) {
      const size_t q = (size_t)i * w + j;
      if (cam.lens) camera_ray<1>(cam.cm, cam.lx, j, i, out[q], out[N + q], out[2 * N + q]);
      else camera_ray<0>(cam.cm, cam.lx, j, i, out[q], out[N + q], out[2 * N + q]);
    }
  FILE* f = fopen(path, "wb");
  if (!f) return 4;
  fwrite(out.data(), sizeof(double), out.size(), f);
  fclose(f);
  return 0;
}

static int mode_bevmaps(int model, int uw, int uh, int n, int bw, int bh, const char* path) {
  double K[9], D[14], P[9], H[9];
  if (n < 0 || n > 14 || !read_doubles(K, 9) || !read_doubles(D, n) || !read_doubles(P, 9) || !read_doubles(H, 9)) return 2;
  Camera cam;
  if (cam.setup(model, K, D, n, nullptr, P, uw, uh) != LENS_OK) return 3;
  WarpMapsArgs a;
  memset(&a, 0, sizeof a);
  a.cm = cam.cm; a.lx = cam.lx;
  if (!inv3(H, a.hm.M)) memset(a.hm.M, 0, sizeof a.hm.M);
  a.sw = uw; a.sh = uh; a.dw = bw; a.dh = bh;
  const size_t N = (size_t)bw * bh;
  std::vector<short> m1(2 * N);
  std::vector<unsigned short> m2(N);
  for (int y = 0; y < bh; ++y)
    for (int x = 0; x < bw; ++x) {   // k_warp_maps<1, LENS>
      const size_t q = (size_t)y * bw + x;
      if (cam.lens) warp_maps_pixel<1, 1>(a, x, y, m1[2 * q], m1[2 * q + 1], m2[q]);
      else warp_maps_pixel<1, 0>(a, x, y, m1[2 * q], m1[2 * q + 1], m2[q]);
    }
  return write_planes(path, m1.data(), m2.data(), N);
}

int main(int argc, char** argv) {
  if (argc == 9 && !strcmp(argv[1], "maps"))
    return mode_maps(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]), atoi(argv[7]), argv[8]);
  if (argc == 9 && !strcmp(argv[1], "bevmaps"))
    return mode_bevmaps(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]), atoi(argv[7]), argv[8]);
  if (argc == 8 && !strcmp(argv[1], "rays"))
    return mode_rays(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]), argv[7]);
  fprintf(stderr, "usage: lens_models maps|bevmaps|rays ...\n");
  return 1;
}
