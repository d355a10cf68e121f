// Host build of the kernels' float-map code: the CV_32FC1 / CV_32FC2 map build (undistort_map_f32_px<LENS>, after the
// camera set-up bevk_api.cu does), cv2.convertMaps (convert_map_px) and the float-map gathers (MODE 4 of gather_frames,
// gather_taps_frames and gather4_frames).  Built and run by tests/test_host_float_maps.py with nvcc (host code only is
// executed), compared there with live cv2.
//   float_maps maps <model> <w> <h> <n_dist> <has_R> <m1type> <out.bin>
//       stdin: K[9] D[n_dist] R[9 if has_R] P[9] as C99 hex floats; out: float map1 then (CV_32FC1) map2
//   float_maps convert <intype> <has_map2> <outtype> <nn> <w> <h> <in.bin> <out.bin>
//       in: map1 then map2 (when present); out: map1 then map2 (when the conversion writes one)
//   float_maps remap <channels> <interp> <m1type> <sw> <sh> <dw> <dh> <words> <in.bin> <out.bin>
//       interp: cv2.INTER_* (INTER_AREA read as INTER_LINEAR).  in: float map1, map2 (CV_32FC1), then the dense source
//       image; out: the dense destination image.  words = 1 runs
//       k_gather4's body (3 channels, INTER_LINEAR, dw % 4 == 0).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_gather4.cuh"

using namespace bevk;

static bool read_doubles(double* v, int n) {
  for (int i = 0; i < n; ++i) {
    char tok[64];
    if (scanf("%63s", tok) != 1) return false;
    v[i] = strtod(tok, nullptr);
  }
  return true;
}

static int mode_maps(int model, int w, int h, int n, int has_r, int m1type, const char* path) {
  double K[9], D[16], R[9], P[9];
  if (n < 0 || n > 16 || !read_doubles(K, 9) || !read_doubles(D, n) || (has_r && !read_doubles(R, 9)) || !read_doubles(P, 9))
    return 2;
  CamModel cm;
  LensExt lx;
  bool lens = false;
  if (lens_model(model, K, D, n, has_r ? R : nullptr, P, w, h, &cm, &lx, &lens) != LENS_OK) return 3;
  const bool walks = rays_walk(cm, has_r ? R : nullptr);
  lens = lens || walks;
  std::vector<double> xs(w), rays;
  if (xs_table_applies(cm)) { fill_xs_table(cm, xs.data()); cm.xs = xs.data(); }
  if (walks) {
    rays.resize((size_t)ray_row_len(cm) * h * 3);
    for (int i = 0; i < h; ++i) walk_rays(cm, i, rays.data());
    lx.rays = rays.data();
  }
  const size_t N = (size_t)w * h;
  std::vector<float> m1(2 * N), m2(N);
  float* y = m1type == MAP_32FC1 ? m2.data() : nullptr;
  for (int i = 0; i < h; ++i)
    for (int j = 0; j < w; ++j) {   // k_undistort_map_f32<LENS>
      if (lens) undistort_map_f32_px<1>(cm, lx, j, i, m1.data(), y);
      else undistort_map_f32_px<0>(cm, lx, j, i, m1.data(), y);
    }
  FILE* f = fopen(path, "wb");
  if (!f) return 4;
  fwrite(m1.data(), 4, y ? N : 2 * N, f);
  if (y) fwrite(m2.data(), 4, N, f);
  fclose(f);
  return 0;
}

static size_t bytes1(int t) { return t == MAP_32FC2 ? 8 : 4; }
static size_t bytes2(int t) { return t == MAP_16SC2 ? 2 : 4; }

static int mode_convert(int intype, int has2, int outtype, int nn, int w, int h, const char* in, const char* out) {
  const size_t N = (size_t)w * h;
  std::vector<uint8_t> i1(N * 8), i2(N * 4), o1(N * 8), o2(N * 4);
  FILE* f = fopen(in, "rb");
  if (!f) return 4;
  if (fread(i1.data(), bytes1(intype), N, f) != N || (has2 && fread(i2.data(), bytes2(intype), N, f) != N)) return 5;
  fclose(f);
  const bool write2 = outtype != MAP_32FC2 && !(outtype == MAP_16SC2 && nn);
  ConvertMapsArgs a{i1.data(), has2 ? i2.data() : nullptr, intype, o1.data(), write2 ? o2.data() : nullptr, outtype,
                    nn != 0 && outtype == MAP_16SC2, (long long)N};
  for (long long i = 0; i < (long long)N; ++i) convert_map_px(a, i);
  f = fopen(out, "wb");
  if (!f) return 4;
  fwrite(o1.data(), bytes1(outtype), N, f);
  if (write2) fwrite(o2.data(), bytes2(outtype), N, f);
  fclose(f);
  return 0;
}

template <int C>
static void grid(const GatherArgs& a, int interp, const short* tabs, bool words) {
  for (int y = 0; y < a.dh; ++y) {
    if (words) {
      if (C == 3)
        for (int x = 0; x < a.dw; x += 4) gather4_frames<4, 1>(a, x, y, 0);
      continue;
    }
    for (int x = 0; x < a.dw; ++x) {
      if (interp == 0) gather_frames<4, C, 0>(a, x, y, 0);
      else if (interp == 1 || interp == 3) gather_frames<4, C, 1>(a, x, y, 0);
      else if (interp == 2) gather_taps_frames<4, C, 4>(a, tabs, x, y, 0);
      else gather_taps_frames<4, C, 8>(a, tabs + INTERP_TAB_LANCZOS4, x, y, 0);
    }
  }
}

static int mode_remap(int ch, int interp, int m1type, int sw, int sh, int dw, int dh, int words, const char* in, const char* out) {
  const size_t N = (size_t)dw * dh, S = (size_t)sw * sh * ch;
  std::vector<float> m1(2 * N + 8), m2(N + 8);
  std::vector<uint8_t> src(S + 16), dst(N * ch);
  FILE* f = fopen(in, "rb");
  if (!f) return 4;
  const size_t n1 = m1type == MAP_32FC2 ? 2 * N : N;
  if (fread(m1.data(), 4, n1, f) != n1 || (m1type == MAP_32FC1 && fread(m2.data(), 4, N, f) != N) ||
      fread(src.data(), 1, S, f) != S)
    return 5;
  fclose(f);
  std::vector<short> tabs(INTERP_TAB_SHORTS);
  build_interp_tabs(tabs.data());
  GatherArgs a{};
  a.src = src.data(); a.sw = sw; a.sh = sh; a.spitch = (long long)sw * ch;
  a.dst = dst.data(); a.dw = dw; a.dh = dh; a.dpitch = (long long)dw * ch;
  a.n = 1;
  a.fmap1 = m1.data(); a.fmap2 = m1type == MAP_32FC1 ? m2.data() : nullptr;
  if (ch == 1) grid<1>(a, interp, tabs.data(), false);
  else if (ch == 3) grid<3>(a, interp, tabs.data(), words != 0);
  else grid<4>(a, interp, tabs.data(), false);
  f = fopen(out, "wb");
  if (!f) return 4;
  fwrite(dst.data(), 1, dst.size(), f);
  fclose(f);
  return 0;
}

int main(int argc, char** argv) {
  if (argc == 9 && !strcmp(argv[1], "maps"))
    return mode_maps(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]), atoi(argv[7]), argv[8]);
  if (argc == 10 && !strcmp(argv[1], "convert"))
    return mode_convert(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]), atoi(argv[7]), argv[8],
                        argv[9]);
  if (argc == 12 && !strcmp(argv[1], "remap"))
    return mode_remap(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]), atoi(argv[7]), atoi(argv[8]),
                      atoi(argv[9]), argv[10], argv[11]);
  fprintf(stderr, "usage: float_maps maps|convert|remap ...\n");
  return 1;
}
