// Host form of the 16U, 16S and 32F gathers: the per-thread bodies gather_frames<..., T> (NEAREST, LINEAR) and
// gather_taps_frames<..., T> (CUBIC, LANCZOS4, with the float rows of build_interp_rows), from the library's own headers,
// driven over the device's grid -- x, y and the grid-z frame groups of GATHER_NB -- in every MODE: CV_16SC2 maps (0),
// the camera model (1), a homography (2), an affine matrix (3), float maps (4), the camera model through float maps (5).
//
//   remap_depth run <in.bin> <out.bin>
//     in : records of int32 mode, channels, interp (cv2.INTER_*: 0, 1, 2, 4), depth (2 16U, 3 16S, 5 32F), sw, sh, dw,
//          dh, n, arg (mode 0: map2 present; 3: WARP_INVERSE_MAP; 4: m1type), then int64 spitch, sistride (bytes);
//          mode 0: map1 int16[dh][dw][2], then map2 uint16[dh][dw] if present; modes 1, 5: float64 K[9], D[5], P[9],
//          model; mode 2: float64 H[9] (inverted here as bevk_warp_perspective inverts it); mode 3: float64 M[6]
//          (inverted unless WARP_INVERSE_MAP, as bevk_warp_affine does); mode 4: float map1 ([dh][dw][2] for CV_32FC2,
//          else [dh][dw] and map2 [dh][dw]); then the source bytes ((n-1)*sistride + (sh-1)*spitch + sw*channels*esize)
//     out: per record the n dense destination images; modes 1 and 5 follow them with the maps the model gives
//          (mode 1: map1 int16[dh][dw][2], map2 uint16[dh][dw] as k_undistort_map writes them; mode 5: float x and y
//          planes [dh][dw] as k_undistort_map_f32 writes them)
// Built by tests/test_host_remap_depth.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_kernels.cuh"

using namespace bevk;

template <int MODE, int C, class T>
static void grid(const GatherArgs& a, int interp, const float* rows) {
  for (int f0 = 0; f0 < a.n; f0 += GATHER_NB)
    for (int y = 0; y < a.dh; ++y)
      for (int x = 0; x < a.dw; ++x) {
        if (interp == 0) gather_frames<MODE, C, 0, 0, T>(a, x, y, f0);
        else if (interp == 1) gather_frames<MODE, C, 1, 0, T>(a, x, y, f0);
        else if (interp == 2) gather_taps_frames<MODE, C, 4, 0, T>(a, rows, x, y, f0);
        else gather_taps_frames<MODE, C, 8, 0, T>(a, rows + INTERP_ROWS_LANCZOS4, x, y, f0);
      }
}

template <int MODE, class T>
static void run_ch(const GatherArgs& a, int ch, int interp, const float* rows) {
  if (ch == 1) grid<MODE, 1, T>(a, interp, rows);
  else if (ch == 3) grid<MODE, 3, T>(a, interp, rows);
  else grid<MODE, 4, T>(a, interp, rows);
}

template <int MODE>
static void run_depth(const GatherArgs& a, int depth, int ch, int interp, const float* rows) {
  if (depth == 2) run_ch<MODE, uint16_t>(a, ch, interp, rows);
  else if (depth == 3) run_ch<MODE, int16_t>(a, ch, interp, rows);
  else run_ch<MODE, float>(a, ch, interp, rows);
}

int main(int argc, char** argv) {
  if (argc != 4 || strcmp(argv[1], "run")) {
    fprintf(stderr, "usage: remap_depth run <in.bin> <out.bin>\n");
    return 2;
  }
  std::vector<float> rows(INTERP_ROWS_FLOATS);
  build_interp_rows(rows.data());
  FILE* fi = fopen(argv[2], "rb");
  FILE* fo = fopen(argv[3], "wb");
  if (!fi || !fo) return 4;
  int32_t h[10];
  long long records = 0;
  while (fread(h, 4, 10, fi) == 10) {
    const int mode = h[0], ch = h[1], interp = h[2], depth = h[3], sw = h[4], sh = h[5], dw = h[6], dh = h[7], n = h[8],
              arg = h[9];
    const int es = depth == 5 ? 4 : 2, px = ch * es;
    int64_t st[2];
    if (fread(st, 8, 2, fi) != 2) return 5;
    GatherArgs a{};
    a.sw = sw; a.sh = sh; a.spitch = st[0]; a.sistride = st[1]; a.n = n;
    a.dw = dw; a.dh = dh; a.dpitch = (long long)dw * px; a.distride = (long long)dh * dw * px;
    const size_t npx = (size_t)dw * dh;
    std::vector<short2> m1(npx);
    std::vector<unsigned short> m2(npx);
    std::vector<float> f1(2 * npx), f2(npx);
    std::vector<double> xs;
    if (mode == 0) {
      if (fread(m1.data(), 4, npx, fi) != npx || (arg && fread(m2.data(), 2, npx, fi) != npx)) return 5;
      a.map1 = m1.data(); a.map2 = arg ? m2.data() : nullptr;
    } else if (mode == 1 || mode == 5) {
      double K[9], D[5], P[9], model;
      if (fread(K, 8, 9, fi) != 9 || fread(D, 8, 5, fi) != 5 || fread(P, 8, 9, fi) != 9 || fread(&model, 8, 1, fi) != 1) return 5;
      memset(&a.cm, 0, sizeof a.cm);
      if (!inv3(P, a.cm.iR)) return 3;
      for (int i = 0; i < 5; ++i) a.cm.k[i] = D[i];
      a.cm.fx = K[0]; a.cm.fy = K[4]; a.cm.cx = K[2]; a.cm.cy = K[5];
      a.cm.model = (int)model; a.cm.w = dw; a.cm.h = dh;
      if (xs_table_applies(a.cm)) {   // as bevk_api.cu attaches it (attach_xs_table)
        xs.resize(dw);
        fill_xs_table(a.cm, xs.data());
        a.cm.xs = xs.data();
      }
    } else if (mode == 2) {
      double H[9];
      if (fread(H, 8, 9, fi) != 9) return 5;
      if (!inv3(H, a.hm.M)) memset(a.hm.M, 0, sizeof a.hm.M);   // make_homog
    } else if (mode == 3) {
      double M[6];
      if (fread(M, 8, 6, fi) != 6) return 5;
      if (arg) memcpy(a.hm.M, M, sizeof M);
      else inv_affine(M, a.hm.M);
    } else {
      const bool c2 = arg == MAP_32FC2;
      if (fread(f1.data(), 4, c2 ? 2 * npx : npx, fi) != (c2 ? 2 * npx : npx) || (!c2 && fread(f2.data(), 4, npx, fi) != npx))
        return 5;
      a.fmap1 = f1.data(); a.fmap2 = c2 ? nullptr : f2.data();
    }
    const size_t sbytes = (size_t)((n - 1) * st[1] + (sh - 1) * st[0] + (int64_t)sw * px);
    std::vector<uint8_t> src(sbytes + 64, 0);
    std::vector<uint8_t> dst((size_t)n * npx * px, 0);
    if (fread(src.data(), 1, sbytes, fi) != sbytes) return 5;
    a.src = src.data(); a.dst = dst.data();
    switch (mode) {
      case 0: run_depth<0>(a, depth, ch, interp, rows.data()); break;
      case 1: run_depth<1>(a, depth, ch, interp, rows.data()); break;
      case 2: run_depth<2>(a, depth, ch, interp, rows.data()); break;
      case 3: run_depth<3>(a, depth, ch, interp, rows.data()); break;
      case 4: run_depth<4>(a, depth, ch, interp, rows.data()); break;
      default: run_depth<5>(a, depth, ch, interp, rows.data());
    }
    fwrite(dst.data(), 1, dst.size(), fo);
    if (mode == 1 || mode == 5) {   // the model's maps: k_undistort_map's and k_undistort_map_f32's arithmetic
      for (int y = 0; y < dh; ++y)
        for (int x = 0; x < dw; ++x) {
          if (mode == 5) {
            undistort_map_f32_px<0>(a.cm, a.lx, x, y, f1.data(), f2.data());
            continue;
          }
          double u, v;
          short mx, my;
          unsigned short fr;
          undistort_point(a.cm, x, y, u, v);
          quantise_uv(u, v, mx, my, fr, pack_saturates(a.cm.model, x, dw));
          m1[(size_t)y * dw + x] = make_short2(mx, my);
          m2[(size_t)y * dw + x] = fr;
        }
      if (mode == 1) {
        fwrite(m1.data(), 4, npx, fo);
        fwrite(m2.data(), 2, npx, fo);
      } else {
        fwrite(f1.data(), 4, npx, fo);
        fwrite(f2.data(), 4, npx, fo);
      }
    }
    ++records;
  }
  fclose(fi);
  fclose(fo);
  printf("run: records=%lld\n", records);
  return 0;
}
