// Host form of k_gather_taps (INTER_CUBIC / INTER_LANCZOS4): the per-thread body gather_taps_frames and the weight
// tables of build_interp_tabs, from the library's own headers, driven over the device's grid -- x, y and the grid-z frame
// groups of GATHER_NB -- in all three modes: maps (0), the camera model evaluated per pixel (1), a homography (2).
//
//   remap_interp run <in.bin> <out.bin>
//     in : records of int32 mode, channels, ks (4 cubic, 8 Lanczos4), sw, sh, dw, dh, n, then int64 spitch, sistride;
//          mode 0: map1 (int16[dh][dw][2]), map2 (uint16[dh][dw]); mode 1: float64 K[9], D[5], P[9], model;
//          mode 2: float64 H[9] (cv2.warpPerspective's matrix; inverted here as bevk_warp_perspective inverts it);
//          then the source bytes ((n-1)*sistride + (sh-1)*spitch + sw*channels)
//     out: per record the n dense destination images (dh * dw * channels each); mode 1 follows them with the maps the
//          model gives (map1 int16[dh][dw][2], map2 uint16[dh][dw], as k_undistort_map writes them)
// Built by tests/test_host_remap_interp.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_kernels.cuh"

using namespace bevk;

template <int MODE, int C, int KS>
static void grid(const GatherArgs& a, const short* tab) {
  for (int f0 = 0; f0 < a.n; f0 += GATHER_NB)
    for (int y = 0; y < a.dh; ++y)
      for (int x = 0; x < a.dw; ++x) gather_taps_frames<MODE, C, KS>(a, tab, x, y, f0);
}

template <int MODE>
static void run_mode(const GatherArgs& a, int ch, int ks, const short* tabs) {
  const short* t4 = tabs;
  const short* t8 = tabs + INTERP_TAB_LANCZOS4;
  if (ks == 4) {
    if (ch == 1) grid<MODE, 1, 4>(a, t4); else if (ch == 3) grid<MODE, 3, 4>(a, t4); else grid<MODE, 4, 4>(a, t4);
  } else {
    if (ch == 1) grid<MODE, 1, 8>(a, t8); else if (ch == 3) grid<MODE, 3, 8>(a, t8); else grid<MODE, 4, 8>(a, t8);
  }
}

int main(int argc, char** argv) {
  if (argc != 4 || strcmp(argv[1], "run")) {
    fprintf(stderr, "usage: remap_interp run <in.bin> <out.bin>\n");
    return 2;
  }
  std::vector<short> tabs(INTERP_TAB_SHORTS);
  build_interp_tabs(tabs.data());
  FILE* fi = fopen(argv[2], "rb");
  FILE* fo = fopen(argv[3], "wb");
  if (!fi || !fo) return 4;
  int32_t h[8];
  long long records = 0;
  while (fread(h, 4, 8, fi) == 8) {
    const int mode = h[0], ch = h[1], ks = h[2], sw = h[3], sh = h[4], dw = h[5], dh = h[6], n = h[7];
    int64_t st[2];
    if (fread(st, 8, 2, fi) != 2) return 5;
    GatherArgs a{};
    a.sw = sw; a.sh = sh; a.spitch = st[0]; a.sistride = st[1]; a.n = n;
    a.dw = dw; a.dh = dh; a.dpitch = (long long)dw * ch; a.distride = (long long)dh * dw * ch;
    const size_t npx = (size_t)dw * dh;
    std::vector<short2> m1(npx);
    std::vector<unsigned short> m2(npx);
    std::vector<double> xs;
    if (mode == 0) {
      if (fread(m1.data(), 4, npx, fi) != npx || fread(m2.data(), 2, npx, fi) != npx) return 5;
      a.map1 = m1.data(); a.map2 = m2.data();
    } else if (mode == 1) {
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
    } else {
      double H[9];
      if (fread(H, 8, 9, fi) != 9) return 5;
      if (!inv3(H, a.hm.M)) memset(a.hm.M, 0, sizeof a.hm.M);   // make_homog
    }
    const size_t sbytes = (size_t)((n - 1) * st[1] + (sh - 1) * st[0] + (int64_t)sw * ch);
    std::vector<uint8_t> src(sbytes + 64, 0);
    std::vector<uint8_t> dst((size_t)n * npx * ch, 0);
    if (fread(src.data(), 1, sbytes, fi) != sbytes) return 5;
    a.src = src.data(); a.dst = dst.data();
    if (mode == 0) run_mode<0>(a, ch, ks, tabs.data());
    else if (mode == 1) run_mode<1>(a, ch, ks, tabs.data());
    else run_mode<2>(a, ch, ks, tabs.data());
    fwrite(dst.data(), 1, dst.size(), fo);
    if (mode == 1) {   // the model's maps, k_undistort_map's arithmetic
      for (int y = 0; y < dh; ++y)
        for (int x = 0; x < dw; ++x) {
          double u, v;
          short mx, my;
          unsigned short fr;
          undistort_point(a.cm, x, y, u, v);
          quantise_uv(u, v, mx, my, fr, pack_saturates(a.cm.model, x, dw));
          m1[(size_t)y * dw + x] = make_short2(mx, my);
          m2[(size_t)y * dw + x] = fr;
        }
      fwrite(m1.data(), 4, npx, fo);
      fwrite(m2.data(), 2, npx, fo);
    }
    ++records;
  }
  fclose(fi);
  fclose(fo);
  printf("run: records=%lld\n", records);
  return 0;
}
