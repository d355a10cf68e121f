// Host form of the gathers under cv2's border modes: the per-thread bodies of k_gather_border, k_gather_taps_border and
// k_gather4_border -- gather_frames_border (NEAREST, LINEAR), gather_taps_frames<..., BD = true> (CUBIC, LANCZOS4) and
// gather4_frames<..., BD = true> (the 3-channel LINEAR word path) -- from the library's own headers, with the border
// built by make_border as bevk_api.cu builds it, driven over the device's grid in every MODE (0 CV_16SC2 maps, 1 camera model, 2 homography, 3 affine matrix, 4 float maps, 5 camera model through float maps).
//
//   remap_border run <in.bin> <out.bin>
//     in : records of int32 mode, channels, interp (cv2.INTER_*: 0, 1, 2, 4), depth (0 8U, 2 16U, 3 16S, 5 32F), sw, sh,
//          dw, dh, n, arg (mode 0: map2 present; 3: WARP_INVERSE_MAP; 4: m1type), border mode, words (1: gather4_frames),
//          float64 border value[4], int64 spitch, sistride (bytes); the mode's payload as tests/host/remap_depth.cu reads
//          it; the source bytes ((n-1)*sistride + (sh-1)*spitch + sw*channels*esize); then the n dense destination
//          images as they are before the call (BORDER_TRANSPARENT leaves some pixels alone)
//     out: per record the n dense destination images; modes 1 and 5 follow them with the model's maps, as remap_depth
//   remap_border index <in.bin> <out.bin>
//     in : int32 count, then count pairs of int32 (n, mode); out: per pair border_index(p, n, mode) as int32 for every p
//          in [-32776, 32775] (the int16 map range widened by the Lanczos4 window)
// Built by tests/test_host_remap_border.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_gather4.cuh"

using namespace bevk;

template <int MODE, int C, class T>
static void grid(const GatherArgs& a, int interp, const void* w) {
  for (int f0 = 0; f0 < a.n; f0 += GATHER_NB)
    for (int y = 0; y < a.dh; ++y)
      for (int x = 0; x < a.dw; ++x) {
        if (interp == 0) gather_frames_border<MODE, C, 0, 0, T>(a, x, y, f0);
        else if (interp == 1) gather_frames_border<MODE, C, 1, 0, T>(a, x, y, f0);
        else if (interp == 2) gather_taps_frames<MODE, C, 4, 0, T, true>(a, static_cast<const TapWeights<T>*>(w), x, y, f0);
        else gather_taps_frames<MODE, C, 8, 0, T, true>(a, static_cast<const TapWeights<T>*>(w), x, y, f0);
      }
}

template <int MODE, class T>
static void run_ch(const GatherArgs& a, int ch, int interp, const void* w) {
  if (ch == 1) grid<MODE, 1, T>(a, interp, w);
  else if (ch == 3) grid<MODE, 3, T>(a, interp, w);
  else grid<MODE, 4, T>(a, interp, w);
}

template <int MODE>
static void run_mode(const GatherArgs& a, int depth, int ch, int interp, bool words, const short* tabs, const float* rows) {
  if (words) {   // the frame groups and single-frame form k_gather4 launches
    for (int f0 = 0; f0 < a.n; f0 += GATHER_NB)
      for (int y = 0; y < a.dh; ++y)
        for (int x4 = 0; x4 < a.dw; x4 += 4) {
          if (a.n == 1) gather4_frames<MODE, 1, Ldg, 0, true>(a, x4, y, f0);
          else gather4_frames<MODE, GATHER_NB, Ldg, 0, true>(a, x4, y, f0);
        }
    return;
  }
  const bool lanczos = interp == 4;
  if (depth == 0) run_ch<MODE, uint8_t>(a, ch, interp, tabs + (lanczos ? INTERP_TAB_LANCZOS4 : 0));
  else if (depth == 2) run_ch<MODE, uint16_t>(a, ch, interp, rows + (lanczos ? INTERP_ROWS_LANCZOS4 : 0));
  else if (depth == 3) run_ch<MODE, int16_t>(a, ch, interp, rows + (lanczos ? INTERP_ROWS_LANCZOS4 : 0));
  else run_ch<MODE, float>(a, ch, interp, rows + (lanczos ? INTERP_ROWS_LANCZOS4 : 0));
}

static int index_table(FILE* fi, FILE* fo) {
  int32_t count;
  if (fread(&count, 4, 1, fi) != 1) return 5;
  std::vector<int32_t> out;
  for (int i = 0; i < count; ++i) {
    int32_t nm[2];
    if (fread(nm, 4, 2, fi) != 2) return 5;
    out.clear();
    for (int p = -32776; p <= 32775; ++p) out.push_back(border_index(p, nm[0], nm[1]));
    fwrite(out.data(), 4, out.size(), fo);
  }
  return 0;
}

int main(int argc, char** argv) {
  if (argc != 4 || (strcmp(argv[1], "run") && strcmp(argv[1], "index"))) {
    fprintf(stderr, "usage: remap_border run|index <in.bin> <out.bin>\n");
    return 2;
  }
  FILE* fi = fopen(argv[2], "rb");
  FILE* fo = fopen(argv[3], "wb");
  if (!fi || !fo) return 4;
  if (!strcmp(argv[1], "index")) {
    const int r = index_table(fi, fo);
    fclose(fi);
    fclose(fo);
    return r;
  }
  std::vector<short> tabs(INTERP_TAB_SHORTS);
  build_interp_tabs(tabs.data());
  std::vector<float> rows(INTERP_ROWS_FLOATS);
  build_interp_rows(rows.data());
  int32_t h[12];
  long long records = 0;
  while (fread(h, 4, 12, fi) == 12) {
    const int mode = h[0], ch = h[1], interp = h[2], depth = h[3], sw = h[4], sh = h[5], dw = h[6], dh = h[7], n = h[8],
              arg = h[9], border = h[10], words = h[11];
    const int es = depth == 5 ? 4 : depth == 0 ? 1 : 2, px = ch * es;
    double bv[4];
    int64_t st[2];
    if (fread(bv, 8, 4, fi) != 4 || fread(st, 8, 2, fi) != 2) return 5;
    GatherArgs a{};
    a.bd = make_border(border, depth, bv);
    a.sw = sw; a.sh = sh; a.spitch = st[0]; a.sistride = st[1]; a.n = n;
    a.dw = dw; a.dh = dh; a.dpitch = (long long)dw * px; a.distride = (long long)dh * dw * px;
    const size_t npx = (size_t)dw * dh;
    std::vector<short2> m1(npx);
    std::vector<unsigned short> m2(npx);
    std::vector<float> f1(2 * npx + 4), f2(npx + 4);   // + 4: gather4_frames' float4 loads of the last pixels
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
    if (fread(src.data(), 1, sbytes, fi) != sbytes || fread(dst.data(), 1, dst.size(), fi) != dst.size()) return 5;
    a.src = src.data(); a.dst = dst.data();
    switch (mode) {
      case 0: run_mode<0>(a, depth, ch, interp, words, tabs.data(), rows.data()); break;
      case 1: run_mode<1>(a, depth, ch, interp, words, tabs.data(), rows.data()); break;
      case 2: run_mode<2>(a, depth, ch, interp, words, tabs.data(), rows.data()); break;
      case 3: run_mode<3>(a, depth, ch, interp, words, tabs.data(), rows.data()); break;
      case 4: run_mode<4>(a, depth, ch, interp, words, tabs.data(), rows.data()); break;
      default: run_mode<5>(a, depth, ch, interp, words, tabs.data(), rows.data());
    }
    fwrite(dst.data(), 1, dst.size(), fo);
    if (mode == 1 || mode == 5) {   // the model's maps, for cv2.remap to follow
      for (int y = 0; y < dh; ++y)
        for (int x = 0; x < dw; ++x) {
          if (mode == 5) {
            undistort_map_f32_px<0>(a.cm, a.lx, x, y, f1.data(), f2.data());
            continue;
          }
          short mx, my;
          unsigned short fr;
          model_entry<0>(a.cm, a.lx, x, y, mx, my, fr);
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
