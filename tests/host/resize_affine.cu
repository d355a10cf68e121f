// Host form of k_resize and of the warpAffine gathers (MODE 3 of gather_frames / gather_taps_frames / gather4_frames):
// the per-thread bodies from the library's own headers, driven over the device's grid -- x (x4 for the word path), y and
// the grid-z frame groups.
//
//   resize_affine run <in.bin> <out.bin>
//     in : records of int32 op (0 resize, 1 warpAffine), channels, sw, sh, dw, dh, n, interp, then int64 spitch,
//          sistride; op 0: float64 fx, fy (0, 0: the dsize form; then dw, dh are 0 and taken from fx, fy as cv2 does);
//          op 1: float64 M[6], int32 flags (interp | 16 = WARP_INVERSE_MAP), int32 word (1: the 4-pixel word path);
//          then the source bytes ((n-1)*sistride + (sh-1)*spitch + sw*channels)
//     out: per record int32 dw, dh, kind (resize_kind; -1 for warpAffine), then n dense images (dh * dw * channels each)
// Built by tests/test_host_resize_affine.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_gather4.cuh"
#include "../../cameracalibration_b200/csrc/bevk_resize.cuh"

using namespace bevk;

template <int C, int KIND>
static void resize_grid(const ResizeArgs& a) {
  for (int f0 = 0; f0 < a.n; f0 += GATHER_NB)
    for (int y = 0; y < a.dh; ++y)
      for (int x = 0; x < a.dw; ++x) resize_frames<C, KIND, GATHER_NB>(a, x, y, f0);
}
template <int C>
static void resize_c(const ResizeArgs& a, int kind) {
  switch (kind) {
    case RZ_NEAREST: resize_grid<C, RZ_NEAREST>(a); break;
    case RZ_LINEAR: resize_grid<C, RZ_LINEAR>(a); break;
    case RZ_AREA_LINEAR: resize_grid<C, RZ_AREA_LINEAR>(a); break;
    case RZ_AREA_FAST: resize_grid<C, RZ_AREA_FAST>(a); break;
    default: resize_grid<C, RZ_AREA>(a);
  }
}

template <int C, int LINEAR>
static void affine_grid(const GatherArgs& a) {
  for (int f0 = 0; f0 < a.n; f0 += GATHER_NB)
    for (int y = 0; y < a.dh; ++y)
      for (int x = 0; x < a.dw; ++x) gather_frames<3, C, LINEAR>(a, x, y, f0);
}
template <int C, int KS>
static void affine_taps(const GatherArgs& a, const short* tab) {
  for (int f0 = 0; f0 < a.n; f0 += GATHER_NB)
    for (int y = 0; y < a.dh; ++y)
      for (int x = 0; x < a.dw; ++x) gather_taps_frames<3, C, KS>(a, tab, x, y, f0);
}

int main(int argc, char** argv) {
  if (argc != 4 || strcmp(argv[1], "run")) {
    fprintf(stderr, "usage: resize_affine run <in.bin> <out.bin>\n");
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
    const int op = h[0], ch = h[1], sw = h[2], sh = h[3], n = h[6], interp = h[7];
    int dw = h[4], dh = h[5];
    int64_t st[2];
    if (fread(st, 8, 2, fi) != 2) return 5;
    double M[6] = {0, 0, 0, 0, 0, 0};
    int32_t fl[2] = {0, 0};
    ResizeArgs r{};
    int kind = -1;
    if (op == 0) {
      if (fread(&r.inv_x, 8, 1, fi) != 1 || fread(&r.inv_y, 8, 1, fi) != 1) return 5;
      if (!resize_geometry(sw, sh, &dw, &dh, &r.inv_x, &r.inv_y)) return 3;
      kind = resize_kind(interp, r);
    } else if (fread(M, 8, 6, fi) != 6 || fread(fl, 4, 2, fi) != 2) {
      return 5;
    }
    const size_t sbytes = (size_t)((n - 1) * st[1] + (sh - 1) * st[0] + (int64_t)sw * ch);
    std::vector<uint8_t> src(sbytes, 0);
    if (fread(src.data(), 1, sbytes, fi) != sbytes) return 5;
    std::vector<uint8_t> dst((size_t)n * dw * dh * ch, 0);
    if (op == 0) {
      r.src = src.data(); r.sw = sw; r.sh = sh; r.spitch = st[0]; r.sistride = st[1]; r.n = n;
      r.dst = dst.data(); r.dw = dw; r.dh = dh; r.dpitch = (long long)dw * ch; r.distride = (long long)dh * dw * ch;
      if (ch == 1) resize_c<1>(r, kind); else if (ch == 3) resize_c<3>(r, kind); else resize_c<4>(r, kind);
    } else {
      GatherArgs a{};
      a.src = src.data(); a.sw = sw; a.sh = sh; a.spitch = st[0]; a.sistride = st[1]; a.n = n;
      a.dst = dst.data(); a.dw = dw; a.dh = dh; a.dpitch = (long long)dw * ch; a.distride = (long long)dh * dw * ch;
      if (fl[0] & 16) memcpy(a.hm.M, M, sizeof M);
      else inv_affine(M, a.hm.M);
      int in = fl[0] & 15;
      if (in == 3) in = 1;   // INTER_AREA reads as INTER_LINEAR
      if (fl[1]) {           // the word path: 3 channels, LINEAR, dw % 4 == 0
        if (ch != 3 || in != 1 || dw % 4) return 6;
        for (int f0 = 0; f0 < n; f0 += GATHER_NB)
          for (int y = 0; y < dh; ++y)
            for (int x4 = 0; x4 < dw; x4 += 4) gather4_frames<3, GATHER_NB>(a, x4, y, f0);
      } else if (in == 2 || in == 4) {
        const short* t = tabs.data() + (in == 2 ? 0 : INTERP_TAB_LANCZOS4);
        if (in == 2) { if (ch == 1) affine_taps<1, 4>(a, t); else if (ch == 3) affine_taps<3, 4>(a, t); else affine_taps<4, 4>(a, t); }
        else { if (ch == 1) affine_taps<1, 8>(a, t); else if (ch == 3) affine_taps<3, 8>(a, t); else affine_taps<4, 8>(a, t); }
      } else if (in == 1) {
        if (ch == 1) affine_grid<1, 1>(a); else if (ch == 3) affine_grid<3, 1>(a); else affine_grid<4, 1>(a);
      } else {
        if (ch == 1) affine_grid<1, 0>(a); else if (ch == 3) affine_grid<3, 0>(a); else affine_grid<4, 0>(a);
      }
    }
    const int32_t hdr[3] = {dw, dh, kind};
    fwrite(hdr, 4, 3, fo);
    fwrite(dst.data(), 1, dst.size(), fo);
    ++records;
  }
  fclose(fi);
  fclose(fo);
  printf("run: records=%lld\n", records);
  return 0;
}
