// CPU harness of the YUV plane descriptor (tests/test_host_yuv_planes.py): the host forms of k_yuv_spans' work item
// (yuv_group) and k_vsum_yuv's (yuv_vsum_2x2) reading frames through YuvFrame, from the library's own headers.  nvcc
// compiles it; only host code runs.
//
//   yuv_planes layout <fmt 1=NV12|2=I420> <FW> <FH>
//     The dense instance of the descriptor (yuv_dense_layout, yuv_dense_frame) against yuv_chroma_rows on every chroma row,
//     and yuv_dense_planes' frame addressing.  Prints "layout: checked=N fails=M".
//   yuv_planes run <fmt> <in.bin> <out.bin>
//     in : int64[5] = NC, FW, FH, balance, arena bytes; int64[NC][6] = plane offsets into the arena (Y, UV / U, V) and
//          pitches; int32[NC][FH][2] the spans to convert; the arena.
//     Writes the BGR copy stack uint8[NC][FH][FW][3] (0xA5 where nothing is converted) and prints the V sums, the
//     luminance offsets and a read audit: how many of the bytes the conversion and the V sum read lie outside the
//     frame's plane rectangles (rows of FW, FW or FW/2 bytes at each pitch).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_bev.cuh"
#include "../../cameracalibration_b200/csrc/bevk_kernels.cuh"
#include "../../cameracalibration_b200/csrc/bevk_plan.cuh"

using namespace bevk;

template <int FMT>
static int layout(int FW, int FH) {
  long long off[3], pitch[3], checked = 0, fails = 0;
  yuv_dense_layout<FMT>(FW, FH, off, pitch);
  static uint8_t dummy[1];
  const uint8_t* base = dummy;   // addresses only: nothing is read
  const YuvFrame fr = yuv_dense_frame<FMT>(base, FW, FH);
  const long long stride = (long long)FW * FH * 3 / 2 + 7;
  const YuvFrame fr3 = yuv_dense_planes<FMT>(base, stride, FW, FH).frame(3);
  for (int p = 0; p < 3; ++p) {
    ++checked;
    if (fr.plane[p] != base + off[p] || fr.pitch[p] != pitch[p] || fr3.plane[p] != base + 3 * stride + off[p] ||
        fr3.pitch[p] != pitch[p]) {
      printf("plane %d: offset %lld pitch %lld\n", p, (long long)(fr.plane[p] - base), fr.pitch[p]);
      ++fails;
    }
  }
  if (pitch[0] != FW || pitch[1] != (FMT == YUV_NV12 ? FW : FW / 2) || off[1] != (long long)FW * FH ||
      (FMT == YUV_I420 && (pitch[2] != FW / 2 || off[2] != (long long)FW * FH + (long long)FW * FH / 4))) {
    printf("dense layout differs from cv2's\n");
    ++fails;
  }
  for (int cy = 0; cy < FH / 2; ++cy) {
    long long uo, vo;
    yuv_chroma_rows<FMT>(FW, FH, FW, cy, uo, vo);
    const uint8_t *u, *v;
    yuv_chroma_ptrs<FMT>(fr, cy, u, v);
    ++checked;
    if (u - base != uo || v - base != vo) {
      if (fails < 20) printf("chroma row %d: planes (%lld, %lld), yuv_chroma_rows (%lld, %lld)\n", cy, (long long)(u - base),
                             (long long)(v - base), uo, vo);
      ++fails;
    }
  }
  for (int y = 0; y < FH; ++y) {   // Y rows: FW bytes apart from the buffer's start
    ++checked;
    if (fr.plane[0] + (long long)y * fr.pitch[0] != base + (long long)y * FW) ++fails;
  }
  printf("layout: checked=%lld fails=%lld\n", checked, fails);
  return fails ? 1 : 0;
}

template <int FMT>
static int run(const char* in_path, const char* out_path) {
  FILE* fi = fopen(in_path, "rb");
  if (!fi) return 2;
  long long hd[5];
  if (fread(hd, 8, 5, fi) != 5) return 2;
  const int NC = (int)hd[0], FW = (int)hd[1], FH = (int)hd[2], bal = (int)hd[3];
  const size_t arena_bytes = (size_t)hd[4];
  std::vector<long long> geo((size_t)NC * 6);
  std::vector<int2> spans((size_t)NC * FH);
  std::vector<uint8_t> arena(arena_bytes);
  if (fread(geo.data(), 8, geo.size(), fi) != geo.size() || fread(spans.data(), sizeof(int2), spans.size(), fi) != spans.size() ||
      fread(arena.data(), 1, arena.size(), fi) != arena.size())
    return 2;
  fclose(fi);
  const int np = FMT == YUV_NV12 ? 2 : 3;
  const long long rows[3] = {FH, FH / 2, FH / 2}, row_bytes[3] = {FW, FMT == YUV_NV12 ? FW : FW / 2, FW / 2};
  std::vector<YuvFrame> frames(NC);
  for (int k = 0; k < NC; ++k) {
    for (int p = 0; p < 3; ++p) {
      const int q = p < np ? p : 1;
      frames[k].plane[p] = arena.data() + geo[6 * k + q];
      frames[k].pitch[p] = geo[6 * k + 3 + q];
    }
  }

  // ---- read audit: every byte the work items and the V sum read lies inside one of the frame's plane rectangles
  long long checked = 0, fails = 0;
  auto check = [&](int k, const uint8_t* a, const char* what) {
    ++checked;
    const long long d0 = a - arena.data();
    bool ok = false;
    for (int p = 0; p < np && !ok; ++p) {
      const long long d = d0 - geo[6 * k + p], pitch = geo[6 * k + 3 + p];
      ok = d >= 0 && d / pitch < rows[p] && d % pitch < row_bytes[p];
    }
    if (!ok && fails < 20) printf("%s of frame %d reads arena byte %lld outside its planes\n", what, k, d0);
    fails += !ok;
  };
  for (int k = 0; k < NC; ++k) {
    const YuvFrame& fr = frames[k];
    for (int y = 0; y < FH; ++y) {
      int g0, g1;
      span_groups(spans[(size_t)k * FH + y], g0, g1);
      const uint8_t *u, *v;
      yuv_chroma_ptrs<FMT>(fr, y >> 1, u, v);
      for (int g = g0; g < g1; ++g) {
        const int x0 = 4 * g, n = std::min(4, FW - x0);
        for (int j = 0; j < n; ++j) check(k, fr.plane[0] + (long long)y * fr.pitch[0] + x0 + j, "yuv_group Y");
        for (int j = 0; j < n / 2; ++j) {
          check(k, u + yuv_chroma_step<FMT>() * ((x0 >> 1) + j), "yuv_group U");
          check(k, v + yuv_chroma_step<FMT>() * ((x0 >> 1) + j), "yuv_group V");
        }
      }
    }
    for (int cy = 0; cy < FH / 2; ++cy) {
      const uint8_t *u, *v;
      yuv_chroma_ptrs<FMT>(fr, cy, u, v);
      for (int cx = 0; cx < FW / 2; ++cx) {
        const uint8_t* y = fr.plane[0] + (long long)(2 * cy) * fr.pitch[0] + 2 * cx;
        const uint8_t* r[6] = {y, y + 1, y + fr.pitch[0], y + fr.pitch[0] + 1, u + yuv_chroma_step<FMT>() * cx,
                               v + yuv_chroma_step<FMT>() * cx};
        for (const uint8_t* a : r) check(k, a, "yuv_vsum_2x2");
      }
    }
  }

  // ---- BALANCE part 1: k_vsum_yuv's sums over whole frames, k_delta's offsets
  std::vector<unsigned long long> vsum(NC, 0);
  for (int k = 0; k < NC; ++k)
    for (int cy = 0; cy < FH / 2; ++cy)
      for (int cx = 0; cx < FW / 2; ++cx) vsum[k] += yuv_vsum_2x2<FMT>(frames[k], cx, cy);
  std::vector<int> delta(NC, 0);
  if (bal) lum_deltas(vsum.data(), NC, (double)FW * (double)FH, delta.data());
  printf("vsum:");
  for (int k = 0; k < NC; ++k) printf(" %llu", vsum[k]);
  printf("\ndelta:");
  for (int k = 0; k < NC; ++k) printf(" %d", delta[k]);
  printf("\n");

  // ---- k_yuv_spans: every work item (group) of every row's span
  std::vector<int> tab(512, 0);   // ensure_hsv's tables
  for (int i = 1; i < 256; ++i) {
    tab[i] = (int)std::nearbyint((255 << 12) / (1. * i));
    tab[256 + i] = (int)std::nearbyint((180 << 12) / (6. * i));
  }
  std::vector<uint8_t> out((size_t)NC * FW * FH * 3, 0xA5);
  for (int k = 0; k < NC; ++k)
    for (int y = 0; y < FH; ++y) {
      int g0, g1;
      span_groups(spans[(size_t)k * FH + y], g0, g1);
      for (int g = g0; g < g1; ++g) {
        int c[12];
        const int n = bal ? yuv_group<FMT, true>(frames[k], FW, y, g, delta[k], tab.data(), c)
                          : yuv_group<FMT, false>(frames[k], FW, y, g, 0, tab.data(), c);
        uint8_t* o = out.data() + ((size_t)k * FH + y) * FW * 3 + 12 * (size_t)g;
        for (int j = 0; j < 3 * n; ++j) o[j] = (uint8_t)c[j];
      }
    }
  FILE* fo = fopen(out_path, "wb");
  if (!fo || fwrite(out.data(), 1, out.size(), fo) != out.size()) return 3;
  fclose(fo);
  printf("audit: checked=%lld fails=%lld\n", checked, fails);
  return fails ? 1 : 0;
}

int main(int argc, char** argv) {
  if (argc == 5 && !strcmp(argv[1], "layout")) {
    const int fmt = atoi(argv[2]), FW = atoi(argv[3]), FH = atoi(argv[4]);
    if (fmt == YUV_NV12) return layout<YUV_NV12>(FW, FH);
    if (fmt == YUV_I420) return layout<YUV_I420>(FW, FH);
  }
  if (argc == 5 && !strcmp(argv[1], "run")) {
    const int fmt = atoi(argv[2]);
    if (fmt == YUV_NV12) return run<YUV_NV12>(argv[3], argv[4]);
    if (fmt == YUV_I420) return run<YUV_I420>(argv[3], argv[4]);
  }
  fprintf(stderr, "usage: yuv_planes layout <1|2> <FW> <FH> | yuv_planes run <1|2> <in.bin> <out.bin>\n");
  return 2;
}
