// CPU harness of the packed YUV 4:2:2 source path (tests/test_host_yuv422.py): the host forms of k_yuv_spans' work item
// (yuv_group), of k_vsum_yuv's (yuv_vsum_pair) and of the ingest plan (yuv_windows, yuv_dma_rects) for YUYV and UYVY,
// from the library's own headers.  nvcc compiles it; only host code runs.
//
//   yuv422 plan <fmt 3=YUYV|4=UYVY> <in.bin> <out.bin>
//     in : int32[8] = NC, FW, FH, BW, BH, nearest, balance, has_maps; with has_maps per camera map1 int16[BH][BW][2],
//          map2 uint16[BH][BW], mask uint8[BH][BW]; then NC dense frames uint8[FH][FW][2].
//     The sampled spans come from the tile-plan compiler (every column of every row without maps).  Writes the BGR copy
//     stack the pre-pass leaves, uint8[NC][FH][FW][3] (0xA5 where nothing is converted), followed by the spans
//     int32[NC][FH][2], and prints the V sums, the luminance offsets, the ingest byte counts per frame-set (windows, DMA
//     rectangles; BGR's for comparison) and how many of the bytes the pre-pass reads lie outside the windows / rectangles
//     the ingest fetches.
//   yuv422 pitched <fmt> <in.bin> <out.bin>
//     in : int64[5] = NC, FW, FH, balance, arena bytes; int64[NC][2] = the plane's offset into the arena and its pitch;
//          int32[NC][FH][2] the spans to convert; the arena.
//     Writes the copy stack as above (without the spans) and prints the V sums, the luminance offsets and a read audit:
//     how many of the bytes the conversion and the V sum read lie outside the frame's plane rectangle (FH rows of 2 FW
//     bytes at the pitch).
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

static std::vector<int> hsv_tables() {   // ensure_hsv's tables
  std::vector<int> tab(512, 0);
  for (int i = 1; i < 256; ++i) {
    tab[i] = (int)std::nearbyint((255 << 12) / (1. * i));
    tab[256 + i] = (int)std::nearbyint((180 << 12) / (6. * i));
  }
  return tab;
}

// k_vsum_yuv's sums and k_delta's offsets over the frames, printed; then k_yuv_spans over every group of every span into
// a copy stack (0xA5 elsewhere).
template <int FMT>
static std::vector<uint8_t> convert(const std::vector<YuvFrame>& frames, const std::vector<int2>& spans, int FW, int FH, bool bal) {
  const int NC = (int)frames.size();
  std::vector<unsigned long long> vsum(NC, 0);
  for (int k = 0; k < NC; ++k)
    for (int y = 0; y < yuv_chroma_rows_of<FMT>(FH); ++y)
      for (int cx = 0; cx < FW / 2; ++cx) vsum[k] += yuv_vsum_sample<FMT>(frames[k], cx, y);
  std::vector<int> delta(NC, 0);
  if (bal) lum_deltas(vsum.data(), NC, (double)FW * (double)FH, delta.data());
  printf("vsum:");
  for (int k = 0; k < NC; ++k) printf(" %llu", vsum[k]);
  printf("\ndelta:");
  for (int k = 0; k < NC; ++k) printf(" %d", delta[k]);
  printf("\n");
  const std::vector<int> tab = hsv_tables();
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
  return out;
}

// Every byte offset (within its frame's plane, as row * pitch + column) that the pre-pass and the V sum read: the group's
// pixel pairs [2 x0, 2 x0 + 2n) of its row, and each pixel pair [4 cx, 4 cx + 4) of every row.
template <typename F>
static void reads(const int2* sp, int FW, int FH, bool vsum, F&& visit) {
  for (int y = 0; y < FH; ++y) {
    int g0, g1;
    span_groups(sp[y], g0, g1);
    for (int g = g0; g < g1; ++g) {
      const int x0 = 4 * g, n = std::min(4, FW - x0);
      for (int j = 0; j < 2 * n; ++j) visit(y, 2 * x0 + j);
    }
    if (vsum)
      for (int j = 0; j < 2 * FW; ++j) visit(y, j);
  }
}

template <int FMT>
static int plan(const char* in_path, const char* out_path) {
  FILE* fi = fopen(in_path, "rb");
  if (!fi) return 2;
  int hd[8];
  if (fread(hd, 4, 8, fi) != 8) return 2;
  const int NC = hd[0], FW = hd[1], FH = hd[2], BW = hd[3], BH = hd[4], nearest = hd[5], bal = hd[6], has_maps = hd[7];
  const size_t npx = (size_t)BW * BH, row = (size_t)FW * 2, fbytes = row * FH;
  std::vector<std::vector<short>> m1(NC);
  std::vector<std::vector<unsigned short>> m2(NC);
  std::vector<std::vector<uint8_t>> mk(NC);
  if (has_maps)
    for (int k = 0; k < NC; ++k) {
      m1[k].resize(npx * 2); m2[k].resize(npx); mk[k].resize(npx);
      if (fread(m1[k].data(), 4, npx, fi) != npx || fread(m2[k].data(), 2, npx, fi) != npx || fread(mk[k].data(), 1, npx, fi) != npx) return 2;
    }
  std::vector<uint8_t> data((size_t)NC * fbytes);
  if (fread(data.data(), 1, data.size(), fi) != data.size()) return 2;
  fclose(fi);

  std::vector<int2> spans((size_t)NC * FH, make_int2(0, FW));
  if (has_maps) {
    BevPlan bp;
    std::vector<const short*> p1(NC);
    std::vector<const unsigned short*> p2(NC);
    std::vector<const uint8_t*> pm(NC);
    for (int k = 0; k < NC; ++k) { p1[k] = m1[k].data(); p2[k] = m2[k].data(); pm[k] = mk[k].data(); }
    build_bev_plan(NC, FW, FH, BW, BH, nearest != 0, p1.data(), p2.data(), pm.data(), bp);
    spans = bp.spans;
  }
  std::vector<YuvFrame> frames(NC);
  for (int k = 0; k < NC; ++k) frames[k] = yuv_dense_frame<FMT>(data.data() + k * fbytes, FW, FH);
  const std::vector<uint8_t> out = convert<FMT>(frames, spans, FW, FH, bal != 0);
  FILE* fo = fopen(out_path, "wb");
  if (!fo || fwrite(out.data(), 1, out.size(), fo) != out.size() || fwrite(spans.data(), sizeof(int2), spans.size(), fo) != spans.size())
    return 3;
  fclose(fo);
  if (!has_maps) return 0;

  // ---- ingest plan: windows (page-locked) and DMA rectangles (pageable, 1..3 bands) against the pre-pass's reads
  long long fetch = 0, dma = 0, bgr_fetch = 0, bgr_dma = 0, checked = 0, fails = 0;
  for (int k = 0; k < NC; ++k) {
    const int2* sp = spans.data() + (size_t)k * FH;
    std::vector<int4> win(FH);
    yuv_windows(FMT, sp, FW, FH, win.data());
    fetch += yuv_window_bytes(win.data(), FH);
    for (int y = 0; y < FH; ++y) {   // bevk_bev_finalize's span_fetch_bytes
      if (sp[y].y > sp[y].x) bgr_fetch += std::min<int>(FW * 3, (3 * sp[y].y + 12 + 15) & ~15) - (std::max(0, 3 * sp[y].x - 12) & ~15);
      const int4 w = win[y];
      if (w.x < 0 || w.y > (int)row || w.x > w.y || w.z != 0 || w.w != 0 || (w.x & 15) || ((w.y & 15) && w.y != (int)row)) {
        printf("bad window cam %d row %d: %d %d %d %d\n", k, y, w.x, w.y, w.z, w.w);
        ++fails;
      }
    }
    std::vector<std::vector<uint8_t>> in_rect(3, std::vector<uint8_t>(fbytes, 0));
    for (int nb = 1; nb <= 3; ++nb) {
      int box[BEVK_MAX_BANDS][4];
      plan_bands(sp, FW, FH, nb, box);
      std::vector<int4> rects;
      yuv_dma_rects(FMT, box, nb, FW, FH, rects);
      for (const int4& r : rects) {
        if (r.x < 0 || r.x + r.y > FH || r.z < 0 || r.z + r.w > (int)row || r.y <= 0 || r.w <= 0 || (r.z & 3) || (r.w & 3)) {
          printf("bad rect cam %d: %d %d %d %d\n", k, r.x, r.y, r.z, r.w);
          ++fails;
          continue;
        }
        for (int yy = r.x; yy < r.x + r.y; ++yy) memset(in_rect[nb - 1].data() + (size_t)yy * row + r.z, 1, r.w);
        if (nb == 2) dma += (long long)r.y * r.w;
      }
      if (nb == 2)
        for (int b = 0; b < nb; ++b) bgr_dma += (long long)(box[b][1] - box[b][0]) * (box[b][3] - box[b][2]);
    }
    reads(sp, FW, FH, false, [&](int y, int col) {
      ++checked;
      const int4 w = win[y];
      bool ok = col >= w.x && col < w.y;
      for (int b = 0; b < 3; ++b) ok = ok && in_rect[b][(size_t)y * row + col];
      if (!ok && fails < 20) printf("read outside the ingest: cam %d byte (%d, %d)\n", k, y, col);
      fails += !ok;
    });
  }
  printf("bytes: fetch=%lld dma=%lld bgr_fetch=%lld bgr_dma=%lld\n", fetch, dma, bgr_fetch, bgr_dma);
  printf("coverage: checked=%lld fails=%lld\n", checked, fails);
  return fails ? 1 : 0;
}

template <int FMT>
static int pitched(const char* in_path, const char* out_path) {
  FILE* fi = fopen(in_path, "rb");
  if (!fi) return 2;
  long long hd[5];
  if (fread(hd, 8, 5, fi) != 5) return 2;
  const int NC = (int)hd[0], FW = (int)hd[1], FH = (int)hd[2], bal = (int)hd[3];
  std::vector<long long> geo((size_t)NC * 2);
  std::vector<int2> spans((size_t)NC * FH);
  std::vector<uint8_t> arena((size_t)hd[4]);
  if (fread(geo.data(), 8, geo.size(), fi) != geo.size() || fread(spans.data(), sizeof(int2), spans.size(), fi) != spans.size() ||
      fread(arena.data(), 1, arena.size(), fi) != arena.size())
    return 2;
  fclose(fi);
  std::vector<YuvFrame> frames(NC);
  for (int k = 0; k < NC; ++k)
    for (int p = 0; p < 3; ++p) {   // planes 1 and 2 are never read: bevk_bev_run_yuv_planes' rule
      frames[k].plane[p] = arena.data() + geo[2 * k];
      frames[k].pitch[p] = geo[2 * k + 1];
    }
  // ---- read audit: every byte read lies inside the frame's plane rectangle
  long long checked = 0, fails = 0;
  for (int k = 0; k < NC; ++k)
    reads(spans.data() + (size_t)k * FH, FW, FH, true, [&](int y, int col) {
      ++checked;
      const long long a = geo[2 * k] + (long long)y * geo[2 * k + 1] + col;
      const long long d = a - geo[2 * k], pitch = geo[2 * k + 1];
      const bool ok = a >= 0 && a < (long long)arena.size() && d >= 0 && d / pitch < FH && d % pitch < 2LL * FW;
      if (!ok && fails < 20) printf("frame %d reads arena byte %lld outside its plane\n", k, a);
      fails += !ok;
    });
  const std::vector<uint8_t> out = convert<FMT>(frames, spans, FW, FH, bal != 0);
  FILE* fo = fopen(out_path, "wb");
  if (!fo || fwrite(out.data(), 1, out.size(), fo) != out.size()) return 3;
  fclose(fo);
  printf("audit: checked=%lld fails=%lld\n", checked, fails);
  return fails ? 1 : 0;
}

int main(int argc, char** argv) {
  if (argc == 5) {
    const int fmt = atoi(argv[2]);
    if (!strcmp(argv[1], "plan") && fmt == YUV_YUYV) return plan<YUV_YUYV>(argv[3], argv[4]);
    if (!strcmp(argv[1], "plan") && fmt == YUV_UYVY) return plan<YUV_UYVY>(argv[3], argv[4]);
    if (!strcmp(argv[1], "pitched") && fmt == YUV_YUYV) return pitched<YUV_YUYV>(argv[3], argv[4]);
    if (!strcmp(argv[1], "pitched") && fmt == YUV_UYVY) return pitched<YUV_UYVY>(argv[3], argv[4]);
  }
  fprintf(stderr, "usage: yuv422 plan|pitched <3|4> <in.bin> <out.bin>\n");
  return 2;
}
