// CPU harness of the YUV 4:2:0 source path (tests/test_host_yuv.py): the host forms of k_yuv_spans' work item
// (yuv_group), of k_vsum_yuv's (yuv_vsum_2x2) and the ingest plan (yuv_windows, yuv_dma_rects) from the library's own
// headers.  nvcc compiles it; only host code runs.
//
//   yuv <fmt 1=NV12|2=I420> <in.bin> <out.bin>
//     in : int32[8] = NC, FW, FH, BW, BH, nearest, balance, has_maps; with has_maps per camera map1 int16[BH][BW][2],
//          map2 uint16[BH][BW], mask uint8[BH][BW]; then NC frames uint8[FH*3/2][FW].
//     The sampled spans come from the tile-plan compiler (every column of every row without maps).  Writes the BGR copy
//     stack the pre-pass leaves, uint8[NC][FH][FW][3] (0xA5 where nothing is converted), followed by the spans
//     int32[NC][FH][2], and prints the V sums, the
//     luminance offsets, the ingest byte counts per frame-set (windows, DMA rectangles; BGR's for comparison) and how
//     many of the bytes the pre-pass reads lie outside the windows / rectangles the ingest fetches.
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
static int run(const char* in_path, const char* out_path) {
  FILE* fi = fopen(in_path, "rb");
  if (!fi) return 2;
  int hd[8];
  if (fread(hd, 4, 8, fi) != 8) return 2;
  const int NC = hd[0], FW = hd[1], FH = hd[2], BW = hd[3], BH = hd[4], nearest = hd[5], bal = hd[6], has_maps = hd[7];
  const size_t npx = (size_t)BW * BH, fbytes = (size_t)FW * FH * 3 / 2, rows = (size_t)FH * 3 / 2;
  std::vector<std::vector<short>> m1(NC);
  std::vector<std::vector<unsigned short>> m2(NC);
  std::vector<std::vector<uint8_t>> mk(NC);
  if (has_maps)
    for (int k = 0; k < NC; ++k) {
      m1[k].resize(npx * 2); m2[k].resize(npx); mk[k].resize(npx);
      if (fread(m1[k].data(), 4, npx, fi) != npx || fread(m2[k].data(), 2, npx, fi) != npx || fread(mk[k].data(), 1, npx, fi) != npx) return 2;
    }
  std::vector<uint8_t> frames((size_t)NC * fbytes);
  if (fread(frames.data(), 1, frames.size(), fi) != frames.size()) return 2;
  fclose(fi);

  // ---- the sampled spans, as bevk_bev_finalize derives them
  std::vector<int2> spans((size_t)NC * FH, make_int2(0, FW));
  BevPlan plan;
  if (has_maps) {
    std::vector<const short*> p1(NC);
    std::vector<const unsigned short*> p2(NC);
    std::vector<const uint8_t*> pm(NC);
    for (int k = 0; k < NC; ++k) { p1[k] = m1[k].data(); p2[k] = m2[k].data(); pm[k] = mk[k].data(); }
    build_bev_plan(NC, FW, FH, BW, BH, nearest != 0, p1.data(), p2.data(), pm.data(), plan);
    spans = plan.spans;
  }

  // ---- BALANCE part 1: k_vsum_yuv's sums over whole frames, k_delta's offsets
  std::vector<unsigned long long> vsum(NC, 0);
  for (int k = 0; k < NC; ++k)
    for (int cy = 0; cy < FH / 2; ++cy)
      for (int cx = 0; cx < FW / 2; ++cx) vsum[k] += yuv_vsum_2x2<FMT>(frames.data() + k * fbytes, FW, FH, cx, cy);
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
        const int n = bal ? yuv_group<FMT, true>(frames.data() + k * fbytes, FW, FH, y, g, delta[k], tab.data(), c)
                          : yuv_group<FMT, false>(frames.data() + k * fbytes, FW, FH, y, g, 0, tab.data(), c);
        uint8_t* o = out.data() + ((size_t)k * FH + y) * FW * 3 + 12 * (size_t)g;
        for (int j = 0; j < 3 * n; ++j) o[j] = (uint8_t)c[j];
      }
    }
  FILE* fo = fopen(out_path, "wb");
  if (!fo || fwrite(out.data(), 1, out.size(), fo) != out.size() || fwrite(spans.data(), sizeof(int2), spans.size(), fo) != spans.size())
    return 3;
  fclose(fo);
  if (!has_maps) return 0;

  // ---- ingest plan: windows (page-locked) and DMA rectangles (pageable, 1..3 bands) against the pre-pass's reads
  long long fetch = 0, dma = 0, bgr_fetch = 0, bgr_dma = 0, checked = 0, fails = 0;
  for (int k = 0; k < NC; ++k) {
    const int2* sp = spans.data() + (size_t)k * FH;
    std::vector<int4> win(rows);
    yuv_windows(FMT, sp, FW, FH, win.data());
    fetch += yuv_window_bytes(win.data(), (int)rows);
    for (int y = 0; y < FH; ++y)   // bevk_bev_finalize's span_fetch_bytes
      if (sp[y].y > sp[y].x) bgr_fetch += std::min<int>(FW * 3, (3 * sp[y].y + 12 + 15) & ~15) - (std::max(0, 3 * sp[y].x - 12) & ~15);
    for (int y = 0; y < (int)rows; ++y) {
      const int4 w = win[y];
      if (w.x < 0 || w.y > FW || w.z < 0 || w.w > FW || (w.x & 15) || (w.z & 15) || ((w.y & 15) && w.y != FW) ||
          ((w.w & 15) && w.w != FW)) {
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
        if (r.x < 0 || r.x + r.y > (int)rows || r.z < 0 || r.z + r.w > FW || r.y <= 0 || r.w <= 0) {
          printf("bad rect cam %d: %d %d %d %d\n", k, r.x, r.y, r.z, r.w);
          ++fails;
          continue;
        }
        for (int yy = r.x; yy < r.x + r.y; ++yy) memset(in_rect[nb - 1].data() + (size_t)yy * FW + r.z, 1, r.w);
        if (nb == 2) dma += (long long)r.y * r.w;
      }
      if (nb == 2)
        for (int b = 0; b < nb; ++b) bgr_dma += (long long)(box[b][1] - box[b][0]) * (box[b][3] - box[b][2]);
    }
    auto check = [&](long long off, int y) {
      ++checked;
      const int r = (int)(off / FW), col = (int)(off % FW);
      const int4 w = win[r];
      bool ok = (col >= w.x && col < w.y) || (col >= w.z && col < w.w);
      for (int b = 0; b < 3; ++b) ok = ok && in_rect[b][off];
      if (!ok && fails < 20) printf("read outside the ingest: cam %d row %d byte (%d, %d)\n", k, y, r, col);
      fails += !ok;
    };
    for (int y = 0; y < FH; ++y) {   // the bytes yuv_group reads, group by group
      int g0, g1;
      span_groups(sp[y], g0, g1);
      long long uo, vo;
      yuv_chroma_rows<FMT>(FW, FH, FW, y >> 1, uo, vo);
      for (int g = g0; g < g1; ++g) {
        const int x0 = 4 * g, n = std::min(4, FW - x0);
        for (int j = 0; j < n; ++j) check((long long)y * FW + x0 + j, y);
        for (int j = 0; j < n / 2; ++j) {
          check(uo + yuv_chroma_step<FMT>() * ((x0 >> 1) + j), y);
          check(vo + yuv_chroma_step<FMT>() * ((x0 >> 1) + j), y);
        }
      }
    }
  }
  printf("bytes: fetch=%lld dma=%lld bgr_fetch=%lld bgr_dma=%lld\n", fetch, dma, bgr_fetch, bgr_dma);
  printf("coverage: checked=%lld fails=%lld\n", checked, fails);
  return fails ? 1 : 0;
}

int main(int argc, char** argv) {
  if (argc == 5 && !strcmp(argv[1], "yuv")) {
    const int fmt = atoi(argv[2]);
    if (fmt == YUV_NV12) return run<YUV_NV12>(argv[3], argv[4]);
    if (fmt == YUV_I420) return run<YUV_I420>(argv[3], argv[4]);
  }
  fprintf(stderr, "usage: yuv yuv <1|2> <in.bin> <out.bin>\n");
  return 2;
}
