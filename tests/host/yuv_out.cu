// CPU harness of the YUV 4:2:0 canvas output (tests/test_host_yuv_out.py): the host form of k_canvas_yuv's work item
// (canvas_yuv_item) from the library's own header, over whole canvases.  nvcc compiles it; only host code runs.
//
//   yuv_out <fmt 1=NV12|2=I420> <gain 0|1> <in.bin> <out.bin>
//     in : int32[5] = BW, BH, batch, has_car, out_off; with gain the channel sums uint64[batch][3]; with has_car the car
//          uint8[BH][BW][3]; then the BGR canvases uint8[batch][BH][BW][3].
//     The YUV canvases go to a 4-byte aligned buffer + out_off (0..3), so that the word path and the byte path the kernel
//     picks for that alignment both run.  Writes uint8[batch][BH*3/2][BW] and prints "words: 0|1".
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_kernels.cuh"

using namespace bevk;

template <int FMT, bool GAIN>
static int run(const char* in_path, const char* out_path) {
  FILE* fi = fopen(in_path, "rb");
  if (!fi) return 2;
  int hd[5];
  if (fread(hd, 4, 5, fi) != 5) return 2;
  const int BW = hd[0], BH = hd[1], batch = hd[2], has_car = hd[3], out_off = hd[4];
  const size_t cbytes = (size_t)BW * BH * 3, ybytes = cbytes / 2;
  std::vector<unsigned long long> csum(GAIN ? (size_t)batch * 3 : 0);
  if (GAIN && fread(csum.data(), 8, csum.size(), fi) != csum.size()) return 2;
  std::vector<uint8_t> car(has_car ? cbytes : 0);
  if (has_car && fread(car.data(), 1, cbytes, fi) != cbytes) return 2;
  std::vector<uint32_t> canvas_words((cbytes * batch + 3) / 4);   // library scratch is aligned
  uint8_t* canvas = reinterpret_cast<uint8_t*>(canvas_words.data());
  if (fread(canvas, 1, cbytes * batch, fi) != cbytes * batch) return 2;
  fclose(fi);
  std::vector<uint32_t> out_words((ybytes * batch + 8) / 4, 0xA5A5A5A5u);
  uint8_t* out = reinterpret_cast<uint8_t*>(out_words.data()) + out_off;

  CanvasYuvArgs a{canvas, out, BW, BH, GAIN ? csum.data() : nullptr, GAIN && has_car ? car.data() : nullptr, (double)BW * BH};
  const bool words = canvas_yuv_words(a);
  std::vector<uint8_t> tab(768, 0);
  for (int b = 0; b < batch; ++b) {
    if (GAIN) {   // gain_table's entries (the kernel fills them with the threads of a CTA)
      double gain[3];
      gray_world_gains(csum.data() + 3 * b, a.npix, gain);
      for (int i = 0; i < 768; ++i) tab[i] = gain_entry(gain[i >> 8], i & 255);
    }
    const int ng = (BW + 3) >> 2;
    for (int cy = 0; cy < BH / 2; ++cy)
      for (int g = 0; g < ng; ++g) canvas_yuv_item<FMT, GAIN>(a, b, tab.data(), cy, g, words);
  }
  printf("words: %d\n", words ? 1 : 0);
  FILE* fo = fopen(out_path, "wb");
  if (!fo || fwrite(out, 1, ybytes * batch, fo) != ybytes * batch) return 3;
  fclose(fo);
  return 0;
}

int main(int argc, char** argv) {
  if (argc == 6 && !strcmp(argv[1], "yuv_out")) {
    const int fmt = atoi(argv[2]), gain = atoi(argv[3]);
    if (fmt == YUV_NV12) return gain ? run<YUV_NV12, true>(argv[4], argv[5]) : run<YUV_NV12, false>(argv[4], argv[5]);
    if (fmt == YUV_I420) return gain ? run<YUV_I420, true>(argv[4], argv[5]) : run<YUV_I420, false>(argv[4], argv[5]);
  }
  fprintf(stderr, "usage: yuv_out yuv_out <1|2> <0|1> <in.bin> <out.bin>\n");
  return 2;
}
