// Host form of the encoder's BALANCE source (bevk_jpeg_enc.cuh GainSrc): a raw composed BEV canvas, its channel sums and
// an optional car are encoded serially through the same __host__ __device__ functions the device runs -- the gain table
// of gray_world_gains + gain_entry (k_gain's), the saturating car, the sampling, FDCT, Huffman codes and stuffing -- so
// tests/test_host_bev_jpeg.py can compare the streams with cv2.imencode(cv2.add(color_balance(canvas), car)).
//
//   bev_jpeg <in.bin> <out.bin>
//     in : records of int32 width, height, quality, has_car, uint64 csum[3], the canvas (width*height*3 bytes, BGR,
//          dense), then the car (same size) when has_car
//     out: per record uint64 stream size, the stream
// Built by tests/test_host_bev_jpeg.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_jpeg_enc.cuh"

using namespace bevk;
using namespace bevk::jpeg;

template <class Src>
static std::vector<uint8_t> encode(const Src& src, int W, int H, int quality) {
  Tables t;
  make_tables(quality, &t);
  const Geom g = geom(W, H);
  const long long nblk = blocks_per_image(g);
  std::vector<int16_t> coef((size_t)nblk * 64);
  for (long long b = 0; b < nblk; ++b) {     // k_jpeg_blocks
    const int m = (int)(b / 6), k = (int)(b % 6), mx = m % g.mcux, my = m / g.mcux;
    int16_t* out = &coef[(size_t)b * 64];
    if (is_dummy(g, mx, my, k)) { memset(out, 0, 128); continue; }
    int d[64];
    load_block(src, g, mx, my, k, d);
    fdct_islow(d);
    quantise(d, t.qdiv[k < 4 ? 0 : 1]);
    for (int j = 0; j < 64; ++j) out[j] = (int16_t)d[t.zz[j]];
  }
  std::vector<uint32_t> words((size_t)(entropy_bound_bits(W, H) / 32 + 2), 0u);
  BitWriter wr(words.data(), 0);
  unsigned long long pos = 0;
  int pred[3] = {0, 0, 0}, dc_y = 0;
  for (long long b = 0; b < nblk; ++b) {     // DC prediction in scan order, entropy coding
    const int m = (int)(b / 6), k = (int)(b % 6), mx = m % g.mcux, my = m / g.mcux;
    const int t_ = k < 4 ? 0 : 1, comp = k < 4 ? 0 : k - 3;
    const int dc = is_dummy(g, mx, my, k) ? dc_y : coef[(size_t)b * 64];
    if (k < 4) dc_y = dc;
    BitCount cnt;
    emit_dc(dc - pred[comp], t.dc[t_], cnt);
    emit_ac(Zigzag16{&coef[(size_t)b * 64]}, t.ac[t_], cnt);
    emit_dc(dc - pred[comp], t.dc[t_], wr);
    emit_ac(Zigzag16{&coef[(size_t)b * 64]}, t.ac[t_], wr);
    pos += cnt.n;
    pred[comp] = dc;
  }
  const int pad = (int)((8 - (pos & 7)) & 7);
  if (pad) wr.put((1u << pad) - 1u, pad);
  wr.flush();
  const size_t nbytes = (size_t)((pos + 7) >> 3);
  std::vector<uint8_t> s(kHeaderBytes + 2 * nbytes + 2);
  make_header(W, H, quality, s.data());
  const size_t o = kHeaderBytes + stuff_copy(reinterpret_cast<const uint8_t*>(words.data()), (int)nbytes, s.data() + kHeaderBytes);
  s[o] = 0xff;
  s[o + 1] = 0xd9;
  s.resize(o + 2);
  return s;
}

int main(int argc, char** argv) {
  if (argc != 3) { fprintf(stderr, "usage: bev_jpeg <in.bin> <out.bin>\n"); return 2; }
  FILE* fi = fopen(argv[1], "rb");
  FILE* fo = fopen(argv[2], "wb");
  if (!fi || !fo) return 4;
  int32_t hdr[4];
  while (fread(hdr, 4, 4, fi) == 4) {
    const int W = hdr[0], H = hdr[1], q = hdr[2], has_car = hdr[3];
    unsigned long long csum[3];
    if (fread(csum, 8, 3, fi) != 3) return 5;
    const size_t bytes = (size_t)W * H * 3;
    std::vector<uint8_t> canvas(bytes), car(has_car ? bytes : 0);
    if (fread(canvas.data(), 1, bytes, fi) != bytes) return 5;
    if (has_car && fread(car.data(), 1, bytes, fi) != bytes) return 5;
    double gain[3];                          // what every CTA of k_jpeg_blocks<GainSrc> builds for this image
    gray_world_gains(csum, (double)W * (double)H, gain);
    uint8_t tab[768];
    for (int j = 0; j < 768; ++j) tab[j] = gain_entry(gain[j >> 8], j & 255);
    const GainSrc src{canvas.data(), 3ll * W, tab, has_car ? car.data() : nullptr, 3ll * W};
    const std::vector<uint8_t> s = encode(src, W, H, q);
    const uint64_t n = s.size();
    fwrite(&n, 8, 1, fo);
    fwrite(s.data(), 1, s.size(), fo);
  }
  fclose(fi);
  fclose(fo);
  return 0;
}
