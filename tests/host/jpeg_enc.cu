// Host form of the device JPEG encoder (bevk_jpeg_enc.cuh): the same __host__ __device__ stage functions -- sampling
// with the edge rules, islow FDCT, quantisation, dummy blocks, DC prediction, Huffman codes, the bit writer, byte
// stuffing -- run serially over whole images, so tests/test_host_jpeg.py can compare the streams with cv2.imencode.
//
//   jpeg_enc <in.bin> <out.bin>
//     in : records of int32 width, height, quality, then width*height*3 bytes (BGR, dense)
//     out: per record uint64 stream size, uint64 bevk_jpeg_encode_bound, uint64 entropy-coded bits (without the pad),
//          the stream
// Built by tests/test_host_jpeg.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_jpeg_enc.cuh"

using namespace bevk::jpeg;

static std::vector<uint8_t> encode(const uint8_t* img, int W, int H, int quality, unsigned long long* bits) {
  Tables t;
  make_tables(quality, &t);
  const Geom g = geom(W, H);
  const long long nblk = blocks_per_image(g);
  std::vector<int16_t> coef((size_t)nblk * 64);
  // stage 1: samples -> FDCT -> quantised zigzag coefficients (dummy blocks all zero)
  for (long long b = 0; b < nblk; ++b) {
    const int m = (int)(b / 6), k = (int)(b % 6), mx = m % g.mcux, my = m / g.mcux;
    int16_t* out = &coef[(size_t)b * 64];
    if (is_dummy(g, mx, my, k)) { memset(out, 0, 128); continue; }
    int d[64];
    load_block(img, 3ll * W, g, mx, my, k, d);
    fdct_islow(d);
    quantise(d, t.qdiv[k < 4 ? 0 : 1]);
    for (int j = 0; j < 64; ++j) out[j] = (int16_t)d[t.zz[j]];
  }
  // stage 2: DC prediction in scan order (a dummy's DC is the block before it in its MCU), entropy coding
  const unsigned long long cap_bits = entropy_bound_bits(W, H);
  std::vector<uint32_t> words((size_t)(cap_bits / 32 + 2), 0u);
  BitWriter wr(words.data(), 0);
  unsigned long long pos = 0;
  int pred[3] = {0, 0, 0}, dc_y = 0;
  for (long long b = 0; b < nblk; ++b) {
    const int m = (int)(b / 6), k = (int)(b % 6), mx = m % g.mcux, my = m / g.mcux;
    const int t_ = k < 4 ? 0 : 1, comp = k < 4 ? 0 : k - 3;
    int dc;
    if (is_dummy(g, mx, my, k)) dc = dc_y;
    else dc = coef[(size_t)b * 64];
    if (k < 4) dc_y = dc;
    const int16_t* c = &coef[(size_t)b * 64];
    BitCount cnt;
    emit_dc(dc - pred[comp], t.dc[t_], cnt);
    emit_ac(Zigzag16{c}, t.ac[t_], cnt);
    const unsigned long long start = pos;
    emit_dc(dc - pred[comp], t.dc[t_], wr);
    emit_ac(Zigzag16{c}, t.ac[t_], wr);
    pos += cnt.n;
    if (wr.w * 32 + wr.n != (long long)pos) { fprintf(stderr, "bit count mismatch at block %lld (start %llu)\n", b, start); exit(3); }
    if (cnt.n > (unsigned)kMaxBlockBits) { fprintf(stderr, "block %lld: %u bits > bound\n", b, cnt.n); exit(3); }
    pred[comp] = dc;
  }
  *bits = pos;
  const int pad = (int)((8 - (pos & 7)) & 7);
  if (pad) wr.put((1u << pad) - 1u, pad);
  wr.flush();
  const size_t nbytes = (size_t)((pos + 7) >> 3);
  const uint8_t* bytes = reinterpret_cast<const uint8_t*>(words.data());
  // stage 3: header, stuffed entropy-coded segment (chunk by chunk, as k_jpeg_stuff copies), EOI
  std::vector<uint8_t> s(kHeaderBytes + 2 * nbytes + 2);
  make_header(W, H, quality, s.data());
  size_t o = kHeaderBytes;
  for (size_t off = 0; off < nbytes; off += kChunk) {
    const int n = (int)(nbytes - off < (size_t)kChunk ? nbytes - off : kChunk);
    const int ff = count_ff(bytes + off, n);
    const int w = stuff_copy(bytes + off, n, s.data() + o);
    if (w != n + ff) { fprintf(stderr, "stuffing count mismatch\n"); exit(3); }
    o += w;
  }
  s[o++] = 0xff;
  s[o++] = 0xd9;
  s.resize(o);
  return s;
}

int main(int argc, char** argv) {
  if (argc != 3) { fprintf(stderr, "usage: jpeg_enc <in.bin> <out.bin>\n"); return 2; }
  FILE* fi = fopen(argv[1], "rb");
  FILE* fo = fopen(argv[2], "wb");
  if (!fi || !fo) return 4;
  int32_t hdr[3];
  while (fread(hdr, 4, 3, fi) == 3) {
    const int W = hdr[0], H = hdr[1], q = hdr[2];
    std::vector<uint8_t> img((size_t)W * H * 3);
    if (fread(img.data(), 1, img.size(), fi) != img.size()) return 5;
    unsigned long long bits = 0;
    const std::vector<uint8_t> s = encode(img.data(), W, H, q, &bits);
    const uint64_t meta[3] = {s.size(), encode_bound(W, H), bits};
    fwrite(meta, 8, 3, fo);
    fwrite(s.data(), 1, s.size(), fo);
  }
  fclose(fi);
  fclose(fo);
  return 0;
}
