// Host form of the device PNG encoder (bevk_png_enc.cuh): png::normalise turns the IMWRITE_PNG_* list into Opts, then
// the same __host__ __device__ stage functions the kernels run -- filter choice and filtered rows, the Z_RLE /
// Z_HUFFMAN_ONLY parse, per-block trees and block type, symbol codes, zlib header, Adler-32, IDAT framing and CRC-32 --
// run serially over whole images, so tests/test_host_png.py can compare the streams with cv2.imencode(".png", img,
// params).  It also checks the case the device pipeline relies on: a block zlib would see without its start in the
// window (raw span > window - 262) never comes out stored.
//
//   png_enc <in.bin> <out.bin>
//     in : records of int32 width, height, n, n ints of params, then width*height*3 bytes (BGR, dense)
//     out: per record int32 normalise result (0 ok, 1 refused as an argument, 2 unsupported), int32 class bits (below),
//          uint64 stream size, uint64 encode bound, the stream (empty unless the result is 0)
// Class bits: 0 stored block, 1 static, 2 dynamic, 3 empty final block, 4 match of 258, 5 match of 3, 6 run of exactly
// 3 bytes, 7 match across a row boundary, 8..12 filter 0..4 chosen by the adaptive heuristic, 13 window-reduced zlib
// header, 14 more than one IDAT, 15 Adler-32 split across two IDATs.
// Built by tests/test_host_png.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_png_enc.cuh"

using namespace bevk::png;

static unsigned g_classes;

static void put_be32(std::vector<uint8_t>& o, uint32_t v) {
  for (int k = 3; k >= 0; --k) o.push_back((uint8_t)(v >> (8 * k)));
}
static void put_chunk(std::vector<uint8_t>& o, const char* type, const uint8_t* data, size_t n) {
  put_be32(o, (uint32_t)n);
  const size_t at = o.size();
  o.insert(o.end(), type, type + 4);
  o.insert(o.end(), data, data + n);
  put_be32(o, crc32(&o[at], (long long)n + 4));
}

static std::vector<uint8_t> encode(const uint8_t* img, int W, int H, const Opts& o) {
  const long long rb = row_bytes(W), N = image_bytes(W, H), pitch = 3ll * W;
  const int filters = row_filters(o.filters, W, H);
  const bool adaptive = (filters & (filters - 1)) != 0;
  std::vector<uint8_t> f((size_t)N);
  for (int y = 0; y < H; ++y) {
    const uint8_t* cur = img + y * pitch;
    const uint8_t* prev = y ? cur - pitch : nullptr;
    unsigned long long sum[5] = {0, 0, 0, 0, 0};
    for (int t = 0; t < 5; ++t)
      for (long long i = 0; i < pitch; ++i) sum[t] += filter_cost(filter_byte(t, cur, prev, i));
    const int t = choose_filter(filters, sum);
    if (adaptive) g_classes |= 1u << (8 + t);
    uint8_t* row = &f[(size_t)(y * rb)];
    row[0] = (uint8_t)t;
    for (long long i = 0; i < pitch; ++i) row[1 + i] = filter_byte(t, cur, prev, i);
  }
  // parse
  std::vector<uint16_t> sym;
  std::vector<long long> pos;
  long long s = 0;
  for (long long p = 0; p < N; ++p) {
    if (run_start(f.data(), p)) {
      s = p;
      long long e = p;
      while (e < N && f[e] == f[p]) ++e;
      if (e - p == 3 && o.strategy == kZRle) g_classes |= 1u << 6;
    }
    const int v = o.strategy == kZRle ? rle_symbol(f.data(), N, p, s) : f[p];
    if (v < 0) continue;
    if (v >= 256) {
      const int len = v - 256 + 3;
      if (len == 258) g_classes |= 1u << 4;
      if (len == 3) g_classes |= 1u << 5;
      if ((p + len - 1) / rb != p / rb) g_classes |= 1u << 7;
    }
    sym.push_back((uint16_t)v);
    pos.push_back(p);
  }
  const long long nsym = (long long)sym.size(), nblk = nsym / kBlockSyms + 1;
  const long long wsize = 1ll << window_bits(N);
  std::vector<uint32_t> words((size_t)(zlib_bound(N) / 4 + 4), 0);
  BitSink out{words.data(), 16};
  std::vector<uint32_t> hdr(kHdrWords);
  TreeWork* w = new TreeWork;
  for (long long b = 0; b < nblk; ++b) {
    const long long s0 = b * kBlockSyms, s1 = std::min(nsym, s0 + kBlockSyms);
    const long long raw0 = s0 < nsym ? pos[(size_t)s0] : N, raw1 = s1 < nsym ? pos[(size_t)s1] : N;
    memset(w, 0, sizeof *w);
    for (long long j = s0; j < s1; ++j) {
      const int v = sym[(size_t)j];
      if (v < 256) w->lt[v].fc++;
      else { w->lt[257 + length_code(v - 256 + 3)].fc++; w->dt[0].fc++; }
    }
    w->lt[kEndBlock].fc = 1;
    unsigned hb = 0;
    std::fill(hdr.begin(), hdr.end(), 0u);
    const int type = decide_block(*w, (unsigned long long)(raw1 - raw0), &hb, hdr.data());
    if (raw1 - raw0 > wsize - 262 && type == kStored) {
      fprintf(stderr, "block %lld: %lld raw bytes (window %lld) chosen stored\n", b, raw1 - raw0, wsize);
      exit(3);
    }
    g_classes |= 1u << type;
    if (s0 == nsym) g_classes |= 1u << 3;
    const bool last = b == nblk - 1;
    out.put((unsigned)(type << 1) + last, 3);
    if (type == kStored) {
      out.pos = (out.pos + 7) & ~7ull;
      const unsigned len = (unsigned)(raw1 - raw0);
      out.put(len, 16);
      out.put(~len & 0xffff, 16);
      for (long long p = raw0; p < raw1; ++p) out.put(f[(size_t)p], 8);
    } else {
      for (unsigned k = 0; k < hb; ++k) out.put((hdr[k >> 5] >> (k & 31)) & 1, 1);
      for (long long j = s0; j < s1; ++j) {
        uint32_t v;
        const int n = symbol_code(w->lt, w->dt, sym[(size_t)j], &v);
        out.put(v, n);
      }
      out.put(w->lt[kEndBlock].fc, w->lt[kEndBlock].dl);
    }
    if (last) out.pos = (out.pos + 7) & ~7ull;
  }
  delete w;
  const long long zbytes = (long long)(out.pos / 8) + 4;
  std::vector<uint8_t> z((size_t)zbytes);
  memcpy(z.data(), words.data(), (size_t)(zbytes - 4));
  zlib_header(N, z.data());
  Adler a{0, 0, 0};
  for (long long p = 0; p < N; ++p) a = adler_cat(a, Adler{f[(size_t)p], f[(size_t)p], 1});
  const uint32_t ad = adler_final(a);
  for (int k = 0; k < 4; ++k) z[(size_t)(zbytes - 4 + k)] = (uint8_t)(ad >> (24 - 8 * k));
  if (z[0] != 0x78) g_classes |= 1u << 13;
  if (zbytes > kIdatBytes) g_classes |= 1u << 14;
  if ((zbytes - 4) / kIdatBytes != (zbytes - 1) / kIdatBytes) g_classes |= 1u << 15;
  // PNG
  std::vector<uint8_t> png = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  uint8_t ihdr[13] = {(uint8_t)(W >> 24), (uint8_t)(W >> 16), (uint8_t)(W >> 8), (uint8_t)W,
                      (uint8_t)(H >> 24), (uint8_t)(H >> 16), (uint8_t)(H >> 8), (uint8_t)H, 8, 2, 0, 0, 0};
  put_chunk(png, "IHDR", ihdr, 13);
  for (long long c = 0; c < zbytes; c += kIdatBytes) put_chunk(png, "IDAT", &z[(size_t)c], (size_t)std::min<long long>(kIdatBytes, zbytes - c));
  put_chunk(png, "IEND", nullptr, 0);
  if ((long long)png.size() != png_bytes(zbytes) || (long long)png.size() > encode_bound(W, H)) {
    fprintf(stderr, "size %zu vs framing %lld / bound %lld\n", png.size(), png_bytes(zbytes), encode_bound(W, H));
    exit(4);
  }
  return png;
}

int main(int argc, char** argv) {
  if (argc != 3) { fprintf(stderr, "usage: png_enc in.bin out.bin\n"); return 2; }
  FILE* fi = fopen(argv[1], "rb");
  FILE* fo = fopen(argv[2], "wb");
  if (!fi || !fo) { perror("open"); return 2; }
  int head[3];
  while (fread(head, 4, 3, fi) == 3) {
    const int W = head[0], H = head[1], n = head[2];
    std::vector<int> params((size_t)n);
    if (n && fread(params.data(), 4, (size_t)n, fi) != (size_t)n) return 2;
    std::vector<uint8_t> img((size_t)W * H * 3);
    if (fread(img.data(), 1, img.size(), fi) != img.size()) return 2;
    Opts o;
    const int ok = normalise(params.data(), n, &o);
    g_classes = 0;
    std::vector<uint8_t> png;
    if (ok == 0) png = encode(img.data(), W, H, o);
    const int32_t rec[2] = {ok, (int32_t)g_classes};
    const uint64_t sz[2] = {png.size(), (uint64_t)encode_bound(W, H)};
    fwrite(rec, 4, 2, fo);
    fwrite(sz, 8, 2, fo);
    fwrite(png.data(), 1, png.size(), fo);
  }
  fclose(fo);
  return 0;
}
