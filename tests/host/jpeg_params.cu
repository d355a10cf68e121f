// Host form of the device JPEG encoder under cv2.imwrite's JPEG parameters (bevk_jpeg_enc.cuh): jpeg::normalise turns
// the (key, value) list into Opts, then the same __host__ __device__ stage functions the kernels run -- sampling in the
// general MCU layout, islow FDCT, quantisation with the luma / chroma tables, dummy blocks, DC prediction with the restart
// reset, symbol counts and optimal tables, Huffman codes, the bit writer, interval pads, byte stuffing, RSTn markers,
// header -- run serially over whole images, so tests/test_host_jpeg_params.py can compare
// the streams with cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q] + params).
//
//   jpeg_params <in.bin> <out.bin>
//     in : records of int32 width, height, quality, n, n ints of params, then width*height*3 bytes (BGR, dense)
//     out: per record int32 ok (normalise accepted the list), hy, vy, qy, qc, rst, optimize, progressive; uint64 stream
//          size, uint64 encode bound under the options, uint64 entropy-coded bits (without pads), uint64 mask of the
//          interval pad lengths seen (bit p: a pad of p bits), uint64 1 if some interval's data ends in 0xFF before a
//          marker, the stream.  A list the encoder does not write (ok 0, or progressive set) has no stream (size 0).
// Built by tests/test_host_jpeg_params.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_jpeg_enc.cuh"

using namespace bevk::jpeg;

struct CountSymbols {   // block_symbols callback: counts of table 2 * tb + class
  long long (*freq)[257];
  int tb;
  __host__ __device__ void operator()(int cls, int sym) const { freq[2 * tb + cls][sym]++; }
};
static unsigned long long g_padmask, g_ffend;

static std::vector<uint8_t> encode(const uint8_t* img, int W, int H, const Opts& o, unsigned long long* bits) {
  Tables t;
  make_tables(o, &t);
  const Geom g = geom(W, H, o);
  const int ny = g.hy * g.vy, bpm = ny + 2;
  const long long nblk = blocks_per_image(g), mcus = (long long)g.mcux * g.mcuy;
  std::vector<int16_t> coef((size_t)nblk * 64);
  // stage 1: samples -> FDCT -> quantised zigzag coefficients (dummy blocks all zero)
  for (long long b = 0; b < nblk; ++b) {
    const int m = (int)(b / bpm), k = (int)(b % bpm), mx = m % g.mcux, my = m / g.mcux;
    int16_t* out = &coef[(size_t)b * 64];
    if (is_dummy(g, mx, my, k)) { memset(out, 0, 128); continue; }
    int d[64];
    load_block(img, 3ll * W, g, mx, my, k, d);
    fdct_islow(d);
    quantise(d, t.qdiv[k < ny ? 0 : 1]);
    for (int j = 0; j < 64; ++j) out[j] = (int16_t)d[t.zz[j]];
  }
  // stage 2: DC differences per component in scan order (a dummy's DC is the block before it in its MCU), the
  // predictors reset to 0 at the first MCU of every restart interval
  std::vector<int> diff((size_t)nblk);
  int pred[3] = {0, 0, 0}, dc_y = 0;
  for (long long b = 0; b < nblk; ++b) {
    const int m = (int)(b / bpm), k = (int)(b % bpm), mx = m % g.mcux, my = m / g.mcux;
    if (k == 0 && o.rst && m % o.rst == 0) pred[0] = pred[1] = pred[2] = 0;
    const int comp = k < ny ? 0 : k - ny + 1;
    const int dc = is_dummy(g, mx, my, k) ? dc_y : coef[(size_t)b * 64];
    if (k < ny) dc_y = dc;
    diff[(size_t)b] = dc - pred[comp];
    pred[comp] = dc;
  }
  // optimised tables: symbol counts per table (DC0, AC0, DC1, AC1), then jpeg_gen_optimal_table and the codes
  uint8_t hbits[4][16], hvals[4][256];
  if (o.optimize) {
    static long long freq[4][257];
    memset(freq, 0, sizeof freq);
    for (long long b = 0; b < nblk; ++b) {
      const int tb = (int)(b % bpm) < ny ? 0 : 1;
      block_symbols(diff[(size_t)b], Zigzag16{&coef[(size_t)b * 64]}, CountSymbols{freq, tb});
    }
    for (int q = 0; q < 4; ++q) gen_optimal_table(freq[q], hbits[q], hvals[q]);
    for (int c = 0; c < 2; ++c) {
      huff_codes(hbits[2 * c], hvals[2 * c], t.dc[c], 12);
      huff_codes(hbits[2 * c + 1], hvals[2 * c + 1], t.ac[c], 256);
    }
  }
  // stage 3: entropy coding, each restart interval padded with 1 bits to a byte; interval starts in bytes
  const long long nint = intervals(g, o);
  std::vector<uint32_t> words((size_t)(entropy_bound_bits(g, o) / 32 + 2), 0u);
  std::vector<unsigned long long> istart;
  BitWriter wr(words.data(), 0);
  unsigned long long pos = 0, raw = 0;
  const int maxbits = o.optimize ? kMaxBlockBitsOpt : kMaxBlockBits;
  for (long long b = 0; b < nblk; ++b) {
    const int m = (int)(b / bpm), k = (int)(b % bpm), t_ = k < ny ? 0 : 1;
    if (k == 0 && (m == 0 || (o.rst && m % o.rst == 0))) istart.push_back(pos >> 3);
    const int16_t* c = &coef[(size_t)b * 64];
    BitCount cnt;
    emit_dc(diff[(size_t)b], t.dc[t_], cnt);
    emit_ac(Zigzag16{c}, t.ac[t_], cnt);
    emit_dc(diff[(size_t)b], t.dc[t_], wr);
    emit_ac(Zigzag16{c}, t.ac[t_], wr);
    pos += cnt.n;
    raw += cnt.n;
    if (cnt.n > (unsigned)maxbits) { fprintf(stderr, "block %lld: %u bits > bound\n", b, cnt.n); exit(3); }
    const bool last = k == bpm - 1 && (m == mcus - 1 || (o.rst && (m + 1) % o.rst == 0));
    if (last) {
      const int pad = (int)((8 - (pos & 7)) & 7);
      if (pad) wr.put((1u << pad) - 1u, pad);
      pos += pad;
      g_padmask |= 1ull << pad;
    }
    if (wr.w * 32 + wr.n != (long long)pos) { fprintf(stderr, "bit count mismatch at block %lld\n", b); exit(3); }
  }
  if ((long long)istart.size() != nint) { fprintf(stderr, "%zu intervals, expected %lld\n", istart.size(), nint); exit(3); }
  *bits = raw;
  wr.flush();
  const size_t nbytes = (size_t)(pos >> 3);
  const uint8_t* bytes = reinterpret_cast<const uint8_t*>(words.data());
  // stage 4: header, stuffed entropy-coded segment with RSTn before every interval but the first, EOI
  std::vector<uint8_t> s(kMaxHeaderBytes + 2 * nbytes + 2 * nint + 2);
  make_header(W, H, o, s.data());
  size_t off_out = (size_t)header_bytes(o);
  if (o.optimize) {
    std::vector<uint8_t> common(s.begin(), s.begin() + off_out);
    off_out = (size_t)optimal_header(common.data(), (int)common.size(), hbits, hvals, s.data());
  }
  size_t next = 1;
  for (size_t p = 0; p < nbytes; ++p) {
    if (next < istart.size() && istart[next] == p) {
      g_ffend |= bytes[p - 1] == 0xff;
      s[off_out++] = 0xff;
      s[off_out++] = (uint8_t)(0xd0 + ((next - 1) & 7));
      ++next;
    }
    off_out += stuff_copy(bytes + p, 1, s.data() + off_out);
  }
  s[off_out++] = 0xff;
  s[off_out++] = 0xd9;
  s.resize(off_out);
  return s;
}

int main(int argc, char** argv) {
  if (argc != 3) { fprintf(stderr, "usage: jpeg_params <in.bin> <out.bin>\n"); return 2; }
  FILE* fi = fopen(argv[1], "rb");
  FILE* fo = fopen(argv[2], "wb");
  if (!fi || !fo) return 4;
  int32_t hdr[4];
  while (fread(hdr, 4, 4, fi) == 4) {
    const int W = hdr[0], H = hdr[1], q = hdr[2], n = hdr[3];
    std::vector<int> params((size_t)(n > 0 ? n : 0) + 1);
    if (n > 0 && fread(params.data(), 4, (size_t)n, fi) != (size_t)n) return 5;
    std::vector<uint8_t> img((size_t)W * H * 3);
    if (fread(img.data(), 1, img.size(), fi) != img.size()) return 5;
    Opts o;
    const int ok = normalise(q, params.data(), n, &o) ? 1 : 0;
    std::vector<uint8_t> s;
    unsigned long long bits = 0, bound = 0;
    g_padmask = g_ffend = 0;
    if (ok && !o.progressive) {
      s = encode(img.data(), W, H, o, &bits);
      bound = encode_bound(geom(W, H, o), o);
    }
    const int32_t meta32[8] = {ok, o.hy, o.vy, o.qy, o.qc, o.rst, o.optimize, o.progressive};
    const uint64_t meta[5] = {s.size(), bound, bits, g_padmask, g_ffend};
    fwrite(meta32, 4, 8, fo);
    fwrite(meta, 8, 5, fo);
    fwrite(s.data(), 1, s.size(), fo);
  }
  fclose(fi);
  fclose(fo);
  return 0;
}
