// Host form of the grey and BGRA stages of the device encoders (bevk_jpeg_enc.cuh, bevk_png_enc.cuh): the same
// __host__ __device__ functions the kernels run, serially over whole images, so tests/test_host_encode_channels.py can
// compare them with cv2.imencode.
//   JPEG  channel_opts, the sample load of C-channel images, FDCT, quantisation, DC prediction with the restart reset,
//         optimal tables, Huffman coding, pads, stuffing, RSTn, the one-component header: whole baseline streams
//   PNG   the filter stage with bpp C (BGRA -> RGBA) and the IHDR colour type: the filtered bytes zlib compresses; under
//         a hash-chain list (levels 4..9, DEFAULT / FILTERED / FIXED) also the whole zlib stream, whose parse depends on
//         the row length C * W + 1 at the window slides
//
//   encode_channels <in.bin> <out.bin>
//     in : records of int32 format (0 JPEG, 1 PNG), width, height, channels, quality, n, n ints of params, then
//          width*height*channels bytes (dense)
//     out: per record int32 status (0 ok, 1 list refused, 2 progressive: no stream), int32 colour type (PNG) or header
//          bytes (JPEG), int32 class bits (below), uint64 bound, uint64 size, uint64 zlib size, the JPEG stream or the
//          PNG filtered bytes, then the PNG's zlib stream (hash-chain lists only; else empty)
// Class bits (hash-chain PNG, as tests/host/png_lazy.cu numbers them): 18 a head at k w_size exactly MAX_DIST back made
// NIL by the parse (lazy_chain's extra literal), 19 such a head searched, 20 such a head NIL whatever the parse (the
// input ends before (k + 1) w_size, or a row ends at (k + 1) w_size - 1).
// Built by tests/test_host_encode_channels.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_jpeg_enc.cuh"
#include "../../cameracalibration_b200/csrc/bevk_jpeg_prog.cuh"
#include "../../cameracalibration_b200/csrc/bevk_png_enc.cuh"

using namespace bevk;

struct CountSymbols {
  long long (*freq)[257];
  int tb;
  void operator()(int cls, int sym) const { freq[2 * tb + cls][sym]++; }
};

static std::vector<uint8_t> jpeg_encode(const uint8_t* img, int W, int H, int C, const jpeg::Opts& o) {
  using namespace jpeg;
  Tables t;
  make_tables(o, &t);
  const Geom g = geom(W, H, o);
  const int ny = g.hy * g.vy, bpm = mcu_blocks(g);
  const long long nblk = blocks_per_image(g), mcus = (long long)g.mcux * g.mcuy;
  std::vector<int16_t> coef((size_t)nblk * 64);
  for (long long b = 0; b < nblk; ++b) {
    const int m = (int)(b / bpm), k = (int)(b % bpm), mx = m % g.mcux, my = m / g.mcux;
    int16_t* out = &coef[(size_t)b * 64];
    if (is_dummy(g, mx, my, k)) { memset(out, 0, 128); continue; }
    int d[64];
    load_block(img, (long long)C * W, g, C, mx, my, k, d);
    fdct_islow(d);
    quantise(d, t.qdiv[k < ny ? 0 : 1]);
    for (int j = 0; j < 64; ++j) out[j] = (int16_t)d[t.zz[j]];
  }
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
  uint8_t hbits[4][16], hvals[4][256];
  if (o.optimize) {
    static long long freq[4][257];
    memset(freq, 0, sizeof freq);
    for (long long b = 0; b < nblk; ++b)
      block_symbols(diff[(size_t)b], Zigzag16{&coef[(size_t)b * 64]}, CountSymbols{freq, (int)(b % bpm) < ny ? 0 : 1});
    for (int q = 0; q < (o.nc == 1 ? 2 : 4); ++q) gen_optimal_table(freq[q], hbits[q], hvals[q]);
    for (int c = 0; c < (o.nc == 1 ? 1 : 2); ++c) {
      huff_codes(hbits[2 * c], hvals[2 * c], t.dc[c], 12);
      huff_codes(hbits[2 * c + 1], hvals[2 * c + 1], t.ac[c], 256);
    }
  }
  std::vector<uint32_t> words((size_t)(entropy_bound_bits(g, o) / 32 + 2), 0u);
  std::vector<unsigned long long> istart;
  BitWriter wr(words.data(), 0);
  unsigned long long pos = 0;
  for (long long b = 0; b < nblk; ++b) {
    const int m = (int)(b / bpm), k = (int)(b % bpm), tb = k < ny ? 0 : 1;
    if (k == 0 && (m == 0 || (o.rst && m % o.rst == 0))) istart.push_back(pos >> 3);
    BitCount cnt;
    emit_dc(diff[(size_t)b], t.dc[tb], cnt);
    emit_ac(Zigzag16{&coef[(size_t)b * 64]}, t.ac[tb], cnt);
    emit_dc(diff[(size_t)b], t.dc[tb], wr);
    emit_ac(Zigzag16{&coef[(size_t)b * 64]}, t.ac[tb], wr);
    pos += cnt.n;
    if (k == bpm - 1 && (m == mcus - 1 || (o.rst && (m + 1) % o.rst == 0))) {
      const int pad = (int)((8 - (pos & 7)) & 7);
      if (pad) wr.put((1u << pad) - 1u, pad);
      pos += pad;
    }
  }
  if ((long long)istart.size() != intervals(g, o)) { fprintf(stderr, "interval count\n"); exit(3); }
  wr.flush();
  const size_t nbytes = (size_t)(pos >> 3);
  const uint8_t* bytes = reinterpret_cast<const uint8_t*>(words.data());
  std::vector<uint8_t> s(kMaxHeaderBytes + 2 * nbytes + 2 * istart.size() + 2);
  make_header(W, H, o, s.data());
  size_t off = (size_t)header_bytes(o);
  if (o.optimize) {
    std::vector<uint8_t> common(s.begin(), s.begin() + off);
    off = (size_t)optimal_header(common.data(), (int)common.size(), hbits, hvals, s.data(), o.nc);
  }
  size_t next = 1;
  for (size_t p = 0; p < nbytes; ++p) {
    if (next < istart.size() && istart[next] == p) {
      s[off++] = 0xff;
      s[off++] = (uint8_t)(0xd0 + ((next - 1) & 7));
      ++next;
    }
    off += stuff_copy(bytes + p, 1, s.data() + off);
  }
  s[off++] = 0xff;
  s[off++] = 0xd9;
  s.resize(off);
  return s;
}

template <int C>
static std::vector<uint8_t> png_filtered(const uint8_t* img, int W, int H, const png::Opts& o) {
  using namespace png;
  const long long rb = row_bytes(W, C), pitch = (long long)C * W;
  const int filters = row_filters(o.filters, W, H);
  std::vector<uint8_t> f((size_t)image_bytes(W, H, C));
  for (int y = 0; y < H; ++y) {
    const uint8_t* cur = img + y * pitch;
    const uint8_t* prev = y ? cur - pitch : nullptr;
    unsigned long long sum[5] = {0, 0, 0, 0, 0};
    for (int t = 0; t < 5; ++t)
      for (long long i = 0; i < pitch; ++i) sum[t] += filter_cost(filter_byte<C>(t, cur, prev, i));
    const int t = choose_filter(filters, sum);
    uint8_t* row = &f[(size_t)(y * rb)];
    row[0] = (uint8_t)t;
    for (long long i = 0; i < pitch; ++i) row[1 + i] = filter_byte<C>(t, cur, prev, i);
  }
  return f;
}

// zlib's deflate_slow over filtered bytes f with rows of rb bytes, as the device runs it: lazy_match per position over
// serial hash chains, lazy_chain from canonical position to canonical position, then blocks, trees, codes, header and
// Adler-32 (the same steps as tests/host/png_lazy.cu, for any row length).
static std::vector<uint8_t> zlib_lazy(const std::vector<uint8_t>& f, long long rb, const png::Opts& o, unsigned* classes) {
  using namespace png;
  const long long N = (long long)f.size();
  std::vector<unsigned> prev((size_t)N, 0u), head(1 << 15, 0u);
  for (long long p = 0; p + 3 <= N; ++p) {
    const unsigned h = hash3(f.data(), p);
    prev[(size_t)p] = head[h];
    head[h] = (unsigned)p;
  }
  std::vector<MatchRec> recs((size_t)N);
  for (long long p = 0; p < N; ++p) recs[(size_t)p] = lazy_match(f.data(), N, prev.data(), p, o.level, o.strategy, rb);
  const RecAt rec{recs.data()};
  const LazyCfg cfg = lazy_cfg(o.level);
  const long long w = 1ll << window_bits(N), maxd = w - kMinLookahead;
  std::vector<uint16_t> sym, dist;
  std::vector<long long> pos;
  for (long long s = 0; s < N;) {
    const Chain ch = lazy_chain(s, N, o.level, rb, rec);
    for (unsigned k = 0; k < ch.lits; ++k) { sym.push_back(f[(size_t)(s + k)]); dist.push_back(0); pos.push_back(s + k); }
    int pl = 2;   // the steps of this chain: classify the searches that meet a head at k w_size exactly MAX_DIST back
    for (long long x = s; x <= s + ch.lits + (ch.m != 0) && x < N; ++x) {
      const long long hd = prev[(size_t)x];
      if (N - x >= 3 && pl < cfg.lazy && hd && x - hd == maxd && hd % w == 0)
        *classes |= (N < hd + w || (hd + w - 1) % rb == 0) ? 1u << 20 : 1u << 19;
      const MatchRec r = rec(x);
      const uint32_t m = (pl >= cfg.good ? r.quarter : r.full) & ~kKwHead;
      if (rec_len(m) > pl) pl = rec_len(m);
    }
    if (ch.m) {
      const long long x = s + ch.lits;
      const int len = rec_len(ch.m);
      sym.push_back((uint16_t)(256 + len - 3)); dist.push_back((uint16_t)rec_dist(ch.m)); pos.push_back(x);
      if (ch.extra) {
        sym.push_back(f[(size_t)(x + len)]); dist.push_back(0); pos.push_back(x + len);
        *classes |= 1u << 18;
      }
    }
    s = ch.next;
  }
  const long long nsym = (long long)sym.size();
  const bool tail_lit = nsym > 0 && sym.back() < 256 && pos.back() == N - 1;
  const long long nblk = nsym % kBlockSyms == 0 && tail_lit ? nsym / kBlockSyms : nsym / kBlockSyms + 1;
  std::vector<uint32_t> words((size_t)(zlib_bound(N) / 4 + 4), 0);
  BitSink out{words.data(), 16};
  std::vector<uint32_t> hdr(kHdrWords);
  TreeWork* tw = new TreeWork;
  for (long long b = 0; b < nblk; ++b) {
    const long long s0 = b * kBlockSyms, s1 = std::min(nsym, s0 + kBlockSyms);
    const long long raw0 = s0 < nsym ? pos[(size_t)s0] : N, raw1 = s1 < nsym ? pos[(size_t)s1] : N;
    memset(tw, 0, sizeof *tw);
    for (long long j = s0; j < s1; ++j) {
      const int v = sym[(size_t)j];
      if (v < 256) tw->lt[v].fc++;
      else { tw->lt[257 + length_code(v - 256 + 3)].fc++; tw->dt[dist_code(dist[(size_t)j])].fc++; }
    }
    tw->lt[kEndBlock].fc = 1;
    unsigned hb = 0;
    std::fill(hdr.begin(), hdr.end(), 0u);
    const int type = decide_block(*tw, (unsigned long long)(raw1 - raw0), &hb, hdr.data(), o.strategy == kZFixed);
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
        uint64_t v;
        const int n = symbol_code(tw->lt, tw->dt, sym[(size_t)j], dist[(size_t)j], &v);
        out.put((uint32_t)v, n < 32 ? n : 32);
        if (n > 32) out.put((uint32_t)(v >> 32), n - 32);
      }
      out.put(tw->lt[kEndBlock].fc, tw->lt[kEndBlock].dl);
    }
    if (last) out.pos = (out.pos + 7) & ~7ull;
  }
  delete tw;
  const long long zbytes = (long long)(out.pos / 8) + 4;
  std::vector<uint8_t> z((size_t)zbytes);
  memcpy(z.data(), words.data(), (size_t)(zbytes - 4));
  zlib_header(N, z.data(), zlib_flevel(o));
  Adler a{0, 0, 0};
  for (long long p = 0; p < N; ++p) a = adler_cat(a, Adler{f[(size_t)p], f[(size_t)p], 1});
  const uint32_t ad = adler_final(a);
  for (int k = 0; k < 4; ++k) z[(size_t)(zbytes - 4 + k)] = (uint8_t)(ad >> (24 - 8 * k));
  return z;
}

int main(int argc, char** argv) {
  if (argc != 3) { fprintf(stderr, "usage: encode_channels <in.bin> <out.bin>\n"); return 2; }
  FILE* fi = fopen(argv[1], "rb");
  FILE* fo = fopen(argv[2], "wb");
  if (!fi || !fo) return 4;
  int32_t hdr[6];
  while (fread(hdr, 4, 6, fi) == 6) {
    const int fmt = hdr[0], W = hdr[1], H = hdr[2], C = hdr[3], q = hdr[4], n = hdr[5];
    std::vector<int> params((size_t)(n > 0 ? n : 0) + 1);
    if (n > 0 && fread(params.data(), 4, (size_t)n, fi) != (size_t)n) return 5;
    std::vector<uint8_t> img((size_t)W * H * C);
    if (fread(img.data(), 1, img.size(), fi) != img.size()) return 5;
    int32_t status = 0, info = 0;
    unsigned classes = 0;
    uint64_t bound = 0;
    std::vector<uint8_t> s, z;
    if (fmt == 0) {
      jpeg::Opts o;
      if (!jpeg::normalise(q, params.data(), n, &o)) status = 1;
      o = jpeg::channel_opts(o, C);
      const jpeg::Geom g = jpeg::geom(W, H, o);
      bound = o.progressive ? jpeg::prog::progressive_bound(g, o.rst) : jpeg::encode_bound(g, o);
      info = jpeg::header_bytes(o);
      if (status == 0 && o.progressive) status = 2;
      if (status == 0) s = jpeg_encode(img.data(), W, H, C, o);
    } else {
      png::Opts o;
      status = png::normalise(params.data(), n, &o, true);
      info = png::colour_type(C);
      bound = (uint64_t)png::encode_bound(W, H, C);
      if (status == 0)
        s = C == 1 ? png_filtered<1>(img.data(), W, H, o) : C == 4 ? png_filtered<4>(img.data(), W, H, o)
                   : png_filtered<3>(img.data(), W, H, o);
      if (status == 0 && png::lazy_parse(o)) z = zlib_lazy(s, png::row_bytes(W, C), o, &classes);
    }
    const int32_t meta32[3] = {status, info, (int32_t)classes};
    const uint64_t meta[3] = {bound, s.size(), z.size()};
    fwrite(meta32, 4, 3, fo);
    fwrite(meta, 8, 3, fo);
    fwrite(s.data(), 1, s.size(), fo);
    fwrite(z.data(), 1, z.size(), fo);
  }
  fclose(fi);
  fclose(fo);
  return 0;
}
