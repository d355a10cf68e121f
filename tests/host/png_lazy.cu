// Host form of the device PNG encoder's hash-chain path (bevk_png_enc.cuh, levels 4..9 under Z_DEFAULT_STRATEGY,
// Z_FILTERED and Z_FIXED): png::normalise(..., hash_chain = true) reads the IMWRITE_PNG_* list, then the same
// __host__ __device__ functions the kernels run -- filters, lazy_match per position, lazy_chain from canonical position
// to canonical position, per-block trees and block type, symbol codes, zlib header, Adler-32, IDAT framing -- run
// serially over whole images, so tests/test_host_png_lazy.py can compare the streams with cv2.imencode(".png", img,
// params).  The chains' prev[] comes from a serial head table here (the device sorts positions by hash).  It also checks
// the case the device relies on: a block zlib would see without its start in the window (raw span > window - 262)
// never comes out stored.
//
//   png_lazy <in.bin> <out.bin>
//     in : records of int32 width, height, n, n ints of params, then width*height*3 bytes (BGR, dense)
//     out: per record int32 normalise result (0 ok, 1 refused as an argument, 2 unsupported, 3 accepted but not a
//          hash-chain list), int32 class bits (below), uint64 stream size, uint64 encode bound, the stream
// Class bits: 0 window slide, 1 reduced window, 2 more than one block, 3 empty final block, 4 stored block, 5 match of
// 258, 6 nice_match exit before the chain ends, 7 chain cut at max_chain, 8 quarter chain differs from the full one at
// a step that uses it, 9 TOO_FAR drop, 10 Z_FILTERED drop, 11 head candidate at exactly MAX_DIST, 12 chain successor at
// exactly MAX_DIST (cut), 13 hash collision in a chain, 14 match ending at the end of the stream with the comparison
// reaching past it, 15 dynamic block with more than one distance code, 16 final block ending in the literal flushed
// without a block split (16383k symbols, no empty block), 17 static block under Z_FIXED, 18 head at k w_size exactly
// MAX_DIST back made NIL by the parse (the step before lies below the last row end before (k + 1) w_size minus 262:
// lazy_chain's extra literal), 19 such a head searched (the window was full), 20 such a head NIL whatever the parse
// (the input ends before (k + 1) w_size, or a row ends at (k + 1) w_size - 1).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_png_enc.cuh"

using namespace bevk::png;

static unsigned g_classes;
static long long g_rb;   // row bytes of the image being encoded

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

// Instrument: the same walk as lazy_match, classifying what it meets at a step's search.
static void probe(const std::vector<uint8_t>& f, long long N, const std::vector<unsigned>& prev, long long p, int level,
                  int strategy, int pl) {
  const LazyCfg c = lazy_cfg(level);
  if (N - p < 3 || pl >= c.lazy) return;
  const long long head = prev[(size_t)p], w = 1ll << window_bits(N), maxd = w - kMinLookahead;
  if (head == 0 || p - head > maxd) return;
  if (p - head == maxd) g_classes |= 1u << 11;
  if (p - head == maxd && head % w == 0) {
    if (N < head + w || (head + w - 1) % g_rb == 0) g_classes |= 1u << 20;
    else g_classes |= 1u << 19;
  }
  const int la = (int)std::min<long long>(N - p, kMaxMatch), nice = std::min(c.nice, la);
  const int chain = pl >= c.good ? c.chain >> 2 : c.chain;
  const long long limit = p > maxd ? p - maxd : 0;
  int best = 2, seen = 0;
  long long bestd = 0, cur = head;
  const unsigned h = hash3(f.data(), p);
  for (;;) {
    if (hash3(f.data(), cur) != h) { fprintf(stderr, "chain of %lld holds %lld of another hash\n", p, cur); exit(5); }
    if (f[(size_t)cur] != f[(size_t)p] || f[(size_t)cur + 1] != f[(size_t)p + 1] || f[(size_t)cur + 2] != f[(size_t)p + 2])
      g_classes |= 1u << 13;
    int len = 0;
    while (len < la && f[(size_t)(cur + len)] == f[(size_t)(p + len)]) ++len;
    if (len > best) {
      best = len;
      bestd = p - cur;
      if (len >= nice) {
        if (len == la && la < kMaxMatch) g_classes |= 1u << 14;
        else if (prev[(size_t)cur] > limit && seen + 1 < chain) g_classes |= 1u << 6;
        break;
      }
    }
    if (++seen == chain) {
      if (prev[(size_t)cur] > limit) g_classes |= 1u << 7;
      break;
    }
    const long long nx = prev[(size_t)cur];
    if (nx <= limit) {
      if (nx != 0 && p - nx == maxd) g_classes |= 1u << 12;
      break;
    }
    cur = nx;
  }
  if (best > pl && best <= 5 && best >= 3) {
    if (strategy == kZFiltered) g_classes |= 1u << 10;
    else if (best == 3 && bestd > kTooFar) g_classes |= 1u << 9;
  }
}

static std::vector<uint8_t> encode(const uint8_t* img, int W, int H, const Opts& o) {
  const long long rb = row_bytes(W), N = image_bytes(W, H), pitch = 3ll * W;
  const int filters = row_filters(o.filters, W, H);
  std::vector<uint8_t> f((size_t)N);
  g_rb = rb;
  for (int y = 0; y < H; ++y) {
    const uint8_t* cur = img + y * pitch;
    const uint8_t* prev = y ? cur - pitch : nullptr;
    unsigned long long sum[5] = {0, 0, 0, 0, 0};
    for (int t = 0; t < 5; ++t)
      for (long long i = 0; i < pitch; ++i) sum[t] += filter_cost(filter_byte(t, cur, prev, i));
    const int t = choose_filter(filters, sum);
    uint8_t* row = &f[(size_t)(y * rb)];
    row[0] = (uint8_t)t;
    for (long long i = 0; i < pitch; ++i) row[1 + i] = filter_byte(t, cur, prev, i);
  }
  // hash chains: prev[p] = the nearest earlier position with p's hash (0: none)
  std::vector<unsigned> prev((size_t)N, 0u), head(1 << 15, 0u);
  for (long long p = 0; p + 3 <= N; ++p) {
    const unsigned h = hash3(f.data(), p);
    prev[(size_t)p] = head[h];
    head[h] = (unsigned)p;
  }
  std::vector<MatchRec> recs((size_t)N);
  for (long long p = 0; p < N; ++p) recs[(size_t)p] = lazy_match(f.data(), N, prev.data(), p, o.level, o.strategy, rb);
  const RecAt rec{recs.data()};
  // parse: canonical position to canonical position from 0
  const LazyCfg cfg = lazy_cfg(o.level);
  std::vector<uint16_t> sym;
  std::vector<uint16_t> dist;
  std::vector<long long> pos;
  const long long w = 1ll << window_bits(N);
  if (window_bits(N) < 15) g_classes |= 1u << 1;
  for (long long s = 0; s < N;) {
    const Chain ch = lazy_chain(s, N, o.level, rb, rec);
    for (unsigned k = 0; k < ch.lits; ++k) {
      sym.push_back(f[(size_t)(s + k)]); dist.push_back(0); pos.push_back(s + k);
    }
    // the steps of this chain: s .. s + lits (+ 1 when a match ends it); probe their searches
    int pl = 2;
    for (long long x = s; x <= s + ch.lits + (ch.m != 0) && x < N; ++x) {
      probe(f, N, prev, x, o.level, o.strategy, pl);
      const MatchRec r = rec(x);
      if (pl >= cfg.good && pl < cfg.lazy && (r.quarter & ~kKwHead) != (r.full & ~kKwHead)) g_classes |= 1u << 8;
      const uint32_t m = (pl >= cfg.good ? r.quarter : r.full) & ~kKwHead;
      if (rec_len(m) > pl) pl = rec_len(m);
    }
    if (ch.m) {
      const long long x = s + ch.lits;
      const int len = rec_len(ch.m);
      if (len == kMaxMatch) g_classes |= 1u << 5;
      sym.push_back((uint16_t)(256 + len - 3)); dist.push_back((uint16_t)rec_dist(ch.m)); pos.push_back(x);
      if (ch.extra) {
        sym.push_back(f[(size_t)(x + len)]); dist.push_back(0); pos.push_back(x + len);
        g_classes |= 1u << 18;
      }
    }
    if (ch.next > w + w - kMinLookahead) g_classes |= 1u << 0;
    s = ch.next;
  }
  const long long nsym = (long long)sym.size();
  const bool tail_lit = nsym > 0 && sym.back() < 256 && pos.back() == N - 1;
  const long long nblk = nsym % kBlockSyms == 0 && tail_lit ? nsym / kBlockSyms : nsym / kBlockSyms + 1;
  if (nblk > 1) g_classes |= 1u << 2;
  if (nsym % kBlockSyms == 0 && tail_lit) g_classes |= 1u << 16;
  std::vector<uint32_t> words((size_t)(zlib_bound(N) / 4 + 4), 0);
  BitSink out{words.data(), 16};
  std::vector<uint32_t> hdr(kHdrWords);
  TreeWork* tw = new TreeWork;
  for (long long b = 0; b < nblk; ++b) {
    const long long s0 = b * kBlockSyms, s1 = std::min(nsym, s0 + kBlockSyms);
    const long long raw0 = s0 < nsym ? pos[(size_t)s0] : N, raw1 = s1 < nsym ? pos[(size_t)s1] : N;
    memset(tw, 0, sizeof *tw);
    int ndist = 0;
    for (long long j = s0; j < s1; ++j) {
      const int v = sym[(size_t)j];
      if (v < 256) tw->lt[v].fc++;
      else {
        tw->lt[257 + length_code(v - 256 + 3)].fc++;
        if (tw->dt[dist_code(dist[(size_t)j])].fc++ == 0) ++ndist;
      }
    }
    tw->lt[kEndBlock].fc = 1;
    unsigned hb = 0;
    std::fill(hdr.begin(), hdr.end(), 0u);
    const int type = decide_block(*tw, (unsigned long long)(raw1 - raw0), &hb, hdr.data(), o.strategy == kZFixed);
    if (raw1 - raw0 > w - kMinLookahead && type == kStored) {
      fprintf(stderr, "block %lld: %lld raw bytes (window %lld) chosen stored\n", b, raw1 - raw0, w);
      exit(3);
    }
    if (type == kStored) g_classes |= 1u << 4;
    if (type == kDynamic && ndist > 1) g_classes |= 1u << 15;
    if (type == kStatic && o.strategy == kZFixed) g_classes |= 1u << 17;
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
  if (argc != 3) { fprintf(stderr, "usage: png_lazy in.bin out.bin\n"); return 2; }
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
    int ok = normalise(params.data(), n, &o, true);
    if (ok == 0 && !lazy_parse(o)) ok = 3;
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
