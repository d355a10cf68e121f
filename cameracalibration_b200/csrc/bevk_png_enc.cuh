// bevk_png_enc.cuh -- PNG encoder on the device (sm_90a), byte-identical to cv2.imwrite / cv2.imencode('.png') for
// 8-bit BGR images under cv2's default settings and its Z_RLE / Z_HUFFMAN_ONLY strategies, and under zlib's hash-chain
// parse at levels 4..9 (deflate_slow; the "parse (deflate_slow ...)" section and DESIGN.md section 2).
//
// cv2 writes PNG through libpng 1.6 and zlib 1.2.11.  With no parameters it asks for the SUB filter on every row,
// zlib level 1 and strategy Z_RLE; IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY asks for literals only.  Under those two strategies
// zlib's parse is a closed-form function of the filtered bytes (deflate_rle / deflate_huff), so every stage runs in
// parallel and the stream still comes out byte for byte:
//   filter     libpng swaps BGR to RGB, then filters each row: SUB, or with a compression level (or a filter list) the
//              png_write_find_filter heuristic -- the least sum of min(v, 256 - v) over the filters allowed, the first
//              filter winning a tie, the row before row 0 all zeros; 1-row images drop UP / AVG / PAETH and 1-column
//              images SUB / AVG / PAETH, an empty set becoming NONE (png_write_start_row)
//   parse      Z_RLE: a run of n equal filtered bytes (runs cross rows) is 1 literal, floor((n-1)/258) matches of 258 at
//              distance 1, then r = (n-1) mod 258 as one match if r >= 3, else r literals.  Z_HUFFMAN_ONLY: literals
//   blocks     16383 symbols each (zlib's lit_bufsize - 1 at memLevel 8); a stream whose symbol count is a multiple of
//              16383 ends with an empty final block (Z_FINISH after the flush of the full one)
//   trees      zlib 1.2.11 trees.c: build_tree with pqdownheap's depth tie-break, gen_bitlen's overflow repair at 15
//              bits, the forced second code of a tree with fewer than two symbols, scan_tree / send_tree run-length
//              codes, bl_order and max_blindex; stored / static / dynamic chosen from opt_len and static_len as
//              _tr_flush_block does.  A stored block is byte-aligned after its 3 header bits.
//   zlib       CMF/FLG from libpng's png_deflate_claim window rule and optimize_cmf (FLEVEL 0 under both strategies),
//              Adler-32 of the filtered stream, big-endian
//   PNG        signature, IHDR (colour type 2, depth 8), the zlib stream in IDAT chunks of 8192 bytes (the last one
//              shorter), IEND; every chunk with its CRC-32
// Everything per row, per position and per block is __host__ __device__: tests/host/png_enc.cu runs the same functions
// serially over whole images and compares the stream with live cv2.imencode.
//
// Device pipeline for a group of equal-sized images (bevk_api.cu: png_group):
//   k_png_filter   one CTA per row: BGR -> RGB, the filter choice, the filtered row, the row's Adler-32 sums
//   scan           inclusive max-scan (CUB) of run starts: every position's run start
//   scan           exclusive sum (CUB) of "a symbol starts here": every symbol's index
//   k_png_setup    symbols, blocks and block ranges per image
//   k_png_compact  one thread per position: the symbol (u16: < 256 literal, 256 + len - 3 match) at its index, and the
//                  raw start of every block
//   (levels 4..9 instead of the two scans and k_png_compact: k_png_keys + a CUB radix sort by (image, hash) and
//    k_png_prev -- each position's chain predecessor; k_png_match -- lazy_match per position; k_png_next -- every
//    position's next canonical position; k_png_jump -- pointer doubling marking each image's parse; k_png_count + a CUB
//    scan -- symbol indices; k_png_lazy_compact -- symbols, distances and block raw starts)
//   k_png_tree     one CTA per block: histograms, then one thread builds the trees and picks the block type
//   k_png_layout   one thread per image: block bit offsets in order (stored blocks byte-aligned), stream sizes,
//                  zlib header and Adler-32 trailer; k_png_offsets: compacted output offsets
//   k_png_pack     one CTA per block: header and tree bits, then every symbol's code at its offset (block scan of the
//                  code lengths); words shared with neighbours take atomicOr; stored blocks copy their bytes
//   k_png_frame    one warp per IDAT chunk: copies its bytes into the compacted PNG and computes its CRC-32 (per-lane
//                  CRCs combined with crc32_combine's x^(8n) mod P); chunk 0 and the last write signature, IHDR, IEND
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>

namespace bevk {
namespace png {

// cv2.IMWRITE_PNG_* keys and values
constexpr int kKeyCompression = 16, kKeyStrategy = 17, kKeyBilevel = 18, kKeyFilter = 19, kKeyZlibBuffer = 20;
constexpr int kFilterNone = 8, kFilterSub = 16, kFilterUp = 32, kFilterAvg = 64, kFilterPaeth = 128;
constexpr int kFilterFast = 56, kFilterAll = 248;
constexpr int kZDefault = 0, kZFiltered = 1, kZHuffmanOnly = 2, kZRle = 3, kZFixed = 4;

constexpr int kBlockSyms = 16383;    // symbols per deflate block (zlib lit_bufsize - 1, memLevel 8)
constexpr int kIdatBytes = 8192;     // libpng's zbuffer size: zlib bytes per IDAT chunk
constexpr int kMaxMatch = 258;
constexpr int kLCodes = 286, kDCodes = 30, kBLCodes = 19, kHeapSize = 2 * kLCodes + 1;
constexpr int kEndBlock = 256;
constexpr int kHdrWords = 72;        // a dynamic block header: 14 + 19 * 3 + (286 + 30) * 7 bits < 72 words
constexpr int kPngHead = 33;         // signature + IHDR chunk
constexpr int kPngTail = 12;         // IEND chunk
constexpr long long kMaxImageBytes = 0x7fff0000ll;   // filtered bytes per image: indices stay 32-bit

enum BlockType { kStored = 0, kStatic = 1, kDynamic = 2 };

struct Opts {
  int level = 1, strategy = kZRle, filters = kFilterSub;
  bool operator!=(const Opts& o) const { return level != o.level || strategy != o.strategy || filters != o.filters; }
};

// cv2 4.13's reading of the IMWRITE_PNG_* list (grfmt_png.cpp), in order: COMPRESSION resets the strategy to
// Z_DEFAULT_STRATEGY and clamps the level to [0, 9]; STRATEGY outside 0..4 becomes Z_RLE; FILTER outside
// {NONE, SUB, UP, AVG, PAETH, FAST, ALL} becomes SUB and replaces whatever filters the level implies.  No level: SUB and
// level 1; a level: every filter (libpng's default).  Returns 0, 1 for a list cv2 does not take (odd length, unknown
// key) or 2 for one the encoder does not reproduce: level 0 (deflate_stored, whose blocks follow libpng's output
// buffer), a hash-chain strategy (DEFAULT, FILTERED, FIXED), BILEVEL != 0 (not a 3-channel format) and ZLIBBUFFER_SIZE.
// With hash_chain, a hash-chain strategy at levels 4..9 (zlib's deflate_slow) is taken too; levels 1..3 under those
// strategies (deflate_fast, whose chains depend on its parse) stay refused.
inline int normalise(const int* p, int n, Opts* o, bool hash_chain = false) {
  if (n < 0 || (n & 1) || (n && !p)) return 1;
  int level = -1, strategy = kZRle, filter = -1;
  bool bilevel = false, zbuf = false;
  for (int i = 0; i < n; i += 2) {
    const int v = p[i + 1];
    switch (p[i]) {
      case kKeyCompression: strategy = kZDefault; level = v < 0 ? 0 : v > 9 ? 9 : v; break;
      case kKeyStrategy: strategy = v >= kZDefault && v <= kZFixed ? v : kZRle; break;
      case kKeyBilevel: bilevel = v != 0; break;
      case kKeyFilter:
        filter = (v == kFilterNone || v == kFilterSub || v == kFilterUp || v == kFilterAvg || v == kFilterPaeth ||
                  v == kFilterFast || v == kFilterAll) ? v : kFilterSub;
        break;
      case kKeyZlibBuffer: zbuf = true; break;
      default: return 1;
    }
  }
  o->level = level < 0 ? 1 : level;
  o->strategy = strategy;
  o->filters = filter >= 0 ? filter : level < 0 ? kFilterSub : kFilterAll;
  if (bilevel || zbuf || o->level == 0) return 2;
  if (strategy != kZRle && strategy != kZHuffmanOnly && !(hash_chain && o->level >= 4)) return 2;
  return 0;
}
__host__ __device__ inline bool lazy_parse(const Opts& o) { return o.strategy != kZRle && o.strategy != kZHuffmanOnly; }

// zlib 1.2.11's configuration_table for deflate_slow (levels 4..9): good_length, max_lazy, nice_length, max_chain
struct LazyCfg { int good, lazy, nice, chain; };
__host__ __device__ inline LazyCfg lazy_cfg(int level) {
  switch (level) {
    case 4: return {4, 4, 16, 16};
    case 5: return {8, 16, 32, 32};
    case 6: return {8, 16, 128, 128};
    case 7: return {8, 32, 128, 256};
    case 8: return {32, 128, 258, 1024};
    default: return {32, 258, 258, 4096};
  }
}
// FLEVEL of the zlib header (deflate.c): 0 under Z_HUFFMAN_ONLY / Z_RLE / Z_FIXED or below level 2, 1 for levels 2..5,
// 2 for level 6, 3 above
__host__ __device__ inline int zlib_flevel(const Opts& o) {
  if (o.strategy >= kZHuffmanOnly || o.level < 2) return 0;
  return o.level < 6 ? 1 : o.level == 6 ? 2 : 3;
}

// ------------------------------------------------------------------ geometry and bounds
__host__ __device__ inline long long row_bytes(int W) { return 3ll * W + 1; }
__host__ __device__ inline long long image_bytes(int W, int H) { return row_bytes(W) * H; }
// Blocks of an image of N filtered bytes: nsym / 16383 + 1 (a full last block is followed by an empty one), nsym <= N.
__host__ __device__ inline long long max_blocks(long long N) { return N / kBlockSyms + 1; }
// Every block costs at most its raw bytes + 5: a stored block is 3 bits, a pad to the byte, LEN, NLEN and the bytes,
// and zlib only codes a block when that comes out below the stored size + 4 (DESIGN.md section 2).
__host__ __device__ inline long long zlib_bound(long long N) { return 2 + N + 5 * max_blocks(N) + 4; }
__host__ __device__ inline long long idat_chunks(long long zbytes) { return (zbytes + kIdatBytes - 1) / kIdatBytes; }
__host__ __device__ inline long long png_bytes(long long zbytes) { return kPngHead + zbytes + 12 * idat_chunks(zbytes) + kPngTail; }
__host__ __device__ inline long long encode_bound(int W, int H) { return png_bytes(zlib_bound(image_bytes(W, H))); }

// Filters libpng tries on a W x H image (png_write_start_row).
__host__ __device__ inline int row_filters(int filters, int W, int H) {
  if (H == 1) filters &= ~(kFilterUp | kFilterAvg | kFilterPaeth);
  if (W == 1) filters &= ~(kFilterSub | kFilterAvg | kFilterPaeth);
  return filters ? filters : kFilterNone;
}

// ------------------------------------------------------------------ filters
// Byte i of a row in RGB order read from a BGR row.
__host__ __device__ inline int rgb_at(const uint8_t* row, long long i) { return row[i - 2 * (i % 3) + 2]; }
__host__ __device__ inline int paeth(int a, int b, int c) {
  const int p = b - c, q = a - c;
  const int pa = p < 0 ? -p : p, pb = q < 0 ? -q : q, pc = p + q < 0 ? -(p + q) : p + q;
  return (pa <= pb && pa <= pc) ? a : pb <= pc ? b : c;
}
// Filtered byte i (0 .. 3W-1) of filter type t (0 NONE .. 4 PAETH); prev NULL is a row of zeros.
__host__ __device__ inline uint8_t filter_byte(int t, const uint8_t* cur, const uint8_t* prev, long long i) {
  const int x = rgb_at(cur, i);
  const int a = i >= 3 ? rgb_at(cur, i - 3) : 0;
  const int b = prev ? rgb_at(prev, i) : 0;
  const int c = prev && i >= 3 ? rgb_at(prev, i - 3) : 0;
  int pred = 0;
  switch (t) {
    case 1: pred = a; break;
    case 2: pred = b; break;
    case 3: pred = (a + b) >> 1; break;
    case 4: pred = paeth(a, b, c); break;
    default: break;
  }
  return (uint8_t)(x - pred);
}
__host__ __device__ inline unsigned filter_cost(uint8_t v) { return v < 128 ? v : 256 - v; }
// png_write_find_filter's choice from the five sums: one filter allowed -> that one; otherwise the least sum over the
// allowed filters in the order NONE, SUB, UP, AVG, PAETH, the first one winning a tie.
__host__ __device__ inline int choose_filter(int filters, const unsigned long long sum[5]) {
  for (int t = 0; t < 5; ++t)
    if (filters == (kFilterNone << t)) return t;
  int best = 0;
  unsigned long long mins = ~0ull;
  for (int t = 0; t < 5; ++t)
    if ((filters & (kFilterNone << t)) && sum[t] < mins) { mins = sum[t]; best = t; }
  return best;
}

// ------------------------------------------------------------------ checksums
// Adler-32 as (s1, s2) sums of a segment without the initial 1: s1 = sum x_i, s2 = sum (len - i) x_i, both mod 65521.
constexpr unsigned kAdlerMod = 65521;
struct Adler { unsigned s1, s2; unsigned long long len; };
__host__ __device__ inline Adler adler_cat(Adler a, Adler b) {
  Adler r;
  r.s1 = (a.s1 + b.s1) % kAdlerMod;
  r.s2 = (unsigned)((a.s2 + (unsigned long long)(b.len % kAdlerMod) * a.s1 + b.s2) % kAdlerMod);
  r.len = a.len + b.len;
  return r;
}
__host__ __device__ inline uint32_t adler_final(Adler a) {
  const unsigned s1 = (1 + a.s1) % kAdlerMod;
  const unsigned s2 = (unsigned)((a.len % kAdlerMod + a.s2) % kAdlerMod);
  return (s2 << 16) | s1;
}

constexpr uint32_t kCrcPoly = 0xedb88320u;
__host__ __device__ inline uint32_t crc_update(uint32_t crc, const uint8_t* p, long long n) {   // raw: no pre/post inversion
  for (long long i = 0; i < n; ++i) {
    crc ^= p[i];
    for (int k = 0; k < 8; ++k) crc = (crc >> 1) ^ (kCrcPoly & (0u - (crc & 1)));
  }
  return crc;
}
__host__ __device__ inline uint32_t crc32(const uint8_t* p, long long n) { return ~crc_update(~0u, p, n); }
// a * b mod P in zlib's reflected representation (x^0 is bit 31)
__host__ __device__ inline uint32_t multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ kCrcPoly : b >> 1;
  }
  return p;
}
// x^(8 n) mod P
__host__ __device__ inline uint32_t x8nmodp(unsigned long long n) {
  uint32_t p = 1u << 31, sq = 1u << 23;   // x^0, x^8
  while (n) {
    if (n & 1) p = multmodp(sq, p);
    sq = multmodp(sq, sq);
    n >>= 1;
  }
  return p;
}
// crc32 of A || B from crc32(A), crc32(B) and |B| (zlib's crc32_combine)
__host__ __device__ inline uint32_t crc_combine(uint32_t ca, uint32_t cb, unsigned long long lenb) {
  return multmodp(x8nmodp(lenb), ca) ^ cb;
}

// ------------------------------------------------------------------ zlib header
// png_deflate_claim: windowBits 15, reduced while the image plus zlib's 262-byte lookahead fits in half the window
// (images of at most 16384 filtered bytes), at least 9 (zlib turns 8 into 9); then optimize_cmf lowers CINFO while the
// image fits in half the window it names.  FLEVEL is 0 under Z_RLE and Z_HUFFMAN_ONLY.
__host__ __device__ inline int window_bits(long long N) {
  int wb = 15;
  if (N <= 16384) {
    unsigned half = 1u << (wb - 1);
    while ((unsigned long long)N + 262 <= half) { half >>= 1; --wb; }
  }
  return wb < 9 ? 9 : wb;
}
__host__ __device__ inline void zlib_header(long long N, uint8_t out[2], int flevel = 0) {
  unsigned cinfo = (unsigned)window_bits(N) - 8;
  if (N <= 16384) {
    unsigned half = 1u << (cinfo + 7);
    if ((unsigned long long)N <= half) {
      do { half >>= 1; --cinfo; } while (cinfo > 0 && (unsigned long long)N <= half);
    }
  }
  const unsigned cmf = (cinfo << 4) | 8, h = (cmf << 8) | ((unsigned)flevel << 6);
  out[0] = (uint8_t)cmf;
  out[1] = (uint8_t)((h & 0xff) + 31 - h % 31);
}

// ------------------------------------------------------------------ parse (Z_RLE / Z_HUFFMAN_ONLY)
// Symbol of position p of a filtered stream f[0, N) whose run starts at s (f[s-1] != f[s] or s == 0): -1 none (inside a
// match), < 256 a literal, 256 + len - 3 a match of len bytes at distance 1.  Positions at k = p - s: 0 is the literal;
// 1 + 258 j are match starts while 3 or more bytes of the run remain from there; the last 1-2 bytes of a run whose
// remainder is short are literals.
__host__ __device__ inline int rle_symbol(const uint8_t* f, long long N, long long p, long long s) {
  const long long k = p - s;
  if (k == 0) return f[p];
  const long long q = (k - 1) % kMaxMatch, kc = p - q;   // the match start this position belongs to
  const uint8_t v = f[s];
  int m = 0;
  while (m < (q == 0 ? kMaxMatch : 3) && kc + m < N && f[kc + m] == v) ++m;
  if (m >= 3) return q == 0 ? 256 + m - 3 : -1;
  return f[p];
}
__host__ __device__ inline bool run_start(const uint8_t* f, long long p) { return p == 0 || f[p] != f[p - 1]; }

// ------------------------------------------------------------------ parse (deflate_slow, levels 4..9; DESIGN.md section 2)
// zlib's hash chains hold every earlier position with the same 3-byte hash (deflate_slow inserts the inside of its
// matches too, and only skips the last 2 bytes of the stream, which nothing later can reach), so each position's
// longest_match over the full chain and over a quarter of it (prev_length >= good_match) is a function of the
// filtered bytes alone.  prev[p] is the nearest earlier position with p's hash (0: none; position 0 is zlib's NIL).
constexpr int kTooFar = 4096, kMinLookahead = 262;
constexpr uint32_t kKwHead = 1u << 31;   // see lazy_match
__host__ __device__ inline unsigned hash3(const uint8_t* f, long long p) {
  return (((unsigned)f[p] << 10) ^ ((unsigned)f[p + 1] << 5) ^ f[p + 2]) & 0x7fff;
}
// A match as deflate_slow weighs it: (len << 16) | dist, or 0 for none or for one zlib drops (Z_FILTERED: len <= 5;
// TOO_FAR: len 3 farther than 4096).
__host__ __device__ inline uint32_t match_rec(int len, long long dist, int strategy) {
  if (len < 3 || (len <= 5 && (strategy == kZFiltered || (len == 3 && dist > kTooFar)))) return 0;
  return ((uint32_t)len << 16) | (uint32_t)dist;
}
__host__ __device__ inline int rec_len(uint32_t m) { return (int)((m >> 16) & 0x1ff); }
__host__ __device__ inline int rec_dist(uint32_t m) { return (int)(m & 0xffff); }
// Common prefix of f[a..] and f[p..] (a < p), at most lim bytes.
__host__ __device__ inline int common_len(const uint8_t* f, long long a, long long p, int lim) {
#ifdef __CUDA_ARCH__
  const uint8_t *x = f + a, *y = f + p;
  int n = 0;
  while (n + 4 <= lim) {   // 4 bytes at a time from aligned words
    const uintptr_t ux = (uintptr_t)(x + n), uy = (uintptr_t)(y + n);
    const uint32_t* wx = reinterpret_cast<const uint32_t*>(ux & ~(uintptr_t)3);
    const uint32_t* wy = reinterpret_cast<const uint32_t*>(uy & ~(uintptr_t)3);
    const uint32_t vx = __funnelshift_r(wx[0], (ux & 3) ? wx[1] : 0u, (unsigned)(ux & 3) * 8);
    const uint32_t vy = __funnelshift_r(wy[0], (uy & 3) ? wy[1] : 0u, (unsigned)(uy & 3) * 8);
    const uint32_t d = vx ^ vy;
    if (d) return n + (__ffs(d) - 1) / 8;
    n += 4;
  }
  while (n < lim && x[n] == y[n]) ++n;
  return n;
#else
  int n = 0;
  while (n < lim && f[a + n] == f[p + n]) ++n;
  return n;
#endif
}
struct MatchRec { uint32_t full, quarter; };
// longest_match at position p of an N-byte stream under level / strategy, once with max_chain candidates (full) and
// once with max_chain / 4 (quarter): the nearest candidate of the greatest length wins, the walk stops at nice_match
// (at most the lookahead), lengths stop at 258 and at the end of the stream.  The head is taken at distance <=
// MAX_DIST = w_size - 262, chain successors at < MAX_DIST.  Bytes past the end of the stream (zlib's window there holds
// zeros or stale bytes) cannot change the winner: a candidate reaching the end is already >= nice_match, so the walk
// stops at the first one.
// One head needs the parse: at T = k w_size + MAX_DIST (k >= 1) a head at k w_size is zlib's NIL when the window
// slides before T's search, which it does unless the window is full then -- that is, unless the input ends or the row
// read last ends at (k + 1) w_size - 1 (then it is none here), or the last parse step before T lies at or below the
// last row end before (k + 1) w_size minus 262 (lazy_chain checks that, flagged by kKwHead).
__host__ __device__ inline MatchRec lazy_match(const uint8_t* f, long long N, const unsigned* prev, long long p, int level,
                                               int strategy, long long rb) {
  MatchRec r{0, 0};
  const long long la = N - p;
  if (la < 3) return r;
  const long long head = prev[p], w = 1ll << window_bits(N), maxd = w - kMinLookahead;
  if (head == 0 || p - head > maxd) return r;
  uint32_t flag = 0;
  if (p - head == maxd && head % w == 0) {
    if (N < head + w || (head + w - 1) % rb == 0) return r;
    flag = kKwHead;
  }
  const LazyCfg c = lazy_cfg(level);
  const int lim = la < kMaxMatch ? (int)la : kMaxMatch, nice = c.nice < lim ? c.nice : lim, quarter = c.chain >> 2;
  const long long limit = p > maxd ? p - maxd : 0;
  int best = 2, seen = 0;
  long long bestd = 0, cur = head;
  bool have_q = false;
  for (;;) {
    if (f[cur + best] == f[p + best] && f[cur] == f[p] && f[cur + 1] == f[p + 1]) {   // longest_match's quick test
      const int len = common_len(f, cur, p, lim);
      if (len > best) {
        best = len;
        bestd = p - cur;
        if (len >= nice) break;
      }
    }
    if (++seen == quarter) { r.quarter = match_rec(best, bestd, strategy); have_q = true; }
    if (seen == c.chain) break;
    cur = prev[cur];
    if (cur <= limit) break;
  }
  r.full = match_rec(best, bestd, strategy);
  if (!have_q) r.quarter = r.full;
  r.full |= flag;
  r.quarter |= flag;
  return r;
}

// From a canonical position s (no pending match, prev_length MIN_MATCH - 1) deflate_slow's lazy steps run to the next
// canonical position: lits literals from s, then (m != 0) the match m at s + lits, then (extra) one literal at its end.
// Each lazy replacement is strictly longer, so a chain takes at most 256 steps.  rec(p) gives lazy_match's MatchRec.
struct Chain { unsigned lits; uint32_t m; bool extra; long long next; };
template <class Rec>
__host__ __device__ inline Chain lazy_chain(long long s, long long N, int level, long long rb, Rec rec) {
  const LazyCfg c = lazy_cfg(level);
  uint32_t m = rec(s).full & ~kKwHead;
  if (!m) return Chain{1, 0, false, s + 1};
  long long x = s;
  for (;;) {
    const int pl = rec_len(m);
    if (pl >= c.lazy) break;
    const MatchRec r = rec(x + 1);
    const uint32_t m2 = (pl >= c.good ? r.quarter : r.full) & ~kKwHead;
    if (rec_len(m2) <= pl) break;
    m = m2;
    ++x;
  }
  Chain ch{(unsigned)(x - s), m, false, x + rec_len(m)};
  const long long t = ch.next;   // the match is emitted by the step at x + 1; the next step is t
  if (t < N && (rec(t).full & kKwHead)) {
    const long long row_end = (t + kMinLookahead - 1) / rb * rb;   // last row end before t + 262 = (k + 1) w_size
    if (x + 1 <= row_end - kMinLookahead) { ch.extra = true; ch.next = t + 1; }   // the window slid: no search at t
  }
  return ch;
}
__host__ __device__ inline unsigned chain_symbols(const Chain& ch) { return ch.lits + (ch.m != 0) + ch.extra; }

// ------------------------------------------------------------------ deflate tables
// Length code (0..28) of a match length 3..258; zlib codes 258 as code 28 (285), not as 284 + 31.
__host__ __device__ inline int length_code(int len) {
  const int lc = len - 3;
  if (lc == 255) return 28;
  if (lc < 8) return lc;
  int xb = 1, base = 8, code = 8;
  while (lc >= base + (4 << xb)) { base += 4 << xb; code += 4; ++xb; }
  return code + ((lc - base) >> xb);
}
__host__ __device__ inline int length_extra(int code) { return code < 8 || code == 28 ? 0 : (code - 4) >> 2; }
__host__ __device__ inline int length_base(int code) {   // base of lc = len - 3
  if (code == 28) return 255;
  if (code < 8) return code;
  const int xb = length_extra(code);
  return (4 << xb) + ((code & 3) << xb);
}
// Distance code (0..29) of a distance 1..32768, its extra bits and the base of dist - 1 (zlib's d_code / base_dist)
__host__ __device__ inline int dist_code(int dist) {
  const unsigned d = (unsigned)dist - 1;
  if (d < 4) return (int)d;
  int nb = 31;
  while (!(d >> nb)) --nb;
  return 2 * nb + (int)((d >> (nb - 1)) & 1);
}
__host__ __device__ inline int dist_extra(int code) { return code < 4 ? 0 : (code - 2) >> 1; }
__host__ __device__ inline int dist_base(int code) { return code < 4 ? code : (2 + (code & 1)) << dist_extra(code); }
__host__ __device__ inline int static_llen(int n) { return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8; }
__host__ __device__ inline unsigned bit_reverse(unsigned code, int len) {
  unsigned r = 0;
  for (int i = 0; i < len; ++i) { r = (r << 1) | (code & 1); code >>= 1; }
  return r;
}
// Static literal/length code of n (bit-reversed, as zlib sends it)
__host__ __device__ inline unsigned static_lcode(int n) {
  unsigned c;
  if (n < 144) c = 0x30 + n;
  else if (n < 256) c = 0x190 + (n - 144);
  else if (n < 280) c = n - 256;
  else c = 0xc0 + (n - 280);
  return bit_reverse(c, static_llen(n));
}
__host__ __device__ inline int bl_order(int i) {
  const uint8_t t[kBLCodes] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  return t[i];
}

// ------------------------------------------------------------------ trees (zlib 1.2.11 trees.c)
struct Node { uint32_t fc; uint16_t dl; };   // fc: Freq, later Code; dl: Dad, later Len (zlib's unions)
// Frequencies of one block and the state build_tree needs.  Leaves 0..285 (literal/length), 0..29 (distance), 0..18
// (code lengths); internal nodes follow the leaves.
struct TreeWork {
  Node lt[kHeapSize], dt[2 * kDCodes + 1], bt[2 * kBLCodes + 1];
  int heap[kHeapSize];
  uint8_t depth[kHeapSize];
  uint16_t bl_count[16];
  int heap_len, heap_max, lmax, dmax, blmax;
  unsigned long long opt_len, static_len;
};

__host__ __device__ inline bool smaller(const Node* t, int n, int m, const uint8_t* depth) {
  return t[n].fc < t[m].fc || (t[n].fc == t[m].fc && depth[n] <= depth[m]);
}
__host__ __device__ inline void pqdownheap(TreeWork& s, const Node* t, int k) {
  const int v = s.heap[k];
  int j = k << 1;
  while (j <= s.heap_len) {
    if (j < s.heap_len && smaller(t, s.heap[j + 1], s.heap[j], s.depth)) j++;
    if (smaller(t, v, s.heap[j], s.depth)) break;
    s.heap[k] = s.heap[j];
    k = j;
    j <<= 1;
  }
  s.heap[k] = v;
}

// kind 0: literal/length (static lengths, extra bits from code 257), 1: distance (static length 5, zlib's extra_dbits),
// 2: bit lengths (no static tree, extra 2/3/7 for 16/17/18).
__host__ __device__ inline int tree_extra(int kind, int n) {
  if (kind == 0) return n >= 257 ? length_extra(n - 257) : 0;
  if (kind == 1) return n < 4 ? 0 : (n - 2) >> 1;
  return n == 16 ? 2 : n == 17 ? 3 : n == 18 ? 7 : 0;
}
__host__ __device__ inline int tree_static_len(int kind, int n) { return kind == 0 ? static_llen(n) : 5; }

__host__ __device__ inline void gen_bitlen(TreeWork& s, Node* tree, int max_code, int kind) {
  const int max_length = kind == 2 ? 7 : 15;
  int overflow = 0;
  for (int b = 0; b <= 15; b++) s.bl_count[b] = 0;
  tree[s.heap[s.heap_max]].dl = 0;
  int h;
  for (h = s.heap_max + 1; h < kHeapSize; h++) {
    const int n = s.heap[h];
    int bits = tree[tree[n].dl].dl + 1;
    if (bits > max_length) bits = max_length, overflow++;
    tree[n].dl = (uint16_t)bits;
    if (n > max_code) continue;
    s.bl_count[bits]++;
    const int xbits = tree_extra(kind, n);
    const unsigned long long f = tree[n].fc;
    s.opt_len += f * (unsigned)(bits + xbits);
    if (kind != 2) s.static_len += f * (unsigned)(tree_static_len(kind, n) + xbits);
  }
  if (overflow == 0) return;
  do {
    int bits = max_length - 1;
    while (s.bl_count[bits] == 0) bits--;
    s.bl_count[bits]--;
    s.bl_count[bits + 1] += 2;
    s.bl_count[max_length]--;
    overflow -= 2;
  } while (overflow > 0);
  for (int bits = max_length; bits != 0; bits--) {
    int n = s.bl_count[bits];
    while (n != 0) {
      const int m = s.heap[--h];
      if (m > max_code) continue;
      if ((unsigned)tree[m].dl != (unsigned)bits) {
        s.opt_len += ((unsigned long long)bits - tree[m].dl) * tree[m].fc;
        tree[m].dl = (uint16_t)bits;
      }
      n--;
    }
  }
}

__host__ __device__ inline void gen_codes(Node* tree, int max_code, const uint16_t* bl_count) {
  uint16_t next_code[16];
  unsigned code = 0;
  for (int bits = 1; bits <= 15; bits++) {
    code = (code + bl_count[bits - 1]) << 1;
    next_code[bits] = (uint16_t)code;
  }
  for (int n = 0; n <= max_code; n++) {
    const int len = tree[n].dl;
    if (len == 0) continue;
    tree[n].fc = bit_reverse(next_code[len]++, len);
  }
}

// build_tree over tree[0, elems): lengths in dl, codes in fc; returns max_code.
__host__ __device__ inline int build_tree(TreeWork& s, Node* tree, int elems, int kind) {
  int max_code = -1;
  s.heap_len = 0;
  s.heap_max = kHeapSize;
  for (int n = 0; n < elems; n++) {
    if (tree[n].fc != 0) {
      s.heap[++s.heap_len] = max_code = n;
      s.depth[n] = 0;
    } else {
      tree[n].dl = 0;
    }
  }
  while (s.heap_len < 2) {   // at least two codes of non-zero frequency
    const int node = s.heap[++s.heap_len] = (max_code < 2 ? ++max_code : 0);
    tree[node].fc = 1;
    s.depth[node] = 0;
    s.opt_len--;
    if (kind != 2) s.static_len -= tree_static_len(kind, node);
  }
  for (int n = s.heap_len / 2; n >= 1; n--) pqdownheap(s, tree, n);
  int node = elems;
  do {
    const int n = s.heap[1];
    s.heap[1] = s.heap[s.heap_len--];
    pqdownheap(s, tree, 1);
    const int m = s.heap[1];
    s.heap[--s.heap_max] = n;
    s.heap[--s.heap_max] = m;
    tree[node].fc = tree[n].fc + tree[m].fc;
    s.depth[node] = (uint8_t)((s.depth[n] >= s.depth[m] ? s.depth[n] : s.depth[m]) + 1);
    tree[n].dl = tree[m].dl = (uint16_t)node;
    s.heap[1] = node++;
    pqdownheap(s, tree, 1);
  } while (s.heap_len >= 2);
  s.heap[--s.heap_max] = s.heap[1];
  gen_bitlen(s, tree, max_code, kind);
  gen_codes(tree, max_code, s.bl_count);
  return max_code;
}

// scan_tree (count) / send_tree (emit) over tree lengths 0..max_code; tree[max_code + 1].dl is the 0xffff guard.
template <class Emit>
__host__ __device__ inline void walk_tree(const Node* tree, int max_code, Emit emit) {
  int prevlen = -1, nextlen = tree[0].dl, count = 0, max_count = 7, min_count = 4;
  if (nextlen == 0) max_count = 138, min_count = 3;
  for (int n = 0; n <= max_code; n++) {
    const int curlen = nextlen;
    nextlen = tree[n + 1].dl;
    if (++count < max_count && curlen == nextlen) continue;
    if (count < min_count) {
      do { emit(curlen, 0); } while (--count != 0);
    } else if (curlen != 0) {
      if (curlen != prevlen) { emit(curlen, 0); count--; }
      emit(16, count - 3);
    } else if (count <= 10) {
      emit(17, count - 3);
    } else {
      emit(18, count - 11);
    }
    count = 0;
    prevlen = curlen;
    if (nextlen == 0) max_count = 138, min_count = 3;
    else if (curlen == nextlen) max_count = 6, min_count = 3;
    else max_count = 7, min_count = 4;
  }
}

// Bits of a block header or of a whole serial stream, LSB first as zlib's send_bits.
struct BitSink {
  uint32_t* words;
  unsigned long long pos;
  __host__ __device__ void put(uint32_t v, int n) {
    for (int i = 0; i < n; ++i, ++pos)
      if ((v >> i) & 1) words[pos >> 5] |= 1u << (pos & 31);
  }
};

// One block's decision (_tr_flush_block of zlib 1.2.11), from frequencies already in w.lt / w.dt (EOB included) and the
// block's raw length.  Builds the trees, fills w.lt / w.dt with the codes of the block type chosen (the static codes
// for a static block) and returns the type; *hdr_bits: the bits after the 3-bit block header that precede the symbols
// (dynamic tree description), written to hdr when non-NULL.
// fixed (Z_FIXED): the static code unless the stored block is no larger (stored weighed against the static size).
__host__ __device__ inline int decide_block(TreeWork& w, unsigned long long stored_len, unsigned* hdr_bits, uint32_t* hdr,
                                            bool fixed = false) {
  w.opt_len = w.static_len = 0;
  w.lmax = build_tree(w, w.lt, kLCodes, 0);
  w.dmax = build_tree(w, w.dt, kDCodes, 1);
  // build_bl_tree
  for (int i = 0; i < kBLCodes; ++i) w.bt[i].fc = 0;
  w.lt[w.lmax + 1].dl = 0xffff;
  w.dt[w.dmax + 1].dl = 0xffff;
  auto count = [&](int sym, int) { w.bt[sym].fc++; };
  walk_tree(w.lt, w.lmax, count);
  walk_tree(w.dt, w.dmax, count);
  build_tree(w, w.bt, kBLCodes, 2);
  int max_blindex;
  for (max_blindex = kBLCodes - 1; max_blindex >= 3; max_blindex--)
    if (w.bt[bl_order(max_blindex)].dl != 0) break;
  w.opt_len += 3 * ((unsigned long long)max_blindex + 1) + 5 + 5 + 4;
  w.blmax = max_blindex;
  unsigned long long opt_lenb = (w.opt_len + 3 + 7) >> 3;
  const unsigned long long static_lenb = (w.static_len + 3 + 7) >> 3;
  if (static_lenb <= opt_lenb || fixed) opt_lenb = static_lenb;
  int type;
  if (stored_len + 4 <= opt_lenb) type = kStored;
  else if (static_lenb == opt_lenb) type = kStatic;
  else type = kDynamic;
  *hdr_bits = 0;
  if (type == kDynamic) {
    uint32_t scratch = 0;
    BitSink sink{hdr ? hdr : &scratch, 0};
    const bool real = hdr != nullptr;
    auto put = [&](uint32_t v, int n) {
      if (real) sink.put(v, n);
      else sink.pos += n;
    };
    put((unsigned)(w.lmax + 1 - 257), 5);
    put((unsigned)(w.dmax + 1 - 1), 5);
    put((unsigned)(max_blindex + 1 - 4), 4);
    for (int r = 0; r <= max_blindex; r++) put(w.bt[bl_order(r)].dl, 3);
    auto send = [&](int sym, int extra) {
      put(w.bt[sym].fc, w.bt[sym].dl);
      if (sym == 16) put((unsigned)extra, 2);
      else if (sym == 17) put((unsigned)extra, 3);
      else if (sym == 18) put((unsigned)extra, 7);
    };
    walk_tree(w.lt, w.lmax, send);
    walk_tree(w.dt, w.dmax, send);
    *hdr_bits = (unsigned)sink.pos;
  } else if (type == kStatic) {
    for (int n = 0; n < kLCodes; ++n) { w.lt[n].fc = static_lcode(n); w.lt[n].dl = (uint16_t)static_llen(n); }
    for (int n = 0; n < kDCodes; ++n) { w.dt[n].fc = bit_reverse(n, 5); w.dt[n].dl = 5; }
  }
  return type;
}

// Code of symbol sym (< 256 literal, else a match) under lt / dt: value (LSB first) and bit count.
__host__ __device__ inline int symbol_code(const Node* lt, const Node* dt, int sym, uint32_t* v) {
  if (sym < 256) { *v = lt[sym].fc; return lt[sym].dl; }
  const int len = sym - 256 + 3, code = length_code(len), xb = length_extra(code);
  const int ll = lt[257 + code].dl;
  uint32_t val = lt[257 + code].fc;
  int n = ll;
  if (xb) { val |= (uint32_t)(len - 3 - length_base(code)) << n; n += xb; }
  val |= dt[0].fc << n;
  *v = val;
  return n + dt[0].dl;
}
// The same for a match at any distance: at most 15 + 5 + 15 + 13 = 48 bits.
__host__ __device__ inline int symbol_code(const Node* lt, const Node* dt, int sym, int dist, uint64_t* v) {
  if (sym < 256) { *v = lt[sym].fc; return lt[sym].dl; }
  const int len = sym - 256 + 3, code = length_code(len), xb = length_extra(code);
  const int ll = lt[257 + code].dl;
  uint64_t val = lt[257 + code].fc;
  int n = ll;
  if (xb) { val |= (uint64_t)(len - 3 - length_base(code)) << n; n += xb; }
  const int dc = dist_code(dist), dx = dist_extra(dc);
  val |= (uint64_t)dt[dc].fc << n;
  n += dt[dc].dl;
  if (dx) { val |= (uint64_t)(dist - 1 - dist_base(dc)) << n; n += dx; }
  *v = val;
  return n;
}


// ------------------------------------------------------------------ device pipeline
// Per block of image i, block j at index i * maxb + j (maxb = max_blocks(N)): blocks past an image's count are idle.
struct Blk {
  unsigned raw0;                 // first filtered byte of the block (N for an empty final block)
  int type;
  unsigned hdr_bits;             // dynamic tree description bits
  unsigned long long bits;       // coded block: 3 + hdr_bits + symbols + EOB (stored blocks: computed by the layout)
  unsigned long long off;        // bit offset of the block header in the image's zlib stream
};
struct PngArgs {
  const uint8_t* img;
  long long istride, pitch;
  int W, H, n, filters, strategy;
  long long N, maxb, zwords, maxchunks;
  uint8_t* f;                    // [n][N] filtered rows
  Adler* rowad;                  // [n][H] Adler-32 sums per row
  const unsigned* runs;          // [n * N] run start (group position)
  const unsigned* symidx;        // [n * N + 1] exclusive sum of symbol starts
  uint16_t* syms;                // [n][N] symbols of image i from i * N
  unsigned* nsym;                // [n]
  Blk* blk;                      // [n * maxb]
  uint32_t* codes;               // [n * maxb][kLCodes + kDCodes] (len << 16) | code
  uint32_t* hdr;                 // [n * maxb][kHdrWords]
  uint32_t* zw;                  // [n][zwords] zlib streams
  unsigned long long* zbytes;    // [n]
  unsigned long long* sizes;     // [n] PNG stream sizes
  unsigned long long* out_off;   // [n] offsets in out
  unsigned long long* base;      // running end of the compacted output (one value)
  uint8_t* out;
  unsigned* nblk;                // [n] blocks per image
  // hash-chain parse (levels 4..9); dists NULL under Z_RLE / Z_HUFFMAN_ONLY (every match at distance 1)
  int level, flevel;
  const unsigned* prev;          // [n * N] nearest earlier position of the same hash (image-relative, 0 none)
  MatchRec* recs;                // [n * N] lazy_match per position
  unsigned* jump;                // [n * N] next canonical position (group index, kEnd past the image), then doubled
  unsigned* jump2;
  uint8_t* mark;                 // [n * N] canonical position on the parse from the image start
  unsigned* cnt;                 // [n * N + 1] symbols of each canonical position's chain
  uint16_t* dists;               // [n][N] match distances beside syms
};
constexpr int kPngThreads = 256;
constexpr unsigned kEnd = 0xffffffffu;

__device__ inline void or_bits(uint32_t* words, unsigned long long pos, uint32_t v, int n) {
  if (!v || !n) return;
  const unsigned long long sh = (unsigned long long)v << (pos & 31);
  atomicOr(words + (pos >> 5), (uint32_t)sh);
  if ((pos & 31) + n > 32) atomicOr(words + (pos >> 5) + 1, (uint32_t)(sh >> 32));
}

// Symbol at group position p, or -1.
__device__ inline int group_symbol(const PngArgs& a, unsigned p) {
  const unsigned i = (unsigned)(p / a.N), base = (unsigned)(i * a.N);
  if (a.strategy != kZRle) return a.f[p];
  return rle_symbol(a.f + base, a.N, p - base, a.runs[p] - base);
}
struct RunStartKey {   // p where a run starts (image starts included), 0 elsewhere: max-scanned into every run's start
  const uint8_t* f;
  long long N;
  __host__ __device__ unsigned operator()(unsigned p) const { return (p % N == 0 || f[p] != f[p - 1]) ? p : 0u; }
};
struct SymbolFlag {
  PngArgs a;
  unsigned total;
  __device__ unsigned operator()(unsigned p) const { return p < total && group_symbol(a, p) >= 0 ? 1u : 0u; }
};
struct MaxOp {
  __device__ unsigned operator()(unsigned x, unsigned y) const { return x > y ? x : y; }
};

__global__ void __launch_bounds__(kPngThreads) k_png_filter(PngArgs a) {
  using Reduce = cub::BlockReduce<unsigned long long, kPngThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  __shared__ int s_t;
  const int r = blockIdx.x, i = r / a.H, y = r % a.H;
  const uint8_t* cur = a.img + i * a.istride + y * a.pitch;
  const uint8_t* prev = y ? cur - a.pitch : nullptr;
  const long long pitch = 3ll * a.W, rb = pitch + 1;
  const int filters = row_filters(a.filters, a.W, a.H);
  if (filters & (filters - 1)) {
    unsigned long long sum[5];
    for (int t = 0; t < 5; ++t) {
      unsigned long long v = 0;
      if (filters & (kFilterNone << t))
        for (long long k = threadIdx.x; k < pitch; k += kPngThreads) v += filter_cost(filter_byte(t, cur, prev, k));
      sum[t] = Reduce(tmp).Sum(v);
      __syncthreads();
    }
    if (threadIdx.x == 0) s_t = choose_filter(filters, sum);
  } else if (threadIdx.x == 0) {
    unsigned long long sum[5] = {0, 0, 0, 0, 0};
    s_t = choose_filter(filters, sum);
  }
  __syncthreads();
  const int t = s_t;
  uint8_t* dst = a.f + i * a.N + y * rb;
  unsigned long long s1 = 0, s2 = 0;
  for (long long k = threadIdx.x; k < rb; k += kPngThreads) {
    const uint8_t v = k ? filter_byte(t, cur, prev, k - 1) : (uint8_t)t;
    dst[k] = v;
    s1 += v;
    s2 += (unsigned long long)(rb - k) * v;
  }
  s1 = Reduce(tmp).Sum(s1);
  __syncthreads();
  s2 = Reduce(tmp).Sum(s2);
  if (threadIdx.x == 0) a.rowad[r] = Adler{(unsigned)(s1 % kAdlerMod), (unsigned)(s2 % kAdlerMod), (unsigned long long)rb};
}

__global__ void k_png_setup(PngArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const unsigned ns = a.strategy == kZRle || a.dists ? a.symidx[(i + 1) * a.N] - a.symidx[i * a.N] : (unsigned)a.N;
  a.nsym[i] = ns;
  // deflate_slow tallies a literal left pending at the end without the block-full check: a last block of exactly 16383
  // symbols ending in the literal of the last byte is not followed by an empty one
  const bool tail_lit = a.dists && a.mark[(i + 1) * a.N - 1];
  a.nblk[i] = ns / kBlockSyms + 1 - (ns && ns % kBlockSyms == 0 && tail_lit);
  if (ns % kBlockSyms == 0 && !(ns && tail_lit)) a.blk[i * a.maxb + ns / kBlockSyms].raw0 = (unsigned)a.N;   // the empty final block
}

// ---- hash-chain parse: hash sort keys, prev[], lazy_match per position, canonical chains, their list ranking
// Sort key of group position p: image and 3-byte hash, or past every image for the last 2 bytes (never inserted).
struct HashKey {
  const uint8_t* f;
  long long N;
  unsigned n;
  __host__ __device__ unsigned operator()(unsigned p) const {
    const unsigned i = (unsigned)(p / N);
    const long long q = p - (long long)i * N;
    return q + 3 <= N ? (i << 15) | hash3(f, p) : n << 15;
  }
};
__global__ void k_png_keys(HashKey h, unsigned* key, unsigned* pos, unsigned total) {
  for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p < total; p += gridDim.x * blockDim.x) {
    key[p] = h(p);
    pos[p] = p;
  }
}
__global__ void k_png_prev(const unsigned* key, const unsigned* pos, unsigned* prev, unsigned total, long long N) {
  for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x) {
    const unsigned p = pos[k], base = (unsigned)(p / N * N);
    prev[p] = k && key[k] == key[k - 1] ? pos[k - 1] - base : 0u;
  }
}
__global__ void k_png_match(PngArgs a) {
  const unsigned total = (unsigned)(a.n * a.N);
  const long long rb = row_bytes(a.W);
  for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p < total; p += gridDim.x * blockDim.x) {
    const unsigned i = (unsigned)(p / a.N), base = (unsigned)(i * a.N);
    a.recs[p] = lazy_match(a.f + base, a.N, a.prev + base, p - base, a.level, a.strategy, rb);
  }
}
struct RecAt {
  const MatchRec* r;
  __host__ __device__ MatchRec operator()(long long p) const { return r[p]; }
};
__device__ inline Chain group_chain(const PngArgs& a, unsigned p, unsigned* base) {
  const unsigned i = (unsigned)(p / a.N);
  *base = (unsigned)(i * a.N);
  return lazy_chain(p - *base, a.N, a.level, row_bytes(a.W), RecAt{a.recs + *base});
}
// Every position's chain as if it were canonical: the next canonical position; image starts are on the parse.
__global__ void k_png_next(PngArgs a) {
  const unsigned total = (unsigned)(a.n * a.N);
  for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p < total; p += gridDim.x * blockDim.x) {
    unsigned base;
    const Chain ch = group_chain(a, p, &base);
    a.jump[p] = ch.next < a.N ? base + (unsigned)ch.next : kEnd;
    a.mark[p] = p == base;
  }
}
// One doubling round: after round r, jump is next^(2^(r+1)) and the marks hold the first 2^(r+1) positions of every
// image's parse (a mark set early in the round only adds a later position of the same parse).
__global__ void k_png_jump(const unsigned* jump, unsigned* jump2, uint8_t* mark, unsigned total) {
  for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p < total; p += gridDim.x * blockDim.x) {
    const unsigned j = jump[p];
    if (j == kEnd) { jump2[p] = kEnd; continue; }
    if (mark[p]) mark[j] = 1;
    jump2[p] = jump[j];
  }
}
__global__ void k_png_count(PngArgs a) {
  const unsigned total = (unsigned)(a.n * a.N);
  for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p <= total; p += gridDim.x * blockDim.x) {
    unsigned base, c = 0;
    if (p < total && a.mark[p]) c = chain_symbols(group_chain(a, p, &base));
    a.cnt[p] = c;
  }
}
// Symbols of every canonical position's chain at their indices, and the raw start of every block.
__global__ void k_png_lazy_compact(PngArgs a) {
  const unsigned total = (unsigned)(a.n * a.N);
  for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p < total; p += gridDim.x * blockDim.x) {
    if (!a.mark[p]) continue;
    unsigned base;
    const Chain ch = group_chain(a, p, &base);
    const unsigned i = (unsigned)(p / a.N), q = p - base;
    unsigned j = a.symidx[p] - a.symidx[base];
    auto put = [&](unsigned at, int v, int d) {
      a.syms[base + j] = (uint16_t)v;
      a.dists[base + j] = (uint16_t)d;
      if (j % kBlockSyms == 0) a.blk[i * a.maxb + j / kBlockSyms].raw0 = at;
      ++j;
    };
    for (unsigned k = 0; k < ch.lits; ++k) put(q + k, a.f[p + k], 0);
    if (ch.m) {
      const int len = rec_len(ch.m);
      put(q + ch.lits, 256 + len - 3, rec_dist(ch.m));
      if (ch.extra) put(q + ch.lits + len, a.f[p + ch.lits + len], 0);
    }
  }
}

__global__ void k_png_compact(PngArgs a) {
  const unsigned total = (unsigned)(a.n * a.N);
  for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p < total; p += gridDim.x * blockDim.x) {
    const int v = group_symbol(a, p);
    if (v < 0) continue;
    const unsigned i = (unsigned)(p / a.N), base = (unsigned)(i * a.N);
    const unsigned j = a.strategy == kZRle ? a.symidx[p] - a.symidx[base] : p - base;
    a.syms[base + j] = (uint16_t)v;
    if (j % kBlockSyms == 0) a.blk[i * a.maxb + j / kBlockSyms].raw0 = p - base;
  }
}

__device__ inline bool block_range(const PngArgs& a, long long b, int* i, unsigned* s0, unsigned* cnt, bool* last) {
  *i = (int)(b / a.maxb);
  const unsigned j = (unsigned)(b % a.maxb), ns = a.nsym[*i], nblk = a.nblk[*i];
  if (j >= nblk) return false;
  *s0 = j * kBlockSyms;
  *cnt = min((unsigned)kBlockSyms, ns - *s0);
  *last = j == nblk - 1;
  return true;
}

__global__ void __launch_bounds__(kPngThreads) k_png_tree(PngArgs a) {
  using Reduce = cub::BlockReduce<unsigned long long, kPngThreads>;
  __shared__ TreeWork w;
  __shared__ typename Reduce::TempStorage tmp;
  const long long b = blockIdx.x;
  int i;
  unsigned s0, cnt;
  bool last;
  if (!block_range(a, b, &i, &s0, &cnt, &last)) return;
  for (int k = threadIdx.x; k < kHeapSize; k += kPngThreads) w.lt[k].fc = 0;
  for (int k = threadIdx.x; k < 2 * kDCodes + 1; k += kPngThreads) w.dt[k].fc = 0;
  __syncthreads();
  const uint16_t* sy = a.syms + i * a.N + s0;
  const uint16_t* dy = a.dists ? a.dists + i * a.N + s0 : nullptr;
  for (unsigned k = threadIdx.x; k < cnt; k += kPngThreads) {
    const int v = sy[k];
    if (v < 256) atomicAdd(&w.lt[v].fc, 1u);
    else { atomicAdd(&w.lt[257 + length_code(v - 256 + 3)].fc, 1u); atomicAdd(&w.dt[dy ? dist_code(dy[k]) : 0].fc, 1u); }
  }
  __syncthreads();
  __shared__ int s_type;
  __shared__ unsigned s_hb;
  if (threadIdx.x == 0) {
    w.lt[kEndBlock].fc = 1;
    uint32_t* hdr = a.hdr + b * kHdrWords;
    for (int k = 0; k < kHdrWords; ++k) hdr[k] = 0;
    const unsigned raw0 = a.blk[b].raw0, raw1 = last ? (unsigned)a.N : a.blk[b + 1].raw0;
    s_type = decide_block(w, raw1 - raw0, &s_hb, hdr, a.strategy == kZFixed);
  }
  __syncthreads();
  if (s_type == kStored) {
    if (threadIdx.x == 0) { a.blk[b].type = kStored; a.blk[b].hdr_bits = 0; a.blk[b].bits = 0; }
    return;
  }
  uint32_t* codes = a.codes + b * (kLCodes + kDCodes);
  for (int k = threadIdx.x; k < kLCodes; k += kPngThreads) codes[k] = ((uint32_t)w.lt[k].dl << 16) | w.lt[k].fc;
  for (int k = threadIdx.x; k < kDCodes; k += kPngThreads) codes[kLCodes + k] = ((uint32_t)w.dt[k].dl << 16) | w.dt[k].fc;
  unsigned long long bits = 0;
  for (unsigned k = threadIdx.x; k < cnt; k += kPngThreads) {
    uint64_t v;
    bits += symbol_code(w.lt, w.dt, sy[k], dy ? dy[k] : 1, &v);
  }
  bits = Reduce(tmp).Sum(bits);
  if (threadIdx.x == 0) {
    a.blk[b].type = s_type;
    a.blk[b].hdr_bits = s_hb;
    a.blk[b].bits = 3 + s_hb + bits + w.lt[kEndBlock].dl;
  }
}

__global__ void k_png_layout(PngArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const unsigned nblk = a.nblk[i];
  unsigned long long pos = 16;
  for (unsigned j = 0; j < nblk; ++j) {
    Blk& bk = a.blk[i * a.maxb + j];
    bk.off = pos;
    if (bk.type == kStored) {
      const unsigned raw1 = j + 1 < nblk ? a.blk[i * a.maxb + j + 1].raw0 : (unsigned)a.N;
      pos = ((pos + 3 + 7) & ~7ull) + 32 + 8ull * (raw1 - bk.raw0);
    } else {
      pos += bk.bits;
    }
  }
  pos = (pos + 7) & ~7ull;
  const unsigned long long zb = pos / 8 + 4;
  uint8_t* z = reinterpret_cast<uint8_t*>(a.zw + i * a.zwords);
  zlib_header(a.N, z, a.flevel);
  Adler ad{0, 0, 0};
  for (int y = 0; y < a.H; ++y) ad = adler_cat(ad, a.rowad[(long long)i * a.H + y]);
  const uint32_t v = adler_final(ad);
  for (int k = 0; k < 4; ++k) z[zb - 4 + k] = (uint8_t)(v >> (24 - 8 * k));
  a.zbytes[i] = zb;
  a.sizes[i] = (unsigned long long)png_bytes((long long)zb);
}

__global__ void k_png_offsets(PngArgs a) {
  unsigned long long o = *a.base;
  for (int i = 0; i < a.n; ++i) { a.out_off[i] = o; o += a.sizes[i]; }
  *a.base = o;
}

__global__ void __launch_bounds__(kPngThreads) k_png_pack(PngArgs a) {
  using Scan = cub::BlockScan<unsigned, kPngThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ Node lt[kLCodes], dt[kDCodes];
  __shared__ unsigned long long s_pos;
  const long long b = blockIdx.x;
  int i;
  unsigned s0, cnt;
  bool last;
  if (!block_range(a, b, &i, &s0, &cnt, &last)) return;
  const Blk bk = a.blk[b];
  uint32_t* words = a.zw + i * a.zwords;
  if (threadIdx.x == 0) or_bits(words, bk.off, (uint32_t)(bk.type << 1) + last, 3);
  if (bk.type == kStored) {
    const unsigned raw1 = last ? (unsigned)a.N : a.blk[b + 1].raw0, len = raw1 - bk.raw0;
    const unsigned long long at = ((bk.off + 3 + 7) & ~7ull) >> 3;
    const uint8_t* src = a.f + i * a.N + bk.raw0;
    for (unsigned k = threadIdx.x; k < len + 4; k += kPngThreads) {
      const unsigned v = k == 0 ? len & 255 : k == 1 ? len >> 8 : k == 2 ? ~len & 255 : k == 3 ? (~len >> 8) & 255 : src[k - 4];
      or_bits(words, (at + k) * 8, v, 8);
    }
    return;
  }
  const uint32_t* codes = a.codes + b * (kLCodes + kDCodes);
  for (int k = threadIdx.x; k < kLCodes; k += kPngThreads) { lt[k].fc = codes[k] & 0xffff; lt[k].dl = (uint16_t)(codes[k] >> 16); }
  for (int k = threadIdx.x; k < kDCodes; k += kPngThreads) {
    dt[k].fc = codes[kLCodes + k] & 0xffff; dt[k].dl = (uint16_t)(codes[kLCodes + k] >> 16);
  }
  const uint32_t* hdr = a.hdr + b * kHdrWords;
  for (unsigned k = threadIdx.x; k * 32 < bk.hdr_bits; k += kPngThreads)
    or_bits(words, bk.off + 3 + 32ull * k, hdr[k], (int)min(32u, bk.hdr_bits - 32 * k));
  if (threadIdx.x == 0) s_pos = bk.off + 3 + bk.hdr_bits;
  __syncthreads();
  const uint16_t* sy = a.syms + i * a.N + s0;
  const uint16_t* dy = a.dists ? a.dists + i * a.N + s0 : nullptr;
  for (unsigned k0 = 0; k0 < cnt; k0 += kPngThreads) {
    const unsigned k = k0 + threadIdx.x;
    uint64_t v = 0;
    const unsigned n = k < cnt ? (unsigned)symbol_code(lt, dt, sy[k], dy ? dy[k] : 1, &v) : 0u;
    unsigned off, tile;
    Scan(tmp).ExclusiveSum(n, off, tile);
    const unsigned long long p0 = s_pos;
    or_bits(words, p0 + off, (uint32_t)v, (int)min(n, 32u));
    if (n > 32) or_bits(words, p0 + off + 32, (uint32_t)(v >> 32), (int)n - 32);
    __syncthreads();
    if (threadIdx.x == 0) s_pos = p0 + tile;
    __syncthreads();
  }
  if (threadIdx.x == 0) or_bits(words, s_pos, lt[kEndBlock].fc, lt[kEndBlock].dl);
}

// One warp per IDAT chunk of image i: the chunk's bytes into the compacted PNG, its CRC-32 from the lanes' CRCs.
__global__ void __launch_bounds__(kPngThreads) k_png_frame(PngArgs a) {
  const long long wid = ((long long)blockIdx.x * kPngThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= a.n * a.maxchunks) return;
  const int i = (int)(wid / a.maxchunks);
  const long long c = wid % a.maxchunks;
  const unsigned long long zb = a.zbytes[i], nch = (unsigned long long)idat_chunks((long long)zb);
  if ((unsigned long long)c >= nch) return;
  uint8_t* o = a.out + a.out_off[i];
  const uint8_t* z = reinterpret_cast<const uint8_t*>(a.zw + i * a.zwords) + c * kIdatBytes;
  const unsigned len = (unsigned)min((unsigned long long)kIdatBytes, zb - c * kIdatBytes);
  uint8_t* dst = o + kPngHead + c * (kIdatBytes + 12);
  const unsigned seg = (len + 31) / 32, b0 = min(len, lane * seg), b1 = min(len, b0 + seg);
  for (unsigned k = b0; k < b1; ++k) dst[8 + k] = z[k];
  uint32_t crc = crc32(z + b0, b1 - b0);
  unsigned long long n = b1 - b0;
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t oc = __shfl_down_sync(0xffffffffu, crc, d);
    const unsigned long long on = __shfl_down_sync(0xffffffffu, n, d);
    if ((lane & (2 * d - 1)) == 0) { crc = crc_combine(crc, oc, on); n += on; }
  }
  if (lane == 0) {
    const uint8_t type[4] = {'I', 'D', 'A', 'T'};
    const uint32_t cc = crc_combine(crc32(type, 4), crc, len);
    for (int k = 0; k < 4; ++k) { dst[k] = (uint8_t)(len >> (24 - 8 * k)); dst[4 + k] = type[k]; dst[8 + len + k] = (uint8_t)(cc >> (24 - 8 * k)); }
    if (c == 0) {
      const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
      for (int k = 0; k < 8; ++k) o[k] = sig[k];
      uint8_t h[17] = {0, 0, 0, 13, 'I', 'H', 'D', 'R',
                       (uint8_t)(a.W >> 24), (uint8_t)(a.W >> 16), (uint8_t)(a.W >> 8), (uint8_t)a.W,
                       (uint8_t)(a.H >> 24), (uint8_t)(a.H >> 16), (uint8_t)(a.H >> 8), (uint8_t)a.H, 8};
      for (int k = 0; k < 17; ++k) o[8 + k] = h[k];
      const uint8_t rest[4] = {2, 0, 0, 0};
      for (int k = 0; k < 4; ++k) o[25 + k] = rest[k];
      const uint32_t hc = crc32(o + 12, 17);
      for (int k = 0; k < 4; ++k) o[29 + k] = (uint8_t)(hc >> (24 - 8 * k));
    }
    if ((unsigned long long)c == nch - 1) {
      const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xae, 0x42, 0x60, 0x82};
      uint8_t* e = o + kPngHead + zb + 12 * nch;
      for (int k = 0; k < 12; ++k) e[k] = iend[k];
    }
  }
}

}  // namespace png
}  // namespace bevk
