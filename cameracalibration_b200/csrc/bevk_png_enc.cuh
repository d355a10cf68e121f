// bevk_png_enc.cuh -- PNG encoder on the device (sm_90a), byte-identical to cv2.imwrite / cv2.imencode('.png') for
// 8-bit BGR images under cv2's default settings and its Z_RLE / Z_HUFFMAN_ONLY strategies.
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
inline int normalise(const int* p, int n, Opts* o) {
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
  if (bilevel || zbuf || o->level == 0 || (strategy != kZRle && strategy != kZHuffmanOnly)) return 2;
  return 0;
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
__host__ __device__ inline void zlib_header(long long N, uint8_t out[2]) {
  unsigned cinfo = (unsigned)window_bits(N) - 8;
  if (N <= 16384) {
    unsigned half = 1u << (cinfo + 7);
    if ((unsigned long long)N <= half) {
      do { half >>= 1; --cinfo; } while (cinfo > 0 && (unsigned long long)N <= half);
    }
  }
  const unsigned cmf = (cinfo << 4) | 8;
  out[0] = (uint8_t)cmf;
  out[1] = (uint8_t)(31 - (cmf << 8) % 31);
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
__host__ __device__ inline int decide_block(TreeWork& w, unsigned long long stored_len, unsigned* hdr_bits, uint32_t* hdr) {
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
  if (static_lenb <= opt_lenb) opt_lenb = static_lenb;
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
};
constexpr int kPngThreads = 256;

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
  const unsigned ns = a.strategy == kZRle ? a.symidx[(i + 1) * a.N] - a.symidx[i * a.N] : (unsigned)a.N;
  a.nsym[i] = ns;
  if (ns % kBlockSyms == 0) a.blk[i * a.maxb + ns / kBlockSyms].raw0 = (unsigned)a.N;   // the empty final block
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
  const unsigned j = (unsigned)(b % a.maxb), ns = a.nsym[*i], nblk = ns / kBlockSyms + 1;
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
  for (unsigned k = threadIdx.x; k < cnt; k += kPngThreads) {
    const int v = sy[k];
    if (v < 256) atomicAdd(&w.lt[v].fc, 1u);
    else { atomicAdd(&w.lt[257 + length_code(v - 256 + 3)].fc, 1u); atomicAdd(&w.dt[0].fc, 1u); }
  }
  __syncthreads();
  __shared__ int s_type;
  __shared__ unsigned s_hb;
  if (threadIdx.x == 0) {
    w.lt[kEndBlock].fc = 1;
    uint32_t* hdr = a.hdr + b * kHdrWords;
    for (int k = 0; k < kHdrWords; ++k) hdr[k] = 0;
    const unsigned raw0 = a.blk[b].raw0, raw1 = last ? (unsigned)a.N : a.blk[b + 1].raw0;
    s_type = decide_block(w, raw1 - raw0, &s_hb, hdr);
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
    uint32_t v;
    bits += symbol_code(w.lt, w.dt, sy[k], &v);
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
  const unsigned ns = a.nsym[i], nblk = ns / kBlockSyms + 1;
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
  zlib_header(a.N, z);
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
  for (unsigned k0 = 0; k0 < cnt; k0 += kPngThreads) {
    const unsigned k = k0 + threadIdx.x;
    uint32_t v = 0;
    const unsigned n = k < cnt ? (unsigned)symbol_code(lt, dt, sy[k], &v) : 0u;
    unsigned off, tile;
    Scan(tmp).ExclusiveSum(n, off, tile);
    const unsigned long long p0 = s_pos;
    or_bits(words, p0 + off, v, (int)n);
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
