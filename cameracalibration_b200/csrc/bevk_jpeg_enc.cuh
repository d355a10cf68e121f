// bevk_jpeg_enc.cuh -- baseline JPEG encoder on the device (sm_90a), byte-identical to cv2.imwrite / cv2.imencode.
//
// cv2 writes JPEG through libjpeg-turbo's baseline compressor: fixed Annex K Huffman tables, 4:2:0 by default, islow
// integer DCT, no restart markers.  That path is integer arithmetic end to end with no data-dependent choices, so the
// stream can be reproduced byte for byte:
//   colour     Y/Cb/Cr from BGR with libjpeg's 16-bit fixed-point constants (jccolor.c)
//   sampling   luma h x v per MCU (IMWRITE_JPEG_SAMPLING_FACTOR: 1x1, 2x1, 1x2, 2x2, 4x1), Cb and Cr 1x1; an MCU is
//              8h x 8v pixels and h*v + 2 blocks (Y row-major, Cb, Cr).  Chroma is the mean of h x v pixels:
//              1x1 copy, 2x1 (a + b + 0/1) >> 1, 2x2 (sum + 1/2) >> 2 (biases alternating along the row), 1x2 and
//              4x1 (sum + n/2) / n (jcsample.c fullsize / h2v1 / h2v2 / int_downsample)
//   edges      luma replicated to whole blocks; chroma sources replicated to 8h*ceil(W/8h) columns, source rows
//              clamped to H-1, chroma rows past ceil(H/v) repeat the last chroma row (jcsample.c + jcprepct.c)
//   dummies    luma blocks outside ceil(W/8) x ceil(H/8) inside an MCU: AC 0, DC = quantised DC of the block before
//              it in the MCU (jccoefct.c); chroma blocks are never dummies
//   quality    IMWRITE_JPEG_LUMA_QUALITY / CHROMA_QUALITY give each table its own quality (normalise())
//   restart    IMWRITE_JPEG_RST_INTERVAL: DRI, DC predictors reset per interval, each interval 1-padded to a byte and
//              followed by RSTn (n cycling 0..7) except the last
//   optimise   IMWRITE_JPEG_OPTIMIZE: per-image tables from the symbol counts (gen_optimal_table), DHTs per image
//   FDCT       jfdctint.c (CONST_BITS 13, PASS1_BITS 2), output scaled by 8; quantised as sign * ((|c| + d/2) / d)
//   entropy    DC differences per component in scan order, AC (run, size) with ZRL / EOB, 0xFF stuffing, 1-bit pad
// Everything per block is __host__ __device__: tests/host/jpeg_enc.cu runs the same functions serially over a whole
// image and compares the stream with live cv2.imencode.
//
// Grey and BGRA images (cv2.imencode of [H][W] / [H][W][1] and [H][W][4]):
//   grey       one component (JCS_GRAYSCALE): an MCU is one 8x8 block, ceil(W/8) x ceil(H/8) blocks in raster order,
//              edges replicated, the sample is the byte itself (libjpeg's grayscale pass-through); only quantisation
//              table 0 at the luma quality and DHT DC0 / AC0; SAMPLING_FACTOR does not reach the stream (a one-component
//              scan is non-interleaved); the restart interval counts blocks.  Header: kGreyHeaderBytes
//   BGRA       cv2 drops alpha: the colour samples are read with a 4-byte pixel stride and the stream is the BGR one
//
// The default (no parameters) is the 4:2:0 instance: geom(W, H), make_tables(q, ...), make_header(W, H, q, ...) and
// encode_bound(W, H) are the general forms at Opts{2, 2, q, q}.
//
// Device pipeline for n equal-sized images (bevk_api.cu: jpeg_enqueue, then enc_collect copies the streams out):
//   k_jpeg_blocks  one thread per 8x8 block: BGR -> samples with the edge rules, FDCT, quantise, int16 zigzag
//                  coefficients (128 B per block) and the block's AC bit count
//   (k_jpeg_blocks, k_jpeg_dc and k_jpeg_pack are instantiated per luma sampling HY x VY: the MCU layout is constant;
//    grey images take the NC = 1 instances, one block per MCU, and k_jpeg_blocks loads C = 1, 3 or 4 bytes per pixel)
//   k_jpeg_dc      DC differences (dummy blocks resolved), bits per block
//   scan           exclusive sum of bits per block (CUB): every block's bit offset in its image's stream
//   k_jpeg_zero    clears the used words of each image's bit buffer
//   k_jpeg_pack    every block writes its codes at its offset; words shared with neighbours take atomicOr
//   k_jpeg_ffcount 0xFF bytes per 128-byte chunk; scan (CUB); k_jpeg_layout: stream sizes, compact offsets, header + EOI
//   k_jpeg_stuff   chunk copy with a 0x00 after every 0xFF, into the compacted output (and RSTn at interval starts)
// OPTIMIZE adds k_jpeg_count (symbol counts), k_jpeg_huff (tables, codes, per-image headers) and k_jpeg_bits (bits per
// block under them) before the scan; RST_INTERVAL adds k_jpeg_intervals (padded bits per interval) and its scan after it.
//
// The encoder reads finished images only: BEV canvases under BALANCE (bevk_bev_run_to_jpeg / bevk_bev_frames_to_jpeg)
// get colour balance and the car from k_gain before k_jpeg_blocks loads them.  Applying the gains in the load stage
// instead was measured slower on H100 than k_gain followed by this encoder (DESIGN.md section 11).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <type_traits>

namespace bevk {
namespace jpeg {

constexpr int kHeaderBytes = 623;             // SOI + APP0 + 2 DQT + SOF0 + 4 DHT + SOS
constexpr int kMaxBlockBits = 11 + 11 + 63 * (16 + 10);   // DC code + value, 63 AC codes (<= 16 bits) + values (<= 10)
constexpr int kMaxBlockBitsOpt = 16 + 11 + 63 * (16 + 10); // the same with optimised tables: a DC code can take 16 bits
constexpr int kHeaderPrefix = 177;            // SOI + APP0 + 2 DQT + SOF0: the header bytes before the DHTs
constexpr int kAnnexKDhtBytes = 432;          // the four Annex K DHT segments (DC 33 + AC 183 bytes per table)
constexpr int kDriBytes = 6;                  // DRI segment, written when restart intervals are on
constexpr int kMaxHeaderBytes = kHeaderBytes + kDriBytes;   // optimal DHTs are never longer than Annex K's
constexpr int kChunk = 128;                   // bytes per thread of the stuffing pass
constexpr int kMaxDim = 65500;                // JPEG_MAX_DIMENSION of libjpeg
constexpr int kGreyHeaderPrefix = 102;        // grey: SOI + APP0 + DQT 0 + SOF0 with one component
constexpr int kGreyAnnexKDhtBytes = 216;      // grey: DHT DC0 + AC0
constexpr int kGreyHeaderBytes = 328;         // grey: prefix + DHT DC0 AC0 + SOS with one component

// Per-quality tables the kernels read (built on the host, copied into shared memory per CTA).
struct Tables {
  uint32_t ac[2][256];     // (length << 16) | code per AC symbol (run << 4 | size); [0] luma, [1] chroma
  uint32_t dc[2][12];      // the same per DC category
  uint16_t qdiv[2][64];    // 8 * quantisation step, natural order
  uint8_t zz[64];          // zigzag index -> natural index
};

// ------------------------------------------------------------------ geometry
struct Geom {
  int W, H, mcux, mcuy, wb, hb;   // MCUs across / down, luma blocks across / down that hold image samples
  int hy, vy;                     // luma blocks per MCU across / down
  int nc;                         // components: 3 (YCbCr) or 1 (grey: hy = vy = 1)
};
__host__ __device__ inline Geom geom(int W, int H, int hy, int vy) {
  Geom g;
  g.W = W; g.H = H;
  g.mcux = (W + 8 * hy - 1) / (8 * hy); g.mcuy = (H + 8 * vy - 1) / (8 * vy);
  g.wb = (W + 7) / 8; g.hb = (H + 7) / 8;
  g.hy = hy; g.vy = vy;
  g.nc = 3;
  return g;
}
__host__ __device__ inline Geom geom(int W, int H) { return geom(W, H, 2, 2); }
// blocks per MCU: the hy*vy luma blocks, then Cb and Cr (none for grey)
__host__ __device__ inline int mcu_blocks(const Geom& g) { return g.hy * g.vy + (g.nc == 1 ? 0 : 2); }
// blocks of one image in scan order: MCU raster, per MCU the hy*vy luma blocks row-major, Cb, Cr
__host__ __device__ inline long long blocks_per_image(const Geom& g) { return (long long)g.mcux * g.mcuy * mcu_blocks(g); }

// luma block k (0..HY*VY-1) of MCU (mx, my) lies outside the image's blocks: a dummy (AC 0, DC of the block before it)
template <int HY, int VY>
__host__ __device__ inline bool is_dummy_s(const Geom& g, int mx, int my, int k) {
  return k < HY * VY && (HY * mx + k % HY >= g.wb || VY * my + k / HY >= g.hb);
}
__host__ __device__ inline bool is_dummy(const Geom& g, int mx, int my, int k) {
  return k < g.hy * g.vy && (g.hy * mx + k % g.hy >= g.wb || g.vy * my + k / g.hy >= g.hb);
}

// cv2's IMWRITE_JPEG_QUALITY clamp to [0, 100], then libjpeg's jpeg_quality_scaling maps 0 to 1
__host__ __device__ inline int clamp_quality(int q) { return q <= 0 ? 1 : q > 100 ? 100 : q; }

// ------------------------------------------------------------------ colour conversion and sampling (jccolor.c, jcsample.c)
__host__ __device__ inline int ycc_y(int b, int g, int r) { return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16; }
__host__ __device__ inline int ycc_cb(int b, int g, int r) { return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16; }
__host__ __device__ inline int ycc_cr(int b, int g, int r) { return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16; }

__host__ __device__ inline int ld8(const uint8_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// pixel (x, y) of a BGR (C 3) or BGRA (C 4) image with rows pitch bytes apart
template <int C = 3>
__host__ __device__ inline void bgr_at(const uint8_t* img, long long pitch, int x, int y, int& b, int& g, int& r) {
  const uint8_t* p = img + y * pitch + (long long)C * x;
  b = ld8(p); g = ld8(p + 1); r = ld8(p + 2);
}

// Sample (r, c) of block k of MCU (mx, my): luma (k < HY*VY) or Cb (k == HY*VY) / Cr after HY x VY subsampling, of an
// image of C channels (1 grey: the byte itself, HY = VY = 1; 3 BGR; 4 BGRA, alpha unread).
template <int HY, int VY, int C = 3>
__host__ __device__ inline int block_sample(const uint8_t* img, long long pitch, const Geom& g, int mx, int my, int k, int r, int c) {
  constexpr int NY = HY * VY;
  if (k < NY) {
    int x = (HY * mx + k % HY) * 8 + c, y = (VY * my + k / HY) * 8 + r;
    x = x < g.W ? x : g.W - 1;
    y = y < g.H ? y : g.H - 1;
    if constexpr (C == 1) return ld8(img + y * pitch + x);
    int b, gg, rr;
    bgr_at<C>(img, pitch, x, y, b, gg, rr);
    return ycc_y(b, gg, rr);
  }
  const int last = (g.H + VY - 1) / VY - 1;              // chroma rows past ceil(H/VY) repeat the last one
  int cy = my * 8 + r;
  cy = cy < last ? cy : last;
  const int cx = mx * 8 + c;
  int s = 0;
  for (int i = 0; i < VY; ++i) {
    const int y = VY * cy + i < g.H ? VY * cy + i : g.H - 1;
    for (int j = 0; j < HY; ++j) {
      const int x = HY * cx + j < g.W ? HY * cx + j : g.W - 1;
      int b, gg, rr;
      bgr_at<C>(img, pitch, x, y, b, gg, rr);
      s += k == NY ? ycc_cb(b, gg, rr) : ycc_cr(b, gg, rr);
    }
  }
  if (NY == 1) return s;                                 // fullsize_downsample
  if (HY == 2 && VY == 1) return (s + (c & 1)) >> 1;     // h2v1_downsample's alternating bias 0, 1
  if (HY == 2 && VY == 2) return (s + 1 + (c & 1)) >> 2; // h2v2_downsample's alternating bias 1, 2
  return (s + NY / 2) / NY;                              // int_downsample
}

// Call f(integral_constant<HY>, integral_constant<VY>) for one of the five luma samplings cv2 writes.
template <class F>
inline auto with_sampling(int hy, int vy, F&& f) {
  using std::integral_constant;
  if (hy == 1 && vy == 1) return f(integral_constant<int, 1>{}, integral_constant<int, 1>{});
  if (hy == 2 && vy == 1) return f(integral_constant<int, 2>{}, integral_constant<int, 1>{});
  if (hy == 1 && vy == 2) return f(integral_constant<int, 1>{}, integral_constant<int, 2>{});
  if (hy == 4 && vy == 1) return f(integral_constant<int, 4>{}, integral_constant<int, 1>{});
  return f(integral_constant<int, 2>{}, integral_constant<int, 2>{});
}

// The 64 samples of a block, level-shifted (sample - 128), natural order.
template <int HY, int VY, int C = 3>
__host__ __device__ inline void load_block_s(const uint8_t* img, long long pitch, const Geom& g, int mx, int my, int k, int* d) {
  for (int r = 0; r < 8; ++r)
    for (int c = 0; c < 8; ++c) d[r * 8 + c] = block_sample<HY, VY, C>(img, pitch, g, mx, my, k, r, c) - 128;
}
inline void load_block(const uint8_t* img, long long pitch, const Geom& g, int mx, int my, int k, int* d) {
  with_sampling(g.hy, g.vy, [&](auto hy, auto vy) { load_block_s<hy(), vy()>(img, pitch, g, mx, my, k, d); });
}
// the same for an image of `channels` (1, 3 or 4) channels
inline void load_block(const uint8_t* img, long long pitch, const Geom& g, int channels, int mx, int my, int k, int* d) {
  if (channels == 1) return load_block_s<1, 1, 1>(img, pitch, g, mx, my, k, d);
  if (channels == 3) return load_block(img, pitch, g, mx, my, k, d);
  with_sampling(g.hy, g.vy, [&](auto hy, auto vy) { load_block_s<hy(), vy(), 4>(img, pitch, g, mx, my, k, d); });
}

// ------------------------------------------------------------------ forward DCT (jfdctint.c, islow) and quantisation
__host__ __device__ inline int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

template <int PASS>
__host__ __device__ inline void fdct_line(int* p, int step) {
  constexpr int CB = 13, P1 = 2, SH = PASS == 0 ? CB - P1 : CB + P1;
  const int t0 = p[0] + p[7 * step], t7 = p[0] - p[7 * step];
  const int t1 = p[step] + p[6 * step], t6 = p[step] - p[6 * step];
  const int t2 = p[2 * step] + p[5 * step], t5 = p[2 * step] - p[5 * step];
  const int t3 = p[3 * step] + p[4 * step], t4 = p[3 * step] - p[4 * step];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  if (PASS == 0) {
    p[0] = (t10 + t11) * (1 << P1);
    p[4 * step] = (t10 - t11) * (1 << P1);
  } else {
    p[0] = descale(t10 + t11, P1);
    p[4 * step] = descale(t10 - t11, P1);
  }
  int z1 = (t12 + t13) * 4433;
  p[2 * step] = descale(z1 + t13 * 6270, SH);
  p[6 * step] = descale(z1 - t12 * 15137, SH);
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * 9633;
  const int a4 = t4 * 2446, a5 = t5 * 16819, a6 = t6 * 25172, a7 = t7 * 12299;
  z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;
  z3 += z5; z4 += z5;
  p[7 * step] = descale(a4 + z1 + z3, SH);
  p[5 * step] = descale(a5 + z2 + z4, SH);
  p[3 * step] = descale(a6 + z2 + z3, SH);
  p[step] = descale(a7 + z1 + z4, SH);
}

// In place on 64 level-shifted samples (natural order); the result is the DCT scaled by 8.
__host__ __device__ inline void fdct_islow(int* d) {
  for (int r = 0; r < 8; ++r) fdct_line<0>(d + 8 * r, 1);
  for (int c = 0; c < 8; ++c) fdct_line<1>(d + c, 8);
}

// In place, natural order: sign(c) * ((|c| + d/2) / d) with d = 8 * Q[k]
__host__ __device__ inline void quantise(int* d, const uint16_t* qdiv) {
  for (int k = 0; k < 64; ++k) {
    const int q = qdiv[k], v = d[k];
    const int a = ((v < 0 ? -v : v) + (q >> 1)) / q;
    d[k] = v < 0 ? -a : a;
  }
}

// ------------------------------------------------------------------ Huffman coding of one block
__host__ __device__ inline int nbits(int a) {   // size category of |v| = a
#ifdef __CUDA_ARCH__
  return 32 - __clz(a);
#else
  return a ? 32 - __builtin_clz((unsigned)a) : 0;
#endif
}

template <class Sink>
__host__ __device__ inline void put_sym(Sink& s, uint32_t e) { s.put(e & 0xffffu, (int)(e >> 16)); }

template <class Sink>
__host__ __device__ inline void emit_dc(int diff, const uint32_t* dc, Sink& s) {
  const int n = nbits(diff < 0 ? -diff : diff);
  put_sym(s, dc[n]);
  if (n) s.put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1u), n);
}

// coefficient accessors for emit_ac: quantised natural-order ints read through the zigzag table, or stored zigzag int16
struct ZigzagOf {
  const int* d;
  const uint8_t* zz;
  __host__ __device__ int operator()(int j) const { return d[zz[j]]; }
};
struct Zigzag16 {
  const int16_t* c;
  __host__ __device__ int operator()(int j) const {
#ifdef __CUDA_ARCH__
    return __ldg(c + j);
#else
    return c[j];
#endif
  }
};

// get(i) = zigzag coefficient i (1..63)
template <class Get, class Sink>
__host__ __device__ inline void emit_ac(const Get& get, const uint32_t* ac, Sink& s) {
  int run = 0;
  for (int i = 1; i < 64; ++i) {
    const int v = get(i);
    if (v == 0) { ++run; continue; }
    for (; run > 15; run -= 16) put_sym(s, ac[0xf0]);     // ZRL
    const int n = nbits(v < 0 ? -v : v);
    put_sym(s, ac[(run << 4) | n]);
    s.put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << n) - 1u), n);
    run = 0;
  }
  if (run) put_sym(s, ac[0x00]);                          // EOB
}

// f(table class, symbol) for every Huffman symbol of one block: class 0 the DC category of diff, class 1 the AC
// (run, size) symbols with ZRL and EOB -- what emit_dc / emit_ac code, and what libjpeg's htest_one_block counts.
template <class Get, class F>
__host__ __device__ inline void block_symbols(int diff, const Get& get, F&& f) {
  f(0, nbits(diff < 0 ? -diff : diff));
  int run = 0;
  for (int i = 1; i < 64; ++i) {
    const int v = get(i);
    if (v == 0) { ++run; continue; }
    for (; run > 15; run -= 16) f(1, 0xf0);
    f(1, (run << 4) | nbits(v < 0 ? -v : v));
    run = 0;
  }
  if (run) f(1, 0x00);
}

struct BitCount {
  unsigned n = 0;
  __host__ __device__ void put(uint32_t, int len) { n += (unsigned)len; }
};

// MSB-first bit writer into 32-bit words whose bytes sit in stream order in memory.  Writers of neighbouring blocks
// share the words at their boundaries, so the device form ORs atomically into a zeroed buffer.
struct BitWriter {
  uint32_t* words;
  long long w;        // word the next full 32 bits go to
  uint64_t acc = 0;
  int n;              // bits pending in acc (the first word starts with `start % 32` zero bits)
  __host__ __device__ BitWriter(uint32_t* base, unsigned long long start) : words(base), w((long long)(start >> 5)), n((int)(start & 31)) {}
  __host__ __device__ static void or_word(uint32_t* p, uint32_t v) {
#ifdef __CUDA_ARCH__
    atomicOr(p, __byte_perm(v, 0, 0x0123));
#else
    *p |= __builtin_bswap32(v);
#endif
  }
  __host__ __device__ void put(uint32_t code, int len) {   // len <= 16
    acc = (acc << len) | code;
    n += len;
    if (n >= 32) {
      n -= 32;
      or_word(words + w++, (uint32_t)(acc >> n));
    }
  }
  __host__ __device__ void flush() {
    if (n > 0) or_word(words + w, (uint32_t)(acc << (32 - n)));
  }
};

// Stream bytes with a 0x00 after every 0xFF (the entropy-coded segment's byte stuffing).
__host__ __device__ inline int count_ff(const uint8_t* p, int n) {
  int k = 0;
  for (int i = 0; i < n; ++i) k += p[i] == 0xff;
  return k;
}
__host__ __device__ inline int stuff_copy(const uint8_t* p, int n, uint8_t* out) {
  int o = 0;
  for (int i = 0; i < n; ++i) {
    out[o++] = p[i];
    if (p[i] == 0xff) out[o++] = 0;
  }
  return o;
}

// Worst-case stream size: header, every block at its longest code, all of it doubled by stuffing, pad, EOI.
__host__ __device__ inline unsigned long long entropy_bound_bits(const Geom& g) {
  return (unsigned long long)blocks_per_image(g) * kMaxBlockBits + 7;
}
__host__ __device__ inline unsigned long long entropy_bound_bits(int W, int H) { return entropy_bound_bits(geom(W, H)); }
__host__ __device__ inline unsigned long long encode_bound(const Geom& g) {
  return kHeaderBytes + 2 * (entropy_bound_bits(g) / 8) + 2;
}
__host__ __device__ inline unsigned long long encode_bound(int W, int H) { return encode_bound(geom(W, H)); }

// jpeg_gen_optimal_table (jchuff.c): the length-limited Huffman code of one table from its symbol counts freq[0..255]
// (freq[256] is the reserved code point; freq is consumed).  libjpeg picks the two smallest non-zero counts, the
// larger symbol on ties, starting each search at 1e9; lengths above 16 are folded down as in K.3 (Adjust_BITS); the
// longest length loses one code (the all-ones code word).  bits[16] and vals[] get BITS / HUFFVAL; returns #vals.
__host__ __device__ inline int gen_optimal_table(long long* freq, uint8_t* bits16, uint8_t* vals) {
  constexpr int kMaxClen = 32;
  unsigned char codesize[257];
  short others[257];
  int bits[kMaxClen + 1];
  for (int i = 0; i < 257; ++i) { codesize[i] = 0; others[i] = -1; }
  for (int i = 0; i <= kMaxClen; ++i) bits[i] = 0;
  freq[256] = 1;
  for (;;) {
    int c1 = -1, c2 = -1;
    long long v = 1000000000ll;
    for (int i = 0; i <= 256; ++i)
      if (freq[i] && freq[i] <= v) { v = freq[i]; c1 = i; }
    v = 1000000000ll;
    for (int i = 0; i <= 256; ++i)
      if (freq[i] && freq[i] <= v && i != c1) { v = freq[i]; c2 = i; }
    if (c2 < 0) break;
    freq[c1] += freq[c2];
    freq[c2] = 0;
    codesize[c1]++;
    while (others[c1] >= 0) { c1 = others[c1]; codesize[c1]++; }
    others[c1] = (short)c2;
    codesize[c2]++;
    while (others[c2] >= 0) { c2 = others[c2]; codesize[c2]++; }
  }
  for (int i = 0; i <= 256; ++i)
    if (codesize[i]) bits[codesize[i] < kMaxClen ? codesize[i] : kMaxClen]++;
  int i = kMaxClen;
  for (; i > 16; --i)
    while (bits[i] > 0) {
      int j = i - 2;
      while (bits[j] == 0) --j;
      bits[i] -= 2;
      bits[i - 1]++;
      bits[j + 1] += 2;
      bits[j]--;
    }
  while (bits[i] == 0) --i;
  bits[i]--;
  for (int l = 1; l <= 16; ++l) bits16[l - 1] = (uint8_t)bits[l];
  int p = 0;
  for (int l = 1; l <= kMaxClen; ++l)
    for (int j = 0; j <= 255; ++j)
      if (codesize[j] == l) vals[p++] = (uint8_t)j;
  return p;
}

// A stream's header with optimised tables: the common header's prefix (SOI .. SOF0), DHT DC0 AC0 DC1 AC1 from bits[t]
// / vals[t] (t = 2 * table + class; DC0 AC0 only for grey, nc 1), then the common header's tail (DRI, SOS).  Returns
// the header's length.
__host__ __device__ inline int optimal_header(const uint8_t* common, int common_len, const uint8_t (*bits)[16],
                                              const uint8_t (*vals)[256], uint8_t* out, int nc = 3) {
  const int prefix = nc == 1 ? kGreyHeaderPrefix : kHeaderPrefix, dhts = nc == 1 ? kGreyAnnexKDhtBytes : kAnnexKDhtBytes;
  int o = 0;
  for (int k = 0; k < prefix; ++k) out[o++] = common[k];
  for (int t = 0; t < (nc == 1 ? 2 : 4); ++t) {
    int n = 0;
    for (int l = 0; l < 16; ++l) n += bits[t][l];
    const int len = 2 + 1 + 16 + n;
    out[o++] = 0xff; out[o++] = 0xc4; out[o++] = (uint8_t)(len >> 8); out[o++] = (uint8_t)len;
    out[o++] = (uint8_t)(((t & 1) << 4) | (t >> 1));
    for (int l = 0; l < 16; ++l) out[o++] = bits[t][l];
    for (int k = 0; k < n; ++k) out[o++] = vals[t][k];
  }
  for (int k = prefix + dhts; k < common_len; ++k) out[o++] = common[k];
  return o;
}

// ------------------------------------------------------------------ cv2.imwrite's JPEG parameters (grfmt_jpeg.cpp)
enum ParamKey {   // cv2.IMWRITE_JPEG_*
  kQuality = 1, kProgressive = 2, kOptimize = 3, kRstInterval = 4, kLumaQuality = 5, kChromaQuality = 6, kSamplingFactor = 7
};
// What a (key, value) list means for the stream, normalised as cv2 does.
struct Opts {
  int hy = 2, vy = 2;       // luma blocks per MCU across / down (Cb, Cr 1x1)
  int qy = 95, qc = 95;     // quality of the luma / chroma quantisation table, 1..100
  int rst = 0;              // restart interval in MCUs, 0..65535
  int optimize = 0, progressive = 0;
  int nc = 3;               // components: 3 (BGR / BGRA images) or 1 (grey)
  bool operator==(const Opts& o) const {
    return hy == o.hy && vy == o.vy && qy == o.qy && qc == o.qc && rst == o.rst && optimize == o.optimize &&
           progressive == o.progressive && nc == o.nc;
  }
  bool operator!=(const Opts& o) const { return !(*this == o); }
};
// quality (the IMWRITE_JPEG_QUALITY of the call) and n ints of (key, value) pairs -> *o.  False for odd n or a key
// outside 1..7.  The rules are cv2's:
//   QUALITY          clamped to [0, 100], 0 acts as 1
//   LUMA_QUALITY     ignored below 0; otherwise min(v, 100) replaces QUALITY, for the chroma table too unless
//                    CHROMA_QUALITY is given (in either order)
//   CHROMA_QUALITY   ignored below 0 or without LUMA_QUALITY; min(v, 100) otherwise.  Luma != chroma forces 4:4:4
//   SAMPLING_FACTOR  0x111111 / 0x211111 / 0x121111 / 0x221111 / 0x411111 (Y h << 20 | v << 16); anything else 4:2:0
//   RST_INTERVAL     clamped to [0, 65535]
//   OPTIMIZE, PROGRESSIVE  on above 0 (cv2 4.13 reads them as 0 / 1: values below 0 act as 0)
inline bool normalise(int quality, const int* params, int n, Opts* o) {
  if (n < 0 || (n & 1) || (n && !params)) return false;
  int luma = -1, chroma = -1, sampling = 0;
  Opts r;
  quality = quality < 0 ? 0 : quality > 100 ? 100 : quality;
  for (int i = 0; i < n; i += 2) {
    const int v = params[i + 1];
    switch (params[i]) {
      case kQuality: quality = v < 0 ? 0 : v > 100 ? 100 : v; break;
      case kProgressive: r.progressive = v > 0; break;
      case kOptimize: r.optimize = v > 0; break;
      case kRstInterval: r.rst = v < 0 ? 0 : v > 65535 ? 65535 : v; break;
      case kLumaQuality:
        if (v >= 0) {
          luma = v < 100 ? v : 100;
          quality = luma;
          if (chroma < 0) chroma = luma;
        }
        break;
      case kChromaQuality:
        if (v >= 0) chroma = v < 100 ? v : 100;
        break;
      case kSamplingFactor:
        sampling = (v == 0x111111 || v == 0x211111 || v == 0x121111 || v == 0x221111 || v == 0x411111) ? v : 0;
        break;
      default: return false;
    }
  }
  if (sampling) { r.hy = (sampling >> 20) & 15; r.vy = (sampling >> 16) & 15; }
  r.qy = r.qc = clamp_quality(quality);
  if (luma >= 0 && chroma >= 0) {
    r.qy = clamp_quality(luma);
    r.qc = clamp_quality(chroma);
    if (luma != chroma) r.hy = r.vy = 1;
  }
  *o = r;
  return true;
}
inline Opts default_opts(int quality) {
  Opts o;
  normalise(quality, nullptr, 0, &o);
  return o;
}
// The options for an image of `channels` channels: grey has one component in 1x1 MCUs (cv2's SAMPLING_FACTOR and the
// chroma quality do not reach its stream; the luma quality is table 0's); BGRA is BGR.
inline Opts channel_opts(Opts o, int channels) {
  if (channels == 1) { o.nc = 1; o.hy = o.vy = 1; }
  return o;
}
inline Geom geom(int W, int H, const Opts& o) {
  Geom g = geom(W, H, o.hy, o.vy);
  g.nc = o.nc;
  return g;
}

// Restart intervals of one image (1 without restart markers): each is byte-aligned with a 1-bit pad and followed by
// RSTn except the last, so each adds up to 7 pad bits and a 2-byte marker.
inline long long intervals(const Geom& g, const Opts& o) {
  const long long mcus = (long long)g.mcux * g.mcuy;
  return o.rst ? (mcus + o.rst - 1) / o.rst : 1;
}
inline unsigned long long entropy_bound_bits(const Geom& g, const Opts& o) {
  return (unsigned long long)blocks_per_image(g) * (o.optimize ? kMaxBlockBitsOpt : kMaxBlockBits) + 7ull * intervals(g, o);
}
inline int header_bytes(const Opts& o) { return (o.nc == 1 ? kGreyHeaderBytes : kHeaderBytes) + (o.rst ? kDriBytes : 0); }
// The params bound: header, entropy bits with every interval's pad, doubled by stuffing, markers, EOI.  With no params
// this is encode_bound(W, H).
inline unsigned long long encode_bound(const Geom& g, const Opts& o) {
  return header_bytes(o) + 2 * (entropy_bound_bits(g, o) / 8) + 2 * (intervals(g, o) - 1) + 2;
}

// ------------------------------------------------------------------ host: tables and header (jcparam.c, Annex K)
namespace annex_k {
static const uint8_t kLumaQ[64] = {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57,
                                   69, 56, 14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64,
                                   81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
static const uint8_t kChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                                     99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
static const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
// BITS (codes per length 1..16) and HUFFVAL of K.3 (DC) and K.5 (AC), luma then chroma
static const uint8_t kDcBits[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
static const uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t kAcBits[2][16] = {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d}, {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
static const uint8_t kAcVals[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
     0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
     0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
     0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
     0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
     0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
     0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
     0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
     0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
     0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
     0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
     0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
     0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
     0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
     0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
     0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
     0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};
}  // namespace annex_k

// jpeg_quality_scaling + jpeg_add_quant_table(force_baseline): natural-order steps of table t (0 luma, 1 chroma)
inline void quant_steps(int quality, int t, int* q) {
  const int qq = clamp_quality(quality), scale = qq < 50 ? 5000 / qq : 200 - 2 * qq;
  const uint8_t* base = t ? annex_k::kChromaQ : annex_k::kLumaQ;
  for (int k = 0; k < 64; ++k) {
    const int v = (base[k] * scale + 50) / 100;
    q[k] = v < 1 ? 1 : v > 255 ? 255 : v;
  }
}

// Canonical code assignment (Annex C): (length << 16) | code per symbol
__host__ __device__ inline void huff_codes(const uint8_t* bits, const uint8_t* vals, uint32_t* table, int n_table) {
  for (int i = 0; i < n_table; ++i) table[i] = 0;
  uint32_t code = 0;
  int k = 0;
  for (int len = 1; len <= 16; ++len) {
    for (int i = 0; i < bits[len - 1]; ++i) table[vals[k++]] = ((uint32_t)len << 16) | code++;
    code <<= 1;
  }
}

inline void make_tables(const Opts& o, Tables* t) {
  memset(t, 0, sizeof *t);
  for (int c = 0; c < 2; ++c) {
    int q[64];
    quant_steps(c ? o.qc : o.qy, c, q);
    for (int k = 0; k < 64; ++k) t->qdiv[c][k] = (uint16_t)(8 * q[k]);
    huff_codes(annex_k::kDcBits[c], annex_k::kDcVals, t->dc[c], 12);
    huff_codes(annex_k::kAcBits[c], annex_k::kAcVals[c], t->ac[c], 256);
  }
  memcpy(t->zz, annex_k::kZigzag, 64);
}
inline void make_tables(int quality, Tables* t) { make_tables(default_opts(quality), t); }

// SOI, APP0 (JFIF 1.01, no units, 1x1), DQT 0 (qy) and DQT 1 (qc), SOF0 (Y hy x vy table 0, Cb/Cr 1x1 table 1),
// DHT DC0 AC0 DC1 AC1, SOS (Y 0/0, Cb 1/1, Cr 1/1, Ss 0 Se 63 Ah/Al 0): kHeaderBytes bytes.  Grey (o.nc 1): DQT 0,
// SOF0 with one component (1x1, table 0), DHT DC0 AC0, SOS with one component: kGreyHeaderBytes.
inline void make_header(int W, int H, const Opts& o, uint8_t* out) {
  const int nt = o.nc == 1 ? 1 : 2;   // quantisation and Huffman table pairs
  uint8_t* p = out;
  auto b = [&](int v) { *p++ = (uint8_t)v; };
  auto w16 = [&](int v) { b(v >> 8); b(v & 255); };
  b(0xff); b(0xd8);
  b(0xff); b(0xe0); w16(16);
  for (const char ch : {'J', 'F', 'I', 'F', '\0'}) b(ch);
  b(1); b(1); b(0); w16(1); w16(1); b(0); b(0);
  for (int t = 0; t < nt; ++t) {
    int q[64];
    quant_steps(t ? o.qc : o.qy, t, q);
    b(0xff); b(0xdb); w16(67); b(t);
    for (int k = 0; k < 64; ++k) b(q[annex_k::kZigzag[k]]);
  }
  b(0xff); b(0xc0); w16(8 + 3 * o.nc); b(8); w16(H); w16(W); b(o.nc);
  b(1); b((o.hy << 4) | o.vy); b(0);
  if (o.nc == 3) {
    b(2); b(0x11); b(1);
    b(3); b(0x11); b(1);
  }
  for (int t = 0; t < nt; ++t) {
    for (int cls = 0; cls < 2; ++cls) {
      const uint8_t* bits = cls ? annex_k::kAcBits[t] : annex_k::kDcBits[t];
      const uint8_t* vals = cls ? annex_k::kAcVals[t] : annex_k::kDcVals;
      int n = 0;
      for (int i = 0; i < 16; ++i) n += bits[i];
      b(0xff); b(0xc4); w16(2 + 1 + 16 + n); b((cls << 4) | t);
      for (int i = 0; i < 16; ++i) b(bits[i]);
      for (int i = 0; i < n; ++i) b(vals[i]);
    }
  }
  if (o.rst) { b(0xff); b(0xdd); w16(4); w16(o.rst); }   // DRI
  b(0xff); b(0xda); w16(6 + 2 * o.nc); b(o.nc);
  b(1); b(0x00);
  if (o.nc == 3) {
    b(2); b(0x11);
    b(3); b(0x11);
  }
  b(0); b(63); b(0);
}
inline void make_header(int W, int H, int quality, uint8_t* out) { make_header(W, H, default_opts(quality), out); }

// ------------------------------------------------------------------ device pipeline
struct EncArgs {
  const uint8_t* img;            // image i at img + i * istride, rows at pitch, BGR
  long long istride, pitch;
  int n;
  Geom g;
  long long nblk;                // blocks per image
  const Tables* tabs;
  int16_t* coef;                 // [n * nblk][64] zigzag
  unsigned long long* bits;      // [n * nblk] bits per block
  unsigned long long* offs;      // [n * nblk] exclusive scan of bits (over the whole batch)
  int* dcdiff;                   // [n * nblk]
  uint32_t* words;               // image i's entropy bits at words + i * words_img
  long long words_img;
  int chunks_img;                // kChunk-byte chunks per image region
  unsigned* ffcnt;               // [n * chunks_img] 0xFF bytes per chunk
  unsigned* ffscan;              // exclusive scan of ffcnt (over the whole batch)
  const uint8_t* header;         // kHeaderBytes
  uint8_t* out;                  // compacted streams
  unsigned long long* out_off;   // [n]
  unsigned long long* sizes;     // [n]
  // restart intervals (rst > 0): nint per image; ilen / iofs [n * nint]: padded bits per interval and their exclusive
  // scan over the batch
  int rst;
  long long nint;
  unsigned long long* ilen;
  unsigned long long* iofs;
  // optimised tables: counts [n][4][256] (DC0, AC0, DC1, AC1), each image's codes and header ([n][kMaxHeaderBytes],
  // hlen[n] bytes); otherwise every image takes `header` (hlen0 bytes) and tabs
  unsigned long long* counts;
  struct Huff { uint32_t ac[2][256]; uint32_t dc[2][12]; }* huff;
  uint8_t* hdrs;
  int* hlen;
  int hlen0;
};
using Huff = EncArgs::Huff;

constexpr int kBlockThreads = 128;
constexpr int kBlockPad = 65;    // ints per thread's block in shared memory: odd stride, conflict-free

__device__ inline void load_tables(Tables* s, const Tables* g) {
  const uint32_t* src = reinterpret_cast<const uint32_t*>(g);
  uint32_t* dst = reinterpret_cast<uint32_t*>(s);
  for (int i = threadIdx.x; i < (int)(sizeof(Tables) / 4); i += blockDim.x) dst[i] = src[i];
}

// bits of image i's entropy-coded data, without the final pad (with restart intervals: every interval padded)
__device__ inline unsigned long long image_bits(const EncArgs& a, int i) {
  if (a.rst) {
    const long long l = (long long)(i + 1) * a.nint - 1;
    return a.iofs[l] + a.ilen[l] - a.iofs[(long long)i * a.nint];
  }
  const long long last = (long long)(i + 1) * a.nblk - 1;
  return a.offs[last] + a.bits[last] - a.offs[(long long)i * a.nblk];
}
__device__ inline int header_len(const EncArgs& a, int i) { return a.hlen ? a.hlen[i] : a.hlen0; }

// blocks per MCU of an NC-component layout
template <int HY, int VY, int NC>
constexpr int kBpm = HY * VY + (NC == 1 ? 0 : 2);

template <int HY, int VY, int C = 3>
__global__ void __launch_bounds__(kBlockThreads) k_jpeg_blocks(EncArgs a) {
  constexpr int NY = HY * VY, BPM = kBpm<HY, VY, C == 1 ? 1 : 3>;   // luma blocks and blocks per MCU
  __shared__ Tables st;
  __shared__ int sblk[kBlockThreads * kBlockPad];
  load_tables(&st, a.tabs);
  const long long b = (long long)blockIdx.x * kBlockThreads + threadIdx.x;
  __syncthreads();
  if (b >= a.nblk * a.n) return;
  const int i = (int)(b / a.nblk);
  const long long local = b - i * a.nblk;
  const int m = (int)(local / BPM), k = (int)(local - (long long)BPM * m);
  const int mx = m % a.g.mcux, my = m / a.g.mcux;
  int16_t* out = a.coef + b * 64;
  const int t = k < NY ? 0 : 1;
  if (is_dummy_s<HY, VY>(a.g, mx, my, k)) {
    uint4* o = reinterpret_cast<uint4*>(out);
    for (int j = 0; j < 8; ++j) o[j] = make_uint4(0, 0, 0, 0);
    a.bits[b] = st.ac[0][0] >> 16;                         // EOB only
    return;
  }
  int* d = sblk + threadIdx.x * kBlockPad;
  load_block_s<HY, VY, C>(a.img + i * a.istride, a.pitch, a.g, mx, my, k, d);
  fdct_islow(d);
  quantise(d, st.qdiv[t]);
  const uint8_t* zz = st.zz;
  BitCount cnt;
  emit_ac(ZigzagOf{d, zz}, st.ac[t], cnt);
  for (int j = 0; j < 64; j += 2) {
    const unsigned lo = (uint16_t)d[zz[j]], hi = (uint16_t)d[zz[j + 1]];
    reinterpret_cast<unsigned*>(out)[j >> 1] = lo | (hi << 16);
  }
  a.bits[b] = cnt.n;
}

// quantised DC of block k of MCU m (image-local block index base): a dummy takes the DC of the block before it
template <int HY, int VY>
__device__ inline int resolved_dc(const EncArgs& a, long long mcu_base, int mx, int my, int k) {
  while (k > 0 && is_dummy_s<HY, VY>(a.g, mx, my, k)) --k;
  return a.coef[(mcu_base + k) * 64];
}

template <int HY, int VY, int NC = 3>
__global__ void k_jpeg_dc(EncArgs a) {
  constexpr int NY = HY * VY, BPM = kBpm<HY, VY, NC>;
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.nblk * a.n) return;
  const int i = (int)(b / a.nblk);
  const long long local = b - i * a.nblk;
  const int m = (int)(local / BPM), k = (int)(local - (long long)BPM * m);
  const int mx = m % a.g.mcux, my = m / a.g.mcux;
  const long long base = b - k;                           // block 0 of this MCU
  const int dc = resolved_dc<HY, VY>(a, base, mx, my, k);
  int pred = 0;
  if (k > 0 && k < NY) pred = resolved_dc<HY, VY>(a, base, mx, my, k - 1);
  else if (m > 0 && (a.rst == 0 || m % a.rst != 0)) {      // predictors restart at 0 with every restart interval
    const int pm = m - 1;
    pred = resolved_dc<HY, VY>(a, base - BPM, pm % a.g.mcux, pm / a.g.mcux, k == 0 ? NY - 1 : k);
  }
  const int diff = dc - pred;
  a.dcdiff[b] = diff;
  BitCount cnt;
  emit_dc(diff, a.tabs->dc[k < NY ? 0 : 1], cnt);
  a.bits[b] += cnt.n;
}

// clear the words image i's bits will occupy (the pad stays inside the last one)
__global__ void k_jpeg_zero(EncArgs a) {
  for (int i = 0; i < a.n; ++i) {
    const long long used = (long long)((image_bits(a, i) + 31) >> 5);
    uint32_t* w = a.words + i * a.words_img;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < used; j += (long long)gridDim.x * blockDim.x) w[j] = 0;
  }
}

// kOpt: the image's own codes (k_jpeg_huff) instead of the shared Annex K tables; kRst: byte-aligned restart intervals
template <int HY, int VY, bool kOpt, bool kRst, int NC = 3>
__global__ void __launch_bounds__(kBlockThreads) k_jpeg_pack(EncArgs a) {
  constexpr int NY = HY * VY, BPM = kBpm<HY, VY, NC>;
  __shared__ Tables st;
  if constexpr (!kOpt) load_tables(&st, a.tabs);
  __syncthreads();
  const long long b = (long long)blockIdx.x * kBlockThreads + threadIdx.x;
  if (b >= a.nblk * a.n) return;
  const int i = (int)(b / a.nblk);
  const long long local = b - i * a.nblk;
  const int t = (int)(local % BPM) < NY ? 0 : 1;
  const uint32_t* dc = kOpt ? a.huff[i].dc[t] : st.dc[t];
  const uint32_t* ac = kOpt ? a.huff[i].ac[t] : st.ac[t];
  unsigned long long start;
  bool last;
  unsigned long long ibits;                               // bits of the block's interval up to its end
  if constexpr (kRst) {
    const long long m = local / BPM, j = m / a.rst, first = (long long)i * a.nblk + j * a.rst * BPM;
    const long long mend = (j + 1) * a.rst < (long long)a.g.mcux * a.g.mcuy ? (j + 1) * a.rst : (long long)a.g.mcux * a.g.mcuy;
    start = a.iofs[(long long)i * a.nint + j] - a.iofs[(long long)i * a.nint] + a.offs[b] - a.offs[first];
    last = local == mend * BPM - 1;
    ibits = a.offs[b] + a.bits[b] - a.offs[first];
  } else {
    start = a.offs[b] - a.offs[(long long)i * a.nblk];
    last = local == a.nblk - 1;
    ibits = start + a.bits[b];
  }
  BitWriter wr(a.words + i * a.words_img, start);
  emit_dc(a.dcdiff[b], dc, wr);
  emit_ac(Zigzag16{a.coef + b * 64}, ac, wr);
  if (last) {                                             // an interval's (image's) last block pads its byte with 1 bits
    const int pad = (int)((8 - (ibits & 7)) & 7);
    if (pad) wr.put((1u << pad) - 1u, pad);
  }
  wr.flush();
}

// restart intervals: padded bits of interval j of image i, one thread per interval
__global__ void k_jpeg_intervals(EncArgs a) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.n * a.nint) return;
  const int bpm = mcu_blocks(a.g);
  const long long i = t / a.nint, j = t - i * a.nint, mcus = (long long)a.g.mcux * a.g.mcuy;
  const long long mend = (j + 1) * a.rst < mcus ? (j + 1) * a.rst : mcus;
  const long long first = i * a.nblk + j * a.rst * bpm, last = i * a.nblk + mend * bpm - 1;
  a.ilen[t] = (a.offs[last] + a.bits[last] - a.offs[first] + 7) & ~7ull;
}

// optimised tables, pass 1: symbol counts per image and table.  Each CTA gathers the first two images its blocks
// touch in shared memory and adds those counts once; blocks of further images (small images) add theirs directly.
template <int HY, int VY, int NC = 3>
__global__ void __launch_bounds__(kBlockThreads) k_jpeg_count(EncArgs a) {
  constexpr int NY = HY * VY, BPM = kBpm<HY, VY, NC>;
  __shared__ unsigned sc[2][4 * 256];
  for (int e = threadIdx.x; e < 2 * 4 * 256; e += blockDim.x) (&sc[0][0])[e] = 0;
  __syncthreads();
  const long long b = (long long)blockIdx.x * kBlockThreads + threadIdx.x;
  const int i0 = (int)((long long)blockIdx.x * kBlockThreads / a.nblk);
  if (b < a.nblk * a.n) {
    const int i = (int)(b / a.nblk);
    const int tb = (int)((b - i * a.nblk) % BPM) < NY ? 0 : 1;
    unsigned* s = i - i0 < 2 ? sc[i - i0] : nullptr;
    unsigned long long* g = a.counts + (size_t)i * 1024;
    block_symbols(a.dcdiff[b], Zigzag16{a.coef + b * 64}, [&](int cls, int sym) {
      const int e = (2 * tb + cls) * 256 + sym;
      if (s) atomicAdd(s + e, 1u);
      else atomicAdd(g + e, 1ull);
    });
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 2 * 1024; e += blockDim.x) {
    const int k = e >> 10, i = i0 + k;
    const unsigned v = sc[k][e & 1023];
    if (v && i < a.n) atomicAdd(a.counts + (size_t)i * 1024 + (e & 1023), (unsigned long long)v);
  }
}

// optimised tables, pass 2: one thread per (image, table) runs jpeg_gen_optimal_table and writes the codes; then one
// thread per image writes its header (the common prefix, its four DHTs -- two for grey, NC 1 -- the common DRI / SOS)
constexpr int kHuffThreads = 128;
template <int NC = 3>
__global__ void __launch_bounds__(kHuffThreads) k_jpeg_huff(EncArgs a) {
  __shared__ uint8_t sbits[kHuffThreads][16];
  __shared__ uint8_t svals[kHuffThreads][256];
  const long long t = (long long)blockIdx.x * kHuffThreads + threadIdx.x;
  const int i = (int)(t >> 2), tb = (int)(t & 3);
  if (i < a.n && (NC == 3 || tb < 2)) {
    long long freq[257];
    for (int k = 0; k < 256; ++k) freq[k] = (long long)a.counts[(size_t)i * 1024 + tb * 256 + k];
    gen_optimal_table(freq, sbits[threadIdx.x], svals[threadIdx.x]);
    const int c = tb >> 1;
    if (tb & 1) huff_codes(sbits[threadIdx.x], svals[threadIdx.x], a.huff[i].ac[c], 256);
    else huff_codes(sbits[threadIdx.x], svals[threadIdx.x], a.huff[i].dc[c], 12);
  }
  __syncthreads();
  if (i < a.n && tb == 0) {
    const int q = threadIdx.x;   // this image's four tables are threads q .. q + 3
    a.hlen[i] = optimal_header(a.header, a.hlen0, &sbits[q], &svals[q], a.hdrs + (size_t)i * kMaxHeaderBytes, NC);
  }
}

// optimised tables, pass 3: each block's bits under its image's codes
template <int HY, int VY, int NC = 3>
__global__ void __launch_bounds__(kBlockThreads) k_jpeg_bits(EncArgs a) {
  constexpr int NY = HY * VY, BPM = kBpm<HY, VY, NC>;
  const long long b = (long long)blockIdx.x * kBlockThreads + threadIdx.x;
  if (b >= a.nblk * a.n) return;
  const int i = (int)(b / a.nblk);
  const int t = (int)((b - i * a.nblk) % BPM) < NY ? 0 : 1;
  BitCount cnt;
  emit_dc(a.dcdiff[b], a.huff[i].dc[t], cnt);
  emit_ac(Zigzag16{a.coef + b * 64}, a.huff[i].ac[t], cnt);
  a.bits[b] = cnt.n;
}

__global__ void k_jpeg_ffcount(EncArgs a) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)a.n * a.chunks_img) return;
  const int i = (int)(t / a.chunks_img), c = (int)(t - (long long)i * a.chunks_img);
  const long long nbytes = (long long)((image_bits(a, i) + 7) >> 3), off = (long long)c * kChunk;
  if (off >= nbytes) return;   // unused chunks keep stale counts: only differences within an image are ever read
  const uint8_t* p = reinterpret_cast<const uint8_t*>(a.words + i * a.words_img) + off;
  a.ffcnt[t] = (unsigned)count_ff(p, (int)(nbytes - off < kChunk ? nbytes - off : kChunk));
}

// one CTA: stream sizes and compacted offsets, then every image's header and EOI
__global__ void k_jpeg_layout(EncArgs a) {
  if (threadIdx.x == 0) {
    unsigned long long off = 0;
    for (int i = 0; i < a.n; ++i) {
      const unsigned long long nbytes = (image_bits(a, i) + 7) >> 3;
      const long long c0 = (long long)i * a.chunks_img, cl = c0 + (long long)((nbytes + kChunk - 1) / kChunk) - 1;
      const unsigned ff = a.ffscan[cl] + a.ffcnt[cl] - a.ffscan[c0];
      const unsigned long long size = header_len(a, i) + nbytes + ff + 2 * (a.nint - 1) + 2;
      a.out_off[i] = off;
      a.sizes[i] = size;
      off += size;
    }
  }
  __syncthreads();
  for (long long j = threadIdx.x; j < (long long)a.n * kMaxHeaderBytes; j += blockDim.x) {
    const int i = (int)(j / kMaxHeaderBytes), h = (int)(j - (long long)i * kMaxHeaderBytes);
    if (h < header_len(a, i)) a.out[a.out_off[i] + h] = a.hdrs ? a.hdrs[j] : a.header[h];
  }
  for (int i = threadIdx.x; i < a.n; i += blockDim.x) {
    uint8_t* e = a.out + a.out_off[i] + a.sizes[i] - 2;
    e[0] = 0xff;
    e[1] = 0xd9;
  }
}

// byte where restart interval j of image i starts in its unstuffed data
__device__ inline unsigned long long interval_start(const EncArgs& a, int i, long long j) {
  return (a.iofs[(long long)i * a.nint + j] - a.iofs[(long long)i * a.nint]) >> 3;
}

__global__ void k_jpeg_stuff(EncArgs a) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)a.n * a.chunks_img) return;
  const int i = (int)(t / a.chunks_img), c = (int)(t - (long long)i * a.chunks_img);
  const long long nbytes = (long long)((image_bits(a, i) + 7) >> 3), off = (long long)c * kChunk;
  if (off >= nbytes) return;
  const uint8_t* p = reinterpret_cast<const uint8_t*>(a.words + i * a.words_img) + off;
  const int len = (int)(nbytes - off < kChunk ? nbytes - off : kChunk);
  uint8_t* o = a.out + a.out_off[i] + header_len(a, i) + off + (a.ffscan[t] - a.ffscan[(long long)i * a.chunks_img]);
  if (!a.rst) {
    stuff_copy(p, len, o);
    return;
  }
  // RSTn goes before the first byte of every interval but the first: find the first interval starting at or past off
  long long lo = 1, hi = a.nint;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (interval_start(a, i, mid) < (unsigned long long)off) lo = mid + 1;
    else hi = mid;
  }
  o += 2 * (lo - 1);                                       // the markers before this chunk
  unsigned long long next = lo < a.nint ? interval_start(a, i, lo) : ~0ull;
  for (int k = 0; k < len; ++k) {
    if ((unsigned long long)(off + k) == next) {
      *o++ = 0xff;
      *o++ = (uint8_t)(0xd0 + ((lo - 1) & 7));
      ++lo;
      next = lo < a.nint ? interval_start(a, i, lo) : ~0ull;
    }
    *o++ = p[k];
    if (p[k] == 0xff) *o++ = 0;
  }
}

}  // namespace jpeg
}  // namespace bevk
