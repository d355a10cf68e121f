// bevk_jpeg_prog.cuh -- progressive JPEG on the device (sm_90a), byte-identical to cv2.imencode(".jpg", img,
// [IMWRITE_JPEG_PROGRESSIVE, 1, ...]).
//
// The quantised coefficients are the baseline encoder's (k_jpeg_blocks: dummy blocks, quality rules, sampling factors);
// only the entropy coder differs.  libjpeg-turbo's jpeg_simple_progression script for YCbCr, with tables optimised per
// scan (PROGRESSIVE implies OPTIMIZE in libjpeg):
//   #  components    Ss-Se  Ah Al   tables (DHT before the SOS)
//   0  Y Cb Cr        0-0    0  1   DC0, DC1                 DC first scans: differences of arithmetically shifted DCs
//   1  Y              1-5    0  2   AC0                      AC first scans: |v| >> Al, negative values as the ones'
//   2  Cr             1-63   0  1   AC1                                      complement of the shifted magnitude
//   3  Cb             1-63   0  1   AC1
//   4  Y              6-63   0  2   AC0
//   5  Y              1-63   2  1   AC0                      AC refinement: newly non-zero (r, 1) + sign, correction
//   6  Y Cb Cr        0-0    1  0   none                     DC refinement: bit Al of each DC, no Huffman code
//   7  Cr             1-63   1  0   AC1
//   8  Cb             1-63   1  0   AC1
//   9  Y              1-63   1  0   AC0
// Grey images (one component, Geom.nc 1) take libjpeg's script for other colour spaces, six scans of component 0:
//   0  DC 0-0 Ah 0 Al 1 (DC0)   1  AC 1-5 0/2 (AC0)   2  AC 6-63 0/2   3  AC 1-63 2/1   4  DC 0-0 1/0 (none)
//   5  AC 1-63 1/0
// with five tables per image (DC0, then one AC table per AC scan).  Every grey scan is non-interleaved: blocks in raster
// order, the restart interval counting blocks.  The functions below read the component count from Geom.nc; the
// kernels are instantiated per count (NC) so that it is a constant there.
// Interleaved scans code every MCU (dummy blocks included); a single-component scan codes that component's own blocks in
// raster order: ceil(W/8) x ceil(H/8) luma blocks, one chroma block per MCU.  The restart interval counts MCUs in
// interleaved scans and blocks in single-component scans; RSTn numbering starts at 0 in every scan.
//
// End-of-band runs.  AC scans code a block with no symbol as one more block of the pending EOB run (EOBn symbol + n
// bits), and in refinement scans the correction bits of those blocks ride along after the EOBn code.  libjpeg flushes
// the run before a block's first symbol, when it reaches 0x7FFF blocks, when more than kCorrFlush (937 =
// MAX_CORR_BITS - 64 + 1) correction bits are buffered, at a restart and at the end of the scan.  Per block that is:
//   BlockRun{sym, e, c}: the block emits a symbol (the run is flushed before it), then contributes e (0 / 1) blocks and c
//   correction bits to the run that follows its last symbol.
// Serially (tests/host/jpeg_progressive.cu, libjpeg's order) the run is a counter.  In parallel (the kernels) every flush is placed after a
// block x:
//   hard    x is the last block of its interval, or block x + 1 emits a symbol: always a flush
//   next    from a run starting at block j, the first block x >= j at which the run's e or c sums reach 0x7FFF or pass
//           937 (binary search over inclusive prefix sums), or the hard block ending j's segment, whichever is first;
//           next(j) = x + 1
//   marks   the run starts that are reached: every scan start and every block after a hard flush, then pointer doubling
//           along next() marks the rest (marking a node of the chain twice is harmless)
// A flush writes nothing when its run is empty (e sum 0).
//
// Bound (progressive_bound): per block and scan at most DC first 16 + 11, DC refinement 1, AC first 26 bits per
// coefficient of the band (a 16-bit code + up to 10 value bits; a ZRL stands for 16 coefficients), AC refinement 18 per
// coefficient (code, sign, one correction bit), plus one EOBn code with its bits (16 + 14) per block in AC scans (every
// non-empty run ends at a distinct block).  So 28 bits per block of an interleaved scan and 4026 per luma / 2832 per
// chroma block of the single-component scans, 7 pad bits per interval, all doubled by stuffing, plus the frame header,
// the ten scan headers (kProgHeaderBytes), RST markers and EOI.
#pragma once
#include "bevk_jpeg_enc.cuh"

namespace bevk {
namespace jpeg {
namespace prog {

constexpr int kScans = 10;             // scans of the YCbCr script: the most of any script (the strides of the buffers)
constexpr int kTables = 10;            // per image: DC0 DC1 (scan 0), then one AC table per AC scan
__host__ __device__ constexpr int scans(int nc) { return nc == 1 ? 6 : kScans; }
__host__ __device__ constexpr int tables(int nc) { return nc == 1 ? 5 : kTables; }
constexpr int kEobMax = 0x7FFF;        // EOB run length that forces a flush
constexpr int kCorrFlush = 937;        // more buffered correction bits than this force a flush
constexpr int kPrefixBytes = kHeaderPrefix;   // SOI APP0 DQT DQT SOF2 (grey: SOI APP0 DQT SOF2, kGreyHeaderPrefix)
constexpr int kDcDhtMax = 4 + 1 + 16 + 12;    // DHT segment of a DC table (categories 0..11)
constexpr int kAcDhtMax = 4 + 1 + 16 + 176;   // of an AC table (EOB0..14, ZRL, (r, 1..10))
constexpr int kMaxScanHeader = kAcDhtMax + 10; // one scan's DHT + SOS, the largest (AC) form
constexpr int kProgHeaderBytes = 2 * kDcDhtMax + kDriBytes + 14 + 8 * kMaxScanHeader + 14;   // all ten scan headers
constexpr int kGreyProgHeaderBytes = kDcDhtMax + kDriBytes + 10 + 4 * kMaxScanHeader + 10;  // the six grey ones
__host__ __device__ constexpr int prefix_bytes(int nc) { return nc == 1 ? kGreyHeaderPrefix : kPrefixBytes; }
__host__ __device__ constexpr int prog_header_bytes(int nc) { return nc == 1 ? kGreyProgHeaderBytes : kProgHeaderBytes; }
constexpr int kDcBits = 16 + 11, kLumaAcBits = 26 * 5 + 26 * 58 + 2 * 18 * 63 + 4 * 30, kChromaAcBits = 26 * 63 + 18 * 63 + 2 * 30;

struct Scan {
  int comp;          // 0 Y, 1 Cb, 2 Cr, 3 all three interleaved
  int ss, se, ah, al;
};
__host__ __device__ inline Scan script(int s) {
  switch (s) {
    case 0: return {3, 0, 0, 0, 1};
    case 1: return {0, 1, 5, 0, 2};
    case 2: return {2, 1, 63, 0, 1};
    case 3: return {1, 1, 63, 0, 1};
    case 4: return {0, 6, 63, 0, 2};
    case 5: return {0, 1, 63, 2, 1};
    case 6: return {3, 0, 0, 1, 0};
    case 7: return {2, 1, 63, 1, 0};
    case 8: return {1, 1, 63, 1, 0};
    default: return {0, 1, 63, 1, 0};
  }
}
__host__ __device__ inline Scan grey_script(int s) {
  switch (s) {
    case 0: return {0, 0, 0, 0, 1};
    case 1: return {0, 1, 5, 0, 2};
    case 2: return {0, 6, 63, 0, 2};
    case 3: return {0, 1, 63, 2, 1};
    case 4: return {0, 0, 0, 1, 0};
    default: return {0, 1, 63, 1, 0};
  }
}
__host__ __device__ inline Scan script(int nc, int s) { return nc == 1 ? grey_script(s) : script(s); }
// the image's table slot of AC scan s (slots 0 / 1 are scan 0's DC0 / DC1; scan 6 has none; grey: slot 0 is DC0,
// scan 4 has none)
__host__ __device__ inline int ac_slot(int nc, int s) { return nc == 1 ? (s < 4 ? s : s - 1) : s < 6 ? s + 1 : s; }
__host__ __device__ inline int ac_slot(int s) { return ac_slot(3, s); }
__host__ __device__ inline bool is_ac(int nc, int s) { return script(nc, s).ss > 0; }
__host__ __device__ inline bool is_ac(int s) { return is_ac(3, s); }

// The pairs of a list with PROGRESSIVE and OPTIMIZE mapped in place to the 0 / 1 cv2 4.13 stores (values below 0 as 0,
// above 1 as 1).  normalise() reads the flags the same way, so mapping first changes no Opts; the serial host encoder
// (tests/host/jpeg_progressive.cu) maps its lists with it.
inline void read_flags(int* params, int n) {
  for (int i = 0; i + 1 < n; i += 2)
    if (params[i] == kProgressive || params[i] == kOptimize) params[i + 1] = params[i + 1] > 0 ? 1 : 0;
}

// ------------------------------------------------------------------ which blocks a scan codes
// The functions of a Geom read the component count from g.nc; their forms with a leading nc take it as an argument,
// which the kernels pass as the constant NC (the Geom itself stays in kernel parameter space).
__host__ __device__ inline int mcu_blocks(int nc, const Geom& g) { return g.hy * g.vy + (nc == 1 ? 0 : 2); }
__host__ __device__ inline long long scan_blocks(const Geom& g, int s) {
  const int c = script(g.nc, s).comp;
  return c == 3 ? blocks_per_image(g) : c == 0 ? (long long)g.wb * g.hb : (long long)g.mcux * g.mcuy;
}
__host__ __device__ inline int unit_blocks(int nc, const Geom& g, int s) { return script(nc, s).comp == 3 ? mcu_blocks(nc, g) : 1; }
__host__ __device__ inline int unit_blocks(const Geom& g, int s) { return unit_blocks(g.nc, g, s); }
// restart intervals of scan s (1 without restarts)
__host__ __device__ inline long long scan_intervals(const Geom& g, int s, int rst) {
  const long long units = scan_blocks(g, s) / unit_blocks(g, s);
  return rst ? (units + rst - 1) / rst : 1;
}
// image-local coefficient slot (MCU-major, as k_jpeg_blocks writes them) of block j of scan s
__host__ __device__ inline long long scan_slot(int nc, const Geom& g, int s, long long j) {
  const int c = script(nc, s).comp, bpm = mcu_blocks(nc, g);
  if (c == 3) return j;
  if (c > 0) return j * bpm + g.hy * g.vy + c - 1;
  const long long by = j / g.wb, bx = j - by * g.wb;
  return ((by / g.vy) * g.mcux + bx / g.hy) * bpm + (by % g.vy) * g.hy + bx % g.hy;
}
__host__ __device__ inline long long scan_slot(const Geom& g, int s, long long j) { return scan_slot(g.nc, g, s, j); }
// component of block j of scan s
__host__ __device__ inline int scan_comp(int nc, const Geom& g, int s, long long j) {
  const int c = script(nc, s).comp;
  if (c != 3) return c;
  const int ny = g.hy * g.vy, k = (int)(j % (ny + 2));
  return k < ny ? 0 : k - ny + 1;
}
__host__ __device__ inline int scan_comp(const Geom& g, int s, long long j) { return scan_comp(g.nc, g, s, j); }

// Offsets of one image's scans: scan s's blocks are [blk[s], blk[s + 1]) and its intervals [seg[s], seg[s + 1]) of the
// image's blocks and intervals (segments) in scan order.  A script of fewer than kScans scans is followed by empty ones
// (blk[s] = blk[scans], seg[s] = seg[scans]), so kScans entries stand for every script.
struct Layout {
  long long blk[kScans + 1];
  long long seg[kScans + 1];
};
__host__ __device__ inline Layout layout(const Geom& g, int rst) {
  Layout l;
  l.blk[0] = l.seg[0] = 0;
  for (int s = 0; s < kScans; ++s) {
    const bool in = s < scans(g.nc);
    l.blk[s + 1] = l.blk[s] + (in ? scan_blocks(g, s) : 0);
    l.seg[s + 1] = l.seg[s] + (in ? scan_intervals(g, s, rst) : 0);
  }
  return l;
}
__host__ __device__ inline int scan_of(const long long* base, long long j) {   // base[s] <= j < base[s + 1]
  int s = 0;
  while (s < kScans - 1 && j >= base[s + 1]) ++s;
  return s;
}

// ------------------------------------------------------------------ point transforms and per-block symbols
__host__ __device__ inline int dc_point(int v, int al) { return v >> al; }   // arithmetic: IRIGHT_SHIFT of libjpeg

// Quantised DC of image-local slot b (MCU-major) with dummy blocks resolved (the DC of the block before it in the MCU);
// dc(b) reads slot b's stored DC.
template <class DC>
__host__ __device__ inline int resolved_dc_at(int nc, const Geom& g, long long b, const DC& dc) {
  const int bpm = mcu_blocks(nc, g);
  const long long m = b / bpm;
  int k = (int)(b - m * bpm);
  const int mx = (int)(m % g.mcux), my = (int)(m / g.mcux);
  while (k > 0 && is_dummy(g, mx, my, k)) --k;
  return dc(m * bpm + k);
}
template <class DC>
__host__ __device__ inline int resolved_dc_at(const Geom& g, long long b, const DC& dc) { return resolved_dc_at(g.nc, g, b, dc); }
// DC first scan: the difference coded for block j (= slot j) of an interleaved scan with point transform al; the
// predictor is the previous block of the same component, 0 at the start of every restart interval.  A grey DC scan
// (one block per MCU) is the same arithmetic over its blocks in raster order.
template <class DC>
__host__ __device__ inline int dc_first_diff(int nc, const Geom& g, int rst, long long j, int al, const DC& dc) {
  const int ny = g.hy * g.vy, bpm = mcu_blocks(nc, g);
  const long long m = j / bpm;
  const int k = (int)(j - m * bpm);
  const int v = dc_point(resolved_dc_at(nc, g, j, dc), al);
  long long p = -1;
  if (k > 0 && k < ny) p = j - 1;
  else if (m > 0 && (rst == 0 || m % rst != 0)) p = (m - 1) * bpm + (k == 0 ? ny - 1 : k);
  return v - (p < 0 ? 0 : dc_point(resolved_dc_at(nc, g, p, dc), al));
}
template <class DC>
__host__ __device__ inline int dc_first_diff(const Geom& g, int rst, long long j, int al, const DC& dc) {
  return dc_first_diff(g.nc, g, rst, j, al, dc);
}

struct BlockRun {
  int sym;   // the block emits at least one Huffman symbol
  int e;     // blocks it adds to the EOB run after its last symbol (0 / 1)
  int c;     // correction bits it adds to that run
};

template <class Sink>
__host__ __device__ inline void put_bits(Sink& s, unsigned long long v, int n) {   // n <= 64, MSB first
  while (n > 16) { n -= 16; s.put((uint32_t)(v >> n) & 0xffffu, 16); }
  if (n) s.put((uint32_t)v & ((1u << n) - 1u), n);
}

// Sinks: sym(symbol) for a Huffman symbol, put(bits, n <= 16) for raw bits
template <class W>
struct CodeSink {   // Huffman codes into a bit writer / counter
  const uint32_t* codes;
  W& w;
  __host__ __device__ void sym(int v) { put_sym(w, codes[v]); }
  __host__ __device__ void put(uint32_t v, int n) { w.put(v, n); }
};
template <class F>
struct SymSink {    // symbols only (counting)
  F f;
  __host__ __device__ void sym(int v) { f(v); }
  __host__ __device__ void put(uint32_t, int) {}
};

// AC first scan over zigzag coefficients ss..se of one block (get(k) = zigzag coefficient k)
template <class Get, class Sink>
__host__ __device__ inline BlockRun ac_first(const Get& get, int ss, int se, int al, Sink& s) {
  int r = 0, any = 0;
  for (int k = ss; k <= se; ++k) {
    const int v = get(k);
    const int a = (v < 0 ? -v : v) >> al;
    if (a == 0) { ++r; continue; }
    for (; r > 15; r -= 16) s.sym(0xf0);
    const int n = nbits(a);
    s.sym((r << 4) | n);
    s.put((uint32_t)(v < 0 ? ~a : a) & ((1u << n) - 1u), n);
    r = 0;
    any = 1;
  }
  return {any, r > 0, 0};
}

// AC refinement scan: newly non-zero coefficients (|v| >> al == 1) get (r, 1) and a sign bit; coefficients non-zero
// before get one correction bit, buffered until the next symbol.  ZRLs are emitted only up to the last newly non-zero
// coefficient.  The correction bits left after the last symbol go to tail(bits, n) (MSB first, n <= 63).
template <class Get, class Sink, class Tail>
__host__ __device__ inline BlockRun ac_refine(const Get& get, int ss, int se, int al, Sink& s, Tail&& tail) {
  int eob = -1;
  for (int k = ss; k <= se; ++k) {
    const int v = get(k);
    if (((v < 0 ? -v : v) >> al) == 1) eob = k;
  }
  int r = 0, br = 0, any = 0;
  unsigned long long buf = 0;
  for (int k = ss; k <= se; ++k) {
    const int v = get(k);
    const int a = (v < 0 ? -v : v) >> al;
    if (a == 0) { ++r; continue; }
    while (r > 15 && k <= eob) {
      s.sym(0xf0);
      r -= 16;
      put_bits(s, buf, br);
      buf = 0; br = 0;
      any = 1;
    }
    if (a > 1) { buf = (buf << 1) | (unsigned)(a & 1); ++br; continue; }
    s.sym((r << 4) | 1);
    s.put(v < 0 ? 0u : 1u, 1);
    put_bits(s, buf, br);
    buf = 0; br = 0; r = 0;
    any = 1;
  }
  tail(buf, br);
  return {any, (r > 0 || br > 0) ? 1 : 0, br};
}
struct NoTail {
  __host__ __device__ void operator()(unsigned long long, int) const {}
};

// Block j of AC scan s of an nc-component script: its own symbols and bits into `s` (get(k) = zigzag coefficient k)
template <class Get, class Sink, class Tail>
__host__ __device__ inline BlockRun ac_block(int nc, int scan, const Get& get, Sink& s, Tail&& tail) {
  const Scan sc = script(nc, scan);
  if (sc.ah == 0) return ac_first(get, sc.ss, sc.se, sc.al, s);
  return ac_refine(get, sc.ss, sc.se, sc.al, s, tail);
}
template <class Get, class Sink, class Tail>
__host__ __device__ inline BlockRun ac_block(int scan, const Get& get, Sink& s, Tail&& tail) {
  return ac_block(3, scan, get, s, tail);
}

// EOBn: the symbol of a run of E >= 1 blocks, followed by n = floor(log2 E) bits of E
__host__ __device__ inline int eob_bits_n(unsigned e) { return nbits((int)e) - 1; }
template <class Sink>
__host__ __device__ inline void emit_eob(Sink& s, unsigned e) {
  const int n = eob_bits_n(e);
  s.sym(n << 4);
  if (n) s.put(e & ((1u << n) - 1u), n);
}

// ------------------------------------------------------------------ the run state machine, in parallel form
// Flush after block x, given inclusive prefix sums over the scan's blocks of e (pe), c (pc) and hard (ph, the count of
// blocks after which a hard flush falls), read through accessors taking absolute indices.  From a run starting at j
// (first block j, last block of the scan `last`): the block after which that run is flushed.
template <class PE, class PC, class PH>
__host__ __device__ inline long long run_end(long long j, long long last, const PE& pe, const PC& pc, const PH& ph,
                                             long long eob_max = kEobMax, long long corr = kCorrFlush) {
  // hard end: the first x >= j with ph(x) > ph(j - 1)
  const unsigned long long h0 = j ? ph(j - 1) : 0;
  long long lo = j, hi = last;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (ph(mid) > h0) hi = mid; else lo = mid + 1;
  }
  const long long hend = lo;
  // threshold: the first x in [j, hend] with e sum >= eob_max or c sum > corr
  const unsigned long long e0 = j ? pe(j - 1) : 0, c0 = j ? pc(j - 1) : 0;
  lo = j; hi = hend;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (pe(mid) - e0 >= (unsigned long long)eob_max || pc(mid) - c0 > (unsigned long long)corr) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// ------------------------------------------------------------------ headers
// The frame header: common_header's SOI .. SOF0 with SOF2's marker (make_header(W, H, o) of the baseline encoder)
// (prefix_bytes(o.nc) bytes)
inline void frame_prefix(int W, int H, const Opts& o, uint8_t* out) {
  uint8_t full[kMaxHeaderBytes];
  make_header(W, H, o, full);
  const int n = prefix_bytes(o.nc);
  memcpy(out, full, n);
  out[n - (10 + 3 * o.nc) + 1] = 0xc2;   // SOF0 -> SOF2
}

// DHT of one optimised table: class cls, id, bits[16] / vals
__host__ __device__ inline int dht(uint8_t* out, int cls, int id, const uint8_t* bits, const uint8_t* vals) {
  int n = 0;
  for (int l = 0; l < 16; ++l) n += bits[l];
  const int len = 2 + 1 + 16 + n;
  int o = 0;
  out[o++] = 0xff; out[o++] = 0xc4; out[o++] = (uint8_t)(len >> 8); out[o++] = (uint8_t)len;
  out[o++] = (uint8_t)((cls << 4) | id);
  for (int l = 0; l < 16; ++l) out[o++] = bits[l];
  for (int k = 0; k < n; ++k) out[o++] = vals[k];
  return o;
}

// Scan s's header: its DHTs (tables of slots t, bits[t] / vals[t]), DRI before scan 0's SOS when rst > 0, SOS
__host__ __device__ inline int scan_header(int nc, int s, int rst, const uint8_t (*bits)[16], const uint8_t (*vals)[256],
                                           uint8_t* out) {
  const Scan sc = script(nc, s);
  int o = 0;
  if (sc.ss == 0 && sc.ah == 0) {
    o += dht(out + o, 0, 0, bits[0], vals[0]);
    if (sc.comp == 3) o += dht(out + o, 0, 1, bits[1], vals[1]);
  } else if (sc.ss > 0) {
    o += dht(out + o, 1, sc.comp ? 1 : 0, bits[ac_slot(nc, s)], vals[ac_slot(nc, s)]);
  }
  if (s == 0 && rst) {
    out[o++] = 0xff; out[o++] = 0xdd; out[o++] = 0; out[o++] = 4;
    out[o++] = (uint8_t)(rst >> 8); out[o++] = (uint8_t)rst;
  }
  const int ns = sc.comp == 3 ? 3 : 1;   // components in the scan
  out[o++] = 0xff; out[o++] = 0xda; out[o++] = 0; out[o++] = (uint8_t)(6 + 2 * ns); out[o++] = (uint8_t)ns;
  for (int c = 0; c < 3; ++c) {
    if (sc.comp != 3 && sc.comp != c) continue;
    out[o++] = (uint8_t)(c + 1);
    out[o++] = sc.ss == 0 ? (sc.ah == 0 && c ? 0x10 : 0x00) : (c ? 0x01 : 0x00);
  }
  out[o++] = (uint8_t)sc.ss; out[o++] = (uint8_t)sc.se; out[o++] = (uint8_t)((sc.ah << 4) | sc.al);
  return o;
}
__host__ __device__ inline int scan_header(int s, int rst, const uint8_t (*bits)[16], const uint8_t (*vals)[256], uint8_t* out) {
  return scan_header(3, s, rst, bits, vals, out);
}

// ------------------------------------------------------------------ bound
// (the grey script's AC scans are the luma scans of the YCbCr one, and it has no chroma scans)
inline unsigned long long total_intervals(const Geom& g, int rst) {
  unsigned long long ints = 0;
  for (int s = 0; s < scans(g.nc); ++s) ints += scan_intervals(g, s, rst);
  return ints;
}
inline unsigned long long entropy_bound_bits(const Geom& g, int rst) {
  unsigned long long bits = 0;
  bits += (unsigned long long)blocks_per_image(g) * (kDcBits + 1);
  bits += (unsigned long long)g.wb * g.hb * kLumaAcBits + (g.nc == 1 ? 0ull : 2ull * g.mcux * g.mcuy * kChromaAcBits);
  return bits + 7 * total_intervals(g, rst);
}
inline unsigned long long progressive_bound(const Geom& g, int rst) {
  return prefix_bytes(g.nc) + prog_header_bytes(g.nc) + 2 * ((entropy_bound_bits(g, rst) + 7) / 8) +
         2 * (total_intervals(g, rst) - scans(g.nc)) + 2;
}


// ------------------------------------------------------------------ device pipeline (bevk_api.cu: jpeg_prog_enqueue)
// After k_jpeg_blocks, over the n * T blocks of all scans of all images (T = Layout.blk[10] per image, the "scan blocks";
// global index J), and the n * S restart intervals ("segments", S = Layout.seg[10]):
//   k_jpeg_prog_desc    per scan block: BlockRun (AC scans) -> desc bits; DC scans code a symbol or a bit per block
//   k_jpeg_prog_hard    marks the blocks after which a hard flush falls; inclusive sums of e, c and hard (CUB)
//   k_jpeg_prog_next    next(J) = run_end(J) + 1 and the roots (scan starts, blocks after a hard flush)
//   k_jpeg_prog_jump    pointer doubling: marks every run start that is reached; a max-scan gives each block its run start
//   k_jpeg_prog_count   symbol counts per image and table (own symbols + the EOBn of each flush)
//   k_jpeg_prog_huff    ten optimal tables per image, their codes, and the ten scan headers
//   k_jpeg_prog_bits    bits per scan block (own bits + a flush's EOBn code, its bits and the run's correction bits)
//   k_jpeg_prog_segs    padded bits per segment and the bytes inserted before it (scan header or RSTn); scans (CUB)
//   k_jpeg_prog_pack    every block writes its codes; correction bits go after the EOBn of their run's flush
//   k_jpeg_prog_ffcount / k_jpeg_prog_layout / k_jpeg_prog_stuff  stuffing, sizes, frame header + EOI, and the data
//                       with each scan's header and the RSTn markers put in front of their segments
// Scratch: 53 bytes per scan block (about 5.3 scan blocks per coefficient block at 4:2:0) besides the 128-byte
// coefficient blocks, 16 per segment and 12 KB per image of tables and headers.
constexpr int kHdrStride = 256;   // bytes per (image, scan) header slot (>= kMaxScanHeader)
enum : uint32_t { kDescSym = 1u, kDescE = 2u, kDescHard = 1u << 9 };
__host__ __device__ inline int desc_c(uint32_t d) { return (int)((d >> 2) & 127u); }

struct ProgArgs {
  int n, rst;
  Geom g;
  long long nblk;                // coefficient blocks per image
  Layout L;
  long long T, S;                // scan blocks and segments per image
  const int16_t* coef;
  uint32_t* desc;                // [n * T]
  unsigned long long *pe, *pc;   // [n * T] inclusive sums of e and c
  unsigned* ph;                  // [n * T] inclusive sums of hard
  unsigned *jump, *jump2;        // [n * T + 1]
  uint8_t* mark;                 // [n * T + 1]
  unsigned* rs;                  // [n * T] run start of each block
  unsigned* counts;              // [n][kTables][256]
  uint32_t* codes;               // [n][kTables][256]
  uint8_t* hdrs;                 // [n][kScans][kHdrStride]
  int* hlen;                     // [n][kScans]
  unsigned long long *bits, *offs;   // [n * T]
  unsigned long long *ilen, *iofs;   // [n * S]
  unsigned *ins, *insx;              // [n * S]
  uint32_t* words;
  long long words_img;
  int chunks_img;
  unsigned *ffcnt, *ffscan;
  const uint8_t* prefix;         // prefix_bytes(g.nc)
  uint8_t* out;
  unsigned long long *out_off, *sizes;
};

struct ScanPos {   // where global scan block J lies
  int i, s;
  long long j, first, last;   // index in its scan; the global indices of the scan's first and last blocks
};
__device__ inline ScanPos scan_pos(const ProgArgs& a, long long J) {
  ScanPos p;
  p.i = (int)(J / a.T);
  const long long l = J - p.i * a.T;
  p.s = scan_of(a.L.blk, l);
  p.j = l - a.L.blk[p.s];
  p.first = J - p.j;
  p.last = p.first + (a.L.blk[p.s + 1] - a.L.blk[p.s]) - 1;
  return p;
}
// segment (image-local) of block j of scan s, and the global index of its last block
template <int NC>
__device__ inline long long seg_of(const ProgArgs& a, int s, long long j) {
  return a.L.seg[s] + (a.rst ? j / unit_blocks(NC, a.g, s) / a.rst : 0);
}
template <int NC>
__device__ inline bool interval_last(const ProgArgs& a, const ScanPos& p) {
  if (p.j == p.last - p.first) return true;
  const int ub = unit_blocks(NC, a.g, p.s);
  return a.rst && (p.j + 1) % ub == 0 && ((p.j + 1) / ub) % a.rst == 0;
}

struct CoefDC {   // DC of image-local slot b of image i
  const int16_t* c;
  __device__ int operator()(long long b) const { return __ldg(c + b * 64); }
};
struct PE { const unsigned long long* p; __device__ unsigned long long operator()(long long i) const { return p[i]; } };
struct PH { const unsigned* p; __device__ unsigned long long operator()(long long i) const { return p[i]; } };

// the run of flush block J: (E, C) of the run ending at J when a flush falls after J (mark[J + 1]), else E = 0
__device__ inline void flush_run(const ProgArgs& a, long long J, unsigned& E, unsigned& C) {
  E = C = 0;
  if (!a.mark[J + 1]) return;
  const long long s0 = a.rs[J];
  E = (unsigned)(a.pe[J] - (s0 ? a.pe[s0 - 1] : 0));
  C = (unsigned)(a.pc[J] - (s0 ? a.pc[s0 - 1] : 0));
}

template <int NC = 3>
__global__ void k_jpeg_prog_desc(ProgArgs a) {
  const long long J = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (J >= a.n * a.T) return;
  const ScanPos p = scan_pos(a, J);
  if (!is_ac(NC, p.s)) { a.desc[J] = kDescSym | kDescHard; return; }
  struct Null { __device__ void sym(int) {} __device__ void put(uint32_t, int) {} } ns;
  const int16_t* c = a.coef + ((long long)p.i * a.nblk + scan_slot(NC, a.g, p.s, p.j)) * 64;
  const BlockRun r = ac_block(NC, p.s, Zigzag16{c}, ns, NoTail{});
  a.desc[J] = (r.sym ? kDescSym : 0u) | (r.e ? kDescE : 0u) | ((uint32_t)r.c << 2);
}

template <int NC = 3>
__global__ void k_jpeg_prog_hard(ProgArgs a) {
  const long long J = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (J >= a.n * a.T) return;
  const ScanPos p = scan_pos(a, J);
  if (!is_ac(NC, p.s)) return;
  if (interval_last<NC>(a, p) || (a.desc[J + 1] & kDescSym)) a.desc[J] |= kDescHard;
}

struct DescE { __host__ __device__ unsigned long long operator()(uint32_t d) const { return (d & kDescE) ? 1ull : 0ull; } };
struct DescC { __host__ __device__ unsigned long long operator()(uint32_t d) const { return (unsigned long long)desc_c(d); } };
struct DescH { __host__ __device__ unsigned operator()(uint32_t d) const { return (d & kDescHard) ? 1u : 0u; } };
struct MarkIndex {   // J if block J starts a reached run, else 0
  const uint8_t* mark;
  __host__ __device__ unsigned operator()(unsigned J) const { return mark[J] ? J : 0u; }
};
struct MaxU { __host__ __device__ unsigned operator()(unsigned x, unsigned y) const { return x > y ? x : y; } };

template <int NC = 3>
__global__ void k_jpeg_prog_next(ProgArgs a) {
  const long long N = a.n * a.T, J = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (J > N) return;
  if (J == N) { a.jump[N] = (unsigned)N; a.mark[N] = 1; return; }
  const ScanPos p = scan_pos(a, J);
  a.mark[J] = p.j == 0 || (a.desc[J - 1] & kDescHard) ? 1 : 0;
  a.jump[J] = (unsigned)(is_ac(NC, p.s) ? run_end(J, p.last, PE{a.pe}, PE{a.pc}, PH{a.ph}) + 1 : J + 1);
}

// one round of pointer doubling: marked nodes mark their jump target, then every jump doubles
__global__ void k_jpeg_prog_jump(const unsigned* jump, unsigned* jump2, uint8_t* mark, long long total) {
  const long long J = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (J > total) return;
  const unsigned t = jump[J];
  if (mark[J]) mark[t] = 1;
  jump2[J] = jump[t];
}

template <int NC, class Sink>
__device__ inline void dc_first_emit(const ProgArgs& a, const ScanPos& p, Sink& s) {
  const int diff = dc_first_diff(NC, a.g, a.rst, p.j, script(NC, p.s).al, CoefDC{a.coef + (long long)p.i * a.nblk * 64});
  const int n = nbits(diff < 0 ? -diff : diff);
  s.sym(n);
  if (n) s.put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1u), n);
}
template <int NC>
__device__ inline int dc_refine_bit(const ProgArgs& a, const ScanPos& p) {
  return (resolved_dc_at(NC, a.g, p.j, CoefDC{a.coef + (long long)p.i * a.nblk * 64}) >> script(NC, p.s).al) & 1;
}
template <int NC>
__device__ inline int table_of(const ProgArgs& a, const ScanPos& p) {
  return is_ac(NC, p.s) ? ac_slot(NC, p.s) : scan_comp(NC, a.g, p.s, p.j) ? 1 : 0;
}

template <int NC = 3>
__global__ void k_jpeg_prog_count(ProgArgs a) {
  const long long J = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (J >= a.n * a.T) return;
  const ScanPos p = scan_pos(a, J);
  const Scan sc = script(NC, p.s);
  if (sc.ss == 0 && sc.ah) return;
  unsigned* cnt = a.counts + ((size_t)p.i * kTables + table_of<NC>(a, p)) * 256;
  auto add = [cnt](int v) { atomicAdd(cnt + v, 1u); };
  SymSink<decltype(add)> s{add};
  if (sc.ss == 0) { dc_first_emit<NC>(a, p, s); return; }
  const int16_t* c = a.coef + ((long long)p.i * a.nblk + scan_slot(NC, a.g, p.s, p.j)) * 64;
  ac_block(NC, p.s, Zigzag16{c}, s, NoTail{});
  unsigned E, C;
  flush_run(a, J, E, C);
  if (E) add(eob_bits_n(E) << 4);
}

constexpr int kProgHuffImages = 12, kProgHuffThreads = kProgHuffImages * kTables;
template <int NC = 3>
__global__ void __launch_bounds__(kProgHuffThreads) k_jpeg_prog_huff(ProgArgs a) {
  __shared__ uint8_t sbits[kProgHuffImages][kTables][16];
  __shared__ uint8_t svals[kProgHuffImages][kTables][256];
  const int li = threadIdx.x / kTables, t = threadIdx.x % kTables;
  const int i = blockIdx.x * kProgHuffImages + li;
  if (i < a.n && t < tables(NC)) {
    long long freq[257];
    for (int k = 0; k < 256; ++k) freq[k] = a.counts[((size_t)i * kTables + t) * 256 + k];
    gen_optimal_table(freq, sbits[li][t], svals[li][t]);
    huff_codes(sbits[li][t], svals[li][t], a.codes + ((size_t)i * kTables + t) * 256, 256);
  }
  __syncthreads();
  if (i < a.n && t < scans(NC))   // thread t writes scan t's header
    a.hlen[i * kScans + t] = scan_header(NC, t, a.rst, sbits[li], svals[li], a.hdrs + ((size_t)i * kScans + t) * kHdrStride);
}

template <int NC = 3>
__global__ void k_jpeg_prog_bits(ProgArgs a) {
  const long long J = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (J >= a.n * a.T) return;
  const ScanPos p = scan_pos(a, J);
  const Scan sc = script(NC, p.s);
  if (sc.ss == 0 && sc.ah) { a.bits[J] = 1; return; }
  const uint32_t* codes = a.codes + ((size_t)p.i * kTables + table_of<NC>(a, p)) * 256;
  BitCount cnt;
  CodeSink<BitCount> s{codes, cnt};
  if (sc.ss == 0) {
    dc_first_emit<NC>(a, p, s);
  } else {
    const int16_t* c = a.coef + ((long long)p.i * a.nblk + scan_slot(NC, a.g, p.s, p.j)) * 64;
    ac_block(NC, p.s, Zigzag16{c}, s, NoTail{});
    unsigned E, C;
    flush_run(a, J, E, C);
    if (E) { emit_eob(s, E); cnt.n += C; }
  }
  a.bits[J] = cnt.n;
}

// segment g of image i: its scan, index within the scan, and its first and last global scan blocks
template <int NC>
__device__ inline void seg_blocks(const ProgArgs& a, int i, long long g, int& s, long long& t, long long& first, long long& last) {
  s = scan_of(a.L.seg, g);
  t = g - a.L.seg[s];
  const long long per = a.rst ? (long long)a.rst * unit_blocks(NC, a.g, s) : a.L.blk[s + 1] - a.L.blk[s];
  const long long base = (long long)i * a.T + a.L.blk[s], end = (long long)i * a.T + a.L.blk[s + 1];
  first = base + t * per;
  last = (first + per < end ? first + per : end) - 1;
}

template <int NC = 3>
__global__ void k_jpeg_prog_segs(ProgArgs a) {
  const long long G = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (G >= a.n * a.S) return;
  const int i = (int)(G / a.S);
  int s;
  long long t, first, last;
  seg_blocks<NC>(a, i, G - i * a.S, s, t, first, last);
  a.ilen[G] = (a.offs[last] + a.bits[last] - a.offs[first] + 7) & ~7ull;
  a.ins[G] = t == 0 ? (unsigned)a.hlen[i * kScans + s] : 2u;
}

__device__ inline unsigned long long prog_image_bits(const ProgArgs& a, int i) {
  const long long l = (long long)(i + 1) * a.S - 1;
  return a.iofs[l] + a.ilen[l] - a.iofs[(long long)i * a.S];
}

__global__ void k_jpeg_prog_zero(ProgArgs a) {
  for (int i = 0; i < a.n; ++i) {
    const long long used = (long long)((prog_image_bits(a, i) + 31) >> 5);
    uint32_t* w = a.words + i * a.words_img;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < used; j += (long long)gridDim.x * blockDim.x) w[j] = 0;
  }
}

// bit position of scan block J in its image's region
template <int NC>
__device__ inline unsigned long long block_pos(const ProgArgs& a, const ScanPos& p, long long J) {
  const long long g = seg_of<NC>(a, p.s, p.j), G = (long long)p.i * a.S + g;
  int s;
  long long t, first, last;
  seg_blocks<NC>(a, p.i, g, s, t, first, last);
  return a.iofs[G] - a.iofs[(long long)p.i * a.S] + a.offs[J] - a.offs[first];
}

template <int NC = 3>
__global__ void k_jpeg_prog_pack(ProgArgs a) {
  const long long J = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (J >= a.n * a.T) return;
  const ScanPos p = scan_pos(a, J);
  const Scan sc = script(NC, p.s);
  uint32_t* words = a.words + p.i * a.words_img;
  const unsigned long long pos = block_pos<NC>(a, p, J);
  BitWriter wr(words, pos);
  if (sc.ss == 0 && sc.ah) {
    wr.put((uint32_t)dc_refine_bit<NC>(a, p), 1);
  } else {
    CodeSink<BitWriter> s{a.codes + ((size_t)p.i * kTables + table_of<NC>(a, p)) * 256, wr};
    if (sc.ss == 0) {
      dc_first_emit<NC>(a, p, s);
    } else {
      const int16_t* c = a.coef + ((long long)p.i * a.nblk + scan_slot(NC, a.g, p.s, p.j)) * 64;
      // this block's correction bits after its last symbol go to its run's flush: after the EOBn code of block x
      auto tail = [&](unsigned long long v, int n) {
        if (!n) return;
        const long long s0 = a.rs[J];
        const long long x = run_end(s0, p.last, PE{a.pe}, PE{a.pc}, PH{a.ph});
        const unsigned long long c0 = s0 ? a.pc[s0 - 1] : 0;
        const unsigned long long crun = a.pc[x] - c0;
        const unsigned long long at = block_pos<NC>(a, p, x) + a.bits[x] - crun + (J ? a.pc[J - 1] : 0) - c0;
        BitWriter tw(words, at);
        put_bits(tw, v, n);
        tw.flush();
      };
      ac_block(NC, p.s, Zigzag16{c}, s, tail);
      unsigned E, C;
      flush_run(a, J, E, C);
      if (E) emit_eob(s, E);
    }
  }
  wr.flush();
  if (interval_last<NC>(a, p)) {   // an interval's last block pads its byte with 1 bits
    const unsigned long long end = pos + a.bits[J];
    const int pad = (int)((8 - (end & 7)) & 7);
    if (pad) {
      BitWriter pw(words, end);
      pw.put((1u << pad) - 1u, pad);
      pw.flush();
    }
  }
}

__global__ void k_jpeg_prog_ffcount(ProgArgs a) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)a.n * a.chunks_img) return;
  const int i = (int)(t / a.chunks_img), c = (int)(t - (long long)i * a.chunks_img);
  const long long nbytes = (long long)(prog_image_bits(a, i) >> 3), off = (long long)c * kChunk;
  if (off >= nbytes) return;
  const uint8_t* p = reinterpret_cast<const uint8_t*>(a.words + i * a.words_img) + off;
  a.ffcnt[t] = (unsigned)count_ff(p, (int)(nbytes - off < kChunk ? nbytes - off : kChunk));
}

__device__ inline unsigned inserted_before(const ProgArgs& a, int i, long long g) {   // bytes inserted before segment g
  const long long G0 = (long long)i * a.S;
  if (g < a.S) return a.insx[G0 + g] - a.insx[G0];
  return a.insx[G0 + a.S - 1] + a.ins[G0 + a.S - 1] - a.insx[G0];
}

template <int NC = 3>
__global__ void k_jpeg_prog_layout(ProgArgs a) {
  if (threadIdx.x == 0) {
    unsigned long long off = 0;
    for (int i = 0; i < a.n; ++i) {
      const unsigned long long nbytes = prog_image_bits(a, i) >> 3;
      const long long c0 = (long long)i * a.chunks_img, cl = c0 + (long long)((nbytes + kChunk - 1) / kChunk) - 1;
      const unsigned ff = a.ffscan[cl] + a.ffcnt[cl] - a.ffscan[c0];
      const unsigned long long size = prefix_bytes(NC) + inserted_before(a, i, a.S) + nbytes + ff + 2;
      a.out_off[i] = off;
      a.sizes[i] = size;
      off += size;
    }
  }
  __syncthreads();
  for (long long j = threadIdx.x; j < (long long)a.n * prefix_bytes(NC); j += blockDim.x) {
    const int i = (int)(j / prefix_bytes(NC)), h = (int)(j - (long long)i * prefix_bytes(NC));
    a.out[a.out_off[i] + h] = a.prefix[h];
  }
  for (int i = threadIdx.x; i < a.n; i += blockDim.x) {
    uint8_t* e = a.out + a.out_off[i] + a.sizes[i] - 2;
    e[0] = 0xff;
    e[1] = 0xd9;
  }
}

// the byte where segment g of image i starts in its unstuffed data
__device__ inline unsigned long long seg_start(const ProgArgs& a, int i, long long g) {
  return (a.iofs[(long long)i * a.S + g] - a.iofs[(long long)i * a.S]) >> 3;
}

template <int NC = 3>
__global__ void k_jpeg_prog_stuff(ProgArgs a) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)a.n * a.chunks_img) return;
  const int i = (int)(t / a.chunks_img), c = (int)(t - (long long)i * a.chunks_img);
  const long long nbytes = (long long)(prog_image_bits(a, i) >> 3), off = (long long)c * kChunk;
  if (off >= nbytes) return;
  const uint8_t* p = reinterpret_cast<const uint8_t*>(a.words + i * a.words_img) + off;
  const int len = (int)(nbytes - off < kChunk ? nbytes - off : kChunk);
  long long lo = 0, hi = a.S;   // the first segment starting at or past off
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (seg_start(a, i, mid) < (unsigned long long)off) lo = mid + 1;
    else hi = mid;
  }
  uint8_t* o = a.out + a.out_off[i] + prefix_bytes(NC) + inserted_before(a, i, lo) + off +
               (a.ffscan[t] - a.ffscan[(long long)i * a.chunks_img]);
  unsigned long long next = lo < a.S ? seg_start(a, i, lo) : ~0ull;
  for (int k = 0; k < len; ++k) {
    while ((unsigned long long)(off + k) == next) {   // scan header or RSTn before segment lo
      const int s = scan_of(a.L.seg, lo);
      const long long ts = lo - a.L.seg[s];
      if (ts == 0) {
        const uint8_t* h = a.hdrs + ((size_t)i * kScans + s) * kHdrStride;
        const int n = a.hlen[i * kScans + s];
        for (int q = 0; q < n; ++q) *o++ = h[q];
      } else {
        *o++ = 0xff;
        *o++ = (uint8_t)(0xd0 + ((ts - 1) & 7));
      }
      ++lo;
      next = lo < a.S ? seg_start(a, i, lo) : ~0ull;
    }
    *o++ = p[k];
    if (p[k] == 0xff) *o++ = 0;
  }
}

}  // namespace prog
}  // namespace jpeg
}  // namespace bevk
