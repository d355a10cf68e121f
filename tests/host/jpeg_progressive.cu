// Host form of the progressive JPEG coder (bevk_jpeg_prog.cuh): the baseline encoder's quantised coefficients, then the
// ten scans with libjpeg's serial EOB-run / correction-bit state machine, per-scan optimal tables, headers, pads, RSTn and
// stuffing, run serially over whole images so tests/test_host_jpeg_progressive.py can compare the streams with
// cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q] + params).  Every AC scan is also resolved in the kernels'
// parallel form (run_end over prefix sums, pointer doubling over the run starts); its flush points must equal the
// serial ones.
//
//   jpeg_progressive <in.bin> <out.bin> [mutation]
//     in : records of int32 width, height, quality, n, n ints of params, then width*height*3 bytes (BGR, dense)
//     out: per record int32 ok, progressive, parallel_ok; uint64 flushes by cause (symbol, 0x7FFF, correction bits,
//          restart, end of scan), uint64 bound, uint64 stream size, the stream (none unless ok and progressive)
//     mutation (evidence that the corpus pins these rules): 1 flush at more than 1000 correction bits instead of 937,
//          2 scans 3 and 4 swapped, 3 DC shifted logically instead of arithmetically
// Built by tests/test_host_jpeg_progressive.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_jpeg_prog.cuh"

using namespace bevk::jpeg;
using namespace bevk::jpeg::prog;

enum Cause { kSym, kEob, kCorr, kRestart, kEnd };
static int g_mutation = 0;

struct Bits {   // the entropy-coded data of one scan: a bit list, Huffman codes or symbol counts
  std::vector<uint8_t> b;
  const uint32_t* codes = nullptr;
  long long* freq = nullptr;
  void put(uint32_t v, int n) { for (int i = n - 1; i >= 0; --i) b.push_back((v >> i) & 1); }
  void sym(int v) {
    if (freq) freq[v]++;
    else put_sym(*this, codes[v]);
  }
  void pad() { while (b.size() & 7) b.push_back(1); }
};

struct Flush { long long x; int cause; };

// One scan, serially as libjpeg codes it.  ints receives the byte offset of every restart interval in out.b.
static void serial_scan(const Geom& g, const Opts& o, int s, const std::vector<int16_t>& coef, Bits& out, const uint32_t* const* codes,
                        long long** freq, int corr, std::vector<Flush>* log, std::vector<size_t>* ints) {
  const Scan sc = script(s);
  const long long nb = scan_blocks(g, s);
  const int ub = unit_blocks(g, s);
  auto dc = [&](long long b) {
    const int v = coef[(size_t)b * 64];
    return v;
  };
  unsigned E = 0;
  std::vector<uint8_t> B;
  auto use = [&](int slot) { out.codes = codes ? codes[slot] : nullptr; out.freq = freq ? freq[slot] : nullptr; };
  auto flush = [&](long long x, int cause) {
    if (E) {
      use(ac_slot(s));
      emit_eob(out, E);
      for (uint8_t bit : B) out.put(bit, 1);
      if (log) log->push_back({x, cause});
    }
    E = 0;
    B.clear();
  };
  for (long long j = 0; j < nb; ++j) {
    const long long unit = j / ub;
    if (j % ub == 0) {
      if (o.rst && unit % o.rst == 0 && j > 0) {
        flush(j - 1, kRestart);
        out.pad();
      }
      if (o.rst && unit % o.rst == 0) ints->push_back(out.b.size() / 8);
      if (!o.rst && j == 0) ints->push_back(0);
    }
    const long long slot = scan_slot(g, s, j);
    if (sc.ss == 0) {
      if (sc.ah == 0) {
        int diff;
        if (g_mutation == 3) {   // logical shift of the DC values
          auto lsh = [&](long long b) { return (int)((unsigned)resolved_dc_at(g, b, dc) >> sc.al); };
          const int ny = g.hy * g.vy, bpm = ny + 2;
          const long long m = j / bpm;
          const int k = (int)(j - m * bpm);
          long long p = -1;
          if (k > 0 && k < ny) p = j - 1;
          else if (m > 0 && (o.rst == 0 || m % o.rst != 0)) p = (m - 1) * bpm + (k == 0 ? ny - 1 : k);
          diff = lsh(j) - (p < 0 ? 0 : lsh(p));
        } else {
          diff = dc_first_diff(g, o.rst, j, sc.al, dc);
        }
        use(scan_comp(g, s, j) ? 1 : 0);
        const int n = nbits(diff < 0 ? -diff : diff);
        out.sym(n);
        if (n) out.put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1u), n);
      } else {
        out.put((uint32_t)(resolved_dc_at(g, slot, dc) >> sc.al) & 1u, 1);
      }
      continue;
    }
    use(ac_slot(s));
    struct First {   // flushes the pending run before the block's first symbol
      Bits& o;
      bool first = true;
      decltype(flush)& f;
      long long j;
      void sym(int v) {
        if (first) { first = false; f(j - 1, kSym); }
        o.sym(v);
      }
      void put(uint32_t v, int n) { o.put(v, n); }
    } fs{out, true, flush, j};
    const int16_t* c = &coef[(size_t)slot * 64];
    std::vector<uint8_t> tail;
    const BlockRun r = ac_block(s, Zigzag16{c}, fs, [&](unsigned long long v, int n) {
      for (int i = n - 1; i >= 0; --i) tail.push_back((v >> i) & 1);
    });
    if (r.e) {
      ++E;
      B.insert(B.end(), tail.begin(), tail.end());
      if (E == (unsigned)kEobMax) flush(j, kEob);
      else if ((int)B.size() > corr) flush(j, kCorr);
    }
  }
  flush(nb - 1, kEnd);
  out.pad();
}

// The kernels' parallel resolution of scan s's runs: the blocks after which a non-empty run is flushed.
static std::vector<long long> parallel_flushes(const Geom& g, const Opts& o, int s, const std::vector<int16_t>& coef, int corr) {
  const long long nb = scan_blocks(g, s);
  const int ub = unit_blocks(g, s);
  std::vector<BlockRun> br((size_t)nb);
  for (long long j = 0; j < nb; ++j) {
    SymSink<void (*)(int)> none{[](int) {}};
    br[(size_t)j] = ac_block(s, Zigzag16{&coef[(size_t)scan_slot(g, s, j) * 64]}, none, NoTail{});
  }
  auto interval_last = [&](long long x) {
    if (x == nb - 1) return true;
    return o.rst && ((x + 1) % ub == 0) && ((x + 1) / ub) % o.rst == 0;
  };
  std::vector<unsigned long long> pe((size_t)nb), pc((size_t)nb), ph((size_t)nb);
  unsigned long long se = 0, sc = 0, sh = 0;
  std::vector<int> hard((size_t)nb);
  for (long long x = 0; x < nb; ++x) {
    hard[(size_t)x] = interval_last(x) || br[(size_t)x + 1].sym;
    se += br[(size_t)x].e; sc += br[(size_t)x].c; sh += hard[(size_t)x];
    pe[(size_t)x] = se; pc[(size_t)x] = sc; ph[(size_t)x] = sh;
  }
  auto PE = [&](long long i) { return pe[(size_t)i]; };
  auto PC = [&](long long i) { return pc[(size_t)i]; };
  auto PH = [&](long long i) { return ph[(size_t)i]; };
  std::vector<long long> jump((size_t)nb + 1), jump2((size_t)nb + 1);
  std::vector<uint8_t> mark((size_t)nb + 1, 0);
  for (long long j = 0; j < nb; ++j) {
    jump[(size_t)j] = run_end(j, nb - 1, PE, PC, PH, kEobMax, corr) + 1;
    mark[(size_t)j] = j == 0 || hard[(size_t)j - 1];
  }
  jump[(size_t)nb] = nb;
  mark[(size_t)nb] = 1;
  for (long long span = 1; span < 2 * (nb + 1); span *= 2) {   // pointer doubling
    for (long long j = 0; j <= nb; ++j)
      if (mark[(size_t)j]) mark[(size_t)jump[(size_t)j]] = 1;
    for (long long j = 0; j <= nb; ++j) jump2[(size_t)j] = jump[(size_t)jump[(size_t)j]];
    jump.swap(jump2);
  }
  std::vector<long long> out;
  long long start = 0;
  for (long long x = 0; x < nb; ++x) {
    if (!mark[(size_t)x + 1]) continue;
    if (pe[(size_t)x] - (start ? pe[(size_t)start - 1] : 0)) out.push_back(x);
    start = x + 1;
  }
  return out;
}

// libjpeg's stuffing: 0x00 after every 0xFF
static void stuff(const std::vector<uint8_t>& bits, size_t from, size_t to, std::vector<uint8_t>& s) {
  for (size_t p = from; p < to; ++p) {
    uint8_t v = 0;
    for (int k = 0; k < 8; ++k) v = (uint8_t)((v << 1) | bits[p * 8 + k]);
    s.push_back(v);
    if (v == 0xff) s.push_back(0);
  }
}

static std::vector<uint8_t> encode(const uint8_t* img, int W, int H, const Opts& o, unsigned long long* causes, int* par_ok) {
  Tables t;
  make_tables(o, &t);
  const Geom g = geom(W, H, o);
  const int ny = g.hy * g.vy, bpm = ny + 2;
  const long long nblk = blocks_per_image(g);
  std::vector<int16_t> coef((size_t)nblk * 64);
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
  const int corr = g_mutation == 1 ? 1000 : kCorrFlush;
  int order[kScans];
  for (int s = 0; s < kScans; ++s) order[s] = s;
  if (g_mutation == 2) { order[2] = 3; order[3] = 2; }
  std::vector<uint8_t> st(kPrefixBytes);
  frame_prefix(W, H, o, st.data());
  for (int k = 0; k < kScans; ++k) {
    const int s = order[k];
    // pass 1: symbol counts of this scan's tables, then jpeg_gen_optimal_table
    static long long freq[kTables][257];
    memset(freq, 0, sizeof freq);
    long long* fp[kTables];
    for (int q = 0; q < kTables; ++q) fp[q] = freq[q];
    Bits count;
    std::vector<size_t> ints;
    serial_scan(g, o, s, coef, count, nullptr, fp, corr, nullptr, &ints);
    uint8_t hb[kTables][16] = {}, hv[kTables][256] = {};
    static uint32_t codes[kTables][256];
    const uint32_t* cp[kTables];
    for (int q = 0; q < kTables; ++q) {
      cp[q] = codes[q];
      bool used = false;
      for (int v = 0; v < 256; ++v) used |= freq[q][v] != 0;
      if (!used) continue;
      gen_optimal_table(freq[q], hb[q], hv[q]);
      huff_codes(hb[q], hv[q], codes[q], 256);
    }
    // pass 2: the scan's data
    Bits data;
    std::vector<Flush> log;
    ints.clear();
    serial_scan(g, o, s, coef, data, cp, nullptr, corr, &log, &ints);
    for (const Flush& f : log) causes[f.cause]++;
    if (is_ac(s)) {
      const std::vector<long long> par = parallel_flushes(g, o, s, coef, corr);
      bool same = par.size() == log.size();
      for (size_t i = 0; same && i < par.size(); ++i) same = par[i] == log[i].x;
      if (!same) *par_ok = 0;
    }
    uint8_t hdr[kMaxScanHeader + 2 * kDcDhtMax + kDriBytes + 14];
    const int hl = scan_header(s, o.rst, hb, hv, hdr);
    st.insert(st.end(), hdr, hdr + hl);
    const size_t nbytes = data.b.size() / 8;
    for (size_t i = 0; i < ints.size(); ++i) {
      if (i) { st.push_back(0xff); st.push_back((uint8_t)(0xd0 + ((i - 1) & 7))); }
      stuff(data.b, ints[i], i + 1 < ints.size() ? ints[i + 1] : nbytes, st);
    }
  }
  st.push_back(0xff);
  st.push_back(0xd9);
  return st;
}

int main(int argc, char** argv) {
  if (argc < 3) { fprintf(stderr, "usage: jpeg_progressive <in.bin> <out.bin> [mutation]\n"); return 2; }
  if (argc > 3) g_mutation = atoi(argv[3]);
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
    read_flags(params.data(), n);
    Opts o;
    const int ok = normalise(q, params.data(), n, &o) ? 1 : 0;
    std::vector<uint8_t> s;
    unsigned long long causes[5] = {0, 0, 0, 0, 0}, bound = 0;
    int par_ok = 1;
    if (ok && o.progressive) {
      s = encode(img.data(), W, H, o, causes, &par_ok);
      bound = progressive_bound(geom(W, H, o), o.rst);
    }
    const int32_t meta32[3] = {ok, o.progressive, par_ok};
    const uint64_t meta[7] = {causes[0], causes[1], causes[2], causes[3], causes[4], bound, s.size()};
    fwrite(meta32, 4, 3, fo);
    fwrite(meta, 8, 7, fo);
    fwrite(s.data(), 1, s.size(), fo);
  }
  fclose(fi);
  fclose(fo);
  return 0;
}
