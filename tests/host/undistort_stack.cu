// Host form of the batched stand-alone gathers (bevk_undistort_stack): the per-thread bodies of k_gather
// (gather_frames) and k_gather4 (gather4_frames) from the library's own headers, driven over the same grid the
// device launches -- x, y and the grid-z frame groups of GATHER_NB -- so the frame loop and the 64-bit per-frame
// addressing run on a CPU.  Every 32-bit tap word and every tap byte is audited against the frame layout.
//
//   undistort_stack run <in.bin> <out.bin>
//     in : records of int32 mode (0 map, 1 fused model), channels, linear, words (1: the 4-pixel word path), sw, sh, dw,
//          dh, n, src_off (base address % 4), then int64 spitch, sistride, dpitch, distride; mode 0: map1 (int16[dh][dw][2]),
//          map2 (uint16[dh][dw]); mode 1: float64 K[9], D[5], P[9], model; then the source bytes
//          ((n-1)*sistride + (sh-1)*spitch + sw*channels) and the destination's initial bytes (same rule)
//     out: per record the destination bytes after the gather
//   undistort_stack audit
//     word audit of gather_px over frames whose right edge falls at every byte phase: the taps of every source
//     position around the frame (in and out of it) are gathered from 2-frame batches with tight and padded pitches
// Every load outside its frame row's bytes (word loads: rounded out to whole 32-bit words), or misaligned, fails the
// run (exit 1).  Built by tests/test_host_undistort_stack.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_device.cuh"
#include "../../cameracalibration_b200/csrc/bevk_gather4.cuh"

using namespace bevk;

// the frame layout the loads are audited against
static struct Layout {
  const uint8_t* base = nullptr;
  long long sistride = 0, spitch = 0;
  int n = 0, sw = 0, sh = 0, ch = 0;
  long long words = 0, bytes = 0, bad = 0;
} g;

// the frame row the address falls into: false outside every row's pitch; row_lo/row_hi: the row's bytes
[[maybe_unused]] static bool locate(const uint8_t* p, long long& row_lo, long long& row_hi) {
  const long long a = (long long)(p - g.base);
  if (a < 0) return false;
  const long long f = g.n > 1 ? a / g.sistride : 0;
  if (f >= g.n) return false;
  const long long r = (a - f * g.sistride) / g.spitch;
  if (r >= g.sh) return false;
  row_lo = f * g.sistride + r * g.spitch;
  row_hi = row_lo + (long long)g.sw * g.ch;
  return true;
}

// __host__ __device__ only to match gather_px's qualifiers: the harness never compiles a kernel that uses it
struct Audit {
  __host__ __device__ static unsigned w32(const uint8_t* p) {
#ifdef __CUDA_ARCH__
    return 0u;
#else
    ++g.words;
    long long lo, hi;
    const long long a = (long long)(p - g.base);
    // the row's bytes rounded out to whole words, in absolute addresses
    const uintptr_t b = reinterpret_cast<uintptr_t>(g.base), q = reinterpret_cast<uintptr_t>(p);
    if (!locate(p, lo, hi) || (q & 3) != 0 || q < ((b + lo) & ~(uintptr_t)3) || q + 4 > ((b + hi + 3) & ~(uintptr_t)3)) {
      if (g.bad++ < 10) fprintf(stderr, "word load at frame offset %lld outside its row's words\n", a);
      return 0u;
    }
    return ldg32(p);
#endif
  }
  __host__ __device__ static int b8(const uint8_t* p) {
#ifdef __CUDA_ARCH__
    return 0;
#else
    ++g.bytes;
    long long lo, hi;
    const long long a = (long long)(p - g.base);
    if (!locate(p, lo, hi) || a < lo || a >= hi) {
      if (g.bad++ < 10) fprintf(stderr, "byte load at frame offset %lld outside its row\n", a);
      return 0;
    }
    return ldg8(p);
#endif
  }
};

static void* alloc(size_t bytes) {   // 64-byte aligned (k_gather4's 16-byte map loads)
  void* p = nullptr;
  if (posix_memalign(&p, 64, bytes + 64)) return nullptr;
  memset(p, 0, bytes + 64);
  return p;
}

// the device grid: blockIdx.z frame groups, then every (x, y) thread of k_gather / k_gather4
template <int MODE>
static void run_grid(const GatherArgs& a, int ch, int linear, int words) {
  for (int f0 = 0; f0 < a.n; f0 += GATHER_NB)
    for (int y = 0; y < a.dh; ++y) {
      if (words) {
        for (int x4 = 0; x4 < a.dw; x4 += 4) {     // the kernel the library launches for this n
          if (a.n == 1) gather4_frames<MODE, 1, Audit>(a, x4, y, f0);
          else gather4_frames<MODE, GATHER_NB, Audit>(a, x4, y, f0);
        }
        continue;
      }
      for (int x = 0; x < a.dw; ++x) {
        if (linear) {
          if (ch == 1) gather_frames<MODE, 1, 1>(a, x, y, f0);
          else if (ch == 3) gather_frames<MODE, 3, 1>(a, x, y, f0);
          else gather_frames<MODE, 4, 1>(a, x, y, f0);
        } else {
          if (ch == 1) gather_frames<MODE, 1, 0>(a, x, y, f0);
          else if (ch == 3) gather_frames<MODE, 3, 0>(a, x, y, f0);
          else gather_frames<MODE, 4, 0>(a, x, y, f0);
        }
      }
    }
}

static int mode_run(const char* in_path, const char* out_path) {
  FILE* fi = fopen(in_path, "rb");
  FILE* fo = fopen(out_path, "wb");
  if (!fi || !fo) return 4;
  int32_t h[10];
  while (fread(h, 4, 10, fi) == 10) {
    const int mode = h[0], ch = h[1], linear = h[2], words = h[3], sw = h[4], sh = h[5], dw = h[6], dh = h[7], n = h[8], off = h[9];
    int64_t st[4];
    if (fread(st, 8, 4, fi) != 4) return 5;
    GatherArgs a{};
    std::vector<double> xs;
    a.sw = sw; a.sh = sh; a.spitch = st[0]; a.sistride = st[1]; a.dw = dw; a.dh = dh; a.dpitch = st[2]; a.distride = st[3]; a.n = n;
    const size_t npx = (size_t)dw * dh;
    short2* m1 = static_cast<short2*>(alloc(npx * 4));
    unsigned short* m2 = static_cast<unsigned short*>(alloc(npx * 2));
    if (mode == 0) {
      if (fread(m1, 4, npx, fi) != npx || fread(m2, 2, npx, fi) != npx) return 5;
      a.map1 = m1; a.map2 = m2;
    } else {
      double K[9], D[5], P[9], model;
      if (fread(K, 8, 9, fi) != 9 || fread(D, 8, 5, fi) != 5 || fread(P, 8, 9, fi) != 9 || fread(&model, 8, 1, fi) != 1) return 5;
      memset(&a.cm, 0, sizeof a.cm);
      if (!inv3(P, a.cm.iR)) return 3;
      for (int i = 0; i < 5; ++i) a.cm.k[i] = D[i];
      a.cm.fx = K[0]; a.cm.fy = K[4]; a.cm.cx = K[2]; a.cm.cy = K[5];
      a.cm.model = (int)model; a.cm.w = dw; a.cm.h = dh;
      if (xs_table_applies(a.cm)) {   // as bevk_api.cu attaches it (attach_xs_table)
        xs.resize(dw);
        fill_xs_table(a.cm, xs.data());
        a.cm.xs = xs.data();
      }
    }
    const size_t sbytes = (size_t)((n - 1) * st[1] + (sh - 1) * st[0] + (int64_t)sw * ch);
    const size_t dbytes = (size_t)((n - 1) * st[3] + (dh - 1) * st[2] + (int64_t)dw * ch);
    uint8_t* sbuf = static_cast<uint8_t*>(alloc(sbytes + 4));
    uint8_t* dbuf = static_cast<uint8_t*>(alloc(dbytes));
    if (!sbuf || !dbuf || fread(sbuf + off, 1, sbytes, fi) != sbytes || fread(dbuf, 1, dbytes, fi) != dbytes) return 5;
    a.src = sbuf + off; a.dst = dbuf;
    g.base = a.src; g.sistride = n > 1 ? st[1] : 0; g.spitch = st[0]; g.n = n; g.sw = sw; g.sh = sh; g.ch = ch;
    if (mode == 0) run_grid<0>(a, ch, linear, words);
    else run_grid<1>(a, ch, linear, words);
    fwrite(dbuf, 1, dbytes, fo);
    free(m1); free(m2); free(sbuf); free(dbuf);
  }
  fclose(fi);
  fclose(fo);
  printf("run: words=%lld bytes=%lld bad=%lld\n", g.words, g.bytes, g.bad);
  return g.bad ? 1 : 0;
}

static int mode_audit() {
  long long phase_hits[4] = {0, 0, 0, 0};   // word-path taps of the rightmost inside position, by 3 * sx % 4
  for (int sw = 2; sw <= 17; ++sw)
    for (int pad = 0; pad <= 4; pad += 4)
      for (int ipad = 0; ipad <= 4; ipad += 4) {
        const int sh = 3, n = 2;
        const long long spitch = ((3ll * sw + 3) & ~3ll) + pad, sistride = sh * spitch + ipad;
        // one output pixel per source position (sx, sy) in [-2, sw] x [-2, sh], every fraction pattern in turn
        std::vector<int2> pos;
        for (int sy = -2; sy <= sh; ++sy)
          for (int sx = -2; sx <= sw; ++sx) pos.push_back(make_int2(sx, sy));
        const int dw = (int)((pos.size() + 3) & ~(size_t)3), dh = 1;
        short2* m1 = static_cast<short2*>(alloc((size_t)dw * 4));
        unsigned short* m2 = static_cast<unsigned short*>(alloc((size_t)dw * 2));
        for (int i = 0; i < dw; ++i) {
          const int2 p = pos[(size_t)i % pos.size()];
          m1[i] = make_short2((short)p.x, (short)p.y);
          m2[i] = (unsigned short)((i * 37) & 1023);
          if (p.x == sw - 2 && p.y >= 0 && p.y + 1 < sh) ++phase_hits[(3 * p.x) & 3];
        }
        const size_t sbytes = (size_t)((n - 1) * sistride + (sh - 1) * spitch + 3ll * sw);
        uint8_t* sbuf = static_cast<uint8_t*>(alloc(sbytes));
        uint8_t* dbuf = static_cast<uint8_t*>(alloc((size_t)n * dw * 3));
        for (size_t i = 0; i < sbytes; ++i) sbuf[i] = (uint8_t)(i * 131 + 7);
        GatherArgs a{};
        a.src = sbuf; a.sw = sw; a.sh = sh; a.spitch = spitch; a.sistride = sistride; a.n = n;
        a.dst = dbuf; a.dw = dw; a.dh = dh; a.dpitch = 3ll * dw; a.distride = 3ll * dw;
        a.map1 = m1; a.map2 = m2;
        g.base = sbuf; g.sistride = sistride; g.spitch = spitch; g.n = n; g.sw = sw; g.sh = sh; g.ch = 3;
        run_grid<0>(a, 3, 1, 1);
        free(m1); free(m2); free(sbuf); free(dbuf);
      }
  printf("audit: words=%lld bytes=%lld bad=%lld edge_phases=%lld,%lld,%lld,%lld\n", g.words, g.bytes, g.bad, phase_hits[0],
         phase_hits[1], phase_hits[2], phase_hits[3]);
  return g.bad ? 1 : 0;
}

int main(int argc, char** argv) {
  if (argc == 4 && !strcmp(argv[1], "run")) return mode_run(argv[2], argv[3]);
  if (argc == 2 && !strcmp(argv[1], "audit")) return mode_audit();
  fprintf(stderr, "usage: undistort_stack run <in.bin> <out.bin> | undistort_stack audit\n");
  return 2;
}
