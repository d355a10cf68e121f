// Host form of the camera-sharded compose and of the gathered luminance offsets: compose_column (the per-thread body of
// k_compose_slabs<UNIT, BAL>, bevk_shard.cuh) driven over the device's grid, with BAL's channel sums reduced per CTA in
// 32 bits and added to u64 sums as the kernel does; and gathered_deltas (k_delta's body, bevk_kernels.cuh) over world
// blocks of V sums.  tests/test_host_shard_compose.py compares both with NumPy.
//
//   shard_compose compose <in.bin> <out.bin>
//     in : records of int32 unit (8 or 1), bal, world, batch, BW, BH, has_car, out_off; int64 slab_bytes, rank_stride;
//          int32 rect[world][4] (x0, y0, x1, y1); the slabs (world * rank_stride bytes); the car (BW*BH*3) when has_car
//     out: per record the canvases (batch*BH*BW*3 bytes), then uint64 csum[batch][3] when bal
//   shard_compose delta <in.bin> <out.bin>
//     in : records of int32 world, batch, n_cam; float64 npix; uint64 blocks[world][batch][n_cam]
//     out: per record int32 delta[batch][n_cam] (gathered_deltas), then int32 delta[batch][n_cam] of lum_deltas on the
//          column sums merged here
// Built by tests/test_host_shard_compose.py with nvcc; only host code runs.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_kernels.cuh"
#include "../../cameracalibration_b200/csrc/bevk_shard.cuh"

using namespace bevk;

static bool rd(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n; }

template <int UNIT, bool BAL>
static void compose_grid(const ComposeArgs& a, unsigned long long* csum) {
  const int units = UNIT == 8 ? a.BW * 3 / 8 : a.BW * 3;
  const int gx = (units + 255) / 256, gy = (a.BH + COMPOSE_ROWS - 1) / COMPOSE_ROWS;
  for (int b = 0; b < a.batch; ++b)
    for (int by = 0; by < gy; ++by)
      for (int bx = 0; bx < gx; ++bx) {
        unsigned cta[3] = {0, 0, 0};   // the kernel's 32-bit CTA total
        for (int t = 0; t < 256; ++t) {
          const int xb = (bx * 256 + t) * UNIT;
          if (xb >= a.BW * 3) continue;
          unsigned s[3] = {0, 0, 0};
          compose_column<UNIT, BAL>(a, b, by * COMPOSE_ROWS, xb, s);
          for (int k = 0; k < 3; ++k) cta[k] += s[k];
        }
        if (BAL)
          for (int k = 0; k < 3; ++k) csum[3 * b + k] += cta[k];
      }
}

static int mode_compose(FILE* in, FILE* out) {
  int32_t h[8];
  int n = 0;
  while (rd(in, h, sizeof h)) {
    const int unit = h[0], bal = h[1], world = h[2], batch = h[3], BW = h[4], BH = h[5], has_car = h[6], off = h[7];
    int64_t sb[2];
    if (!rd(in, sb, sizeof sb) || world < 1 || world > SHARD_MAX_RANKS) return 2;
    ComposeArgs a{};
    a.world = world; a.batch = batch; a.BW = BW; a.BH = BH; a.slab_bytes = sb[0]; a.rank_stride = sb[1];
    for (int r = 0; r < world; ++r) {
      int32_t q[4];
      if (!rd(in, q, sizeof q)) return 2;
      a.rect[r] = SlabRect{q[0], q[1], q[2], q[3]};
    }
    std::vector<uint8_t> slabs((size_t)world * sb[1] + 8), car(has_car ? (size_t)BW * BH * 3 : 0);
    if (!rd(in, slabs.data(), (size_t)world * sb[1])) return 2;
    if (has_car && !rd(in, car.data(), car.size())) return 2;
    const size_t canvas = (size_t)batch * BH * BW * 3;
    std::vector<uint64_t> obuf((canvas + off + 16) / 8 + 1, 0x5a5a5a5a5a5a5a5aull);   // 8-byte aligned base
    uint8_t* o = reinterpret_cast<uint8_t*>(obuf.data()) + off;
    a.slabs = slabs.data(); a.car = has_car ? car.data() : nullptr; a.out = o;
    std::vector<unsigned long long> csum((size_t)batch * 3, 0ull);
    a.csum = csum.data();
    if (unit == 8 && bal) compose_grid<8, true>(a, csum.data());
    else if (unit == 8) compose_grid<8, false>(a, csum.data());
    else if (bal) compose_grid<1, true>(a, csum.data());
    else compose_grid<1, false>(a, csum.data());
    fwrite(o, 1, canvas, out);
    if (bal) fwrite(csum.data(), 8, csum.size(), out);
    ++n;
  }
  printf("compose records=%d\n", n);
  return 0;
}

static int mode_delta(FILE* in, FILE* out) {
  int32_t h[3];
  int n = 0;
  while (rd(in, h, sizeof h)) {
    const int world = h[0], batch = h[1], n_cam = h[2];
    double npix;
    if (!rd(in, &npix, 8) || n_cam < 1 || n_cam > BEVK_MAX_CAMERAS_K) return 2;
    std::vector<unsigned long long> blocks((size_t)world * batch * n_cam);
    if (!rd(in, blocks.data(), blocks.size() * 8)) return 2;
    std::vector<int32_t> got((size_t)batch * n_cam), merged_d((size_t)batch * n_cam);
    for (int b = 0; b < batch; ++b) {   // k_delta's thread b
      gathered_deltas(blocks.data() + (size_t)b * n_cam, (long long)batch * n_cam, world, n_cam, npix, got.data() + (size_t)b * n_cam);
      unsigned long long merged[BEVK_MAX_CAMERAS_K] = {};
      for (int w = 0; w < world; ++w)
        for (int c = 0; c < n_cam; ++c) merged[c] += blocks[((size_t)w * batch + b) * n_cam + c];
      lum_deltas(merged, n_cam, npix, merged_d.data() + (size_t)b * n_cam);
    }
    fwrite(got.data(), 4, got.size(), out);
    fwrite(merged_d.data(), 4, merged_d.size(), out);
    ++n;
  }
  printf("delta records=%d\n", n);
  return 0;
}

int main(int argc, char** argv) {
  if (argc != 4) { fprintf(stderr, "usage: shard_compose compose|delta <in.bin> <out.bin>\n"); return 2; }
  FILE* in = fopen(argv[2], "rb");
  FILE* out = fopen(argv[3], "wb");
  if (!in || !out) return 2;
  const int r = !strcmp(argv[1], "compose") ? mode_compose(in, out) : !strcmp(argv[1], "delta") ? mode_delta(in, out) : 2;
  fclose(in);
  fclose(out);
  return r;
}
