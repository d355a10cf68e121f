// l2_model.cu -- a model of the DRAM traffic of one k_bev_tma step, for comparing unit orders on the CPU.
// Driven by tools/l2_model.py, which builds the LUT planes and masks of the bench geometry and writes <in.bin>.
//
//   l2_model <in.bin> <batch> <order mode> <order k> [l2 MB] [CTAs] [promotion bytes] [hints]
//   in.bin: int32 NC FW FH BW BH nearest, then per camera int16x2 map1 [BH][BW], uint16 map2 [BH][BW], uint8 mask [BH][BW]
//
// The plan is the product's (build_tma_plan, FS 7936, 4 entry groups per slot, max-mult 4), its tiles put in the
// candidate order (candidate_order); the units are decoded as the kernel decodes them, or group-major per window for the
// window candidates (unit_tile).  Model, and what it leaves out:
//   * 2 x 132 persistent CTAs take units off the counter in order; a unit lasts its tile's plan cost (the same estimate
//     the cost sort uses).  A CTA picks its next unit when it finishes the last one (greedy list schedule).
//   * a unit's ring slots (one per item and pass) are spread evenly over its duration; each slot touches the LUT bytes of
//     the item (re-read per pass) and the box rows of its frame-sets (clipped to the frame, widened to the tensor map's
//     L2 promotion granule); a GATHER slot touches the 32-B sectors of its entries' taps.  The tile's canvas rows are
//     written at the end of the unit.  All accesses of a slot happen at one instant; the accesses of all slots are
//     replayed in time order through one LRU of 32-B sectors.
//   * L2 is one cache of `l2 MB` (the H100's two partitions and their duplication are not modelled, nor set
//     associativity, nor the L1); writes allocate and are written back once each.
//   * hints (bit mask, as the kernel's cache policies): 1 LUT evict_last (evicted only when nothing else is left), 2 canvas
//     stores evict_first, 4 source boxes evict_first (inserted at the LRU end).
//   * two steps are replayed back to back (graph replays); the second is reported.
// Output: one JSON line.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <queue>
#include <vector>

#include "../cameracalibration_b200/csrc/bevk_plan_tma.cuh"

using namespace bevk;

namespace {

struct Lru {   // sectors 0..n-1; two lists: normal and evict_last; evict_first inserts at the normal list's LRU end
  std::vector<int> prev, next;
  std::vector<unsigned char> state;   // 0 absent, 1 normal, 2 last
  long long cap, size = 0;
  int head[3], tail[3];               // sentinel-free lists per state (index 1, 2)
  explicit Lru(long long n, long long cap_) : prev(n, -1), next(n, -1), state(n, 0), cap(cap_) {
    for (int i = 0; i < 3; ++i) head[i] = tail[i] = -1;
  }
  void unlink(int s) {
    const int l = state[s];
    if (prev[s] >= 0) next[prev[s]] = next[s]; else head[l] = next[s];
    if (next[s] >= 0) prev[next[s]] = prev[s]; else tail[l] = prev[s];
    prev[s] = next[s] = -1;
  }
  void push_front(int s, int l) {   // most recently used
    state[s] = (unsigned char)l;
    prev[s] = -1; next[s] = head[l];
    if (head[l] >= 0) prev[head[l]] = s; else tail[l] = s;
    head[l] = s;
  }
  void push_back(int s, int l) {    // next to be evicted
    state[s] = (unsigned char)l;
    next[s] = -1; prev[s] = tail[l];
    if (tail[l] >= 0) next[tail[l]] = s; else head[l] = s;
    tail[l] = s;
  }
  // hint: 0 normal, 1 evict_last, 2 evict_first.  Returns true on a hit.
  bool touch(int s, int hint) {
    const bool hit = state[s] != 0;
    if (hit) unlink(s); else ++size;
    if (hint == 1) push_front(s, 2);
    else if (hint == 2) push_back(s, 1);
    else push_front(s, 1);
    while (size > cap) {
      const int l = tail[1] >= 0 ? 1 : 2;
      const int v = tail[l];
      unlink(v);
      state[v] = 0;
      --size;
    }
    return hit;
  }
};

// Unit -> (position in the tile list, frame-set group).  window 1 is the kernel's decode (tile u / groups, group
// u % groups); window K models group-major windows of K tiles (only the last window may be shorter).
int unit_tile(long long unit, int groups, int window, int n_tiles, int& group) {
  const int u = (int)unit, per = window * groups, w = u / per, r = u - w * per, t0 = w * window;
  const int kw = std::min(window, n_tiles - t0);
  group = r / kw;
  return t0 + (r - group * kw);
}

// Candidate tile orders over tx x ty tiles (row-major indices, cost[i]); sets the window of the unit decode.
//   0  by decreasing cost (the order before the Hilbert curve)
//   1  the product's tile_order with the cheapest k % last (k = 0: the plain Hilbert curve)
//   2  the Hilbert curve cut into blocks of k tiles, blocks by decreasing cost, groups inner
//   3  the same blocks as windows of k tiles, group-major inside a window
std::vector<int> candidate_order(int tx, int ty, const std::vector<long long>& cost, int mode, int k, int& window) {
  const int n_tiles = tx * ty;
  window = 1;
  if (mode == 1) return tile_order(tx, ty, cost, k);
  std::vector<int> order(n_tiles);
  for (int i = 0; i < n_tiles; ++i) order[i] = i;
  if (mode == 0) {
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return cost[a] > cost[b]; });
    return order;
  }
  order = tile_order(tx, ty, cost, 0);
  k = std::max(1, k);
  const int n_blocks = (n_tiles + k - 1) / k;
  std::vector<long long> bcost(n_blocks, 0);
  for (int i = 0; i < n_tiles; ++i) bcost[i / k] += cost[order[i]];
  std::vector<int> blocks(n_blocks);
  for (int b = 0; b < n_blocks; ++b) blocks[b] = b;
  std::stable_sort(blocks.begin(), blocks.end(), [&](int a, int b) {   // a partial block stays last (window decode)
    const bool pa = (a + 1) * k > n_tiles, pb = (b + 1) * k > n_tiles;
    if (pa != pb) return pb;
    return bcost[a] > bcost[b];
  });
  std::vector<int> out;
  for (int b : blocks)
    for (int i = b * k; i < std::min(n_tiles, (b + 1) * k); ++i) out.push_back(order[i]);
  if (mode == 3) window = k;
  return out;
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 5) {
    fprintf(stderr, "usage: l2_model <in.bin> <batch> <order mode> <order k> [l2 MB] [CTAs] [promotion] [hints]\n");
    return 1;
  }
  const int batch = atoi(argv[2]), mode = atoi(argv[3]), order_k = atoi(argv[4]);
  const double l2_mb = argc > 5 ? atof(argv[5]) : 50.0;
  const int n_cta = argc > 6 ? atoi(argv[6]) : 264;
  const int promo = argc > 7 ? atoi(argv[7]) : 128;
  const int hints = argc > 8 ? atoi(argv[8]) : 0;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  int hdr[6];
  if (fread(hdr, 4, 6, f) != 6) return 3;
  const int NC = hdr[0], FW = hdr[1], FH = hdr[2], BW = hdr[3], BH = hdr[4];
  const bool nearest = hdr[5] != 0;
  const size_t npx = (size_t)BW * BH;
  std::vector<std::vector<short>> m1(NC, std::vector<short>(npx * 2));
  std::vector<std::vector<unsigned short>> m2(NC, std::vector<unsigned short>(npx));
  std::vector<std::vector<uint8_t>> mk(NC, std::vector<uint8_t>(npx));
  std::vector<const short*> p1(NC);
  std::vector<const unsigned short*> p2(NC);
  std::vector<const uint8_t*> pm(NC);
  for (int k = 0; k < NC; ++k) {
    if (fread(m1[k].data(), 4, npx, f) != npx || fread(m2[k].data(), 2, npx, f) != npx || fread(mk[k].data(), 1, npx, f) != npx) return 4;
    p1[k] = m1[k].data(); p2[k] = m2[k].data(); pm[k] = mk[k].data();
  }
  fclose(f);
  const int FS = 7936;
  TmaPlan plan;
  build_tma_plan(NC, FW, FH, BW, BH, nearest, p1.data(), p2.data(), pm.data(), FS, true, plan, 4, 4);
  int window = 1;
  {   // the plan's tiles back in row-major order, then in the candidate order
    const int tx = (BW + TILE - 1) / TILE, ty = (BH + TILE - 1) / TILE;
    std::vector<int4> rm(plan.tiles.size());
    std::vector<long long> cost(plan.tiles.size());
    for (size_t i = 0; i < plan.tiles.size(); ++i) {
      const int idx = plan.tiles[i].y / TILE * tx + plan.tiles[i].x / TILE;
      rm[idx] = plan.tiles[i]; cost[idx] = plan.tile_cost[i];
    }
    const std::vector<int> order = candidate_order(tx, ty, cost, mode, order_k, window);
    for (size_t i = 0; i < order.size(); ++i) { plan.tiles[i] = rm[order[i]]; plan.tile_cost[i] = cost[order[i]]; }
  }

  const int NB = batch >= 4 ? 4 : 1, groups = (batch + NB - 1) / NB;
  const int n_tiles = (int)plan.tiles.size();
  const long long n_units = (long long)n_tiles * groups;
  const long long pitch = (long long)FW * 3, frame_bytes = pitch * FH, canvas_bytes = (long long)BW * BH * 3;
  const long long lut_bytes = (long long)plan.lut.size() * 16;
  // dense sector spaces: frames | LUT | canvases
  const long long src_sec = (long long)batch * NC * frame_bytes / 32 + 1, lut_sec = lut_bytes / 32,
                  out_sec = ((long long)batch * canvas_bytes + 31) / 32;
  const long long n_sec = src_sec + lut_sec + out_sec;

  // ---- schedule: greedy list schedule of the units over the CTAs
  struct Slot { double t; int unit, item, pass; };   // item -1: the unit's write-out
  std::vector<Slot> slots;
  std::priority_queue<std::pair<double, int>, std::vector<std::pair<double, int>>, std::greater<>> ctas;
  for (int c = 0; c < n_cta; ++c) ctas.push({0.0, c});
  std::vector<double> finish(n_cta, 0.0);
  for (long long u = 0; u < n_units; ++u) {
    int g = 0;
    const int ti = unit_tile(u, groups, window, n_tiles, g);
    const int4 t = plan.tiles[ti];
    const int nb = std::min(NB, batch - g * NB);
    const double dur = (double)plan.tile_cost[ti] * nb / NB;
    auto [t0, c] = ctas.top();
    ctas.pop();
    std::vector<Slot> us;
    for (int it = t.z; it < t.z + t.w; ++it) {
      const TmaItem& I = plan.items[it];
      const int fpp = (I.flags & ITEM_GATHER) ? nb : std::min(NB, 4 * FS / I.fs_bytes);
      for (int p = 0; p < nb; p += fpp) us.push_back({0.0, (int)u, it, p});
    }
    for (size_t i = 0; i < us.size(); ++i) { us[i].t = t0 + dur * (double)i / (double)us.size(); slots.push_back(us[i]); }
    slots.push_back({t0 + dur, (int)u, -1, 0});
    finish[c] = t0 + dur;
    ctas.push({t0 + dur, c});
  }
  std::stable_sort(slots.begin(), slots.end(), [](const Slot& a, const Slot& b) { return a.t < b.t; });
  const double t_end = *std::max_element(finish.begin(), finish.end());
  double t_first = t_end;
  for (double v : finish) if (v > 0) t_first = std::min(t_first, v);

  // ---- replay
  Lru lru(n_sec, (long long)(l2_mb * 1e6 / 32));
  std::vector<unsigned char> seen(n_sec, 0);   // per step: bit 0 box sector, bit 1 sampled sector, bit 2 counted write
  long long rd_src = 0, rd_lut = 0, wr = 0, box_sum = 0, box_union = 0, sampled = 0, gather_sec = 0;
  auto src_range = [&](long long a, long long b, int gran, bool box, bool count) {   // frame-stack bytes [a, b)
    a = a / gran * gran; b = (b + gran - 1) / gran * gran;
    for (long long s = a / 32; s < b / 32; ++s) {
      if (!lru.touch((int)s, (hints & 4) ? 2 : 0) && count) rd_src += 32;
      if (count && box && !(seen[s] & 1)) { seen[s] |= 1; ++box_union; }
    }
  };
  for (int step = 0; step < 2; ++step) {
    const bool count = step == 1;
    std::fill(seen.begin(), seen.end(), 0);
    for (const Slot& sl : slots) {
      int g = 0;
      const int ti = unit_tile(sl.unit, groups, window, n_tiles, g);
      const int4 t = plan.tiles[ti];
      const int b0 = g * NB, nb = std::min(NB, batch - b0);
      if (sl.item < 0) {   // write-out of the tile's rows, every frame-set of the unit
        for (int j = 0; j < nb; ++j)
          for (int y = t.y; y < std::min(t.y + TILE, BH); ++y) {
            const long long a = (long long)(b0 + j) * canvas_bytes + ((long long)y * BW + t.x) * 3;
            const long long b = a + (long long)(std::min(t.x + TILE, BW) - t.x) * 3;
            for (long long s = a / 32; s <= (b - 1) / 32; ++s) {
              const long long q = src_sec + lut_sec + s;
              lru.touch((int)q, (hints & 2) ? 2 : 0);
              if (count && !(seen[q] & 4)) { seen[q] |= 4; wr += 32; }
            }
          }
        continue;
      }
      const TmaItem& I = plan.items[sl.item];
      const int nk = I.k1 - I.k0;
      // LUT entries of the item (every pass reads them again)
      const long long la = (long long)I.lut_block * TILE * TILE * 16 + (long long)I.k0 * 4096;
      for (long long s = la / 32; s < (la + (long long)nk * 4096) / 32; ++s)
        if (!lru.touch((int)(src_sec + s), (hints & 1) ? 1 : 0) && count) rd_lut += 32;
      if (I.flags & ITEM_GATHER) {
        for (int j = 0; j < nb; ++j) {
          const long long fb = (long long)((b0 + j) * NC + I.cam) * frame_bytes;
          for (int i = I.k0 * 256; i < I.k1 * 256; ++i) {
            const uint4 e = plan.lut[(size_t)I.lut_block * TILE * TILE + i];
            if (!(e.w & T_ACTIVE) || (e.w & T_SLOW)) continue;
            const long long off = e.x & ~3u, len = ((e.w >> 17) & 3u) == 3u ? 12 : 8;
            for (int r = 0; r < 2; ++r) {
              src_range(fb + off + r * pitch, fb + off + r * pitch + len, 32, false, count);
              if (count) gather_sec += 1;
            }
          }
        }
        continue;
      }
      const int fpp = std::min(NB, 4 * FS / I.fs_bytes), np = std::min(fpp, nb - sl.pass);
      const int2 shape = plan.shapes[I.shape];
      for (int j = 0; j < np; ++j) {
        const long long fb = (long long)((b0 + sl.pass + j) * NC + I.cam) * frame_bytes;
        if (count) box_sum += I.tx_bytes;
        const long long c0 = std::max<long long>(0, (long long)I.xw * 4), c1 = std::min<long long>(pitch, (long long)(I.xw + shape.x) * 4);
        if (c1 <= c0) continue;
        for (int r = std::max(0, I.y); r < std::min(FH, I.y + shape.y); ++r)
          src_range(fb + r * pitch + c0, fb + r * pitch + c1, promo, true, count);
      }
    }
  }
  // sampled sectors: the taps of every active entry inside the frame (bench.py algorithmic_bytes), per frame-set
  {
    std::vector<unsigned char> mark((size_t)(NC * frame_bytes / 32 + 1), 0);
    long long per_set = 0;
    for (const TmaItem& I : plan.items)
      for (int i = I.k0 * 256; i < I.k1 * 256; ++i) {
        const uint4 e = plan.lut[(size_t)I.lut_block * TILE * TILE + i];
        if (!(e.w & T_ACTIVE)) continue;
        long long sx, sy;
        if (I.flags & ITEM_GATHER) {
          if (e.w & T_SLOW) continue;
          sy = e.x / pitch; sx = (e.x % pitch) / 3;
        } else {
          const long long row = e.x / I.pitch, w0 = I.xw + (e.x % I.pitch) / 4, sh = (e.w >> 27) & 3u;
          sy = I.y + row; sx = (w0 * 4 + sh) / 3;
        }
        if (sx < 0 || sx + 1 >= FW || sy < 0 || sy + 1 >= FH) continue;
        for (int r = 0; r < 2; ++r) {
          const long long off = (long long)I.cam * frame_bytes + (sy + r) * pitch + sx * 3;
          for (long long s = off / 32; s <= (off + 5) / 32; ++s)
            if (!mark[s]) { mark[s] = 1; ++per_set; }
        }
      }
    sampled = per_set * 32 * batch;
  }
  printf("{\"order\": %d, \"k\": %d, \"window\": %d, \"batch\": %d, \"tiles\": %d, \"units\": %lld, \"l2_mb\": %.1f, \"ctas\": %d, "
         "\"promotion\": %d, \"hints\": %d, \"box_bytes\": %lld, \"box_union_bytes\": %lld, \"sampled_bytes\": %lld, "
         "\"dram_read_src\": %lld, \"dram_read_lut\": %lld, \"dram_write\": %lld, \"lut_bytes\": %lld, \"finish_spread\": %.4f}\n",
         mode, order_k, window, batch, n_tiles, n_units, l2_mb, n_cta, promo, hints, box_sum, box_union * 32, sampled, rd_src,
         rd_lut, wr, lut_bytes, (t_end - t_first) / t_end);
  return 0;
}
