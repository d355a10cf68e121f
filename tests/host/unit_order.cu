// unit_order.cu -- k_bev_tma's unit hand-out on the host: the tile order of the plan compiler (tile_order) decoded the way
// the producer decodes a unit (tile u / groups, frame-set group u % groups) must cover every (tile, group) exactly once,
// and the units that survive the output-window skip of camera-sharded slabs must be exactly the window's tiles times the
// groups.
//
//   unit_order <tx> <ty> <batch> <tail percent> <seed> [ox oy ox1 oy1]
// prints "ok units=<n> kept=<k>" or the first violation (exit 1).
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "../../cameracalibration_b200/csrc/bevk_plan_tma.cuh"

using namespace bevk;

int main(int argc, char** argv) {
  if (argc != 6 && argc != 10) { fprintf(stderr, "usage\n"); return 2; }
  const int tx = atoi(argv[1]), ty = atoi(argv[2]), batch = atoi(argv[3]), tail = atoi(argv[4]);
  std::mt19937 rng(atoi(argv[5]));
  const int n_tiles = tx * ty;
  std::vector<long long> cost(n_tiles);
  for (auto& c : cost) c = 64 + (long long)(rng() % 4) * (rng() % 5000);   // ties and a spread, like real plans
  const std::vector<int> order = tile_order(tx, ty, cost, tail);
  // the tile list is a permutation of the tiles
  std::vector<int> seen_tile(n_tiles, 0);
  for (int t : order) {
    if (t < 0 || t >= n_tiles || seen_tile[t]++) { printf("tile %d repeated or out of range\n", t); return 1; }
  }
  if ((int)order.size() != n_tiles) { printf("tile list has %zu of %d tiles\n", order.size(), n_tiles); return 1; }
  // the kernel's frame-sets per unit: 4 for batches of at least 4, else 1 (bevk_api.cu render)
  const int NB = batch >= 4 ? 4 : 1, groups = (batch + NB - 1) / NB;
  const long long n_units = (long long)n_tiles * groups;
  std::vector<int> seen(n_units, 0);
  int ox = 0, oy = 0, ox1 = tx * TILE, oy1 = ty * TILE;
  if (argc == 10) { ox = atoi(argv[6]); oy = atoi(argv[7]); ox1 = atoi(argv[8]); oy1 = atoi(argv[9]); }
  long long kept = 0;
  for (long long u = 0; u < n_units; ++u) {
    const int pos = (int)(u / groups), g = (int)(u % groups);   // k_bev_tma's producer
    if (pos < 0 || pos >= n_tiles || g < 0 || g >= groups) { printf("unit %lld -> position %d group %d out of range\n", u, pos, g); return 1; }
    const long long id = (long long)order[pos] * groups + g;
    if (seen[id]++) { printf("unit %lld repeats tile %d group %d\n", u, order[pos], g); return 1; }
    // the producer's window skip (bevk_bev_tma.cuh): tiles outside [ox,ox1) x [oy,oy1) post nothing
    const int x0 = (order[pos] % tx) * TILE, y0 = (order[pos] / tx) * TILE;
    if (!(x0 >= ox1 || x0 + TILE <= ox || y0 >= oy1 || y0 + TILE <= oy)) ++kept;
  }
  long long want = 0;
  for (int t = 0; t < n_tiles; ++t) {
    const int x0 = (t % tx) * TILE, y0 = (t / tx) * TILE;
    if (!(x0 >= ox1 || x0 + TILE <= ox || y0 >= oy1 || y0 + TILE <= oy)) want += groups;
  }
  if (kept != want) { printf("window keeps %lld units, want %lld\n", kept, want); return 1; }
  printf("ok units=%lld kept=%lld\n", n_units, kept);
  return 0;
}
