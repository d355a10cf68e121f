// bevk_shard.cuh -- camera-per-GPU sharding of the BEV path: slab geometry and the compose kernel.
//
// The reference composes the four masked camera images with a cv2.add chain (SurroundBirdEyeView/surroundBEV.py:316-320).
// A saturating sum of non-negative bytes does not depend on the order (min(min(a+b,255)+c,255) == min(a+b+c,255)), so
// the chain can be cut anywhere: rank r renders only its cameras -- into a SLAB, the tile-aligned bounding box of the
// union of their masks, 0.9-1.2 MB instead of the 3 MB canvas at 1000x1000 -- one all-gather moves the slabs over
// NVLink, and every rank composes them.  k_compose_slabs is that compose (+ the car overlay, :323-324).
#pragma once
#include "bevk_bev.cuh"

namespace bevk {

constexpr int SHARD_MAX_RANKS = 8;

struct SlabRect { int ox, oy, ox1, oy1; };   // canvas pixels [ox,ox1) x [oy,oy1); empty when ox1 <= ox

// ranks' cameras: contiguous blocks, the first n_cam % world ranks get one more (cameracalibration_b200/sharding.py:block_range)
inline void shard_block(int n, int rank, int world, int* lo, int* hi) {
  const int base = n / world, extra = n % world;
  *lo = rank * base + (rank < extra ? rank : extra);
  *hi = *lo + base + (rank < extra ? 1 : 0);
}

// tile-aligned bounding box of the union of the masks of cameras [lo,hi), clipped to the canvas
inline SlabRect slab_rect(const uint8_t* const* masks, int lo, int hi, int BW, int BH) {
  int x0 = BW, y0 = BH, x1 = 0, y1 = 0;
  for (int k = lo; k < hi; ++k)
    for (int y = 0; y < BH; ++y) {
      const uint8_t* row = masks[k] + (size_t)y * BW;
      int a = 0, b = BW - 1;
      while (a < BW && !row[a]) ++a;
      if (a == BW) continue;
      while (!row[b]) --b;
      if (a < x0) x0 = a;
      if (b + 1 > x1) x1 = b + 1;
      if (y < y0) y0 = y;
      y1 = y + 1;
    }
  SlabRect r{0, 0, 0, 0};
  if (x1 <= x0 || y1 <= y0) return r;
  r.ox = x0 / TILE * TILE; r.oy = y0 / TILE * TILE;
  r.ox1 = (x1 + TILE - 1) / TILE * TILE; r.oy1 = (y1 + TILE - 1) / TILE * TILE;
  if (r.ox1 > BW) r.ox1 = BW;
  if (r.oy1 > BH) r.oy1 = BH;
  return r;
}

struct ComposeArgs {
  const uint8_t* slabs;            // rank r, frame-set b at slabs + r * rank_stride + b * slab_bytes
  long long slab_bytes, rank_stride;
  int world, batch, BW, BH;
  SlabRect rect[SHARD_MAX_RANKS];
  const uint8_t* car;              // dense canvas or null
  uint8_t* out;                    // [batch][BH][BW][3]
  unsigned long long* csum;        // BAL: channel sums [batch][3] of the composed canvases (zeroed by the caller)
};

// grid (chunks of 256 units per canvas row, groups of COMPOSE_ROWS canvas rows, frame-sets): no index arithmetic beyond
// adds.  UNIT bytes per thread and row: 8 when canvas rows are whole 8-byte words (BW % 8 == 0; every slab edge then falls
// on an 8-byte boundary: tile-aligned x is a multiple of 96 bytes, the canvas edge a multiple of 8), else 1.
constexpr int COMPOSE_ROWS = 4;

// One thread's work: bytes [xb, xb + UNIT) of canvas rows y0 .. y0 + COMPOSE_ROWS - 1 of frame-set b.  Without BAL the
// car is added.  With BAL the raw canvas is written (colour balance and then the car follow in k_gain) and each byte
// written is added to sums[channel], the channel being its offset in the canvas row mod 3 (a row starts on a pixel).
// Host-capable: tests/host/shard_compose.cu drives it over the device's grid.
template <int UNIT, bool BAL>
__host__ __device__ __forceinline__ void compose_column(const ComposeArgs& a, int b, int y0, int xb, unsigned* sums) {
  const int row_bytes = a.BW * 3;
  uint8_t* out = a.out + (size_t)b * row_bytes * a.BH;
  unsigned rel[3] = {0, 0, 0};     // BAL: sums of the bytes at xb + k, k % 3 == 0, 1, 2
#pragma unroll
  for (int dy = 0; dy < COMPOSE_ROWS; ++dy) {
    const int y = y0 + dy;
    if (y >= a.BH) break;
    const size_t off = (size_t)y * row_bytes + xb;
    unsigned lo = 0, hi = 0;
#pragma unroll
    for (int r = 0; r < SHARD_MAX_RANKS; ++r) {
      if (r >= a.world) break;
      const SlabRect q = a.rect[r];
      if (y < q.oy || y >= q.oy1 || xb < q.ox * 3 || xb >= q.ox1 * 3) continue;
      const uint8_t* p = a.slabs + (size_t)r * a.rank_stride + (size_t)b * a.slab_bytes + (size_t)(y - q.oy) * ((q.ox1 - q.ox) * 3) + (xb - q.ox * 3);
      // plain loads (not the read-only path): in peer-store mode other GPUs wrote this memory
      if (UNIT == 8) { const uint2 v = *reinterpret_cast<const uint2*>(p); lo = lane_addus4(lo, v.x); hi = lane_addus4(hi, v.y); }
      else lo = min(255u, lo + *p);
    }
    if (!BAL && a.car) {
#ifdef __CUDA_ARCH__
      if (UNIT == 8) { const uint2 v = __ldg(reinterpret_cast<const uint2*>(a.car + off)); lo = __vaddus4(lo, v.x); hi = __vaddus4(hi, v.y); }
      else lo = min(255u, lo + __ldg(a.car + off));
#else
      if (UNIT == 8) { const uint2 v = *reinterpret_cast<const uint2*>(a.car + off); lo = lane_addus4(lo, v.x); hi = lane_addus4(hi, v.y); }
      else lo = min(255u, lo + a.car[off]);
#endif
    }
    if (UNIT == 8) *reinterpret_cast<uint2*>(out + off) = make_uint2(lo, hi);
    else out[off] = (uint8_t)lo;
    if (BAL) {
      if (UNIT == 8) {   // bytes k = 0..3 of lo, 4..7 of hi
        rel[0] += (lo & 255u) + (lo >> 24) + ((hi >> 16) & 255u);
        rel[1] += ((lo >> 8) & 255u) + (hi & 255u) + (hi >> 24);
        rel[2] += ((lo >> 16) & 255u) + ((hi >> 8) & 255u);
      } else {
        rel[0] += lo;
      }
    }
  }
  if (BAL) {
    const int ph = xb % 3;
    sums[ph] += rel[0];
    sums[ph == 2 ? 0 : ph + 1] += rel[1];
    sums[ph == 0 ? 2 : ph - 1] += rel[2];
  }
}

#ifdef __CUDACC__
// BAL: 32-bit partials per thread (at most COMPOSE_ROWS * 3 * 255 per channel), warp shuffles, then one u64 atomic per
// channel and CTA (a CTA's sum stays below 256 * COMPOSE_ROWS * 8 * 255 < 2^32).
template <int UNIT, bool BAL = false>
__global__ void __launch_bounds__(256) k_compose_slabs(ComposeArgs a) {
  const int b = blockIdx.z;
  const int xb = (blockIdx.x * 256 + threadIdx.x) * UNIT;
  if (!BAL) {
    if (xb >= a.BW * 3) return;
    compose_column<UNIT, false>(a, b, blockIdx.y * COMPOSE_ROWS, xb, nullptr);
    return;
  }
  unsigned s[3] = {0, 0, 0};
  if (xb < a.BW * 3) compose_column<UNIT, true>(a, b, blockIdx.y * COMPOSE_ROWS, xb, s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s[0] += __shfl_xor_sync(0xffffffffu, s[0], o);
    s[1] += __shfl_xor_sync(0xffffffffu, s[1], o);
    s[2] += __shfl_xor_sync(0xffffffffu, s[2], o);
  }
  __shared__ unsigned part[8][3];
  if ((threadIdx.x & 31) == 0) { part[threadIdx.x >> 5][0] = s[0]; part[threadIdx.x >> 5][1] = s[1]; part[threadIdx.x >> 5][2] = s[2]; }
  __syncthreads();
  if (threadIdx.x < 3) {
    unsigned t = 0;
    for (int w = 0; w < 8; ++w) t += part[w][threadIdx.x];
    if (t) atomicAdd(a.csum + 3 * b + threadIdx.x, (unsigned long long)t);
  }
}
#endif

}  // namespace bevk
