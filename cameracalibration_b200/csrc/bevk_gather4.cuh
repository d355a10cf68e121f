// bevk_gather4.cuh -- 4-pixels-per-thread form of the stand-alone gathers for 3-channel INTER_LINEAR:
// cv2.remap with resident maps (MODE 0; Camera.undistort / InCalibrator.undistort / Tools/undistort.py,
// surroundBEV.py:110-111, intrinsicCalib.py:193-195, undistort.py:66), the same with the camera model
// evaluated in-kernel (MODE 1), cv2.warpPerspective (MODE 2; extrinsicCalib.py:166-169) and cv2.warpAffine
// (MODE 3; extrinsicCalib.py:58), and cv2.remap / undistortion with float maps (MODE 4 and 5).
// Same tap machinery as the fused BEV kernel (aligned 32-bit words, funnel shift, PRMT, DP2A);
// each thread produces 12 output bytes per frame and stores them as three 32-bit words.  Over a
// batch it resolves its 4 pixels' taps once and gathers them from NB = GATHER_NB frames (see k_gather).
// The generic k_gather stays for 1/4-channel images, INTER_NEAREST, sizes that are not multiples
// of 4 and caller memory that is not 4-byte aligned.
#pragma once
#include "bevk_bev.cuh"
#include "bevk_kernels.cuh"

namespace bevk {

// Tap loads of gather_px: read-only global loads.  tests/host/undistort_stack.cu substitutes a loader that records
// every address it is asked for.
struct Ldg {
  __host__ __device__ __forceinline__ static unsigned w32(const uint8_t* p) { return ldg32(p); }
  __host__ __device__ __forceinline__ static int b8(const uint8_t* p) { return ldg8(p); }
};

// one output pixel: fixed-point source position -> packed B | G<<8 | R<<16.  BD (k_gather4_border): a window not wholly
// inside takes its taps through border_window instead (bd: any mode but BORDER_TRANSPARENT, which gather4_ok sends to
// k_gather_border); a window the border value fills is the Q10 sum of four border taps, which is the value itself.
// The word loads read nothing outside the taps' own rows, rounded out to whole 32-bit words, so frames need no
// slack after them: `inside` means both taps of each row, bytes [off, off + 6) with off = 3 * sx, lie in the row.
// The loaded words start at off_al = off & ~3 and off_al + 4, and at off_al + 8 only when off % 4 == 3.  Each of
// them holds a byte of [off, off + 6): off itself; off_al + 4, which is in [off + 1, off + 4]; off_al + 8 = off + 5.
// With the row's first byte on a 4-byte boundary (src, spitch 4-aligned; checked by the host), every word loaded
// is therefore one of the row's own words.
template <class LD = Ldg, bool BD = false>
__host__ __device__ __forceinline__ unsigned gather_px(const uint8_t* __restrict__ src, unsigned spitch, int sw, int sh, int sx, int sy,
                                              unsigned fx, unsigned fy, const Border& bd = Border{}) {
  const bool inside = sx >= 0 && sy >= 0 && sx + 1 < sw && sy + 1 < sh;
  if constexpr (BD) {
    if (!inside) {
      int xs[2], ys[2], p[4][3];
      const bool fill = border_window<2>(bd, sx, sy, sw, sh, xs, ys) != BW_TAPS;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int tx = xs[t & 1], ty = ys[t >> 1];
        if (!fill && (tx | ty) >= 0) {
          const uint8_t* q = src + (size_t)ty * spitch + 3 * tx;
          p[t][0] = LD::b8(q); p[t][1] = LD::b8(q + 1); p[t][2] = LD::b8(q + 2);
        } else { p[t][0] = bd.v[0]; p[t][1] = bd.v[1]; p[t][2] = bd.v[2]; }
      }
      const unsigned ob = (unsigned)bilerp_q10(p[0][0], p[1][0], p[2][0], p[3][0], (int)fx, (int)fy);
      const unsigned og = (unsigned)bilerp_q10(p[0][1], p[1][1], p[2][1], p[3][1], (int)fx, (int)fy);
      const unsigned orr = (unsigned)bilerp_q10(p[0][2], p[1][2], p[2][2], p[3][2], (int)fx, (int)fy);
      return ob | (og << 8) | (orr << 16);
    }
  }
  if (inside) {
    const unsigned off = (unsigned)sy * spitch + 3u * (unsigned)sx;
    const unsigned off_al = off & ~3u, sh8 = (off & 3u) * 8u;
    const bool third = (sh8 == 24u);
    const uint8_t* q0 = src + off_al;
    const uint8_t* q1 = q0 + spitch;
    const unsigned a0 = LD::w32(q0), a1 = LD::w32(q0 + 4), a2 = third ? LD::w32(q0 + 8) : 0u;
    const unsigned b0 = LD::w32(q1), b1 = LD::w32(q1 + 4), b2 = third ? LD::w32(q1 + 8) : 0u;
    const unsigned w11 = fx * fy, w01 = (fx << 5) - w11, w10 = (fy << 5) - w11, w00 = 1024u - (fx << 5) - (fy << 5) + w11;
    return interp_fast(sh8, w00 | (w01 << 16), w10 | (w11 << 16), 65536u, a0, a1, a2, b0, b1, b2);
  }
  int p[4][3];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int tx = sx + (t & 1), ty = sy + (t >> 1);
    if ((unsigned)tx < (unsigned)sw && (unsigned)ty < (unsigned)sh) {
      const uint8_t* q = src + (size_t)ty * spitch + 3 * tx;
      p[t][0] = LD::b8(q); p[t][1] = LD::b8(q + 1); p[t][2] = LD::b8(q + 2);
    } else { p[t][0] = p[t][1] = p[t][2] = 0; }
  }
  const unsigned ob = (unsigned)bilerp_q10(p[0][0], p[1][0], p[2][0], p[3][0], (int)fx, (int)fy);
  const unsigned og = (unsigned)bilerp_q10(p[0][1], p[1][1], p[2][1], p[3][1], (int)fx, (int)fy);
  const unsigned orr = (unsigned)bilerp_q10(p[0][2], p[1][2], p[2][2], p[3][2], (int)fx, (int)fy);
  return ob | (og << 8) | (orr << 16);
}

// One thread of k_gather4: output pixels x4 .. x4 + 3 of row y, frames [f0, min(n, f0 + NB)).  Host-capable
// (tests/host/undistort_stack.cu).  Requirements checked by the host (gather4_ok in bevk_api.cu): channels == 3,
// INTER_LINEAR, dw % 4 == 0; src, dst, both row pitches and (n > 1) both image strides multiples of 4; spitch * sh < 2^31
// (gather_px's 32-bit offsets within a frame).
template <int MODE, int NB, class LD = Ldg, int LENS = 0, bool BD = false>
__host__ __device__ __forceinline__ void gather4_frames(const GatherArgs& a, int x4, int y, int f0) {
  short mx[4], my[4];
  unsigned short fr[4];
  if (MODE == 0) {
    const size_t i = (size_t)y * a.dw + x4;
    const int4 m = *reinterpret_cast<const int4*>(a.map1 + i);        // 4 x (short x, short y)
    const uint2 f = *reinterpret_cast<const uint2*>(a.map2 + i);      // 4 x uint16
    mx[0] = (short)(m.x & 0xffff); my[0] = (short)(m.x >> 16);
    mx[1] = (short)(m.y & 0xffff); my[1] = (short)(m.y >> 16);
    mx[2] = (short)(m.z & 0xffff); my[2] = (short)(m.z >> 16);
    mx[3] = (short)(m.w & 0xffff); my[3] = (short)(m.w >> 16);
    fr[0] = (unsigned short)(f.x & 0xffffu); fr[1] = (unsigned short)(f.x >> 16);
    fr[2] = (unsigned short)(f.y & 0xffffu); fr[3] = (unsigned short)(f.y >> 16);
  } else if (MODE == 4) {   // 16-byte map loads: the host checks the maps' alignment (gather4_ok)
    const size_t i = (size_t)y * a.dw + x4;
    float X[4], Y[4];
    if (a.fmap2) {
      const float4 p = *reinterpret_cast<const float4*>(a.fmap1 + i), q = *reinterpret_cast<const float4*>(a.fmap2 + i);
      X[0] = p.x; X[1] = p.y; X[2] = p.z; X[3] = p.w;
      Y[0] = q.x; Y[1] = q.y; Y[2] = q.z; Y[3] = q.w;
    } else {
      const float4 p = *reinterpret_cast<const float4*>(a.fmap1 + 2 * i), q = *reinterpret_cast<const float4*>(a.fmap1 + 2 * i + 4);
      X[0] = p.x; Y[0] = p.y; X[1] = p.z; Y[1] = p.w;
      X[2] = q.x; Y[2] = q.y; X[3] = q.z; Y[3] = q.w;
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) quantise_xy(X[q], Y[q], false, mx[q], my[q], fr[q]);
  }
  int sx[4], sy[4], fx[4], fy[4];
  unsigned px[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (MODE == 0 || MODE == 4) split_entry(mx[q], my[q], fr[q], false, sx[q], sy[q], fx[q], fy[q]);
    else source_pos<MODE, LENS>(a, x4 + q, y, false, sx[q], sy[q], fx[q], fy[q]);
    // one frame (launched only for n = 1, so f0 = 0): gather each pixel as soon as its taps are known, as the
    // single-frame kernel always did -- about half the registers of the batch form, twice the occupancy
    if (NB == 1) px[q] = gather_px<LD, BD>(a.src, (unsigned)a.spitch, a.sw, a.sh, sx[q], sy[q], fx[q], fy[q], a.bd);
  }
  const int nf = a.n - f0 < NB ? a.n - f0 : NB;
  const uint8_t* s = a.src + (long long)f0 * a.sistride;
  uint8_t* d = a.dst + (long long)f0 * a.distride + (long long)y * a.dpitch + (long long)x4 * 3;
  for (int f = 0; f < nf; ++f, s += a.sistride, d += a.distride) {
    if (NB != 1) {
#pragma unroll
      for (int q = 0; q < 4; ++q) px[q] = gather_px<LD, BD>(s, (unsigned)a.spitch, a.sw, a.sh, sx[q], sy[q], fx[q], fy[q], a.bd);
    }
    unsigned* o = reinterpret_cast<unsigned*>(NB == 1 ? a.dst + (long long)y * a.dpitch + (long long)x4 * 3 : d);
    o[0] = lane_perm(px[0], px[1], 0x4210);   // B0 G0 R0 B1
    o[1] = lane_perm(px[1], px[2], 0x5421);   // G1 R1 B2 G2
    o[2] = lane_perm(px[2], px[3], 0x6542);   // R2 B3 G3 R3
    if (NB == 1) break;
  }
}

// NB = frames per thread: GATHER_NB over a batch, 1 for a single frame (n = 1 then compiles to the single-frame body
// and keeps its register count and occupancy; the batch form needs about twice the registers).
template <int MODE, int NB, int LENS>
__global__ void __launch_bounds__(256) k_gather4(GatherArgs a) {
  const int x4 = (blockIdx.x * 32 + (threadIdx.x & 31)) * 4;
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x4 >= a.dw || y >= a.dh) return;
  gather4_frames<MODE, NB, Ldg, LENS>(a, x4, y, blockIdx.z * NB);
}

// k_gather4 under cv2's other border modes and values but BORDER_TRANSPARENT (gather_px's BD form)
template <int MODE, int NB, int LENS>
__global__ void __launch_bounds__(256) k_gather4_border(GatherArgs a) {
  const int x4 = (blockIdx.x * 32 + (threadIdx.x & 31)) * 4;
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x4 >= a.dw || y >= a.dh) return;
  gather4_frames<MODE, NB, Ldg, LENS, true>(a, x4, y, blockIdx.z * NB);
}

}  // namespace bevk
