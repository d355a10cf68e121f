// bevk_api.cu -- C ABI of libbevk.so (see include/bevk.h) over the sm_90a kernels.
// Host side: argument checks, 3x3 inverses the way OpenCV computes them, device
// buffer management, the tile-plan compiler, stream ordering.  No CPU fallback.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "../../include/bevk.h"
#include "bevk_kernels.cuh"
#include "bevk_bev.cuh"
#include "bevk_gather4.cuh"
#include "bevk_plan.cuh"
#include "bevk_bev_tma.cuh"
#include "bevk_plan_tma.cuh"
#include "bevk_shard.cuh"
#include "bevk_jpeg_enc.cuh"
#include "bevk_jpeg_prog.cuh"
#include "bevk_png_enc.cuh"
#include "bevk_resize.cuh"
#include "bevk_points.cuh"

#include <cub/device/device_scan.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include <dlfcn.h>
#include <nvtx3/nvToolsExt.h>   // header-only: ranges cost nothing unless a profiler injects itself

using namespace bevk;

// k_bev_tma configurations built into the library: FS = bytes of one frame-set's staged source box (a ring slot holds 4 FS
// of boxes), STAGES = ring slots, MINCTAS = resident CTAs per SM the register budget is set for, EG = LUT-entry groups per
// slot (the plan's items never span more).  The first entry is the default; BEVK_TMA_CFG="<FS>,<STAGES>,<EG>" (read at
// bevk_bev_finalize) selects another one for tuning runs.  Measured on H100 (bench.py default workload, 400 W power limit):
// with two CTAs per SM the largest slots that fit win (0.206 ms per step at FS 4096 -> 0.199 ms at FS 7936); a third,
// smaller stage does not pay.  7936: 2 x (2 x 48256 + 16896 + 1056) + static/reserved = 233024 of the SM's 233472 bytes.
#define BEVK_TMA_CONFIGS(X) X(7936, 2, 2, 4) X(7680, 2, 2, 4) X(6144, 2, 2, 4) X(5120, 2, 2, 4) X(4096, 2, 2, 4) X(4096, 3, 2, 2) X(4096, 2, 3, 2)
struct TmaConfig { int fs, stages, min_ctas, eg; };
#define X(FS, ST, MC, EG) {FS, ST, MC, EG},
static const TmaConfig kTmaConfigs[] = {BEVK_TMA_CONFIGS(X)};
#undef X
static const int kNumTmaConfigs = (int)(sizeof kTmaConfigs / sizeof kTmaConfigs[0]);
constexpr int kMaxTmaConfigs = 8;   // bevk_ctx::tma_grid
static_assert(sizeof kTmaConfigs / sizeof kTmaConfigs[0] <= kMaxTmaConfigs, "grow bevk_ctx::tma_grid");


// ------------------------------------------------------------------ errors
static thread_local std::string g_err;
static int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
#define CU(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
      return fail(e_ == cudaErrorMemoryAllocation ? BEVK_ERR_OOM : BEVK_ERR_CUDA, "%s: %s (%s:%d)", #call, \
                  cudaGetErrorString(e_), __FILE__, __LINE__);                                     \
  } while (0)
#define RET(call)             \
  do {                        \
    int r_ = (call);          \
    if (r_ != BEVK_OK) return r_; \
  } while (0)

// NVTX range for the lifetime of a scope (visible in nsys / ncu timelines: ingest, render, read-back)
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

// ------------------------------------------------------------------ small helpers
// bytes rounded up to a multiple of 256: frames in a stack start 256-byte aligned
static size_t pad256(size_t bytes) { return (bytes + 255) & ~size_t(255); }

// Device memory owned by the ctx: grown by ensure(), freed with its owner.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  int ensure(size_t n) {
    if (n <= cap) return BEVK_OK;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    n = pad256(n);
    CU(cudaMalloc(&p, n + 256));   // 256 B of slack: the kernels' 32-bit tap loads may touch 3 bytes past a frame
    cap = n;
    return BEVK_OK;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

// A camera of either model (K, D, R, P) as the kernels take it (lens_model): CamModel, LensExt and whether it needs the
// LENS = 1 instances.  D lengths cv2 refuses are refused.
struct Lens {
  CamModel cm;
  LensExt lx;
  bool full = false;
  bool walks = false;   // R makes the rays depend on the row (rays_walk): they are walked first (k_walk_rays)
};

static int make_model(int model, const double* K, const double* D, int n_dist, const double* R, const double* P, int w, int h,
                      Lens* L) {
  if (!K || !P || (n_dist > 0 && !D)) return fail(BEVK_ERR_ARG, "null K/D/P");
  if (model != BEVK_MODEL_FISHEYE && model != BEVK_MODEL_PINHOLE) return fail(BEVK_ERR_ARG, "bad camera model %d", model);
  if (w <= 0 || h <= 0) return fail(BEVK_ERR_ARG, "bad map size %dx%d", w, h);
  switch (lens_model(model, K, D, n_dist, R, P, w, h, &L->cm, &L->lx, &L->full)) {
    case LENS_BAD_COUNT:
      return fail(BEVK_ERR_ARG, model == BEVK_MODEL_FISHEYE ? "fisheye D has %d coefficients, cv2 takes 4 (or 0)"
                                                           : "pinhole D has %d coefficients, cv2 takes 0, 4, 5, 8, 12 or 14", n_dist);
    case LENS_SINGULAR: return fail(BEVK_ERR_ARG, R ? "P * R is singular" : "P is singular");
  }
  L->walks = rays_walk(L->cm, R);
  L->full = L->full || L->walks;
  return BEVK_OK;
}

// The D of the entry points that take no R (bevk_undistort_map, bevk_undistorter_set, bevk_bev_set_camera), as they have
// always read it: a pinhole D of 8, 12 or 14 coefficients in full, the first 5 (zero-padded) of any other count; a
// fisheye D's first 4.
struct LegacyDist {
  double d[14] = {};
  const double* D;
  int n;
  LegacyDist(int model, const double* src, int n_dist) : D(src), n(n_dist) {
    if (dist_count_ok(model, n_dist) || (n_dist > 0 && !src)) return;   // a count cv2 takes, or a null D: as given
    n = model == BEVK_MODEL_FISHEYE ? 4 : 5;
    if (n_dist > 0) memcpy(d, src, sizeof(double) * std::min(n, n_dist));
    D = d;
  }
};

static int make_homog(const double* H, Homog* hm) {
  if (!H) return fail(BEVK_ERR_ARG, "null H");
  if (!inv3(H, hm->M)) memset(hm->M, 0, sizeof hm->M);   // cv::invert leaves zeros for a singular matrix
  return BEVK_OK;
}

static dim3 grid2d(int w, int h) { return dim3((w + 31) / 32, (h + 7) / 8); }

// ------------------------------------------------------------------ context
struct Undistorter {
  bool valid = false, fused = false;
  int m1type = MAP_16SC2;         // the maps the slot follows: CV_16SC2 + CV_16UC1, CV_32FC1 or CV_32FC2
  Lens lens;
  DevBuf map1, map2;              // resident: CV_16SC2 + CV_16UC1, CV_32FC1's x and y planes, or CV_32FC2 in map1
  DevBuf xs;                      // cm.xs of a fused slot
  DevBuf rays;                    // lx.rays of a fused pinhole slot whose rays walk: its block starts (walk_rays)
};

struct BevCam {
  bool has_maps = false, has_mask = false;
  DevBuf map1, map2;              // device BEV maps
  std::vector<uint8_t> mask;      // host mask
};

struct bevk_ctx {
  int device = 0;
  int n_sm = 1;                             // streaming multiprocessors of the device: sizes the grid-stride launches
  cudaStream_t own = nullptr, stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_switch = nullptr;
  cudaStream_t copy_stream = nullptr;                      // H2D side of the host-pointer pipeline
  cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr};
  bool timed = false;
  long long launches = 0;
  DevBuf s_src, s_dst, s_m1, s_m2, s_o1, s_o2;   // scratch for the host-pointer entry points
  DevBuf s_xs;                                   // cm.xs of bevk_undistort_map and bevk_bev_set_camera
  DevBuf s_rays;                                 // lx.rays of a map build whose rays depend on the row
  DevBuf d_wtab;                                 // INTER_CUBIC and INTER_LANCZOS4 weight tables (build_interp_tabs), then
                                                 // their float 1-D rows for 16U / 16S / 32F sources (build_interp_rows)
  Undistorter und[8];
  // BEV engine
  int n_cam = 0, FW = 0, FH = 0, BW = 0, BH = 0;
  BevCam cam[BEVK_MAX_CAMERAS];
  bool planned = false;
  long long n_tiles = 0, n_items = 0, span_px = 0;
  int nb_override = 0;   // BEVK_NB tuning override, read at finalize
  int bev_interp = BEVK_INTER_LINEAR;   // cv2.remap interpolation the BEV LUT is compiled for
  int n_bands = 1;
  bool zero_copy_ok = true;                 // BEVK_ZEROCOPY=0 forces the DMA path
  DevBuf d_hptrs;                           // device copy of the mapped host frame pointers (per half)
  const uint8_t** h_hptrs = nullptr;        // pinned staging of those pointers
  cudaEvent_t ev_hp[2] = {nullptr, nullptr};
  long long span_fetch_bytes = 0;           // bytes k_fetch_spans moves per frame-set
  long long last_h2d_bytes = 0;             // host->device bytes of the last bevk_bev_run call
  int cam_box[BEVK_MAX_CAMERAS][BEVK_MAX_BANDS][4] = {};   // per camera and band: sampled rows [y0,y1), bytes [bx0,bx1)
  // YUV sources, per format (NV12, I420, YUYV, UYVY): page-locked ingest windows [camera][buffer rows: FH*3/2 for 4:2:0,
  // FH for 4:2:2] and their bytes per frame-set, and
  // the DMA rectangles of pageable frames per camera
  DevBuf d_yuv_win[4];
  long long yuv_fetch_bytes[4] = {0, 0, 0, 0};
  std::vector<int4> yuv_rects[4][BEVK_MAX_CAMERAS];
  DevBuf d_tiles, d_items, d_lut, d_hsv;
  int bev_grid[6] = {0, 0, 0, 0, 0, 0};   // resident CTAs of k_bev<BAL, NB>: index = 3*BAL + {NB=1:0, 4:1, 8:2}
  DevBuf d_frames, d_canvas, d_car, d_vsum, d_delta, d_csum;
  DevBuf d_spans, d_bal;                    // BALANCE: sampled row spans per camera, balanced frame copies
  DevBuf d_out_bgr, d_out_yuv;              // YUV output: BGR canvases of the device entry points, YUV canvases of bevk_bev_run
  DevBuf d_user_ptrs;                       // bevk_bev_run_frames: device copy of the caller's frame table
  std::vector<const void*> user_tab;        // ... and what it currently holds
  DevBuf d_yuv_tab;                         // bevk_bev_run_yuv_surfaces: device copy of the plane table, plane-major
  std::vector<const void*> yuv_tab;         // ... and what it currently holds
  // TMA-staged kernel (bevk_bev_tma.cuh): its plan, and the tensor maps of the frame stacks seen recently
  bool tma_planned = false;
  int tma_stage_bytes = 0;
  long long tma_items = 0, tma_box_bytes = 0, tma_entries = 0, tma_gather_entries = 0;
  std::vector<int2> tma_shapes;
  DevBuf d_ttiles, d_titems, d_tlut, d_unit_counter;
  struct MapSet { const void* base = nullptr; long long stride = 0, frames = 0; DevBuf d; unsigned long long used = 0; };
  MapSet maps[4];
  unsigned long long map_clock = 0;
  int tma_cfg = 0;                          // index into kTmaConfigs
  int tma_backoff_ns = 0;                   // BEVK_TMA_BACKOFF (read at finalize): producer poll interval when the ring is full
  int tma_grid[kMaxTmaConfigs][4] = {};                  // [config] resident CTAs of k_bev_tma<BAL, NB>: index = 2*BAL + {NB=1:0, 4:1}
  int last_path = 0;                        // 1: k_bev (global-offset gather), 2: k_bev_tma
  int gather_path = 0;                      // stand-alone gathers: 4 = k_gather4 (word path), 1 = k_gather (byte path),
                                            // 2 = k_gather_taps (CUBIC / LANCZOS4)
  // multi-GPU sharding (bevk_shard_*): partition, slab geometry, NCCL communicator
  struct Shard {
    bool configured = false, geometry = false;
    int policy = 0, rank = 0, world = 1;
    int cam_lo[SHARD_MAX_RANKS] = {}, cam_hi[SHARD_MAX_RANKS] = {};
    SlabRect rect[SHARD_MAX_RANKS] = {};
    long long slab_bytes = 0;
    void* comm = nullptr;                   // ncclComm_t
    DevBuf d_slabs;
    DevBuf d_vsums;                         // BALANCE: V sums [world][batch][n_cam], block r from rank r
    long long last_link_bytes = 0;
    // peer-store exchange (bevk_bev_run_scattered): this rank's receive buffer [2 halves][world][own_max][slab_bytes],
    // the same buffer of every peer mapped through CUDA IPC, and a 4-byte-per-rank scratch for the step barrier
    void* recv = nullptr; size_t recv_bytes = 0; int prepared_batch = 0, own_max = 0;
    void* peer_recv[SHARD_MAX_RANKS] = {}; bool attached = false;
    DevBuf d_flag;
    unsigned step = 0;
  } shard;
  // nvJPEG ingest (bevk_jpeg_decode): library handle + decoder state, created on first use
  void* jpeg_handle = nullptr; void* jpeg_state = nullptr;
  DevBuf d_jpeg_frames, d_jpeg_canvas;
  // The streams of every encoder (JPEG, progressive JPEG, PNG) on their way to the host: two slots, so that one batch can
  // be encoded while the streams of the one before are still being copied out on out_stream.  A slot's `out` holds the
  // compacted streams and its `meta` their offsets [n], sizes [n] and running end [1].
  struct EncOut {
    DevBuf out[2], meta[2];
    unsigned long long* h_sizes[2] = {nullptr, nullptr};   // page-locked copies of a slot's stream sizes
    size_t h_sizes_cap[2] = {0, 0};
    cudaStream_t out_stream = nullptr;                      // D2H of the streams
    cudaEvent_t ev_sizes[2] = {nullptr, nullptr}, ev_out_free[2] = {nullptr, nullptr};
  } enc_out;
  // JPEG encoder (bevk_jpeg_encode, bevk_jpeg_encode_params): the cv2.imwrite parameters of bevk_jpeg_set_params, the
  // header (baseline) or frame prefix (progressive) and tables of the last (width, height, normalised options), and the
  // work buffers of both entropy coders.
  struct JpegEnc {
    std::vector<int> params;
    int w = 0, h = 0;
    jpeg::Opts o{0, 0, -1, -1};
    uint8_t header[jpeg::kMaxHeaderBytes] = {};
    DevBuf d_header, d_tabs, coef, bits, offs, dcdiff, words, ffcnt, ffscan, scan_tmp;
    DevBuf ilen, iofs, counts, huff, hdrs, hlen;   // restart intervals (segments); optimised tables
    DevBuf desc, pe, pc, ph, jump, jump2, mark, rs, codes, ins, insx;   // progressive only (bevk_jpeg_prog.cuh)
  } enc;
  // PNG encoder (bevk_png_encode): the cv2.imwrite parameters of bevk_png_set_params and the work buffers of one group
  // of images (bevk_png_enc.cuh).
  struct PngEnc {
    std::vector<int> params;
    DevBuf f, rowad, runs, symidx, syms, nsym, blk, codes, hdr, zw, zbytes, scan_tmp;
    DevBuf nblk, keys, keys2, pos, pos2, prev, recs, jump, jump2, mark, cnt, dists;   // nblk; the hash-chain parse
  } png;
  // CUDA graphs captured from the device-pointer entry points (bevk_graph_*)
  bool capturing = false;
  long long capture_launches0 = 0;
  struct Graph { cudaGraph_t g = nullptr; cudaGraphExec_t x = nullptr; long long kernels = 0; };
  std::vector<Graph> graphs;
  ~bevk_ctx();   // releases every handle that is set: safe on a partly built ctx; the DevBufs free themselves
};

static int use(bevk_ctx* c) {
  if (!c) return fail(BEVK_ERR_ARG, "null ctx");
  CU(cudaSetDevice(c->device));
  return BEVK_OK;
}

// The table of OpenCV's running _x per column (bevk_device.cuh, xs_table_applies) into buf, with cm->xs pointing at it;
// rays that depend on the row keep cm->xs null.  buf must outlive every kernel launched with *cm.
static int attach_xs_table(bevk_ctx* c, DevBuf& buf, CamModel* cm) {
  cm->xs = nullptr;
  if (!xs_table_applies(*cm)) return BEVK_OK;
  if (c->capturing) return fail(BEVK_ERR_ARG, "a camera model cannot be set up inside a graph capture");
  std::vector<double> xs((size_t)cm->w);
  fill_xs_table(*cm, xs.data());
  RET(buf.ensure(xs.size() * sizeof(double)));
  CU(cudaMemcpyAsync(buf.p, xs.data(), xs.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  cm->xs = buf.as<double>();
  return BEVK_OK;
}
#define LAUNCHED(c)                 \
  do {                              \
    (c)->launches++;                \
    CU(cudaGetLastError());         \
  } while (0)

// All bevk_* functions get C linkage from their declarations in include/bevk.h.

int bevk_version(void) { return 100; }
const char* bevk_last_error(void) { return g_err.c_str(); }

int bevk_ctx_create(int device, bevk_ctx** out) {
  if (!out) return fail(BEVK_ERR_ARG, "null out");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    return fail(BEVK_ERR_CUDA, "no CUDA device (%s); libbevk has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= n) return fail(BEVK_ERR_ARG, "device %d out of range [0,%d)", device, n);
  CU(cudaSetDevice(device));
  bevk_ctx* c = new (std::nothrow) bevk_ctx;
  if (!c) return fail(BEVK_ERR_OOM, "host allocation failed");
  c->device = device;
  cudaError_t e0 = cudaDeviceGetAttribute(&c->n_sm, cudaDevAttrMultiProcessorCount, device);
  cudaError_t e1 = e0 == cudaSuccess ? cudaStreamCreateWithFlags(&c->own, cudaStreamNonBlocking) : e0;
  cudaError_t e2 = e1 == cudaSuccess ? cudaEventCreate(&c->ev0) : e1;
  cudaError_t e3 = e2 == cudaSuccess ? cudaEventCreate(&c->ev1) : e2;
  if (e3 != cudaSuccess) {
    delete c;
    return fail(BEVK_ERR_CUDA, "context setup: %s", cudaGetErrorString(e3));
  }
  c->stream = c->own;
  // The weight tables of INTER_CUBIC / INTER_LANCZOS4 are uploaded here, so that the enqueue-only gathers
  // (bevk_undistort_stack, also under graph capture) never allocate or copy.
  static const std::vector<short> tabs = [] {
    std::vector<short> t(INTERP_TAB_SHORTS + INTERP_ROWS_FLOATS * 2);
    build_interp_tabs(t.data());
    float rows[INTERP_ROWS_FLOATS];
    build_interp_rows(rows);
    memcpy(t.data() + INTERP_TAB_SHORTS, rows, sizeof rows);
    return t;
  }();
  int r = c->d_wtab.ensure(tabs.size() * sizeof(short));
  if (r == BEVK_OK) {
    cudaError_t e4 = cudaMemcpyAsync(c->d_wtab.p, tabs.data(), tabs.size() * sizeof(short), cudaMemcpyHostToDevice, c->own);
    if (e4 == cudaSuccess) e4 = cudaStreamSynchronize(c->own);
    if (e4 != cudaSuccess) r = fail(BEVK_ERR_CUDA, "weight table upload: %s", cudaGetErrorString(e4));
  }
  if (r != BEVK_OK) {
    delete c;
    return r;
  }
  *out = c;
  return BEVK_OK;
}

static void shard_release(bevk_ctx* c);
static void jpeg_release(bevk_ctx* c);

bevk_ctx::~bevk_ctx() {
  shard_release(this);
  jpeg_release(this);
  for (auto& g : graphs) { if (g.x) cudaGraphExecDestroy(g.x); if (g.g) cudaGraphDestroy(g.g); }
  for (cudaEvent_t e : {ev0, ev1, ev_switch, ev_in[0], ev_in[1], ev_free[0], ev_free[1], ev_hp[0], ev_hp[1], enc_out.ev_sizes[0],
                        enc_out.ev_sizes[1], enc_out.ev_out_free[0], enc_out.ev_out_free[1]})
    if (e) cudaEventDestroy(e);
  for (cudaStream_t s : {copy_stream, enc_out.out_stream, own})
    if (s) cudaStreamDestroy(s);
  for (void* p : {(void*)h_hptrs, (void*)enc_out.h_sizes[0], (void*)enc_out.h_sizes[1]})
    if (p) cudaFreeHost(p);
}

int bevk_ctx_destroy(bevk_ctx* c) {
  if (!c) return BEVK_OK;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();   // not c->stream: a caller-owned stream handed to bevk_ctx_set_stream may be gone by now
  delete c;
  return BEVK_OK;
}

// A stream and its events, created all or nothing: on failure every handle is destroyed and left null, so that the next
// call tries again.
static int create_stream_set(cudaStream_t* s, std::initializer_list<cudaEvent_t*> events) {
  cudaError_t e = cudaStreamCreateWithFlags(s, cudaStreamNonBlocking);
  for (cudaEvent_t* ev : events)
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(ev, cudaEventDisableTiming);
  if (e == cudaSuccess) return BEVK_OK;
  for (cudaEvent_t* ev : events) { if (*ev) cudaEventDestroy(*ev); *ev = nullptr; }
  if (*s) cudaStreamDestroy(*s);
  *s = nullptr;
  return fail(e == cudaErrorMemoryAllocation ? BEVK_ERR_OOM : BEVK_ERR_CUDA, "stream set-up: %s", cudaGetErrorString(e));
}

int bevk_ctx_set_stream(bevk_ctx* c, void* s) {
  RET(use(c));
  cudaStream_t next = s ? reinterpret_cast<cudaStream_t>(s) : c->own;
  if (next == c->stream) return BEVK_OK;
  if (c->capturing) return fail(BEVK_ERR_ARG, "cannot change the stream inside a graph capture");
  // Everything this ctx enqueued so far (kernels that read its cached tables, uploads that wrote them) is ordered before
  // whatever it enqueues on the new stream: no host synchronisation, no table is dropped.
  if (!c->ev_switch) CU(cudaEventCreateWithFlags(&c->ev_switch, cudaEventDisableTiming));
  if (cudaEventRecord(c->ev_switch, c->stream) == cudaSuccess) CU(cudaStreamWaitEvent(next, c->ev_switch, 0));
  else cudaGetLastError();   // the old (caller-owned) stream is gone: nothing of it can still be running
  c->stream = next;
  return BEVK_OK;
}

int bevk_ctx_sync(bevk_ctx* c) {
  RET(use(c));
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

int bevk_device_pci_bus_id(int device, char* out, int len) {
  if (!out || len < 16) return fail(BEVK_ERR_ARG, "bus id buffer too small");
  CU(cudaDeviceGetPCIBusId(out, len, device));
  return BEVK_OK;
}

int bevk_host_alloc(uint64_t bytes, void** out) {
  if (!out) return fail(BEVK_ERR_ARG, "null out");
  CU(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
  return BEVK_OK;
}
int bevk_host_free(void* p) {
  if (p) CU(cudaFreeHost(p));
  return BEVK_OK;
}

// ------------------------------------------------------------------ K1
// The walked rays of L (walk_rays, k_walk_rays) into buf, with L->lx.rays pointing at them: 24 bytes per map entry for the
// fisheye (126 MB at 2560 x 2048), 3 for the pinhole's block starts.
static int walk_into(bevk_ctx* c, DevBuf& buf, Lens* L) {
  const CamModel& cm = L->cm;
  if (c->capturing) return fail(BEVK_ERR_ARG, "a camera model cannot be set up inside a graph capture");
  RET(buf.ensure((size_t)ray_row_len(cm) * cm.h * 3 * sizeof(double)));
  if (cm.model == BEVK_MODEL_PINHOLE) k_walk_rays<1><<<(cm.h + 127) / 128, 128, 0, c->stream>>>(cm, buf.as<double>());
  else k_walk_rays<0><<<(cm.h + 127) / 128, 128, 0, c->stream>>>(cm, buf.as<double>());
  LAUNCHED(c);
  L->lx.rays = buf.as<double>();
  return BEVK_OK;
}

// Bytes per entry of a map pair of type m1type: map1 and map2 (0: none, as for CV_32FC2).
static void map_entry_bytes(int m1type, size_t* b1, size_t* b2) {
  *b1 = m1type == MAP_32FC2 ? 8 : 4;
  *b2 = m1type == MAP_16SC2 ? 2 : m1type == MAP_32FC1 ? 4 : 0;
}

// k_undistort_map (CV_16SC2 + CV_16UC1) or k_undistort_map_f32 (CV_32FC1, CV_32FC2) of L into the pair (m1, m2): cm.w x
// cm.h entries.  A camera whose rays depend on the row walks them into scratch first (walk_into), as cv2 walks each row,
// unless L already carries them (a fused slot's); the scratch is freed again once the map is built, so that a ctx does
// not hold it between set-ups.
static int build_map(bevk_ctx* c, Lens L, DevBuf& m1, DevBuf& m2, int m1type = MAP_16SC2) {
  const CamModel& cm = L.cm;
  const size_t n = (size_t)cm.w * cm.h;
  size_t b1, b2;
  map_entry_bytes(m1type, &b1, &b2);
  RET(m1.ensure(n * b1));
  if (b2) RET(m2.ensure(n * b2));
  const bool scratch = L.walks && !L.lx.rays;
  if (scratch) RET(walk_into(c, c->s_rays, &L));
  if (m1type != MAP_16SC2) {
    float* y = m1type == MAP_32FC1 ? m2.as<float>() : nullptr;
    if (L.full) k_undistort_map_f32<1><<<grid2d(cm.w, cm.h), 256, 0, c->stream>>>(cm, L.lx, m1.as<float>(), y);
    else k_undistort_map_f32<0><<<grid2d(cm.w, cm.h), 256, 0, c->stream>>>(cm, L.lx, m1.as<float>(), y);
  } else if (L.full) {
    k_undistort_map<1><<<grid2d(cm.w, cm.h), 256, 0, c->stream>>>(cm, L.lx, m1.as<short2>(), m2.as<unsigned short>());
  } else {
    k_undistort_map<0><<<grid2d(cm.w, cm.h), 256, 0, c->stream>>>(cm, L.lx, m1.as<short2>(), m2.as<unsigned short>());
  }
  LAUNCHED(c);
  if (scratch) {   // the map kernel reads the rays: wait for it before the scratch goes
    CU(cudaStreamSynchronize(c->stream));
    c->s_rays.release();
  }
  return BEVK_OK;
}

// n entries of the device map pair (m1, m2) to the caller's host maps, then wait for them
static int download_maps(bevk_ctx* c, const void* m1, const void* m2, size_t n, int16_t* map1, uint16_t* map2) {
  CU(cudaMemcpyAsync(map1, m1, n * 4, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaMemcpyAsync(map2, m2, n * 2, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

int bevk_undistort_rectify_map(bevk_ctx* c, int model, const double K[9], const double* D, int n_dist, const double* R,
                               const double P[9], int w, int h, int16_t* map1, uint16_t* map2) {
  RET(use(c));
  if (!map1 || !map2) return fail(BEVK_ERR_ARG, "null output map");
  Lens L;
  RET(make_model(model, K, D, n_dist, R, P, w, h, &L));
  RET(attach_xs_table(c, c->s_xs, &L.cm));
  RET(build_map(c, L, c->s_m1, c->s_m2));
  return download_maps(c, c->s_m1.p, c->s_m2.p, (size_t)w * h, map1, map2);
}

// n entries of a device float map pair of type m1type (CV_32FC1 / CV_32FC2) to the caller's host maps, then wait
static int download_maps_f32(bevk_ctx* c, const void* m1, const void* m2, size_t n, int m1type, float* map1, float* map2) {
  size_t b1, b2;
  map_entry_bytes(m1type, &b1, &b2);
  CU(cudaMemcpyAsync(map1, m1, n * b1, cudaMemcpyDeviceToHost, c->stream));
  if (b2) CU(cudaMemcpyAsync(map2, m2, n * b2, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

// The float map types a camera can be built into: CV_32FC1 for both models, CV_32FC2 for the pinhole only, as
// cv2.fisheye.initUndistortRectifyMap asserts on CV_32FC2.
static int check_f32_type(int model, int m1type) {
  if (m1type != MAP_32FC1 && m1type != MAP_32FC2)
    return fail(BEVK_ERR_ARG, "m1type %d: float maps are CV_32FC1 (%d) or CV_32FC2 (%d)", m1type, MAP_32FC1, MAP_32FC2);
  if (model == BEVK_MODEL_FISHEYE && m1type == MAP_32FC2)
    return fail(BEVK_ERR_ARG, "cv2.fisheye.initUndistortRectifyMap builds CV_16SC2 or CV_32FC1 maps, not CV_32FC2");
  return BEVK_OK;
}
// ... and the host maps such a build writes: CV_32FC1 needs both planes
static int check_f32_maps(int model, int m1type, const void* map1, const void* map2) {
  RET(check_f32_type(model, m1type));
  if (!map1 || (m1type == MAP_32FC1 && !map2)) return fail(BEVK_ERR_ARG, "null output map");
  return BEVK_OK;
}

int bevk_undistort_rectify_map_f32(bevk_ctx* c, int model, const double K[9], const double* D, int n_dist, const double* R,
                                   const double P[9], int w, int h, int m1type, float* map1, float* map2) {
  RET(use(c));
  RET(check_f32_maps(model, m1type, map1, map2));
  Lens L;
  RET(make_model(model, K, D, n_dist, R, P, w, h, &L));
  RET(attach_xs_table(c, c->s_xs, &L.cm));
  RET(build_map(c, L, c->s_m1, c->s_m2, m1type));
  return download_maps_f32(c, c->s_m1.p, c->s_m2.p, (size_t)w * h, m1type, map1, map2);
}

int bevk_undistort_map(bevk_ctx* c, int model, const double K[9], const double* D, int n_dist, const double P[9], int w,
                       int h, int16_t* map1, uint16_t* map2) {
  const LegacyDist d(model, D, n_dist);
  return bevk_undistort_rectify_map(c, model, K, d.D, d.n, nullptr, P, w, h, map1, map2);
}

// ------------------------------------------------------------------ image operations
// remap, undistort, warpPerspective, warpAffine and resize are each an ImageOp (what the operation adds to the frames,
// checked by its builder, which enqueues nothing) run over an ImageBatch (the frames it reads and writes) by launch().
// The host forms run it over dense scratch (host_image), the device forms over the caller's frames (device_image).

// k_gather4's word path: 32-bit tap loads need every source row to start on a 4-byte boundary (base, row pitch and, over
// a batch, image stride), and its 32-bit stores the same of the destination (padded rows are fine).  Anything else,
// e.g. caller memory at an odd address, takes k_gather's byte path; so does BORDER_TRANSPARENT, which leaves pixels
// alone that k_gather4's three-word stores of four pixels would write.
// An image's cv2 type (CV_8UC1 .. CV_32FC4): the depth (CV_8U 0, CV_16U 2, CV_16S 3, CV_32F 5), the channels and the bytes
// of one element.  Rows, images and base pointers of a wider depth are element-aligned (check_image).
struct PixType {
  int depth, channels, esize;
  long long px() const { return (long long)channels * esize; }   // bytes per pixel
};
static PixType u8(int channels) { return PixType{0, channels, 1}; }

// a cv2 type code of the image gathers: 8U, 16U, 16S and 32F; 8S and 16F, which cv2.remap refuses, and 64F are refused
static int pix_type(int type, PixType* t) {
  if (type < 0 || type >= (512 << 3)) return fail(BEVK_ERR_ARG, "image type %d is not a cv2 type code", type);
  const int depth = type & 7;
  static const int esize[8] = {1, 0, 2, 2, 0, 4, 0, 0};
  if (!esize[depth])
    return fail(BEVK_ERR_UNSUPPORTED, "image type %d: depth %d; the gathers take CV_8U, CV_16U, CV_16S and CV_32F images",
                type, depth);
  *t = PixType{depth, (type >> 3) + 1, esize[depth]};
  return BEVK_OK;
}

static bool gather4_ok(const GatherArgs& a, PixType t, int interp, int mode) {
  const int channels = t.esize == 1 ? t.channels : 0;   // the word path is 8-bit only
  const uintptr_t al = reinterpret_cast<uintptr_t>(a.src) | reinterpret_cast<uintptr_t>(a.dst) | (uintptr_t)a.spitch |
                       (uintptr_t)a.dpitch | (a.n > 1 ? (uintptr_t)(a.sistride | a.distride) : 0);
  return channels == 3 && interp == BEVK_INTER_LINEAR && a.bd.mode != BORDER_TRANSPARENT && (a.dw % 4) == 0 && (al & 3) == 0 &&
         a.spitch < (1ll << 31) / std::max(1, a.sh) && (mode != 0 || a.map2 != nullptr) &&
         (mode != 4 || ((reinterpret_cast<uintptr_t>(a.fmap1) | reinterpret_cast<uintptr_t>(a.fmap2)) & 15) == 0);   // float4 loads
}

// The interpolation flag of the image gathers: INTER_AREA is read as INTER_LINEAR, as cv2.remap and cv2.warpPerspective
// read it; anything but NEAREST, LINEAR, CUBIC and LANCZOS4 is refused.
static int gather_interp(int* interp) {
  if (*interp == BEVK_INTER_AREA) *interp = BEVK_INTER_LINEAR;
  if (*interp != BEVK_INTER_NEAREST && *interp != BEVK_INTER_LINEAR && *interp != BEVK_INTER_CUBIC && *interp != BEVK_INTER_LANCZOS4)
    return fail(BEVK_ERR_UNSUPPORTED, "interp %d", *interp);
  return BEVK_OK;
}

// n >= 1 frames: source and destination images, rows `pitch` bytes apart and images `istride` bytes apart (0 when n = 1)
struct ImageBatch {
  const uint8_t* src; int sw, sh; long long spitch, sistride;
  uint8_t* dst; int dw, dh; long long dpitch, distride;
  int n;
};

constexpr int OP_RESIZE = 6;   // ImageOp::mode after the gathers' MODE 0..5

struct ImageOp {
  int mode = 0;                     // the gathers' MODE (0 maps, 1 camera model, 2 homography, 3 affine, 4 float maps,
                                    // 5 camera model through float maps) or OP_RESIZE
  bool lens = false;                // MODE 1 / 5: the camera needs the LENS = 1 instances (lens_model)
  int interp = 0;                   // a gather's interpolation after gather_interp; a resize's body (resize_kind)
  GatherArgs g{};                   // a gather's maps, camera model or inverse matrix
  ResizeArgs r{};                   // a resize's scales
  int slot = -1, dw = 0, dh = 0;    // an undistorter slot and the size of the images it writes
  // bevk_remap*: the bytes of the caller's maps in g.map1 / g.map2, 0 for none.  host_launch uploads host maps once every
  // check has passed; device_image refuses images written over device maps.
  size_t map1_bytes = 0, map2_bytes = 0;
};

// a (GatherArgs or ResizeArgs) with its frame fields taken from b
template <class Args>
static Args with_frames(Args a, const ImageBatch& b) {
  a.src = b.src; a.sw = b.sw; a.sh = b.sh; a.spitch = b.spitch; a.sistride = b.sistride;
  a.dst = b.dst; a.dw = b.dw; a.dh = b.dh; a.dpitch = b.dpitch; a.distride = b.distride;
  a.n = b.n;
  return a;
}

// bd: a border other than a zero BORDER_CONSTANT, which the _border kernels take; the zero-constant kernels keep their
// machine code
template <int MODE, int LENS, class T>
static void gather_t(bevk_ctx* c, const GatherArgs& a, int channels, int interp, bool bd, unsigned gz) {
  const dim3 g((a.dw + 31) / 32, (a.dh + 7) / 8, gz);
#define GO(C, L)                                                                      \
  (bd ? k_gather_border<MODE, C, L, LENS, T><<<g, 256, 0, c->stream>>>(a)             \
      : k_gather<MODE, C, L, LENS, T><<<g, 256, 0, c->stream>>>(a))
#define TAPS(C, KS)                                                                   \
  (bd ? k_gather_taps_border<MODE, C, KS, LENS, T><<<g, 256, 0, c->stream>>>(a, wt)   \
      : k_gather_taps<MODE, C, KS, LENS, T><<<g, 256, 0, c->stream>>>(a, wt))
  if (interp == BEVK_INTER_CUBIC || interp == BEVK_INTER_LANCZOS4) {
    const TapWeights<T>* wt;
    if constexpr (sizeof(T) == 1) wt = c->d_wtab.as<short>() + (interp == BEVK_INTER_CUBIC ? 0 : INTERP_TAB_LANCZOS4);
    else wt = reinterpret_cast<const float*>(c->d_wtab.as<short>() + INTERP_TAB_SHORTS) +
              (interp == BEVK_INTER_CUBIC ? 0 : INTERP_ROWS_LANCZOS4);
    if (interp == BEVK_INTER_CUBIC) {
      if (channels == 1) TAPS(1, 4); else if (channels == 3) TAPS(3, 4); else TAPS(4, 4);
    } else {
      if (channels == 1) TAPS(1, 8); else if (channels == 3) TAPS(3, 8); else TAPS(4, 8);
    }
  } else if (interp == BEVK_INTER_LINEAR) {
    if (channels == 1) GO(1, 1); else if (channels == 3) GO(3, 1); else GO(4, 1);
  } else {
    if (channels == 1) GO(1, 0); else if (channels == 3) GO(3, 0); else GO(4, 0);
  }
#undef GO
#undef TAPS
}

template <int MODE, int LENS>
static void gather(bevk_ctx* c, const GatherArgs& a, PixType t, int interp, bool words, unsigned gz) {
  bool bd = a.bd.mode != BORDER_CONSTANT;
  for (unsigned char v : a.bd.v) bd |= v != 0;
  if (words) {
    // 4 output pixels per thread, 32-bit tap loads and 12-byte stores
    const dim3 g4((a.dw / 4 + 31) / 32, (a.dh + 7) / 8, gz);
    if (bd) {
      if (a.n == 1) k_gather4_border<MODE, 1, LENS><<<g4, 256, 0, c->stream>>>(a);
      else k_gather4_border<MODE, GATHER_NB, LENS><<<g4, 256, 0, c->stream>>>(a);
    } else {
      if (a.n == 1) k_gather4<MODE, 1, LENS><<<g4, 256, 0, c->stream>>>(a);
      else k_gather4<MODE, GATHER_NB, LENS><<<g4, 256, 0, c->stream>>>(a);
    }
    return;
  }
  switch (t.depth) {
    case 0: gather_t<MODE, LENS, uint8_t>(c, a, t.channels, interp, bd, gz); break;
    case 2: gather_t<MODE, LENS, uint16_t>(c, a, t.channels, interp, bd, gz); break;
    case 3: gather_t<MODE, LENS, int16_t>(c, a, t.channels, interp, bd, gz); break;
    default: gather_t<MODE, LENS, float>(c, a, t.channels, interp, bd, gz);
  }
}

template <int C, int KIND>
static void resize_c(bevk_ctx* c, const ResizeArgs& a, dim3 g) {
  if (a.n > 1) k_resize<C, KIND, GATHER_NB><<<g, 256, 0, c->stream>>>(a);
  else k_resize<C, KIND, 1><<<g, 256, 0, c->stream>>>(a);
}
template <int C>
static void resize_k(bevk_ctx* c, const ResizeArgs& a, int kind, dim3 g) {
  switch (kind) {
    case RZ_NEAREST: resize_c<C, RZ_NEAREST>(c, a, g); break;
    case RZ_LINEAR: resize_c<C, RZ_LINEAR>(c, a, g); break;
    case RZ_AREA_LINEAR: resize_c<C, RZ_AREA_LINEAR>(c, a, g); break;
    case RZ_AREA_FAST: resize_c<C, RZ_AREA_FAST>(c, a, g); break;
    default: resize_c<C, RZ_AREA>(c, a, g);
  }
}

// Enqueue op over b.n >= 1 frames.  grid.z = frame groups of GATHER_NB, at most 65535 per launch; a single frame takes
// the kernels' single-frame form (NB = 1), which keeps the register count and speed of the one-frame kernel.
static int launch(bevk_ctx* c, const ImageOp& op, const ImageBatch& b, PixType t) {
  const bool words = op.mode != OP_RESIZE && gather4_ok(with_frames(op.g, b), t, op.interp, op.mode);
  const int channels = t.channels;
  const int per_launch = 65535 * GATHER_NB;
  for (int f0 = 0; f0 < b.n; f0 += per_launch) {
    ImageBatch p = b;
    p.n = std::min(per_launch, b.n - f0);
    p.src += (long long)f0 * b.sistride;
    p.dst += (long long)f0 * b.distride;
    const unsigned gz = (unsigned)((p.n + GATHER_NB - 1) / GATHER_NB);
    if (op.mode != OP_RESIZE) {
      const GatherArgs a = with_frames(op.g, p);
      switch (op.mode) {
        case 0: gather<0, 0>(c, a, t, op.interp, words, gz); break;
        case 1:
          if (op.lens) gather<1, 1>(c, a, t, op.interp, words, gz);
          else gather<1, 0>(c, a, t, op.interp, words, gz);
          break;
        case 2: gather<2, 0>(c, a, t, op.interp, words, gz); break;
        case 3: gather<3, 0>(c, a, t, op.interp, words, gz); break;
        case 4: gather<4, 0>(c, a, t, op.interp, words, gz); break;
        default:
          if (op.lens) gather<5, 1>(c, a, t, op.interp, words, gz);
          else gather<5, 0>(c, a, t, op.interp, words, gz);
      }
    } else {
      const ResizeArgs a = with_frames(op.r, p);
      const dim3 g((a.dw + 31) / 32, (a.dh + 7) / 8, gz);
      if (channels == 1) resize_k<1>(c, a, op.interp, g);
      else if (channels == 3) resize_k<3>(c, a, op.interp, g);
      else resize_k<4>(c, a, op.interp, g);
    }
    LAUNCHED(c);
  }
  const bool taps = op.interp == BEVK_INTER_CUBIC || op.interp == BEVK_INTER_LANCZOS4;
  c->gather_path = op.mode == OP_RESIZE ? 3 : words ? 4 : taps ? 2 : 1;
  return BEVK_OK;
}

// ---- the operations' builders: each makes the refusals of its operation's own arguments and fills a default op
// dw x dh CV_16SC2 + CV_16UC1 maps, map2 null for NEAREST without fractions
static int remap_op(const int16_t* map1, const uint16_t* map2, int interp, int dw, int dh, ImageOp* op) {
  if (!map1) return fail(BEVK_ERR_ARG, "null map1");
  RET(gather_interp(&interp));
  if (interp != BEVK_INTER_NEAREST && !map2) return fail(BEVK_ERR_ARG, "interpolation %d needs map2", interp);
  op->interp = interp;
  const size_t n = (size_t)dw * dh;
  op->g.map1 = reinterpret_cast<const short2*>(map1); op->g.map2 = map2;
  op->map1_bytes = n * 4; op->map2_bytes = map2 ? n * 2 : 0;
  return BEVK_OK;
}

// dw x dh float maps: map2 null means map1 is CV_32FC2
static int remap_f32_op(const float* map1, const float* map2, int interp, int dw, int dh, ImageOp* op) {
  if (!map1) return fail(BEVK_ERR_ARG, "null map1");
  RET(gather_interp(&interp));
  op->mode = 4;
  op->interp = interp;
  const size_t n = (size_t)dw * dh;
  op->g.fmap1 = map1; op->g.fmap2 = map2;
  op->map1_bytes = map2 ? n * 4 : n * 8; op->map2_bytes = map2 ? n * 4 : 0;
  return BEVK_OK;
}

static int need_undistorter(bevk_ctx* c, int slot) {
  if (slot < 0 || slot >= 8 || !c->und[slot].valid) return fail(BEVK_ERR_ARG, "undistorter slot %d not set", slot);
  return BEVK_OK;
}

// a slot's resident map (MODE 0, float: 4) or, fused, its camera model (MODE 1, float: 5); the images it writes are the
// map's size
static int undistort_op(bevk_ctx* c, int slot, int interp, ImageOp* op) {
  RET(need_undistorter(c, slot));
  RET(gather_interp(&interp));
  const Undistorter& u = c->und[slot];
  const bool f32 = u.m1type != MAP_16SC2;
  op->mode = u.fused ? (f32 ? 5 : 1) : (f32 ? 4 : 0);
  op->interp = interp;
  if (u.fused) { op->g.cm = u.lens.cm; op->g.lx = u.lens.lx; op->lens = u.lens.full; }
  else if (f32) { op->g.fmap1 = u.map1.as<float>(); op->g.fmap2 = u.m1type == MAP_32FC1 ? u.map2.as<float>() : nullptr; }
  else { op->g.map1 = u.map1.as<short2>(); op->g.map2 = u.map2.as<unsigned short>(); }
  op->slot = slot; op->dw = u.lens.cm.w; op->dh = u.lens.cm.h;
  return BEVK_OK;
}

static int perspective_op(const double* H, int interp, ImageOp* op) {
  RET(gather_interp(&interp));
  op->mode = 2;
  op->interp = interp;
  return make_homog(H, &op->g.hm);
}

// flags -> interpolation (gather_interp's) and the inverse map in hm.M[0..5]
static int affine_op(const double* M, int flags, ImageOp* op) {
  if (!M) return fail(BEVK_ERR_ARG, "null M");
  if (flags & ~(7 | BEVK_WARP_INVERSE_MAP)) return fail(BEVK_ERR_UNSUPPORTED, "warpAffine flags %d", flags);
  int interp = flags & 7;
  RET(gather_interp(&interp));
  op->mode = 3;
  op->interp = interp;
  if (flags & BEVK_WARP_INVERSE_MAP) memcpy(op->g.hm.M, M, 6 * sizeof(double));
  else inv_affine(M, op->g.hm.M);
  return BEVK_OK;
}

// interp and cv2's size rule (resize_geometry): the scales and the body
static int resize_op(int sw, int sh, int dw, int dh, double fx, double fy, int interp, ImageOp* op) {
  if (interp != BEVK_INTER_NEAREST && interp != BEVK_INTER_LINEAR && interp != BEVK_INTER_AREA)
    return fail(BEVK_ERR_UNSUPPORTED, "resize interp %d: INTER_NEAREST, INTER_LINEAR and INTER_AREA only", interp);
  if (sw <= 0 || sh <= 0 || dw <= 0 || dh <= 0) return fail(BEVK_ERR_ARG, "bad size %dx%d -> %dx%d", sw, sh, dw, dh);
  op->mode = OP_RESIZE;
  ResizeArgs& a = op->r;
  if (fx == 0. && fy == 0.) {
    a.inv_x = (double)dw / sw; a.inv_y = (double)dh / sh;
  } else {
    int w = 0, h = 0;
    a.inv_x = fx; a.inv_y = fy;
    if (!resize_geometry(sw, sh, &w, &h, &a.inv_x, &a.inv_y))
      return fail(BEVK_ERR_ARG, "fx %g, fy %g give no image from %dx%d", fx, fy, sw, sh);
    if (w != dw || h != dh) return fail(BEVK_ERR_ARG, "fx %g, fy %g make %dx%d images, the caller expects %dx%d", fx, fy, w, h, dw, dh);
  }
  op->interp = resize_kind(interp, a);
  return BEVK_OK;
}

// ---- the two paths: the source is checked, then the destination (an undistorter slot's size first)
static int check_op_size(const ImageOp& op, int dw, int dh) {
  if (op.slot >= 0 && (dw != op.dw || dh != op.dh))   // the caller sized dst for another map: never write past it
    return fail(BEVK_ERR_ARG, "undistorter slot %d holds a %dx%d map, the caller expects %dx%d", op.slot, op.dw, op.dh, dw, dh);
  return BEVK_OK;
}

static int check_image(const void* p, int w, int h, int64_t stride, PixType t, const char* what) {
  if (!p) return fail(BEVK_ERR_ARG, "null %s", what);
  if (w <= 0 || h <= 0) return fail(BEVK_ERR_ARG, "bad %s size %dx%d", what, w, h);
  if (t.channels != 1 && t.channels != 3 && t.channels != 4) return fail(BEVK_ERR_UNSUPPORTED, "channels must be 1, 3 or 4");
  if (stride < (int64_t)w * t.px()) return fail(BEVK_ERR_ARG, "%s stride %lld < row bytes", what, (long long)stride);
  if ((reinterpret_cast<uintptr_t>(p) | (uintptr_t)stride) % t.esize)
    return fail(BEVK_ERR_ARG, "%s base %p and row stride %lld must be multiples of the %d-byte element", what, p,
                (long long)stride, t.esize);
  return BEVK_OK;
}

static int upload_image(bevk_ctx* c, DevBuf& buf, const void* src, int w, int h, int64_t stride, PixType t) {
  const size_t row = (size_t)(w * t.px());
  RET(buf.ensure(row * h));
  if ((size_t)stride == row) CU(cudaMemcpyAsync(buf.p, src, row * h, cudaMemcpyHostToDevice, c->stream));   // dense: one DMA
  else CU(cudaMemcpy2DAsync(buf.p, row, src, (size_t)stride, row, h, cudaMemcpyHostToDevice, c->stream));
  return BEVK_OK;
}
static int download_image(bevk_ctx* c, const DevBuf& buf, void* dst, int w, int h, int64_t stride, PixType t) {
  const size_t row = (size_t)(w * t.px());
  if ((size_t)stride == row) CU(cudaMemcpyAsync(dst, buf.p, row * h, cudaMemcpyDeviceToHost, c->stream));
  else CU(cudaMemcpy2DAsync(dst, (size_t)stride, buf.p, row, row, h, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

// Host path, without the read-back: a checked host frame uploaded to c->s_src and op run into c->s_dst.  Both are dense
// (row pitch w times the pixel bytes), so k_gather4's word-path choice sees the same pitches whatever the caller's strides.
// BORDER_TRANSPARENT leaves some destination pixels as they are: the caller's dst (dstride) is uploaded into c->s_dst first.
static int host_launch(bevk_ctx* c, ImageOp op, const void* src, int sw, int sh, int64_t sstride, PixType t, int dw, int dh,
                       const void* dst = nullptr, int64_t dstride = 0) {
  RET(upload_image(c, c->s_src, src, sw, sh, sstride, t));
  if (op.mode != OP_RESIZE && op.g.bd.mode == BORDER_TRANSPARENT) RET(upload_image(c, c->s_dst, dst, dw, dh, dstride, t));
  else RET(c->s_dst.ensure((size_t)dw * dh * t.px()));
  if (op.map1_bytes) {
    RET(c->s_m1.ensure(op.map1_bytes));
    CU(cudaMemcpyAsync(c->s_m1.p, op.g.map1, op.map1_bytes, cudaMemcpyHostToDevice, c->stream));
    op.g.map1 = c->s_m1.as<short2>();
  }
  if (op.map2_bytes) {
    RET(c->s_m2.ensure(op.map2_bytes));
    CU(cudaMemcpyAsync(c->s_m2.p, op.g.map2, op.map2_bytes, cudaMemcpyHostToDevice, c->stream));
    op.g.map2 = c->s_m2.as<unsigned short>();
  }
  const ImageBatch b{c->s_src.as<uint8_t>(), sw, sh, sw * t.px(), 0, c->s_dst.as<uint8_t>(), dw, dh, dw * t.px(), 0, 1};
  return launch(c, op, b, t);
}

// Host path: one host image through op into another, which the call has written when it returns.
static int host_image(bevk_ctx* c, const ImageOp& op, const void* src, int sw, int sh, int64_t sstride, PixType t, void* dst,
                      int dw, int dh, int64_t dstride) {
  RET(check_image(src, sw, sh, sstride, t, "src"));
  RET(check_op_size(op, dw, dh));
  RET(check_image(dst, dw, dh, dstride, t, "dst"));
  RET(host_launch(c, op, src, sw, sh, sstride, t, dw, dh, dst, dstride));
  return download_image(c, c->s_dst, dst, dw, dh, dstride, t);
}

// The source side of the device-batch calls: a frame, n >= 1, and an image stride that covers an image when n > 1.
static int check_stack_src(const void* d_src, int64_t sis, int sw, int sh, int64_t srs, PixType t, int n) {
  if (n < 1) return fail(BEVK_ERR_ARG, "n must be >= 1, got %d", n);
  RET(check_image(d_src, sw, sh, srs, t, "src"));
  if (n > 1 && sis < (int64_t)(sh - 1) * srs + sw * t.px())
    return fail(BEVK_ERR_ARG, "src image stride %lld is smaller than one image", (long long)sis);
  if (n > 1 && sis % t.esize)
    return fail(BEVK_ERR_ARG, "src image stride %lld must be a multiple of the %d-byte element", (long long)sis, t.esize);
  return BEVK_OK;
}

// The destination side of the device-batch calls, given a checked source: rows, an image stride that covers an image
// (n > 1), and byte ranges [first, last] of the whole batch on each side that do not overlap -- an output that overwrites
// frames still to be read is refused.
static int check_stack_dst(const void* d_src, int64_t sis, int sw, int sh, int64_t srs, PixType t, int n, const void* d_dst,
                           int64_t dis, int dw, int dh, int64_t drs) {
  RET(check_image(d_dst, dw, dh, drs, t, "dst"));
  const int64_t dimg = (int64_t)(dh - 1) * drs + dw * t.px();
  if (n > 1 && dis < dimg) return fail(BEVK_ERR_ARG, "dst image stride %lld is smaller than one image", (long long)dis);
  if (n > 1 && dis % t.esize)
    return fail(BEVK_ERR_ARG, "dst image stride %lld must be a multiple of the %d-byte element", (long long)dis, t.esize);
  const uintptr_t s0 = reinterpret_cast<uintptr_t>(d_src), d0 = reinterpret_cast<uintptr_t>(d_dst);
  const uintptr_t s1 = s0 + (uintptr_t)(n > 1 ? (n - 1) * sis : 0) + (uintptr_t)((int64_t)(sh - 1) * srs + sw * t.px());
  const uintptr_t d1 = d0 + (uintptr_t)(n > 1 ? (n - 1) * dis : 0) + (uintptr_t)dimg;
  if (s0 < d1 && d0 < s1) return fail(BEVK_ERR_ARG, "the destination range overlaps the source frames");
  return BEVK_OK;
}

// the caller's n device frames; an image stride only matters when n > 1
static ImageBatch device_batch(const void* d_src, int64_t sis, int sw, int sh, int64_t srs, int n, void* d_dst, int64_t dis,
                               int dw, int dh, int64_t drs) {
  return ImageBatch{reinterpret_cast<const uint8_t*>(d_src), sw, sh, srs, n > 1 ? sis : 0,
                    reinterpret_cast<uint8_t*>(d_dst), dw, dh, drs, n > 1 ? dis : 0, n};
}

// Device path: n device frames through op, enqueued only.  It allocates and copies nothing, so a graph can capture it.
static int device_image(bevk_ctx* c, const ImageOp& op, const void* d_src, int64_t sis, int sw, int sh, int64_t srs, PixType t,
                        int n, void* d_dst, int64_t dis, int dw, int dh, int64_t drs) {
  RET(check_stack_src(d_src, sis, sw, sh, srs, t, n));
  RET(check_op_size(op, dw, dh));
  RET(check_stack_dst(d_src, sis, sw, sh, srs, t, n, d_dst, dis, dw, dh, drs));
  if (op.map1_bytes) {   // the caller's maps: the images written must not overwrite them
    const uintptr_t d0 = reinterpret_cast<uintptr_t>(d_dst);
    const uintptr_t d1 = d0 + (uintptr_t)(n > 1 ? (n - 1) * dis : 0) + (uintptr_t)((int64_t)(dh - 1) * drs + dw * t.px());
    const uintptr_t x0 = reinterpret_cast<uintptr_t>(op.g.map1), x1 = x0 + op.map1_bytes;
    const uintptr_t y0 = reinterpret_cast<uintptr_t>(op.g.map2), y1 = y0 + op.map2_bytes;
    if ((x0 < d1 && d0 < x1) || (y0 < d1 && d0 < y1)) return fail(BEVK_ERR_ARG, "the destination range overlaps the maps");
  }
  return launch(c, op, device_batch(d_src, sis, sw, sh, srs, n, d_dst, dis, dw, dh, drs), t);
}

// cv2's borderMode and borderValue for a gather op of images of type t: the mode (BORDER_CONSTANT 0 .. BORDER_TRANSPARENT
// 5; anything else, BORDER_ISOLATED included, refused as cv2 refuses it) and the value converted to t's depth, once, here
// (make_border; NULL means zeros).  cv2 4.13 leaves remap's arithmetic in a few border cases; exactly those are refused:
// LINEAR (and AREA, read as LINEAR) under BORDER_TRANSPARENT at 32F, whose windows across the edge cv2 sums another way,
// and warpPerspective NEAREST / LINEAR at 16S under BORDER_REPLICATE and BORDER_TRANSPARENT (DESIGN.md section 2).
static int set_border(ImageOp* op, PixType t, int mode, const double* value) {
  if (mode < BORDER_CONSTANT || mode > BORDER_TRANSPARENT)
    return fail(BEVK_ERR_ARG, "border mode %d: the gathers take cv2's BORDER_CONSTANT (0) .. BORDER_TRANSPARENT (5)", mode);
  const bool linear = op->interp == BEVK_INTER_LINEAR, nearest = op->interp == BEVK_INTER_NEAREST;
  if ((t.depth == 5 && linear && mode == BORDER_TRANSPARENT) ||
      (op->mode == 2 && t.depth == 3 && (linear || nearest) && (mode == BORDER_REPLICATE || mode == BORDER_TRANSPARENT)))
    return fail(BEVK_ERR_UNSUPPORTED, "%s with interp %d at depth %d under border mode %d: cv2 computes it with another body "
                "than cv2.remap's", op->mode == 2 ? "warpPerspective" : "a gather", op->interp, t.depth, mode);
  double v[4] = {0, 0, 0, 0};
  if (value) memcpy(v, value, sizeof v);
  op->g.bd = make_border(mode, t.depth, v);
  return BEVK_OK;
}

// ---- the entry points
// Each uint8 entry point is its _typed sibling at CV_8UC(channels); the sibling reads a cv2 type code (pix_type) first,
// and is its _border sibling at BORDER_CONSTANT with a zero value.
static int remap_image(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, PixType t, const int16_t* map1,
                       const uint16_t* map2, int dw, int dh, void* dst, int64_t dstride, int interp, int border, const double* bval) {
  ImageOp op;
  RET(remap_op(map1, map2, interp, dw, dh, &op));
  RET(set_border(&op, t, border, bval));
  return host_image(c, op, src, sw, sh, sstride, t, dst, dw, dh, dstride);
}
int bevk_remap(bevk_ctx* c, const uint8_t* src, int sw, int sh, int64_t sstride, int channels, const int16_t* map1,
               const uint16_t* map2, int dw, int dh, uint8_t* dst, int64_t dstride, int interp) {
  RET(use(c));
  return remap_image(c, src, sw, sh, sstride, u8(channels), map1, map2, dw, dh, dst, dstride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_remap_typed(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, int type, const int16_t* map1,
                     const uint16_t* map2, int dw, int dh, void* dst, int64_t dstride, int interp) {
  return bevk_remap_border(c, src, sw, sh, sstride, type, map1, map2, dw, dh, dst, dstride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_remap_border(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, int type, const int16_t* map1,
                     const uint16_t* map2, int dw, int dh, void* dst, int64_t dstride, int interp, int border_mode,
                      const double border_value[4]) {
  RET(use(c));
  PixType t;
  RET(pix_type(type, &t));
  return remap_image(c, src, sw, sh, sstride, t, map1, map2, dw, dh, dst, dstride, interp, border_mode, border_value);
}

static int remap_f32_image(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, PixType t, const float* map1,
                           const float* map2, int dw, int dh, void* dst, int64_t dstride, int interp, int border, const double* bval) {
  ImageOp op;
  RET(remap_f32_op(map1, map2, interp, dw, dh, &op));
  RET(set_border(&op, t, border, bval));
  return host_image(c, op, src, sw, sh, sstride, t, dst, dw, dh, dstride);
}
int bevk_remap_f32(bevk_ctx* c, const uint8_t* src, int sw, int sh, int64_t sstride, int channels, const float* map1,
                   const float* map2, int dw, int dh, uint8_t* dst, int64_t dstride, int interp) {
  RET(use(c));
  return remap_f32_image(c, src, sw, sh, sstride, u8(channels), map1, map2, dw, dh, dst, dstride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_remap_f32_typed(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, int type, const float* map1,
                         const float* map2, int dw, int dh, void* dst, int64_t dstride, int interp) {
  return bevk_remap_f32_border(c, src, sw, sh, sstride, type, map1, map2, dw, dh, dst, dstride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_remap_f32_border(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, int type, const float* map1,
                         const float* map2, int dw, int dh, void* dst, int64_t dstride, int interp, int border_mode,
                          const double border_value[4]) {
  RET(use(c));
  PixType t;
  RET(pix_type(type, &t));
  return remap_f32_image(c, src, sw, sh, sstride, t, map1, map2, dw, dh, dst, dstride, interp, border_mode, border_value);
}

static int remap_f32_frames(bevk_ctx* c, const void* d_src, int64_t src_image_stride, int sw, int sh, int64_t src_row_stride,
                            PixType t, int n, const float* d_map1, const float* d_map2, void* d_dst, int64_t dst_image_stride,
                            int dw, int dh, int64_t dst_row_stride, int interp, int border, const double* bval) {
  ImageOp op;
  RET(remap_f32_op(d_map1, d_map2, interp, dw, dh, &op));
  RET(set_border(&op, t, border, bval));
  return device_image(c, op, d_src, src_image_stride, sw, sh, src_row_stride, t, n, d_dst, dst_image_stride, dw, dh,
                      dst_row_stride);
}
int bevk_remap_f32_stack(bevk_ctx* c, const void* d_src, int64_t src_image_stride, int sw, int sh, int64_t src_row_stride,
                         int channels, int n, const float* d_map1, const float* d_map2, void* d_dst, int64_t dst_image_stride,
                         int dw, int dh, int64_t dst_row_stride, int interp) {
  RET(use(c));
  return remap_f32_frames(c, d_src, src_image_stride, sw, sh, src_row_stride, u8(channels), n, d_map1, d_map2, d_dst,
                          dst_image_stride, dw, dh, dst_row_stride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_remap_f32_stack_typed(bevk_ctx* c, const void* d_src, int64_t src_image_stride, int sw, int sh, int64_t src_row_stride,
                               int type, int n, const float* d_map1, const float* d_map2, void* d_dst, int64_t dst_image_stride,
                               int dw, int dh, int64_t dst_row_stride, int interp) {
  return bevk_remap_f32_stack_border(c, d_src, src_image_stride, sw, sh, src_row_stride, type, n, d_map1, d_map2, d_dst,
                                     dst_image_stride, dw, dh, dst_row_stride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_remap_f32_stack_border(bevk_ctx* c, const void* d_src, int64_t src_image_stride, int sw, int sh, int64_t src_row_stride,
                               int type, int n, const float* d_map1, const float* d_map2, void* d_dst, int64_t dst_image_stride,
                               int dw, int dh, int64_t dst_row_stride, int interp, int border_mode,
                                const double border_value[4]) {
  RET(use(c));
  PixType t;
  RET(pix_type(type, &t));
  return remap_f32_frames(c, d_src, src_image_stride, sw, sh, src_row_stride, t, n, d_map1, d_map2, d_dst, dst_image_stride,
                          dw, dh, dst_row_stride, interp, border_mode, border_value);
}

// ------------------------------------------------------------------ cached-map undistortion
// A slot following maps of type m1type: CV_16SC2 + CV_16UC1 (bevk_undistorter_set_rectify), CV_32FC1 or CV_32FC2
// (bevk_undistorter_set_f32).
static int set_undistorter(bevk_ctx* c, int slot, int model, const double K[9], const double* D, int n_dist, const double* R,
                           const double P[9], int dw, int dh, int fused, int m1type) {
  RET(use(c));
  if (slot < 0 || slot >= 8) return fail(BEVK_ERR_ARG, "slot %d out of range", slot);
  Undistorter& u = c->und[slot];
  u.valid = false;
  Lens& L = u.lens;
  RET(make_model(model, K, D, n_dist, R, P, dw, dh, &L));
  u.fused = fused != 0;
  u.m1type = m1type;
  if (u.fused && L.walks && model == BEVK_MODEL_FISHEYE)
    return fail(BEVK_ERR_UNSUPPORTED, "a fused fisheye slot cannot follow cv2's running ray sums when R makes the rays depend "
                "on the row; set up a map-resident slot (fused = 0) for this camera");
  if (u.fused) {   // the gathers evaluate the model per pixel: the slot keeps its column table or its block starts
    RET(attach_xs_table(c, u.xs, &L.cm));
    if (L.walks) RET(walk_into(c, u.rays, &L));
    else u.rays.release();
  } else {         // the table (and walked rays) are read once, by the map build, from scratch
    u.xs.release();
    u.rays.release();
    RET(attach_xs_table(c, c->s_xs, &L.cm));
    RET(build_map(c, L, u.map1, u.map2, m1type));
    L.cm.xs = nullptr;
  }
  u.valid = true;
  return BEVK_OK;
}

int bevk_undistorter_set_rectify(bevk_ctx* c, int slot, int model, const double K[9], const double* D, int n_dist,
                                 const double* R, const double P[9], int dw, int dh, int fused) {
  return set_undistorter(c, slot, model, K, D, n_dist, R, P, dw, dh, fused, MAP_16SC2);
}

int bevk_undistorter_set_f32(bevk_ctx* c, int slot, int model, const double K[9], const double* D, int n_dist,
                             const double* R, const double P[9], int dw, int dh, int fused, int m1type) {
  RET(check_f32_type(model, m1type));
  return set_undistorter(c, slot, model, K, D, n_dist, R, P, dw, dh, fused, m1type);
}

int bevk_undistorter_set(bevk_ctx* c, int slot, int model, const double K[9], const double* D, int n_dist,
                         const double P[9], int dw, int dh, int fused) {
  const LegacyDist d(model, D, n_dist);
  return bevk_undistorter_set_rectify(c, slot, model, K, d.D, d.n, nullptr, P, dw, dh, fused);
}

int bevk_undistorter_maps(bevk_ctx* c, int slot, int16_t* map1, uint16_t* map2) {
  RET(use(c));
  RET(need_undistorter(c, slot));
  if (!map1 || !map2) return fail(BEVK_ERR_ARG, "null output map");
  Undistorter& u = c->und[slot];
  if (u.m1type != MAP_16SC2)
    return fail(BEVK_ERR_ARG, "undistorter slot %d follows CV_32F maps (type %d): read them with bevk_undistorter_maps_f32",
                slot, u.m1type);
  const bool resident = !u.fused;   // a fused slot has no resident map: evaluate into scratch
  if (!resident) RET(build_map(c, u.lens, c->s_m1, c->s_m2));
  return download_maps(c, resident ? u.map1.p : c->s_m1.p, resident ? u.map2.p : c->s_m2.p, (size_t)u.lens.cm.w * u.lens.cm.h,
                       map1, map2);
}

int bevk_undistorter_maps_f32(bevk_ctx* c, int slot, float* map1, float* map2) {
  RET(use(c));
  RET(need_undistorter(c, slot));
  Undistorter& u = c->und[slot];
  if (u.m1type == MAP_16SC2)
    return fail(BEVK_ERR_ARG, "undistorter slot %d follows CV_16SC2 maps: read them with bevk_undistorter_maps", slot);
  RET(check_f32_maps(u.lens.cm.model, u.m1type, map1, map2));
  const bool resident = !u.fused;
  if (!resident) RET(build_map(c, u.lens, c->s_m1, c->s_m2, u.m1type));
  return download_maps_f32(c, resident ? u.map1.p : c->s_m1.p, resident ? u.map2.p : c->s_m2.p,
                           (size_t)u.lens.cm.w * u.lens.cm.h, u.m1type, map1, map2);
}

// ------------------------------------------------------------------ cv2.convertMaps
int bevk_convert_maps(bevk_ctx* c, const void* map1, const void* map2, int m1type, int w, int h, int dstm1type,
                      int nninterpolation, void* dst1, void* dst2, int on_device) {
  RET(use(c));
  const auto known = [](int t) { return t == MAP_16SC2 || t == MAP_32FC1 || t == MAP_32FC2; };
  if (!known(m1type) || !known(dstm1type))
    return fail(BEVK_ERR_ARG, "map types %d -> %d: cv2.convertMaps converts between CV_16SC2 (%d), CV_32FC1 (%d) and "
                "CV_32FC2 (%d)", m1type, dstm1type, MAP_16SC2, MAP_32FC1, MAP_32FC2);
  if (m1type == dstm1type) return fail(BEVK_ERR_ARG, "map type %d -> %d: nothing to convert", m1type, dstm1type);
  if (w <= 0 || h <= 0) return fail(BEVK_ERR_ARG, "bad map size %dx%d", w, h);
  const bool nn = nninterpolation != 0 && dstm1type == MAP_16SC2;
  if (!map1 || (m1type == MAP_32FC1 && !map2)) return fail(BEVK_ERR_ARG, "null source map");
  if (!dst1 || ((dstm1type == MAP_32FC1 || (dstm1type == MAP_16SC2 && !nn)) && !dst2))
    return fail(BEVK_ERR_ARG, "null destination map");
  const long long n = (long long)w * h;
  size_t i1, i2, o1, o2;
  map_entry_bytes(m1type, &i1, &i2);
  map_entry_bytes(dstm1type, &o1, &o2);
  if (m1type != MAP_32FC1 && !map2) i2 = 0;   // CV_16SC2 without map2
  if (nn) o2 = 0;
  ConvertMapsArgs a{map1, i2 ? map2 : nullptr, m1type, dst1, o2 ? dst2 : nullptr, dstm1type, nn, n};
  if (!on_device) {   // host maps: through scratch, then wait
    if (c->capturing) return fail(BEVK_ERR_ARG, "host maps cannot be converted inside a graph capture");
    RET(c->s_m1.ensure(n * i1));
    if (i2) RET(c->s_m2.ensure(n * i2));
    RET(c->s_o1.ensure(n * o1));
    if (o2) RET(c->s_o2.ensure(n * o2));
    CU(cudaMemcpyAsync(c->s_m1.p, map1, n * i1, cudaMemcpyHostToDevice, c->stream));
    if (i2) CU(cudaMemcpyAsync(c->s_m2.p, map2, n * i2, cudaMemcpyHostToDevice, c->stream));
    a.in1 = c->s_m1.p; a.in2 = i2 ? c->s_m2.p : nullptr;
    a.out1 = c->s_o1.p; a.out2 = o2 ? c->s_o2.p : nullptr;
  }
  const long long blocks = std::min<long long>((n + 255) / 256, (long long)c->n_sm * 16);
  k_convert_maps<<<(unsigned)blocks, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  if (!on_device) {
    CU(cudaMemcpyAsync(dst1, c->s_o1.p, n * o1, cudaMemcpyDeviceToHost, c->stream));
    if (o2) CU(cudaMemcpyAsync(dst2, c->s_o2.p, n * o2, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
  }
  return BEVK_OK;
}

// ------------------------------------------------------------------ point functions (bevk_points.cuh)
template <int OP, int MODEL, class T>
static void launch_points(bevk_ctx* c, const PointCam& pc, const void* src, void* dst, long long n) {
  const long long blocks = std::min<long long>((n + 255) / 256, (long long)c->n_sm * 16);
  k_points<OP, MODEL, T><<<(unsigned)blocks, 256, 0, c->stream>>>(pc, (const T*)src, (T*)dst, n);
}

// One point call: checks, then host points through scratch (waits) or device points (only enqueued).  The output
// may alias the input exactly (same element count per point); any other overlap is refused.
static int points_call(bevk_ctx* c, int op, int model, const PointCam& pc, const void* src, void* dst, int64_t n, int depth,
                       int on_device) {
  if (depth != BEVK_CV_32F && depth != BEVK_CV_64F)
    return fail(BEVK_ERR_ARG, "point depth %d: BEVK_CV_32F (%d) or BEVK_CV_64F (%d)", depth, BEVK_CV_32F, BEVK_CV_64F);
  if (depth == BEVK_CV_64F && model == BEVK_MODEL_FISHEYE && op != PT_PERSPECTIVE)
    return fail(BEVK_ERR_UNSUPPORTED, "float64 fisheye points: cv2 uses glibc's tan / atan, which the device cannot "
                "reproduce to the last bit");
  if (n < 0) return fail(BEVK_ERR_ARG, "n must be >= 0, got %lld", (long long)n);
  if (n == 0) return BEVK_OK;
  if (!src || !dst) return fail(BEVK_ERR_ARG, "null points");
  const size_t es = depth == BEVK_CV_64F ? 8 : 4, in_bytes = (size_t)n * (op == PT_PROJECT ? 3 : 2) * es,
               out_bytes = (size_t)n * 2 * es;
  const char *s0 = (const char*)src, *d0 = (const char*)dst;
  const bool same = src == dst && op != PT_PROJECT;
  if (!same && s0 < d0 + out_bytes && d0 < s0 + in_bytes) return fail(BEVK_ERR_ARG, "the output overlaps the input points");
  const void* in = src;
  void* out = dst;
  if (!on_device) {
    if (c->capturing) return fail(BEVK_ERR_ARG, "host points cannot be mapped inside a graph capture");
    RET(c->s_src.ensure(in_bytes));
    RET(c->s_dst.ensure(out_bytes));
    CU(cudaMemcpyAsync(c->s_src.p, src, in_bytes, cudaMemcpyHostToDevice, c->stream));
    in = c->s_src.p;
    out = c->s_dst.p;
  }
  const bool f64 = depth == BEVK_CV_64F;
  if (op == PT_UNDISTORT && model == BEVK_MODEL_FISHEYE) launch_points<PT_UNDISTORT, 0, float>(c, pc, in, out, n);
  else if (op == PT_UNDISTORT) f64 ? launch_points<PT_UNDISTORT, 1, double>(c, pc, in, out, n)
                                   : launch_points<PT_UNDISTORT, 1, float>(c, pc, in, out, n);
  else if (op == PT_PROJECT && model == BEVK_MODEL_FISHEYE) launch_points<PT_PROJECT, 0, float>(c, pc, in, out, n);
  else if (op == PT_PROJECT) f64 ? launch_points<PT_PROJECT, 1, double>(c, pc, in, out, n)
                                 : launch_points<PT_PROJECT, 1, float>(c, pc, in, out, n);
  else if (op == PT_DISTORT) launch_points<PT_DISTORT, 0, float>(c, pc, in, out, n);
  else f64 ? launch_points<PT_PERSPECTIVE, 0, double>(c, pc, in, out, n) : launch_points<PT_PERSPECTIVE, 0, float>(c, pc, in, out, n);
  CU(cudaGetLastError());
  LAUNCHED(c);
  if (!on_device) {
    CU(cudaMemcpyAsync(dst, out, out_bytes, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
  }
  return BEVK_OK;
}

static int point_camera(int op, int model, const double* K, const double* D, int n_dist, const double* R, int n_r,
                        const double* P, const double* t, double alpha, int crit, int max_count, double eps, PointCam* pc) {
  if (model != BEVK_MODEL_FISHEYE && model != BEVK_MODEL_PINHOLE) return fail(BEVK_ERR_ARG, "bad camera model %d", model);
  if (!K) return fail(BEVK_ERR_ARG, "null K");
  if (n_dist > 0 && !D) return fail(BEVK_ERR_ARG, "null D");
  if (R && !(n_r == 9 || (n_r == 3 && model == BEVK_MODEL_FISHEYE)))
    return fail(BEVK_ERR_ARG, "R has %d entries: a 3x3 matrix (9)%s", n_r, model == BEVK_MODEL_FISHEYE ? " or an rvec (3)" : "");
  switch (points_camera(op, model, K, D, n_dist, R, n_r, P, t, alpha, crit, max_count, eps, pc)) {
    case PTS_BAD_COUNT:
      return fail(BEVK_ERR_ARG, model == BEVK_MODEL_FISHEYE ? "fisheye D has %d coefficients, cv2 takes 4 (or 0)"
                                                            : "pinhole D has %d coefficients, cv2 takes 4, 5, 8, 12 or 14 (or 0)",
                  n_dist);
    case PTS_BAD_CRITERIA:
      return fail(BEVK_ERR_UNSUPPORTED, "criteria type %d without COUNT: cv2 iterates without bound", crit);
    case PTS_TOO_MANY_ITERATIONS:
      return fail(BEVK_ERR_UNSUPPORTED, "criteria max_count %d: at most %d iterations per point", max_count,
                  MAX_POINT_ITERATIONS);
    case PTS_EPS_UNFOLLOWED:
      return fail(BEVK_ERR_UNSUPPORTED, "cv2.undistortPointsIter's EPS criterion (its reprojection-error stop) is not "
                  "followed; use COUNT");
    default: return BEVK_OK;
  }
}

int bevk_undistort_points(bevk_ctx* c, int model, const void* src, void* dst, int64_t n, int depth, const double* K,
                          const double* D, int n_dist, const double* R, int n_r, const double* P, int criteria_type,
                          int max_count, double epsilon, int on_device) {
  RET(use(c));
  PointCam pc;
  RET(point_camera(PT_UNDISTORT, model, K, D, n_dist, R, n_r, P, nullptr, 0., criteria_type, max_count, epsilon, &pc));
  return points_call(c, PT_UNDISTORT, model, pc, src, dst, n, depth, on_device);
}

int bevk_project_points(bevk_ctx* c, int model, const void* obj, void* dst, int64_t n, int depth, const double* rvec,
                        const double* tvec, const double* K, const double* D, int n_dist, double alpha, int on_device) {
  RET(use(c));
  if (!rvec || !tvec) return fail(BEVK_ERR_ARG, "null rvec / tvec");
  PointCam pc;
  RET(point_camera(PT_PROJECT, model, K, D, n_dist, nullptr, 0, nullptr, tvec, alpha, CRIT_COUNT, 0, 0., &pc));
  rodrigues(rvec, pc.RR);
  return points_call(c, PT_PROJECT, model, pc, obj, dst, n, depth, on_device);
}

int bevk_fisheye_distort_points(bevk_ctx* c, const void* src, void* dst, int64_t n, int depth, const double* K,
                                const double* D, int n_dist, double alpha, int on_device) {
  RET(use(c));
  PointCam pc;
  RET(point_camera(PT_DISTORT, BEVK_MODEL_FISHEYE, K, D, n_dist, nullptr, 0, nullptr, nullptr, alpha, CRIT_COUNT, 0, 0., &pc));
  return points_call(c, PT_DISTORT, BEVK_MODEL_FISHEYE, pc, src, dst, n, depth, on_device);
}

int bevk_perspective_transform(bevk_ctx* c, const void* src, void* dst, int64_t n, int depth, const double* M, int on_device) {
  RET(use(c));
  if (!M) return fail(BEVK_ERR_ARG, "null M");
  PointCam pc;
  memset(&pc, 0, sizeof pc);
  memcpy(pc.RR, M, sizeof pc.RR);
  return points_call(c, PT_PERSPECTIVE, BEVK_MODEL_PINHOLE, pc, src, dst, n, depth, on_device);
}

int bevk_invert3(const double* S, double* T) {
  if (!S || !T) return fail(BEVK_ERR_ARG, "null matrix");
  if (!inv3(S, T)) return fail(BEVK_ERR_ARG, "singular matrix");
  return BEVK_OK;
}

static int undistort_image(bevk_ctx* c, int slot, const void* src, int sw, int sh, int64_t sstride, PixType t, void* dst, int dw,
                           int dh, int64_t dstride, int interp, int border, const double* bval) {
  ImageOp op;
  RET(undistort_op(c, slot, interp, &op));
  RET(set_border(&op, t, border, bval));
  return host_image(c, op, src, sw, sh, sstride, t, dst, dw, dh, dstride);
}
int bevk_undistort(bevk_ctx* c, int slot, const uint8_t* src, int sw, int sh, int64_t sstride, int channels,
                   uint8_t* dst, int dw, int dh, int64_t dstride, int interp) {
  RET(use(c));
  return undistort_image(c, slot, src, sw, sh, sstride, u8(channels), dst, dw, dh, dstride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_undistort_typed(bevk_ctx* c, int slot, const void* src, int sw, int sh, int64_t sstride, int type, void* dst, int dw,
                         int dh, int64_t dstride, int interp) {
  return bevk_undistort_border(c, slot, src, sw, sh, sstride, type, dst, dw, dh, dstride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_undistort_border(bevk_ctx* c, int slot, const void* src, int sw, int sh, int64_t sstride, int type, void* dst, int dw,
                         int dh, int64_t dstride, int interp, int border_mode,
                          const double border_value[4]) {
  RET(use(c));
  PixType t;
  RET(pix_type(type, &t));
  return undistort_image(c, slot, src, sw, sh, sstride, t, dst, dw, dh, dstride, interp, border_mode, border_value);
}

// ------------------------------------------------------------------ undistortion of device frame batches
int bevk_undistort_stack(bevk_ctx* c, int slot, const void* d_src, int64_t src_image_stride, int sw, int sh, int64_t src_row_stride,
                         int channels, int n, void* d_dst, int64_t dst_image_stride, int dw, int dh, int64_t dst_row_stride,
                         int interp) {
  RET(use(c));
  // this entry point's contract: INTER_NEAREST and INTER_LINEAR, every other value refused
  if (interp != BEVK_INTER_LINEAR && interp != BEVK_INTER_NEAREST)
    return fail(BEVK_ERR_UNSUPPORTED, "interp %d: bevk_undistort_stack takes INTER_NEAREST and INTER_LINEAR, "
                "bevk_undistort_stack_interp every cv2 flag", interp);
  return bevk_undistort_stack_interp(c, slot, d_src, src_image_stride, sw, sh, src_row_stride, channels, n, d_dst,
                                     dst_image_stride, dw, dh, dst_row_stride, interp);
}

static int undistort_frames(bevk_ctx* c, int slot, const void* d_src, int64_t src_image_stride, int sw, int sh,
                            int64_t src_row_stride, PixType t, int n, void* d_dst, int64_t dst_image_stride, int dw, int dh,
                            int64_t dst_row_stride, int interp, int border, const double* bval) {
  ImageOp op;
  RET(undistort_op(c, slot, interp, &op));
  RET(set_border(&op, t, border, bval));
  return device_image(c, op, d_src, src_image_stride, sw, sh, src_row_stride, t, n, d_dst, dst_image_stride, dw, dh,
                      dst_row_stride);
}
int bevk_undistort_stack_interp(bevk_ctx* c, int slot, const void* d_src, int64_t src_image_stride, int sw, int sh,
                                int64_t src_row_stride, int channels, int n, void* d_dst, int64_t dst_image_stride, int dw, int dh,
                                int64_t dst_row_stride, int interp) {
  RET(use(c));
  return undistort_frames(c, slot, d_src, src_image_stride, sw, sh, src_row_stride, u8(channels), n, d_dst, dst_image_stride,
                          dw, dh, dst_row_stride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_undistort_stack_interp_typed(bevk_ctx* c, int slot, const void* d_src, int64_t src_image_stride, int sw, int sh,
                                      int64_t src_row_stride, int type, int n, void* d_dst, int64_t dst_image_stride, int dw,
                                      int dh, int64_t dst_row_stride, int interp) {
  return bevk_undistort_stack_interp_border(c, slot, d_src, src_image_stride, sw, sh, src_row_stride, type, n, d_dst,
                                            dst_image_stride, dw, dh, dst_row_stride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_undistort_stack_interp_border(bevk_ctx* c, int slot, const void* d_src, int64_t src_image_stride, int sw, int sh,
                                      int64_t src_row_stride, int type, int n, void* d_dst, int64_t dst_image_stride, int dw,
                                      int dh, int64_t dst_row_stride, int interp, int border_mode,
                                       const double border_value[4]) {
  RET(use(c));
  PixType t;
  RET(pix_type(type, &t));
  return undistort_frames(c, slot, d_src, src_image_stride, sw, sh, src_row_stride, t, n, d_dst, dst_image_stride, dw, dh,
                          dst_row_stride, interp, border_mode, border_value);
}

int bevk_undistort_last_path(bevk_ctx* c) { return c ? c->gather_path : 0; }

// ------------------------------------------------------------------ K4 / K2
// cv2 4.13's warpPerspective and warpAffine compute a few wider-source cases with warp-specific bodies whose pixels
// differ from cv2.remap through the same 1/32-px positions, which is what the gathers compute: warpPerspective LINEAR
// (and AREA, read as LINEAR) at 16UC3 / 16UC4 and NEAREST at 32FC1 / 32FC4; warpAffine NEAREST at 16UC4 and at 16S with
// any channel count, with or without WARP_INVERSE_MAP.  Exactly those are refused rather than given other pixels than
// cv2's; every other depth, channel count and interpolation follows remap (DESIGN.md section 2).
static int check_warp_depth(const ImageOp& op, PixType t) {
  const bool nearest = op.interp == BEVK_INTER_NEAREST, linear = op.interp == BEVK_INTER_LINEAR;
  const bool leaves = op.mode == 2 ? (t.depth == 2 && linear && t.channels != 1) || (t.depth == 5 && nearest && t.channels != 3)
                                   : nearest && (t.depth == 3 || (t.depth == 2 && t.channels == 4));
  if (leaves)
    return fail(BEVK_ERR_UNSUPPORTED, "%s with interp %d at depth %d, %d channels: cv2 computes it with another body than "
                "cv2.remap's", op.mode == 2 ? "warpPerspective" : "warpAffine", op.interp, t.depth, t.channels);
  return BEVK_OK;
}

static int perspective_image(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, PixType t, const double H[9],
                             void* dst, int dw, int dh, int64_t dstride, int interp, int border, const double* bval) {
  ImageOp op;
  RET(perspective_op(H, interp, &op));
  RET(check_warp_depth(op, t));
  RET(set_border(&op, t, border, bval));
  return host_image(c, op, src, sw, sh, sstride, t, dst, dw, dh, dstride);
}
int bevk_warp_perspective(bevk_ctx* c, const uint8_t* src, int sw, int sh, int64_t sstride, int channels,
                          const double H[9], uint8_t* dst, int dw, int dh, int64_t dstride, int interp) {
  RET(use(c));
  return perspective_image(c, src, sw, sh, sstride, u8(channels), H, dst, dw, dh, dstride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_warp_perspective_typed(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, int type, const double H[9],
                                void* dst, int dw, int dh, int64_t dstride, int interp) {
  return bevk_warp_perspective_border(c, src, sw, sh, sstride, type, H, dst, dw, dh, dstride, interp, BORDER_CONSTANT, nullptr);
}
int bevk_warp_perspective_border(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, int type, const double H[9],
                                void* dst, int dw, int dh, int64_t dstride, int interp, int border_mode,
                                 const double border_value[4]) {
  RET(use(c));
  PixType t;
  RET(pix_type(type, &t));
  return perspective_image(c, src, sw, sh, sstride, t, H, dst, dw, dh, dstride, interp, border_mode, border_value);
}

// ------------------------------------------------------------------ cv2.warpAffine
static int affine_image(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, PixType t, const double M[6], void* dst,
                        int dw, int dh, int64_t dstride, int flags, int border, const double* bval) {
  ImageOp op;
  RET(affine_op(M, flags, &op));
  RET(check_warp_depth(op, t));
  RET(set_border(&op, t, border, bval));
  return host_image(c, op, src, sw, sh, sstride, t, dst, dw, dh, dstride);
}
int bevk_warp_affine(bevk_ctx* c, const uint8_t* src, int sw, int sh, int64_t sstride, int channels, const double M[6],
                     uint8_t* dst, int dw, int dh, int64_t dstride, int flags) {
  RET(use(c));
  return affine_image(c, src, sw, sh, sstride, u8(channels), M, dst, dw, dh, dstride, flags, BORDER_CONSTANT, nullptr);
}
int bevk_warp_affine_typed(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, int type, const double M[6], void* dst,
                           int dw, int dh, int64_t dstride, int flags) {
  return bevk_warp_affine_border(c, src, sw, sh, sstride, type, M, dst, dw, dh, dstride, flags, BORDER_CONSTANT, nullptr);
}
int bevk_warp_affine_border(bevk_ctx* c, const void* src, int sw, int sh, int64_t sstride, int type, const double M[6], void* dst,
                           int dw, int dh, int64_t dstride, int flags, int border_mode,
                            const double border_value[4]) {
  RET(use(c));
  PixType t;
  RET(pix_type(type, &t));
  return affine_image(c, src, sw, sh, sstride, t, M, dst, dw, dh, dstride, flags, border_mode, border_value);
}

static int affine_frames(bevk_ctx* c, const void* d_src, int64_t src_image_stride, int sw, int sh, int64_t src_row_stride,
                         PixType t, int n, const double M[6], void* d_dst, int64_t dst_image_stride, int dw, int dh,
                         int64_t dst_row_stride, int flags, int border, const double* bval) {
  ImageOp op;
  RET(affine_op(M, flags, &op));
  RET(check_warp_depth(op, t));
  RET(set_border(&op, t, border, bval));
  return device_image(c, op, d_src, src_image_stride, sw, sh, src_row_stride, t, n, d_dst, dst_image_stride, dw, dh,
                      dst_row_stride);
}
int bevk_warp_affine_stack(bevk_ctx* c, const void* d_src, int64_t src_image_stride, int sw, int sh, int64_t src_row_stride,
                           int channels, int n, const double M[6], void* d_dst, int64_t dst_image_stride, int dw, int dh,
                           int64_t dst_row_stride, int flags) {
  RET(use(c));
  return affine_frames(c, d_src, src_image_stride, sw, sh, src_row_stride, u8(channels), n, M, d_dst, dst_image_stride, dw, dh,
                       dst_row_stride, flags, BORDER_CONSTANT, nullptr);
}
int bevk_warp_affine_stack_typed(bevk_ctx* c, const void* d_src, int64_t src_image_stride, int sw, int sh, int64_t src_row_stride,
                                 int type, int n, const double M[6], void* d_dst, int64_t dst_image_stride, int dw, int dh,
                                 int64_t dst_row_stride, int flags) {
  return bevk_warp_affine_stack_border(c, d_src, src_image_stride, sw, sh, src_row_stride, type, n, M, d_dst, dst_image_stride,
                                       dw, dh, dst_row_stride, flags, BORDER_CONSTANT, nullptr);
}
int bevk_warp_affine_stack_border(bevk_ctx* c, const void* d_src, int64_t src_image_stride, int sw, int sh, int64_t src_row_stride,
                                 int type, int n, const double M[6], void* d_dst, int64_t dst_image_stride, int dw, int dh,
                                 int64_t dst_row_stride, int flags, int border_mode,
                                  const double border_value[4]) {
  RET(use(c));
  PixType t;
  RET(pix_type(type, &t));
  return affine_frames(c, d_src, src_image_stride, sw, sh, src_row_stride, t, n, M, d_dst, dst_image_stride, dw, dh,
                       dst_row_stride, flags, border_mode, border_value);
}

// ------------------------------------------------------------------ cv2.resize
int bevk_resize(bevk_ctx* c, const uint8_t* src, int sw, int sh, int64_t sstride, int channels, uint8_t* dst, int dw, int dh,
                int64_t dstride, double fx, double fy, int interp) {
  RET(use(c));
  ImageOp op;
  RET(resize_op(sw, sh, dw, dh, fx, fy, interp, &op));
  return host_image(c, op, src, sw, sh, sstride, u8(channels), dst, dw, dh, dstride);
}

int bevk_resize_stack(bevk_ctx* c, const void* d_src, int64_t src_image_stride, int sw, int sh, int64_t src_row_stride,
                      int channels, int n, void* d_dst, int64_t dst_image_stride, int dw, int dh, int64_t dst_row_stride,
                      double fx, double fy, int interp) {
  RET(use(c));
  ImageOp op;
  RET(resize_op(sw, sh, dw, dh, fx, fy, interp, &op));
  return device_image(c, op, d_src, src_image_stride, sw, sh, src_row_stride, u8(channels), n, d_dst, dst_image_stride, dw, dh,
                      dst_row_stride);
}

int bevk_warp_maps(bevk_ctx* c, const int16_t* map1, const uint16_t* map2, int sw, int sh, const double H[9], int dw,
                   int dh, int16_t* out1, uint16_t* out2) {
  RET(use(c));
  if (!map1 || !map2 || !out1 || !out2) return fail(BEVK_ERR_ARG, "null map pointer");
  if (sw <= 0 || sh <= 0 || dw <= 0 || dh <= 0) return fail(BEVK_ERR_ARG, "bad size");
  WarpMapsArgs a{};
  RET(make_homog(H, &a.hm));
  const size_t ns = (size_t)sw * sh, nd = (size_t)dw * dh;
  RET(c->s_m1.ensure(ns * 4));
  RET(c->s_m2.ensure(ns * 2));
  RET(c->s_o1.ensure(nd * 4));
  RET(c->s_o2.ensure(nd * 2));
  CU(cudaMemcpyAsync(c->s_m1.p, map1, ns * 4, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemcpyAsync(c->s_m2.p, map2, ns * 2, cudaMemcpyHostToDevice, c->stream));
  a.in1 = c->s_m1.as<short2>(); a.in2 = c->s_m2.as<unsigned short>(); a.sw = sw; a.sh = sh;
  a.out1 = c->s_o1.as<short2>(); a.out2 = c->s_o2.as<unsigned short>(); a.dw = dw; a.dh = dh;
  k_warp_maps<0, 0><<<grid2d(dw, dh), 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  return download_maps(c, c->s_o1.p, c->s_o2.p, nd, out1, out2);
}

// ------------------------------------------------------------------ BEV engine: setup
int bevk_bev_configure(bevk_ctx* c, int n_cam, int fw, int fh, int bw, int bh) {
  RET(use(c));
  if (n_cam < 1 || n_cam > BEVK_MAX_CAMERAS) return fail(BEVK_ERR_ARG, "n_cam %d out of range", n_cam);
  if (fw <= 0 || fh <= 0 || bw <= 0 || bh <= 0) return fail(BEVK_ERR_ARG, "bad geometry");
  if (fw > 32767 || fh > 32767) return fail(BEVK_ERR_UNSUPPORTED, "frames larger than 32767 px");
  // k_bev_tma passes a tile's origin to its consumers as x | y << 16: the last tile of a 65536-px row starts at 65504
  if (bw > 65536 || bh > 65536) return fail(BEVK_ERR_UNSUPPORTED, "canvas %d x %d: wider or taller than 65536 px", bw, bh);
  if ((long long)fw * fh * 3 + 16 > 0xffffffffLL) return fail(BEVK_ERR_UNSUPPORTED, "frame too large for 32-bit offsets");
  c->n_cam = n_cam; c->FW = fw; c->FH = fh; c->BW = bw; c->BH = bh;
  c->bev_interp = BEVK_INTER_LINEAR;
  c->planned = false;
  c->tma_planned = false;
  for (auto& k : c->cam) { k.has_maps = false; k.has_mask = false; k.mask.clear(); }
  return BEVK_OK;
}

static int need_cam(bevk_ctx* c, int cam) {
  if (c->n_cam == 0) return fail(BEVK_ERR_ARG, "bevk_bev_configure not called");
  if (cam < 0 || cam >= c->n_cam) return fail(BEVK_ERR_ARG, "camera %d out of range", cam);
  return BEVK_OK;
}

static int need_plan(bevk_ctx* c) {
  return c->planned ? BEVK_OK : fail(BEVK_ERR_ARG, "bevk_bev_finalize not called");
}

int bevk_bev_set_camera_model(bevk_ctx* c, int cam, int model, const double K[9], const double* D, int n_dist,
                              const double P[9], int und_w, int und_h, const double H[9]) {
  RET(use(c));
  RET(need_cam(c, cam));
  WarpMapsArgs a{};
  Lens L;
  RET(make_model(model, K, D, n_dist, nullptr, P, und_w, und_h, &L));
  a.cm = L.cm; a.lx = L.lx;
  RET(attach_xs_table(c, c->s_xs, &a.cm));
  RET(make_homog(H, &a.hm));
  BevCam& k = c->cam[cam];
  const size_t n = (size_t)c->BW * c->BH;
  RET(k.map1.ensure(n * 4));
  RET(k.map2.ensure(n * 2));
  a.sw = und_w; a.sh = und_h;
  a.out1 = k.map1.as<short2>(); a.out2 = k.map2.as<unsigned short>(); a.dw = c->BW; a.dh = c->BH;
  if (L.full) k_warp_maps<1, 1><<<grid2d(c->BW, c->BH), 256, 0, c->stream>>>(a);
  else k_warp_maps<1, 0><<<grid2d(c->BW, c->BH), 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  k.has_maps = true;
  c->planned = false;
  return BEVK_OK;
}

int bevk_bev_set_camera(bevk_ctx* c, int cam, const double K[9], const double D[4], const double P[9], int und_w,
                        int und_h, const double H[9]) {
  return bevk_bev_set_camera_model(c, cam, BEVK_MODEL_FISHEYE, K, D, 4, P, und_w, und_h, H);
}

int bevk_bev_set_maps(bevk_ctx* c, int cam, const int16_t* map1, const uint16_t* map2) {
  RET(use(c));
  RET(need_cam(c, cam));
  if (!map1 || !map2) return fail(BEVK_ERR_ARG, "null map");
  BevCam& k = c->cam[cam];
  const size_t n = (size_t)c->BW * c->BH;
  RET(k.map1.ensure(n * 4));
  RET(k.map2.ensure(n * 2));
  CU(cudaMemcpyAsync(k.map1.p, map1, n * 4, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemcpyAsync(k.map2.p, map2, n * 2, cudaMemcpyHostToDevice, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  k.has_maps = true;
  c->planned = false;
  return BEVK_OK;
}

int bevk_bev_get_maps(bevk_ctx* c, int cam, int16_t* map1, uint16_t* map2) {
  RET(use(c));
  RET(need_cam(c, cam));
  BevCam& k = c->cam[cam];
  if (!k.has_maps) return fail(BEVK_ERR_ARG, "camera %d has no maps", cam);
  if (!map1 || !map2) return fail(BEVK_ERR_ARG, "null map");
  const size_t n = (size_t)c->BW * c->BH;
  CU(cudaMemcpyAsync(map1, k.map1.p, n * 4, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaMemcpyAsync(map2, k.map2.p, n * 2, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

int bevk_bev_set_interpolation(bevk_ctx* c, int interp) {
  RET(use(c));
  if (c->n_cam == 0) return fail(BEVK_ERR_ARG, "bevk_bev_configure not called");
  if (interp != BEVK_INTER_LINEAR && interp != BEVK_INTER_NEAREST) return fail(BEVK_ERR_UNSUPPORTED, "interp %d", interp);
  c->bev_interp = interp;
  c->planned = false;
  return BEVK_OK;
}

int bevk_bev_set_mask(bevk_ctx* c, int cam, const uint8_t* mask) {
  RET(use(c));
  RET(need_cam(c, cam));
  if (!mask) return fail(BEVK_ERR_ARG, "null mask");
  BevCam& k = c->cam[cam];
  k.mask.assign(mask, mask + (size_t)c->BW * c->BH);
  k.has_mask = true;
  c->planned = false;
  return BEVK_OK;
}

int bevk_blend_masks(bevk_ctx* c, const uint8_t* polys, const int32_t* lines, int bw, int bh, uint8_t* out) {
  RET(use(c));
  if (!polys || !lines || !out) return fail(BEVK_ERR_ARG, "null argument");
  if (bw <= 0 || bh <= 0) return fail(BEVK_ERR_ARG, "bad size");
  const size_t n = (size_t)bw * bh * 4;
  RET(c->s_src.ensure(n));
  RET(c->s_dst.ensure(n));
  CU(cudaMemcpyAsync(c->s_src.p, polys, n, cudaMemcpyHostToDevice, c->stream));
  BlendArgs a{};
  a.polys = c->s_src.as<uint8_t>(); a.out = c->s_dst.as<uint8_t>(); a.w = bw; a.h = bh;
  for (int i = 0; i < 8; ++i) for (int j = 0; j < 4; ++j) a.lines[i][j] = lines[i * 4 + j];
  k_blend_masks<<<grid2d(bw, bh), 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  CU(cudaMemcpyAsync(out, c->s_dst.p, n, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

// the instantiations of one k_bev_tma configuration: {BAL=0,NB=1}, {0,4}, {1,1}, {1,4}, and the peer-store forms of the first two
struct TmaFns { const void* fn[6]; };
static TmaFns tma_fns(int cfg) {
  int i = 0;
#define X(FS, ST, MC, EG)                                                                                              \
  if (i++ == cfg)                                                                                                      \
    return TmaFns{{(const void*)k_bev_tma<false, 1, FS, ST, MC, EG>, (const void*)k_bev_tma<false, 4, FS, ST, MC, EG>,   \
                   (const void*)k_bev_tma<true, 1, FS, ST, MC, EG>, (const void*)k_bev_tma<true, 4, FS, ST, MC, EG>,     \
                   (const void*)k_bev_tma<false, 1, FS, ST, MC, EG, true>, (const void*)k_bev_tma<false, 4, FS, ST, MC, EG, true>}};
  BEVK_TMA_CONFIGS(X)
#undef X
  return TmaFns{{nullptr, nullptr, nullptr, nullptr, nullptr, nullptr}};
}

// the instantiations of k_bev: index = 3*BAL + {NB=1:0, 4:1, 8:2}
static const void* const kBevFns[6] = {(const void*)k_bev<false, 1>, (const void*)k_bev<false, 4>, (const void*)k_bev<false, 8>,
                                       (const void*)k_bev<true, 1>, (const void*)k_bev<true, 4>, (const void*)k_bev<true, 8>};
static const int kBevNb[6] = {1, 4, 8, 1, 4, 8};

// OpenCV's 8-bit HSV division tables (color_hsv: sdiv_table / hdiv_table180, hsv_shift = 12), uploaded once per ctx
static int ensure_hsv(bevk_ctx* c) {
  if (c->d_hsv.p) return BEVK_OK;
  std::vector<int> tab(512, 0);
  for (int i = 1; i < 256; ++i) {
    tab[i] = (int)std::nearbyint((255 << 12) / (1. * i));
    tab[256 + i] = (int)std::nearbyint((180 << 12) / (6. * i));
  }
  RET(c->d_hsv.ensure(512 * sizeof(int)));
  CU(cudaMemcpyAsync(c->d_hsv.p, tab.data(), 512 * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

// Tile-plan compiler: LUT maps + masks -> per-tile item lists and thread-ordered LUT blocks.
int bevk_bev_finalize(bevk_ctx* c) {
  RET(use(c));
  if (c->n_cam == 0) return fail(BEVK_ERR_ARG, "bevk_bev_configure not called");
  const int BW = c->BW, BH = c->BH, FW = c->FW, FH = c->FH, NC = c->n_cam;
  const size_t npx = (size_t)BW * BH;
  std::vector<std::vector<short>> m1(NC);
  std::vector<std::vector<unsigned short>> m2(NC);
  for (int k = 0; k < NC; ++k) {
    if (!c->cam[k].has_maps) return fail(BEVK_ERR_ARG, "camera %d has no maps", k);
    if (!c->cam[k].has_mask) return fail(BEVK_ERR_ARG, "camera %d has no mask", k);
    m1[k].resize(npx * 2);
    m2[k].resize(npx);
    CU(cudaMemcpyAsync(m1[k].data(), c->cam[k].map1.p, npx * 4, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(m2[k].data(), c->cam[k].map2.p, npx * 2, cudaMemcpyDeviceToHost, c->stream));
  }
  CU(cudaStreamSynchronize(c->stream));
  c->nb_override = 0;
  if (const char* env = getenv("BEVK_NB")) {   // tuning override of the frame-sets per work unit: 1, 4 or 8
    const int v = atoi(env);
    if (v == 1 || v == 4 || v == 8) c->nb_override = v;
  }
  BevPlan plan;
  {
    std::vector<const short*> p1(NC);
    std::vector<const unsigned short*> p2(NC);
    std::vector<const uint8_t*> pm(NC);
    for (int k = 0; k < NC; ++k) { p1[k] = m1[k].data(); p2[k] = m2[k].data(); pm[k] = c->cam[k].mask.data(); }
    build_bev_plan(NC, FW, FH, BW, BH, c->bev_interp == BEVK_INTER_NEAREST, p1.data(), p2.data(), pm.data(), plan);
  }
  std::vector<int4>& tiles = plan.tiles;
  std::vector<BevItem>& items = plan.items;
  std::vector<uint4>& lut = plan.lut;
  std::vector<int2>& spans = plan.spans;
  c->n_tiles = (long long)tiles.size();
  c->n_items = (long long)items.size();
  RET(c->d_tiles.ensure(tiles.size() * sizeof(int4)));
  RET(c->d_items.ensure(std::max<size_t>(1, items.size()) * sizeof(BevItem)));
  RET(c->d_lut.ensure(std::max<size_t>(1, lut.size()) * sizeof(uint4)));
  CU(cudaMemcpyAsync(c->d_tiles.p, tiles.data(), tiles.size() * sizeof(int4), cudaMemcpyHostToDevice, c->stream));
  if (!items.empty()) {
    CU(cudaMemcpyAsync(c->d_items.p, items.data(), items.size() * sizeof(BevItem), cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->d_lut.p, lut.data(), lut.size() * sizeof(uint4), cudaMemcpyHostToDevice, c->stream));
  }
  RET(c->d_spans.ensure(spans.size() * sizeof(int2)));
  CU(cudaMemcpyAsync(c->d_spans.p, spans.data(), spans.size() * sizeof(int2), cudaMemcpyHostToDevice, c->stream));
  c->span_px = 0;
  for (const auto& sp : spans) c->span_px += sp.y - sp.x;
  // Host-path ingest: page-locked frames are read span by span (k_fetch_spans), pageable ones as a few DMA
  // rectangles per frame (plan_bands); BALANCE needs whole frames (its V means cover them).
  c->zero_copy_ok = true;
  if (const char* env = getenv("BEVK_ZEROCOPY")) c->zero_copy_ok = atoi(env) != 0;
  c->span_fetch_bytes = 0;
  for (const auto& sp : spans)
    if (sp.y > sp.x) c->span_fetch_bytes += std::min<int>(FW * 3, (3 * sp.y + 12 + 15) & ~15) - (std::max(0, 3 * sp.x - 12) & ~15);
  c->n_bands = 2;
  if (const char* env = getenv("BEVK_BANDS")) c->n_bands = std::max(1, std::min(BEVK_MAX_BANDS, atoi(env)));
  for (int k = 0; k < NC; ++k) plan_bands(spans.data() + (size_t)k * FH, FW, FH, c->n_bands, c->cam_box[k]);
  // YUV ingest of the same spans: 4:2:2 needs an even width, 4:2:0 an even size (other sizes: those calls are refused)
  for (int fmt = YUV_NV12; fmt <= YUV_UYVY && FW % 2 == 0; ++fmt) {
    const bool packed = fmt == YUV_YUYV || fmt == YUV_UYVY;
    if (!packed && FH % 2) continue;
    const int rows = packed ? FH : FH * 3 / 2;
    std::vector<int4> win((size_t)NC * rows);
    for (int k = 0; k < NC; ++k) {
      yuv_windows(fmt, spans.data() + (size_t)k * FH, FW, FH, win.data() + (size_t)k * rows);
      yuv_dma_rects(fmt, c->cam_box[k], c->n_bands, FW, FH, c->yuv_rects[fmt - 1][k]);
    }
    c->yuv_fetch_bytes[fmt - 1] = yuv_window_bytes(win.data(), NC * rows);
    RET(c->d_yuv_win[fmt - 1].ensure(win.size() * sizeof(int4)));
    CU(cudaMemcpyAsync(c->d_yuv_win[fmt - 1].p, win.data(), win.size() * sizeof(int4), cudaMemcpyHostToDevice, c->stream));
    CU(cudaStreamSynchronize(c->stream));   // win goes out of scope before the next format
  }
  RET(ensure_hsv(c));
  CU(cudaStreamSynchronize(c->stream));
  // ---- the TMA-staged kernel's plan (frames whose row pitch is a multiple of 16 bytes)
  c->tma_planned = false;
  c->tma_cfg = 0;
  if (const char* env = getenv("BEVK_TMA_CFG")) {   // "FS,slots,groups" of a built configuration; anything else is an error
    int fs = 0, st = 0, eg = 0, found = -1;
    if (sscanf(env, "%d,%d,%d", &fs, &st, &eg) == 3)
      for (int i = 0; i < kNumTmaConfigs; ++i)
        if (kTmaConfigs[i].fs == fs && kTmaConfigs[i].stages == st && kTmaConfigs[i].eg == eg) found = i;
    if (found < 0) return fail(BEVK_ERR_ARG, "BEVK_TMA_CFG=%s matches no built configuration (BEVK_TMA_CONFIGS)", env);
    c->tma_cfg = found;
  }
  c->tma_stage_bytes = kTmaConfigs[c->tma_cfg].fs;
  c->tma_backoff_ns = 0;
  if (const char* env = getenv("BEVK_TMA_BACKOFF")) c->tma_backoff_ns = std::max(0, atoi(env));
  {
    TmaPlan tp;
    std::vector<const short*> p1(NC);
    std::vector<const unsigned short*> p2(NC);
    std::vector<const uint8_t*> pm(NC);
    for (int k = 0; k < NC; ++k) { p1[k] = m1[k].data(); p2[k] = m2[k].data(); pm[k] = c->cam[k].mask.data(); }
    const char* env = getenv("BEVK_TMA");
    const bool want = !(env && atoi(env) == 0) && ((unsigned)FW * 3u) % 16u == 0;
    if (want) {
      const char* mm = getenv("BEVK_TMA_MAXMULT");   // tuning: largest multi-pass box (1, 2 or 4 FS); larger boxes become GATHER items
      build_tma_plan(NC, FW, FH, BW, BH, c->bev_interp == BEVK_INTER_NEAREST, p1.data(), p2.data(), pm.data(), c->tma_stage_bytes, true, tp,
                     kTmaConfigs[c->tma_cfg].eg, mm ? std::max(1, std::min(4, atoi(mm))) : 4);
      RET(c->d_ttiles.ensure(tp.tiles.size() * sizeof(int4)));
      RET(c->d_titems.ensure(std::max<size_t>(1, tp.items.size()) * sizeof(TmaItem)));
      RET(c->d_tlut.ensure(std::max<size_t>(1, tp.lut.size()) * sizeof(uint4)));
      CU(cudaMemcpyAsync(c->d_ttiles.p, tp.tiles.data(), tp.tiles.size() * sizeof(int4), cudaMemcpyHostToDevice, c->stream));
      if (!tp.items.empty()) {
        CU(cudaMemcpyAsync(c->d_titems.p, tp.items.data(), tp.items.size() * sizeof(TmaItem), cudaMemcpyHostToDevice, c->stream));
        CU(cudaMemcpyAsync(c->d_tlut.p, tp.lut.data(), tp.lut.size() * sizeof(uint4), cudaMemcpyHostToDevice, c->stream));
      }
      CU(cudaStreamSynchronize(c->stream));
      c->tma_shapes = tp.shapes;
      c->tma_items = (long long)tp.items.size(); c->tma_box_bytes = tp.box_bytes;
      c->tma_entries = tp.tma_entries; c->tma_gather_entries = tp.gather_entries;
      for (auto& m : c->maps) m.base = nullptr;   // tensor maps are per shape table
      c->tma_planned = true;
    }
  }
  if (c->tma_planned && c->tma_grid[c->tma_cfg][0] == 0) {
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, c->device));
    const TmaFns f = tma_fns(c->tma_cfg);
    const int nb[6] = {1, 4, 1, 4, 1, 4};
    for (int i = 0; i < 6; ++i) {
      int per_sm = 0;
      const size_t smem = bev_tma_smem_bytes(nb[i], kTmaConfigs[c->tma_cfg].fs, kTmaConfigs[c->tma_cfg].stages, kTmaConfigs[c->tma_cfg].eg);
      CU(cudaFuncSetAttribute(f.fn[i], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      // two CTAs of the default configuration fill the SM's shared memory to within 448 bytes: ask for the full carve-out
      CU(cudaFuncSetAttribute(f.fn[i], cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
      CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, f.fn[i], TMA_THREADS, smem));
      if (i < 4) c->tma_grid[c->tma_cfg][i] = std::max(1, per_sm) * prop.multiProcessorCount;
    }
  }
  if (c->bev_grid[0] == 0) {   // persistent grid = resident CTAs of each variant
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, c->device));
    for (int i = 0; i < 6; ++i) {
      int per_sm = 0;
      const size_t smem = bev_smem_bytes(i >= 3, kBevNb[i]);
      CU(cudaFuncSetAttribute(kBevFns[i], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kBevFns[i], 256, smem));
      c->bev_grid[i] = std::max(1, per_sm) * prop.multiProcessorCount;
    }
  }
  c->planned = true;
  c->shard.geometry = false;   // slabs follow the masks
  return BEVK_OK;
}

int bevk_bev_plan_info(bevk_ctx* c, int64_t* n_tiles, int64_t* n_items, int64_t* lut_bytes) {
  RET(use(c));
  RET(need_plan(c));
  if (n_tiles) *n_tiles = c->n_tiles;
  if (n_items) *n_items = c->n_items;
  if (lut_bytes) *lut_bytes = c->n_items * TILE * TILE * (int64_t)sizeof(uint4);
  return BEVK_OK;
}

int bevk_bev_tma_plan_info(bevk_ctx* c, int64_t* n_items, int64_t* n_shapes, int64_t* box_bytes, int64_t* tma_entries,
                           int64_t* gather_entries) {
  RET(use(c));
  RET(need_plan(c));
  const bool t = c->tma_planned;
  if (n_items) *n_items = t ? c->tma_items : 0;
  if (n_shapes) *n_shapes = t ? (int64_t)c->tma_shapes.size() : 0;
  if (box_bytes) *box_bytes = t ? c->tma_box_bytes : 0;
  if (tma_entries) *tma_entries = t ? c->tma_entries : 0;
  if (gather_entries) *gather_entries = t ? c->tma_gather_entries : 0;
  return BEVK_OK;
}

int64_t bevk_bev_last_h2d_bytes(bevk_ctx* c) { return c ? c->last_h2d_bytes : 0; }

constexpr int kInFlags = BEVK_FLAG_NV12 | BEVK_FLAG_I420 | BEVK_FLAG_YUYV | BEVK_FLAG_UYVY;
constexpr int kOutFlags = BEVK_FLAG_OUT_NV12 | BEVK_FLAG_OUT_I420;

static bool packed_format(int fmt) { return fmt == YUV_YUYV || fmt == YUV_UYVY; }

// Bytes of one dense frame of pixel format fmt (0 = BGR).
static int64_t frame_bytes_of(const bevk_ctx* c, int fmt) {
  const int64_t px = (int64_t)c->FW * c->FH;
  return !fmt ? 3 * px : packed_format(fmt) ? 2 * px : 3 * px / 2;
}

// The source and canvas formats of a call from its flags: *fmt 0 = BGR, YUV_NV12, YUV_I420, YUV_YUYV, YUV_UYVY; *ofmt
// 0 = BGR, YUV_NV12, YUV_I420.  `accepts` holds kInFlags if entry point fn reads YUV frames and kOutFlags if it writes
// YUV canvases; the others are refused rather than read a YUV buffer as BGR or write BGR where YUV was asked for.  YUV
// 4:2:0 needs an even frame or canvas size and 4:2:2 an even frame width, as cv2 does.
static int read_flags(bevk_ctx* c, int flags, int accepts, const char* fn, int* fmt, int* ofmt) {
  const int yuv = flags & kInFlags, o = flags & kOutFlags;
  *fmt = *ofmt = 0;
  if (yuv && !(accepts & kInFlags)) return fail(BEVK_ERR_UNSUPPORTED, "%s takes BGR frames only (no YUV flags)", fn);
  if (yuv & (yuv - 1)) return fail(BEVK_ERR_ARG, "the input flags BEVK_FLAG_NV12, _I420, _YUYV and _UYVY are exclusive");
  if (yuv & (BEVK_FLAG_YUYV | BEVK_FLAG_UYVY)) {
    if (c->FW & 1) return fail(BEVK_ERR_UNSUPPORTED, "YUV 4:2:2 frames need an even width, not %d", c->FW);
    *fmt = yuv == BEVK_FLAG_YUYV ? YUV_YUYV : YUV_UYVY;
  } else if (yuv) {
    if ((c->FW | c->FH) & 1) return fail(BEVK_ERR_UNSUPPORTED, "YUV 4:2:0 frames need an even size, not %d x %d", c->FW, c->FH);
    *fmt = yuv == BEVK_FLAG_NV12 ? YUV_NV12 : YUV_I420;
  }
  if (o && !(accepts & kOutFlags)) return fail(BEVK_ERR_UNSUPPORTED, "%s writes BGR canvases only (no output flags)", fn);
  if (!o) return BEVK_OK;
  if (o == kOutFlags) return fail(BEVK_ERR_ARG, "BEVK_FLAG_OUT_NV12 and BEVK_FLAG_OUT_I420 are exclusive");
  if ((c->BW | c->BH) & 1) return fail(BEVK_ERR_UNSUPPORTED, "YUV 4:2:0 canvases need an even size, not %d x %d", c->BW, c->BH);
  *ofmt = o == BEVK_FLAG_OUT_NV12 ? YUV_NV12 : YUV_I420;
  return BEVK_OK;
}

int bevk_bev_host_copy_bytes(bevk_ctx* c, int flags, int64_t* h2d, int64_t* d2h) {
  RET(use(c));
  RET(need_plan(c));
  int fmt = 0, ofmt = 0;
  RET(read_flags(c, flags, kInFlags | kOutFlags, "bevk_bev_host_copy_bytes", &fmt, &ofmt));
  int64_t up = 0;
  for (int k = 0; k < c->n_cam; ++k) {
    if (flags & BEVK_FLAG_BALANCE) { up += frame_bytes_of(c, fmt); continue; }
    if (fmt) {
      for (const int4& r : c->yuv_rects[fmt - 1][k]) up += (int64_t)r.y * r.w;
      continue;
    }
    for (int bnd = 0; bnd < c->n_bands; ++bnd)
      up += (int64_t)(c->cam_box[k][bnd][1] - c->cam_box[k][bnd][0]) * (c->cam_box[k][bnd][3] - c->cam_box[k][bnd][2]);
  }
  if (h2d) *h2d = up;
  if (d2h) *d2h = (int64_t)c->BW * c->BH * (ofmt ? 3 : 6) / 2;
  return BEVK_OK;
}

// ------------------------------------------------------------------ BEV engine: run
// The frames of a call are a Frames (bevk_device.cuh).  Stacks are what the TMA-staged kernel's 3-D tensor maps describe;
// every other kernel reads either form.

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    else
      cudaGetLastError();
  }
  return fn;
}

// Tensor maps (one per box shape of the plan) of the frame stack (base, stride, frames): uint32[frames][FH][pitch/4].
static int stack_maps(bevk_ctx* c, const uint8_t* base, long long stride, long long frames, const uint8_t** d_maps) {
  bevk_ctx::MapSet* slot = &c->maps[0];
  for (auto& m : c->maps) {
    if (m.base == base && m.stride == stride && m.frames >= frames) { m.used = ++c->map_clock; *d_maps = m.d.as<uint8_t>(); return BEVK_OK; }
    if (m.used < slot->used) slot = &m;
  }
  EncodeTiledFn enc = encode_tiled();
  if (!enc) return fail(BEVK_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled is not available from this driver");
  static_assert(sizeof(CUtensorMap) == TMA_DESC_BYTES, "tensor map size");
  const size_t n = c->tma_shapes.size();
  std::vector<CUtensorMap> maps(std::max<size_t>(1, n));
  const cuuint64_t dims[3] = {(cuuint64_t)c->FW * 3u / 4u, (cuuint64_t)c->FH, (cuuint64_t)frames};
  const cuuint64_t strides[2] = {(cuuint64_t)c->FW * 3u, (cuuint64_t)stride};
  const cuuint32_t estr[3] = {1, 1, 1};
  for (size_t i = 0; i < n; ++i) {
    const cuuint32_t box[3] = {(cuuint32_t)c->tma_shapes[i].x, (cuuint32_t)c->tma_shapes[i].y, 1};
    const CUresult r = enc(&maps[i], CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<uint8_t*>(base), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
      return fail(BEVK_ERR_CUDA, "cuTensorMapEncodeTiled(box %u x %u words, stride %lld) failed: %d", box[0], box[1], stride, (int)r);
  }
  // the slot being replaced may still be read by launches in flight on this stream: stream order protects it
  RET(slot->d.ensure(maps.size() * sizeof(CUtensorMap)));
  CU(cudaMemcpyAsync(slot->d.p, maps.data(), maps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice, c->stream));
  CU(cudaStreamSynchronize(c->stream));   // maps is a stack-lifetime staging vector
  slot->base = base; slot->stride = stride; slot->frames = frames; slot->used = ++c->map_clock;
  *d_maps = slot->d.as<uint8_t>();
  return BEVK_OK;
}

static int launch_bev_tma(bevk_ctx* c, const TmaParams& P, int nbu, bool bal) {
  const long long units = c->n_tiles * ((P.batch + nbu - 1) / nbu);
  const int variant = (bal ? 2 : 0) + (nbu == 4 ? 1 : 0);
  const TmaConfig cfg = kTmaConfigs[c->tma_cfg];
  const unsigned blocks = (unsigned)std::max<long long>(1, std::min<long long>(units, c->tma_grid[c->tma_cfg][variant]));
  const size_t smem = bev_tma_smem_bytes(nbu, cfg.fs, cfg.stages, cfg.eg);
  const bool scatter = P.world != 0;   // peer-store output: only without BALANCE (render runs windows without it)
#ifdef BEVK_TRACE
  // slot timeline (tools/gpu/trace_slots.py): the 12th launch of the process records clock64 stamps of the first 8 CTAs
  // into BEVK_TRACE_FILE; a -DBEVK_TRACE build is for this measurement only
  static unsigned long long* d_trace = nullptr;
  static int n_launch = 0;
  constexpr size_t kTraceWords = 8 * 512 * 16;
  TmaParams PT = P;
  const char* trace_file = getenv("BEVK_TRACE_FILE");
  if (trace_file) {
    if (!d_trace) CU(cudaMalloc(&d_trace, kTraceWords * 8));
    if (++n_launch == 12) { CU(cudaMemsetAsync(d_trace, 0, kTraceWords * 8, c->stream)); PT.trace = d_trace; }
  }
  void* args[] = {&PT};
#else
  void* args[] = {const_cast<TmaParams*>(&P)};
#endif
  CU(cudaLaunchKernel(tma_fns(c->tma_cfg).fn[scatter ? 4 + (nbu == 4 ? 1 : 0) : variant], dim3(blocks), dim3(TMA_THREADS), args, smem, c->stream));
  LAUNCHED(c);
#ifdef BEVK_TRACE
  if (trace_file && n_launch == 12) {
    CU(cudaStreamSynchronize(c->stream));
    std::vector<unsigned long long> h(kTraceWords);
    CU(cudaMemcpy(h.data(), d_trace, kTraceWords * 8, cudaMemcpyDeviceToHost));
    if (FILE* f = fopen(trace_file, "wb")) { fwrite(h.data(), 8, h.size(), f); fclose(f); }
  }
#endif
  return BEVK_OK;
}

// Output window of a render: the full canvas by default; camera-sharded runs render the tile-aligned bounding box of
// their cameras' masks ("slab") with its own pitch and frame-set stride.
struct OutWin {
  int pitch = 0, ox = 0, oy = 0, ox1 = 0, oy1 = 0; long long stride = 0;
  // scattered mode (peer stores): frame-set b -> peer[b % world] + src_off + (b / world) * stride
  uint8_t* peer[SHARD_MAX_RANKS] = {}; int world = 0; long long src_off = 0;
};

// k_vsum over the frames of camera range `cr` (`nr` of them): vsum[frame] += its V sum
static void launch_vsum(bevk_ctx* c, Frames srcs, CamRange cr, int nr, unsigned long long* vsum) {
  const long long frame_bytes = (long long)c->FW * 3 * c->FH;
  const int blocks = (int)std::max<long long>(1, std::min<long long>(c->n_sm * 4 / std::max(1, std::min(nr, 64)) + 1, frame_bytes / (48 * 256) + 1));
  k_vsum<<<dim3(blocks, nr), 256, 0, c->stream>>>(srcs, frame_bytes, vsum, cr);
}

// luminance_balance deltas of `batch` frame-sets into d_delta, from the V-sum blocks [world][batch][n_cam]; without
// blocks (null) from d_vsum, zeroed and then filled by vsum_kernel(d_vsum), which enqueues one kernel
template <class VsumLaunch>
static int lum_deltas(bevk_ctx* c, int batch, const unsigned long long* vsum_blocks, int world, VsumLaunch vsum_kernel) {
  const int nf = batch * c->n_cam;
  RET(c->d_delta.ensure((size_t)nf * 4));
  if (!vsum_blocks) {
    RET(c->d_vsum.ensure((size_t)nf * 8));
    CU(cudaMemsetAsync(c->d_vsum.p, 0, (size_t)nf * 8, c->stream));
    vsum_kernel(c->d_vsum.as<unsigned long long>());
    LAUNCHED(c);
    vsum_blocks = c->d_vsum.as<unsigned long long>();
    world = 1;
  }
  k_delta<<<(batch + 127) / 128, 128, 0, c->stream>>>(vsum_blocks, c->n_cam, batch, world, (double)c->FW * (double)c->FH,
                                                       c->d_delta.as<int>());
  LAUNCHED(c);
  return BEVK_OK;
}

// BALANCE pre-pass of the fused render: luminance_balance of the frames of cameras [lo, hi) of every frame-set, once
// per sampled source pixel, into balanced copies (d_bal: frame b * n_cam + cam at the 256-byte padded stride) that the
// ordinary fused gather then reads; *bal_src describes them.  The V sums come from k_vsum over those frames
// (vsum_blocks null: single GPU, where the range is every camera), or from the `world` blocks [world][batch][n_cam]
// that camera-sharded ranks filled with their own cameras' sums and exchanged.  Other cameras' copies are neither
// written nor read.  The caller checks batch * n_cam <= 65535.
static int balance_prepass(bevk_ctx* c, Frames src, int batch, int lo, int hi, const unsigned long long* vsum_blocks, int world,
                           Frames* bal_src) {
  const int nf = batch * c->n_cam, nr = batch * (hi - lo);
  const CamRange cr{lo, hi - lo, c->n_cam};
  RET(lum_deltas(c, batch, vsum_blocks, world, [&](unsigned long long* vsum) { launch_vsum(c, src, cr, nr, vsum); }));
  const size_t fpad = pad256((size_t)c->FW * 3 * c->FH);
  RET(c->d_bal.ensure(fpad * nf));
  k_lum_spans<<<dim3((c->FH + LUM_ROWS - 1) / LUM_ROWS, nr), 128, 0, c->stream>>>(src, c->d_bal.as<uint8_t>(), (long long)fpad,
                                                                                 c->d_spans.as<int2>(), cr, c->FW, c->FH,
                                                                                 c->d_delta.as<int>(), c->d_hsv.as<int>());
  LAUNCHED(c);
  *bal_src = Frames(c->d_bal.p, (long long)fpad);
  return BEVK_OK;
}

// YUV pre-pass of the fused render: the sampled spans of every frame converted to BGR (and, with BALANCE, balanced) into
// the copy stack d_bal, laid out as balance_prepass leaves it; *bgr_src describes it.  With BALANCE the V sums come from
// k_vsum_yuv over the whole converted frames first.  The caller checks batch * n_cam <= 65535.
template <int FMT>
static int yuv_prepass_fmt(bevk_ctx* c, Frames src, const YuvPlanes* planes, int batch, bool bal, Frames* bgr_src) {
  const int nf = batch * c->n_cam;
  const CamRange cr{0, c->n_cam, c->n_cam};
  const YuvPlanes in = planes ? *planes : yuv_dense_planes<FMT>(src.base, src.stride, c->FW, c->FH);
  if (bal) {
    const int blocks = std::max(1, std::min(yuv_chroma_rows_of<FMT>(c->FH), c->n_sm * 4 / std::max(1, std::min(nf, 64)) + 1));
    RET(lum_deltas(c, batch, nullptr, 1, [&](unsigned long long* vsum) {
      k_vsum_yuv<FMT><<<dim3(blocks, nf), 256, 0, c->stream>>>(in, c->FW, c->FH, vsum, cr);
    }));
  }
  const size_t fpad = pad256((size_t)c->FW * 3 * c->FH);
  RET(c->d_bal.ensure(fpad * nf));
  const dim3 grid((c->FH + LUM_ROWS - 1) / LUM_ROWS, nf);
  if (bal)
    k_yuv_spans<FMT, true><<<grid, 128, 0, c->stream>>>(in, c->d_bal.as<uint8_t>(), (long long)fpad, c->d_spans.as<int2>(), cr,
                                                        c->FW, c->FH, c->d_delta.as<int>(), c->d_hsv.as<int>());
  else
    k_yuv_spans<FMT, false><<<grid, 128, 0, c->stream>>>(in, c->d_bal.as<uint8_t>(), (long long)fpad, c->d_spans.as<int2>(), cr,
                                                         c->FW, c->FH, nullptr, nullptr);
  LAUNCHED(c);
  *bgr_src = Frames(c->d_bal.p, (long long)fpad);
  return BEVK_OK;
}

// The frames are `planes` when given, else the dense stack src (cv2's single-buffer layout).
static int yuv_prepass(bevk_ctx* c, int fmt, Frames src, const YuvPlanes* planes, int batch, bool bal, Frames* bgr_src) {
  switch (fmt) {
    case YUV_NV12: return yuv_prepass_fmt<YUV_NV12>(c, src, planes, batch, bal, bgr_src);
    case YUV_I420: return yuv_prepass_fmt<YUV_I420>(c, src, planes, batch, bal, bgr_src);
    case YUV_YUYV: return yuv_prepass_fmt<YUV_YUYV>(c, src, planes, batch, bal, bgr_src);
    default: return yuv_prepass_fmt<YUV_UYVY>(c, src, planes, batch, bal, bgr_src);
  }
}

// colour balance of `batch` full canvases from their channel sums, then the car (null: none), in place
static int launch_gain(bevk_ctx* c, uint8_t* out, int batch, const unsigned long long* csum, const uint8_t* car) {
  const long long canvas_bytes = (long long)c->BW * c->BH * 3;
  const int blocks = (int)std::max<long long>(1, std::min<long long>(canvas_bytes / (12 * 256) + 1, c->n_sm * 8 / std::max(1, std::min(batch, 64)) + 1));
  k_gain<<<dim3(blocks, batch), 256, 0, c->stream>>>(out, canvas_bytes, (double)c->BW * (double)c->BH, csum, car);
  LAUNCHED(c);
  return BEVK_OK;
}

// What every check and launch of one render reads.  The frames are `planes` when given (YUV only; src is then planes->f[0]),
// else src: a frame stack or a device table of frame pointers, and dense YUV frames come as a stack.  Without a window
// the render writes whole canvases of format ofmt to out: BGR straight there, YUV as BGR into `scratch` (dense, 4-byte
// aligned, batch canvases) and converted from there by k_canvas_yuv.  A window (a shard's slab, or peer stores, where out
// is null) renders the cameras [cam_lo, cam_hi) without car or colour balance: under BALANCE its caller has balanced
// the frames of src already, and the balance of the canvases follows the compose.
struct RenderReq {
  Frames src; const YuvPlanes* planes = nullptr; int fmt = 0;   // the source and its pixel format
  int batch = 0; bool bal = false; const void* car = nullptr;
  void* out = nullptr; int ofmt = 0;                            // the canvases and their format
  const OutWin* win = nullptr;
  int cam_lo = 0, cam_hi = BEVK_MAX_CAMERAS;
  uint8_t* scratch = nullptr;
};

// Every refusal of a render, before anything is enqueued.
static int render_check(bevk_ctx* c, const RenderReq& q) {
  RET(need_plan(c));
  if ((!q.src.table && !q.src.base) || (!q.out && !(q.win && q.win->world))) return fail(BEVK_ERR_ARG, "null device pointer");
  if (q.batch < 1 || q.batch > 65535) return fail(BEVK_ERR_ARG, "batch %d out of range [1,65535]", q.batch);
  if ((q.bal || q.fmt) && (long long)q.batch * c->n_cam > 65535)
    return fail(BEVK_ERR_ARG, "batch %d x %d cameras exceeds the 65535 frames of a BALANCE or YUV call", q.batch, c->n_cam);
  if (q.fmt && (q.win || q.cam_lo != 0 || q.cam_hi < c->n_cam)) return fail(BEVK_ERR_UNSUPPORTED, "YUV frames render whole canvases only");
  if (q.fmt && !q.planes && q.src.table) return fail(BEVK_ERR_UNSUPPORTED, "dense YUV frames come as a frame stack");
  return BEVK_OK;
}

// k_canvas_yuv over `batch` BGR canvases (dense, 4-byte aligned scratch) into `batch` YUV canvases at out (any alignment).
// csum non-null: the canvases are raw BALANCE renders with those channel sums, and colour balance and the car come first.
static int launch_canvas_yuv(bevk_ctx* c, int ofmt, const uint8_t* canvases, int batch, const unsigned long long* csum,
                             const void* d_car, void* out) {
  CanvasYuvArgs a{canvases, reinterpret_cast<uint8_t*>(out), c->BW, c->BH, csum, csum ? reinterpret_cast<const uint8_t*>(d_car) : nullptr,
                  (double)c->BW * (double)c->BH};
  const long long items = (long long)((c->BW + 3) / 4) * (c->BH / 2);
  const dim3 grid((unsigned)std::max<long long>(1, std::min<long long>(items / 256 + 1, c->n_sm * 8 / std::max(1, std::min(batch, 64)) + 1)),
                  (unsigned)batch);
  if (ofmt == YUV_NV12) {
    if (csum) k_canvas_yuv<YUV_NV12, true><<<grid, 256, 0, c->stream>>>(a);
    else k_canvas_yuv<YUV_NV12, false><<<grid, 256, 0, c->stream>>>(a);
  } else {
    if (csum) k_canvas_yuv<YUV_I420, true><<<grid, 256, 0, c->stream>>>(a);
    else k_canvas_yuv<YUV_I420, false><<<grid, 256, 0, c->stream>>>(a);
  }
  LAUNCHED(c);
  return BEVK_OK;
}

// One render that render_check passed: the BALANCE or YUV pre-pass, the fused kernel, then k_gain (BGR canvases under
// BALANCE) or k_canvas_yuv (YUV canvases, which under BALANCE applies colour balance and the car itself).  Only enqueues.
static int render(bevk_ctx* c, const RenderReq& q) {
  NvtxRange nvtx_render("bevk render (fused BEV kernels)");
  const bool bal = q.bal && !q.win;
  const int nf = q.batch * c->n_cam;
  RenderParams R{};
  R.n_cam = c->n_cam; R.FW = c->FW; R.FH = c->FH; R.pitch = (unsigned)c->FW * 3u;
  R.out = reinterpret_cast<uint8_t*>(q.ofmt ? q.scratch : q.out); R.BW = c->BW; R.BH = c->BH;
  R.canvas_bytes = (long long)c->BW * c->BH * 3;
  R.out_pitch = c->BW * 3; R.ox = 0; R.oy = 0; R.ox1 = c->BW; R.oy1 = c->BH;
  const OutWin* w = q.win;   // null: the whole canvas
  if (w) { R.canvas_bytes = w->stride; R.out_pitch = w->pitch; R.ox = w->ox; R.oy = w->oy; R.ox1 = w->ox1; R.oy1 = w->oy1; }
  R.car = reinterpret_cast<const uint8_t*>(q.car);
  R.cam_lo = q.cam_lo; R.cam_hi = q.cam_hi;
  R.n_tiles = (int)c->n_tiles; R.batch = q.batch;
  // frame-sets per work unit: 4 amortises the LUT decode over a batch; 1 for single frames
  int nbu = q.batch >= 4 ? 4 : 1;
  if (c->nb_override) nbu = c->nb_override;
  Frames gsrc = q.src;                         // what the fused gather reads
  if (bal) {
    RET(c->d_csum.ensure((size_t)q.batch * 24));
    CU(cudaMemsetAsync(c->d_csum.p, 0, (size_t)q.batch * 24, c->stream));
    if (!q.fmt) RET(balance_prepass(c, q.src, q.batch, 0, c->n_cam, nullptr, 1, &gsrc));
    R.csum = c->d_csum.as<unsigned long long>();
  }
  if (q.fmt) RET(yuv_prepass(c, q.fmt, q.src, q.planes, q.batch, bal, &gsrc));   // BGR copies of the sampled spans (balanced with BALANCE)
  // TMA-staged kernel for frame stacks (16-byte aligned base and stride); global-offset gather otherwise
  const bool use_tma = c->tma_planned && !gsrc.table && (reinterpret_cast<uintptr_t>(gsrc.base) & 15) == 0 && (gsrc.stride & 15) == 0 &&
                       gsrc.stride >= (long long)R.pitch * c->FH && (nbu == 1 || nbu == 4);
  if (use_tma) {
    TmaParams T{R};
    T.tiles = c->d_ttiles.as<int4>(); T.items = c->d_titems.as<TmaItem>(); T.lut = c->d_tlut.as<uint4>();
    RET(stack_maps(c, gsrc.base, gsrc.stride, nf, &T.maps));
    T.base = gsrc.base; T.frame_stride = gsrc.stride;
    T.backoff_ns = c->tma_backoff_ns;
    if (w && w->world) { for (int r = 0; r < SHARD_MAX_RANKS; ++r) T.peer[r] = w->peer[r]; T.world = w->world; T.src_off = w->src_off; }
    RET(c->d_unit_counter.ensure(256));
    CU(cudaMemsetAsync(c->d_unit_counter.p, 0, 4, c->stream));
    T.unit_counter = c->d_unit_counter.as<unsigned>();
    RET(launch_bev_tma(c, T, nbu, bal));
    c->last_path = 2;
  } else {
    if (w && w->world) return fail(BEVK_ERR_UNSUPPORTED, "peer-store output needs the TMA-staged kernel (a 16-byte friendly frame stack)");
    BevParams P{R};
    P.tiles = c->d_tiles.as<int4>(); P.items = c->d_items.as<BevItem>(); P.lut = c->d_lut.as<uint4>();
    P.srcs = gsrc;
    const long long units = c->n_tiles * ((q.batch + nbu - 1) / nbu);
    const int variant = (bal ? 3 : 0) + (nbu == 8 ? 2 : (nbu == 4 ? 1 : 0));
    const unsigned bev_blocks = (unsigned)std::max<long long>(1, std::min<long long>(units, c->bev_grid[variant]));
    void* args[] = {&P};
    CU(cudaLaunchKernel(kBevFns[variant], dim3(bev_blocks), dim3(256), args, bev_smem_bytes(bal, nbu), c->stream));
    LAUNCHED(c);
    c->last_path = 1;
  }
  if (q.ofmt) return launch_canvas_yuv(c, q.ofmt, q.scratch, q.batch, R.csum, q.car, q.out);
  if (bal) RET(launch_gain(c, R.out, q.batch, R.csum, R.car));
  return BEVK_OK;
}

// bevk_last_kernel_ms reads the window between ev0 and ev1 that a timed call records around its kernels (not inside a
// graph capture); c->timed says that they hold the last timed call's window, and untimed calls clear it.
static int time_begin(bevk_ctx* c) {
  if (!c->capturing) CU(cudaEventRecord(c->ev0, c->stream));
  return BEVK_OK;
}

static int time_end(bevk_ctx* c) {
  if (!c->capturing) CU(cudaEventRecord(c->ev1, c->stream));
  c->timed = true;
  return BEVK_OK;
}

// The device entry points: one checked, timed render.  YUV canvases are rendered through d_out_bgr over the whole batch.
// Rendering in chunks of 8 frame-sets, so that the conversion reads canvases still in L2, was slower: the fused kernels
// lose more on the smaller batches than the conversion gains (DESIGN.md section 4).
static int render_timed(bevk_ctx* c, RenderReq q) {
  RET(render_check(c, q));
  if (q.ofmt) {
    RET(c->d_out_bgr.ensure((size_t)c->BW * c->BH * 3 * q.batch));
    q.scratch = c->d_out_bgr.as<uint8_t>();
  }
  RET(time_begin(c));
  RET(render(c, q));
  return time_end(c);
}

// A whole-canvas render request of the entry point fn with the given flags (`accepts`: see read_flags).
static int canvas_req(bevk_ctx* c, const char* fn, int flags, int accepts, Frames src, int batch, const void* d_car, void* d_out,
                      RenderReq* q) {
  RET(read_flags(c, flags, accepts, fn, &q->fmt, &q->ofmt));
  q->src = src; q->batch = batch; q->bal = (flags & BEVK_FLAG_BALANCE) != 0; q->car = d_car; q->out = d_out;
  return BEVK_OK;
}

int bevk_bev_run_device(bevk_ctx* c, const void* d_srcs, int batch, const void* d_car, int flags, void* d_out) {
  RET(use(c));
  RenderReq q;
  RET(canvas_req(c, "bevk_bev_run_device", flags, kOutFlags, Frames(d_srcs), batch, d_car, d_out, &q));
  return render_timed(c, q);
}

// frames[i] == frames[0] + i * stride with a 16-byte friendly stride?  (a frame stack: the TMA-staged kernel applies)
static bool affine_table(const void* const* frames, size_t n, long long* stride) {
  const uintptr_t b = reinterpret_cast<uintptr_t>(frames[0]);
  if (n == 1) { *stride = 1ll << 32; return (b & 15) == 0; }   // a single frame is a stack of one
  const long long st = (long long)(reinterpret_cast<uintptr_t>(frames[1]) - b);
  if (st <= 0 || (st & 15) || (b & 15)) return false;
  for (size_t i = 2; i < n; ++i)
    if (reinterpret_cast<uintptr_t>(frames[i]) != b + (uintptr_t)st * i) return false;
  *stride = st;
  return true;
}

// The host table tab in the device buffer d, whose contents `cached` remembers: uploaded only when they change.  The
// source is pageable, so the driver stages it before returning, and stream order protects launches still reading the
// old table.  A failed upload leaves nothing cached, so that the next call uploads again.
static int upload_table(bevk_ctx* c, const void* const* tab, size_t n, DevBuf& d, std::vector<const void*>& cached, const char* what) {
  if (cached.size() == n && memcmp(cached.data(), tab, n * sizeof(void*)) == 0) return BEVK_OK;
  RET(d.ensure(n * sizeof(void*)));
  cached.assign(tab, tab + n);
  const cudaError_t e = cudaMemcpyAsync(d.p, cached.data(), n * sizeof(void*), cudaMemcpyHostToDevice, c->stream);
  if (e != cudaSuccess) {
    cached.clear();
    return fail(BEVK_ERR_CUDA, "%s upload: %s", what, cudaGetErrorString(e));
  }
  return BEVK_OK;
}

// The frames of a host table of device pointers as render reads them: a frame stack when the table describes one
// (no table upload at all), else the ctx's device copy of the table.
static int frames_src(bevk_ctx* c, const void* const* frames, int batch, Frames* src) {
  if (batch < 1) return fail(BEVK_ERR_ARG, "batch must be >= 1");
  const size_t n = (size_t)batch * c->n_cam;
  for (size_t i = 0; i < n; ++i)
    if (!frames[i] || (reinterpret_cast<uintptr_t>(frames[i]) & 3)) return fail(BEVK_ERR_ARG, "frame %zu null or not 4-byte aligned", i);
  long long stride = 0;
  if (c->tma_planned && affine_table(frames, n, &stride)) {
    *src = Frames(frames[0], stride);
    return BEVK_OK;
  }
  RET(upload_table(c, frames, n, c->d_user_ptrs, c->user_tab, "frame table"));
  *src = Frames(c->d_user_ptrs.p);
  return BEVK_OK;
}

int bevk_bev_run_frames(bevk_ctx* c, const void* const* frames, int batch, const void* d_car, int flags, void* d_out) {
  RET(use(c));
  RET(need_plan(c));
  if (!frames || !d_out) return fail(BEVK_ERR_ARG, "null pointer");
  RenderReq q;
  RET(canvas_req(c, "bevk_bev_run_frames", flags, kOutFlags, Frames(), batch, d_car, d_out, &q));
  RET(frames_src(c, frames, batch, &q.src));
  return render_timed(c, q);
}

// A frame stack of pixel format fmt.  BGR frames need 4-byte alignment; YUV frames are read byte- or word-wise by
// k_vsum_yuv / k_yuv_spans only, so any base and stride will do.
static int check_stack(bevk_ctx* c, const void* d_frames, int64_t frame_stride, int fmt = 0) {
  if (!d_frames) return fail(BEVK_ERR_ARG, "null frame stack");
  if (fmt) {
    if (frame_stride < frame_bytes_of(c, fmt))
      return fail(BEVK_ERR_ARG, "frame_stride %lld smaller than a YUV %s frame", (long long)frame_stride,
                  packed_format(fmt) ? "4:2:2" : "4:2:0");
    return BEVK_OK;
  }
  if (reinterpret_cast<uintptr_t>(d_frames) & 3) return fail(BEVK_ERR_ARG, "frame stack not 4-byte aligned");
  if (frame_stride < (int64_t)c->FW * c->FH * 3 || (frame_stride & 3)) return fail(BEVK_ERR_ARG, "frame_stride %lld smaller than a frame or not a multiple of 4", (long long)frame_stride);
  return BEVK_OK;
}

int bevk_bev_run_stack(bevk_ctx* c, const void* d_frames, int64_t frame_stride, int batch, const void* d_car, int flags, void* d_out) {
  RET(use(c));
  RenderReq q;
  RET(canvas_req(c, "bevk_bev_run_stack", flags, kInFlags | kOutFlags, Frames(d_frames, frame_stride), batch, d_car, d_out, &q));
  RET(check_stack(c, d_frames, frame_stride, q.fmt));
  return render_timed(c, q);
}

// The request of the two plane entry points, before anything is enqueued: a YUV flag and pitches that cover their
// planes' rows (plane 1 not for 4:2:2, plane 2 only for I420).
static int yuv_planes_req(bevk_ctx* c, const char* fn, const int64_t* pitch, int batch, const void* d_car, int flags, void* d_out,
                          RenderReq* q, int* n_planes) {
  RET(need_plan(c));
  RET(canvas_req(c, fn, flags, kInFlags | kOutFlags, Frames(), batch, d_car, d_out, q));
  const int fmt = q->fmt;
  if (!fmt) return fail(BEVK_ERR_ARG, "YUV planes need BEVK_FLAG_NV12, _I420, _YUYV or _UYVY");
  if (!pitch) return fail(BEVK_ERR_ARG, "null pitch array");
  *n_planes = packed_format(fmt) ? 1 : fmt == YUV_NV12 ? 2 : 3;
  const int row[3] = {packed_format(fmt) ? 2 * c->FW : c->FW, fmt == YUV_NV12 ? c->FW : c->FW / 2, c->FW / 2};
  for (int p = 0; p < *n_planes; ++p)
    if (pitch[p] < row[p]) return fail(BEVK_ERR_ARG, "pitch[%d] %lld smaller than the plane's %d-byte rows", p, (long long)pitch[p], row[p]);
  return BEVK_OK;
}

int bevk_bev_run_yuv_planes(bevk_ctx* c, const void* d_base, int64_t frame_stride, const int64_t offset[3], const int64_t pitch[3],
                            int batch, const void* d_car, int flags, void* d_out) {
  RET(use(c));
  RenderReq q;
  int np = 0;
  RET(yuv_planes_req(c, "bevk_bev_run_yuv_planes", pitch, batch, d_car, flags, d_out, &q, &np));
  if (!d_base || !offset) return fail(BEVK_ERR_ARG, "null surface pool or offset array");
  YuvPlanes planes;
  for (int p = 0; p < 3; ++p) {
    const int k = p < np ? p : np - 1;   // NV12: plane 2, 4:2:2: planes 1 and 2 are never read
    planes.f[p] = Frames(static_cast<const uint8_t*>(d_base) + offset[k], frame_stride);
    planes.pitch[p] = pitch[k];
  }
  q.src = planes.f[0]; q.planes = &planes;
  return render_timed(c, q);
}

int bevk_bev_run_yuv_surfaces(bevk_ctx* c, const void* const* surfaces, const int64_t pitch[3], int batch, const void* d_car,
                              int flags, void* d_out) {
  RET(use(c));
  RenderReq q;
  int np = 0;
  RET(yuv_planes_req(c, "bevk_bev_run_yuv_surfaces", pitch, batch, d_car, flags, d_out, &q, &np));
  if (!surfaces) return fail(BEVK_ERR_ARG, "null plane table");
  YuvPlanes planes;
  q.src = Frames(surfaces); q.planes = &planes;   // checked before the table is read; the render reads the planes
  RET(render_check(c, q));
  const size_t n = (size_t)batch * c->n_cam;
  std::vector<const void*> tab(3 * n, nullptr);   // plane-major: plane p of frame i at [p * n + i]
  for (size_t i = 0; i < n; ++i)
    for (int p = 0; p < np; ++p) {
      if (!surfaces[3 * i + p]) return fail(BEVK_ERR_ARG, "plane %d of frame %zu is null", p, i);
      tab[p * n + i] = surfaces[3 * i + p];
    }
  for (int p = np; p < 3; ++p)   // NV12: plane 2, 4:2:2: planes 1 and 2 are never read
    std::copy(tab.begin() + (np - 1) * n, tab.begin() + np * n, tab.begin() + p * n);
  RET(upload_table(c, tab.data(), tab.size(), c->d_yuv_tab, c->yuv_tab, "plane table"));
  const void* const* d_tab = c->d_yuv_tab.as<const void*>();
  for (int p = 0; p < 3; ++p) {
    planes.f[p] = Frames(d_tab + p * n);
    planes.pitch[p] = pitch[p < np ? p : np - 1];
  }
  q.src = planes.f[0];
  return render_timed(c, q);
}

// The cameras [cam_lo, cam_hi) of src into whole BGR canvases, without car or colour balance.
static int render_cams(bevk_ctx* c, Frames src, int batch, int cam_lo, int cam_hi, void* d_out) {
  if (cam_lo < 0 || cam_hi > c->n_cam || cam_lo > cam_hi) return fail(BEVK_ERR_ARG, "bad camera range [%d,%d)", cam_lo, cam_hi);
  RenderReq q;
  q.src = src; q.batch = batch; q.out = d_out; q.cam_lo = cam_lo; q.cam_hi = cam_hi;
  return render_timed(c, q);
}

int bevk_bev_run_stack_cams(bevk_ctx* c, const void* d_frames, int64_t frame_stride, int batch, int cam_lo, int cam_hi, void* d_out) {
  RET(use(c));
  RET(check_stack(c, d_frames, frame_stride));
  return render_cams(c, Frames(d_frames, frame_stride), batch, cam_lo, cam_hi, d_out);
}

int bevk_bev_last_path(bevk_ctx* c) { return c ? c->last_path : 0; }

int bevk_bev_run_device_cams(bevk_ctx* c, const void* d_srcs, int batch, int cam_lo, int cam_hi, void* d_out) {
  RET(use(c));
  return render_cams(c, Frames(d_srcs), batch, cam_lo, cam_hi, d_out);
}

int bevk_sat_sum_device(bevk_ctx* c, const void* const* parts, int n, uint64_t bytes, const void* d_car, void* d_out) {
  RET(use(c));
  if (!parts || !d_out || n < 1 || n > BEVK_MAX_CAMERAS) return fail(BEVK_ERR_ARG, "bad partial list");
  SatSumArgs a{};
  for (int i = 0; i < n; ++i) {
    if (!parts[i] || (reinterpret_cast<uintptr_t>(parts[i]) & 15)) return fail(BEVK_ERR_ARG, "partial %d null or not 16-B aligned", i);
    a.parts[i] = reinterpret_cast<const uint8_t*>(parts[i]);
  }
  if ((reinterpret_cast<uintptr_t>(d_out) & 15) || (d_car && (reinterpret_cast<uintptr_t>(d_car) & 15)))
    return fail(BEVK_ERR_ARG, "out/car not 16-B aligned");
  a.n = n; a.bytes = bytes; a.car = reinterpret_cast<const uint8_t*>(d_car); a.out = reinterpret_cast<uint8_t*>(d_out);
  const int blocks = (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)c->n_sm * 8, bytes / (16 * 256) + 1));
  k_sat_sum<<<blocks, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  return BEVK_OK;
}

// Host frames into the two halves of the ctx staging stack (d_frames), chunk by chunk on the copy stream: the state one
// call of bevk_bev_run / bevk_bev_run_to_jpeg shares between its chunks.
struct HostIngest {
  size_t row = 0, fbytes = 0, fpad = 0, cbytes = 0;
  int fmt = 0, rows = 0;                  // pixel format (0 = BGR) and buffer rows of a frame (FH; FH * 3 / 2 for 4:2:0)
  int ofmt = 0;                           // canvas format, and the bytes of one canvas in it
  size_t obytes = 0;
  int chunk = 0;
  bool zero_copy = false;
  const void* d_car = nullptr;            // the car overlay on the device, or null
  std::vector<const uint8_t*> dev_view;   // zero-copy: device views of the page-locked frames
};

// The caller's host car canvas (null: none) into d_car on the ctx stream; *d_car: the device copy, or null.
static int upload_car(bevk_ctx* c, const uint8_t* car, const void** d_car) {
  *d_car = nullptr;
  if (!car) return BEVK_OK;
  const size_t cbytes = (size_t)c->BW * c->BH * 3;
  RET(c->d_car.ensure(cbytes));
  CU(cudaMemcpyAsync(c->d_car.p, car, cbytes, cudaMemcpyHostToDevice, c->stream));
  *d_car = c->d_car.p;
  return BEVK_OK;
}

// h->fmt and h->ofmt come from read_flags.
static int ingest_setup(bevk_ctx* c, const uint8_t* const* srcs, int64_t src_stride, int batch, const uint8_t* car, int flags,
                        HostIngest* h) {
  RET(need_plan(c));
  if (!srcs) return fail(BEVK_ERR_ARG, "null host pointer");
  if (batch < 1) return fail(BEVK_ERR_ARG, "batch must be >= 1");
  const int fmt = h->fmt, ofmt = h->ofmt;
  // a YUV 4:2:0 frame is uint8[FH * 3 / 2][FW] and a 4:2:2 one uint8[FH][FW][2], rows at the same stride; it is staged as
  // it is and converted on the device
  const bool packed = packed_format(fmt);
  const int rows = fmt && !packed ? c->FH * 3 / 2 : c->FH;
  const size_t row = (size_t)c->FW * (!fmt ? 3 : packed ? 2 : 1), fbytes = row * rows, fpad = pad256(fbytes);
  if (src_stride < (int64_t)row) return fail(BEVK_ERR_ARG, "src_stride %lld < row bytes", (long long)src_stride);
  const size_t cbytes = (size_t)c->BW * c->BH * 3;
  h->row = row; h->fbytes = fbytes; h->fpad = fpad; h->cbytes = cbytes; h->rows = rows;
  h->obytes = ofmt ? cbytes / 2 : cbytes;
  // Two-deep pipeline over chunks of frame-sets: the H2D copies of chunk i+1 run on the copy
  // stream while chunk i is rendered and its canvases go back on the main stream, so the two
  // PCIe directions overlap and the kernel hides under the copies.
  int chunk = std::min(batch, 4);   // 4 frame-sets = one kernel work group; finer chunks shorten pipeline fill / drain
  if (const char* env = getenv("BEVK_CHUNK")) chunk = std::max(1, std::min(std::min(batch, 8), atoi(env)));
  h->chunk = chunk;
  const size_t set_frames = (size_t)c->n_cam;
  RET(c->d_frames.ensure(fpad * set_frames * chunk * 2));
  RET(c->d_canvas.ensure(cbytes * chunk * 2));
  if (ofmt) RET(c->d_out_yuv.ensure(h->obytes * chunk * 2));
  if (!c->copy_stream)
    RET(create_stream_set(&c->copy_stream, {&c->ev_in[0], &c->ev_in[1], &c->ev_free[0], &c->ev_free[1], &c->ev_hp[0], &c->ev_hp[1]}));
  RET(upload_car(c, car, &h->d_car));
  // the copy stream must not start before work already queued on the main stream (e.g. the car upload,
  // or a previous call's D2H that still reads the canvases) has been ordered
  CU(cudaEventRecord(c->ev_free[0], c->stream));
  CU(cudaEventRecord(c->ev_free[1], c->stream));
  // Page-locked host frames whose rows are 16-byte friendly are ingested by k_fetch_spans (the SMs read
  // only the sampled row spans over PCIe); anything else goes through DMA copies.
  bool zero_copy = !(flags & BEVK_FLAG_BALANCE) && (row % 16 == 0) && (src_stride % 16 == 0) && c->zero_copy_ok;
  h->dev_view.assign((size_t)batch * c->n_cam, nullptr);
  if (zero_copy) {
    for (size_t i = 0; i < h->dev_view.size() && zero_copy; ++i) {
      cudaPointerAttributes at{};
      if (!srcs[i] || cudaPointerGetAttributes(&at, srcs[i]) != cudaSuccess || at.type != cudaMemoryTypeHost || !at.devicePointer ||
          (reinterpret_cast<uintptr_t>(at.devicePointer) & 15)) {
        zero_copy = false;
        cudaGetLastError();   // a pageable pointer makes cudaPointerGetAttributes fail on old drivers: not an error here
      } else {
        h->dev_view[i] = static_cast<const uint8_t*>(at.devicePointer);
      }
    }
  }
  if (zero_copy) {
    RET(c->d_hptrs.ensure(sizeof(void*) * set_frames * chunk * 2));
    if (!c->h_hptrs) CU(cudaHostAlloc(reinterpret_cast<void**>(&c->h_hptrs), sizeof(void*) * BEVK_MAX_CAMERAS * 8 * 2, cudaHostAllocDefault));
  }
  h->zero_copy = zero_copy;
  c->last_h2d_bytes = 0;
  return BEVK_OK;
}

// Frame-sets [b0, b0 + nb) into staging half `half` on the copy stream, and the main stream made to wait for them.  *fsrc:
// the staged frames as render reads them (a frame stack, so the TMA-staged kernel serves them too).
static int ingest_chunk(bevk_ctx* c, const HostIngest& h, const uint8_t* const* srcs, int64_t src_stride, int flags, int b0, int nb,
                        int half, Frames* fsrc) {
  const size_t set_frames = (size_t)c->n_cam, row = h.row, fbytes = h.fbytes, fpad = h.fpad;
  const int chunk = h.chunk;
  uint8_t* dframes = c->d_frames.as<uint8_t>() + (size_t)half * chunk * set_frames * fpad;
  NvtxRange nvtx_ingest("bevk ingest (H2D / zero-copy spans)");
  CU(cudaStreamWaitEvent(c->copy_stream, c->ev_free[half], 0));   // this half's previous chunk has been rendered
  if (h.zero_copy) {
    const uint8_t** hp = c->h_hptrs + (size_t)half * chunk * set_frames;
    // the pinned pointer staging area of this half was consumed by the copy two chunks ago (ordered by ev_free + stream order)
    CU(cudaEventSynchronize(c->ev_hp[half]));
    for (int i = 0; i < nb * c->n_cam; ++i) hp[i] = h.dev_view[(size_t)b0 * c->n_cam + i];
    const uint8_t** dhp = c->d_hptrs.as<const uint8_t*>() + (size_t)half * chunk * set_frames;
    CU(cudaMemcpyAsync(dhp, hp, sizeof(void*) * nb * c->n_cam, cudaMemcpyHostToDevice, c->copy_stream));
    CU(cudaEventRecord(c->ev_hp[half], c->copy_stream));
    if (h.fmt) {
      k_fetch_yuv<<<dim3(h.rows, nb * c->n_cam), 128, 0, c->copy_stream>>>(
          dhp, dframes, (long long)fpad, c->d_yuv_win[h.fmt - 1].as<int4>(), c->n_cam, h.rows, (long long)src_stride, (int)row);
      c->last_h2d_bytes += (long long)c->yuv_fetch_bytes[h.fmt - 1] * nb;
    } else {
      k_fetch_spans<<<dim3(c->FH, nb * c->n_cam), 128, 0, c->copy_stream>>>(
          dhp, dframes, (long long)fpad, c->d_spans.as<int2>(), c->n_cam, c->FH, (long long)src_stride, (int)row);
      c->last_h2d_bytes += (long long)c->span_fetch_bytes * nb;
    }
    LAUNCHED(c);
  }
  for (int i = 0; i < nb * c->n_cam && !h.zero_copy; ++i) {
    const uint8_t* s = srcs[(size_t)b0 * c->n_cam + i];
    if (!s) return fail(BEVK_ERR_ARG, "null frame pointer %d", b0 * c->n_cam + i);
    uint8_t* d = dframes + (size_t)i * fpad;
    if (flags & BEVK_FLAG_BALANCE) {   // luminance_balance averages V over the whole raw frame: everything goes up
      if ((size_t)src_stride == row) CU(cudaMemcpyAsync(d, s, fbytes, cudaMemcpyHostToDevice, c->copy_stream));
      else CU(cudaMemcpy2DAsync(d, row, s, (size_t)src_stride, row, h.rows, cudaMemcpyHostToDevice, c->copy_stream));
      c->last_h2d_bytes += (long long)fbytes;
    } else if (h.fmt) {                // the Y rows of this camera's band boxes and their chroma rows (yuv_dma_rects)
      for (const int4& r : c->yuv_rects[h.fmt - 1][i % c->n_cam]) {
        CU(cudaMemcpy2DAsync(d + (size_t)r.x * row + r.z, row, s + (size_t)r.x * src_stride + r.z, (size_t)src_stride, (size_t)r.w,
                             (size_t)r.y, cudaMemcpyHostToDevice, c->copy_stream));
        c->last_h2d_bytes += (long long)r.y * r.w;
      }
    } else {                           // only the rectangle of the frame this camera's LUT can sample
      for (int bnd = 0; bnd < c->n_bands; ++bnd) {
        const int* bx = c->cam_box[i % c->n_cam][bnd];
        if (bx[1] > bx[0]) {
          CU(cudaMemcpy2DAsync(d + (size_t)bx[0] * row + bx[2], row, s + (size_t)bx[0] * src_stride + bx[2],
                               (size_t)src_stride, (size_t)(bx[3] - bx[2]), (size_t)(bx[1] - bx[0]), cudaMemcpyHostToDevice,
                               c->copy_stream));
          c->last_h2d_bytes += (long long)(bx[3] - bx[2]) * (bx[1] - bx[0]);
        }
      }
    }
  }
  CU(cudaEventRecord(c->ev_in[half], c->copy_stream));
  CU(cudaStreamWaitEvent(c->stream, c->ev_in[half], 0));
  *fsrc = Frames(dframes, (long long)fpad);
  return BEVK_OK;
}

// One chunk of a host-frame call: frame-sets [b0, b0 + nb) ingested into staging half `half` and rendered into canvas
// half `half` of d_canvas (*dcanvas), after which the staging half is free again.  With a YUV canvas format the BGR
// canvases in d_canvas are converted into half `half` of d_out_yuv, and *dcanvas points there.
static int render_chunk(bevk_ctx* c, const HostIngest& h, const uint8_t* const* srcs, int64_t src_stride, int flags, int b0, int nb,
                        int half, uint8_t** dcanvas) {
  RenderReq q;
  RET(ingest_chunk(c, h, srcs, src_stride, flags, b0, nb, half, &q.src));
  q.scratch = c->d_canvas.as<uint8_t>() + (size_t)half * h.chunk * h.cbytes;
  *dcanvas = h.ofmt ? c->d_out_yuv.as<uint8_t>() + (size_t)half * h.chunk * h.obytes : q.scratch;
  q.fmt = h.fmt; q.batch = nb; q.bal = (flags & BEVK_FLAG_BALANCE) != 0; q.car = h.d_car; q.out = *dcanvas; q.ofmt = h.ofmt;
  RET(render_check(c, q));
  RET(render(c, q));
  CU(cudaEventRecord(c->ev_free[half], c->stream));
  return BEVK_OK;
}

int bevk_bev_run(bevk_ctx* c, const uint8_t* const* srcs, int64_t src_stride, int batch, const uint8_t* car, int flags,
                 uint8_t* out) {
  NvtxRange nvtx_call("bevk_bev_run (host frames -> host canvases)");
  RET(use(c));
  RET(need_plan(c));
  if (!srcs || !out) return fail(BEVK_ERR_ARG, "null host pointer");
  HostIngest h;
  RET(read_flags(c, flags, kInFlags | kOutFlags, "bevk_bev_run", &h.fmt, &h.ofmt));
  RET(ingest_setup(c, srcs, src_stride, batch, car, flags, &h));
  c->timed = false;
  for (int b0 = 0, half = 0; b0 < batch; b0 += h.chunk, half ^= 1) {
    const int nb = std::min(h.chunk, batch - b0);
    uint8_t* dcanvas = nullptr;
    RET(render_chunk(c, h, srcs, src_stride, flags, b0, nb, half, &dcanvas));
    NvtxRange nvtx_d2h("bevk read-back (D2H canvases)");
    CU(cudaMemcpyAsync(out + (size_t)b0 * h.obytes, dcanvas, h.obytes * nb, cudaMemcpyDeviceToHost, c->stream));
  }
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

// ------------------------------------------------------------------ stand-alone helpers
static int stream_blocks(const bevk_ctx* c, long long n_items) {
  return (int)std::max<long long>(1, std::min<long long>(c->n_sm * 8LL, (n_items + 255) / 256));
}

int bevk_apply_mask(bevk_ctx* c, const uint8_t* img, const uint8_t* mask, int w, int h, int blend, uint8_t* out) {
  RET(use(c));
  if (!img || !mask || !out || w <= 0 || h <= 0) return fail(BEVK_ERR_ARG, "bad argument");
  const size_t npx = (size_t)w * h;
  RET(c->s_src.ensure(npx * 3));
  RET(c->s_m1.ensure(npx));
  RET(c->s_dst.ensure(npx * 3));
  CU(cudaMemcpyAsync(c->s_src.p, img, npx * 3, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemcpyAsync(c->s_m1.p, mask, npx, cudaMemcpyHostToDevice, c->stream));
  k_apply_mask<<<stream_blocks(c, npx), 256, 0, c->stream>>>(c->s_src.as<uint8_t>(), c->s_m1.as<uint8_t>(),
                                                          c->s_dst.as<uint8_t>(), (long long)npx, blend);
  LAUNCHED(c);
  CU(cudaMemcpyAsync(out, c->s_dst.p, npx * 3, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

int bevk_color_balance(bevk_ctx* c, const uint8_t* img, int w, int h, uint8_t* out) {
  RET(use(c));
  if (!img || !out || w <= 0 || h <= 0) return fail(BEVK_ERR_ARG, "bad argument");
  const size_t npx = (size_t)w * h;
  RET(c->s_dst.ensure(npx * 3));
  RET(c->d_csum.ensure(24));
  CU(cudaMemcpyAsync(c->s_dst.p, img, npx * 3, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemsetAsync(c->d_csum.p, 0, 24, c->stream));
  k_chan_sum<<<stream_blocks(c, npx), 256, 0, c->stream>>>(c->s_dst.as<uint8_t>(), (long long)npx,
                                                        c->d_csum.as<unsigned long long>());
  LAUNCHED(c);
  k_gain<<<dim3(stream_blocks(c, npx / 4 + 1), 1), 256, 0, c->stream>>>(c->s_dst.as<uint8_t>(), (long long)npx * 3, (double)npx,
                                                                   c->d_csum.as<unsigned long long>(), nullptr);
  LAUNCHED(c);
  CU(cudaMemcpyAsync(out, c->s_dst.p, npx * 3, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

int bevk_luminance_balance(bevk_ctx* c, const uint8_t* const* imgs, int n, int w, int h, uint8_t* const* outs) {
  RET(use(c));
  if (!imgs || !outs || n < 1 || n > BEVK_MAX_CAMERAS || w <= 0 || h <= 0) return fail(BEVK_ERR_ARG, "bad argument");
  RET(ensure_hsv(c));
  const size_t fbytes = (size_t)w * h * 3, fpad = pad256(fbytes);
  RET(c->s_src.ensure(fpad * n));
  RET(c->s_dst.ensure(fpad * n));
  RET(c->d_vsum.ensure(8 * n));
  RET(c->d_delta.ensure(4 * n));
  uint8_t* const d_in = c->s_src.as<uint8_t>();
  uint8_t* const d_out = c->s_dst.as<uint8_t>();
  for (int i = 0; i < n; ++i) {
    if (!imgs[i] || !outs[i]) return fail(BEVK_ERR_ARG, "null frame %d", i);
    CU(cudaMemcpyAsync(d_in + i * fpad, imgs[i], fbytes, cudaMemcpyHostToDevice, c->stream));
  }
  CU(cudaMemsetAsync(c->d_vsum.p, 0, 8 * n, c->stream));
  k_vsum<<<dim3(stream_blocks(c, fbytes / 48 + 1) / n + 1, n), 256, 0, c->stream>>>(Frames(d_in, (long long)fpad), (long long)fbytes,
                                                                                 c->d_vsum.as<unsigned long long>(), CamRange{0, n, n});
  LAUNCHED(c);
  k_delta<<<1, 32, 0, c->stream>>>(c->d_vsum.as<unsigned long long>(), n, 1, 1, (double)w * (double)h, c->d_delta.as<int>());
  LAUNCHED(c);
  k_lum_apply<<<dim3(stream_blocks(c, (long long)w * h) / n + 1, n), 256, 0, c->stream>>>(d_in, d_out, (long long)fpad, w, h,
                                                                                       c->d_delta.as<int>(), c->d_hsv.as<int>());
  LAUNCHED(c);
  for (int i = 0; i < n; ++i)
    CU(cudaMemcpyAsync(outs[i], d_out + i * fpad, fbytes, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

// ------------------------------------------------------------------ multi-GPU sharding (one process per GPU)
// NCCL is loaded at run time (dlopen): libbevk.so has no link-time dependency on it, and a process that already holds
// a libnccl.so.2 (torch's) shares it.
namespace {
struct NcclId { char b[128]; };   // ncclUniqueId (passed by value to ncclCommInitRank)
struct Nccl {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, NcclId, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool ok = false;
};
Nccl& nccl() {
  static Nccl n;
  static bool tried = false;
  if (!tried) {
    tried = true;
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
      n.lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (n.lib) break;
    }
    if (n.lib) {
      n.GetUniqueId = reinterpret_cast<decltype(n.GetUniqueId)>(dlsym(n.lib, "ncclGetUniqueId"));
      n.CommInitRank = reinterpret_cast<decltype(n.CommInitRank)>(dlsym(n.lib, "ncclCommInitRank"));
      n.CommDestroy = reinterpret_cast<decltype(n.CommDestroy)>(dlsym(n.lib, "ncclCommDestroy"));
      n.AllGather = reinterpret_cast<decltype(n.AllGather)>(dlsym(n.lib, "ncclAllGather"));
      n.GetErrorString = reinterpret_cast<decltype(n.GetErrorString)>(dlsym(n.lib, "ncclGetErrorString"));
      n.ok = n.GetUniqueId && n.CommInitRank && n.CommDestroy && n.AllGather && n.GetErrorString;
    }
  }
  return n;
}
const int kNcclUint8 = 1;   // ncclUint8 (nccl.h: ncclInt8 = 0, ncclUint8 = 1)
}  // namespace

static void shard_peers_release(bevk_ctx* c) {
  bevk_ctx::Shard& s = c->shard;
  for (int r = 0; r < SHARD_MAX_RANKS; ++r) {
    if (s.peer_recv[r] && s.peer_recv[r] != s.recv) cudaIpcCloseMemHandle(s.peer_recv[r]);
    s.peer_recv[r] = nullptr;
  }
  s.attached = false;
}

static void shard_release(bevk_ctx* c) {
  shard_peers_release(c);
  if (c->shard.recv) cudaFree(c->shard.recv);
  c->shard.recv = nullptr; c->shard.recv_bytes = 0; c->shard.prepared_batch = 0;
  c->shard.d_flag.release();
  if (c->shard.comm && nccl().ok) nccl().CommDestroy(c->shard.comm);
  c->shard.comm = nullptr;
  c->shard.d_slabs.release();
  c->shard.d_vsums.release();
}

int bevk_shard_configure(bevk_ctx* c, int policy, int rank, int world) {
  RET(use(c));
  if (policy != BEVK_SHARD_FRAMES && policy != BEVK_SHARD_CAMERAS) return fail(BEVK_ERR_ARG, "bad policy %d", policy);
  if (world < 1 || rank < 0 || rank >= world) return fail(BEVK_ERR_ARG, "rank %d outside world %d", rank, world);
  if (policy == BEVK_SHARD_CAMERAS && world > SHARD_MAX_RANKS)
    return fail(BEVK_ERR_UNSUPPORTED, "camera sharding supports up to %d ranks (there are at most %d cameras)", SHARD_MAX_RANKS, BEVK_MAX_CAMERAS);
  if (c->shard.comm && (c->shard.rank != rank || c->shard.world != world)) shard_release(c);
  c->shard.configured = true; c->shard.geometry = false;
  c->shard.policy = policy; c->shard.rank = rank; c->shard.world = world;
  return BEVK_OK;
}

static int shard_geometry(bevk_ctx* c) {
  bevk_ctx::Shard& s = c->shard;
  if (!s.configured) return fail(BEVK_ERR_ARG, "bevk_shard_configure not called");
  RET(need_plan(c));
  if (s.geometry) return BEVK_OK;
  std::vector<const uint8_t*> pm(c->n_cam);
  for (int k = 0; k < c->n_cam; ++k) pm[k] = c->cam[k].mask.data();
  s.slab_bytes = 0;
  for (int r = 0; r < s.world && r < SHARD_MAX_RANKS; ++r) {
    shard_block(c->n_cam, r, s.world, &s.cam_lo[r], &s.cam_hi[r]);
    s.rect[r] = slab_rect(pm.data(), s.cam_lo[r], s.cam_hi[r], c->BW, c->BH);
    const long long bytes = (long long)(s.rect[r].ox1 - s.rect[r].ox) * (s.rect[r].oy1 - s.rect[r].oy) * 3;
    s.slab_bytes = std::max(s.slab_bytes, bytes);
  }
  s.slab_bytes = (long long)pad256(s.slab_bytes);   // equal counts for the all-gather, 256-byte aligned slabs
  s.geometry = true;
  return BEVK_OK;
}

int bevk_shard_unique_id(void* id, int len) {
  if (!id || len < 128) return fail(BEVK_ERR_ARG, "id buffer must hold 128 bytes");
  if (!nccl().ok) return fail(BEVK_ERR_UNSUPPORTED, "NCCL (libnccl.so.2) could not be loaded: %s", dlerror() ? dlerror() : "missing symbols");
  NcclId u;
  const int r = nccl().GetUniqueId(&u);
  if (r != 0) return fail(BEVK_ERR_CUDA, "ncclGetUniqueId: %s", nccl().GetErrorString(r));
  memcpy(id, &u, 128);
  return BEVK_OK;
}

int bevk_shard_connect(bevk_ctx* c, const void* id, int len) {
  RET(use(c));
  if (!c->shard.configured) return fail(BEVK_ERR_ARG, "bevk_shard_configure not called");
  if (!id || len < 128) return fail(BEVK_ERR_ARG, "id must be the 128 bytes bevk_shard_unique_id produced on one rank");
  if (!nccl().ok) return fail(BEVK_ERR_UNSUPPORTED, "NCCL (libnccl.so.2) could not be loaded");
  if (c->shard.comm) { nccl().CommDestroy(c->shard.comm); c->shard.comm = nullptr; }
  NcclId u;
  memcpy(&u, id, 128);
  const int r = nccl().CommInitRank(&c->shard.comm, c->shard.world, u, c->shard.rank);
  if (r != 0) { c->shard.comm = nullptr; return fail(BEVK_ERR_CUDA, "ncclCommInitRank(rank %d of %d): %s", c->shard.rank, c->shard.world, nccl().GetErrorString(r)); }
  return BEVK_OK;
}

static int check_rank(bevk_ctx* c, int rank) {
  if (rank < 0 || rank >= c->shard.world || rank >= SHARD_MAX_RANKS) return fail(BEVK_ERR_ARG, "rank %d out of range", rank);
  return BEVK_OK;
}

// a device buffer the caller hands in: not null, and `align`-byte aligned
static int check_dev_buf(const void* p, int align, const char* what) {
  if (!p || (reinterpret_cast<uintptr_t>(p) & (align - 1))) return fail(BEVK_ERR_ARG, "%s null or not %d-byte aligned", what, align);
  return BEVK_OK;
}

// does rank r render anything?  (a rank without cameras, or whose cameras' masks are empty, contributes nothing)
static bool has_slab(const bevk_ctx::Shard& s, int r) { return s.rect[r].ox1 > s.rect[r].ox && s.cam_hi[r] > s.cam_lo[r]; }

// the output window of rank r's slabs: its slab rectangle, slab_bytes apart
static OutWin slab_win(const bevk_ctx::Shard& s, int r) {
  const SlabRect q = s.rect[r];
  OutWin w;
  w.pitch = (q.ox1 - q.ox) * 3; w.ox = q.ox; w.oy = q.oy; w.ox1 = q.ox1; w.oy1 = q.oy1; w.stride = s.slab_bytes;
  return w;
}

int bevk_shard_info(bevk_ctx* c, int rank, int* cam_lo, int* cam_hi, int32_t rect[4], int64_t* slab_bytes) {
  RET(use(c));
  RET(shard_geometry(c));
  RET(check_rank(c, rank));
  if (cam_lo) *cam_lo = c->shard.cam_lo[rank];
  if (cam_hi) *cam_hi = c->shard.cam_hi[rank];
  if (rect) { rect[0] = c->shard.rect[rank].ox; rect[1] = c->shard.rect[rank].oy; rect[2] = c->shard.rect[rank].ox1; rect[3] = c->shard.rect[rank].oy1; }
  if (slab_bytes) *slab_bytes = c->shard.slab_bytes;
  return BEVK_OK;
}

// The render of rank r's slabs of `batch` frame-sets into d_slabs[r][batch][slab_bytes], through *w.  Under BALANCE
// slab_prepass points q.src at the balanced copies first.
static RenderReq slab_req(bevk_ctx* c, Frames src, int batch, int r, bool bal, void* d_slabs, OutWin* w) {
  const bevk_ctx::Shard& s = c->shard;
  *w = slab_win(s, r);
  RenderReq q;
  q.src = src; q.batch = batch; q.bal = bal; q.win = w; q.cam_lo = s.cam_lo[r]; q.cam_hi = s.cam_hi[r];
  q.out = reinterpret_cast<uint8_t*>(d_slabs) + (size_t)r * batch * s.slab_bytes;
  return q;
}

// rank r's slabs; a rank without one renders nothing
static int shard_render(bevk_ctx* c, const RenderReq& q, int r) { return has_slab(c->shard, r) ? render(c, q) : BEVK_OK; }

// BALANCE of rank r's slabs: luminance balance of its own cameras from the exchanged V sums [world][batch][n_cam] into
// balanced copies, which q->src then reads
static int slab_prepass(bevk_ctx* c, RenderReq* q, int r, const unsigned long long* d_vsums) {
  const bevk_ctx::Shard& s = c->shard;
  if (!has_slab(s, r)) return BEVK_OK;
  return balance_prepass(c, q->src, q->batch, s.cam_lo[r], s.cam_hi[r], d_vsums, s.world, &q->src);
}

// bal: colour balance after the compose -- k_compose_slabs<.., true> writes the raw canvases and their channel sums,
// then k_gain applies the grey-world gains and the car, as the single-GPU BALANCE render does
static int shard_compose(bevk_ctx* c, const void* d_slabs, int batch, const void* d_car, void* d_out, long long rank_stride = 0,
                         bool bal = false) {
  bevk_ctx::Shard& s = c->shard;
  ComposeArgs a{};
  a.slabs = reinterpret_cast<const uint8_t*>(d_slabs); a.slab_bytes = s.slab_bytes; a.world = std::min(s.world, SHARD_MAX_RANKS);
  a.rank_stride = rank_stride ? rank_stride : (long long)batch * s.slab_bytes;
  a.batch = batch; a.BW = c->BW; a.BH = c->BH;
  for (int r = 0; r < a.world; ++r) a.rect[r] = s.rect[r];
  a.car = bal ? nullptr : reinterpret_cast<const uint8_t*>(d_car); a.out = reinterpret_cast<uint8_t*>(d_out);
  const bool wide = (c->BW % 8) == 0 && (reinterpret_cast<uintptr_t>(d_out) & 7) == 0 && (!a.car || (reinterpret_cast<uintptr_t>(a.car) & 7) == 0) &&
                    (reinterpret_cast<uintptr_t>(d_slabs) & 7) == 0 && (s.slab_bytes & 7) == 0 && (a.rank_stride & 7) == 0;
  if (batch > 65535 || c->BH > 65535 * COMPOSE_ROWS) return fail(BEVK_ERR_UNSUPPORTED, "compose grid too large");
  const int units = wide ? c->BW * 3 / 8 : c->BW * 3;
  const dim3 grid((units + 255) / 256, (c->BH + COMPOSE_ROWS - 1) / COMPOSE_ROWS, batch);
  if (!bal) {
    if (wide) k_compose_slabs<8><<<grid, 256, 0, c->stream>>>(a);
    else k_compose_slabs<1><<<grid, 256, 0, c->stream>>>(a);
    LAUNCHED(c);
    return BEVK_OK;
  }
  RET(c->d_csum.ensure((size_t)batch * 24));
  CU(cudaMemsetAsync(c->d_csum.p, 0, (size_t)batch * 24, c->stream));
  a.csum = c->d_csum.as<unsigned long long>();
  if (wide) k_compose_slabs<8, true><<<grid, 256, 0, c->stream>>>(a);
  else k_compose_slabs<1, true><<<grid, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  return launch_gain(c, a.out, batch, a.csum, reinterpret_cast<const uint8_t*>(d_car));
}

// the V sums of rank `as_rank`'s own cameras into block as_rank of d_vsums[world][batch][n_cam], zero in the other
// columns; other cameras' frames are never read
static int shard_vsum(bevk_ctx* c, Frames src, int batch, int as_rank, unsigned long long* d_vsums) {
  bevk_ctx::Shard& s = c->shard;
  const int lo = s.cam_lo[as_rank], hi = s.cam_hi[as_rank], nf = batch * c->n_cam;
  unsigned long long* blk = d_vsums + (size_t)as_rank * nf;
  CU(cudaMemsetAsync(blk, 0, (size_t)nf * 8, c->stream));
  if (hi <= lo) return BEVK_OK;   // a rank without cameras sends zeros
  launch_vsum(c, src, CamRange{lo, hi - lo, c->n_cam}, batch * (hi - lo), blk);
  LAUNCHED(c);
  return BEVK_OK;
}

int bevk_shard_vsum(bevk_ctx* c, const void* d_frames, int64_t frame_stride, int batch, int as_rank, uint64_t* d_vsums) {
  RET(use(c));
  RET(shard_geometry(c));
  RET(check_stack(c, d_frames, frame_stride));
  RET(check_rank(c, as_rank));
  RET(check_dev_buf(d_vsums, 8, "V-sum buffer"));
  const Frames src(d_frames, frame_stride);
  OutWin w;
  RET(render_check(c, slab_req(c, src, batch, as_rank, true, d_vsums, &w)));   // the limits of the render these sums balance
  return shard_vsum(c, src, batch, as_rank, reinterpret_cast<unsigned long long*>(d_vsums));
}

// bevk_shard_render, and with V sums bevk_shard_render_balanced, whose window starts after its balance pre-pass
static int shard_render_call(bevk_ctx* c, const void* d_frames, int64_t frame_stride, int batch, int as_rank, bool bal,
                             const uint64_t* d_vsums, void* d_slabs) {
  RET(use(c));
  RET(shard_geometry(c));
  RET(check_stack(c, d_frames, frame_stride));
  RET(check_rank(c, as_rank));
  if (bal) RET(check_dev_buf(d_vsums, 8, "V-sum buffer"));
  RET(check_dev_buf(d_slabs, 16, "slab buffer"));
  OutWin w;
  RenderReq q = slab_req(c, Frames(d_frames, frame_stride), batch, as_rank, bal, d_slabs, &w);
  RET(render_check(c, q));
  if (bal) RET(slab_prepass(c, &q, as_rank, reinterpret_cast<const unsigned long long*>(d_vsums)));
  RET(time_begin(c));
  RET(shard_render(c, q, as_rank));
  return time_end(c);
}

int bevk_shard_render_balanced(bevk_ctx* c, const void* d_frames, int64_t frame_stride, int batch, int as_rank, const uint64_t* d_vsums,
                               void* d_slabs) {
  return shard_render_call(c, d_frames, frame_stride, batch, as_rank, true, d_vsums, d_slabs);
}

int bevk_shard_compose_balanced(bevk_ctx* c, const void* d_slabs, int batch, const void* d_car, void* d_out) {
  RET(use(c));
  RET(shard_geometry(c));
  RenderReq q;   // the limits of the canvases the compose balances
  q.src = Frames(d_slabs, 0); q.batch = batch; q.bal = true; q.car = d_car; q.out = d_out;
  RET(render_check(c, q));
  return shard_compose(c, d_slabs, batch, d_car, d_out, 0, true);
}

int bevk_shard_render(bevk_ctx* c, const void* d_frames, int64_t frame_stride, int batch, int as_rank, void* d_slabs) {
  return shard_render_call(c, d_frames, frame_stride, batch, as_rank, false, nullptr, d_slabs);
}

int bevk_shard_compose(bevk_ctx* c, const void* d_slabs, int batch, const void* d_car, void* d_out) {
  RET(use(c));
  RET(shard_geometry(c));
  if (!d_slabs || !d_out || batch < 1) return fail(BEVK_ERR_ARG, "bad argument");
  return shard_compose(c, d_slabs, batch, d_car, d_out);
}

// this rank's V sums into its block of s.d_vsums, then one in-place all-gather of the blocks (none in a world of one);
// *received: the bytes that came from the other ranks
static int shard_exchange_vsums(bevk_ctx* c, Frames src, int batch, long long* received) {
  bevk_ctx::Shard& s = c->shard;
  const size_t blk = (size_t)batch * c->n_cam * 8;
  RET(s.d_vsums.ensure(blk * s.world));
  RET(shard_vsum(c, src, batch, s.rank, s.d_vsums.as<unsigned long long>()));
  *received = 0;
  if (s.world == 1) return BEVK_OK;
  const int r = nccl().AllGather(s.d_vsums.as<uint8_t>() + blk * s.rank, s.d_vsums.p, blk, kNcclUint8, s.comm, c->stream);
  if (r != 0) return fail(BEVK_ERR_CUDA, "ncclAllGather (V sums): %s", nccl().GetErrorString(r));
  *received = (long long)blk * (s.world - 1);
  return BEVK_OK;
}

int bevk_bev_run_sharded(bevk_ctx* c, const void* d_frames, int64_t frame_stride, int batch, const void* d_car, int flags, void* d_out) {
  NvtxRange nvtx_call("bevk_bev_run_sharded (render slabs, all-gather, compose)");
  RET(use(c));
  RenderReq q;
  RET(canvas_req(c, "bevk_bev_run_sharded", flags, 0, Frames(d_frames, frame_stride), batch, d_car, d_out, &q));
  if (!c->shard.configured) return fail(BEVK_ERR_ARG, "bevk_shard_configure not called");
  RET(check_stack(c, d_frames, frame_stride));
  bevk_ctx::Shard& s = c->shard;
  s.last_link_bytes = 0;
  if (s.policy == BEVK_SHARD_FRAMES || s.world == 1) return render_timed(c, q);   // every rank renders its own frame-sets
  RET(render_check(c, q));   // the canvases the compose writes
  if (!s.comm) return fail(BEVK_ERR_ARG, "bevk_shard_connect not called");
  RET(shard_geometry(c));
  const size_t per_rank = (size_t)batch * s.slab_bytes;
  RET(s.d_slabs.ensure(per_rank * s.world));
  c->timed = false;
  OutWin w;
  RenderReq sq = slab_req(c, q.src, batch, s.rank, q.bal, s.d_slabs.p, &w);
  long long vsum_bytes = 0;
  if (q.bal) {
    // luminance_balance needs every camera's V mean: ONE all-gather of the ranks' V-sum blocks before the render
    RET(shard_exchange_vsums(c, q.src, batch, &vsum_bytes));
    RET(slab_prepass(c, &sq, s.rank, s.d_vsums.as<unsigned long long>()));
  }
  RET(shard_render(c, sq, s.rank));
  // ONE all-gather of the slabs (in place: this rank's block is already where it belongs)
  const int r = nccl().AllGather(s.d_slabs.as<uint8_t>() + per_rank * s.rank, s.d_slabs.p, per_rank, kNcclUint8, s.comm, c->stream);
  if (r != 0) return fail(BEVK_ERR_CUDA, "ncclAllGather: %s", nccl().GetErrorString(r));
  s.last_link_bytes = (long long)per_rank * (s.world - 1) + vsum_bytes;
  return shard_compose(c, s.d_slabs.p, batch, d_car, d_out, 0, q.bal);
}

// ---- camera sharding with peer stores: compute and exchange in one kernel ----------------------------------------
// Frame-set b of the batch is OWNED by rank b % world, which ends up with its canvas.  Every rank renders its cameras'
// slabs of ALL frame-sets, and the fused kernel's write-out stores each slab straight into the owner's receive buffer
// over NVLink (CUDA IPC mapping) -- no send buffer, no separate collective; one 4-byte all-gather per step is the
// barrier that tells an owner its slabs have landed, then it composes its own canvases.  Each rank sends and receives
// (world-1)/world of ONE slab set instead of receiving world-1 whole ones as the all-gather form does.
static int own_count(int batch, int rank, int world) { return (batch - rank + world - 1) / world; }

int bevk_shard_prepare(bevk_ctx* c, int batch, void* handle64) {
  RET(use(c));
  RET(shard_geometry(c));
  bevk_ctx::Shard& s = c->shard;
  if (s.policy != BEVK_SHARD_CAMERAS) return fail(BEVK_ERR_ARG, "peer stores belong to the CAMERAS policy");
  if (batch < 1 || !handle64) return fail(BEVK_ERR_ARG, "bad argument");
  CU(cudaStreamSynchronize(c->stream));
  shard_peers_release(c);
  s.own_max = (batch + s.world - 1) / s.world;
  const size_t need = 2 * (size_t)s.world * s.own_max * s.slab_bytes;
  if (need > s.recv_bytes) {   // plain cudaMalloc: IPC handles cannot be taken from pool / async allocations
    if (s.recv) cudaFree(s.recv);
    s.recv = nullptr; s.recv_bytes = 0;
    CU(cudaMalloc(&s.recv, need));
    s.recv_bytes = need;
  }
  CU(cudaMemsetAsync(s.recv, 0, s.recv_bytes, c->stream));   // slabs of ranks without cameras are never written: keep them zero
  CU(cudaStreamSynchronize(c->stream));
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, s.recv));
  static_assert(sizeof h == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle64, &h, 64);
  s.prepared_batch = batch;
  RET(s.d_flag.ensure(sizeof(int) * (SHARD_MAX_RANKS + 1)));
  return BEVK_OK;
}

int bevk_shard_attach(bevk_ctx* c, const void* handles) {
  RET(use(c));
  bevk_ctx::Shard& s = c->shard;
  if (!s.prepared_batch || !handles) return fail(BEVK_ERR_ARG, "bevk_shard_prepare not called");
  shard_peers_release(c);
  for (int r = 0; r < s.world && r < SHARD_MAX_RANKS; ++r) {
    if (r == s.rank) { s.peer_recv[r] = s.recv; continue; }
    cudaIpcMemHandle_t h;
    memcpy(&h, reinterpret_cast<const uint8_t*>(handles) + 64 * r, 64);
    const cudaError_t e = cudaIpcOpenMemHandle(&s.peer_recv[r], h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) { s.peer_recv[r] = nullptr; shard_peers_release(c); return fail(BEVK_ERR_CUDA, "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(e)); }
  }
  s.attached = true;
  return BEVK_OK;
}

int bevk_bev_run_scattered(bevk_ctx* c, const void* d_frames, int64_t frame_stride, int batch, const void* d_car, int flags,
                           void* d_out_own, int* n_own) {
  NvtxRange nvtx_call("bevk_bev_run_scattered (render with peer stores, barrier, compose own)");
  RET(use(c));
  RenderReq q;
  RET(canvas_req(c, "bevk_bev_run_scattered", flags, 0, Frames(d_frames, frame_stride), batch, d_car, d_out_own, &q));
  bevk_ctx::Shard& s = c->shard;
  if (!s.configured || s.policy != BEVK_SHARD_CAMERAS) return fail(BEVK_ERR_ARG, "bevk_shard_configure(CAMERAS) not called");
  RET(check_stack(c, d_frames, frame_stride));
  RET(shard_geometry(c));
  if (!s.comm && s.world > 1) return fail(BEVK_ERR_ARG, "bevk_shard_connect not called");
  if (!s.attached || batch > s.prepared_batch || (batch + s.world - 1) / s.world != s.own_max)
    return fail(BEVK_ERR_ARG, "bevk_shard_prepare / bevk_shard_attach not called for a batch of %d", batch);
  const int mine = own_count(batch, s.rank, s.world);
  if (n_own) *n_own = mine;
  if (mine > 0 && !d_out_own) return fail(BEVK_ERR_ARG, "null output");
  const size_t half = (size_t)s.world * s.own_max * s.slab_bytes, rank_stride = (size_t)s.own_max * s.slab_bytes;
  const unsigned par = s.step & 1u;     // double buffer: a peer may already store step n+1 while this rank composes step n
  OutWin w;
  RenderReq sq = slab_req(c, q.src, batch, s.rank, q.bal, nullptr, &w);
  sq.out = nullptr;
  w.world = s.world; w.src_off = (long long)(par * half + (size_t)s.rank * rank_stride);
  for (int r = 0; r < s.world; ++r) w.peer[r] = reinterpret_cast<uint8_t*>(s.peer_recv[r]);
  RET(render_check(c, sq));
  s.step++;
  s.last_link_bytes = 0;
  c->timed = false;
  long long vsum_bytes = 0;
  if (q.bal) RET(shard_exchange_vsums(c, q.src, batch, &vsum_bytes));
  if (has_slab(s, s.rank)) {
    if (q.bal) RET(slab_prepass(c, &sq, s.rank, s.d_vsums.as<unsigned long long>()));   // the peer-store render reads them
    RET(render(c, sq));
    s.last_link_bytes = (long long)(batch - mine) * s.slab_bytes;   // what this rank stored into its peers
  }
  s.last_link_bytes += vsum_bytes;
  if (s.world > 1) {   // the step barrier: every rank's stores are complete (its kernel has finished) when this returns on the stream
    int* f = s.d_flag.as<int>();
    const int r = nccl().AllGather(f + SHARD_MAX_RANKS, f, 4, kNcclUint8, s.comm, c->stream);
    if (r != 0) return fail(BEVK_ERR_CUDA, "ncclAllGather (step barrier): %s", nccl().GetErrorString(r));
  }
  if (mine > 0) RET(shard_compose(c, reinterpret_cast<const uint8_t*>(s.recv) + par * half, mine, d_car, d_out_own, (long long)rank_stride, q.bal));
  return BEVK_OK;
}

int64_t bevk_shard_last_link_bytes(bevk_ctx* c) { return c ? c->shard.last_link_bytes : 0; }

// ------------------------------------------------------------------ JPEG ingest on the device (nvJPEG, dlopen'ed)
// The reference reads its frames with cv2.imread (SurroundBirdEyeView/surroundBEV.py:328-332, Tools/undistort.py:65):
// decode on the host, then -- here -- 3 bytes per pixel over PCIe.  bevk_jpeg_decode ships the compressed stream
// instead and decodes it straight into the frame stack the BEV / undistort entry points read.
namespace {
struct NvjpegImage { unsigned char* channel[4]; size_t pitch[4]; };
struct Nvjpeg {
  void* lib = nullptr;
  int (*CreateSimple)(void**) = nullptr;
  int (*Destroy)(void*) = nullptr;
  int (*StateCreate)(void*, void**) = nullptr;
  int (*StateDestroy)(void*) = nullptr;
  int (*GetImageInfo)(void*, const unsigned char*, size_t, int*, int*, int*, int*) = nullptr;
  int (*Decode)(void*, void*, const unsigned char*, size_t, int, NvjpegImage*, cudaStream_t) = nullptr;
  bool ok = false;
};
Nvjpeg& nvjpeg() {
  static Nvjpeg n;
  static bool tried = false;
  if (!tried) {
    tried = true;
    for (const char* name : {"libnvjpeg.so.12", "libnvjpeg.so", "/usr/local/cuda/lib64/libnvjpeg.so.12"}) {
      n.lib = dlopen(name, RTLD_NOW | RTLD_LOCAL);
      if (n.lib) break;
    }
    if (n.lib) {
      n.CreateSimple = reinterpret_cast<decltype(n.CreateSimple)>(dlsym(n.lib, "nvjpegCreateSimple"));
      n.Destroy = reinterpret_cast<decltype(n.Destroy)>(dlsym(n.lib, "nvjpegDestroy"));
      n.StateCreate = reinterpret_cast<decltype(n.StateCreate)>(dlsym(n.lib, "nvjpegJpegStateCreate"));
      n.StateDestroy = reinterpret_cast<decltype(n.StateDestroy)>(dlsym(n.lib, "nvjpegJpegStateDestroy"));
      n.GetImageInfo = reinterpret_cast<decltype(n.GetImageInfo)>(dlsym(n.lib, "nvjpegGetImageInfo"));
      n.Decode = reinterpret_cast<decltype(n.Decode)>(dlsym(n.lib, "nvjpegDecode"));
      n.ok = n.CreateSimple && n.Destroy && n.StateCreate && n.StateDestroy && n.GetImageInfo && n.Decode;
    }
  }
  return n;
}
const int kNvjpegOutputBGRI = 6;   // NVJPEG_OUTPUT_BGRI: interleaved BGR in channel[0], what cv2.imread's layout is
}  // namespace

static void jpeg_release(bevk_ctx* c) {
  if (c->jpeg_state && nvjpeg().ok) nvjpeg().StateDestroy(c->jpeg_state);
  if (c->jpeg_handle && nvjpeg().ok) nvjpeg().Destroy(c->jpeg_handle);
  c->jpeg_state = c->jpeg_handle = nullptr;
}

int bevk_jpeg_decode(bevk_ctx* c, const uint8_t* const* jpegs, const uint64_t* sizes, int n, int width, int height, void* d_frames,
                     int64_t frame_stride) {
  NvtxRange nvtx_call("bevk_jpeg_decode (nvJPEG -> frame stack)");
  RET(use(c));
  if (!jpegs || !sizes || !d_frames || n < 1) return fail(BEVK_ERR_ARG, "bad argument");
  if (width <= 0 || height <= 0 || frame_stride < (int64_t)width * height * 3) return fail(BEVK_ERR_ARG, "bad frame geometry / stride");
  if (!nvjpeg().ok) return fail(BEVK_ERR_UNSUPPORTED, "nvJPEG (libnvjpeg.so.12) could not be loaded");
  if (!c->jpeg_handle) {
    int r = nvjpeg().CreateSimple(&c->jpeg_handle);
    if (r != 0) { c->jpeg_handle = nullptr; return fail(BEVK_ERR_CUDA, "nvjpegCreateSimple failed: %d", r); }
    r = nvjpeg().StateCreate(c->jpeg_handle, &c->jpeg_state);
    if (r != 0) { jpeg_release(c); return fail(BEVK_ERR_CUDA, "nvjpegJpegStateCreate failed: %d", r); }
  }
  for (int i = 0; i < n; ++i) {
    if (!jpegs[i] || !sizes[i]) return fail(BEVK_ERR_ARG, "JPEG stream %d is empty", i);
    int comps = 0, sub = 0, w[4] = {0, 0, 0, 0}, h[4] = {0, 0, 0, 0};
    int r = nvjpeg().GetImageInfo(c->jpeg_handle, jpegs[i], (size_t)sizes[i], &comps, &sub, w, h);
    if (r != 0) return fail(BEVK_ERR_ARG, "stream %d is not a JPEG nvJPEG can parse (status %d)", i, r);
    if (w[0] != width || h[0] != height) return fail(BEVK_ERR_ARG, "stream %d is %dx%d, the frame stack holds %dx%d", i, w[0], h[0], width, height);
    NvjpegImage dst{};
    dst.channel[0] = reinterpret_cast<unsigned char*>(d_frames) + (size_t)i * frame_stride;
    dst.pitch[0] = (size_t)width * 3;
    r = nvjpeg().Decode(c->jpeg_handle, c->jpeg_state, jpegs[i], (size_t)sizes[i], kNvjpegOutputBGRI, &dst, c->stream);
    if (r != 0) return fail(BEVK_ERR_CUDA, "nvjpegDecode(stream %d) failed: %d", i, r);
  }
  return BEVK_OK;
}

// BevGenerator.__call__ on JPEG streams: decode the batch into the library's frame stack, render, read the canvases back.
int bevk_bev_run_jpeg(bevk_ctx* c, const uint8_t* const* jpegs, const uint64_t* sizes, int batch, const uint8_t* car, int flags,
                      uint8_t* out) {
  NvtxRange nvtx_call("bevk_bev_run_jpeg (JPEG streams -> host canvases)");
  RET(use(c));
  RenderReq q;
  RET(canvas_req(c, "bevk_bev_run_jpeg", flags, 0, Frames(), batch, nullptr, nullptr, &q));
  RET(need_plan(c));
  if (!jpegs || !sizes || !out || batch < 1) return fail(BEVK_ERR_ARG, "bad argument");
  const size_t fpad = pad256((size_t)c->FW * c->FH * 3), cbytes = (size_t)c->BW * c->BH * 3;
  const int nf = batch * c->n_cam;
  RET(c->d_jpeg_frames.ensure(fpad * nf));
  RET(c->d_jpeg_canvas.ensure(cbytes * batch));
  q.src = Frames(c->d_jpeg_frames.p, (long long)fpad); q.out = c->d_jpeg_canvas.p;
  RET(render_check(c, q));
  RET(bevk_jpeg_decode(c, jpegs, sizes, nf, c->FW, c->FH, c->d_jpeg_frames.p, (int64_t)fpad));
  RET(upload_car(c, car, &q.car));
  c->timed = false;
  RET(render(c, q));
  CU(cudaMemcpyAsync(out, c->d_jpeg_canvas.p, cbytes * batch, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return BEVK_OK;
}

// ------------------------------------------------------------------ encoders: one host path for JPEG and PNG
// Every encoding call runs through enc_chunks: each chunk of images is encoded into one of the two slots of c->enc_out
// (slot_open ... slot_close), and enc_collect copies that slot's streams to the host while the next chunk is encoded.

// What an encoder reads: n images at img + i * istride, rows pitch bytes apart.
struct EncIn {
  const void* img = nullptr;
  long long istride = 0, pitch = 0;
};

// The channel counts the encoders take: grey, BGR, BGRA
static int check_enc_channels(int channels) {
  if (channels != 1 && channels != 3 && channels != 4)
    return fail(BEVK_ERR_UNSUPPORTED, "%d channels: the encoders take 1 (grey), 3 (BGR) or 4 (BGRA)", channels);
  return BEVK_OK;
}

// n device images of `channels` channels of the bevk_*_encode calls, rows row_stride bytes apart, image_stride apart
// (n > 1)
static int check_device_images(const void* d_images, int64_t image_stride, int64_t row_stride, int channels, int n, int w, int h) {
  if (!d_images || n < 1) return fail(BEVK_ERR_ARG, "bad argument");
  const int64_t rb = (int64_t)w * channels;
  if (row_stride < rb) return fail(BEVK_ERR_ARG, "row stride %lld < %lld bytes", (long long)row_stride, (long long)rb);
  if (n > 1 && image_stride < (int64_t)(h - 1) * row_stride + rb)
    return fail(BEVK_ERR_ARG, "image stride %lld is smaller than one image", (long long)image_stride);
  return BEVK_OK;
}

// The encoding calls write host memory and wait for the stream sizes, so they cannot be captured into a graph.
static int enc_call_check(bevk_ctx* c, const uint8_t* out, const uint64_t* sizes) {
  if (c->capturing) return fail(BEVK_ERR_ARG, "the encoding calls synchronise and cannot be captured into a graph");
  if (!out || !sizes) return fail(BEVK_ERR_ARG, "null host pointer");
  return BEVK_OK;
}

// Slot s for the streams of n images, `bytes` at most: its buffers, and the ctx stream ordered after the slot's previous
// streams have been copied out.  An encoder calls it before its first write into the slot.
static int slot_open(bevk_ctx* c, int s, int n, size_t bytes) {
  auto& e = c->enc_out;
  RET(e.out[s].ensure(bytes));
  RET(e.meta[s].ensure((size_t)(2ll * n + 1) * 8));
  if (e.h_sizes_cap[s] < (size_t)n) {
    if (e.h_sizes[s]) CU(cudaFreeHost(e.h_sizes[s]));      // enc_collect waited for its last copy
    e.h_sizes[s] = nullptr; e.h_sizes_cap[s] = 0;
    CU(cudaHostAlloc(reinterpret_cast<void**>(&e.h_sizes[s]), (size_t)n * 8, cudaHostAllocDefault));
    e.h_sizes_cap[s] = (size_t)n;
  }
  CU(cudaStreamWaitEvent(c->stream, e.ev_out_free[s], 0));
  return BEVK_OK;
}

// After an encoder's last kernel into slot s: ev1 (bevk_last_kernel_ms covers the kernels only), then the D2H of the
// stream sizes into page-locked memory and ev_sizes[s].  enc_collect(s) finishes the batch.
static int slot_close(bevk_ctx* c, int s, int n) {
  auto& e = c->enc_out;
  RET(time_end(c));
  CU(cudaMemcpyAsync(e.h_sizes[s], e.meta[s].as<unsigned long long>() + n, (size_t)n * 8, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaEventRecord(e.ev_sizes[s], c->stream));
  return BEVK_OK;
}

// Finish slot s's batch of n: wait for its sizes, store them in sizes[n], and copy streams to the host at out + *used on
// out_stream (not synchronised).  whole: all of the batch's streams or none; otherwise the leading streams that still fit
// in capacity, none once *full (an earlier stream did not fit).  *used grows by the bytes copied.
static int enc_collect(bevk_ctx* c, int s, int n, uint8_t* out, uint64_t capacity, bool whole, uint64_t* sizes, uint64_t* used,
                       bool* full) {
  auto& e = c->enc_out;
  CU(cudaEventSynchronize(e.ev_sizes[s]));
  unsigned long long fit = 0, all = 0;
  for (int i = 0; i < n; ++i) {
    sizes[i] = e.h_sizes[s][i];
    all += sizes[i];
    if (!*full && *used + fit + sizes[i] <= capacity) fit += sizes[i];
    else *full = true;
  }
  if (whole && fit < all) fit = 0;
  if (fit) {
    CU(cudaStreamWaitEvent(e.out_stream, e.ev_sizes[s], 0));
    CU(cudaMemcpyAsync(out + *used, e.out[s].p, fit, cudaMemcpyDeviceToHost, e.out_stream));
    CU(cudaEventRecord(e.ev_out_free[s], e.out_stream));
  }
  *used += fit;
  return BEVK_OK;
}

static int capacity_error(const char* fmt, int n, const uint64_t* sizes, uint64_t capacity) {
  unsigned long long total = 0;
  for (int i = 0; i < n; ++i) total += sizes[i];
  return fail(BEVK_ERR_ARG, "the %d %s streams take %llu bytes, capacity is %llu", n, fmt, total, (unsigned long long)capacity);
}

// Encode n images (n >= 1) chunk by chunk through the two slots.  enqueue(b0, nb, s) enqueues what makes images
// [b0, b0 + nb) and an encoder over them into slot s.  A chunk's streams are collected (wait for their sizes, D2H on
// out_stream) after the next chunk has been enqueued into the other slot.  whole: all streams or none (a single chunk);
// otherwise the leading streams that fit in capacity.  fmt names the format in the capacity error.
template <class Enqueue>
static int enc_chunks(bevk_ctx* c, const char* fmt, int n, int chunk, bool whole, uint8_t* out, uint64_t capacity,
                      uint64_t* sizes, Enqueue enqueue) {
  RET(enc_call_check(c, out, sizes));
  auto& e = c->enc_out;
  if (!e.out_stream) RET(create_stream_set(&e.out_stream, {&e.ev_sizes[0], &e.ev_sizes[1], &e.ev_out_free[0], &e.ev_out_free[1]}));
  uint64_t used = 0;
  bool full = false;
  int s = 0, prev_b0 = -1, prev_nb = 0;
  for (int b0 = 0; b0 < n; b0 += chunk, s ^= 1) {
    const int nb = std::min(chunk, n - b0);
    RET(enqueue(b0, nb, s));
    if (prev_b0 >= 0) RET(enc_collect(c, s ^ 1, prev_nb, out, capacity, whole, sizes + prev_b0, &used, &full));
    prev_b0 = b0; prev_nb = nb;
  }
  RET(enc_collect(c, s ^ 1, prev_nb, out, capacity, whole, sizes + prev_b0, &used, &full));
  CU(cudaStreamSynchronize(e.out_stream));
  return full ? capacity_error(fmt, n, sizes, capacity) : BEVK_OK;
}

// ------------------------------------------------------------------ JPEG encode on the device (bevk_jpeg_enc.cuh)
// The reference writes its results with cv2.imwrite (Tools/undistort.py:72-73, surroundBEV.py:340): D2H of the whole
// image, then libjpeg-turbo on a host core.  Here the encoder runs on the device and only the streams cross PCIe.
static int jpeg_size_check(int width, int height) {
  if (width < 1 || height < 1 || width > jpeg::kMaxDim || height > jpeg::kMaxDim)
    return fail(BEVK_ERR_ARG, "bad JPEG size %dx%d (1..%d)", width, height, jpeg::kMaxDim);
  return BEVK_OK;
}

// A JPEG list: keys 2..7 of cv2.IMWRITE_JPEG_*, normalised by jpeg::normalise under the call's quality.
static int jpeg_params_check(const int* params, int n, int quality, jpeg::Opts* o) {
  if (n < 0 || (n & 1) || (n && !params)) return fail(BEVK_ERR_ARG, "JPEG params: %d ints, need (key, value) pairs", n);
  for (int i = 0; i < n; i += 2)
    if (params[i] < jpeg::kProgressive || params[i] > jpeg::kSamplingFactor)
      return fail(BEVK_ERR_ARG, "JPEG params: key %d (IMWRITE_JPEG_QUALITY is the quality argument of each call; "
                  "keys are 2..7)", params[i]);
  jpeg::normalise(quality, params, n, o);
  return BEVK_OK;
}

// A bevk_jpeg_set_params list.  The calls that read it write baseline streams: PROGRESSIVE asks for another entropy
// coder and is refused, not ignored (the per-call bevk_jpeg_encode_params writes it).
static int jpeg_ctx_params_check(const int* params, int n, jpeg::Opts* o) {
  RET(jpeg_params_check(params, n, 95, o));
  if (o->progressive) return fail(BEVK_ERR_UNSUPPORTED, "JPEG params: IMWRITE_JPEG_PROGRESSIVE is not supported");
  return BEVK_OK;
}

// the ctx's list (bevk_jpeg_set_params checked it) under a call's quality
static jpeg::Opts jpeg_ctx_opts(const bevk_ctx* c, int quality) {
  jpeg::Opts o;
  jpeg::normalise(quality, c->enc.params.data(), (int)c->enc.params.size(), &o);
  return o;
}

static unsigned long long jpeg_bound(int w, int h, const jpeg::Opts& o) {
  const jpeg::Geom g = jpeg::geom(w, h, o);
  return o.progressive ? jpeg::prog::progressive_bound(g, o.rst) : jpeg::encode_bound(g, o);
}

int bevk_jpeg_encode_bound(int width, int height, uint64_t* bytes) {
  return bevk_jpeg_encode_bound_params(width, height, nullptr, 0, bytes);
}

int bevk_jpeg_set_params(bevk_ctx* c, const int* params, int n) {
  RET(use(c));
  jpeg::Opts o;
  RET(jpeg_ctx_params_check(params, n, &o));
  c->enc.params.assign(params, params + n);
  return BEVK_OK;
}

int bevk_jpeg_encode_bound_params(int width, int height, const int* params, int n, uint64_t* bytes) {
  if (!bytes) return fail(BEVK_ERR_ARG, "null bytes");
  RET(jpeg_size_check(width, height));
  jpeg::Opts o;
  RET(jpeg_ctx_params_check(params, n, &o));
  *bytes = jpeg_bound(width, height, o);
  return BEVK_OK;
}

int bevk_jpeg_encode_params_bound(int width, int height, const int* params, int n, uint64_t* bytes) {
  return bevk_jpeg_encode_channels_bound(width, height, 3, params, n, bytes);
}

int bevk_jpeg_encode_channels_bound(int width, int height, int channels, const int* params, int n, uint64_t* bytes) {
  if (!bytes) return fail(BEVK_ERR_ARG, "null bytes");
  RET(check_enc_channels(channels));
  RET(jpeg_size_check(width, height));
  jpeg::Opts o;
  RET(jpeg_params_check(params, n, 95, &o));
  *bytes = jpeg_bound(width, height, jpeg::channel_opts(o, channels));
  return BEVK_OK;
}

// Launch shapes of the baseline kernels: f(HY, VY, NC) as integral constants, for the layout of o (grey: 1, 1, 1)
template <class F>
static int with_layout(const jpeg::Opts& o, F&& f) {
  using std::integral_constant;
  if (o.nc == 1) return f(integral_constant<int, 1>{}, integral_constant<int, 1>{}, integral_constant<int, 1>{});
  return jpeg::with_sampling(o.hy, o.vy, [&](auto hy, auto vy) { return f(hy, vy, integral_constant<int, 3>{}); });
}
// k_jpeg_blocks of layout (HY, VY, NC) over images of C bytes per pixel
template <int HY, int VY, int NC>
static void launch_blocks(int C, unsigned grid, cudaStream_t st, const jpeg::EncArgs& a) {
  using namespace jpeg;
  if constexpr (NC == 1) k_jpeg_blocks<1, 1, 1><<<grid, kBlockThreads, 0, st>>>(a);
  else if (C == 4) k_jpeg_blocks<HY, VY, 4><<<grid, kBlockThreads, 0, st>>>(a);
  else k_jpeg_blocks<HY, VY><<<grid, kBlockThreads, 0, st>>>(a);
}

// Header (baseline) or frame prefix (progressive) into d_header and the tables into d_tabs: they depend on
// (w, h, options) only, so they are uploaded when one of these changes.
static int jpeg_tables(bevk_ctx* c, int w, int h, const jpeg::Opts& o) {
  using namespace jpeg;
  auto& e = c->enc;
  if (w == e.w && h == e.h && o == e.o) return BEVK_OK;
  Tables t;
  make_tables(o, &t);
  if (o.progressive) prog::frame_prefix(w, h, o, e.header);
  else make_header(w, h, o, e.header);
  RET(e.d_header.ensure(kMaxHeaderBytes));
  RET(e.d_tabs.ensure(sizeof(Tables)));
  CU(cudaMemcpyAsync(e.d_header.p, e.header, kMaxHeaderBytes, cudaMemcpyHostToDevice, c->stream));   // pageable: staged
  CU(cudaMemcpyAsync(e.d_tabs.p, &t, sizeof t, cudaMemcpyHostToDevice, c->stream));               // before returning
  e.w = w; e.h = h; e.o = o;
  return BEVK_OK;
}

// Enqueue the baseline encoder over n w x h images of C channels (o = channel_opts(..., C)) into slot s on the ctx
// stream.  The work buffers are single: batches use them one after the other in stream order.
static int jpeg_enqueue(bevk_ctx* c, int s, const EncIn& in, int n, int w, int h, const jpeg::Opts& o, int C = 3) {
  using namespace jpeg;
  auto& e = c->enc;
  RET(jpeg_tables(c, w, h, o));
  const Geom g = geom(w, h, o);
  const long long nblk = blocks_per_image(g), nb = nblk * n;
  const long long nint = intervals(g, o), ni = nint * n;
  const long long words_img = ((long long)((entropy_bound_bits(g, o) + 31) / 32) + 3) & ~3ll;   // 16-byte aligned regions
  const int chunks = (int)((words_img * 4 + kChunk - 1) / kChunk);
  const long long nch = (long long)n * chunks;
  if (nb > INT_MAX || nch > INT_MAX || ni > INT_MAX) return fail(BEVK_ERR_ARG, "batch of %d %dx%d images is too large for one call", n, w, h);
  RET(e.coef.ensure((size_t)nb * 128));
  RET(e.bits.ensure((size_t)nb * 8));
  RET(e.offs.ensure((size_t)nb * 8));
  RET(e.dcdiff.ensure((size_t)nb * 4));
  RET(e.words.ensure((size_t)(n * words_img * 4)));
  const size_t ffcap = e.ffcnt.cap;
  RET(e.ffcnt.ensure((size_t)nch * 4));
  if (e.ffcnt.cap != ffcap) CU(cudaMemsetAsync(e.ffcnt.p, 0, e.ffcnt.cap, c->stream));
  RET(e.ffscan.ensure((size_t)nch * 4));
  if (o.rst) {
    RET(e.ilen.ensure((size_t)ni * 8));
    RET(e.iofs.ensure((size_t)ni * 8));
  }
  if (o.optimize) {
    RET(e.counts.ensure((size_t)n * 1024 * 8));
    RET(e.huff.ensure((size_t)n * sizeof(Huff)));
    RET(e.hdrs.ensure((size_t)n * kMaxHeaderBytes));
    RET(e.hlen.ensure((size_t)n * 4));
  }
  size_t tmp1 = 0, tmp2 = 0;
  CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp1, e.bits.as<unsigned long long>(), e.offs.as<unsigned long long>(), (int)nb));
  CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp2, e.ffcnt.as<unsigned>(), e.ffscan.as<unsigned>(), (int)nch));
  size_t tmp3 = 0;
  if (o.rst) CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp3, e.ilen.as<unsigned long long>(), e.iofs.as<unsigned long long>(), (int)ni));
  const size_t tmp = std::max(std::max(tmp1, tmp2), tmp3);
  RET(e.scan_tmp.ensure(tmp));
  RET(slot_open(c, s, n, (size_t)n * encode_bound(g, o)));

  EncArgs a{};
  a.img = reinterpret_cast<const uint8_t*>(in.img); a.istride = in.istride; a.pitch = in.pitch; a.n = n; a.g = g; a.nblk = nblk;
  a.tabs = e.d_tabs.as<Tables>(); a.coef = e.coef.as<int16_t>(); a.bits = e.bits.as<unsigned long long>();
  a.offs = e.offs.as<unsigned long long>(); a.dcdiff = e.dcdiff.as<int>(); a.words = e.words.as<uint32_t>(); a.words_img = words_img;
  a.chunks_img = chunks; a.ffcnt = e.ffcnt.as<unsigned>(); a.ffscan = e.ffscan.as<unsigned>(); a.header = e.d_header.as<uint8_t>();
  a.out = c->enc_out.out[s].as<uint8_t>(); a.out_off = c->enc_out.meta[s].as<unsigned long long>(); a.sizes = a.out_off + n;
  a.rst = o.rst; a.nint = nint; a.hlen0 = header_bytes(o);
  if (o.rst) { a.ilen = e.ilen.as<unsigned long long>(); a.iofs = e.iofs.as<unsigned long long>(); }
  if (o.optimize) {
    a.counts = e.counts.as<unsigned long long>(); a.huff = e.huff.as<Huff>(); a.hdrs = e.hdrs.as<uint8_t>(); a.hlen = e.hlen.as<int>();
  }
  const unsigned gb = (unsigned)((nb + kBlockThreads - 1) / kBlockThreads), gc = (unsigned)((nch + 255) / 256);
  CU(cudaEventRecord(c->ev0, c->stream));
  RET(with_layout(o, [&](auto hy, auto vy, auto nc) -> int {
    constexpr int HY = hy(), VY = vy(), NC = nc();
    launch_blocks<HY, VY, NC>(C, gb, c->stream, a);
    LAUNCHED(c);
    k_jpeg_dc<HY, VY, NC><<<gb, kBlockThreads, 0, c->stream>>>(a);
    LAUNCHED(c);
    if (o.optimize) {   // per-image tables from the symbol counts, then every block's bits under them
      CU(cudaMemsetAsync(a.counts, 0, (size_t)n * 1024 * 8, c->stream));
      k_jpeg_count<HY, VY, NC><<<gb, kBlockThreads, 0, c->stream>>>(a);
      LAUNCHED(c);
      k_jpeg_huff<NC><<<(unsigned)((4ll * n + kHuffThreads - 1) / kHuffThreads), kHuffThreads, 0, c->stream>>>(a);
      LAUNCHED(c);
      k_jpeg_bits<HY, VY, NC><<<gb, kBlockThreads, 0, c->stream>>>(a);
      LAUNCHED(c);
    }
    CU(cub::DeviceScan::ExclusiveSum(e.scan_tmp.p, tmp1, a.bits, a.offs, (int)nb, c->stream));
    if (o.rst) {        // byte-aligned intervals: their padded lengths and offsets
      k_jpeg_intervals<<<(unsigned)((ni + 255) / 256), 256, 0, c->stream>>>(a);
      LAUNCHED(c);
      CU(cub::DeviceScan::ExclusiveSum(e.scan_tmp.p, tmp3, a.ilen, a.iofs, (int)ni, c->stream));
    }
    k_jpeg_zero<<<c->n_sm * 4, 256, 0, c->stream>>>(a);
    LAUNCHED(c);
    if (o.optimize && o.rst) k_jpeg_pack<HY, VY, true, true, NC><<<gb, kBlockThreads, 0, c->stream>>>(a);
    else if (o.optimize) k_jpeg_pack<HY, VY, true, false, NC><<<gb, kBlockThreads, 0, c->stream>>>(a);
    else if (o.rst) k_jpeg_pack<HY, VY, false, true, NC><<<gb, kBlockThreads, 0, c->stream>>>(a);
    else k_jpeg_pack<HY, VY, false, false, NC><<<gb, kBlockThreads, 0, c->stream>>>(a);
    LAUNCHED(c);
    return BEVK_OK;
  }));
  k_jpeg_ffcount<<<gc, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  CU(cub::DeviceScan::ExclusiveSum(e.scan_tmp.p, tmp2, a.ffcnt, a.ffscan, (int)nch, c->stream));
  k_jpeg_layout<<<1, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  k_jpeg_stuff<<<gc, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  return slot_close(c, s, n);
}

// Enqueue the progressive encoder over n w x h images into slot s: k_jpeg_blocks, then the k_jpeg_prog_* pipeline over
// every scan of every image at once (bevk_jpeg_prog.cuh).  The k_jpeg_prog_* kernels are instantiated per component
// count (NC = o.nc): grey images run the six-scan script.
template <int NC>
static int jpeg_prog_run(bevk_ctx* c, int s, const EncIn& in, int n, int w, int h, const jpeg::Opts& o, int C) {
  using namespace jpeg;
  using namespace jpeg::prog;
  auto& e = c->enc;
  const Geom g = geom(w, h, o);
  const Layout L = layout(g, o.rst);
  const long long nblk = blocks_per_image(g), T = L.blk[kScans], S = L.seg[kScans];
  const long long N = T * n, NS = S * n;
  const long long words_img = ((long long)((prog::entropy_bound_bits(g, o.rst) + 31) / 32) + 3) & ~3ll;
  const int chunks = (int)((words_img * 4 + kChunk - 1) / kChunk);
  const long long nch = (long long)n * chunks;
  if (N >= INT_MAX || NS >= INT_MAX || nch >= INT_MAX)
    return fail(BEVK_ERR_ARG, "batch of %d %dx%d images is too large for one progressive call", n, w, h);
  RET(jpeg_tables(c, w, h, o));
  RET(e.coef.ensure((size_t)(nblk * n) * 128));
  RET(e.desc.ensure((size_t)N * 4));
  RET(e.pe.ensure((size_t)N * 8));
  RET(e.pc.ensure((size_t)N * 8));
  RET(e.ph.ensure((size_t)N * 4));
  RET(e.jump.ensure((size_t)(N + 1) * 4));
  RET(e.jump2.ensure((size_t)(N + 1) * 4));
  RET(e.mark.ensure((size_t)(N + 1)));
  RET(e.rs.ensure((size_t)N * 4));
  RET(e.counts.ensure((size_t)n * kTables * 256 * 4));
  RET(e.codes.ensure((size_t)n * kTables * 256 * 4));
  RET(e.hdrs.ensure((size_t)n * kScans * kHdrStride));
  RET(e.hlen.ensure((size_t)n * kScans * 4));
  RET(e.bits.ensure((size_t)N * 8));
  RET(e.offs.ensure((size_t)N * 8));
  RET(e.ilen.ensure((size_t)NS * 8));
  RET(e.iofs.ensure((size_t)NS * 8));
  RET(e.ins.ensure((size_t)NS * 4));
  RET(e.insx.ensure((size_t)NS * 4));
  RET(e.words.ensure((size_t)(n * words_img * 4)));
  const size_t ffcap = e.ffcnt.cap;
  RET(e.ffcnt.ensure((size_t)nch * 4));
  if (e.ffcnt.cap != ffcap) CU(cudaMemsetAsync(e.ffcnt.p, 0, e.ffcnt.cap, c->stream));
  RET(e.ffscan.ensure((size_t)nch * 4));
  RET(slot_open(c, s, n, (size_t)n * progressive_bound(g, o.rst)));

  ProgArgs a{};
  a.n = n; a.rst = o.rst; a.g = g; a.nblk = nblk; a.L = L; a.T = T; a.S = S;
  a.coef = e.coef.as<int16_t>(); a.desc = e.desc.as<uint32_t>(); a.pe = e.pe.as<unsigned long long>();
  a.pc = e.pc.as<unsigned long long>(); a.ph = e.ph.as<unsigned>(); a.jump = e.jump.as<unsigned>(); a.jump2 = e.jump2.as<unsigned>();
  a.mark = e.mark.as<uint8_t>(); a.rs = e.rs.as<unsigned>(); a.counts = e.counts.as<unsigned>(); a.codes = e.codes.as<uint32_t>();
  a.hdrs = e.hdrs.as<uint8_t>(); a.hlen = e.hlen.as<int>(); a.bits = e.bits.as<unsigned long long>();
  a.offs = e.offs.as<unsigned long long>(); a.ilen = e.ilen.as<unsigned long long>(); a.iofs = e.iofs.as<unsigned long long>();
  a.ins = e.ins.as<unsigned>(); a.insx = e.insx.as<unsigned>(); a.words = e.words.as<uint32_t>(); a.words_img = words_img;
  a.chunks_img = chunks; a.ffcnt = e.ffcnt.as<unsigned>(); a.ffscan = e.ffscan.as<unsigned>(); a.prefix = e.d_header.as<uint8_t>();
  a.out = c->enc_out.out[s].as<uint8_t>(); a.out_off = c->enc_out.meta[s].as<unsigned long long>(); a.sizes = a.out_off + n;

  using ItE = cub::TransformInputIterator<unsigned long long, DescE, const uint32_t*>;
  using ItC = cub::TransformInputIterator<unsigned long long, DescC, const uint32_t*>;
  using ItH = cub::TransformInputIterator<unsigned, DescH, const uint32_t*>;
  using ItM = cub::TransformInputIterator<unsigned, MarkIndex, cub::CountingInputIterator<unsigned>>;
  const ItM itm(cub::CountingInputIterator<unsigned>(0), MarkIndex{a.mark});
  size_t tmp[8] = {};
  CU(cub::DeviceScan::InclusiveSum(nullptr, tmp[0], ItE(a.desc, DescE()), a.pe, (int)N));
  CU(cub::DeviceScan::InclusiveSum(nullptr, tmp[1], ItC(a.desc, DescC()), a.pc, (int)N));
  CU(cub::DeviceScan::InclusiveSum(nullptr, tmp[2], ItH(a.desc, DescH()), a.ph, (int)N));
  CU(cub::DeviceScan::InclusiveScan(nullptr, tmp[3], itm, a.rs, MaxU(), (int)N));
  CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp[4], a.bits, a.offs, (int)N));
  CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp[5], a.ilen, a.iofs, (int)NS));
  CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp[6], a.ins, a.insx, (int)NS));
  CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp[7], a.ffcnt, a.ffscan, (int)nch));
  RET(e.scan_tmp.ensure(*std::max_element(tmp, tmp + 8)));
  void* st = e.scan_tmp.p;

  EncArgs b{};
  b.img = reinterpret_cast<const uint8_t*>(in.img); b.istride = in.istride; b.pitch = in.pitch; b.n = n; b.g = g; b.nblk = nblk;
  b.tabs = e.d_tabs.as<Tables>(); b.coef = e.coef.as<int16_t>(); b.bits = a.bits;   // k_jpeg_blocks' AC bit counts land in scratch
  const unsigned gb = (unsigned)((nblk * n + kBlockThreads - 1) / kBlockThreads);
  const unsigned gN = (unsigned)((N + 255) / 256), gN1 = (unsigned)((N + 1 + 255) / 256), gS = (unsigned)((NS + 255) / 256);
  const unsigned gc = (unsigned)((nch + 255) / 256);
  CU(cudaEventRecord(c->ev0, c->stream));
  RET(with_layout(o, [&](auto hy, auto vy, auto nc) -> int {
    launch_blocks<hy(), vy(), nc()>(C, gb, c->stream, b);
    LAUNCHED(c);
    return BEVK_OK;
  }));
  k_jpeg_prog_desc<NC><<<gN, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  k_jpeg_prog_hard<NC><<<gN, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  CU(cub::DeviceScan::InclusiveSum(st, tmp[0], ItE(a.desc, DescE()), a.pe, (int)N, c->stream));
  CU(cub::DeviceScan::InclusiveSum(st, tmp[1], ItC(a.desc, DescC()), a.pc, (int)N, c->stream));
  CU(cub::DeviceScan::InclusiveSum(st, tmp[2], ItH(a.desc, DescH()), a.ph, (int)N, c->stream));
  k_jpeg_prog_next<NC><<<gN1, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  long long longest = 0;   // the longest scan bounds every chain of run starts
  for (int k = 0; k < kScans; ++k) longest = std::max(longest, L.blk[k + 1] - L.blk[k]);
  for (long long span = 1; span <= longest; span *= 2) {
    k_jpeg_prog_jump<<<gN1, 256, 0, c->stream>>>(a.jump, a.jump2, a.mark, N);
    LAUNCHED(c);
    std::swap(a.jump, a.jump2);
  }
  CU(cub::DeviceScan::InclusiveScan(st, tmp[3], itm, a.rs, MaxU(), (int)N, c->stream));
  CU(cudaMemsetAsync(a.counts, 0, (size_t)n * kTables * 256 * 4, c->stream));
  k_jpeg_prog_count<NC><<<gN, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  k_jpeg_prog_huff<NC><<<(unsigned)((n + kProgHuffImages - 1) / kProgHuffImages), kProgHuffThreads, 0, c->stream>>>(a);
  LAUNCHED(c);
  k_jpeg_prog_bits<NC><<<gN, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  CU(cub::DeviceScan::ExclusiveSum(st, tmp[4], a.bits, a.offs, (int)N, c->stream));
  k_jpeg_prog_segs<NC><<<gS, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  CU(cub::DeviceScan::ExclusiveSum(st, tmp[5], a.ilen, a.iofs, (int)NS, c->stream));
  CU(cub::DeviceScan::ExclusiveSum(st, tmp[6], a.ins, a.insx, (int)NS, c->stream));
  k_jpeg_prog_zero<<<c->n_sm * 4, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  k_jpeg_prog_pack<NC><<<gN, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  k_jpeg_prog_ffcount<<<gc, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  CU(cub::DeviceScan::ExclusiveSum(st, tmp[7], a.ffcnt, a.ffscan, (int)nch, c->stream));
  k_jpeg_prog_layout<NC><<<1, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  k_jpeg_prog_stuff<NC><<<gc, 256, 0, c->stream>>>(a);
  LAUNCHED(c);
  return slot_close(c, s, n);
}
static int jpeg_prog_enqueue(bevk_ctx* c, int s, const EncIn& in, int n, int w, int h, const jpeg::Opts& o, int C = 3) {
  return o.nc == 1 ? jpeg_prog_run<1>(c, s, in, n, w, h, o, C) : jpeg_prog_run<3>(c, s, in, n, w, h, o, C);
}

// Images per chunk of the chunked device-frame calls.  8 canvases (24 MB at 1000^2: they stay in the 50 MB L2) beat the
// whole batch at once on H100 (DESIGN.md section 4); BEVK_JPEG_CHUNK=n sets another size, 0 the whole batch.
static int jpeg_chunk(int n) {
  int chunk = std::min(n, 8);
  if (const char* env = getenv("BEVK_JPEG_CHUNK")) chunk = atoi(env) > 0 ? std::min(n, atoi(env)) : n;
  return chunk;
}

// ------------------------------------------------------------------ BEV canvases straight to JPEG (surroundBEV.py:340)
// BevGenerator.__call__ then cv2.imencode: each chunk of frame-sets is rendered into ctx scratch and encoded there, and
// only the streams come back.  Under BALANCE the render's k_gain applies colour balance and the car to the chunk's
// canvases before the encoder reads them.  The call is checked before the render set-up enqueues anything.
static int to_jpeg_check(bevk_ctx* c, uint8_t* out, uint64_t* sizes) {
  RET(need_plan(c));
  RET(enc_call_check(c, out, sizes));
  return jpeg_size_check(c->BW, c->BH);
}

int bevk_bev_run_to_jpeg(bevk_ctx* c, const uint8_t* const* srcs, int64_t src_stride, int batch, const uint8_t* car, int flags,
                         int quality, uint8_t* out, uint64_t capacity, uint64_t* sizes) {
  NvtxRange nvtx_call("bevk_bev_run_to_jpeg (host frames -> host JPEG streams)");
  RET(use(c));
  HostIngest h;
  RET(read_flags(c, flags, 0, "bevk_bev_run_to_jpeg", &h.fmt, &h.ofmt));
  RET(to_jpeg_check(c, out, sizes));
  const jpeg::Opts o = jpeg_ctx_opts(c, quality);
  RET(ingest_setup(c, srcs, src_stride, batch, car, flags, &h));
  // the ingest chunks are the encoder's: staging half = canvas half = encoder slot
  return enc_chunks(c, "JPEG", batch, h.chunk, false, out, capacity, sizes, [&](int b0, int nb, int half) -> int {
    uint8_t* dcanvas = nullptr;
    RET(render_chunk(c, h, srcs, src_stride, flags, b0, nb, half, &dcanvas));
    return jpeg_enqueue(c, half, EncIn{dcanvas, (long long)h.cbytes, (long long)c->BW * 3}, nb, c->BW, c->BH, o);
  });
}

int bevk_bev_frames_to_jpeg(bevk_ctx* c, const void* const* frames, int batch, const void* d_car, int flags, int quality,
                            uint8_t* out, uint64_t capacity, uint64_t* sizes) {
  NvtxRange nvtx_call("bevk_bev_frames_to_jpeg (device frames -> host JPEG streams)");
  RET(use(c));
  RenderReq q;
  RET(canvas_req(c, "bevk_bev_frames_to_jpeg", flags, 0, Frames(), batch, d_car, nullptr, &q));
  RET(to_jpeg_check(c, out, sizes));
  if (!frames) return fail(BEVK_ERR_ARG, "null pointer");
  const jpeg::Opts o = jpeg_ctx_opts(c, quality);
  Frames src;
  RET(frames_src(c, frames, batch, &src));
  // every chunk is rendered into the same canvas scratch: the next render is stream-ordered after the encoder read it
  const int chunk = jpeg_chunk(batch);
  RET(c->d_canvas.ensure((size_t)c->BW * c->BH * 3 * chunk));
  uint8_t* dcanvas = c->d_canvas.as<uint8_t>();
  return enc_chunks(c, "JPEG", batch, chunk, false, out, capacity, sizes, [&](int b0, int nb, int s) -> int {
    q.src = src;
    if (src.table) q.src.table += (size_t)b0 * c->n_cam;
    else q.src.base += (long long)b0 * c->n_cam * src.stride;
    q.batch = nb; q.out = dcanvas;
    RET(render_check(c, q));
    RET(render(c, q));
    return jpeg_enqueue(c, s, EncIn{dcanvas, (long long)c->BW * c->BH * 3, (long long)c->BW * 3}, nb, c->BW, c->BH, o);
  });
}

// bevk_jpeg_encode is this call under the ctx's list, which bevk_jpeg_set_params checked as this call checks its own.
int bevk_jpeg_encode(bevk_ctx* c, const void* d_images, int64_t image_stride, int64_t row_stride, int n, int width, int height,
                     int quality, uint8_t* out, uint64_t capacity, uint64_t* sizes) {
  NvtxRange nvtx_call("bevk_jpeg_encode (device images -> host JPEG streams)");
  RET(use(c));
  return bevk_jpeg_encode_params(c, c->enc.params.data(), (int)c->enc.params.size(), d_images, image_stride, row_stride, n,
                                 width, height, quality, out, capacity, sizes);
}

// n device images of `channels` channels under a per-call list, as one chunk: all streams or none
static int jpeg_encode_images(bevk_ctx* c, const int* params, int n_params, const void* d_images, int64_t image_stride,
                              int64_t row_stride, int channels, int n, int width, int height, int quality, uint8_t* out,
                              uint64_t capacity, uint64_t* sizes) {
  RET(use(c));
  RET(check_enc_channels(channels));
  jpeg::Opts o;
  RET(jpeg_params_check(params, n_params, quality, &o));
  o = jpeg::channel_opts(o, channels);
  RET(jpeg_size_check(width, height));
  RET(check_device_images(d_images, image_stride, row_stride, channels, n, width, height));
  const EncIn in{d_images, image_stride, row_stride};
  return enc_chunks(c, "JPEG", n, n, true, out, capacity, sizes, [&](int, int, int s) {
    return o.progressive ? jpeg_prog_enqueue(c, s, in, n, width, height, o, channels)
                         : jpeg_enqueue(c, s, in, n, width, height, o, channels);
  });
}

int bevk_jpeg_encode_params(bevk_ctx* c, const int* params, int n_params, const void* d_images, int64_t image_stride,
                            int64_t row_stride, int n, int width, int height, int quality, uint8_t* out, uint64_t capacity,
                            uint64_t* sizes) {
  NvtxRange nvtx_call("bevk_jpeg_encode_params (device images -> host JPEG streams)");
  return jpeg_encode_images(c, params, n_params, d_images, image_stride, row_stride, 3, n, width, height, quality, out,
                            capacity, sizes);
}

int bevk_jpeg_encode_channels(bevk_ctx* c, const int* params, int n_params, const void* d_images, int64_t image_stride,
                              int64_t row_stride, int channels, int n, int width, int height, int quality, uint8_t* out,
                              uint64_t capacity, uint64_t* sizes) {
  NvtxRange nvtx_call("bevk_jpeg_encode_channels (device images -> host JPEG streams)");
  return jpeg_encode_images(c, params, n_params, d_images, image_stride, row_stride, channels, n, width, height, quality,
                            out, capacity, sizes);
}

int bevk_undistort_jpeg(bevk_ctx* c, int slot, const uint8_t* src, int sw, int sh, int64_t sstride, int interp, int quality,
                        uint8_t* out, uint64_t capacity, uint64_t* size) {
  NvtxRange nvtx_call("bevk_undistort_jpeg (host frame -> undistorted JPEG)");
  RET(use(c));
  ImageOp op;
  RET(undistort_op(c, slot, interp, &op));
  RET(check_image(src, sw, sh, sstride, u8(3), "src"));
  RET(jpeg_size_check(op.dw, op.dh));
  const jpeg::Opts o = jpeg_ctx_opts(c, quality);
  return enc_chunks(c, "JPEG", 1, 1, true, out, capacity, size, [&](int, int, int s) -> int {
    RET(host_launch(c, op, src, sw, sh, sstride, u8(3), op.dw, op.dh));
    return jpeg_enqueue(c, s, EncIn{c->s_dst.p, 0, (long long)op.dw * 3}, 1, op.dw, op.dh, o);
  });
}

// Device frames -> undistorted -> JPEG, chunk by chunk as bevk_bev_frames_to_jpeg: chunk i+1 is undistorted into the
// scratch (stream-ordered after chunk i's encoder kernels read it) while chunk i's streams are copied out.
int bevk_undistort_stack_jpeg(bevk_ctx* c, int slot, const void* d_src, int64_t src_image_stride, int sw, int sh,
                              int64_t src_row_stride, int n, int interp, int quality, uint8_t* out, uint64_t capacity,
                              uint64_t* sizes) {
  NvtxRange nvtx_call("bevk_undistort_stack_jpeg (device frames -> undistorted JPEG streams)");
  RET(use(c));
  ImageOp op;
  RET(undistort_op(c, slot, interp, &op));
  RET(check_stack_src(d_src, src_image_stride, sw, sh, src_row_stride, u8(3), n));
  const int dw = op.dw, dh = op.dh;
  RET(jpeg_size_check(dw, dh));
  const jpeg::Opts o = jpeg_ctx_opts(c, quality);
  const int chunk = jpeg_chunk(n);
  const long long ibytes = (long long)dw * dh * 3;
  const ImageBatch b = device_batch(d_src, src_image_stride, sw, sh, src_row_stride, n, nullptr, ibytes, dw, dh, (long long)dw * 3);
  return enc_chunks(c, "JPEG", n, chunk, false, out, capacity, sizes, [&](int b0, int nb, int s) -> int {
    RET(c->s_dst.ensure((size_t)ibytes * chunk));
    ImageBatch part = b;   // frames [b0, b0 + nb) into the dense scratch
    part.src += (long long)b0 * b.sistride;
    part.n = nb;
    part.dst = c->s_dst.as<uint8_t>(); part.distride = ibytes;
    RET(launch(c, op, part, u8(3)));
    return jpeg_enqueue(c, s, EncIn{c->s_dst.p, ibytes, (long long)dw * 3}, nb, dw, dh, o);
  });
}

// ------------------------------------------------------------------ PNG encode on the device (bevk_png_enc.cuh)
// cv2.imwrite('x.png', img) writes through libpng + zlib on a host core.  Under cv2's default settings (SUB, level 1,
// Z_RLE) and Z_HUFFMAN_ONLY zlib's parse has no history, so the device reproduces the stream byte for byte in parallel.
static int png_params_check(const int* params, int n, png::Opts* o, bool hash_chain = false) {
  const int r = png::normalise(params, n, o, hash_chain);
  if (r == 1)
    return fail(BEVK_ERR_ARG, "PNG params: %d ints; need (key, value) pairs with keys 16..20 (cv2.IMWRITE_PNG_*)", n);
  if (r == 2 && hash_chain)
    return fail(BEVK_ERR_UNSUPPORTED, "PNG params: the device encoder writes zlib levels 1..9 under IMWRITE_PNG_STRATEGY_RLE "
                "or _HUFFMAN_ONLY, and levels 4..9 under the other strategies (levels 1..3 there are zlib's deflate_fast; "
                "level 0, BILEVEL and ZLIBBUFFER_SIZE are refused too)");
  if (r == 2)
    return fail(BEVK_ERR_UNSUPPORTED, "PNG params: the device encoder writes zlib levels 1..9 under IMWRITE_PNG_STRATEGY_RLE "
                "or _HUFFMAN_ONLY only (a compression level without a later strategy is zlib's hash-chain LZ77, which "
                "bevk_png_encode_params takes at levels 4..9; level 0, BILEVEL and ZLIBBUFFER_SIZE are refused too)");
  return BEVK_OK;
}

static int png_size_check(int width, int height, int channels = 3) {
  if (width < 1 || height < 1 || png::image_bytes(width, height, channels) > png::kMaxImageBytes)
    return fail(BEVK_ERR_ARG, "bad PNG size %dx%d (at least 1x1, at most %lld filtered bytes)", width, height,
                png::kMaxImageBytes);
  return BEVK_OK;
}

int bevk_png_set_params(bevk_ctx* c, const int* params, int n) {
  RET(use(c));
  png::Opts o;
  RET(png_params_check(params, n, &o));
  c->png.params.assign(params, params + n);
  return BEVK_OK;
}

int bevk_png_encode_bound(int width, int height, const int* params, int n, uint64_t* bytes) {
  if (!bytes) return fail(BEVK_ERR_ARG, "null bytes");
  RET(png_size_check(width, height));
  png::Opts o;
  RET(png_params_check(params, n, &o));
  *bytes = (uint64_t)png::encode_bound(width, height);
  return BEVK_OK;
}

int bevk_png_encode_channels_bound(int width, int height, int channels, uint64_t* bytes) {
  if (!bytes) return fail(BEVK_ERR_ARG, "null bytes");
  RET(check_enc_channels(channels));
  RET(png_size_check(width, height, channels));
  *bytes = (uint64_t)png::encode_bound(width, height, channels);
  return BEVK_OK;
}

// Filtered bytes per group: the group's scans, symbols and run starts take 11 bytes per filtered byte of scratch.  The
// hash-chain parse takes about 50 (sort keys and positions twice, prev, two match records, two jump arrays, marks,
// counts, symbols and distances, the sort's scratch), so its groups are a quarter of the size; a single image larger
// than a group still runs as one group of one, so a hash-chain image needs about 50 B of device memory per filtered
// byte.  Its hash sort keys are (image in group << 15) | hash, 32 bits with the sentinel (group size << 15) of the
// last 2 bytes: at most 2^16 images per group.
constexpr long long kPngGroupBytes = 1ll << 27, kPngLazyGroupBytes = 1ll << 25, kPngLazyGroupImages = 1ll << 16;

// Enqueue the PNG encoder over n width x height images of C channels into slot s, group by group; every group's streams
// land compacted in the slot after the ones before (the running end at meta[2n]).
static int png_enqueue(bevk_ctx* c, int s, const EncIn& in, int n, int width, int height, const png::Opts& o, int C = 3) {
  using namespace png;
  auto& e = c->png;
  const bool lazy = lazy_parse(o);
  const long long N = image_bytes(width, height, C), maxb = max_blocks(N), zb = zlib_bound(N);
  const long long zwords = zb / 4 + 2, maxch = idat_chunks(zb), bound = encode_bound(width, height, C);
  const int g = (int)std::max(1ll, std::min({(long long)n, (lazy ? kPngLazyGroupBytes : kPngGroupBytes) / N,
                                               lazy ? kPngLazyGroupImages : (long long)n}));
  const long long gN = g * N;
  RET(e.f.ensure((size_t)gN + 8));   // common_len's word loads read up to 3 bytes past the last image
  RET(e.nblk.ensure((size_t)g * 4));
  RET(e.rowad.ensure((size_t)g * height * sizeof(Adler)));
  RET(e.syms.ensure((size_t)gN * 2));
  RET(e.nsym.ensure((size_t)g * 4));
  RET(e.blk.ensure((size_t)g * maxb * sizeof(Blk)));
  RET(e.codes.ensure((size_t)g * maxb * (kLCodes + kDCodes) * 4));
  RET(e.hdr.ensure((size_t)g * maxb * kHdrWords * 4));
  RET(e.zw.ensure((size_t)g * zwords * 4));
  RET(e.zbytes.ensure((size_t)g * 8));
  RET(slot_open(c, s, n, (size_t)(n * bound)));
  unsigned long long* meta = c->enc_out.meta[s].as<unsigned long long>();
  using KeyIt = cub::TransformInputIterator<unsigned, RunStartKey, cub::CountingInputIterator<unsigned>>;
  using FlagIt = cub::TransformInputIterator<unsigned, SymbolFlag, cub::CountingInputIterator<unsigned>>;
  PngArgs a{};
  a.istride = in.istride; a.pitch = in.pitch; a.W = width; a.H = height; a.filters = o.filters; a.strategy = o.strategy;
  a.colour = colour_type(C); a.rb = row_bytes(width, C);
  a.N = N; a.maxb = maxb; a.zwords = zwords; a.maxchunks = maxch;
  a.f = e.f.as<uint8_t>(); a.rowad = e.rowad.as<Adler>(); a.syms = e.syms.as<uint16_t>(); a.nsym = e.nsym.as<unsigned>();
  a.blk = e.blk.as<Blk>(); a.codes = e.codes.as<uint32_t>(); a.hdr = e.hdr.as<uint32_t>(); a.zw = e.zw.as<uint32_t>();
  a.zbytes = e.zbytes.as<unsigned long long>(); a.base = meta + 2ll * n; a.out = c->enc_out.out[s].as<uint8_t>();
  a.nblk = e.nblk.as<unsigned>(); a.level = o.level; a.flevel = zlib_flevel(o);
  size_t tmp1 = 0, tmp2 = 0;
  int key_bits = 15;
  while ((1ll << key_bits) <= ((long long)g << 15)) ++key_bits;
  if (lazy) {   // hash sort, prev, match records, jumps, marks, chain symbol counts and their scan, distances
    RET(e.keys.ensure((size_t)gN * 4)); RET(e.keys2.ensure((size_t)gN * 4));
    RET(e.pos.ensure((size_t)gN * 4)); RET(e.pos2.ensure((size_t)gN * 4));
    RET(e.prev.ensure((size_t)gN * 4)); RET(e.recs.ensure((size_t)gN * sizeof(MatchRec)));
    RET(e.jump.ensure((size_t)gN * 4)); RET(e.jump2.ensure((size_t)gN * 4)); RET(e.mark.ensure((size_t)gN));
    RET(e.cnt.ensure((size_t)(gN + 1) * 4)); RET(e.symidx.ensure((size_t)(gN + 1) * 4)); RET(e.dists.ensure((size_t)gN * 2));
    a.prev = e.prev.as<unsigned>(); a.recs = e.recs.as<MatchRec>(); a.mark = e.mark.as<uint8_t>();
    a.cnt = e.cnt.as<unsigned>(); a.symidx = e.symidx.as<unsigned>(); a.dists = e.dists.as<uint16_t>();
    CU(cub::DeviceRadixSort::SortPairs(nullptr, tmp1, e.keys.as<unsigned>(), e.keys2.as<unsigned>(), e.pos.as<unsigned>(),
                                       e.pos2.as<unsigned>(), (int)gN, 0, key_bits));
    CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp2, e.cnt.as<unsigned>(), e.symidx.as<unsigned>(), (int)gN + 1));
    RET(e.scan_tmp.ensure(std::max(tmp1, tmp2)));
  }
  if (o.strategy == kZRle) {   // run starts and symbol indices (Z_HUFFMAN_ONLY: every byte is a symbol at its position)
    RET(e.runs.ensure((size_t)gN * 4));
    RET(e.symidx.ensure((size_t)(gN + 1) * 4));
    a.runs = e.runs.as<unsigned>(); a.symidx = e.symidx.as<unsigned>();
    const cub::CountingInputIterator<unsigned> pos(0);
    CU(cub::DeviceScan::InclusiveScan(nullptr, tmp1, KeyIt(pos, RunStartKey{a.f, N}), e.runs.as<unsigned>(), MaxOp(), (int)gN));
    CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp2, FlagIt(pos, SymbolFlag{a, 0}), e.symidx.as<unsigned>(), (int)gN + 1));
    RET(e.scan_tmp.ensure(std::max(tmp1, tmp2)));
  }
  CU(cudaMemsetAsync(a.base, 0, 8, c->stream));
  CU(cudaEventRecord(c->ev0, c->stream));
  for (int b0 = 0; b0 < n; b0 += g) {
    const int gn = std::min(g, n - b0);
    a.img = reinterpret_cast<const uint8_t*>(in.img) + b0 * in.istride;
    a.n = gn;
    a.out_off = meta + b0;
    a.sizes = meta + n + b0;
    const long long total = gn * N;
    const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, (long long)c->n_sm * 16);
    const unsigned gf = (unsigned)(gn * height);
    if (C == 1) k_png_filter<1><<<gf, kPngThreads, 0, c->stream>>>(a);
    else if (C == 4) k_png_filter<4><<<gf, kPngThreads, 0, c->stream>>>(a);
    else k_png_filter<<<gf, kPngThreads, 0, c->stream>>>(a);
    LAUNCHED(c);
    if (lazy) {
      k_png_keys<<<grid, 256, 0, c->stream>>>(HashKey{a.f, N, (unsigned)gn}, e.keys.as<unsigned>(), e.pos.as<unsigned>(),
                                              (unsigned)total);
      LAUNCHED(c);
      CU(cub::DeviceRadixSort::SortPairs(e.scan_tmp.p, tmp1, e.keys.as<unsigned>(), e.keys2.as<unsigned>(), e.pos.as<unsigned>(),
                                         e.pos2.as<unsigned>(), (int)total, 0, key_bits, c->stream));
      k_png_prev<<<grid, 256, 0, c->stream>>>(e.keys2.as<unsigned>(), e.pos2.as<unsigned>(), e.prev.as<unsigned>(),
                                               (unsigned)total, N);
      LAUNCHED(c);
      k_png_match<<<(unsigned)((total + 127) / 128), 128, 0, c->stream>>>(a);
      LAUNCHED(c);
      a.jump = e.jump.as<unsigned>(); a.jump2 = e.jump2.as<unsigned>();
      k_png_next<<<grid, 256, 0, c->stream>>>(a);
      LAUNCHED(c);
      for (long long len = 1; len < N; len *= 2) {   // a parse has at most N positions
        k_png_jump<<<grid, 256, 0, c->stream>>>(a.jump, a.jump2, a.mark, (unsigned)total);
        LAUNCHED(c);
        std::swap(a.jump, a.jump2);
      }
      k_png_count<<<grid, 256, 0, c->stream>>>(a);
      LAUNCHED(c);
      CU(cub::DeviceScan::ExclusiveSum(e.scan_tmp.p, tmp2, e.cnt.as<unsigned>(), e.symidx.as<unsigned>(), (int)total + 1,
                                       c->stream));
    }
    if (o.strategy == kZRle) {
      const cub::CountingInputIterator<unsigned> pos(0);
      CU(cub::DeviceScan::InclusiveScan(e.scan_tmp.p, tmp1, KeyIt(pos, RunStartKey{a.f, N}), e.runs.as<unsigned>(), MaxOp(), (int)total,
                                        c->stream));
      CU(cub::DeviceScan::ExclusiveSum(e.scan_tmp.p, tmp2, FlagIt(pos, SymbolFlag{a, (unsigned)total}),
                                       e.symidx.as<unsigned>(), (int)total + 1, c->stream));
    }
    k_png_setup<<<(unsigned)((gn + 127) / 128), 128, 0, c->stream>>>(a);
    LAUNCHED(c);
    if (lazy) k_png_lazy_compact<<<grid, 256, 0, c->stream>>>(a);
    else k_png_compact<<<grid, 256, 0, c->stream>>>(a);
    LAUNCHED(c);
    k_png_tree<<<(unsigned)(gn * maxb), kPngThreads, 0, c->stream>>>(a);
    LAUNCHED(c);
    CU(cudaMemsetAsync(a.zw, 0, (size_t)gn * zwords * 4, c->stream));
    k_png_layout<<<(unsigned)((gn + 127) / 128), 128, 0, c->stream>>>(a);
    LAUNCHED(c);
    k_png_offsets<<<1, 1, 0, c->stream>>>(a);
    LAUNCHED(c);
    k_png_pack<<<(unsigned)(gn * maxb), kPngThreads, 0, c->stream>>>(a);
    LAUNCHED(c);
    k_png_frame<<<(unsigned)((gn * maxch * 32 + kPngThreads - 1) / kPngThreads), kPngThreads, 0, c->stream>>>(a);
    LAUNCHED(c);
  }
  return slot_close(c, s, n);
}

// n device images of `channels` channels through the PNG encoder under o, as one chunk: all streams or none
static int png_encode_images(bevk_ctx* c, const png::Opts& o, const void* d_images, int64_t image_stride, int64_t row_stride,
                             int channels, int n, int width, int height, uint8_t* out, uint64_t capacity, uint64_t* sizes) {
  RET(check_enc_channels(channels));
  RET(png_size_check(width, height, channels));
  RET(check_device_images(d_images, image_stride, row_stride, channels, n, width, height));
  const EncIn in{d_images, image_stride, row_stride};
  return enc_chunks(c, "PNG", n, n, true, out, capacity, sizes, [&](int, int, int s) {
    return png_enqueue(c, s, in, n, width, height, o, channels);
  });
}

int bevk_png_encode(bevk_ctx* c, const void* d_images, int64_t image_stride, int64_t row_stride, int n, int width, int height,
                    uint8_t* out, uint64_t capacity, uint64_t* sizes) {
  NvtxRange nvtx_call("bevk_png_encode (device images -> host PNG streams)");
  RET(use(c));
  png::Opts o;
  png::normalise(c->png.params.data(), (int)c->png.params.size(), &o);   // bevk_png_set_params checked the list
  return png_encode_images(c, o, d_images, image_stride, row_stride, 3, n, width, height, out, capacity, sizes);
}

// The parameter list per call, as cv2.imencode takes it; also zlib's hash-chain parse at levels 4..9 (deflate_slow,
// bevk_png_enc.cuh).  The ctx's bevk_png_set_params list is neither read nor changed.
int bevk_png_encode_params(bevk_ctx* c, const int* params, int n_params, const void* d_images, int64_t image_stride,
                           int64_t row_stride, int n, int width, int height, uint8_t* out, uint64_t capacity,
                           uint64_t* sizes) {
  NvtxRange nvtx_call("bevk_png_encode_params (device images -> host PNG streams)");
  return bevk_png_encode_channels(c, params, n_params, d_images, image_stride, row_stride, 3, n, width, height, out,
                                  capacity, sizes);
}

int bevk_png_encode_channels(bevk_ctx* c, const int* params, int n_params, const void* d_images, int64_t image_stride,
                             int64_t row_stride, int channels, int n, int width, int height, uint8_t* out, uint64_t capacity,
                             uint64_t* sizes) {
  NvtxRange nvtx_call("bevk_png_encode_channels (device images -> host PNG streams)");
  RET(use(c));
  png::Opts o;
  RET(png_params_check(params, n_params, &o, true));
  return png_encode_images(c, o, d_images, image_stride, row_stride, channels, n, width, height, out, capacity, sizes);
}

// ------------------------------------------------------------------ CUDA graphs
// Stream capture of whatever the device-pointer entry points enqueue between begin and end; replayed with one call.
int bevk_graph_begin(bevk_ctx* c) {
  RET(use(c));
  if (c->capturing) return fail(BEVK_ERR_ARG, "a capture is already open on this context");
  CU(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
  c->capturing = true;
  c->capture_launches0 = c->launches;
  return BEVK_OK;
}

int bevk_graph_end(bevk_ctx* c, int* graph_id) {
  RET(use(c));
  if (!c->capturing) return fail(BEVK_ERR_ARG, "bevk_graph_begin was not called");
  c->capturing = false;
  bevk_ctx::Graph g;
  cudaError_t e = cudaStreamEndCapture(c->stream, &g.g);
  if (e != cudaSuccess || !g.g) {
    cudaGetLastError();
    return fail(BEVK_ERR_CUDA, "stream capture failed (%s): a call inside the capture allocated or synchronised -- run the same "
                               "calls once before capturing so that every buffer and table exists", cudaGetErrorString(e));
  }
  e = cudaGraphInstantiate(&g.x, g.g, 0);
  if (e != cudaSuccess) { cudaGraphDestroy(g.g); return fail(BEVK_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(e)); }
  g.kernels = c->launches - c->capture_launches0;
  c->launches = c->capture_launches0;            // nothing ran yet: replays are counted by bevk_graph_launch
  size_t slot = 0;
  while (slot < c->graphs.size() && c->graphs[slot].x) ++slot;
  if (slot == c->graphs.size()) c->graphs.push_back(g); else c->graphs[slot] = g;
  if (graph_id) *graph_id = (int)slot;
  return BEVK_OK;
}

int bevk_graph_launch(bevk_ctx* c, int graph_id, int times) {
  RET(use(c));
  if (graph_id < 0 || (size_t)graph_id >= c->graphs.size() || !c->graphs[graph_id].x) return fail(BEVK_ERR_ARG, "no graph %d", graph_id);
  if (times < 1) return fail(BEVK_ERR_ARG, "times must be >= 1");
  if (c->capturing) return fail(BEVK_ERR_ARG, "cannot launch a graph inside a capture");
  for (int i = 0; i < times; ++i) CU(cudaGraphLaunch(c->graphs[graph_id].x, c->stream));
  c->launches += (long long)times * c->graphs[graph_id].kernels;
  return BEVK_OK;
}

int bevk_graph_destroy(bevk_ctx* c, int graph_id) {
  RET(use(c));
  if (graph_id < 0 || (size_t)graph_id >= c->graphs.size() || !c->graphs[graph_id].x) return fail(BEVK_ERR_ARG, "no graph %d", graph_id);
  CU(cudaStreamSynchronize(c->stream));
  cudaGraphExecDestroy(c->graphs[graph_id].x);
  cudaGraphDestroy(c->graphs[graph_id].g);
  c->graphs[graph_id] = bevk_ctx::Graph();
  return BEVK_OK;
}

int64_t bevk_launch_count(bevk_ctx* c) { return c ? c->launches : 0; }

int bevk_last_kernel_ms(bevk_ctx* c, float* ms) {
  RET(use(c));
  if (!ms) return fail(BEVK_ERR_ARG, "null ms");
  if (!c->timed) return fail(BEVK_ERR_ARG, "no timed bevk_bev_run_device, bevk_jpeg_encode or bevk_png_encode call yet");
  CU(cudaEventSynchronize(c->ev1));
  CU(cudaEventElapsedTime(ms, c->ev0, c->ev1));
  return BEVK_OK;
}

