/* bevk.h -- C ABI of libbevk.so, the H100 (sm_90a) surround-BEV warping engine.
 *
 * Drop-in boundary for the per-pixel hot path of dyfcalid/CameraCalibration.  The
 * reference has no FFI of its own (it is pure Python over OpenCV); each entry
 * point below replaces the OpenCV call(s) the reference makes at the cited
 * file:line (paths relative to the reference tree).  INTEGRATION.md shows the
 * ctypes binding a maintainer of the reference would add.
 *
 * Conventions
 *   - plain C, no torch / C++ types; every call returns 0 on success or a negative
 *     bevk_status; bevk_last_error() gives the thread-local message.
 *   - images are uint8, interleaved channels (BGR as cv2.imread gives), row-major,
 *     explicit row stride in bytes.  3x3 matrices are row-major double[9].
 *   - "host" entry points take host pointers and do H2D / D2H inside the call;
 *     "_device" entry points take device pointers on the ctx's device and only
 *     enqueue work on the ctx stream (no synchronisation).
 *   - the caller owns every buffer it passes in (inputs and outputs).
 *   - a ctx is not thread-safe; use one ctx per thread.  No CPU fallback exists:
 *     without a CUDA device bevk_ctx_create fails.
 */
#ifndef BEVK_H
#define BEVK_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct bevk_ctx bevk_ctx;

typedef enum {
  BEVK_OK = 0,
  BEVK_ERR_ARG = -1,         /* bad argument / call order                       */
  BEVK_ERR_CUDA = -2,        /* CUDA runtime error (message has the details)    */
  BEVK_ERR_OOM = -3,
  BEVK_ERR_UNSUPPORTED = -4
} bevk_status;

enum { BEVK_INTER_NEAREST = 0, BEVK_INTER_LINEAR = 1 };          /* cv2.INTER_* values */
enum { BEVK_MAPS_UNDISTORT = 0, BEVK_MAPS_BEV = 1 };
enum { BEVK_MODEL_FISHEYE = 0, BEVK_MODEL_PINHOLE = 1 };
/* bevk_bev_run flags.  BEVK_FLAG_NV12 / BEVK_FLAG_I420 (exclusive; they combine with BALANCE) say the frames are YUV
 * 4:2:0 in cv2's single-buffer layout, uint8[frame_h*3/2][frame_w] (frame_w, frame_h even, else BEVK_ERR_UNSUPPORTED):
 * the Y plane, then NV12: interleaved U,V rows; I420: the U plane, then the V plane, each frame_w/2 x frame_h/2 and
 * packed (two chroma rows per buffer row).  The result is byte for byte cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 /
 * COLOR_YUV2BGR_I420) followed by the BGR call.  Accepted by bevk_bev_run, bevk_bev_run_stack and
 * bevk_bev_host_copy_bytes, and required by bevk_bev_run_yuv_planes / _surfaces (frames as separate, pitched planes);
 * every other entry point with flags refuses them with BEVK_ERR_UNSUPPORTED.
 * BEVK_FLAG_OUT_NV12 / BEVK_FLAG_OUT_I420 (exclusive: both is BEVK_ERR_ARG; they combine with BALANCE, the car and the
 * input flags) say the canvases are written as YUV 4:2:0: canvas b is the dense uint8[bev_h*3/2][bev_w] at
 * out + b * bev_w*bev_h*3/2 (bev_w, bev_h even, else BEVK_ERR_UNSUPPORTED, as cv2 refuses odd sizes), whose bytes are
 * cv2.cvtColor(bgr, COLOR_BGR2YUV_I420) of the BGR canvas `bgr` the same call writes without the flag (OUT_NV12: the
 * same Y plane, then the U and V planes interleaved).  The conversion runs on the device, so only 1.5 bytes per canvas
 * pixel leave it.  Accepted by bevk_bev_run, bevk_bev_run_device, bevk_bev_run_frames, bevk_bev_run_stack and
 * bevk_bev_host_copy_bytes; every other entry point with flags refuses them with BEVK_ERR_UNSUPPORTED.
 * BEVK_FLAG_YUYV / BEVK_FLAG_UYVY say the frames are packed YUV 4:2:2 as UVC / V4L2 and GMSL cameras deliver them,
 * uint8[frame_h][frame_w][2] (cv2's input shape for these codes; frame_w even, else BEVK_ERR_UNSUPPORTED; frame_h may be
 * odd): each row holds pixel pairs of 4 bytes, YUYV: Y0 U0 Y1 V0, UYVY: U0 Y0 V0 Y1, and both pixels of a pair take its
 * U and V.  The result is byte for byte cv2.cvtColor(frame, COLOR_YUV2BGR_YUY2 / COLOR_YUV2BGR_UYVY) followed by the BGR
 * call.  They are accepted wherever the NV12 / I420 flags are and combine with the same flags; the plane entry points
 * take one plane (offset[0] / plane 0, pitch[0] >= 2 * frame_w; entries 1 and 2 are not read).  Any two of the four input
 * flags together are BEVK_ERR_ARG. */
enum { BEVK_FLAG_BALANCE = 1, BEVK_FLAG_NV12 = 2, BEVK_FLAG_I420 = 4, BEVK_FLAG_OUT_NV12 = 8, BEVK_FLAG_OUT_I420 = 16,
       BEVK_FLAG_YUYV = 32, BEVK_FLAG_UYVY = 64 };
#define BEVK_MAX_CAMERAS 8

int bevk_version(void);
const char *bevk_last_error(void);

/* ---- context ------------------------------------------------------------- */
int bevk_ctx_create(int device, bevk_ctx **out);
int bevk_ctx_destroy(bevk_ctx *ctx);
/* Run on an externally owned cudaStream_t (e.g. torch's current stream); NULL
 * restores the ctx's own stream. */
int bevk_ctx_set_stream(bevk_ctx *ctx, void *cuda_stream);
int bevk_ctx_sync(bevk_ctx *ctx);
/* PCI bus id ("0000:1b:00.0") of a CUDA device: lets a multi-process launcher bind each rank to the CPUs and memory
 * of its GPU's NUMA node (/sys/bus/pci/devices/<id>/local_cpulist) before it allocates page-locked buffers. */
int bevk_device_pci_bus_id(int device, char *out, int len);
/* Pinned host memory for callers who want full-rate PCIe copies. */
int bevk_host_alloc(uint64_t bytes, void **out);
int bevk_host_free(void *p);

/* ---- K1: undistortion maps ------------------------------------------------
 * cv2.fisheye.initUndistortRectifyMap(K, D, eye(3), P, (w,h), CV_16SC2)
 *   SurroundBirdEyeView/surroundBEV.py:98-103, Tools/undistort.py:50-52,
 *   IntrinsicCalibration/intrinsicCalib.py:98-103            (model FISHEYE, 4 coeffs)
 * cv2.initUndistortRectifyMap(K, D5, eye(3), P, (w,h), CV_16SC2)
 *   IntrinsicCalibration/intrinsicCalib.py:158-163           (model PINHOLE, 5 coeffs)
 * map1: int16[h][w][2] (x,y integer part), map2: uint16[h][w] (fy*32+fx).        */
int bevk_undistort_map(bevk_ctx *ctx, int model, const double K[9], const double *D, int n_dist,
                       const double P[9], int w, int h, int16_t *map1, uint16_t *map2);

/* ---- K3: cv2.remap(src, map1, map2, interp), BORDER_CONSTANT 0 --------------
 *   surroundBEV.py:110-111,116-117; undistort.py:66; intrinsicCalib.py:193-195
 * channels in {1,3,4}; map2 may be NULL for NEAREST with integer maps.          */
int bevk_remap(bevk_ctx *ctx, const uint8_t *src, int sw, int sh, int64_t sstride, int channels,
               const int16_t *map1, const uint16_t *map2, int dw, int dh,
               uint8_t *dst, int64_t dstride, int interp);

/* ---- cached-map undistortion (the per-frame call of InCalibrator.undistort /
 * Camera.undistort / Tools/undistort.py's loop).  The map is built on the device
 * once per "slot" and never leaves HBM; each frame is one H2D, one gather kernel,
 * one D2H.  fused!=0 skips the map entirely and evaluates the camera model inside
 * the gather kernel (no 6 B/px map traffic; same results).                      */
int bevk_undistorter_set(bevk_ctx *ctx, int slot, int model, const double K[9], const double *D, int n_dist,
                         const double P[9], int dw, int dh, int fused);
int bevk_undistorter_maps(bevk_ctx *ctx, int slot, int16_t *map1, uint16_t *map2);   /* D2H, for parity tests */
/* dw x dh: the destination size the caller allocated; must equal the slot's map size (checked, so a stale handle to
 * a slot that was re-set can never make the library write past dst). */
int bevk_undistort(bevk_ctx *ctx, int slot, const uint8_t *src, int sw, int sh, int64_t sstride, int channels,
                   uint8_t *dst, int dw, int dh, int64_t dstride, int interp);
/* n DEVICE frames (frame i at d_src + i*src_image_stride, rows src_row_stride apart, channels 1/3/4) undistorted
 * through the slot's map or fused model into n DEVICE images (dst_image_stride / dst_row_stride, dw x dh = the slot's
 * size, checked).  Each output pixel's taps are resolved once (map read or camera model) for several frames.  Row
 * strides must cover a row, image strides (read when n > 1) an image; a destination range that overlaps the source
 * range is refused.  3-channel INTER_LINEAR with dw % 4 == 0 takes the 4-pixel word path when both base pointers, both
 * row strides and (n > 1) both image strides are multiples of 4; otherwise the byte path.  Only enqueues on the ctx
 * stream; no allocation or synchronisation, so it can be graph-captured. */
int bevk_undistort_stack(bevk_ctx *ctx, int slot, const void *d_src, int64_t src_image_stride, int sw, int sh,
                         int64_t src_row_stride, int channels, int n, void *d_dst, int64_t dst_image_stride,
                         int dw, int dh, int64_t dst_row_stride, int interp);
/* Which gather the last undistort call (or bevk_remap / bevk_warp_perspective) launched: 4 = k_gather4 (word path),
 * 1 = k_gather (byte path), 0 = none yet. */
int bevk_undistort_last_path(bevk_ctx *ctx);

/* ---- K4: cv2.warpPerspective(src, H, (dw,dh), flags=interp), border 0 --------
 *   ExtrinsicCalibration/extrinsicCalib.py:166-169, surroundBEV.py:113-114      */
int bevk_warp_perspective(bevk_ctx *ctx, const uint8_t *src, int sw, int sh, int64_t sstride, int channels,
                          const double H[9], uint8_t *dst, int dw, int dh, int64_t dstride, int interp);
/* The same call applied to a 16SC2 / 16UC1 map pair (Camera.get_bev_maps,
 * surroundBEV.py:105-108): float-table bilinear, rounded, saturated.            */
int bevk_warp_maps(bevk_ctx *ctx, const int16_t *map1, const uint16_t *map2, int sw, int sh,
                   const double H[9], int dw, int dh, int16_t *out1, uint16_t *out2);

/* ---- the BEV engine (BevGenerator, surroundBEV.py:282-325) ----------------- */
/* frames up to 32767 px a side, canvases up to 65536 (BEVK_ERR_UNSUPPORTED beyond) */
int bevk_bev_configure(bevk_ctx *ctx, int n_cam, int frame_w, int frame_h, int bev_w, int bev_h);
/* Camera.__init__ (surroundBEV.py:82-108): K, D, P = camera_mat_dst, undistorted
 * size (und_w x und_h) and H.  Builds the camera's BEV LUT on the device with the
 * reference's semantics (the undistortion maps themselves warped by H, SURVEY A4)
 * without materialising the und_w x und_h intermediate map.                      */
int bevk_bev_set_camera(bevk_ctx *ctx, int cam, const double K[9], const double D[4], const double P[9],
                        int und_w, int und_h, const double H[9]);
/* Inject / read back a camera's BEV maps (int16[bev_h][bev_w][2], uint16[bev_h][bev_w]). */
int bevk_bev_set_maps(bevk_ctx *ctx, int cam, const int16_t *map1, const uint16_t *map2);
int bevk_bev_get_maps(bevk_ctx *ctx, int cam, int16_t *map1, uint16_t *map2);
/* Mask / BlendMask (surroundBEV.py:119-162, 164-280): uint8[bev_h][bev_w]; 0/255 for
 * the plain path, 0..255 blend weights otherwise (weight = float32(mask/255.0)). */
int bevk_bev_set_mask(bevk_ctx *ctx, int cam, const uint8_t *mask);
/* Interpolation of raw2bev's cv2.remap (surroundBEV.py:116-117 uses INTER_LINEAR; INTER_NEAREST is
 * offered with cv2.remap's exact fixed-point-map semantics).  Call before bevk_bev_finalize. */
int bevk_bev_set_interpolation(bevk_ctx *ctx, int interp);
/* BlendMask.get_blend_mask (surroundBEV.py:270-277) for the 4-camera layout, on the
 * device: polys = the four *unblended* 6-gon masks (uint8[4][bev_h][bev_w], order
 * front,back,left,right), lines = the 8 seam segments FL,FR,BL,BR,LF,LB,RF,RB as
 * int32[8][2][2].  Writes the four blend masks to out (same layout as polys).     */
int bevk_blend_masks(bevk_ctx *ctx, const uint8_t *polys, const int32_t *lines, int bev_w, int bev_h, uint8_t *out);
/* Compile LUTs + masks into the tile plan the fused kernel consumes. */
int bevk_bev_finalize(bevk_ctx *ctx);

/* BevGenerator.__call__ (surroundBEV.py:312-325) for `batch` frame-sets.
 * srcs: batch*n_cam host pointers (frame-set major: set0 cam0..camN-1, set1 ...),
 *       each uint8[frame_h][frame_w][3] with row stride src_stride bytes.
 * car : NULL or uint8[bev_h][bev_w][3] (dense), added after colour balance.
 * out : batch canvases uint8[bev_h][bev_w][3], dense, canvas b at out + b*bev_h*bev_w*3; with BEVK_FLAG_OUT_NV12 /
 *       _I420 uint8[bev_h*3/2][bev_w] at out + b*bev_w*bev_h*3/2, converted on the device, so only those bytes come back.
 * With BEVK_FLAG_NV12 / _I420 each frame is uint8[frame_h*3/2][frame_w] whose rows (Y and chroma alike) are
 * src_stride bytes apart.  Page-locked frames (frame_w and src_stride multiples of 16, no BALANCE) are read by the SMs
 * in the 16-byte windows around the sampled Y spans and the matching chroma bytes; pageable ones go up as the band
 * rectangles of the Y plane plus their chroma rows; with BALANCE whole frames.  On the device the sampled spans are
 * converted to BGR (and balanced) into a copy stack that the TMA-staged kernel renders from.
 * With BEVK_FLAG_YUYV / _UYVY each frame is uint8[frame_h][frame_w][2], rows src_stride bytes apart: page-locked frames
 * (2 * frame_w and src_stride multiples of 16, no BALANCE) bring the 16-byte windows around the sampled spans, pageable
 * ones the band rectangles widened to whole pixel pairs, BALANCE whole frames (2 bytes per pixel). */
int bevk_bev_run(bevk_ctx *ctx, const uint8_t *const *srcs, int64_t src_stride, int batch,
                 const uint8_t *car, int flags, uint8_t *out);
/* Device-resident variant: d_srcs is a DEVICE array of batch*n_cam device pointers
 * (dense frames, row stride frame_w*3); d_car NULL or device; d_out device.  Only
 * enqueues on the ctx stream.                                                    */
int bevk_bev_run_device(bevk_ctx *ctx, const void *d_srcs, int batch, const void *d_car, int flags, void *d_out);
/* Same with the table on the HOST: frames[batch*n_cam] are DEVICE pointers to dense frames (e.g. the
 * data pointers of torch / CuPy / NVDEC buffers; 4-byte aligned).  The library keeps the device copy of
 * the table and re-uploads it only when its contents change, so streaming into fixed buffers costs no
 * copy per call.  Replaces the host frames of BevGenerator.__call__ (surroundBEV.py:312-325) when the
 * decoder already left them on the GPU (SURVEY 8f-2).  Only enqueues on the ctx stream.             */
int bevk_bev_run_frames(bevk_ctx *ctx, const void *const *frames, int batch, const void *d_car, int flags, void *d_out);
/* Frame STACK on the device: frame i (= frame-set i / n_cam, camera i % n_cam) is the dense uint8[frame_h][frame_w][3]
 * at d_frames + i * frame_stride -- e.g. one uint8[batch][n_cam][H][W][3] tensor, or a decoder's surface pool.
 * Replaces the frames of BevGenerator.__call__ (surroundBEV.py:312-325, the cv2.remap inputs of :116-117).  With a
 * 16-byte aligned base and stride (and a row pitch frame_w*3 that is a multiple of 16) the TMA-staged kernel runs:
 * per (canvas tile, camera) one cp.async.bulk.tensor box per frame-set into shared memory; otherwise the
 * pointer-table gather.  bevk_bev_run_frames takes this path by itself when its table describes a stack, and so
 * does bevk_bev_run for its staging buffers.  Only enqueues on the ctx stream.
 * With BEVK_FLAG_NV12 / _I420 frame i is the dense uint8[frame_h*3/2][frame_w] YUV frame at d_frames + i * frame_stride
 * (any base and any stride >= frame_w * frame_h * 3/2); its sampled spans are converted on the device into a 16-byte
 * friendly BGR copy stack, so the TMA-staged kernel renders them whenever a TMA plan exists.  Still only enqueues, so
 * it can be captured into a graph (after one eager call of the same shape).  The same holds with BEVK_FLAG_OUT_NV12 /
 * _I420 (here and in bevk_bev_run_device / _frames): the BGR canvases are rendered into library scratch and converted
 * from there into d_out (any alignment).  With BEVK_FLAG_YUYV / _UYVY frame i is the dense uint8[frame_h][frame_w][2]
 * packed frame at d_frames + i * frame_stride (any base and any stride >= frame_w * frame_h * 2).                     */
int bevk_bev_run_stack(bevk_ctx *ctx, const void *d_frames, int64_t frame_stride, int batch, const void *d_car, int flags,
                       void *d_out);
/* YUV 4:2:0 frames as a video decoder leaves them on the device (NVDEC / DeepStream surfaces, FFmpeg CUDA frames'
 * data[] / linesize[]): each plane at its own address, rows padded to their own pitch.  Plane p of frame i (= frame-set
 * i / n_cam, camera i % n_cam): p = 0 Y (frame_w bytes a row), 1 interleaved U,V (NV12, frame_w bytes) or U (I420,
 * frame_w/2), 2 V (I420, frame_w/2; not read for NV12); row r of it at <plane address> + r * pitch[p], with pitch[p] >=
 * the plane's row bytes.  Pixels within a row are dense.  cv2's single buffer is the case offset = {0, w*h, w*h*5/4},
 * pitch = {w, w/2, w/2} (I420), or offset = {0, w*h}, pitch = {w, w} (NV12).  Needs BEVK_FLAG_NV12 or _I420 (frame_w, frame_h even); combines
 * with BALANCE, the car and BEVK_FLAG_OUT_*; the result is that of bevk_bev_run_stack on the same frames repacked
 * densely, with no repack: only the bytes the conversion samples are read (any base, offset, pitch or stride; odd ones
 * cost byte loads instead of word loads).  Refused with BEVK_ERR_ARG, nothing enqueued: no YUV flag or both, a pitch
 * below its plane's row bytes, a null plane, batch * n_cam > 65535.  With BEVK_FLAG_YUYV / _UYVY a frame is the one
 * packed plane 0 (rows of 2 * frame_w bytes, pitch[0] >= that); offset / pitch / plane entries 1 and 2 are not read.
 * Only enqueues on the ctx stream, so it can be
 * captured into a graph (after one eager call of the same shape).
 * Surface pool: plane p of frame i at d_base + i * frame_stride + offset[p] (a plane may lie before d_base's Y plane). */
int bevk_bev_run_yuv_planes(bevk_ctx *ctx, const void *d_base, int64_t frame_stride, const int64_t offset[3],
                            const int64_t pitch[3], int batch, const void *d_car, int flags, void *d_out);
/* Scattered surfaces: planes[3*i + p] is the DEVICE address of plane p of frame i (a HOST array of batch*n_cam*3
 * pointers; the V entries of NV12 are not read).  The library keeps a device copy of the table and uploads it again only
 * when its contents change, as bevk_bev_run_frames does. */
int bevk_bev_run_yuv_surfaces(bevk_ctx *ctx, const void *const *planes, const int64_t pitch[3], int batch, const void *d_car,
                              int flags, void *d_out);
/* Per-camera partial canvases for camera-sharded multi-GPU runs: rank r renders only
 * cameras [cam_lo, cam_hi) into d_out (zero elsewhere); the saturating sum of the
 * ranks' partials equals the full canvas (balance is not supported in this mode). */
int bevk_bev_run_device_cams(bevk_ctx *ctx, const void *d_srcs, int batch, int cam_lo, int cam_hi, void *d_out);
/* The same over a frame stack (see bevk_bev_run_stack). */
int bevk_bev_run_stack_cams(bevk_ctx *ctx, const void *d_frames, int64_t frame_stride, int batch, int cam_lo, int cam_hi,
                            void *d_out);
/* Saturating sum of n partial canvases (device), optional car, into d_out. */
int bevk_sat_sum_device(bevk_ctx *ctx, const void *const *d_parts_host_array, int n, uint64_t bytes,
                        const void *d_car, void *d_out);

/* ---- stand-alone forms of the reference's per-pixel helpers ----------------------
 * Mask.__call__ / BlendMask.__call__ (surroundBEV.py:161-162, 279-280): dense BGR image
 * uint8[h][w][3], mask uint8[h][w]; blend=0: mask ? px : 0, blend=1: trunc(px*f32(mask/255)). */
int bevk_apply_mask(bevk_ctx *ctx, const uint8_t *img, const uint8_t *mask, int w, int h, int blend, uint8_t *out);
/* color_balance (surroundBEV.py:43-55) of one dense BGR image. */
int bevk_color_balance(bevk_ctx *ctx, const uint8_t *img, int w, int h, uint8_t *out);
/* luminance_balance (surroundBEV.py:57-79) of n (<= 8) dense BGR frames of equal size. */
int bevk_luminance_balance(bevk_ctx *ctx, const uint8_t *const *imgs, int n, int w, int h, uint8_t *const *outs);

/* Introspection for tests / bench */
int bevk_bev_plan_info(bevk_ctx *ctx, int64_t *n_tiles, int64_t *n_items, int64_t *lut_bytes);
/* Bytes bevk_bev_run moves over PCIe per frame-set for the given flags: host->device (without
 * BALANCE only the rectangle of each frame its camera's LUT can sample is uploaded; with BALANCE
 * the whole frames, because the V means cover them) and device->host (the canvas).  With a YUV
 * flag: the Y rectangles and their chroma rows (1.5 bytes per pixel; YUYV / UYVY: the rectangles at 2 bytes per
 * pixel), or whole YUV frames.  With an
 * output flag the canvas is bev_w*bev_h*3/2 bytes. */
int bevk_bev_host_copy_bytes(bevk_ctx *ctx, int flags, int64_t *h2d_per_frame_set, int64_t *d2h_per_frame_set);
/* Host->device bytes the last bevk_bev_run call actually moved (page-locked frames are ingested span
 * by span by the SMs, pageable ones by DMA rectangles, BALANCE uploads whole frames). */
int64_t bevk_bev_last_h2d_bytes(bevk_ctx *ctx);
/* Which fused kernel the last BEV call launched: 1 = k_bev (pointer-table gather), 2 = k_bev_tma (TMA-staged). */
int bevk_bev_last_path(bevk_ctx *ctx);
/* The TMA-staged kernel's plan: work items, tensor-map box shapes, bytes one frame-set's boxes deliver, LUT entries
 * served from staged boxes / by global gathers.  All zero when the plan does not exist (row pitch not a multiple of
 * 16 bytes, or BEVK_TMA=0). */
int bevk_bev_tma_plan_info(bevk_ctx *ctx, int64_t *n_items, int64_t *n_shapes, int64_t *box_bytes, int64_t *tma_entries,
                           int64_t *gather_entries);
/* ---- multi-GPU sharding: one process (one ctx) per GPU ---------------------------------------------------
 * The reference is a single process (no collective anywhere); the path shards two ways:
 *   BEVK_SHARD_FRAMES   every rank renders its own frame-sets with a replica of the plan -- no exchange at all;
 *   BEVK_SHARD_CAMERAS  rank r renders cameras [lo_r, hi_r) (contiguous blocks) of EVERY frame-set into a slab -- the
 *                       tile-aligned bounding box of the union of their masks -- ONE ncclAllGather moves the slabs
 *                       over NVLink, and each rank composes them with the saturating sum, which is exact because
 *                       the cv2.add chain of BevGenerator.__call__ (surroundBEV.py:316-320) is order-independent.
 * NCCL is dlopen'ed (libnccl.so.2) on first use.  Call order: bevk_bev_finalize, bevk_shard_configure on every rank,
 * bevk_shard_unique_id on ONE rank, its 128 bytes carried to the others by the launcher (file, MPI, torch.distributed),
 * bevk_shard_connect on every rank, then bevk_bev_run_sharded per step.  All work is enqueued on the ctx stream. */
enum { BEVK_SHARD_FRAMES = 0, BEVK_SHARD_CAMERAS = 1 };
int bevk_shard_configure(bevk_ctx *ctx, int policy, int rank, int world);
int bevk_shard_unique_id(void *id128, int len);
int bevk_shard_connect(bevk_ctx *ctx, const void *id128, int len);
/* Partition and slab geometry of `rank`: its cameras [cam_lo, cam_hi), its slab rectangle {x0, y0, x1, y1} in canvas
 * pixels, and the (padded, equal for all ranks) bytes of one frame-set's slab. */
int bevk_shard_info(bevk_ctx *ctx, int rank, int *cam_lo, int *cam_hi, int32_t rect[4], int64_t *slab_bytes);
/* BevGenerator.__call__ over a frame stack (see bevk_bev_run_stack) under the configured policy.  CAMERAS: every rank
 * passes the same batch; only the frames of its own cameras are read; every rank ends with all canvases in d_out.
 * BEVK_FLAG_BALANCE under CAMERAS: each rank sums V over its own cameras' frames, one all-gather of those sums
 * (world x batch x n_cam uint64) gives every rank the luminance offsets of every camera, each rank balances and renders
 * its own cameras, and colour balance (then the car) runs on the composed canvases.  The result is byte-identical to
 * the single-GPU BALANCE render; batch x n_cam <= 65535. */
int bevk_bev_run_sharded(bevk_ctx *ctx, const void *d_frames, int64_t frame_stride, int batch, const void *d_car, int flags,
                         void *d_out);
/* CAMERAS policy, fused compute + exchange: frame-set b is OWNED by rank b % world.  Every rank renders its cameras'
 * slabs of all frame-sets and the fused kernel's write-out stores each slab straight into the owner's receive buffer
 * over NVLink (peer memory mapped with CUDA IPC); one 4-byte all-gather per step is the barrier, then each rank composes
 * the canvases it owns (d_out_own[*n_own][bev_h][bev_w][3], frame-sets rank, rank+world, ...).  Per step a rank sends
 * (and receives) (world-1)/world of one slab set, instead of receiving world-1 whole slab sets as the all-gather does.
 * Setup after bevk_shard_connect: bevk_shard_prepare(batch) on every rank gives a 64-byte handle; the launcher gathers
 * the handles of all ranks (rank order, world x 64 bytes) and gives them to bevk_shard_attach.  Frames must be a
 * 16-byte friendly stack (the TMA-staged kernel does the stores).  BEVK_FLAG_BALANCE works as in bevk_bev_run_sharded:
 * the V-sum all-gather comes first, and each rank colour-balances the canvases it owns. */
int bevk_shard_prepare(bevk_ctx *ctx, int batch, void *handle64);
int bevk_shard_attach(bevk_ctx *ctx, const void *handles);
int bevk_bev_run_scattered(bevk_ctx *ctx, const void *d_frames, int64_t frame_stride, int batch, const void *d_car, int flags,
                           void *d_out_own, int *n_own);
/* Bytes this rank received (all-gather) or stored into its peers (scattered) over NVLink in the last sharded call. */
int64_t bevk_shard_last_link_bytes(bevk_ctx *ctx);
/* The two halves of the CAMERAS policy on their own (tests, custom exchanges): render the slabs of rank `as_rank`
 * into d_slabs[as_rank][batch][slab_bytes]; compose d_slabs[world][batch][slab_bytes] (+ car) into canvases. */
int bevk_shard_render(bevk_ctx *ctx, const void *d_frames, int64_t frame_stride, int batch, int as_rank, void *d_slabs);
int bevk_shard_compose(bevk_ctx *ctx, const void *d_slabs, int batch, const void *d_car, void *d_out);
/* The BALANCE halves, in this order: bevk_shard_vsum writes block as_rank of d_vsums[world][batch][n_cam] (8-byte
 * aligned): the V sums of rank as_rank's own cameras, zero in the other columns.  Once every block is there (an
 * all-gather, or every rank on one GPU), bevk_shard_render_balanced renders rank as_rank's balanced slabs and
 * bevk_shard_compose_balanced composes, colour-balances and adds the car.  Only enqueue; batch x n_cam <= 65535. */
int bevk_shard_vsum(bevk_ctx *ctx, const void *d_frames, int64_t frame_stride, int batch, int as_rank, uint64_t *d_vsums);
int bevk_shard_render_balanced(bevk_ctx *ctx, const void *d_frames, int64_t frame_stride, int batch, int as_rank,
                               const uint64_t *d_vsums, void *d_slabs);
int bevk_shard_compose_balanced(bevk_ctx *ctx, const void *d_slabs, int batch, const void *d_car, void *d_out);

/* ---- JPEG ingest on the device ------------------------------------------------------------------------------
 * Replaces cv2.imread in front of the path (surroundBEV.py:328-332, Tools/undistort.py:65): n baseline JPEG streams
 * (host memory) are decoded by nvJPEG (dlopen'ed on first use) into frames 0..n-1 of a device frame stack, BGR
 * interleaved, row pitch width*3 -- the layout bevk_bev_run_stack and bevk_undistort_stack(_jpeg) read.  Only the
 * compressed bytes cross PCIe.  Every stream must decode to width x height.  The pixels are nvJPEG's, which differ from
 * libjpeg-turbo's (cv2) by the decoders' IDCT / upsampling rounding; everything downstream is bit-exact on them.
 * The Huffman stage runs on the calling thread; GPU work is enqueued on the ctx stream. */
int bevk_jpeg_decode(bevk_ctx *ctx, const uint8_t *const *jpegs, const uint64_t *sizes, int n, int width, int height,
                     void *d_frames, int64_t frame_stride);

/* BevGenerator.__call__ (surroundBEV.py:312-325) on JPEG streams: jpegs[batch*n_cam] in frame-set-major order as in
 * bevk_bev_run; decoded on the device, rendered, canvases copied to `out` (host).  Synchronises. */
int bevk_bev_run_jpeg(bevk_ctx *ctx, const uint8_t *const *jpegs, const uint64_t *sizes, int batch, const uint8_t *car, int flags,
                      uint8_t *out);

/* ---- JPEG encode on the device ------------------------------------------------------------------------------------
 * Replaces cv2.imwrite(path, img, [IMWRITE_JPEG_QUALITY, q]) at the end of the path (Tools/undistort.py:72-73,
 * surroundBEV.py:340): the streams are byte-identical to cv2's (libjpeg-turbo baseline: islow DCT, JFIF 1.01 header;
 * by default 4:2:0, Annex K Huffman tables and no restart markers, otherwise as bevk_jpeg_set_params says), and only
 * the compressed bytes cross PCIe.
 * bevk_jpeg_encode_bound: the largest stream a width x height image can produce (sizes the caller's buffer) with no
 * params set.  4:4:4, optimised and restart-marker streams can be larger: size buffers for params with
 * bevk_jpeg_encode_bound_params.                                                                                     */
int bevk_jpeg_encode_bound(int width, int height, uint64_t *bytes);
/* cv2.imwrite's JPEG (key, value) pairs, n ints (n even), applied to every encoding call of this ctx (bevk_jpeg_encode,
 * bevk_undistort_jpeg, bevk_undistort_stack_jpeg, bevk_bev_run_to_jpeg, bevk_bev_frames_to_jpeg) until the next call;
 * n == 0 restores cv2's defaults.  Keys 2..7 as cv2.IMWRITE_JPEG_*, values normalised as cv2 does:
 *   SAMPLING_FACTOR (7)  0x111111 4:4:4, 0x211111 4:2:2, 0x121111 4:4:0, 0x221111 4:2:0, 0x411111 4:1:1; else 4:2:0
 *   LUMA_QUALITY (5)     >= 0: min(v, 100) replaces the call's quality (both tables unless CHROMA_QUALITY is given)
 *   CHROMA_QUALITY (6)   >= 0 and LUMA_QUALITY given: the chroma table's quality; luma != chroma forces 4:4:4
 *   OPTIMIZE (3)         != 0: per-image Huffman tables (libjpeg's jpeg_gen_optimal_table), built on the device
 *   RST_INTERVAL (4)     clamped to [0, 65535] MCUs; > 0 writes DRI and an RSTn marker after every interval but the last
 *   PROGRESSIVE (2)      0 as cv2's default; anything else is BEVK_ERR_UNSUPPORTED (a multi-scan coder)
 * QUALITY (1) is refused (every encoding call takes quality itself), as are other keys and odd n (BEVK_ERR_ARG).  A
 * refused list leaves the ctx's params as they were.  The streams are byte-identical to
 * cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, quality] + params).                                               */
int bevk_jpeg_set_params(bevk_ctx *ctx, const int *params, int n);
/* bevk_jpeg_encode_bound for streams made under `params` (same list and rules).                                       */
int bevk_jpeg_encode_bound_params(int width, int height, const int *params, int n, uint64_t *bytes);
/* n DEVICE images, 3-channel BGR, image i at d_images + i * image_stride, rows row_stride bytes apart (any pitch >= 3 *
 * width).  quality is clamped as cv2 does (to [0, 100]; 0 acts as 1; cv2's default is 95).  The streams are written
 * back to back into HOST memory at out, their sizes to sizes[n]; the call synchronises.  When they need more than
 * capacity bytes the call fails with BEVK_ERR_ARG, still fills sizes[], and writes nothing to out.                    */
int bevk_jpeg_encode(bevk_ctx *ctx, const void *d_images, int64_t image_stride, int64_t row_stride, int n, int width, int height,
                     int quality, uint8_t *out, uint64_t capacity, uint64_t *sizes);
/* bevk_undistort (3 channels) followed by the encoder: Tools/undistort.py:65-73 (imread'ed frame -> remap -> imwrite)
 * without the undistorted image ever leaving the device.  Works with map and fused slots; capacity as above.          */
int bevk_undistort_jpeg(bevk_ctx *ctx, int slot, const uint8_t *src, int sw, int sh, int64_t sstride, int interp, int quality,
                        uint8_t *out, uint64_t capacity, uint64_t *size);
/* bevk_undistort_stack for n 3-channel DEVICE frames, encoded on the device: the streams are byte-identical to
 * cv2.imencode of the undistorted images, back to back in host `out`; sizes[n] is always filled; capacity rule as
 * bevk_bev_frames_to_jpeg (below), and the same chunk pipeline (BEVK_JPEG_CHUNK).  Synchronises; cannot be captured. */
int bevk_undistort_stack_jpeg(bevk_ctx *ctx, int slot, const void *d_src, int64_t src_image_stride, int sw, int sh,
                              int64_t src_row_stride, int n, int interp, int quality,
                              uint8_t *out, uint64_t capacity, uint64_t *sizes);

/* ---- BEV canvases straight to JPEG ----------------------------------------------------------------------------------
 * BevGenerator.__call__ then cv2.imencode('.jpg', surround, [IMWRITE_JPEG_QUALITY, quality]) (surroundBEV.py:312-325,
 * :340): each canvas is rendered into library scratch and encoded on the device, and only the streams (byte-identical to
 * cv2's) cross PCIe.  With BEVK_FLAG_BALANCE the encoder applies colour balance and the car as it loads the raw canvas.
 * Streams go back to back into host `out`, their sizes into sizes[batch], which is always filled for the whole batch.
 * Streams leave chunk by chunk, so when they need more than `capacity` bytes the call fails with BEVK_ERR_ARG after
 * `out` has received the whole streams of the leading frame-sets that fit; nothing is written at or past capacity.
 * quality is clamped as in bevk_jpeg_encode.  Both calls synchronise and cannot be captured into a graph.
 * bevk_bev_run_to_jpeg: `batch` HOST frame-sets laid out as in bevk_bev_run (same chunk pipeline and ingest).         */
int bevk_bev_run_to_jpeg(bevk_ctx *ctx, const uint8_t *const *srcs, int64_t src_stride, int batch, const uint8_t *car, int flags,
                         int quality, uint8_t *out, uint64_t capacity, uint64_t *sizes);
/* The same for DEVICE frames given as a host table of device pointers, as in bevk_bev_run_frames (a table that describes a
 * 16-byte friendly stack takes the TMA-staged kernel).  d_car NULL or device; work runs on the ctx stream.           */
int bevk_bev_frames_to_jpeg(bevk_ctx *ctx, const void *const *frames, int batch, const void *d_car, int flags, int quality,
                            uint8_t *out, uint64_t capacity, uint64_t *sizes);

/* ---- PNG encode on the device -------------------------------------------------------------------------------------
 * Replaces cv2.imwrite('x.png', img, params) / cv2.imencode('.png', ...) for 8-bit 3-channel BGR images: the streams are
 * byte-identical to cv2's (libpng 1.6 + zlib 1.2.11: colour type 2, IDAT chunks of 8192 bytes) and only the compressed
 * bytes cross PCIe.  cv2's defaults (SUB filter, zlib level 1, Z_RLE) and IMWRITE_PNG_STRATEGY_RLE / _HUFFMAN_ONLY are
 * reproduced by every entry; bevk_png_encode_params also reproduces zlib's hash-chain parse (deflate_slow) at levels 4..9
 * under the DEFAULT, FILTERED and FIXED strategies.
 * bevk_png_set_params: cv2.imwrite's PNG (key, value) pairs, n ints (n even), applied to bevk_png_encode on this ctx
 * until the next call; n == 0 restores cv2's defaults.  Keys 16..20 as cv2.IMWRITE_PNG_*, read in order as cv2 4.13 does:
 *   COMPRESSION (16)     clamped to [0, 9]; resets the strategy to DEFAULT and switches to adaptive filtering over all
 *                        five filters (libpng's heuristic); a STRATEGY after it sets the strategy again
 *   STRATEGY (17)        RLE (3) or HUFFMAN_ONLY (2); values outside 0..4 act as RLE
 *   FILTER (19)          NONE 8, SUB 16, UP 32, AVG 64, PAETH 128, FAST 56, ALL 248 (others act as SUB); overrides the
 *                        filters the level implies
 *   BILEVEL (18)         0 only
 * A list that ends at level 0, at the DEFAULT / FILTERED / FIXED strategy, or with BILEVEL != 0 or ZLIBBUFFER_SIZE (20)
 * is BEVK_ERR_UNSUPPORTED; other keys and odd n are BEVK_ERR_ARG.  A refused list leaves the ctx's params as they were.
 * bevk_png_encode_bound: the largest stream a width x height image can produce under `params` (every block at most its
 * filtered bytes + 5, plus zlib header and trailer, signature, IHDR, IDAT framing and IEND).
 * bevk_png_encode: n DEVICE images, image i at d_images + i * image_stride, rows row_stride bytes apart (any pitch >=
 * 3 * width; filtered size (3 * width + 1) * height below 2^31 - 2^16).  The streams are written back to back into HOST
 * memory at out, their sizes to sizes[n]; the call synchronises.  When they need more than capacity bytes the call fails
 * with BEVK_ERR_ARG, still fills sizes[], and writes nothing to out.                                                   */
int bevk_png_set_params(bevk_ctx *ctx, const int *params, int n);
int bevk_png_encode_bound(int width, int height, const int *params, int n, uint64_t *bytes);
int bevk_png_encode(bevk_ctx *ctx, const void *d_images, int64_t image_stride, int64_t row_stride, int n, int width, int height,
                    uint8_t *out, uint64_t capacity, uint64_t *sizes);
/* bevk_png_encode_params: bevk_png_encode with the (key, value) list given per call, as cv2.imencode takes it, read as
 * above except that a list ending at level 4..9 under the DEFAULT (0), FILTERED (1) or FIXED (4) strategy -- [16, 9],
 * cv2.imwrite's level 9 -- is taken too.  Level 0, levels 1..3 under those strategies (a STRATEGY 0 / 1 / 4 without a
 * COMPRESSION is level 1), BILEVEL != 0 and ZLIBBUFFER_SIZE are BEVK_ERR_UNSUPPORTED.  The same contract as
 * bevk_png_encode (the call synchronises, sizes[] always filled, nothing written past capacity, bevk_last_kernel_ms
 * covers it); the ctx's bevk_png_set_params list is neither read nor changed.  bevk_png_encode_bound(w, h, NULL, 0)
 * bounds its streams too: the bound does not depend on the parameters.  The hash-chain parse keeps about 50 bytes of
 * device memory per filtered byte of a group (up to 32 MB of filtered data, or one larger image) in the ctx until it
 * is destroyed: an image of 1.5 G filtered bytes needs about 75 GB and fails with BEVK_ERR_OOM where that is not free. */
int bevk_png_encode_params(bevk_ctx *ctx, const int *params, int n_params, const void *d_images, int64_t image_stride,
                           int64_t row_stride, int n, int width, int height, uint8_t *out, uint64_t capacity,
                           uint64_t *sizes);

/* ---- CUDA graphs over the device-pointer entry points ------------------------------------------------
 * Everything the "_device" / "_stack" / "_frames" entry points enqueue on the ctx stream between begin and end is
 * captured (stream capture) instead of executed, instantiated once, and replayed `times` times by one call --
 * BevGenerator.__call__ (surroundBEV.py:312-325) for a fixed set of device buffers costs one graph launch per
 * frame-set instead of up to five kernel launches and two memsets (BALANCE), and a host that stalls between calls
 * cannot starve the GPU.  Run the same calls once before capturing: a call that has to allocate or build tables
 * inside a capture fails, and bevk_graph_end reports it.  Host-pointer entry points cannot be captured.
 * A graph keeps the device buffers it was captured with: a map slot's maps and a fused fisheye slot's column table
 * (bevk_undistorter_set), and the BEV LUT.  Setting that slot or camera up again after the capture changes what the
 * graph reads (or frees it, if the buffer had to grow); capture again after bevk_undistorter_set /
 * bevk_bev_set_camera.  Those set-up calls (and bevk_undistort_map) cannot themselves be captured.            */
int bevk_graph_begin(bevk_ctx *ctx);
int bevk_graph_end(bevk_ctx *ctx, int *graph_id);
int bevk_graph_launch(bevk_ctx *ctx, int graph_id, int times);
int bevk_graph_destroy(bevk_ctx *ctx, int graph_id);
/* Kernel launches issued by this ctx since creation (bench "gpu_launches"). */
int64_t bevk_launch_count(bevk_ctx *ctx);
/* Milliseconds spent in the last bevk_bev_run_device, bevk_jpeg_encode or bevk_png_encode call's kernels, measured with
 * CUDA events on the ctx stream (synchronises). */
int bevk_last_kernel_ms(bevk_ctx *ctx, float *ms);

#ifdef __cplusplus
}
#endif
#endif /* BEVK_H */
