/*
 * film_b200.h -- C ABI of the H100-native (sm_90a) FILM inference engine (libfilm_b200.so).
 *
 * Drop-in boundary: every entry point replaces one piece of the reference's Python
 * inference wrapper, `eval/interpolator.py` (google-research/frame-interpolation):
 *
 *   film_create            <- Interpolator.__init__  (eval/interpolator.py:135-150,
 *                             tf.saved_model.load at :148)
 *   film_interpolate       <- Interpolator.interpolate (eval/interpolator.py:152-176):
 *                             _pad_to_align (:30-63) -> self._model(inputs) (:170-172,
 *                             i.e. models/film_net/interpolator.py:89-207) -> crop (:175)
 *   film_interpolate_tiled <- Interpolator.__call__ tiled branch
 *                             (eval/interpolator.py:192-206; image_to_patches :66-99,
 *                             patches_to_image :102-126)
 *   film_interpolate_device<- same as film_interpolate with device-resident frames; no
 *                             reference counterpart (the reference pays H2D + D2H + sync
 *                             per call at :171,:176); used by the recursive scheduler
 *                             (eval/util.py:62-91) and the multi-GPU shards.
 *
 * Plain C: pointers and sizes only, no torch / CUDA types in the signatures (a CUDA
 * stream is passed as void*). All frames are float32, NHWC, C-contiguous, 3 channels,
 * nominally in [0,1]; `dt` (B floats) is accepted and ignored exactly like the
 * reference ignores `time` (models/film_net/interpolator.py:102,163). Outputs are
 * NOT clipped (clipping happens in eval/util.py:51 on the reference side).
 *
 * Status codes: 0 ok; 1 bad argument (shape / alignment / divisibility);
 * 2 CUDA error; 3 weight-file mismatch; 4 not supported. film_last_error() returns
 * a human-readable message for the last non-zero status on that handle (or on
 * creation, when handle is NULL).
 *
 * There is no CPU fallback: every entry point fails with status 2 if no sm_90
 * device is present.
 *
 * Threading: a handle owns one CUDA stream, its per-shape plans (activation arenas, CUDA
 * graphs) and its staging buffers, so calls on ONE handle must be serialised by the caller;
 * different handles (one per GPU, or several per GPU when memory allows: ~20 GB per cached
 * 1080p shape) are independent and may be driven from different threads or processes.
 */
#ifndef FILM_B200_H_
#define FILM_B200_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define FILM_API __attribute__((visibility("default")))
#else
#define FILM_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct film_handle film_handle;

enum {
  FILM_OK = 0,
  FILM_ERR_ARG = 1,
  FILM_ERR_CUDA = 2,
  FILM_ERR_WEIGHTS = 3,
  FILM_ERR_UNSUPPORTED = 4
};

/* Per-call engine statistics (all times are device times from CUDA events). */
typedef struct film_profile_t {
  double last_call_ms;        /* event time of the last network call (excl. H2D/D2H)      */
  double last_h2d_ms;         /* host->device copy time of the last host-pointer call     */
  double last_d2h_ms;         /* device->host copy time of the last host-pointer call     */
  double conv_flops;          /* reference-graph conv FLOPs of the last call (2*MAC)      */
  double mma_flops;           /* tensor-core FLOPs actually issued (1 or 3 passes per stage, padded K) */
  double warp_bytes;          /* algorithmic bytes of the warp-gather kernels (rd+wr)      */
  int64_t kernel_launches;    /* kernels launched (or graph nodes replayed) by the last call */
  int64_t arena_bytes;        /* device memory held by the plan used by the last call     */
  int32_t padded_h, padded_w; /* network resolution of the last call                       */
  int32_t used_graph;         /* 1 if the last call replayed a CUDA graph                  */
  int32_t reserved;
} film_profile_t;

/* Loads a FILMW1 weight file (see frame_interpolation_b200/weights.py), repacks the
 * HWIO kernels into the engine's split-bf16 K-major layout on `device_ordinal`,
 * creates the stream.  Replaces tf.saved_model.load (eval/interpolator.py:148). */
FILM_API int film_create(film_handle** out, const char* weights_path, int device_ordinal);

FILM_API void film_destroy(film_handle* h);

/* Host pointers. x0/x1/out: B*H*W*3 floats. align <= 0 disables padding
 * (eval/interpolator.py:149: `align or None`); then H and W must be multiples of 64 unless the
 * option "any_size" is 1.
 * Blocks until `out` is written. */
FILM_API int film_interpolate(film_handle* h, const float* x0, const float* x1, const float* dt,
                     int B, int H, int W, int align, float* out);

/* Host pointers, B == 1. Splits the frame into block_h x block_w non-overlapping tiles
 * (row-major tile order), pads every tile independently to `align`, runs the network
 * per tile, stitches. H % block_h == 0 and W % block_w == 0 or status 1.
 * With the option "tile_overlap" = v > 0 (no reference counterpart) every tile runs on a window that reaches v pixels
 * past each interior tile boundary and neighbouring results are cross-faded over the 2v pixels around the boundary:
 * both frames are uploaded once, the windows run as views of the resident frames, film_stitch_tiles_device blends them,
 * one download.  2v must not exceed the tile height (block_h > 1) or width (block_w > 1), else status 1; at most 64
 * tiles.  film_profile then reports the padded window size. */
FILM_API int film_interpolate_tiled(film_handle* h, const float* x0, const float* x1, const float* dt,
                           int H, int W, int align, int block_h, int block_w, float* out);

/* Device pointers (same layout), row pitches in floats (pitch >= W*3) so a tile of a
 * larger frame can be passed as a strided view. Asynchronous on `cuda_stream`
 * (a cudaStream_t; NULL = the handle's own stream, in which case the call returns after
 * enqueueing; use film_synchronize). */
FILM_API int film_interpolate_device(film_handle* h, const float* d_x0, const float* d_x1,
                            int B, int H, int W, int64_t in_pitch, int align,
                            float* d_out, int64_t out_pitch, void* cuda_stream);

/* Feathered stitch of overlapped tiles, device pointers, asynchronous on `cuda_stream` like film_interpolate_device.
 * Geometry, the same along H and W: a frame axis of length L in b blocks has the core length p = L / b.  b == 1: one
 * window [0, L), nothing is blended.  b > 1: every window has the length q = p + 2 * overlap and window k starts at
 * clamp(k*p - overlap, 0, L - q): border windows are shifted inward, not shortened, so all block_h * block_w windows of
 * a frame have one shape (q_h, q_w).  Tile t (row-major) is read as [q_h][q_w][3] floats at
 * d_tiles + slot_of_tile[t] * tile_stride (tile_stride in floats, >= q_h*q_w*3; slot_of_tile: HOST array of
 * block_h*block_w ints read before the call returns, NULL = identity; a rank-major all-gather buffer is read in place
 * through it).  At the boundary c = k*p between tiles k-1 (value a) and k (value b), for x in [c - overlap, c + overlap):
 * t = (x + 0.5 - (c - overlap)) / (2 * overlap), out = a + t * (b - a); every other pixel comes from the tile whose core
 * contains it; along W first, then along H.  Every output float is written once (no atomics: results are
 * run-to-run identical) through the row pitch out_pitch (floats, >= W*3).  Status 1 unless 0 <= 2 * overlap <= p on
 * every axis with b > 1, block_h * block_w <= 64 and H <= 65535. */
FILM_API int film_stitch_tiles_device(film_handle* h, const float* d_tiles, int64_t tile_stride, const int* slot_of_tile,
                                      int H, int W, int block_h, int block_w, int overlap, float* d_out,
                                      int64_t out_pitch, void* cuda_stream);

/* Recursive mid-point interpolation between two (H, W, 3) host frames, the whole binary tree of
 * eval/util.py:62-91 (`_recursive_generator`) evaluated with every intermediate frame resident in
 * HBM: 2 uploads, 2^times - 1 network calls, 1 download.  `out` receives 2^times + 1 frames in
 * display order INCLUDING both end points (what interpolate_recursively_from_memory yields for one
 * pair, eval/util.py:125-153).  Results are bit-identical to calling film_interpolate recursively. */
FILM_API int film_interpolate_recursive(film_handle* h, const float* frame0, const float* frame1, int H, int W,
                                        int align, int times_to_interpolate, float* out);

/* Frames at arbitrary times between two (H, W, 3) frames: frame i of `out` is the reference graph with mid_time
 * (models/film_net/interpolator.py:159-161, multiply_pyramid) replaced by t_i = times[i]: image 0 is warped with
 * fp32(t * backward_flow), image 1 with fp32((1 - t) * forward_flow) (1 - t an fp32 subtraction), and the side tensor,
 * the warps and the fusion decoder follow.  No reference counterpart: the released weights were supervised at t = 0.5
 * only, so the quality away from 0.5 depends on the weights.  At t = 0.5 frame i is bit-identical to film_interpolate on
 * the same pair, handle options and align.
 * One head (padding, pyramids, features, both flow pyramids) per call, then per time one tail (fusion warps, side
 * tensors, decoder, RGB head); CUDA graphs: one for the head, one for the tail.  The times plan is cached next to the
 * ordinary plan of the shape and keeps feature levels 0-4 of both images alive across the tails: 2.65 GB at 1088x1920
 * (2 images x sum over levels 0-4 of H_l * W_l * C_l x 4 bytes, C_l = 64, 192, 448, 960, 960).  Its arena measured
 * 0.94 GB larger than the ordinary plan's there (H100 80GB HBM3): the decoder finds most of its buffers in blocks the
 * head has released.
 * `times`: HOST array of n_times floats, read before the call returns.  Status 1 for n_times < 1 or a t that is not
 * finite or not in [0, 1] (the message names its index); the frame-size rule (status 4 / option any_size) is the one of
 * film_interpolate.  film_profile covers the whole call: conv_flops = head + n_times x tail, kernel_launches = head ops +
 * n_times x tail ops (the one-thread kernel that stores each t is not counted).
 * film_interpolate_times: host frames, `out` receives n_times frames; blocks until they are written.
 * film_interpolate_times_device: device frames with row pitches like film_interpolate_device, frame i at
 * d_out + i * H * out_pitch; asynchronous on `cuda_stream` (NULL = the handle's stream). */
FILM_API int film_interpolate_times(film_handle* h, const float* x0, const float* x1, const float* times, int n_times,
                                    int H, int W, int align, float* out);
FILM_API int film_interpolate_times_device(film_handle* h, const float* d_x0, const float* d_x1, const float* times,
                                           int n_times, int H, int W, int64_t in_pitch, int align, float* d_out,
                                           int64_t out_pitch, void* cuda_stream);

/* film_interpolate_times on the tiles of film_interpolate_tiled: frame i of `out` is what film_interpolate_tiled computes
 * with the handle's "tile_overlap" v, with every window's mid_time replaced by t_i = times[i].  The windows are those of
 * film_stitch_tiles_device (v = 0: the reference's non-overlapping tiles, each padded on its own to `align`); every
 * window runs what film_interpolate_times runs on its crop, one head and then one tail per time, and per time the window
 * results are stitched by film_stitch_tiles_device (a paste at v = 0).  Consequences: at t = 0.5 frame i is bit-identical
 * to film_interpolate_tiled on the same pair, options, align and overlap; at v = 0 tile k of frame i is bit-identical to
 * film_interpolate_times on tile k's crop; block 1 x 1 is film_interpolate_times.
 * Host frames in; `out` receives n_times frames of (H, W, 3); blocks until they are written.  Both frames are uploaded
 * once, and one times plan of the window shape serves every window (row-major order).  Times are checked as in
 * film_interpolate_times, the geometry as in film_interpolate_tiled (divisibility, 2v <= tile size on every blocked
 * axis, at most 64 tiles: status 1); the frame-size rule (status 4 / option any_size) applies to the window shape.
 * Device scratch, kept by the handle and grown on demand: (2 + n_times) frames plus n_times x tiles windows of float32,
 * i.e. 4 x ((2 + n) x H x W x 3 + n x tiles x q_h x q_w x 3) bytes (8K in 4x4 tiles at v = 0 and n = 7: 9 x 398 MB + 112 x
 * 24.9 MB = 6.4 GB, next to the times plan of the window); a failed allocation is status 2 and names the bytes.
 * film_profile covers the whole call: conv_flops = tiles x (head + n_times x tail), kernel_launches = tiles x (head ops +
 * n_times x tail ops) (the kernels that store t and the stitches are not counted), padded_h / padded_w = the padded
 * window, last_call_ms = every window's network plus the stitches (uploads and download excluded).  With option
 * keep_debug, film_debug_read returns the last window's last time. */
FILM_API int film_interpolate_times_tiled(film_handle* h, const float* x0, const float* x1, const float* times,
                                          int n_times, int H, int W, int align, int block_h, int block_w, float* out);

/* 8-bit front / back end (SURVEY 8f row 3): the frames cross PCIe as uint8 (4x fewer bytes) and the reference's
 * conversions run on the device, bit-identical to the host versions:
 *   in : float32 = uint8 / 255                         (eval/util.py:38-41, read_image)
 *   out: uint8   = trunc(clip(x * 255, 0, 255) + 0.5)  (eval/util.py:51-52, write_image)
 * film_interpolate_u8 == to_uint8(film_interpolate(x0 / 255, x1 / 255)).  film_interpolate_recursive_u8 keeps the
 * recursion on the unquantised float32 mid-frames (like eval/util.py:85-91) and quantises only what it returns. */
FILM_API int film_interpolate_u8(film_handle* h, const uint8_t* x0, const uint8_t* x1, int B, int H, int W, int align,
                                 uint8_t* out);
FILM_API int film_interpolate_recursive_u8(film_handle* h, const uint8_t* frame0, const uint8_t* frame1, int H, int W,
                                           int align, int times_to_interpolate, uint8_t* out);

/* Page-locked host memory for frames (cudaHostAlloc): uploads / downloads of pinned buffers run at
 * PCIe speed instead of through the driver's pageable staging path. The Python wrapper returns its
 * results in pooled buffers allocated here. NULL on failure. */
FILM_API void* film_host_alloc(size_t bytes);
FILM_API void film_host_free(void* p);

FILM_API int film_synchronize(film_handle* h);

/* Fills *out with statistics of the last call on this handle. */
FILM_API int film_profile(film_handle* h, film_profile_t* out);

/* Engine options, set before the first call of a given shape.
 *   "conv_impl"   : 0 = wgmma implicit-GEMM kernels (default, the product path),
 *                   1 = fp32 CUDA-core validation kernels (debug only; used by the
 *                       tests to cross-check the tensor-core path on the device)
 *   "use_graph"   : 1 = capture each shape's schedule in a CUDA graph (default), 0 = eager
 *   "keep_debug"  : 1 = keep every intermediate tensor alive (no arena reuse) so that film_debug_read can
 *                   return it after the call; it changes nothing else, so the same kernels run and the output is
 *                   bit-identical; 0 (default) = activation buffers are recycled inside a plan
 *   "time_ops"    : 1 = run eagerly with one CUDA-event pair per kernel (see film_op_table)
 *   "conv3x3_v2"  : 1 = persistent tap-reuse kernel for 3x3 convs (default), 0 = generic kernel
 *   "conv3x3_2cta": 1 = the streamed-weight 3x3 convs of the large pyramid levels run as (2,1,1) CTA clusters in which
 *                   each CTA loads half of every weight tap and TMA-multicasts it to both, 0 = off (default: the
 *                   paired layers measure slower on H100), 2 = every eligible layer
 *   "conv3x3_halo": wide halo boxes of the persistent kernel -- one (64 ch, 10 px, 18 rows) TMA box per chunk serves all
 *                   nine taps (wgmma descriptors at pixel offsets): 3 = 64- and 32-channel chunks (default),
 *                   2 = 64-channel chunks only, 1 = CTA-pair layers only, 0 = three dx-shifted 8-px boxes
 *   "conv3x3_pxn" : persistent 3x3 layers with Cout = 64 (or single-pass with Cout = 128, 256 or 512), 64-channel chunks
 *                   and a plain or pooled store put the pixels on the wgmma N dimension (m64n128k16 per 64-cout half of
 *                   a 128-cout N tile, weight tap as the M operand, 32x8 tiles): 1 = where 32x8 tiles times N tiles
 *                   still give two waves over the SMs and the layer class measured faster (Cout = 64 and 128; Cout =
 *                   256 with K <= 9216), and for a Cout = 64 layer with a source that skips k-steps (fusion conv_1)
 *                   where 32x8 tiles take at most half the waves of 16x8 tiles (default), 2 = every such layer, 0 = off.
 *                   Wider layers whose source skips k-steps keep the 16x8 form
 *   "fe_conv0_tc" : cfeat_conv_0 (3 -> 64, K = 27): 0 = register-tiled fp32 FMA kernel reading the fp32 image directly
 *                   (default: exact fp32 arithmetic, no widened image tensor), 1 = tensor-core kernel over a 32-channel-
 *                   padded split image
 *   "plane_skip"  : 1 = lo planes that no consumer reads (destinations of single-pass convs) are neither gathered nor
 *                   written (default), 0 = always both planes
 *   "mma_straight": 1 = with resident weights each warpgroup issues a whole activation stage as one wgmma group of
 *                   straight-line code (default), 0 = one wgmma group per tap
 *   "arena_reuse" : 1 = activation buffers are recycled inside a plan by liveness (default), 0 = one buffer per tensor
 *   "fuse_flow_head": 1 = on flow level 0 (32-filter predictor) conv_3, conv_4 and the residual add run in the epilogue of
 *                   conv_2 (default), 2 = also on level 1 (64 filters: measured epilogue-bound, slower), 0 = separate launch
 *   "fuse_rgb_head": 1 = the linear 1x1 RGB head and the crop run in the epilogue of the decoder's last 3x3 conv (default;
 *                   the 64-channel activation is never stored), 0 = separate kernel
 *   "any_size"    : 0 = the padded frame size must be a multiple of 64, anything else fails with status 4 (default),
 *                   1 = any padded size whose level-5 grid is at least 2x2 runs the reference graph (smaller frames
 *                   fail with status 1): pyramid levels floor like its VALID pooling, and a decoder level that is not
 *                   exactly twice the coarser one gets a nearest resize of its own before fusion conv_0.  Only decides
 *                   whether a size is accepted: a 64-aligned size runs the same plan either way
 *   "tile_overlap": film_interpolate_tiled only.  0 = the reference's tiling: non-overlapping tiles, pasted (default),
 *                   v > 0 = every tile is interpolated on a window v pixels larger on each interior side and neighbouring
 *                   results are cross-faded over 2v pixels (see film_stitch_tiles_device); negative values are stored
 *                   as 0.  The output then differs from the reference's, which is why it is never chosen for the caller.
 *                   Not a plan key: the window shape selects the plan, and one frame needs one plan
 *   "use_lanes"   : 1 = enqueue independent branches on separate streams (default 0)
 *   "clear_plans" : (any value) drop every cached (H, W, align) plan -- CUDA graph and activation arena --
 *                   after draining the handle's stream.  Plans are cached per shape and never evicted
 *                   otherwise, except that a shape whose arena cannot be allocated triggers one
 *                   drop-and-retry before FILM_ERR_CUDA is returned. */
/*   "onepass_mask": precision plan -- bit s selects the single-pass product (A_hi x W_hi, fp16 operands, fp32
 *                   accumulate) for stage s (film_stage_count / film_stage_name); every other conv runs the
 *                   three-pass split product.  The default is a measured per-stage plan;
 *                   0 = every conv three-pass (fp32-grade).  "onepass_default" (any value) restores it. */
FILM_API int film_set_option(film_handle* h, const char* name, int value);
/* Reads back any value option of film_set_option, as stored (booleans as 0/1, clamped and masked values after the
 * clamp or mask), or "onepass_default": the default precision plan.  An unknown name returns FILM_ERR_ARG. */
FILM_API int film_get_option(film_handle* h, const char* name, int* value);

/* Stages of the precision plan: film_stage_count() names ("fe_i0_k01", "flow_L3", "fus2_c1", ...), index =
 * bit position in "onepass_mask".  film_stage_name copies the NUL-terminated name into buf. */
FILM_API int film_stage_count(void);
FILM_API int film_stage_name(int stage, char* buf, int buf_size);

/* Debug/parity hook: copies an intermediate tensor of the LAST call to host as float32
 * NHWC. `name` is e.g. "feat0/3" (feature pyramid of image 0, level 3), "flow_fwd/0",
 * "flow_bwd/2", "image", "img/2" (image pyramid level, [2][H_l][W_l][3]).  The destination of
 * every conv op of film_op_table is "out:<op name>" (its cout real channels over all batches;
 * the pooled output of a conv, fused or by fe_pool@L<r>: "pool:<conv op name>"), and so are the
 * outputs of fe_conv0*, fe_split32@L*, fe_im2col@L* and fusion_resize@L* (that one's resized side
 * tensor: "out:fusion_resize@L<i>:side").  "fusion_net/0" is absent when the RGB head is fused.
 * "<name>.hi" / "<name>.lo" return one 16-bit plane of a split tensor as float32 (a plane that
 * was never written reads as zeros).  Returns the element count through *count when dst == NULL. */
FILM_API int film_debug_read(film_handle* h, const char* name, float* dst, int64_t* count);

/* Per-op table of the plan used by the last call, as CSV text
 * "idx,category,name,ms,ref_flops,alg_bytes,form,passes" (category 0 = tensor-core conv, 1 = warp gather,
 * 2 = other bandwidth kernels; form = the kernel of a conv: "3x3" / "3x3_pxn" persistent 3x3 kernel, the latter with
 * pixels on N, "3x3_pair" persistent 3x3 kernel on (2,1,1) CTA-pair clusters (option conv3x3_2cta), "tc" generic
 * wgmma kernel, "simt" validation kernel, empty otherwise; passes = 1 (hi x hi) or 3 (split
 * product) for a category-0 conv, empty otherwise). `ms` is filled by calls made with option "time_ops" = 1
 * (eager run, one CUDA event pair per kernel on the launching stream), else -1.
 * *needed receives the buffer size required. */
FILM_API int film_op_table(film_handle* h, char* buf, int64_t buf_size, int64_t* needed);

FILM_API const char* film_last_error(film_handle* h);

/* Version / build info string: "film_b200 <ver> sm_90a split=fp16x2 mma=...". */
FILM_API const char* film_version(void);

#ifdef __cplusplus
}
#endif
#endif /* FILM_B200_H_ */
