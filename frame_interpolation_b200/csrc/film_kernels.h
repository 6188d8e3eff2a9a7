// Launchers of the bandwidth-bound (non-GEMM) kernels of the FILM engine.
#pragma once
#include <cuda_runtime.h>

#include "film_common.cuh"

namespace film {

// util.py:38-44 -- 2x2/2 VALID average pool of a 3-channel fp32 image batch.
cudaError_t launch_image_pool(const float* in, float* out, int B, int H, int W, cudaStream_t st);

// feature_extractor.py:119 (cfeat_conv_0: 3 -> 64, 3x3 SAME, LeakyReLU): K = 27, HBM-bound.
// w: [27][64] fp32 (k = (ky*3+kx)*3 + ci), writes split output into a channel slice.
cudaError_t launch_conv0_c3(const float* img, int B, int H, int W, const float* w,
                            const float* bias, sp_t* out_hi, sp_t* out_lo, int out_C,
                            int out_c_off, cudaStream_t st);

// Product path of cfeat_conv_0: register-tiled fp32 direct conv (K = 27 is too short for the tensor cores), reads the
// fp32 image level, writes the 64-channel split output [B][H][W][64] (hi plane only when `lo_skip`).
// `pool_out` (nullable): [B][H/2][W/2][3] fp32 -- the 2x2/2 average pool of `img` (util.py:38-44), i.e. the next image
// pyramid level, written from the input patch the conv has staged anyway (H, W even).
cudaError_t launch_fe_conv0(const float* img, int B, int H, int W, const float* w, const float* bias, sp_t* out_hi,
                            sp_t* out_lo, bool lo_skip, float* pool_out, cudaStream_t st);

// im2col-lite for the tensor-core version of cfeat_conv_0: [B][H][W][3] fp32 -> [B][H][W][32] split
// (27 tap x channel values in HWIO order + 5 zero channels, zero outside the image).
cudaError_t launch_im2col3x3(const float* img, int B, int H, int W, sp_t* out_hi, sp_t* out_lo, cudaStream_t st);

// [B][H][W][3] fp32 -> channels 0..7 of a zero-initialised [B][H][W][32] split tensor (3 real channels).
cudaError_t launch_image_to_split32(const float* img, int B, int H, int W, sp_t* out_hi, sp_t* out_lo, cudaStream_t st);

// feature_extractor.py:138-146 -- 2x2/2 VALID average pool of a channel slice of a split tensor.
cudaError_t launch_act_pool(const sp_t* in_hi, const sp_t* in_lo, int in_C, int in_c_off, int B,
                            int H, int W, int Cn, sp_t* out_hi, sp_t* out_lo, int out_C,
                            cudaStream_t st);

// pyramid_flow_estimator.py:154-157 fused: v_up = resize_bilinear(2*v_prev -> HxW);
// warped[d] = warp(feat[1-d], v_up[d]).  feat/warped are [2][H][W][C] split tensors.
cudaError_t launch_flow_warp(const float* v_prev, int Hc, int Wc, const sp_t* feat_hi,
                             const sp_t* feat_lo, int H, int W, int C, float* v_up,
                             sp_t* warped_hi, sp_t* warped_lo, bool hi_only, cudaStream_t st);
// hi_only (both gathers): the destination's only consumers are single-pass convs -> read and write the hi
// planes alone (half the bytes; the lo planes of the destination are left untouched and never read)

// pyramid_flow_estimator.py:77-83,96-97 (conv_3: 1x1 nf->nf/2 LReLU, conv_4: 1x1 ->2 linear)
// fused with :161 (v = v_residual + v).  x: [2][H][W][Cx] split (first nf channels real).
cudaError_t launch_flow_head(const sp_t* x_hi, const sp_t* x_lo, int Cx, int nf, int npix,
                             const float* w3, const float* b3, const float* w4, const float* b4,
                             const float* v_up, float* residual, float* v, cudaStream_t st);

// interpolator.py:159-183: flows scaled by the time, warp of [image, features] pyramids.  `time` is a device scalar t
// (0.5 in the reference graph): warped[0] = warp(feat[0], fp32(t * v[1])), warped[1] = warp(feat[1], fp32((1 - t) * v[0]))
// (k = 0: image 0 by backward flow, k = 1: image 1 by forward flow; v[0] = forward flow, v[1] = backward flow).
cudaError_t launch_fusion_warp(const float* v, const float* time, const sp_t* feat_hi, const sp_t* feat_lo, int H,
                               int W, int C, sp_t* warped_hi, sp_t* warped_lo, bool hi_only, cudaStream_t st);
// one thread stores t into the device scalar `time`: stream-ordered, so a captured graph replayed after it reads t
cudaError_t launch_set_time(float* time, float t, cudaStream_t st);
// fusion.py:133 when the level is not exactly twice the coarser one: TF2 NEAREST resize of channels
// [src_c_off, src_c_off + Cn) of a [B][Hi][Wi][src_C] split tensor into channels [dst_c_off, dst_c_off + Cn) of a
// [B][Ho][Wo][dst_C] one, src = min(floor((dst + 0.5) * in / out), in - 1) per axis (exact integer arithmetic).
// Channel counts and offsets are multiples of 8.  hi_only: the consumer is a single-pass conv -> only the hi planes
// are read and written.
cudaError_t launch_resize_nearest(const sp_t* src_hi, const sp_t* src_lo, int src_C, int src_c_off, int B, int Hi, int Wi,
                                  sp_t* dst_hi, sp_t* dst_lo, int dst_C, int dst_c_off, int Ho, int Wo, int Cn, bool hi_only,
                                  cudaStream_t st);
// side tensor [1][H][W][side_C] split: ch 0-2 warp(img0, t*bwd), 3-5 warp(img1, (1-t)*fwd),
// 6-7 t*bwd, 8-9 (1-t)*fwd, 10-15 zero (t = *time, rounded like launch_fusion_warp).
cudaError_t launch_fusion_side(const float* v, const float* time, const float* img, int H, int W, sp_t* side_hi,
                               sp_t* side_lo, int side_C, cudaStream_t st);

// fusion.py:100-101,139 (1x1 conv 64 -> 3, linear) + crop (eval/interpolator.py:175).
cudaError_t launch_rgb_head(const sp_t* x_hi, const sp_t* x_lo, int Cx, int H, int W,
                            const float* w, const float* b, float* out, int64_t out_pitch,
                            int off_y, int off_x, int out_h, int out_w, cudaStream_t st);

// zero-pad copy (eval/interpolator.py:56): dst [H][W][3] <- src [h][w][3] at (off_y, off_x).
cudaError_t launch_pad_image(const float* src, int64_t src_pitch, int h, int w, float* dst, int H,
                             int W, int off_y, int off_x, cudaStream_t st);

// 8-bit front / back end: eval/util.py:38-41 (uint8 / 255 -> float32) and :51-52 (clip(x * 255, 0, 255) + 0.5 -> uint8)
cudaError_t launch_u8_to_f32(const uint8_t* src, float* dst, int64_t n, cudaStream_t st);
cudaError_t launch_f32_to_u8(const float* src, uint8_t* dst, int64_t n, cudaStream_t st);

// Overlapped tiling (option tile_overlap).  One frame axis of length L = b * p cut into b windows of one length
// q = p + 2v: window k starts at clamp(k*p - v, 0, L - q), so border windows are shifted inward, not shortened.
// An axis with b == 1 has v = 0 (one window, nothing to blend).  0 <= 2v <= p keeps the ramps of consecutive
// boundaries apart: a pixel sees at most two windows per axis.
struct StitchAxis {
  int b, p, v, q, L;
};
__host__ __device__ inline int stitch_origin(const StitchAxis& a, int k) {  // first coordinate of window k
  const int o = k * a.p - a.v;
  return o < 0 ? 0 : (o > a.L - a.q ? a.L - a.q : o);
}
constexpr int kMaxStitchTiles = 64;
struct StitchGeom {
  StitchAxis ay, ax;            // rows, columns
  int slot[kMaxStitchTiles];    // tile t = ty * ax.b + tx lives at tiles + slot[t] * tile_stride
};
// Feathered stitch of [tiles][q_h][q_w][3] fp32 window results into an (H, W, 3) frame with row pitch `out_pitch`
// floats.  Across the boundary c = k*p between windows k-1 (value a) and k (value b), for x in [c - v, c + v):
// t = (x + 0.5 - (c - v)) / 2v, out = a + t * (b - a); elsewhere the pixel of the window whose core holds it.  Along W
// first, then along H.  Gather form: every output float is written once, from at most four windows.
cudaError_t launch_stitch_feather(const float* tiles, int64_t tile_stride, const StitchGeom& g, float* out,
                                  int64_t out_pitch, cudaStream_t st);

// debug: split tensor slice -> fp32 NHWC
cudaError_t launch_unsplit(const sp_t* hi, const sp_t* lo, int C, int c_off, int Cn, int64_t npix,
                           float* out, cudaStream_t st);

}  // namespace film
