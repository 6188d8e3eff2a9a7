// Convolution problem descriptor shared by the wgmma implicit-GEMM kernels
// (film_conv_tc.cu) and the CUDA-core validation kernel (film_kernels.cu).
//
// A "problem" is one Conv2D call site of the reference graph
// (feature_extractor.py:94-99, pyramid_flow_estimator.py:67-72, fusion.py:83-96) viewed as
// an implicit GEMM:  M = B*H*W output-grid pixels, N = Cout, K = sum over sources, 64-channel
// chunks and taps.  The K loop walks (source, chunk, tap) in that order; channel concats of
// the reference (`tf.concat`, feature_extractor.py:191, pyramid_flow_estimator.py:95,
// util.py:142, fusion.py:136) are never materialised -- each concat operand is a source.
#pragma once
#include <cuda.h>
#include <stdint.h>

#include "film_common.cuh"

namespace film {

constexpr int kMaxSrc = 4;
constexpr int kMaxTaps = 9;
constexpr int kChunk = 64;   // default channels per K block (64 x 2 B = one 128 B swizzle row)
                             // ConvProblem::kchunk may be 32 (64 B rows, SWIZZLE_64B) for 32-channel layers
constexpr int kTileM = 128;  // output pixels per CTA tile (tile_h x tile_w)

struct ConvSrc {
  const sp_t* hi;
  const sp_t* lo;
  int C;       // channel stride of the tensor (allocated channels)
  int c_off;   // first channel consumed
  int nchunk;  // number of K-block chunks consumed
  int bswap;   // 1: this source is read with the batch index swapped (b -> B - 1 - b): the coarsest flow level pairs
               // the features of image 0 with the UNWARPED features of image 1 and vice versa
               // (pyramid_flow_estimator.py:148-149), which is the same tensor at the other batch index
};

struct alignas(64) ConvProblem {
  CUtensorMap tm_a_hi[kMaxSrc];
  CUtensorMap tm_a_lo[kMaxSrc];
  CUtensorMap tm_w_hi;
  CUtensorMap tm_w_lo;
  CUtensorMap tm_w_hi_half;  // box [BN/2 x KC]: CTA-pair kernel, each CTA loads (and multicasts) half of every tap
  CUtensorMap tm_w_lo_half;
  ConvSrc src[kMaxSrc];
  int nsrc;
  int B, H, W;              // GEMM-M grid == input grid
  int tile_h, tile_w;       // tile_h * tile_w == 128 (256: persistent kernel with pxn)
  int tiles_y, tiles_x;
  int ntaps;
  int tap_dy[kMaxTaps], tap_dx[kMaxTaps];
  int kchunk;               // channels per K block: 64 or 32
  int ktot;                 // total K (multiple of kchunk)
  const sp_t* w_hi;         // [cout][ktot] K-major
  const sp_t* w_lo;
  const float* bias;        // [cout]
  int cout;
  int act;                  // 1 = LeakyReLU(0.2)
  sp_t* out_hi;
  sp_t* out_lo;
  int out_C, out_c_off;     // channel stride / first channel of the destination slice
  int out_H, out_W;         // destination spatial dims
  int out_sy, out_sx, out_oy, out_ox;  // dest pixel = (y*sy + oy, x*sx + ox)
  // epilogue mode 1 ("flow head", pyramid_flow_estimator.py:77-83,161): this conv is the 1x1
  // nf -> nf/2 LeakyReLU layer; the epilogue applies the final linear 1x1 (nf/2 -> 2) on the
  // fp32 accumulators and adds the upsampled flow:  res = W4^T h + b4 ;  v = res + v_up.
  // epilogue mode 2 ("RGB head", fusion.py:100-101,139 + the crop of eval/interpolator.py:175; persistent single-CTA
  // kernel only): this conv is the decoder's last 3x3 (64 -> 64, LeakyReLU); the epilogue applies the linear 1x1
  // 64 -> 3 output conv on the fp32 activations and writes the cropped fp32 image -- the 64-channel tensor is never
  // stored.  head_w4 = [64][3], head_b4 = [3], head_v = image [crop_h][crop_w][3] with row pitch crop_pitch floats.
  // epilogue mode 3 ("flow head in the last 3x3", persistent single-CTA kernel, Cout <= 64): this conv is conv_2 of a
  // FlowEstimator (pyramid_flow_estimator.py:66-72); the epilogue applies conv_3 (1x1, nf -> nf/2, LeakyReLU, head_w3 =
  // [nf][nf/2], head_b3), conv_4 (1x1 -> 2, linear, head_w4 / head_b4) and the residual add `v = r + v_up` (:161) on the
  // fp32 activations: the nf-channel tensor is never stored and the separate head launch disappears.
  int epi_mode;
  const float* head_w3;
  const float* head_b3;
  int crop_y, crop_x, crop_h, crop_w;
  int64_t crop_pitch;
  const float* head_w4;   // [cout][2]
  const float* head_b4;   // [2]
  const float* head_vup;  // [B][H][W][2] or null (coarsest level)
  float* head_res;        // [B][H][W][2]
  float* head_v;          // [B][H][W][2]
  // persistent 3x3 kernel (film_conv3x3_tc.cu): tiles of 128 pixels (16 x 8, 8 x 16 or 4 x 32; 32 x 8 = 256 pixels
  // with pxn), taps are dx-major, tm_a_* boxes are (KC ch, tile_w px, tile_h + 2 rows), or tile_w + 2 px wide with
  // `halo`.  Pipeline shape chosen on the host:
  int v2_resident;        // 1: all W_hi/W_lo K blocks stay in shared memory for the CTA's lifetime
  int v2_na, v2_nw;       // activation-ring / weight-ring stages
  int v2_grid;            // persistent CTAs
  int v2_part_lo, v2_part_hi;  // activation stages [lo, hi) of every tile read the one source whose chunks hold data in
                               // their first 16-channel k-step only (the 10-of-64 "side" source, the 3-of-32 image
                               // block): the kernel issues that k-step alone there, skipping the zero padding exactly.
                               // lo == hi: no such source.  The generic kernel issues every k-step
  // optional fused 2x2/2 average pool of the (activated, fp32) output tile, written as a second
  // split tensor [B][H/2][W/2][pool_C] (feature_extractor.py:138-146); null = off
  sp_t* pool_hi;
  sp_t* pool_lo;
  int pool_C;
  int group;              // generic kernel: number of consecutive problems launched as grid.z
  int pair;               // 1: persistent 3x3 kernel as (2,1,1) clusters sharing streamed weight taps by TMA multicast
  int halo;               // persistent 3x3 kernel, 16x8 tiles: 1 = ONE (KC ch, 10 px, 18 rows) halo box per chunk serves
                          // all nine taps (descriptors start at pixel granularity, SBO = 10 pixel rows); 0 = three
                          // dx-shifted 8-px boxes.  Set to 1 by the engine to ALLOW it; the plan functions keep or clear it.
  int bn;                 // N tile (32/64/128/256): conv_tc_block_n(cout), or smaller on tiny levels so that
                          // a K-serial problem spreads over more SMs
  int passes;             // MMAs per product: 3 = A_hi*W_hi + A_hi*W_lo + A_lo*W_hi (fp32-grade), 1 = A_hi*W_hi only
                          // (11-bit fp16 operands, fp32 accumulate; only the hi planes of the activations and
                          // weights are loaded).  Chosen per call site by the engine's precision plan
                          // (film_engine.cu).
  int straight;           // persistent kernel, resident weights: 1 = a whole activation stage is one wgmma group issued as
                          // straight-line code (default), 0 = one group per tap
  int out_lo_skip;        // 1: every consumer of the destination reads the hi plane only -> the lo plane is not written
  int pxn;                // persistent kernel, BN = 64 or 128, 64-channel chunks, store / pool epilogue: 1 = pixels on the
                          // wgmma N dimension (D^T = W_tap x A^T, one m64n128k16 per 64-cout half of the N tile, 32x8 tiles
                          // of 128 pixels per consumer warpgroup)
};

// launchers (film_conv_tc.cu / film_kernels.cu)
cudaError_t launch_conv_tc(const ConvProblem* d_prob, const ConvProblem& h_prob, cudaStream_t st);
cudaError_t launch_conv_simt(const ConvProblem* d_prob, const ConvProblem& h_prob, cudaStream_t st);
cudaError_t conv_tc_configure();  // cudaFuncSetAttribute for all instantiations
// persistent 3x3 variant: fills the v2_* fields of `h_prob` (call before uploading the problem)
bool conv3x3_tc_plan(ConvProblem& h_prob, int num_sms);   // false if the shape's smem rings cannot fit
void conv3x3_tc_pick_tile(int H, int W, int B, int cout, int kc, int passes, int ktot, int epi_mode, int num_sms,
                          int& tile_h, int& tile_w);
cudaError_t launch_conv3x3_tc(const ConvProblem* d_prob, const ConvProblem& h_prob, cudaStream_t st);
cudaError_t conv3x3_tc_configure();
}  // namespace film
