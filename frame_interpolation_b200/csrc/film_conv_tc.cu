// wgmma implicit-GEMM convolution for sm_90a (the engine's generic tensor-core kernel).
//
// One CTA computes a 128-pixel (tile_h x tile_w) x BN-channel output tile of one Conv2D
// call site (film_conv.h).  GEMM view: D[128 x BN] += A[128 x 64] * W[BN x 64]^T per K block,
// K blocks = (source, 64-channel chunk, tap).
//
//   warp 8     : TMA producer (warpgroup 2; its registers are handed to the consumers).  Per K block: 4-D tiled
//                TMA loads of the hi and lo planes of the activation box (64 ch, tile_w, tile_h, 1) at the tap-shifted coordinate --
//                out-of-bounds rows/cols are zero-filled by TMA, which IS the SAME padding of
//                tf.keras Conv2D -- plus 2-D loads of the W_hi / W_lo [BN x 64] blocks.
//                Everything lands in SWIZZLE_128B K-major layout (one pixel = one 128 B row).
//   warps 0-7  : two consumer warpgroups, one per 64-pixel half of the tile.  Per K block 4 k-steps x 3 passes
//                A_hi*W_hi + A_hi*W_lo + A_lo*W_hi (split-precision product, fp32 accumulators in registers),
//                then the epilogue from the registers: + bias, LeakyReLU, re-split to hi/lo 16-bit planes, stores
//                into the destination channel slice (which is how channel concats and the NN-upsample parity
//                scatter are realised without extra passes).
//
// mbarrier pipeline: full[s] (TMA -> MMA, tx-count), empty[s] (MMA -> TMA, one arrive per warpgroup once its
// wgmma reading the stage retired).  A watchdog turns a stuck barrier into a trap instead of a hang.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <stdint.h>

#include "film_conv.h"
#include "film_tc_ptx.cuh"

namespace film {

namespace {
using namespace tc;

constexpr int kConsumers = 256;                 // two warpgroups
constexpr int kNumThreads = kConsumers + 128;   // + the producer warpgroup (one active warp)
template <int BN, int KC>
struct TcCfg {
  static constexpr int kABytes = kTileM * KC * 2;  // 16 KiB (KC = 64) or 8 KiB (KC = 32) per plane
  static constexpr int kWBytes = BN * KC * 2;
  static constexpr int kStageBytes = 2 * kABytes + 2 * kWBytes;
  static constexpr int kStages = (BN == 256) ? 2 : (BN == 128) ? 3 : 2;
  // two-accumulator product for BN <= 128: A_hi x W_hi and A_lo x W_hi accumulate into the first BN columns,
  // A_hi x W_lo into the second BN columns (all wgmma of one shape); the epilogue adds the halves
  static constexpr bool kFused = BN <= 128;
  static constexpr int kAccRegs = (kFused ? 2 * BN : BN) / 2;
  // stages + barriers (8 B each) + bias + flow-head weights
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 + BN * 4 + BN * 8 + 16;
};

template <int BN, int KC>
__global__ void __launch_bounds__(kNumThreads, 1) k_conv_tc(const ConvProblem* __restrict__ prob_base) {
  using Cfg = TcCfg<BN, KC>;
  // grid.z selects one of `group` consecutive problems with identical grids (the four parity classes
  // of the NN-upsample + 2x2 conv are one launch)
  const ConvProblem* __restrict__ prob = prob_base + blockIdx.z;
  constexpr int kABytes = Cfg::kABytes;
  extern __shared__ uint8_t smem_raw[];

  // carve shared memory (1024 B alignment required by SWIZZLE_128B)
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (base - raw);
  const uint32_t bar_base = base + Cfg::kStages * Cfg::kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (Cfg::kStages + s); };
  float* bias_smem = reinterpret_cast<float*>(gen_base + Cfg::kStages * Cfg::kStageBytes + 256);
  float* w4_smem = bias_smem + BN;  // [BN][2] + b4[2], flow-head mode only

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // problem fields -> registers once (asm "memory" clobbers would otherwise reload them from global)
  const int nsrc = prob->nsrc, ntaps = prob->ntaps, cout = prob->cout, epi_mode = prob->epi_mode;
  const bool one = prob->passes == 1;   // single-pass product: hi planes only
  const int tile_h = prob->tile_h, tile_w = prob->tile_w, tiles_x = prob->tiles_x, tiles_y = prob->tiles_y;

  // tile coordinates
  int tile = blockIdx.x;
  const int tx = tile % tiles_x;
  tile /= tiles_x;
  const int ty = tile % tiles_y;
  const int b = tile / tiles_y;
  const int y0 = ty * tile_h, x0 = tx * tile_w;
  const int n0 = blockIdx.y * BN;

  int nkb = 0;
  for (int s = 0; s < nsrc; ++s) nkb += prob->src[s].nchunk * ntaps;

  if (warp == 8 && lane == 0) {
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);   // one arrive per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp < 8) {
    for (int i = threadIdx.x; i < BN; i += kConsumers) bias_smem[i] = (n0 + i < cout) ? prob->bias[n0 + i] : 0.f;
    if (epi_mode == 1) {
      for (int i = threadIdx.x; i < 2 * BN; i += kConsumers) w4_smem[i] = (i < 2 * cout) ? prob->head_w4[i] : 0.f;
      if (threadIdx.x < 2) w4_smem[2 * BN + threadIdx.x] = prob->head_b4[threadIdx.x];
    }
  }
  __syncthreads();

  if (warp >= 8) {
    regs_dec<40>();   // registers of the producer warpgroup go to the consumers (168 per thread at launch)
    if (warp > 8) return;
    // ===================== TMA producer (warp-uniform, elected lane issues) =====================
    const CUtensorMap* tm_w_hi = &prob->tm_w_hi;
    const CUtensorMap* tm_w_lo = &prob->tm_w_lo;
    int kb = 0;
    for (int s = 0; s < nsrc; ++s) {
      const int nchunk = prob->src[s].nchunk, c_off = prob->src[s].c_off;
      const int bs = prob->src[s].bswap ? prob->B - 1 - b : b;
      const CUtensorMap* tm_hi = &prob->tm_a_hi[s];
      const CUtensorMap* tm_lo = &prob->tm_a_lo[s];
      for (int ch = 0; ch < nchunk; ++ch) {
        for (int t = 0; t < ntaps; ++t, ++kb) {
          const int stage = kb % Cfg::kStages;
          const uint32_t phase = (uint32_t)(kb / Cfg::kStages) & 1u;
          const int xx = x0 + prob->tap_dx[t], yy = y0 + prob->tap_dy[t];
          mbar_wait(empty_bar(stage), phase ^ 1u);
          if (elect_one()) {
            const uint32_t sa = base + stage * Cfg::kStageBytes;
            mbar_expect_tx(full_bar(stage), one ? (uint32_t)(kABytes + Cfg::kWBytes) : (uint32_t)Cfg::kStageBytes);
            const int cc = c_off + ch * KC;
            tma_load_4d(sa, tm_hi, full_bar(stage), cc, xx, yy, bs);
            tma_load_2d(sa + 2 * kABytes, tm_w_hi, full_bar(stage), kb * KC, n0);
            if (!one) {
              tma_load_4d(sa + kABytes, tm_lo, full_bar(stage), cc, xx, yy, bs);
              tma_load_2d(sa + 2 * kABytes + Cfg::kWBytes, tm_w_lo, full_bar(stage), kb * KC, n0);
            }
          }
          __syncwarp();
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups: MMA + epilogue =====================
  regs_inc<232>();
  const int wg = warp >> 2;                  // which 64-pixel half of the tile
  const uint32_t a_row0 = (uint32_t)(wg * 64 * KC * 2);
  float acc[Cfg::kAccRegs];
#pragma unroll
  for (int i = 0; i < Cfg::kAccRegs; ++i) acc[i] = 0.f;
  int prev_stage = -1;
  for (int kb = 0; kb < nkb; ++kb) {
    const int stage = kb % Cfg::kStages;
    const uint32_t phase = (uint32_t)(kb / Cfg::kStages) & 1u;
    mbar_wait(full_bar(stage), phase);
    const uint32_t sa = base + stage * Cfg::kStageBytes;
    const uint64_t a_hi = make_desc_kc<KC>(sa + a_row0), a_lo = make_desc_kc<KC>(sa + kABytes + a_row0);
    const uint64_t w_hi = make_desc_kc<KC>(sa + 2 * kABytes), w_lo = make_desc_kc<KC>(sa + 2 * kABytes + Cfg::kWBytes);
    const uint32_t first = kb == 0 ? 0u : 1u;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KC / 16; ++k) {
      const uint64_t adv = (uint64_t)(k * 32 >> 4);  // 16 elements x 2 B = 32 B along K
      if (one) {
        wgmma<BN>(acc, a_hi + adv, w_hi + adv, k == 0 ? first : 1u);
      } else if constexpr (Cfg::kFused) {
        wgmma<BN>(acc, a_hi + adv, w_hi + adv, k == 0 ? first : 1u);
        wgmma<BN>(acc + BN / 2, a_hi + adv, w_lo + adv, k == 0 ? first : 1u);
        wgmma<BN>(acc, a_lo + adv, w_hi + adv, 1u);
      } else {
        wgmma<BN>(acc, a_lo + adv, w_hi + adv, k == 0 ? first : 1u);
        wgmma<BN>(acc, a_hi + adv, w_lo + adv, 1u);
        wgmma<BN>(acc, a_hi + adv, w_hi + adv, 1u);
      }
    }
    wgmma_commit();
    // the previous K block's wgmma group has retired once at most this one is in flight: release its stage
    wgmma_wait<1>();
    if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(empty_bar(prev_stage));
    prev_stage = stage;
  }
  wgmma_wait<0>();
  acc_fence<Cfg::kAccRegs>(acc);

  // fragment -> pixels: this thread holds rows r0 = 64 wg + 16 (warp & 3) + lane / 4 and r0 + 8, channel pairs
  // 8j + 2 (lane & 3) + {0, 1}
  const bool fused3 = Cfg::kFused && !one;
  auto value = [&](int h, int j, int e) {
    const int i = 4 * j + 2 * h + e;
    return fused3 ? acc[i] + acc[(i + BN / 2) % Cfg::kAccRegs] : acc[i];
  };
  const int q = lane & 3;
  const float* head_vup = prob->head_vup;
  float* head_res = prob->head_res;
  float* head_v = prob->head_v;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    const int py = y0 + r / tile_w, px = x0 + r % tile_w;
    const bool valid = (py < prob->H) && (px < prob->W);
    const int64_t opix = ((int64_t)b * prob->out_H + ((int64_t)py * prob->out_sy + prob->out_oy)) * prob->out_W +
                         ((int64_t)px * prob->out_sx + prob->out_ox);
    if (epi_mode == 1) {
      // flow head: hidden = LeakyReLU(acc + b3) stays in fp32 registers; 2-wide linear layer + v_up
      float r0 = 0.f, r1 = 0.f;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j + 2 * q + e;
          const float hdn = leaky(value(h, j, e) + bias_smem[c]);
          r0 = fmaf(hdn, w4_smem[c * 2], r0);
          r1 = fmaf(hdn, w4_smem[c * 2 + 1], r1);
        }
      r0 += __shfl_xor_sync(0xffffffffu, r0, 1);
      r1 += __shfl_xor_sync(0xffffffffu, r1, 1);
      r0 += __shfl_xor_sync(0xffffffffu, r0, 2);
      r1 += __shfl_xor_sync(0xffffffffu, r1, 2);
      if (valid && q == 0) {
        float2 res = make_float2(r0 + w4_smem[2 * BN], r1 + w4_smem[2 * BN + 1]);
        float2 tot = res;
        if (head_vup) {
          const float2 u = reinterpret_cast<const float2*>(head_vup)[opix];
          tot.x += u.x;
          tot.y += u.y;
        }
        reinterpret_cast<float2*>(head_res)[opix] = res;
        reinterpret_cast<float2*>(head_v)[opix] = tot;
      }
    } else if (valid) {
      const int act = prob->act;
      sp_t* oh = prob->out_hi + opix * prob->out_C + prob->out_c_off + n0;
      sp_t* ol = prob->out_lo + opix * prob->out_C + prob->out_c_off + n0;
      const bool lo_skip = prob->out_lo_skip != 0;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + 2 * q;
        if (n0 + c >= cout) break;
        float f0 = value(h, j, 0) + bias_smem[c], f1 = value(h, j, 1) + bias_smem[c + 1];
        if (act) {
          f0 = leaky(f0);
          f1 = leaky(f1);
        }
        uint32_t hi, lo;
        if (lo_skip) {
          *reinterpret_cast<uint32_t*>(oh + c) = pack2_hi(f0, f1);
        } else {
          split_pack2(f0, f1, hi, lo);
          *reinterpret_cast<uint32_t*>(oh + c) = hi;
          *reinterpret_cast<uint32_t*>(ol + c) = lo;
        }
      }
    }
  }
}

template <int BN, int KC>
cudaError_t launch_bn(const ConvProblem* d_prob, const ConvProblem& h, cudaStream_t st) {
  dim3 grid(h.B * h.tiles_y * h.tiles_x, (h.cout + BN - 1) / BN, h.group > 1 ? h.group : 1);
  k_conv_tc<BN, KC><<<grid, kNumThreads, TcCfg<BN, KC>::kSmemBytes, st>>>(d_prob);
  return cudaGetLastError();
}

}  // namespace

int conv_tc_block_n(int cout) { return cout >= 256 ? 256 : cout >= 128 ? 128 : cout >= 64 ? 64 : 32; }

cudaError_t conv_tc_configure() {
  cudaError_t e;
#define FILM_CFG(BN, KC)                                                                         \
  e = cudaFuncSetAttribute(k_conv_tc<BN, KC>, cudaFuncAttributeMaxDynamicSharedMemorySize,      \
                           TcCfg<BN, KC>::kSmemBytes);                                           \
  if (e != cudaSuccess) return e;
  FILM_CFG(32, 64) FILM_CFG(64, 64) FILM_CFG(128, 64) FILM_CFG(256, 64) FILM_CFG(32, 32) FILM_CFG(64, 32)
#undef FILM_CFG
  return cudaSuccess;
}

cudaError_t launch_conv_tc(const ConvProblem* d_prob, const ConvProblem& h, cudaStream_t st) {
  const int bn = h.bn;
  if (h.kchunk == 32) {
    if (bn == 64) return launch_bn<64, 32>(d_prob, h, st);
    if (bn == 32) return launch_bn<32, 32>(d_prob, h, st);
    return cudaErrorInvalidValue;  // 32-channel K blocks are only instantiated for Cout <= 64
  }
  switch (bn) {
    case 256: return launch_bn<256, 64>(d_prob, h, st);
    case 128: return launch_bn<128, 64>(d_prob, h, st);
    case 64: return launch_bn<64, 64>(d_prob, h, st);
    default: return launch_bn<32, 64>(d_prob, h, st);
  }
}

}  // namespace film
