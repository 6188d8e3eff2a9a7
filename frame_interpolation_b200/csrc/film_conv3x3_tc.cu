// Persistent wgmma 3x3 convolution with activation-tile reuse across taps (sm_90a).
//
// Why a second kernel: the generic kernel re-loads the same activation pixels once per tap (9 x 32 KiB per
// 64-channel chunk and tile) and serialises prologue / mainloop / epilogue per tile.  Here:
//
//  * Tile = 16 rows x 8 columns of output pixels.  For a 64-channel chunk the producer loads
//    THREE boxes (dx = -1, 0, +1), each (64 ch, 8 px, 18 rows) of both planes: 144 pixel rows
//    of 128 B = 18 KiB per plane.  Because a tile row is exactly one 1024-byte swizzle atom
//    (8 px x 128 B), the operand of tap (dy, dx) is the SAME smem box at byte offset dy * 1024:
//    3 loads serve 9 taps (2.67x less L2 -> smem traffic) with plain, 1024-aligned descriptors.
//  * Weights: if the whole [Cout x K] hi+lo matrix fits (64->64, 128->32, 64->32 ...) it is loaded ONCE per CTA
//    and stays resident; otherwise it streams through its own ring, one tap ([BN x 64] hi+lo) per stage.
//  * Persistent CTAs (grid = #SMs) walk a static tile list; the producer runs ahead into the next tile's stages while
//    the consumers drain the accumulators of the current one.
//  * Two-accumulator product (BN <= 128): A_hi x W_hi and A_lo x W_hi accumulate into columns [0, BN) and A_hi x W_lo
//    into columns [BN, 2 BN) of one register accumulator, all as N = BN wgmma; the epilogue adds the halves.
//  * Pixels on N (kPxN: BN = 64 or 128, 64-channel chunks): a Cout = 64 layer would issue m64n64k16 with both operands
//    read from shared memory, 4 KiB of operand reads per 64x64x16 MACs.  This form computes D^T = W_tap x A^T instead:
//    each 64-row half of the weight tap [BN x 64] is an M = 64 A operand, the activation box the B operand, and each
//    consumer warpgroup owns 128 pixels (16 tile rows of 8) of a 32x8 tile, so every product is one m64n128k16 per
//    64-cout half (3 KiB per 64x64x16 MACs; BN = 128 pixels on M reads 6 KiB per 64x128x16) and each weight tap serves
//    256 pixels instead of 128, half the L2 -> SMEM weight traffic per MAC of the wide layers.  Cout = 256 / 512 run as
//    2 / 4 N tiles of 128.  The three products of the three-pass form share one accumulator per half (the engine runs
//    only single-pass layers at BN = 128: no register room to keep the cross products apart).  The transposed
//    accumulator holds couts on its rows: the epilogue stages each plane and 64-cout half through shared memory with
//    stmatrix.trans and stores whole 128-byte pixel rows; the fused 2x2 pool finds its partners in the thread's own
//    registers (column e ^ 1, row j + 1).
//  * Folded pixels on N (kPxN with BN = 32: the single-pass Cout = 32 convs of the level-0 flow predictor, KC = 64 or
//    32): 32 couts fill only half of M = 64, and m64n32k16 pixels-on-M products read 3 KiB of operands per 32K MACs.
//    Instead one [64 x KC] weight block holds two dy taps of a dx column (rows 0-31 tap dy, rows 32-63 tap dy + 1;
//    film_pack.h), and each warpgroup issues one m64n136k16 over 17 tile rows of the box at tap dy's offset: rows 0-31
//    of the accumulator hold its 16 output rows, rows 32-63 partial sums of the output one tile row up.  Per dx column
//    the pairs are (-1, 0) and (zero weights, +1), six products per chunk instead of nine taps.  The epilogue stages the
//    fp32 sums through shared memory, adds the lower half one pixel row up, and finishes one pixel per thread: the
//    split store, or the fused flow head (conv_3, conv_4 and the residual add) with its weights read as broadcasts.
//
// Roles: warp 8 (warpgroup 2, registers handed to the consumers) = TMA producer (+ L2 prefetch of the next tile's boxes; warp-uniform, one elected lane issues),
// warps 0-7 = two consumer warpgroups, each owning 64 (kPxN: 128) pixels of the tile: wgmma into register
// accumulators, then the epilogue from the registers (folded Cout = 32: through shared memory).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "film_conv.h"
#include "film_tc_ptx.cuh"

namespace film {
namespace {
using namespace tc;

constexpr int kConsumers = 256;
constexpr int kThreads = kConsumers + 128;   // + the producer warpgroup (one active warp)
// Tile shapes: tile_w must be a multiple of 8 pixels (one swizzle atom) and tile_h * tile_w = 128.
// 16x8 has the smallest halo (18/16); 8x16 and 4x32 exist to avoid wave quantisation on small levels.
__host__ __device__ constexpr int a_plane_bytes(int kc, int th, int tw) { return (th + 2) * tw * kc * 2; }
__host__ __device__ constexpr int a_stage_bytes(int kc, int th, int tw) { return 2 * a_plane_bytes(kc, th, tw); }
// Wide-halo mode (16x8 tiles, 32x8 with kPxN): ONE box (KC ch, 10 px, tile_h + 2 rows) per plane and chunk serves all
// nine taps -- the descriptor of tap (dy, dx) starts (dy * 10 + dx) pixel rows into the box and steps 10 pixel rows
// between 8-row groups.  2.4x less L2 -> smem activation traffic than the three dx-shifted boxes.
constexpr int kHaloW = 10;
__host__ __device__ constexpr int halo_box_bytes(int kc, int th) { return (th + 2) * kHaloW * kc * 2; }  // 23,040 for KC = 64, 16 rows
__host__ __device__ constexpr int halo_plane_bytes(int kc, int th) { return (halo_box_bytes(kc, th) + 1023) & ~1023; }  // 1 KiB-aligned planes
// `planes` = 2 (hi + lo, three-pass product) or 1 (single-pass layers load the hi planes only)
__host__ __device__ constexpr int a_stage_bytes_h(int kc, int th, int tw, int halo, int planes = 2) {
  return planes * (halo ? halo_plane_bytes(kc, th) : a_plane_bytes(kc, th, tw));
}
constexpr int kMaxRing = 8;
constexpr int kSmemLimit = 227 * 1024;
constexpr int kBarBytes = 8 * (4 * kMaxRing + 4);
constexpr int kFixedBytes = kBarBytes + 16 + 512 * 4 /*bias*/ + 64 /*src table: 16 ints*/ + 1024 /*align*/ + 64;
// flow-head epilogue (epi_mode 3): W3 [64][32] + b3 / W4 / b4, after the src table
constexpr int kHeadW3 = 64 * 32 * 4, kHeadMisc = 512;
constexpr int kHeadBytes = kHeadW3 + kHeadMisc;
// kPxN store epilogue, after the src table: per consumer warpgroup one plane of 64 pixels x 64 channels
constexpr int kPxnStageWg = 64 * 64 * 2;
constexpr int kPxnStageBytes = 2 * kPxnStageWg;
// folded Cout = 32 pixels-on-N epilogue, after the src table (and the flow head's scratch): per consumer warpgroup the
// fp32 sums of 32 couts x 128 pixels, rows 136 floats apart (conflict-free float2 stores from the fragments and
// conflict-free per-pixel reads)
constexpr int kFoldLd = 136;
constexpr int kFoldStageWg = 32 * kFoldLd * 4;
// shared memory of the epilogue scratch after the src table
inline int epi_scratch_bytes(int epi_mode, int pxn, int bn) {
  if (pxn && bn == 32) return (epi_mode == 3 ? kHeadBytes : 0) + 2 * kFoldStageWg;
  return epi_mode == 3 ? kHeadBytes : pxn ? kPxnStageBytes : 0;
}

// weight rows of one K block: BN, except the folded Cout = 32 pixels-on-N form, whose block holds two dy taps' 32 rows
__host__ __device__ constexpr int w_rows(int bn, int pxn) { return pxn && bn == 32 ? 64 : bn; }
__host__ __device__ inline int w_tap_bytes(int bn, int kc, int planes = 2) { return bn * kc * 2 * planes; }  // [BN x KC] hi (+ lo)

// Variants are template parameters chosen on the host (launch_conv3x3_tc): kPartial = the activation stages
// [v2_part_lo, v2_part_hi) of every tile read a source whose chunks hold data in their first 16-channel k-step only (the
// 10-of-64 "side" source, the 3-of-32 image block); the all-zero k-steps are skipped, and with kPxN the source's weights
// come packed one K block per dx column (film_pack.h), so each block serves three taps; kHalo = wide halo boxes; kOne =
// single-pass product A_hi x W_hi (hi planes only); kRes = resident weights issued as straight-line code (a whole
// activation stage is one wgmma group); kPxN = pixels on N (BN = 64 or 128, KC = 64, 32x8 tiles, store / pool epilogue
// only; BN = 32: the folded form, KC = 64 or 32, single-pass, store or flow-head epilogue).
template <int BN, int KC, bool kPartial, bool kHalo, bool kOne, bool kRes, bool kPxN = false>
__global__ void __launch_bounds__(kThreads, 1) k_conv3x3_tc(const ConvProblem* __restrict__ prob) {
  static_assert(!kPxN || ((BN == 64 || BN == 128) && KC == 64) || (BN == 32 && kOne && !kPartial),
                "pixels on N: one or two M = 64 weight tiles of 64-channel chunks, or the folded single-pass Cout = 32 form");
  extern __shared__ uint8_t smem_raw[];
  constexpr bool one = kOne;
  const int planes = one ? 1 : 2;
  // folded Cout = 32 pixels on N: each K block [64 x KC] holds two dy taps of one dx column, rows 0-31 tap dy and rows
  // 32-63 tap dy + 1, and every product is one m64n136k16 over 17 tile rows of the box at the offset of tap dy.  Rows
  // 32-63 then hold partial sums of the output one tile row up.  The pairs are (-1, 0) and (zero weights, +1): the
  // third tap read at the dy = 0 offset keeps the 17 rows inside the box, where zero weights never meet unloaded bytes
  constexpr bool kFold = kPxN && BN == 32;
  constexpr int kWPlane = w_rows(BN, kPxN) * KC * 2;  // one weight plane of one K block
  const int kWTap = kWPlane * planes;
  const int kTileH = prob->tile_h, kTileW = prob->tile_w;
  constexpr int kHaloTileH = kPxN ? 32 : 16;   // the only tile height of a wide-halo box
  constexpr int kHaloBox = halo_box_bytes(KC, kHaloTileH), kHaloPlane = halo_plane_bytes(KC, kHaloTileH);
  constexpr bool halo = kHalo;   // plan guarantees 16x8 (kPxN: 32x8) tiles
  const int kAPlane = halo ? kHaloPlane : a_plane_bytes(KC, kTileH, kTileW);
  const int kAStage = planes * kAPlane;
  const int kRowStep = kTileW * KC * 2;  // one tile row of pixels = tile_w/8 swizzle atoms
  constexpr bool kFused = BN <= 128 && !kPxN;
  constexpr int kMh = kPxN && !kFold ? BN / 64 : 1;                   // kPxN: M = 64 halves of the weight tile
  constexpr int kPxnN = kFold ? 136 : 128;                            // kPxN: pixel columns of one product
  constexpr int kAccRegs = kPxN ? kPxnN / 2 * kMh : (kFused ? 2 * BN : BN) / 2;   // kPxN: one m64nN f32 per half
  constexpr int kWgPx = kPxN ? 128 : 64;                              // pixels per consumer warpgroup

  // ---- problem fields -> registers, once (the asm "memory" clobbers would otherwise force a
  //      global reload of every P.* access inside the role loops)
  const int NA = prob->v2_na, NW = prob->v2_nw;
  const bool resident = prob->v2_resident != 0;
  const int nsrc = prob->nsrc;
  const int tiles_x = prob->tiles_x, tiles_per_img = prob->tiles_y * prob->tiles_x;
  const int cout = prob->cout;
  const int n_nt = (cout + BN - 1) / BN;                       // N tiles (Cout = 512 -> 2)
  const int ntiles = prob->B * tiles_per_img * n_nt;            // work items (spatial, N), N fastest
  constexpr int kStageTaps = kHalo ? 9 : 3;                     // taps served by one activation stage
  constexpr int kStageMmas = kFold ? 2 * kStageTaps / 3 : kStageTaps;   // products per stage: one per tap or dy pair
  // Pixels on N: the partial source's packed weight blocks each hold k-step 0 of the three dy taps of one dx column.
  // The 16x8 form keeps one block per tap: packing measured no faster there, and it made the BN = 128 and 256 partial
  // instantiations spill about three times as much
  constexpr bool kPacked = kPartial && kPxN;
  const int part_lo = prob->v2_part_lo, part_hi = prob->v2_part_hi;   // kPartial: 1-k-step stages
  int nab = 0;                                                  // activation stages: one halo box or three dx boxes per chunk
  for (int s = 0; s < nsrc; ++s) nab += prob->src[s].nchunk * (kHalo ? 1 : 3);
  // K blocks, in consumption order (source, chunk, dx, dy): one per tap, one per three taps in a packed partial stage,
  // two per dx column when folded
  const int nkb = nab * kStageMmas - (kPacked ? (part_hi - part_lo) * (kStageTaps - kStageTaps / 3) : 0);

  const FastDiv div_nt(n_nt, ntiles), div_img(tiles_per_img, ntiles), div_tx(tiles_x, ntiles);   // tile decode
  // CTA pair (prob->pair, launched as (2,1,1) clusters): the two CTAs of a cluster walk the same work list, each on its
  // own spatial tile of a neighbouring pair, with the same N tile and hence the same weight taps.  Each CTA loads half of
  // every streamed weight tap and multicasts it into both CTAs' weight rings: half the L2 -> SM weight traffic per CTA.
  const bool pair = prob->pair != 0;
  const int rank = pair ? (int)cluster_ctarank() : 0;
  const int nsp = prob->B * tiles_per_img;                      // spatial tiles
  const int nwork = pair ? ((nsp + 1) / 2) * n_nt : ntiles;
  const int w_first = pair ? (int)blockIdx.x >> 1 : (int)blockIdx.x, w_step = pair ? (int)gridDim.x >> 1 : (int)gridDim.x;
  auto decode = [&](int work, int& sp, int& nti) {   // -> spatial tile (>= nsp: the empty partner of an odd count), N tile
    div_nt.divmod(work, sp, nti);
    if (pair) sp = 2 * sp + rank;
  };

  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (base - raw);
  const uint32_t a_base = base;
  const uint32_t w_base = a_base + (uint32_t)NA * kAStage;
  const uint32_t w_bytes = resident ? (uint32_t)nkb * kWTap : (uint32_t)NW * kWTap;
  const uint32_t tail = w_base + w_bytes;
  const uint32_t tail_off = (uint32_t)NA * kAStage + w_bytes;
  // barrier k lives at tail + 8k: a_full[0..7], a_empty[8..15], w_full[16..23], w_empty[24..31]
  float* bias_smem = reinterpret_cast<float*>(gen_base + tail_off + kBarBytes + 16);
  int* src_tab = reinterpret_cast<int*>(gen_base + tail_off + kBarBytes + 16 + 512 * 4);  // {nchunk, c_off} x 4

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    for (int s = 0; s < kMaxRing; ++s) {
      mbar_init(tail + 8u * s, 1);
      mbar_init(tail + 8u * (kMaxRing + s), 2);       // one arrive per consumer warpgroup
      mbar_init(tail + 8u * (2 * kMaxRing + s), 1);
      mbar_init(tail + 8u * (3 * kMaxRing + s), pair ? 4 : 2);   // a pair's weight slot is free once both CTAs read it
    }
    for (int s = 0; s < kMaxSrc; ++s) {
      src_tab[2 * s] = s < nsrc ? prob->src[s].nchunk : 0;
      src_tab[2 * s + 1] = s < nsrc ? prob->src[s].c_off : 0;
      src_tab[2 * kMaxSrc + s] = s < nsrc ? prob->src[s].bswap : 0;
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp < 8)
    for (int i = threadIdx.x; i < n_nt * BN; i += kConsumers) bias_smem[i] = (i < cout) ? prob->bias[i] : 0.f;
  __syncthreads();
  if (pair) cluster_sync_all();   // the peer's barriers are initialised before any multicast or remote arrive
  // a CTA of a pair leaves only together with its peer: the peer's consumers still arrive on this CTA's barriers
  auto leave = [&]() {
    if (pair) cluster_sync_all();
  };

  if (warp >= 8) {
    regs_dec<40>();
    if (warp > 8) {
      leave();
      return;
    }
    // ============================ TMA producer (warp-uniform) ============================
    const CUtensorMap* tm_w_hi = &prob->tm_w_hi;
    const CUtensorMap* tm_w_lo = &prob->tm_w_lo;
    if (resident && elect_one()) {
      // whole weight matrix, once: nkb blocks of [BN x 64] hi then lo
      mbar_expect_tx(tail + 8u * (2 * kMaxRing), (uint32_t)nkb * kWTap);
      for (int kb = 0; kb < nkb; ++kb) {
        tma_load_2d(w_base + kb * kWTap, tm_w_hi, tail + 8u * (2 * kMaxRing), kb * KC, 0);
        if (!one) tma_load_2d(w_base + kb * kWTap + kWPlane, tm_w_lo, tail + 8u * (2 * kMaxRing), kb * KC, 0);
      }
    }
    __syncwarp();
    RingPos ra, rw;   // activation / weight ring positions
    for (int tile = w_first; tile < nwork; tile += w_step) {
      int sp, nti, b, rem, ty, tx;
      decode(tile, sp, nti);
      div_img.divmod(sp, b, rem);   // an empty partner tile decodes to b = B: every TMA box is out of bounds (zeros)
      div_tx.divmod(rem, ty, tx);
      const int n0 = nti * BN, y0 = ty * kTileH, x0 = tx * kTileW;
      {
        // L2 prefetch of this CTA's NEXT spatial tile: first touch of an activation tile is DRAM
        const int nt = tile + w_step;
        int next_sp, nnt;
        decode(nt < nwork ? nt : 0, next_sp, nnt);
        if (nt < nwork && next_sp != sp && next_sp < nsp && elect_one()) {
          int nb, nrem, nty, ntx;
          div_img.divmod(next_sp, nb, nrem);
          div_tx.divmod(nrem, nty, ntx);
          const int ny0 = nty * kTileH, nx0 = ntx * kTileW;
          for (int s = 0; s < nsrc; ++s)
            for (int ch = 0; ch < src_tab[2 * s]; ++ch) {
              // the three dx boxes overlap: boxes at dx = 0 and dx = 2 cover the (tile_w + 2)-px-wide halo
              const int cc = src_tab[2 * s + 1] + ch * KC;
              tma_prefetch_4d(&prob->tm_a_hi[s], cc, nx0 - 1, ny0 - 1, nb);
              if (!one) tma_prefetch_4d(&prob->tm_a_lo[s], cc, nx0 - 1, ny0 - 1, nb);
              if (!halo) {  // (the wide box already spans the halo)
                tma_prefetch_4d(&prob->tm_a_hi[s], cc, nx0 + 1, ny0 - 1, nb);
                if (!one) tma_prefetch_4d(&prob->tm_a_lo[s], cc, nx0 + 1, ny0 - 1, nb);
              }
            }
        }
        __syncwarp();
      }
      int kb = 0, ab = 0;
      for (int s = 0; s < nsrc; ++s) {
        const int nchunk = src_tab[2 * s], c_off = src_tab[2 * s + 1];
        const int bs = src_tab[2 * kMaxSrc + s] ? prob->B - 1 - b : b;
        const CUtensorMap* tm_hi = &prob->tm_a_hi[s];
        const CUtensorMap* tm_lo = &prob->tm_a_lo[s];
        for (int ch = 0; ch < nchunk; ++ch) {
          const int nst = halo ? 1 : 3;   // activation stages of this chunk: one wide halo box or three dx boxes
          for (int dx = 0; dx < nst; ++dx, ++ab) {
            const int st = ra.stage;
            mbar_wait(tail + 8u * (kMaxRing + st), ra.phase ^ 1u);
            if (elect_one()) {
              const uint32_t sa = a_base + st * kAStage, bar = tail + 8u * st;
              mbar_expect_tx(bar, halo ? (uint32_t)(planes * kHaloBox) : (uint32_t)kAStage);
              tma_load_4d(sa, tm_hi, bar, c_off + ch * KC, x0 + dx - 1, y0 - 1, bs);
              if (!one) tma_load_4d(sa + kAPlane, tm_lo, bar, c_off + ch * KC, x0 + dx - 1, y0 - 1, bs);
            }
            __syncwarp();
            ra.advance(NA);
            if (!resident) {
              // weight blocks consumed against this activation stage: one per tap, one per dx column when packed
              const bool packed = kPacked && ab >= part_lo && ab < part_hi;
              const int nblk = packed ? kStageTaps / 3 : kStageMmas;
              for (int t = 0; t < nblk; ++t, ++kb) {
                const int ws = rw.stage;
                mbar_wait(tail + 8u * (3 * kMaxRing + ws), rw.phase ^ 1u);
                if (elect_one()) {
                  const uint32_t sw = w_base + ws * kWTap, bar = tail + 8u * (2 * kMaxRing + ws);
                  mbar_expect_tx(bar, kWTap);
                  if (pair) {   // this CTA's half of the tap's rows, into the same slot of both CTAs
                    const uint32_t hoff = (uint32_t)(rank * (kWPlane / 2));
                    tma_load_2d_mc(sw + hoff, &prob->tm_w_hi_half, bar, kb * KC, n0 + rank * (BN / 2), 3);
                    if (!one) tma_load_2d_mc(sw + kWPlane + hoff, &prob->tm_w_lo_half, bar, kb * KC, n0 + rank * (BN / 2), 3);
                  } else {
                    tma_load_2d(sw, tm_w_hi, bar, kb * KC, n0);
                    if (!one) tma_load_2d(sw + kWPlane, tm_w_lo, bar, kb * KC, n0);
                  }
                }
                __syncwarp();
                rw.advance(NW);
              }
            }
          }
        }
      }
    }
    leave();
    return;
  }

  // ============================ consumer warpgroups: MMA + epilogue ============================
  regs_inc<232>();
  const int wg = warp >> 2;        // pixels [kWgPx wg, kWgPx (wg + 1)) of the tile
  const int q = lane & 3;
  const int H = prob->H, W = prob->W, out_H = prob->out_H, out_W = prob->out_W, out_C = prob->out_C;
  const int out_c_off = prob->out_c_off, act = prob->act;
  sp_t* const out_hi = prob->out_hi;
  sp_t* const out_lo = prob->out_lo;
  // fused 2x2/2 average pool: only for 16x8 tiles, where the 2x2 partners of the pixel in fragment row r0 are the
  // same thread's row r0 + 8 (next tile row) and lane ^ 4 (next column)
  sp_t* const pool_hi = prob->pool_hi;
  sp_t* const pool_lo = prob->pool_lo;
  const int pool_C = prob->pool_C;
  const bool do_pool = pool_hi != nullptr;
  const bool lo_skip = prob->out_lo_skip != 0;
  // RGB-head mode: channel partial sums of the 1x1 64 -> 3 conv, reduced over the four lanes that share a pixel
  const bool rgb = prob->epi_mode == 2;
  const float* const head_w = prob->head_w4;
  float* const rgb_out = prob->head_v;
  const int crop_y = prob->crop_y, crop_x = prob->crop_x, crop_h = prob->crop_h, crop_w = prob->crop_w;
  const int64_t crop_pitch = prob->crop_pitch;
  // flow-head mode (BN <= 64): hidden units = BN / 2; each lane accumulates the partial sums of its channels for every
  // hidden unit, the four lanes of a pixel combine with shuffles and finish the head
  const bool fhead = prob->epi_mode == 3;
  constexpr int kHid = BN <= 64 ? BN / 2 : 1;
  float* const w3s = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(src_tab) + 64);   // [BN][kHid]
  float* const hmisc = w3s + kHeadW3 / 4;                                                  // b3[kHid] | w4[kHid][2] | b4[2]
  if (fhead) {
    if constexpr (BN <= 64) {
      for (int i = threadIdx.x; i < BN * kHid; i += kConsumers) w3s[i] = prob->head_w3[i];
      for (int i = threadIdx.x; i < kHid; i += kConsumers) hmisc[i] = prob->head_b3[i];
      for (int i = threadIdx.x; i < 2 * kHid; i += kConsumers) hmisc[kHid + i] = prob->head_w4[i];
      if (threadIdx.x < 2) hmisc[3 * kHid + threadIdx.x] = prob->head_b4[threadIdx.x];
    }
    asm volatile("bar.sync 1, %0;" ::"r"(kConsumers) : "memory");   // consumer warps only
  }
  const float* const head_vup = prob->head_vup;
  float* const head_res = prob->head_res;
  float* const head_vout = prob->head_v;

  if (resident) mbar_wait(tail + 8u * (2 * kMaxRing), 0);
  const bool is_leader = (threadIdx.x & 127) == 0;
  const uint32_t w_empty_peer = pair ? map_to_cta(tail + 8u * (3 * kMaxRing), (uint32_t)(rank ^ 1)) : 0u;
  auto release_w = [&](int slot) {
    mbar_arrive(tail + 8u * (3 * kMaxRing + slot));
    if (pair) mbar_arrive_cluster(w_empty_peer + 8u * slot);
  };
  {
    constexpr int kWTapC = kWPlane * (kOne ? 1 : 2);
    constexpr uint32_t kPx = KC * 2;            // bytes of one pixel row of a box
    // first pixel row of this warpgroup's pixels inside the box, and the stride between its 8-row groups
    const uint32_t a_row0 = kHalo ? (uint32_t)(wg * (kWgPx / 8) * kHaloW) * kPx : (uint32_t)(wg * kWgPx) * kPx;
    const uint32_t sbo = kHalo ? kHaloW * kPx : 8 * kPx;
    RingPos ra, rw;   // activation / weight ring positions
    float acc[kAccRegs];
    // tap (3 dx + dy, dx-major within the stage) whose box offset product m of an activation stage reads: the folded
    // form's products read at the upper tap of their dy pair, (-1, 0) and (zero, +1) of each dx column
    auto tap_of = [](int m) { return kFold ? (kHalo ? 3 * (m / 2) : 0) + m % 2 : m; };
    // pixels on N: half h of the weight tap (rows 64 h .. 64 h + 63, one 8 KiB run of 1 KiB swizzle atoms) into
    // accumulator registers [64 h, 64 h + 64)
    auto pxn_mma = [&](uint64_t w_hi, uint64_t w_lo, uint64_t a_hi, uint64_t a_lo, uint32_t accf) {
#pragma unroll
      for (int h = 0; h < kMh; ++h) {
        const uint64_t wh = (uint64_t)(h * (64 * KC * 2) >> 4);
        wgmma<kPxnN>(acc + 64 * h, w_hi + wh, a_hi, accf);
        if constexpr (!kOne) {
          wgmma<kPxnN>(acc + 64 * h, w_lo + wh, a_hi, 1u);
          wgmma<kPxnN>(acc + 64 * h, w_hi + wh, a_lo, 1u);
        }
      }
    };
    for (int tile = w_first; tile < nwork; tile += w_step) {
      int kb = 0;
      int rel_a = -1, rel_w = -1;   // stages read by the previous wgmma group, released once it retired
      auto retire = [&](int next_a, int next_w) {
        wgmma_commit();
        wgmma_wait<1>();
        if (is_leader) {
          if (rel_a >= 0) mbar_arrive(tail + 8u * (kMaxRing + rel_a));
          if (rel_w >= 0) release_w(rel_w);
        }
        rel_a = next_a;
        rel_w = next_w;
      };
      // One activation stage whose products each issue kSteps k-steps (a compile-time count: ptxas serialises every
      // wgmma of a kernel in which a runtime condition picks between wgmma sequences, C7520).  kTpb taps share one
      // weight block, their k-steps back to back in it: 3 in a packed partial stage (k-step 0 of each dy tap), else 1
      auto stage = [&](auto ksteps_c, auto tpb_c) {
        constexpr int kSteps = decltype(ksteps_c)::value, kTpb = decltype(tpb_c)::value;
        constexpr int kBlocks = kStageMmas / kTpb;   // weight blocks read against this stage
        const int st = ra.stage;
        mbar_wait(tail + 8u * st, ra.phase);
        const uint32_t sa = a_base + st * kAStage + a_row0;
        const uint32_t lo_off = (uint32_t)(kHalo ? kHaloPlane : kAPlane);
        if constexpr (kRes) {
          // Resident weights: nothing to wait for inside the stage, so all of its taps are one wgmma group issued as
          // straight-line code with compile-time descriptor offsets
          const uint64_t a0 = make_desc_sbo<KC>(sa, sbo);
          const uint64_t lo_delta = (uint64_t)(lo_off >> 4);
          const uint64_t row_delta = (uint64_t)(kRowStep >> 4);
          const uint64_t w0 = make_desc_kc<KC>(w_base + kb * kWTapC);
          const uint32_t first = (kb == 0) ? 0u : 1u;
          wgmma_fence();
#pragma unroll
          for (int mi = 0; mi < kStageMmas; ++mi) {
            const int t = tap_of(mi);
            const uint64_t a_hi = a0 + (kHalo ? (uint64_t)((((t % 3) * kHaloW + t / 3) * kPx) >> 4) : (uint64_t)t * row_delta);
            const uint64_t a_lo = a_hi + lo_delta;
            const uint64_t w_hi = w0 + (uint64_t)(((mi / kTpb) * kWTapC + (mi % kTpb) * kSteps * 32) >> 4);
            const uint64_t w_lo = w_hi + (uint64_t)(kWPlane >> 4);
#pragma unroll
            for (int k = 0; k < kSteps; ++k) {
              const uint64_t adv = (uint64_t)(k * 32 >> 4);
              const uint32_t accf = (mi == 0 && k == 0) ? first : 1u;
              if constexpr (kPxN) {   // D^T += W x A^T: each 64-row half of the weight tap is an M = 64 operand
                pxn_mma(w_hi + adv, w_lo + adv, a_hi + adv, a_lo + adv, accf);
              } else if constexpr (kOne) {
                wgmma<BN>(acc, a_hi + adv, w_hi + adv, accf);
              } else if constexpr (kFused) {
                wgmma<BN>(acc, a_hi + adv, w_hi + adv, accf);
                wgmma<BN>(acc + BN / 2, a_hi + adv, w_lo + adv, accf);
                wgmma<BN>(acc, a_lo + adv, w_hi + adv, 1u);
              } else {
                wgmma<BN>(acc, a_lo + adv, w_hi + adv, accf);
                wgmma<BN>(acc, a_hi + adv, w_lo + adv, 1u);
                wgmma<BN>(acc, a_hi + adv, w_hi + adv, 1u);
              }
            }
          }
          retire(st, -1);
          kb += kBlocks;
        } else {
          for (int blk = 0; blk < kBlocks; ++blk, ++kb) {
            uint32_t sw;
            int ws = -1;
            if (resident) {
              sw = w_base + kb * kWTap;
            } else {
              ws = rw.stage;
              mbar_wait(tail + 8u * (2 * kMaxRing + ws), rw.phase);
              sw = w_base + ws * kWTap;
            }
            const uint32_t first = (kb == 0) ? 0u : 1u;
            wgmma_fence();
#pragma unroll
            for (int u = 0; u < kTpb; ++u) {
              const int t = tap_of(blk * kTpb + u);
              const uint32_t off = kHalo ? (uint32_t)((t % 3) * kHaloW + t / 3) * kPx : (uint32_t)(t * kRowStep);
              const uint64_t a_hi = make_desc_sbo<KC>(sa + off, sbo);
              const uint64_t a_lo = make_desc_sbo<KC>(sa + lo_off + off, sbo);
              const uint64_t wk = (uint64_t)((u * kSteps * 32) >> 4);   // the tap's first k-step inside the block
              const uint64_t w_hi = make_desc_kc<KC>(sw) + wk, w_lo = make_desc_kc<KC>(sw + kWPlane) + wk;
#pragma unroll
              for (int k = 0; k < kSteps; ++k) {
                const uint64_t adv = (uint64_t)(k * 32 >> 4);
                const uint32_t accf = (u == 0 && k == 0) ? first : 1u;
                if constexpr (kPxN) {
                  pxn_mma(w_hi + adv, w_lo + adv, a_hi + adv, a_lo + adv, accf);
                } else if constexpr (kOne) {
                  wgmma<BN>(acc, a_hi + adv, w_hi + adv, accf);
                } else if constexpr (kFused) {
                  wgmma<BN>(acc, a_hi + adv, w_hi + adv, accf);
                  wgmma<BN>(acc + BN / 2, a_hi + adv, w_lo + adv, accf);
                  wgmma<BN>(acc, a_lo + adv, w_hi + adv, 1u);
                } else {
                  wgmma<BN>(acc, a_lo + adv, w_hi + adv, accf);
                  wgmma<BN>(acc, a_hi + adv, w_lo + adv, 1u);
                  wgmma<BN>(acc, a_hi + adv, w_hi + adv, 1u);
                }
              }
            }
            retire(blk == kBlocks - 1 ? st : -1, ws);
            if (!resident) rw.advance(NW);
          }
        }
        ra.advance(NA);
      };
      // the partial source's stages run in a loop of their own: no condition between alternative wgmma sequences
      using Full = std::integral_constant<int, KC / 16>;
      using One = std::integral_constant<int, 1>;
      if constexpr (kPartial) {
        for (int ab = 0; ab < part_lo; ++ab) stage(Full{}, One{});
        for (int ab = part_lo; ab < part_hi; ++ab) stage(One{}, std::integral_constant<int, kPacked ? 3 : 1>{});
        for (int ab = part_hi; ab < nab; ++ab) stage(Full{}, One{});
      } else {
        for (int ab = 0; ab < nab; ++ab) stage(Full{}, One{});
      }
      wgmma_wait<0>();
      if (is_leader) {
        if (rel_a >= 0) mbar_arrive(tail + 8u * (kMaxRing + rel_a));
        if (rel_w >= 0) release_w(rel_w);
      }
      acc_fence<kAccRegs>(acc);

      // ---------------- epilogue from the registers ----------------
      int sp, nti, b, rem, ty, tx;
      decode(tile, sp, nti);
      div_img.divmod(sp, b, rem);
      div_tx.divmod(rem, ty, tx);
      const int n0 = nti * BN;
      const bool live = sp < nsp;   // false: the empty partner of an odd tile count stores nothing
      if constexpr (kFold) {
        // Register 4j + 2h + e holds weight row 16 (warp & 3) + lane / 4 + 8h at box column j (tile row 16 wg + j for
        // rows 0-31, 16 wg + j - 1 for rows 32-63, j = 0 .. 16) and pixel column 2q + e.  The upper warps store their
        // rows' sums, the lower warps add theirs one tile row up, and then each thread finishes one pixel
        float* const stg = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(src_tab) + 64 + (fhead ? kHeadBytes : 0) +
                                                    wg * kFoldStageWg);
        auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory"); };
        const bool lower = (warp & 2) != 0;
        const int r0 = 16 * (warp & 1) + (lane >> 2);
        wg_sync();   // the previous tile's reads are done
        if (!lower) {
#pragma unroll
          for (int j = 0; j < 16; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
              *reinterpret_cast<float2*>(stg + (r0 + 8 * h) * kFoldLd + 8 * j + 2 * q) =
                  make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
        wg_sync();
        if (lower) {
#pragma unroll
          for (int j = 1; j < 17; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float2* d = reinterpret_cast<float2*>(stg + (r0 + 8 * h) * kFoldLd + 8 * (j - 1) + 2 * q);
              const float2 v = *d;
              *d = make_float2(v.x + acc[4 * j + 2 * h], v.y + acc[4 * j + 2 * h + 1]);
            }
        }
        wg_sync();
        const int p = threadIdx.x & 127;
        const int py = ty * kTileH + 16 * wg + (p >> 3), px = tx * kTileW + (p & 7);
        const int64_t opix = ((int64_t)b * out_H + py) * out_W + px;
        float f[32];
#pragma unroll
        for (int c = 0; c < 32; ++c) {
          const float x = stg[c * kFoldLd + p] + bias_smem[c];
          f[c] = act ? leaky(x) : x;
        }
        if (!live || py >= H || px >= W) {
        } else if (fhead) {
          // conv_3 (32 -> 16, bias, LeakyReLU), conv_4 (16 -> 2) and the residual add of the flow head
          float hp[16];
#pragma unroll
          for (int hh = 0; hh < 16; ++hh) hp[hh] = 0.f;
#pragma unroll
          for (int c = 0; c < 32; ++c) {
            const float4* wr = reinterpret_cast<const float4*>(w3s + c * 16);
#pragma unroll
            for (int h4 = 0; h4 < 4; ++h4) {
              const float4 wv = wr[h4];
              hp[4 * h4] = fmaf(f[c], wv.x, hp[4 * h4]);
              hp[4 * h4 + 1] = fmaf(f[c], wv.y, hp[4 * h4 + 1]);
              hp[4 * h4 + 2] = fmaf(f[c], wv.z, hp[4 * h4 + 2]);
              hp[4 * h4 + 3] = fmaf(f[c], wv.w, hp[4 * h4 + 3]);
            }
          }
          float f0 = hmisc[3 * 16], f1 = hmisc[3 * 16 + 1];
#pragma unroll
          for (int hh = 0; hh < 16; ++hh) {
            const float x = leaky(hp[hh] + hmisc[hh]);
            f0 = fmaf(x, hmisc[16 + 2 * hh], f0);
            f1 = fmaf(x, hmisc[16 + 2 * hh + 1], f1);
          }
          float2 res = make_float2(f0, f1), tot = res;
          if (head_vup) {
            const float2 u = reinterpret_cast<const float2*>(head_vup)[opix];
            tot.x += u.x;
            tot.y += u.y;
          }
          reinterpret_cast<float2*>(head_res)[opix] = res;
          reinterpret_cast<float2*>(head_vout)[opix] = tot;
        } else {
          sp_t* const oh = out_hi + opix * out_C + out_c_off;
          sp_t* const ol = out_lo + opix * out_C + out_c_off;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) split_pack2(f[8 * k + 2 * i], f[8 * k + 2 * i + 1], hi[i], lo[i]);
            *reinterpret_cast<uint4*>(oh + 8 * k) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            if (!lo_skip) *reinterpret_cast<uint4*>(ol + 8 * k) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
          }
        }
        continue;
      }
      if constexpr (kPxN && !kFold) {
        // Transposed accumulator: register 64 m + 4j + 2h + e holds cout n0 + 64 m + c0 + 8h and pixel (tile row
        // 16 wg + j, column 2q + e)
        const int c0 = 16 * (warp & 3) + (lane >> 2);
#pragma unroll
        for (int m = 0; m < kMh; ++m) {
          const float bias0 = bias_smem[n0 + 64 * m + c0], bias1 = bias_smem[n0 + 64 * m + c0 + 8];
#pragma unroll
          for (int i = 64 * m; i < 64 * m + 64; ++i) {
            const float f = acc[i] + ((i & 2) ? bias1 : bias0);
            acc[i] = act ? leaky(f) : f;
          }
        }
        const int y_wg = ty * kTileH + 16 * wg, x_t = tx * kTileW;
        if (do_pool) {
          // 2x2 partners in the thread's own registers: the next column is e ^ 1, the next row is j + 1.  The lane of
          // the odd cout (lane ^ 4) hands its sum over, and the even-cout lane stores the pair.  A pooled pixel is
          // written only when its whole 2x2 window is inside the frame (VALID pooling floors odd sizes)
          const int px = x_t + 2 * q;
#pragma unroll
          for (int j = 0; j < 16; j += 2) {
            const int py = y_wg + j;
            const bool ok = live && (py >> 1) < (out_H >> 1) && (px >> 1) < (out_W >> 1) && !(lane & 4);
            const int64_t ppix = ((int64_t)b * (out_H >> 1) + (py >> 1)) * (out_W >> 1) + (px >> 1);
#pragma unroll
            for (int m = 0; m < kMh; ++m)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int i = 64 * m + 4 * j + 2 * h;
                const float v = ((acc[i] + acc[i + 1]) + (acc[i + 4] + acc[i + 5])) * 0.25f;
                const float vn = __shfl_xor_sync(0xffffffffu, v, 4);
                if (ok) {
                  uint32_t hi, lo;
                  split_pack2(v, vn, hi, lo);
                  const int64_t pc = ppix * pool_C + n0 + 64 * m + c0 + 8 * h;
                  *reinterpret_cast<uint32_t*>(pool_hi + pc) = hi;
                  *reinterpret_cast<uint32_t*>(pool_lo + pc) = lo;
                }
              }
          }
        }
        // Split store: each plane and 64-cout half goes through shared memory 64 pixels at a time.  stmatrix.trans
        // writes 8 couts of one pixel as one 16-byte row (chunk cout / 8 of the pixel's 128 bytes, XOR-swizzled by
        // pixel % 8: conflict-free); eight consecutive threads then store one pixel's 128 bytes of the half
        uint8_t* const stg = reinterpret_cast<uint8_t*>(src_tab) + 64 + wg * kPxnStageWg;
        const uint32_t stg_u = smem_u32(stg);
        const int t128 = threadIdx.x & 127;
        auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory"); };
        for (int pl = 0; pl < (lo_skip ? 1 : 2); ++pl) {
          sp_t* const dst = (pl ? out_lo : out_hi) + out_c_off + n0;
#pragma unroll
          for (int m = 0; m < kMh; ++m)
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              wg_sync();   // the previous round's reads are done
#pragma unroll
              for (int jj = 0; jj < 8; jj += 2) {
                uint32_t r[4];   // matrices (j, h) = (jj, 0), (jj, 1), (jj + 1, 0), (jj + 1, 1)
#pragma unroll
                for (int mm = 0; mm < 4; ++mm) {
                  const int i = 64 * m + 4 * (8 * half + jj + (mm >> 1)) + 2 * (mm & 1);
                  if (pl) {
                    uint32_t hi;
                    split_pack2(acc[i], acc[i + 1], hi, r[mm]);
                  } else {
                    r[mm] = pack2_hi(acc[i], acc[i + 1]);
                  }
                }
                // this lane addresses row (lane & 7) of matrix lane >> 3: pixel 8 (jj + lane / 16) + lane % 8 of the half
                const int p = 8 * (jj + (lane >> 4)) + (lane & 7), ch = 2 * (warp & 3) + ((lane >> 3) & 1);
                stmatrix_x4_trans(stg_u + p * 128 + ((ch ^ (p & 7)) << 4), r[0], r[1], r[2], r[3]);
              }
              wg_sync();
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const int idx = 128 * k + t128, p = idx >> 3, ch = idx & 7;
                const int py = y_wg + 8 * half + (p >> 3), px = x_t + (p & 7);
                if (live && py < H && px < W) {
                  const uint4 v = *reinterpret_cast<const uint4*>(stg + p * 128 + ((ch ^ (p & 7)) << 4));
                  const int64_t opix = ((int64_t)b * out_H + py) * out_W + px;
                  *reinterpret_cast<uint4*>(dst + opix * out_C + 64 * m + 8 * ch) = v;
                }
              }
            }
        }
        continue;
      }
      auto value = [&](int h, int j, int e) {
        const int i = 4 * j + 2 * h + e;
        return (kFused && !kOne) ? acc[i] + acc[(i + BN / 2) % kAccRegs] : acc[i];
      };
      // RGB / flow heads: one fragment row (pixel) at a time
#pragma unroll
      for (int h = 0; h < 2 && (fhead || rgb); ++h) {
        const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        const int py = ty * kTileH + r / kTileW, px = tx * kTileW + r % kTileW;
        const bool valid = live && (py < H) && (px < W);
        const int64_t opix = ((int64_t)b * out_H + py) * out_W + px;
        if (fhead) {
          if constexpr (BN <= 64) {
            float hp[kHid];
#pragma unroll
            for (int hh = 0; hh < kHid; ++hh) hp[hh] = 0.f;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int c = 8 * j + 2 * q + e;
                const float x = value(h, j, e) + bias_smem[n0 + c];
                const float f = act ? leaky(x) : x;
                const float4* wr = reinterpret_cast<const float4*>(w3s + c * kHid);
#pragma unroll
                for (int h4 = 0; h4 < kHid / 4; ++h4) {
                  const float4 wv = wr[h4];
                  hp[4 * h4] = fmaf(f, wv.x, hp[4 * h4]);
                  hp[4 * h4 + 1] = fmaf(f, wv.y, hp[4 * h4 + 1]);
                  hp[4 * h4 + 2] = fmaf(f, wv.z, hp[4 * h4 + 2]);
                  hp[4 * h4 + 3] = fmaf(f, wv.w, hp[4 * h4 + 3]);
                }
              }
#pragma unroll
            for (int hh = 0; hh < kHid; ++hh) {
              hp[hh] += __shfl_xor_sync(0xffffffffu, hp[hh], 1);
              hp[hh] += __shfl_xor_sync(0xffffffffu, hp[hh], 2);
            }
            if (q == 0 && valid) {
              float f0 = hmisc[3 * kHid], f1 = hmisc[3 * kHid + 1];
#pragma unroll
              for (int hh = 0; hh < kHid; ++hh) {
                const float x = leaky(hp[hh] + hmisc[hh]);       // conv_3: bias + LeakyReLU
                f0 = fmaf(x, hmisc[kHid + 2 * hh], f0);            // conv_4: linear
                f1 = fmaf(x, hmisc[kHid + 2 * hh + 1], f1);
              }
              float2 res = make_float2(f0, f1), tot = res;
              if (head_vup) {
                const float2 u = reinterpret_cast<const float2*>(head_vup)[opix];
                tot.x += u.x;
                tot.y += u.y;
              }
              reinterpret_cast<float2*>(head_res)[opix] = res;
              reinterpret_cast<float2*>(head_vout)[opix] = tot;
            }
          }
        } else if (rgb) {
          float r0 = 0.f, r1 = 0.f, r2 = 0.f;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = n0 + 8 * j + 2 * q + e;
              float f = value(h, j, e) + bias_smem[c];
              if (act) f = leaky(f);
              r0 = fmaf(f, __ldg(head_w + 3 * c), r0);
              r1 = fmaf(f, __ldg(head_w + 3 * c + 1), r1);
              r2 = fmaf(f, __ldg(head_w + 3 * c + 2), r2);
            }
#pragma unroll
          for (int m = 1; m <= 2; m <<= 1) {
            r0 += __shfl_xor_sync(0xffffffffu, r0, m);
            r1 += __shfl_xor_sync(0xffffffffu, r1, m);
            r2 += __shfl_xor_sync(0xffffffffu, r2, m);
          }
          const int oy = py - crop_y, ox = px - crop_x;
          if (q == 0 && valid && oy >= 0 && oy < crop_h && ox >= 0 && ox < crop_w) {
            float* o = rgb_out + (int64_t)oy * crop_pitch + (int64_t)ox * 3;
            o[0] = r0 + __ldg(prob->head_b4);
            o[1] = r1 + __ldg(prob->head_b4 + 1);
            o[2] = r2 + __ldg(prob->head_b4 + 2);
          }
        }
      }
      if (!fhead && !rgb) {
        // split stores, channel block outermost: both fragment rows of a block are at hand together, so the fused pool
        // combines tile rows y (r0) and y + 1 (r0 + 8) without holding a whole row of partial sums
        bool valid[2];
        int64_t opix[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
          const int py = ty * kTileH + r / kTileW, px = tx * kTileW + r % kTileW;
          valid[h] = live && (py < H) && (px < W);
          opix[h] = ((int64_t)b * out_H + py) * out_W + px;
        }
        // the lane with the even tile column of row r0 owns the pooled pixel (pool implies 16x8 tiles).  It is written
        // only when the whole 2x2 window is inside the frame: VALID pooling floors odd sizes
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int py0 = ty * kTileH + r0 / kTileW, px0 = tx * kTileW + r0 % kTileW;
        const bool pool_ok = live && (py0 >> 1) < (out_H >> 1) && (px0 >> 1) < (out_W >> 1) && !(lane & 4);
        const int64_t ppix = ((int64_t)b * (out_H >> 1) + (py0 >> 1)) * (out_W >> 1) + (px0 >> 1);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = 8 * j + 2 * q;
          if (n0 + c >= cout) break;
          float a[2][2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float f0 = value(h, j, 0) + bias_smem[n0 + c], f1 = value(h, j, 1) + bias_smem[n0 + c + 1];
            if (act) {
              f0 = leaky(f0);
              f1 = leaky(f1);
            }
            if (valid[h]) {
              sp_t* oh = out_hi + opix[h] * out_C + out_c_off + n0;
              if (lo_skip) {
                *reinterpret_cast<uint32_t*>(oh + c) = pack2_hi(f0, f1);
              } else {
                sp_t* ol = out_lo + opix[h] * out_C + out_c_off + n0;
                uint32_t hi, lo;
                split_pack2(f0, f1, hi, lo);
                *reinterpret_cast<uint32_t*>(oh + c) = hi;
                *reinterpret_cast<uint32_t*>(ol + c) = lo;
              }
            }
            if (do_pool) {   // x-pair sums: the next tile column is lane ^ 4
              a[h][0] = f0 + __shfl_xor_sync(0xffffffffu, f0, 4);
              a[h][1] = f1 + __shfl_xor_sync(0xffffffffu, f1, 4);
            }
          }
          if (do_pool && pool_ok) {
            uint32_t hi, lo;
            split_pack2((a[0][0] + a[1][0]) * 0.25f, (a[0][1] + a[1][1]) * 0.25f, hi, lo);
            *reinterpret_cast<uint32_t*>(pool_hi + ppix * pool_C + n0 + c) = hi;
            *reinterpret_cast<uint32_t*>(pool_lo + ppix * pool_C + n0 + c) = lo;
          }
        }
      }
    }
  }
  leave();
}

int smem_bytes_for(const ConvProblem& h, int bn) {
  const int nkb = h.ktot / h.kchunk;
  const int planes = h.passes == 1 ? 1 : 2;
  const int wtap = w_tap_bytes(w_rows(bn, h.pxn), h.kchunk, planes);
  const int w = h.v2_resident ? nkb * wtap : h.v2_nw * wtap;
  return h.v2_na * a_stage_bytes_h(h.kchunk, h.tile_h, h.tile_w, h.halo, planes) + w + kFixedBytes +
         epi_scratch_bytes(h.epi_mode, h.pxn, bn);
}

}  // namespace

int conv_tc_block_n(int cout);

namespace {
// Resident or streamed weights and the ring depths for one tile shape.  A consumer warpgroup releases a stage only once
// the wgmma group AFTER the one that read it has been committed, and that group reads the next stage of the same
// ring: both rings therefore need at least two slots, or producer and consumers wait on each other forever.
// Returns false when the shape cannot get them within the shared-memory budget.
bool ring_depths(int kc, int tile_h, int tile_w, int halo, int planes, int bn, int cout, int ktot, int epi_mode, int pxn,
                 int& resident, int& na, int& nw) {
  const int wtap = w_tap_bytes(w_rows(bn, pxn), kc, planes);
  const int w_all = (ktot / kc) * wtap;
  const int kLimit = kSmemLimit - epi_scratch_bytes(epi_mode, pxn, bn);   // flow-head / pixels-on-N store scratch
  const int kAStage = a_stage_bytes_h(kc, tile_h, tile_w, halo, planes);
  if (cout <= bn && w_all + 2 * kAStage + kFixedBytes <= kLimit) {
    resident = 1;
    const int n = (kLimit - kFixedBytes - w_all) / kAStage;
    const int n_max = halo ? 3 : 6;
    na = n > n_max ? n_max : n;
    nw = 1;
    return true;
  }
  resident = 0;
  na = halo ? 2 : (bn >= 128 ? 2 : 3);
  int n = (kLimit - kFixedBytes - na * kAStage) / wtap;
  if (n < 2 && na > 2) {   // a deeper weight ring matters more than a third activation stage
    na = 2;
    n = (kLimit - kFixedBytes - na * kAStage) / wtap;
  }
  nw = n > kMaxRing ? kMaxRing : n;
  return nw >= 2;
}
}  // namespace

// Tile shape: fewest waves over the SMs first (a 133rd tile costs a whole extra wave on a small
// level), then the smallest halo.  16x8 is required by the fused pool; a shape whose rings do not fit
// (ring_depths) is never picked.
void conv3x3_tc_pick_tile(int H, int W, int B, int cout, int kc, int passes, int ktot, int epi_mode, int num_sms,
                          int& tile_h, int& tile_w) {
  static const int cand[3][2] = {{16, 8}, {8, 16}, {4, 32}};
  const int bn = conv_tc_block_n(cout);   // the engine only ever lowers BN from here, which only shrinks the rings
  const int n_nt = (cout + bn - 1) / bn;
  double best = 1e30;
  tile_h = 16;
  tile_w = 8;
  for (auto& c : cand) {
    int res, na, nw;
    if (!ring_depths(kc, c[0], c[1], 0, passes == 1 ? 1 : 2, bn, cout, ktot, epi_mode, 0, res, na, nw)) continue;
    const long tiles = (long)B * ((H + c[0] - 1) / c[0]) * ((W + c[1] - 1) / c[1]) * n_nt;
    const long waves = (tiles + num_sms - 1) / num_sms;
    const double cost = (double)waves * (c[0] + 2.0) / c[0] * (1.0 + 1e-3 * (c[1] / 8));
    if (cost < best) {
      best = cost;
      tile_h = c[0];
      tile_w = c[1];
    }
  }
}

// Chooses resident/streamed weights and the ring depths for one 3x3 problem; false if its rings cannot fit.
bool conv3x3_tc_plan(ConvProblem& h, int num_sms) {
  const int bn = h.bn;
  const int planes = h.passes == 1 ? 1 : 2;
  const int wtap = w_tap_bytes(w_rows(bn, h.pxn), h.kchunk, planes);
  const int w_all = (h.ktot / h.kchunk) * wtap;
  const bool can_resident = h.cout <= bn;
  const int kLimit = kSmemLimit - epi_scratch_bytes(h.epi_mode, h.pxn, bn);
  // wide halo (the engine allows it per chunk size): 16x8 (pixels on N: 32x8) tiles only; resident weights win when
  // both do not fit
  if (h.halo && (h.tile_h != (h.pxn ? 32 : 16) || h.tile_w != 8 ||
                 (can_resident && w_all + 2 * a_stage_bytes_h(h.kchunk, h.tile_h, h.tile_w, 0, planes) + kFixedBytes <= kLimit &&
                  w_all + 2 * a_stage_bytes_h(h.kchunk, h.tile_h, h.tile_w, 1, planes) + kFixedBytes > kLimit)))
    h.halo = 0;
  bool ok = ring_depths(h.kchunk, h.tile_h, h.tile_w, h.halo, planes, bn, h.cout, h.ktot, h.epi_mode, h.pxn,
                        h.v2_resident, h.v2_na, h.v2_nw);
  if (!ok && h.halo) {
    h.halo = 0;
    ok = ring_depths(h.kchunk, h.tile_h, h.tile_w, 0, planes, bn, h.cout, h.ktot, h.epi_mode, h.pxn, h.v2_resident,
                     h.v2_na, h.v2_nw);
  }
  const int nsp = h.B * h.tiles_y * h.tiles_x, n_nt = (h.cout + bn - 1) / bn;
  if (h.pair) {   // (2,1,1) clusters, one work item = a pair of spatial tiles
    const int nwork = (nsp + 1) / 2 * n_nt, nclu = num_sms / 2;
    h.v2_grid = 2 * (nwork < nclu ? nwork : nclu);
  } else {
    h.v2_grid = nsp * n_nt < num_sms ? nsp * n_nt : num_sms;
  }
  return ok;
}

using ConvKernel = void (*)(const ConvProblem*);
// the folded Cout = 32 pixels-on-N form exists single-pass and without a k-step-skipping source only
template <int BN, int KC, bool kPartial, bool kHalo, bool kOne, bool kRes, bool kPxN>
constexpr ConvKernel kernel_of() {
  if constexpr (kPxN && BN == 32 && (kPartial || !kOne))
    return nullptr;
  else
    return k_conv3x3_tc<BN, KC, kPartial, kHalo, kOne, kRes, kPxN>;
}

template <int BN, int KC, bool kPxN = false>
struct Variants {
  // every (kPartial, kHalo, kOne, kRes) instantiation of one (BN, KC, kPxN) kernel, indexed by the four bits
  static constexpr ConvKernel kFn[16] = {
      kernel_of<BN, KC, false, false, false, false, kPxN>(), kernel_of<BN, KC, false, false, false, true, kPxN>(),
      kernel_of<BN, KC, false, false, true, false, kPxN>(),  kernel_of<BN, KC, false, false, true, true, kPxN>(),
      kernel_of<BN, KC, false, true, false, false, kPxN>(),  kernel_of<BN, KC, false, true, false, true, kPxN>(),
      kernel_of<BN, KC, false, true, true, false, kPxN>(),   kernel_of<BN, KC, false, true, true, true, kPxN>(),
      kernel_of<BN, KC, true, false, false, false, kPxN>(),  kernel_of<BN, KC, true, false, false, true, kPxN>(),
      kernel_of<BN, KC, true, false, true, false, kPxN>(),   kernel_of<BN, KC, true, false, true, true, kPxN>(),
      kernel_of<BN, KC, true, true, false, false, kPxN>(),   kernel_of<BN, KC, true, true, false, true, kPxN>(),
      kernel_of<BN, KC, true, true, true, false, kPxN>(),    kernel_of<BN, KC, true, true, true, true, kPxN>()};
  static cudaError_t configure() {
    for (auto fn : kFn) {
      if (!fn) continue;
      const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
      if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
  }
  static cudaError_t launch(const ConvProblem* d_prob, const ConvProblem& h, cudaStream_t st) {
    if (h.v2_na < 2 || (!h.v2_resident && h.v2_nw < 2)) return cudaErrorInvalidValue;   // see ring_depths
    if (kPxN && (h.pair || h.tile_h != 32 || h.tile_w != 8 || h.epi_mode != (BN == 32 && h.epi_mode == 3 ? 3 : 0)))
      return cudaErrorInvalidValue;
    if (kPxN && BN == 32 && h.pool_hi) return cudaErrorInvalidValue;   // the folded form has no pool epilogue
    const bool partial = h.v2_part_hi > h.v2_part_lo;
    const int idx = (partial ? 8 : 0) | (h.halo ? 4 : 0) | (h.passes == 1 ? 2 : 0) | (h.v2_resident && h.straight ? 1 : 0);
    if (!kFn[idx]) return cudaErrorInvalidValue;   // a form this kernel does not have
    if (!h.pair) {
      kFn[idx]<<<h.v2_grid, kThreads, smem_bytes_for(h, BN), st>>>(d_prob);
      return cudaGetLastError();
    }
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3(h.v2_grid);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem_bytes_for(h, BN);
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kFn[idx], d_prob);
  }
};

cudaError_t conv3x3_tc_configure() {
  cudaError_t e;
#define FILM_CFG(BN, KC)                        \
  e = Variants<BN, KC>::configure();            \
  if (e != cudaSuccess) return e;
  FILM_CFG(32, 64) FILM_CFG(64, 64) FILM_CFG(128, 64) FILM_CFG(256, 64) FILM_CFG(32, 32) FILM_CFG(64, 32)
#undef FILM_CFG
  e = Variants<64, 64, true>::configure();
  if (e != cudaSuccess) return e;
  e = Variants<128, 64, true>::configure();
  if (e != cudaSuccess) return e;
  e = Variants<32, 64, true>::configure();
  if (e != cudaSuccess) return e;
  e = Variants<32, 32, true>::configure();
  if (e != cudaSuccess) return e;
  return cudaSuccess;
}

cudaError_t launch_conv3x3_tc(const ConvProblem* d_prob, const ConvProblem& h, cudaStream_t st) {
  const int bn = h.bn;
  if (h.kchunk == 32) {  // 32-channel K blocks: the 32 -> 32 flow convs and the 3(32) -> 64 first conv
    if (bn == 32) return h.pxn ? Variants<32, 32, true>::launch(d_prob, h, st) : Variants<32, 32>::launch(d_prob, h, st);
    if (bn == 64) return Variants<64, 32>::launch(d_prob, h, st);
    return cudaErrorInvalidValue;
  }
  switch (bn) {
    case 256: return Variants<256, 64>::launch(d_prob, h, st);
    case 128: return h.pxn ? Variants<128, 64, true>::launch(d_prob, h, st) : Variants<128, 64>::launch(d_prob, h, st);
    case 64: return h.pxn ? Variants<64, 64, true>::launch(d_prob, h, st) : Variants<64, 64>::launch(d_prob, h, st);
    default: return h.pxn ? Variants<32, 64, true>::launch(d_prob, h, st) : Variants<32, 64>::launch(d_prob, h, st);
  }
}

}  // namespace film
