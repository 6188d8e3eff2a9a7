// Shared device/host definitions of the FILM engine.
//
// Activation storage ("split" format): every feature tensor is NHWC and stored as TWO
// 16-bit planes, hi = rn16(x) and lo = rn16(x - hi).  Same bytes as fp32, but each plane
// is directly consumable by wgmma (f16 / bf16 operands), and hi + lo carries 16 mantissa bits
// (bf16) -- the 3-pass product  A_hi*W_hi + A_hi*W_lo + A_lo*W_hi  then matches an fp32
// convolution to ~1e-5 relative (measured against the fp64 oracle).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace film {

#ifdef FILM_SPLIT_FP16
typedef __half sp_t;
#define FILM_SPLIT_NAME "fp16x2"
#else
typedef __nv_bfloat16 sp_t;
#define FILM_SPLIT_NAME "bf16x2"
#endif

constexpr float kLeaky = 0.2f;

// Split activation tensor view: [B][H][W][C] per plane, C = allocated channel stride.
struct ActView {
  sp_t* hi;
  sp_t* lo;
  int B, H, W, C;
};

__device__ __forceinline__ float sp_to_float(sp_t v) {
#ifdef FILM_SPLIT_FP16
  return __half2float(v);
#else
  return __bfloat162float(v);
#endif
}
__device__ __forceinline__ sp_t float_to_sp(float v) {
#ifdef FILM_SPLIT_FP16
  return __float2half_rn(v);
#else
  return __float2bfloat16_rn(v);
#endif
}

__device__ __forceinline__ void split2(float x, sp_t& hi, sp_t& lo) {
  hi = float_to_sp(x);
  lo = float_to_sp(x - sp_to_float(hi));
}

// two floats -> packed hi pair / lo pair (little-endian: element 0 in the low half)
#ifndef FILM_SPLIT_FP16
// bf16: one packed convert per plane (F2FP.BF16.F32.PACK_AB), float(bf16) is a 16-bit shift -> 6
// instructions per pair (the gather kernels are instruction-issue bound)
__device__ __forceinline__ void split_pack2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
  hi = *reinterpret_cast<const uint32_t*>(&h2);
  const float ra = a - __uint_as_float(hi << 16);
  const float rb = b - __uint_as_float(hi & 0xffff0000u);
  const __nv_bfloat162 l2 = __floats2bfloat162_rn(ra, rb);
  lo = *reinterpret_cast<const uint32_t*>(&l2);
}
__device__ __forceinline__ void split_pack2_generic(float a, float b, uint32_t& hi, uint32_t& lo) {
#else
// fp16: packed saturating converts (F2FP.SATFINITE.F16.F32.PACK_AB; |x| > 65504 clamps instead of turning into
// inf), the hi halves come back through HADD2.F32 -> 6 instructions per pair, like the bf16 form
__device__ __forceinline__ void split_pack2(float a, float b, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(b - hf.y), "f"(a - hf.x));
}
__device__ __forceinline__ void split_pack2_generic(float a, float b, uint32_t& hi, uint32_t& lo) {
#endif
  sp_t ah, al, bh, bl;
  split2(a, ah, al);
  split2(b, bh, bl);
  hi = (uint32_t)(*reinterpret_cast<unsigned short*>(&ah)) |
       ((uint32_t)(*reinterpret_cast<unsigned short*>(&bh)) << 16);
  lo = (uint32_t)(*reinterpret_cast<unsigned short*>(&al)) |
       ((uint32_t)(*reinterpret_cast<unsigned short*>(&bl)) << 16);
}

__device__ __forceinline__ float sp_bits_to_float(uint32_t bits16) {
#ifdef FILM_SPLIT_FP16
  unsigned short s = (unsigned short)bits16;
  return __half2float(*reinterpret_cast<__half*>(&s));
#else
  return __uint_as_float(bits16 << 16);
#endif
}

// unpack 8 consecutive channels (one uint4 per plane) into fp32: x = hi + lo
__device__ __forceinline__ void unpack8(const uint4& h, const uint4& l, float* v) {
  const uint32_t hw[4] = {h.x, h.y, h.z, h.w};
  const uint32_t lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#ifndef FILM_SPLIT_FP16
    v[2 * i] = __uint_as_float(hw[i] << 16) + __uint_as_float(lw[i] << 16);
    v[2 * i + 1] = __uint_as_float(hw[i] & 0xffff0000u) + __uint_as_float(lw[i] & 0xffff0000u);
#else
    const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[i]));
    const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lw[i]));
    v[2 * i] = hf.x + lf.x;
    v[2 * i + 1] = hf.y + lf.y;
#endif
  }
}

__device__ __forceinline__ void pack8(const float* v, uint4& h, uint4& l) {
  split_pack2(v[0], v[1], h.x, l.x);
  split_pack2(v[2], v[3], h.y, l.y);
  split_pack2(v[4], v[5], h.z, l.z);
  split_pack2(v[6], v[7], h.w, l.w);
}

// 32-byte global accesses: 16 channels of one plane as two 128-bit accesses (sm_90 has no 256-bit load/store).
// Addresses must be 16-byte aligned.
__device__ __forceinline__ void st256(void* p, const uint4& a, const uint4& b) {
  uint4* q = reinterpret_cast<uint4*>(p);
  q[0] = a;
  q[1] = b;
}
__device__ __forceinline__ void ld256_nc(const void* p, uint4& a, uint4& b) {
  const uint4* q = reinterpret_cast<const uint4*>(p);
  a = __ldg(q);
  b = __ldg(q + 1);
}
// 16 consecutive channels: pack to (hi 32 B, lo 32 B) and store
__device__ __forceinline__ void pack_store16(const float* v, sp_t* hi_dst, sp_t* lo_dst) {
  uint4 h0, l0, h1, l1;
  pack8(v, h0, l0);
  pack8(v + 8, h1, l1);
  st256(hi_dst, h0, h1);
  st256(lo_dst, l0, l1);
}
// hi plane only (destinations whose consumers are all single-pass convs)
__device__ __forceinline__ uint32_t pack2_hi(float a, float b) {
#ifdef FILM_SPLIT_FP16
  uint32_t hi;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));
  return hi;
#else
  const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h2);
#endif
}
__device__ __forceinline__ void pack_store16_hi(const float* v, sp_t* hi_dst) {
  uint4 h0, h1;
  h0.x = pack2_hi(v[0], v[1]);   h0.y = pack2_hi(v[2], v[3]);   h0.z = pack2_hi(v[4], v[5]);   h0.w = pack2_hi(v[6], v[7]);
  h1.x = pack2_hi(v[8], v[9]);   h1.y = pack2_hi(v[10], v[11]); h1.z = pack2_hi(v[12], v[13]); h1.w = pack2_hi(v[14], v[15]);
  st256(hi_dst, h0, h1);
}
// unpack 8 / 16 consecutive channels of the hi plane alone (x ~ hi: 11-bit operands of a single-pass conv)
__device__ __forceinline__ void unpack8_hi(const uint4& h, float* v) {
  const uint32_t hw[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#ifndef FILM_SPLIT_FP16
    v[2 * i] = __uint_as_float(hw[i] << 16);
    v[2 * i + 1] = __uint_as_float(hw[i] & 0xffff0000u);
#else
    const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[i]));
    v[2 * i] = hf.x;
    v[2 * i + 1] = hf.y;
#endif
  }
}
__device__ __forceinline__ void load_unpack16_hi(const sp_t* hi_src, float* v) {
  uint4 h0, h1;
  ld256_nc(hi_src, h0, h1);
  unpack8_hi(h0, v);
  unpack8_hi(h1, v + 8);
}
__device__ __forceinline__ void load_unpack16(const sp_t* hi_src, const sp_t* lo_src, float* v) {
  uint4 h0, h1, l0, l1;
  ld256_nc(hi_src, h0, h1);
  ld256_nc(lo_src, l0, l1);
  unpack8(h0, l0, v);
  unpack8(h1, l1, v + 8);
}

__device__ __forceinline__ float leaky(float x) { return x >= 0.f ? x : x * kLeaky; }

}  // namespace film
