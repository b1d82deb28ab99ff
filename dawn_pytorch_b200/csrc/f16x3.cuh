// FP16x3 building blocks shared by every tensor-core product (DESIGN §2, numerics decision 1): x = hi + lo with both pieces
// in fp16, a*b ~= lo(a)*hi(b) + hi(a)*lo(b) + hi(a)*hi(b) with fp32 accumulation.  Two rules for hi exist and each product keeps
// the one its error bound (tests/test_fused_gpu.py) assumes, so the rule is part of the name:
//   _rn     hi = x rounded to 11 significant bits:  |x - hi| <= 2^-11 |x|
//   _trunc  hi = x truncated to 11 significant bits: |x - hi| <= 2^-10 |x|
// Either way hi converts to fp16 exactly (no f16 -> f32 unpack is needed, and the integer ops keep the split off the conversion
// pipe) and lo = x - hi is exact in fp32 and rounded once to fp16.  Below fp16's normal range the conversions go subnormal:
// absolute error <= 2^-25, irrelevant next to O(1) outputs.
#pragma once
#include <cuda_fp16.h>
#include <cmath>
#include <cstdint>
#include <cstring>
#include "common.cuh"

namespace dawn {

// ---------------------------------------------------------------- hi / lo splits
__device__ __forceinline__ float f16_hi_rn(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }
__device__ __forceinline__ float f16_hi_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// (x0, x1) -> packed fp16 hi pair and lo pair (x0 in the low half)
__device__ __forceinline__ void split_f16x2_rn(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const float h0 = f16_hi_rn(x0), h1 = f16_hi_rn(x1);
  const __half2 h = __floats2half2_rn(h0, h1);
  const __half2 l = __floats2half2_rn(x0 - h0, x1 - h1);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void split_f16x2_trunc(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const float h0 = f16_hi_trunc(x0), h1 = f16_hi_trunc(x1);
  const __half2 h = __floats2half2_rn(h0, h1);
  const __half2 l = __floats2half2_rn(x0 - h0, x1 - h1);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
// x -> fp16 hi and lo
__device__ __forceinline__ void split_f16_rn(float x, __half& hi, __half& lo) {
  const float h = f16_hi_rn(x);
  hi = __float2half_rn(h);
  lo = __float2half_rn(x - h);
}
__device__ __forceinline__ void split_f16_trunc(float x, __half& hi, __half& lo) {
  const float h = f16_hi_trunc(x);
  hi = __float2half_rn(h);
  lo = __float2half_rn(x - h);
}

// ---------------------------------------------------------------- mma.sync (warp-level) primitives
// D(16x8, f32) += A(16x16, f16, row) * B(16x8, f16, col)
__device__ __forceinline__ void mma_m16n8k16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// 3-term split product: acc += a_lo*b_hi + a_hi*b_lo + a_hi*b_hi, b = {hi k0-7, hi k8-15, lo k0-7, lo k8-15}
__device__ __forceinline__ void mma3(float (&acc)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], const uint32_t (&b)[4]) {
  mma_m16n8k16(acc, al, b[0], b[1]);
  mma_m16n8k16(acc, ah, b[2], b[3]);
  mma_m16n8k16(acc, ah, b[0], b[1]);
}
// four 8x8 b16 matrices; lane l supplies the address of row (l & 7) of matrix (l >> 3)
__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], const __half* p) {
  const uint32_t addr = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm4_trans(uint32_t (&r)[4], const __half* p) {
  const uint32_t addr = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
  return y;
}

// ---------------------------------------------------------------- LayerNorm statistics of one C-channel row
// The row is held as one float4 per lane by LANES consecutive lanes (C = 4 * LANES).  Two-pass variance from registers;
// returns (mean, 1 / sqrt(biased variance + 1e-5)).
template <int LANES, int C>
__device__ __forceinline__ float2 row_ln_stats(const float4& v) {
  static_assert(C == 4 * LANES, "one float4 per lane");
  float s = (v.x + v.y) + (v.z + v.w);
#pragma unroll
  for (int o = 1; o < LANES; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mu = s * (1.0f / C);
  const float d0 = v.x - mu, d1 = v.y - mu, d2 = v.z - mu, d3 = v.w - mu;
  float ss = (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
#pragma unroll
  for (int o = 1; o < LANES; o <<= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  return make_float2(mu, 1.0f / sqrtf(ss * (1.0f / C) + 1e-5f));
}

// ---------------------------------------------------------------- host side of the weight images
// The exact power of two p with max_abs * p in [1024, 2048) (2^11 for an all-zero matrix).  Weight images are pre-scaled by p so
// that their lo pieces stay fp16-normal; every kernel undoes it with inv_wscale = 1 / p in its epilogue.
inline float f16_prescale(float max_abs) {
  int e = 0;
  if (max_abs > 0.f) std::frexp(max_abs, &e);   // max_abs = m * 2^e, m in [0.5, 1)
  return std::ldexp(1.0f, 11 - e);
}
// v -> fp16 bits of hi = fp16(v) and lo = fp16(v - hi)
inline void split_f16_host(float v, uint16_t& hi, uint16_t& lo) {
  const __half h = __float2half_rn(v);
  const __half l = __float2half_rn(v - __half2float(h));
  memcpy(&hi, &h, 2);
  memcpy(&lo, &l, 2);
}

}  // namespace dawn
