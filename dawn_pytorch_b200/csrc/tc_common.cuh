// Shared device helpers of the wgmma kernels (tc_gemm.cu, tc_conv3.cu, temporal_fused.cu): mbarrier / bulk-copy / wgmma PTX wrappers,
// shared-memory matrix descriptors, the fp16 hi/lo split and the coalesced row store.
#pragma once
#include <cuda_fp16.h>
#include <type_traits>
#include "common.cuh"

namespace dawn {
namespace tc {

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// The dynamic shared-memory base rounded up to 1024 bytes (the 128-byte swizzle repeats every 1024 B).  Offsetting the
// __shared__ pointer itself keeps its address space visible to the compiler, so stores through it compile to STS; a
// round trip through uintptr_t turned them into generic stores.
__device__ __forceinline__ uint8_t* smem_align1024(uint8_t* base) { return base + ((1024u - (smem_u32(base) & 1023u)) & 1023u); }

// Per-warpgroup register budgets (all four warps of the warpgroup execute the same instruction).  The kernel launches with
// the even split its __launch_bounds__ allows; .dec may only lower a warp's count and returns the rest to the CTA's pool, .inc
// may only raise it and waits until the pool holds enough.  ptxas allocates the code after each instruction within its budget.
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// f(integral_constant<int, I>) for I = 0 .. N-1, expanded at compile time: the MMA loops below branch only on constants,
// so no runtime control-flow merge carries accumulator registers that a wgmma may still be writing
template <int I, int N, class F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (I < N) {
    f(std::integral_constant<int, I>{});
    static_for<I + 1, N>(f);
  }
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Relaxed arrive for the A producers: the default .release form compiles to MEMBAR.ALL.CTA, which also waits for the
// producers' outstanding register-prefetch loads (two panels ahead) and serialised the whole prefetch (measured ~1000
// cycles per panel).  Ordering of the operand writes is provided by the preceding fence.proxy.async; the consumer side
// (mbarrier try_wait, acquire) is unchanged.
__device__ __forceinline__ void mbar_arrive_relaxed(uint64_t* bar) {
  asm volatile("mbarrier.arrive.relaxed.cta.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");   // compiler barrier only
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- wgmma (sm_90a warpgroup MMA, accumulators in registers)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across an in-flight wgmma
template <int N>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D(64 x 64, f32) (+)= A(64 x 16, f16, K-major) * B(64 x 16, f16, K-major)^T; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(scale_d)
      : "memory");
}
// D(64 x 96, f32) (+)= A(64 x 16, f16, K-major) * B(96 x 16, f16, K-major)^T; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_m64n96k16(float (&d)[48], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
        "+f"(d[46]), "+f"(d[47])
      : "l"(adesc), "l"(bdesc), "r"(scale_d)
      : "memory");
}
// D(64 x 64, f32) (+)= A(64 x 16, f16, registers) * B(64 x 16, f16, K-major)^T.  Warp w of the warpgroup supplies rows
// 16w .. 16w+15 of A in the mma.sync m16n8k16 A-fragment layout; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
      : "memory");
}

// K-major, 128-byte-swizzled operand: rows of 128 B, 8-row groups `sbo` bytes apart (1024 B for a dense panel), layout SWIZZLE_128B.
// The swizzle follows absolute shared-memory address bits, so an operand may start at any 128-byte row of a 1024-byte-aligned image.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t sbo = 1024) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)((sbo >> 4) & 0x3FFF) << 32) | (1ull << 62);
}

// A consumer warpgroup's 64 x 64 accumulator fragment (rows r0 + [0, 64) of a [128][kStageLd] fp32 tile): the first drain of a tile
// stores, later drains add (round-to-nearest fp32 adds outside the tensor core, see tc_gemm.cu)
constexpr int kStageLd = 68;                  // floats per staged row (64 + 4 pad: conflict-free float4 row reads)
__device__ __forceinline__ void stage_fragment(float* stage, int r0, const float (&d)[32], bool first, int wtid) {
  const int w = wtid >> 5, l = wtid & 31;
  float* p0 = stage + (size_t)(r0 + w * 16 + (l >> 2)) * kStageLd + 2 * (l & 3);
  float* p1 = p0 + 8 * kStageLd;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float2* a = reinterpret_cast<float2*>(p0 + 8 * j);
    float2* b = reinterpret_cast<float2*>(p1 + 8 * j);
    if (first) {
      *a = make_float2(d[4 * j], d[4 * j + 1]);
      *b = make_float2(d[4 * j + 2], d[4 * j + 3]);
    } else {
      const float2 x = *a, y = *b;
      *a = make_float2(x.x + d[4 * j], x.y + d[4 * j + 1]);
      *b = make_float2(y.x + d[4 * j + 2], y.y + d[4 * j + 3]);
    }
  }
}

// byte offset of 16-byte chunk c (0..7) of row r inside a swizzled panel
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4)); }

// (x0, x1) -> packed fp16 hi pair and fp16 lo pair.  hi is rounded to 11 significant bits in fp32 with two integer
// ops (so its fp16 conversion is exact and no f16->f32 unpack is needed: the conversion pipe was the measured
// producer bottleneck); lo = x - hi is exact in fp32 and rounded once to fp16.  Below fp16's normal range the
// conversions go subnormal: absolute error <= 2^-25, irrelevant next to O(1) outputs.
__device__ __forceinline__ void split_f16x2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const float h0 = __uint_as_float((__float_as_uint(x0) + 0x1000u) & 0xFFFFE000u);
  const float h1 = __uint_as_float((__float_as_uint(x1) + 0x1000u) & 0xFFFFE000u);
  const __half2 h = __floats2half2_rn(h0, h1);
  const __half2 l = __floats2half2_rn(x0 - h0, x1 - h1);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// Store this warp's 32 rows x 64 columns (row-per-lane registers) to global memory with full-sector transactions:
// 16 columns at a time go through a per-warp shared-memory buffer so that one store instruction writes 8 rows x 64
// contiguous bytes instead of 32 rows x 16 bytes at a multi-KB stride (measured: the strided form capped the qkv
// projection's output stream at ~1.6 TB/s).
__device__ __forceinline__ void store_rows_coalesced(float* wbuf, const float (&acc)[64], float* out, size_t opix, int ldo,
                                                     int n0, bool rv, int lane) {
  // destination rows of this lane in the read-back phase: r = lane/4 + 8k (fetched once from the owning lanes)
  float* dst[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int r = (lane >> 2) + 8 * k;
    const uint32_t lo = __shfl_sync(0xffffffffu, (uint32_t)opix, r);
    const uint32_t hi = __shfl_sync(0xffffffffu, (uint32_t)((unsigned long long)opix >> 32), r);
    const int ok = __shfl_sync(0xffffffffu, rv ? 1 : 0, r);
    const size_t px = ((size_t)hi << 32) | lo;
    dst[k] = ok ? (out + px * ldo + n0 + (lane & 3) * 4) : nullptr;
  }
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<float4*>(wbuf + lane * 20 + j * 4) =
          make_float4(acc[pass * 16 + j * 4], acc[pass * 16 + j * 4 + 1], acc[pass * 16 + j * 4 + 2], acc[pass * 16 + j * 4 + 3]);
    __syncwarp();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int r = (lane >> 2) + 8 * k;
      const float4 v = *reinterpret_cast<const float4*>(wbuf + r * 20 + (lane & 3) * 4);
      if (dst[k]) *reinterpret_cast<float4*>(dst[k] + pass * 16) = v;
    }
  }
}

}  // namespace tc
}  // namespace dawn
