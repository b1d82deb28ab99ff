// Shared device/host helpers for the DAWN denoising-UNet kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <string>

namespace dawn {

// ---------------------------------------------------------------- error plumbing (no exceptions across the C-ABI)
void set_last_error(const std::string& s);
#define DAWN_CUDA_OK(expr)                                                              \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      ::dawn::set_last_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " @" + \
                             __FILE__ + ":" + std::to_string(__LINE__));                \
      return -2;                                                                        \
    }                                                                                   \
  } while (0)
#define DAWN_LAUNCH_OK() DAWN_CUDA_OK(cudaGetLastError())
#define DAWN_CHECK(cond, msg)                 \
  do {                                        \
    if (!(cond)) {                            \
      ::dawn::set_last_error(msg);            \
      return -1;                              \
    }                                         \
  } while (0)
#define DAWN_TRY(expr)           \
  do {                           \
    int _rc = (expr);            \
    if (_rc != 0) return _rc;    \
  } while (0)

// Clips of one batched pass.  Activations hold frame f of clip b as frame f * clips + b; per-clip GroupNorm statistics (16 doubles),
// FiLM tables and init-conv maps are one slice per clip, found from a row's frame index.
constexpr int kMaxClips = 16;

// ---------------------------------------------------------------- small device helpers
__device__ __forceinline__ float silu(float x) { return x / (1.0f + expf(-x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float quad_sum(float v) {   // the 4 lanes sharing lane/4
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
  return v;
}

// cp.async 16 B global -> shared
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gsrc) : "memory");
}
// cp.async 16 B with zero-fill when !pred (src-size = 0); src must still be a valid address.
__device__ __forceinline__ void cp_async16_zfill(void* smem_dst, const void* gsrc, bool pred) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem_dst);
  const int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// 3xTF32 split: x ~= hi + lo with hi, lo representable in tf32 (10-bit mantissa), round-to-nearest (ties away),
// done with full-rate integer ops: cvt.rna.tf32.f32 issues on a slow conversion pipe and was the measured
// bottleneck of both contraction kernels' operand preparation.
__device__ __forceinline__ uint32_t tf32_rn_bits(uint32_t u) { return (u + 0x1000u) & 0xFFFFE000u; }
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = tf32_rn_bits(__float_as_uint(x));
  lo = tf32_rn_bits(__float_as_uint(x - __uint_as_float(hi)));
}

// D(16x8, f32) += A(16x8, tf32, row) * B(8x8, tf32, col)
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

}  // namespace dawn
