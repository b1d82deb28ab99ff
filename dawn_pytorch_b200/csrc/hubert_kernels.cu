// Kernels of the HuBERT audio encoder that are not contractions (hubert_kernels.cuh): feature-extractor layer 0, the
// LayerNorm (+ GELU) row pass, the positional conv's grouped re-layout, and the encoder's full multi-head attention.
#include <algorithm>

#include "common.cuh"
#include "f16x3.cuh"
#include "gemm.cuh"
#include "hubert_kernels.cuh"

namespace dawn {
namespace {

// ------------------------------------------------------------------------------------------------ LayerNorm row pass
// one warp per row; the lane holds columns 2 lane + 64 j (+1).  Two passes over the row (mean, then centred squares), both read
// from global memory (the row stays in L1).
__device__ __forceinline__ void ln_row_warp(const float* x, float* y, int C, const float* gamma, const float* beta, float eps,
                                            int gelu, int lane) {
  float s = 0.f;
  for (int c = 2 * lane; c < C; c += 64) {
    const float2 v = *reinterpret_cast<const float2*>(x + c);
    s += v.x + v.y;
  }
  const float mu = warp_sum(s) / (float)C;
  float ss = 0.f;
  for (int c = 2 * lane; c < C; c += 64) {
    const float2 v = *reinterpret_cast<const float2*>(x + c);
    const float a = v.x - mu, b = v.y - mu;
    ss += a * a + b * b;
  }
  const float rstd = 1.0f / sqrtf(warp_sum(ss) / (float)C + eps);
  for (int c = 2 * lane; c < C; c += 64) {
    const float2 v = *reinterpret_cast<const float2*>(x + c);
    float a = (v.x - mu) * rstd * gamma[c] + beta[c], b = (v.y - mu) * rstd * gamma[c + 1] + beta[c + 1];
    if (gelu) { a = gelu_erf(a); b = gelu_erf(b); }
    *reinterpret_cast<float2*>(y + c) = make_float2(a, b);
  }
}

constexpr int ROW_WARPS = 8;

__global__ void __launch_bounds__(ROW_WARPS * 32) hb_row_ln_kernel(const float* x, int ld, int M, int C, const float* gamma,
                                                                   const float* beta, float eps, int gelu, float* y, int ldo) {
  const int lane = threadIdx.x & 31;
  for (long long row = (long long)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5); row < M; row += (long long)gridDim.x * ROW_WARPS)
    ln_row_warp(x + row * ld, y + row * ldo, C, gamma, beta, eps, gelu, lane);
}

// layer 0: the warp computes its frame's C conv outputs into the output row, then normalises the row in place
__global__ void __launch_bounds__(ROW_WARPS * 32) hb_conv0_kernel(const float* __restrict__ x, int L, int T0, int M,
                                                                  const float* __restrict__ w, const float* __restrict__ bias, int k,
                                                                  int s, int C, const float* gamma, const float* beta, float eps,
                                                                  float* out) {
  const int lane = threadIdx.x & 31;
  for (long long row = (long long)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5); row < M; row += (long long)gridDim.x * ROW_WARPS) {
    const long long b = row / T0, t = row - b * T0;
    const float* xs = x + b * L + t * s;
    float* o = out + row * C;
    for (int c = lane; c < C; c += 32) {
      float acc = bias ? __ldg(bias + c) : 0.f;
      for (int i = 0; i < k; ++i) acc = fmaf(__ldg(w + (size_t)i * C + c), __ldg(xs + i), acc);
      o[c] = acc;
    }
    __syncwarp();
    ln_row_warp(o, o, C, gamma, beta, eps, 1, lane);
    __syncwarp();
  }
}

__global__ void hb_group_pad_kernel(const float* __restrict__ h, int B, int T, int G, int pad, float* __restrict__ xg) {
  const int Tp = T + 2 * pad;
  const long long n = (long long)G * B * Tp * 16;           // float4s
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i & 15);
    const long long r_all = i >> 4;
    const int r = (int)(r_all % Tp);
    const long long gb = r_all / Tp;
    const int b = (int)(gb % B), g = (int)(gb / B);
    const int t = r - pad;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t >= 0 && t < T) v = __ldg(reinterpret_cast<const float4*>(h + ((size_t)b * T + t) * G * 64 + g * 64) + c4);
    reinterpret_cast<float4*>(xg)[i] = v;
  }
}

// ------------------------------------------------------------------------------------------------ attention
// CTA = (head, sequence, 64 queries); 4 warps, each owns 16 queries.  Per block of 64 keys, K (row-major [key][d]) and V
// (transposed, [d][key]) are split once into fp16 hi / lo in shared memory (the B-operand layouts of mma.sync m16n8k16, rows
// padded to 72 halfs: conflict-free fragment reads).  S = Q K^T (3-term split) -> online softmax in fp32 -> P, whose
// accumulator layout is the A fragment of the next product -> O = O * corr + P V.  Keys past T are zero-filled and masked.
constexpr int AQ = 64, AK = 64, ALD = 72, ATHREADS = 128;

__global__ void __launch_bounds__(ATHREADS) hb_attention_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                                const float* __restrict__ v, int ld, int T, float* __restrict__ out,
                                                                int ldo) {
  __shared__ __align__(16) __half sKh[AK * ALD], sKl[AK * ALD], sVh[kHbHeadDim * ALD], sVl[kHbHeadDim * ALD];
  const int head = blockIdx.x, seq = blockIdx.y, q0 = blockIdx.z * AQ;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const size_t row0 = (size_t)seq * T;
  const int hc = head * kHbHeadDim;

  const int i0 = q0 + warp * 16;
  uint32_t qh[4][4], ql[4][4];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      // a0: (row g, cols 2t..), a1: (row g + 8), a2: (row g, cols 2t + 8..), a3: (row g + 8, cols 2t + 8..)
      const int row = i0 + g + ((r & 1) ? 8 : 0);
      const int col = ks * 16 + 2 * t + ((r & 2) ? 8 : 0);
      float2 x = make_float2(0.f, 0.f);
      if (row < T) x = *reinterpret_cast<const float2*>(q + (row0 + row) * ld + hc + col);
      split_f16x2_rn(x.x, x.y, qh[ks][r], ql[ks][r]);
    }
  float o[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int c = 0; c < 4; ++c) o[n][c] = 0.f;
  float m0 = -1e30f, m1 = -1e30f, l0 = 0.f, l1 = 0.f;

  for (int kb = 0; kb < T; kb += AK) {
    __syncthreads();
    // ---- stage 64 keys: 64 rows x (16 float4 of K + 16 float4 of V)
#pragma unroll 4
    for (int it = 0; it < AK * 32 / ATHREADS; ++it) {
      const int idx = it * ATHREADS + tid;
      const int r = idx >> 5, c = idx & 31;                 // c < 16: K float4 #c, else V float4 #(c - 16)
      const int key = kb + r;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (key < T) x = __ldg(reinterpret_cast<const float4*>((c < 16 ? k : v) + (row0 + key) * ld + hc) + (c & 15));
      if (c < 16) {
        uint32_t h0, l0_, h1, l1_;
        split_f16x2_rn(x.x, x.y, h0, l0_); split_f16x2_rn(x.z, x.w, h1, l1_);
        *reinterpret_cast<uint2*>(&sKh[r * ALD + c * 4]) = make_uint2(h0, h1);
        *reinterpret_cast<uint2*>(&sKl[r * ALD + c * 4]) = make_uint2(l0_, l1_);
      } else {
        const int d = (c - 16) * 4;
        const float xv[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          __half hh, ll;
          split_f16_rn(xv[i], hh, ll);
          sVh[(d + i) * ALD + r] = hh;
          sVl[(d + i) * ALD + r] = ll;
        }
      }
    }
    __syncthreads();
    if (i0 >= T) continue;

    // ---- S = Q K^T: 8 n-tiles of 8 keys, k = 64 dims in 4 steps
    float s[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int c = 0; c < 4; ++c) s[n][c] = 0.f;
      const int krow = n * 8 + g;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const int off = krow * ALD + ks * 16 + 2 * t;
        const uint32_t bk[4] = {*reinterpret_cast<const uint32_t*>(&sKh[off]), *reinterpret_cast<const uint32_t*>(&sKh[off + 8]),
                                *reinterpret_cast<const uint32_t*>(&sKl[off]), *reinterpret_cast<const uint32_t*>(&sKl[off + 8])};
        mma3(s[n], qh[ks], ql[ks], bk);
      }
    }
    // ---- online softmax over rows g (c = 0, 1) and g + 8 (c = 2, 3)
    float mn0 = m0, mn1 = m1;
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const bool ok = kb + n * 8 + 2 * t + (c & 1) < T;
        if (!ok) s[n][c] = -1e30f;
        if (c & 2) mn1 = fmaxf(mn1, s[n][c]); else mn0 = fmaxf(mn0, s[n][c]);
      }
    mn0 = fmaxf(mn0, __shfl_xor_sync(0xffffffffu, mn0, 1)); mn0 = fmaxf(mn0, __shfl_xor_sync(0xffffffffu, mn0, 2));
    mn1 = fmaxf(mn1, __shfl_xor_sync(0xffffffffu, mn1, 1)); mn1 = fmaxf(mn1, __shfl_xor_sync(0xffffffffu, mn1, 2));
    const float corr0 = __expf(m0 - mn0), corr1 = __expf(m1 - mn1);
    m0 = mn0; m1 = mn1;
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const bool ok = kb + n * 8 + 2 * t + (c & 1) < T;
        const float pv = ok ? __expf(s[n][c] - ((c & 2) ? mn1 : mn0)) : 0.f;
        s[n][c] = pv;
        if (c & 2) ps1 += pv; else ps0 += pv;
      }
    l0 = l0 * corr0 + ps0;                                   // per-thread partial sums; quad-reduced at the end
    l1 = l1 * corr1 + ps1;
    // ---- O = O * corr + P V (P: accumulator layout of two n-tiles == A fragment of one k16 step)
    uint32_t ph[4][4], pl[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      split_f16x2_rn(s[2 * ks][0], s[2 * ks][1], ph[ks][0], pl[ks][0]);
      split_f16x2_rn(s[2 * ks][2], s[2 * ks][3], ph[ks][1], pl[ks][1]);
      split_f16x2_rn(s[2 * ks + 1][0], s[2 * ks + 1][1], ph[ks][2], pl[ks][2]);
      split_f16x2_rn(s[2 * ks + 1][2], s[2 * ks + 1][3], ph[ks][3], pl[ks][3]);
    }
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      const int drow = (n * 8 + g) * ALD;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const int off = drow + ks * 16 + 2 * t;
        const uint32_t bv[4] = {*reinterpret_cast<const uint32_t*>(&sVh[off]), *reinterpret_cast<const uint32_t*>(&sVh[off + 8]),
                                *reinterpret_cast<const uint32_t*>(&sVl[off]), *reinterpret_cast<const uint32_t*>(&sVl[off + 8])};
        mma3(acc, ph[ks], pl[ks], bv);
      }
      o[n][0] = o[n][0] * corr0 + acc[0];
      o[n][1] = o[n][1] * corr0 + acc[1];
      o[n][2] = o[n][2] * corr1 + acc[2];
      o[n][3] = o[n][3] * corr1 + acc[3];
    }
  }

  if (i0 >= T) return;
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  const int r0 = i0 + g, r1 = i0 + g + 8;
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    const int col = hc + n * 8 + 2 * t;
    if (r0 < T) *reinterpret_cast<float2*>(out + (row0 + r0) * ldo + col) = make_float2(o[n][0] * inv0, o[n][1] * inv0);
    if (r1 < T) *reinterpret_cast<float2*>(out + (row0 + r1) * ldo + col) = make_float2(o[n][2] * inv1, o[n][3] * inv1);
  }
}

int grid_for(long long items, int per_block) { return (int)std::min<long long>((items + per_block - 1) / per_block, 132 * 16); }

}  // namespace

int launch_hb_conv0(const float* x, int B, int L, const float* w, const float* bias, int k, int s, int C, const float* gamma,
                    const float* beta, float eps, float* out, cudaStream_t st) {
  if (L < k || k < 1 || s < 1 || C < 64 || C % 64 != 0 || C > kHbMaxC) { set_last_error("hubert conv0: bad geometry"); return -1; }
  const int T0 = (L - k) / s + 1;
  const long long M = (long long)B * T0;
  hb_conv0_kernel<<<grid_for(M, ROW_WARPS), ROW_WARPS * 32, 0, st>>>(x, L, T0, (int)M, w, bias, k, s, C, gamma, beta, eps, out);
  DAWN_LAUNCH_OK();
  return 0;
}

int launch_hb_row_ln(const float* x, int ld, int M, int C, const float* gamma, const float* beta, float eps, int gelu, float* y,
                     int ldo, cudaStream_t st) {
  if (C < 64 || C % 64 != 0 || C > kHbMaxC || (ld & 1) || (ldo & 1)) { set_last_error("hubert row LayerNorm: bad geometry"); return -1; }
  if (M <= 0) return 0;
  hb_row_ln_kernel<<<grid_for(M, ROW_WARPS), ROW_WARPS * 32, 0, st>>>(x, ld, M, C, gamma, beta, eps, gelu, y, ldo);
  DAWN_LAUNCH_OK();
  return 0;
}

int launch_hb_group_pad(const float* h, int B, int T, int G, int pad, float* xg, cudaStream_t st) {
  const long long n = (long long)G * B * (T + 2 * pad) * 16;
  if (n <= 0) return 0;
  hb_group_pad_kernel<<<grid_for(n, 256), 256, 0, st>>>(h, B, T, G, pad, xg);
  DAWN_LAUNCH_OK();
  return 0;
}

int launch_hb_attention(const float* q, const float* k, const float* v, int ld, int B, int T, int H, float* out, int ldo,
                        cudaStream_t st) {
  if ((ld & 3) || (ldo & 1) || H < 1 || B < 1 || T < 1 || B > 65535) { set_last_error("hubert attention: bad geometry"); return -1; }
  dim3 grid(H, B, (T + AQ - 1) / AQ);
  hb_attention_kernel<<<grid, ATHREADS, 0, st>>>(q, k, v, ld, T, out, ldo);
  DAWN_LAUNCH_OK();
  return 0;
}

}  // namespace dawn
