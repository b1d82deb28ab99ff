// Kernels of PBnet's transformer decoder (pbnet_kernels.cuh).  The decoder is small (d_model 64, 4 heads, ff 128 in DAWN) and
// runs over every frame of the audio, so the kernels are plain fp32 SIMT: one warp per row for the row kernels, one thread per
// query for the banded attention, which only visits the keys within +-band of its query.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "pbnet_kernels.cuh"

namespace dawn {
namespace {

constexpr int kRowWarps = 8;          // rows per block of the memory and out_ln kernels
constexpr int kFfnWarps = 4;          // rows per block of the FFN kernel (its hidden rows live in shared memory)
constexpr int kProjRows = 8;          // rows per block of the projection kernel
constexpr int kAttnQ = 64;            // queries per block of the attention kernel (one thread each)
constexpr int kAttnK = 64;            // keys per shared-memory tile
constexpr int kMaxNL = kPbMaxD / 32;  // outputs per lane of a row kernel

__global__ void __launch_bounds__(kRowWarps * 32) pb_memory_kernel(const float* __restrict__ aud, const float* __restrict__ z, int Lz,
                                                                   const float* __restrict__ wz, const float* __restrict__ xref, int PE,
                                                                   const float* __restrict__ wp, int bs, int F, int D,
                                                                   float* __restrict__ mem) {
  const int m = blockIdx.x * kRowWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (m >= bs * F) return;
  const int b = m / F, f = m - b * F, NL = D >> 5;
  float acc[kMaxNL];
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t) acc[t] = 0.f;
  const float* zr = z + ((size_t)f * bs + b) * Lz;                 // z is (F, bs, Lz): CAE.generate's layout (cae.py:133)
  for (int k0 = 0; k0 < Lz; k0 += 32) {
    const float zv = (k0 + lane < Lz) ? zr[k0 + lane] : 0.f;
    const int nk = min(32, Lz - k0);
    for (int kk = 0; kk < nk; ++kk) {
      const float zk = __shfl_sync(0xffffffffu, zv, kk);
      const float* w = wz + (size_t)(k0 + kk) * D + lane;
#pragma unroll
      for (int t = 0; t < kMaxNL; ++t)
        if (t < NL) acc[t] = fmaf(zk, w[32 * t], acc[t]);
    }
  }
  const float* xr = xref + (size_t)b * PE;
  for (int p = 0; p < PE; ++p) {
    const float xp = xr[p];
    const float* w = wp + (size_t)p * D + lane;
#pragma unroll
    for (int t = 0; t < kMaxNL; ++t)
      if (t < NL) acc[t] = fmaf(xp, w[32 * t], acc[t]);
  }
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t)
    if (t < NL) mem[(size_t)m * D + lane + 32 * t] = aud[(size_t)m * D + lane + 32 * t] + acc[t];
}

__global__ void __launch_bounds__(256) pb_proj_kernel(const float* __restrict__ x, int ldx, int T, int F, int D,
                                                      const float* __restrict__ w, int hid, int ngroups, PbProjGroups groups,
                                                      float qscale, const float* __restrict__ rot, int npairs, float* __restrict__ out) {
  __shared__ float xs[kProjRows][kPbMaxD];
  const int m0 = blockIdx.x * kProjRows;
  for (int i = threadIdx.x; i < kProjRows * D; i += blockDim.x) {
    const int r = i / D, k = i - r * D;
    xs[r][k] = (m0 + r < T) ? x[(size_t)(m0 + r) * ldx + k] : 0.f;
  }
  __syncthreads();
  const int N = ngroups * hid, npair_cols = N >> 1;
  for (int pc = threadIdx.x; pc < npair_cols; pc += blockDim.x) {
    const int n = 2 * pc;
    float a0[kProjRows], a1[kProjRows];
#pragma unroll
    for (int r = 0; r < kProjRows; ++r) a0[r] = a1[r] = 0.f;
    for (int k = 0; k < D; ++k) {
      const float2 wv = *reinterpret_cast<const float2*>(w + (size_t)k * N + n);
#pragma unroll
      for (int r = 0; r < kProjRows; ++r) {
        a0[r] = fmaf(xs[r][k], wv.x, a0[r]);
        a1[r] = fmaf(xs[r][k], wv.y, a1[r]);
      }
    }
    const int g = n / hid, d = (n - g * hid) & 31, fl = groups.flags[g];
    const bool rotate = (fl & PB_ROTARY) && (d >> 1) < npairs;
#pragma unroll
    for (int r = 0; r < kProjRows; ++r) {
      const int m = m0 + r;
      if (m >= T) break;
      float v0 = a0[r], v1 = a1[r];
      if (fl & PB_SCALE) { v0 *= qscale; v1 *= qscale; }             // q * scale before the rotary (transformerdecoder4.py:62-67)
      if (rotate) {                                                  // t * cos + rotate_half(t) * sin, rotate_half(x0, x1) = (-x1, x0)
        const float2 cs = *reinterpret_cast<const float2*>(rot + ((size_t)(m % F) * npairs + (d >> 1)) * 2);
        const float r0 = v0 * cs.x - v1 * cs.y, r1 = v1 * cs.x + v0 * cs.y;
        v0 = r0; v1 = r1;
      }
      *reinterpret_cast<float2*>(out + (size_t)m * N + n) = make_float2(v0, v1);
    }
  }
}

__global__ void __launch_bounds__(kAttnQ) pb_attention_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk,
                                                              const float* __restrict__ v, int ldv, const float* __restrict__ bias,
                                                              int band, int F, int H, float* __restrict__ out) {
  __shared__ __align__(16) float Ks[kAttnK][32];
  __shared__ __align__(16) float Vs[kAttnK][32];
  const int h = blockIdx.y, b = blockIdx.z, i0 = blockIdx.x * kAttnQ, i = i0 + threadIdx.x;
  const size_t row0 = (size_t)b * F;
  const bool live = i < F;
  float qv[32], acc[32];
  float mx = -INFINITY, l = 0.f;
#pragma unroll
  for (int d = 0; d < 32; d += 4) {
    const float4 t = live ? *reinterpret_cast<const float4*>(q + (row0 + i) * ldq + h * 32 + d) : make_float4(0.f, 0.f, 0.f, 0.f);
    qv[d] = t.x; qv[d + 1] = t.y; qv[d + 2] = t.z; qv[d + 3] = t.w;
    acc[d] = acc[d + 1] = acc[d + 2] = acc[d + 3] = 0.f;
  }
  const float* bh = bias + (size_t)h * (2 * band + 1) + band;       // bh[j - i]
  const int jlo = max(0, i0 - band), jhi = min(F, i0 + kAttnQ + band);
  for (int jt = jlo; jt < jhi; jt += kAttnK) {
    __syncthreads();
    {
      const int j = jt + threadIdx.x;
      float4* kd = reinterpret_cast<float4*>(Ks[threadIdx.x]);
      float4* vd = reinterpret_cast<float4*>(Vs[threadIdx.x]);
      if (j < jhi) {
        const float4* ks = reinterpret_cast<const float4*>(k + (row0 + j) * ldk + h * 32);
        const float4* vs = reinterpret_cast<const float4*>(v + (row0 + j) * ldv + h * 32);
#pragma unroll
        for (int c = 0; c < 8; ++c) { kd[c] = ks[c]; vd[c] = vs[c]; }
      }
    }
    __syncthreads();
    if (!live) continue;
    const int a = max(jt, i - band), e = min(min(jt + kAttnK, jhi), i + band + 1);
    for (int j = a; j < e; ++j) {
      const float* kr = Ks[j - jt];
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) s = fmaf(qv[d], kr[d], s);
      s += bh[j - i];
      if (s > mx) {                                                  // online softmax: rescale what was summed so far
        const float corr = expf(mx - s);
        l *= corr;
#pragma unroll
        for (int d = 0; d < 32; ++d) acc[d] *= corr;
        mx = s;
      }
      const float p = expf(s - mx);
      l += p;
      const float* vr = Vs[j - jt];
#pragma unroll
      for (int d = 0; d < 32; ++d) acc[d] = fmaf(p, vr[d], acc[d]);
    }
  }
  if (!live) return;
  const float inv = 1.f / l;
  float* o = out + (row0 + i) * (size_t)(32 * H) + h * 32;
#pragma unroll
  for (int d = 0; d < 32; d += 4) *reinterpret_cast<float4*>(o + d) = make_float4(acc[d] * inv, acc[d + 1] * inv, acc[d + 2] * inv, acc[d + 3] * inv);
}

// LayerNorm of the warp's row y (lane holds y[lane + 32 t]), biased variance, eps 1e-5, in place
__device__ __forceinline__ void row_layer_norm(float (&y)[kMaxNL], int NL, int D, const float* __restrict__ gamma,
                                               const float* __restrict__ beta, int lane) {
  float s = 0.f;
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t)
    if (t < NL) s += y[t];
  const float mean = warp_sum(s) / (float)D;
  float q = 0.f;
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t)
    if (t < NL) { const float d = y[t] - mean; q = fmaf(d, d, q); }
  const float rstd = 1.f / sqrtf(warp_sum(q) / (float)D + 1e-5f);
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t)
    if (t < NL) { const int c = lane + 32 * t; y[t] = (y[t] - mean) * rstd * gamma[c] + beta[c]; }
}

__global__ void __launch_bounds__(kRowWarps * 32) pb_out_ln_kernel(const float* __restrict__ o, int hid, const float* __restrict__ wo,
                                                                   const float* __restrict__ res, int ldr, const float* __restrict__ gamma,
                                                                   const float* __restrict__ beta, int T, int D, float* __restrict__ x_out) {
  const int m = blockIdx.x * kRowWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (m >= T) return;
  const int NL = D >> 5;
  float y[kMaxNL];
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t) y[t] = 0.f;
  const float* orow = o + (size_t)m * hid;
  for (int k0 = 0; k0 < hid; k0 += 32) {
    const float ov = orow[k0 + lane];
    for (int kk = 0; kk < 32; ++kk) {
      const float ok = __shfl_sync(0xffffffffu, ov, kk);
      const float* w = wo + (size_t)(k0 + kk) * D + lane;
#pragma unroll
      for (int t = 0; t < kMaxNL; ++t)
        if (t < NL) y[t] = fmaf(ok, w[32 * t], y[t]);
    }
  }
  const float* rr = res + (size_t)m * ldr;
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t)
    if (t < NL) y[t] = rr[lane + 32 * t] + y[t];
  row_layer_norm(y, NL, D, gamma, beta, lane);
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t)
    if (t < NL) x_out[(size_t)m * D + lane + 32 * t] = y[t];
}

__global__ void __launch_bounds__(kFfnWarps * 32) pb_ffn_ln_kernel(float* __restrict__ x, int T, int D, const float* __restrict__ w1,
                                                                   const float* __restrict__ b1, int ff, const float* __restrict__ w2,
                                                                   const float* __restrict__ b2, const float* __restrict__ gamma,
                                                                   const float* __restrict__ beta, const float* __restrict__ wf,
                                                                   const float* __restrict__ bf, int nout,
                                                                   const unsigned char* __restrict__ mask, float* __restrict__ out) {
  __shared__ float xs[kFfnWarps][kPbMaxD];
  __shared__ float hs[kFfnWarps][kPbMaxFF];
  const int wi = threadIdx.x >> 5, lane = threadIdx.x & 31, m = blockIdx.x * kFfnWarps + wi;
  if (m >= T) return;
  const int NL = D >> 5;
  float xr[kMaxNL];
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t)
    if (t < NL) { xr[t] = x[(size_t)m * D + lane + 32 * t]; xs[wi][lane + 32 * t] = xr[t]; }
  __syncwarp();
  for (int j = lane; j < ff; j += 32) {                              // linear1 -> F.gelu (erf)
    float a = 0.f;
    for (int k = 0; k < D; ++k) a = fmaf(xs[wi][k], w1[(size_t)k * ff + j], a);
    a += b1[j];
    hs[wi][j] = 0.5f * a * (1.f + erff(a * 0.70710678118654752f));
  }
  __syncwarp();
  float y[kMaxNL];
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t) y[t] = 0.f;
  for (int j = 0; j < ff; ++j) {                                     // linear2
    const float hj = hs[wi][j];
    const float* w = w2 + (size_t)j * D + lane;
#pragma unroll
    for (int t = 0; t < kMaxNL; ++t)
      if (t < NL) y[t] = fmaf(hj, w[32 * t], y[t]);
  }
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t)
    if (t < NL) y[t] = xr[t] + (y[t] + b2[lane + 32 * t]);
  row_layer_norm(y, NL, D, gamma, beta, lane);
  if (wf == nullptr) {
#pragma unroll
    for (int t = 0; t < kMaxNL; ++t)
      if (t < NL) x[(size_t)m * D + lane + 32 * t] = y[t];
    return;
  }
  __syncwarp();
#pragma unroll
  for (int t = 0; t < kMaxNL; ++t)
    if (t < NL) xs[wi][lane + 32 * t] = y[t];
  __syncwarp();
  if (lane < nout) {                                                 // finallayer, then output[~mask] = 0 (reemb5:370-374)
    float a = 0.f;
    for (int c = 0; c < D; ++c) a = fmaf(xs[wi][c], wf[(size_t)c * nout + lane], a);
    out[(size_t)m * nout + lane] = mask[m] ? a + bf[lane] : 0.f;
  }
}

}  // namespace

int launch_pb_memory(const float* aud, const float* z, int Lz, const float* wz, const float* xref, int PE, const float* wp,
                     int bs, int F, int D, float* mem, cudaStream_t st) {
  const int T = bs * F;
  pb_memory_kernel<<<(T + kRowWarps - 1) / kRowWarps, kRowWarps * 32, 0, st>>>(aud, z, Lz, wz, xref, PE, wp, bs, F, D, mem);
  DAWN_LAUNCH_OK();
  return 0;
}

int launch_pb_proj(const float* x, int ldx, int T, int F, int D, const float* w, int hid, int ngroups, PbProjGroups groups,
                   float qscale, const float* rot, int npairs, float* out, cudaStream_t st) {
  pb_proj_kernel<<<(T + kProjRows - 1) / kProjRows, 256, 0, st>>>(x, ldx, T, F, D, w, hid, ngroups, groups, qscale, rot, npairs, out);
  DAWN_LAUNCH_OK();
  return 0;
}

int launch_pb_attention(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* bias, int band,
                        int bs, int F, int H, float* out, cudaStream_t st, int* launches) {
  constexpr int kMaxGridZ = 65535;                                 // clips per launch: gridDim.z's limit
  for (int b0 = 0; b0 < bs; b0 += kMaxGridZ) {
    const size_t r0 = (size_t)b0 * F;
    dim3 grid((F + kAttnQ - 1) / kAttnQ, H, std::min(kMaxGridZ, bs - b0));
    pb_attention_kernel<<<grid, kAttnQ, 0, st>>>(q + r0 * ldq, ldq, k + r0 * ldk, ldk, v + r0 * ldv, ldv, bias, band, F, H,
                                                 out + r0 * 32 * H);
    DAWN_LAUNCH_OK();
    if (launches) ++*launches;
  }
  return 0;
}

int launch_pb_out_ln(const float* o, int hid, const float* wo, const float* res, int ldr, const float* gamma, const float* beta,
                     int T, int D, float* x_out, cudaStream_t st) {
  pb_out_ln_kernel<<<(T + kRowWarps - 1) / kRowWarps, kRowWarps * 32, 0, st>>>(o, hid, wo, res, ldr, gamma, beta, T, D, x_out);
  DAWN_LAUNCH_OK();
  return 0;
}

int launch_pb_ffn_ln(float* x, int T, int D, const float* w1, const float* b1, int ff, const float* w2, const float* b2,
                     const float* gamma, const float* beta, const float* wf, const float* bf, int nout, const unsigned char* mask,
                     float* out, cudaStream_t st) {
  pb_ffn_ln_kernel<<<(T + kFfnWarps - 1) / kFfnWarps, kFfnWarps * 32, 0, st>>>(x, T, D, w1, b1, ff, w2, b2, gamma, beta, wf, bf,
                                                                              nout, mask, out);
  DAWN_LAUNCH_OK();
  return 0;
}

}  // namespace dawn
