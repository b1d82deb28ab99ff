// Spatial linear attention context for 64-channel levels (reference U:602-627), fused:
//
//   per frame f, head h:  ctx[d][e] = sum_n softmax_n(k)[d, n] * v[e, n]      k, v = W_k x^, W_v x^  (x^ = channel LayerNorm of x)
//
// The unfused path wrote k and v (512 of the 768 qkv columns, 1.7 GB per level-0 layer) to HBM and read them back twice.  Here a CTA
// owns a run of pixels of one frame and every warp owns ONE HEAD: it projects K^T and V^T of 16 pixels at a time with mma.sync
// (3-term FP16 split, fp32 accumulate), so that the accumulator fragments of exp(K^T - m) are already the A operand and those of V^T
// the B operand of the context product -- k and v never leave registers.  The softmax over pixels is the FlashAttention recurrence
// with the roles transposed (rows = head dims d, "keys" = pixels): running row maximum m[d], running sum l[d], rescaled ctx rows.
// Each CTA writes its partial (m, l, ctx) per head; sla_merge_kernel combines the partials of a frame, normalises, and composes the
// context with the out-projection into the per-frame 256 x C matrix the output GEMM consumes (as sla_context_kernel did).
#include <cuda_fp16.h>
#include <algorithm>
#include <cmath>
#include <vector>
#include "common.cuh"
#include "f16x3.cuh"
#include "kernels.cuh"
#include "sla_fused.cuh"

namespace dawn {
namespace {

constexpr int C = 64;
constexpr int LD = C + 8;              // halfs per shared-memory row (conflict-free ldmatrix)
constexpr int CHUNK = 64;              // pixels staged per iteration
constexpr int NTH = 256;               // 8 warps = 8 heads
constexpr int PART = 64 + 32 * 32;     // floats per partial: m[32], l[32], ctx[32][32]
constexpr float LOG2E = 1.4426950408889634f;

__global__ void __launch_bounds__(NTH, 1) sla_ctx_kernel(SlaCtxArgs a) {
  extern __shared__ __align__(16) unsigned char sla_smem[];
  __half* Wh = reinterpret_cast<__half*>(sla_smem);     // [512 rows = 8 heads x (k 32 | v 32)][LD], hi
  __half* Wl = Wh + 512 * LD;                           // lo
  __half* Xh = Wl + 512 * LD;                           // [CHUNK][LD] normalised pixels, hi
  __half* Xl = Xh + CHUNK * LD;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3, lm = lane >> 3, lr = lane & 7;
  const int f = blockIdx.y, split = blockIdx.x;
  const int px_lo = split * a.px_per_cta, px_hi = min(a.P, px_lo + a.px_per_cta);

  // all heads' K/V weights: dense [hi|lo][512][64] fp16 in global
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.Wkv);
    for (int i = tid; i < 2 * 512 * C / 8; i += NTH) {
      const int r = i / (C / 8), c8 = i - r * (C / 8);              // r in [0, 1024): hi rows then lo rows
      cp_async16(Wh + r * LD + c8 * 8, src + i);
    }
    cp_async_commit();
  }

  const int head = warp;
  const float kscale = a.inv_wscale * LOG2E;            // k lives in the log2 domain (softmax through ex2)
  float ctx[2][4][4];                                   // [d tile of 16][e tile of 8][frag]
  float mrow[2][2], lrow[2][2];                         // running max / per-thread partial sum of rows (tile, g | g+8)
#pragma unroll
  for (int mi = 0; mi < 2; ++mi) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int c = 0; c < 4; ++c) ctx[mi][j][c] = 0.f;
    mrow[mi][0] = mrow[mi][1] = -1e30f;
    lrow[mi][0] = lrow[mi][1] = 0.f;
  }

  // raw pixels of the next chunk travel in registers while the current chunk is being multiplied
  const int l16 = tid & 15;
  float4 xin[CHUNK / (NTH / 16)];
  auto fetch = [&](int p0) {
#pragma unroll
    for (int i = 0; i < CHUNK / (NTH / 16); ++i) {
      const int px = p0 + i * (NTH / 16) + (tid >> 4);
      xin[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (px < px_hi) xin[i] = __ldg(reinterpret_cast<const float4*>(a.x + ((size_t)f * a.P + px) * a.ldx) + l16);
    }
  };
  fetch(px_lo);

  for (int p0 = px_lo; p0 < px_hi; p0 += CHUNK) {
    __syncthreads();                                    // previous chunk consumed
    // ---------------------------------------------------------------- stage CHUNK pixels: LayerNorm over channels, fp16 hi/lo
#pragma unroll
    for (int i = 0; i < CHUNK / (NTH / 16); ++i) {
      const int r = i * (NTH / 16) + (tid >> 4);
      const float4 v = xin[i];
      const float2 st = row_ln_stats<16, C>(v);
      const float mu = st.x, rs = st.y;
      uint32_t h0, l0, h1, l1;
      split_f16x2_trunc((v.x - mu) * rs, (v.y - mu) * rs, h0, l0); split_f16x2_trunc((v.z - mu) * rs, (v.w - mu) * rs, h1, l1);
      *reinterpret_cast<uint2*>(&Xh[r * LD + l16 * 4]) = make_uint2(h0, h1);
      *reinterpret_cast<uint2*>(&Xl[r * LD + l16 * 4]) = make_uint2(l0, l1);
    }
    cp_async_wait<0>();
    __syncthreads();
    if (p0 + CHUNK < px_hi) fetch(p0 + CHUNK);

    const int ngrp = min(CHUNK, px_hi - p0) >> 4;       // 16-pixel groups (P is a multiple of 16)
    for (int grp = 0; grp < ngrp; ++grp) {
      // ------------------------------------------------------------ K^T, V^T (32 x 16 each) = W_{k,v}[head] (32 x 64) * x^ group^T
      float kt[2][2][4], vt[2][2][4];                   // [row tile][pixel n-tile][frag]
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int c = 0; c < 4; ++c) { kt[mi][nt][c] = 0.f; vt[mi][nt][c] = 0.f; }
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        uint32_t bx[2][4];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
          ldsm4(bx[nt], ((lm & 2) ? Xl : Xh) + (grp * 16 + nt * 8 + lr) * LD + ks * 16 + (lm & 1) * 8);
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {                // row tiles: k rows 0-15, 16-31, v rows 0-15, 16-31
          uint32_t ah[4], al[4];
          const int aoff = (head * 64 + mt * 16 + (lm & 1) * 8 + lr) * LD + ks * 16 + (lm >> 1) * 8;
          ldsm4(ah, Wh + aoff);
          ldsm4(al, Wl + aoff);
          if (mt < 2) { mma3(kt[mt][0], ah, al, bx[0]); mma3(kt[mt][1], ah, al, bx[1]); }
          else { mma3(vt[mt - 2][0], ah, al, bx[0]); mma3(vt[mt - 2][1], ah, al, bx[1]); }
        }
      }
      // ------------------------------------------------------------ online softmax over pixels (rows = head dims)
      uint32_t ph[2][4], pl[2][4];                      // exp(K^T - m) as A fragments of the context product
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        float mx0 = -1e30f, mx1 = -1e30f;
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
          for (int c = 0; c < 4; ++c) kt[mi][nt][c] *= kscale;
          mx0 = fmaxf(mx0, fmaxf(kt[mi][nt][0], kt[mi][nt][1]));
          mx1 = fmaxf(mx1, fmaxf(kt[mi][nt][2], kt[mi][nt][3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float m0 = fmaxf(mrow[mi][0], mx0), m1 = fmaxf(mrow[mi][1], mx1);
        const float c0 = ex2(mrow[mi][0] - m0), c1 = ex2(mrow[mi][1] - m1);
        mrow[mi][0] = m0; mrow[mi][1] = m1;
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          kt[mi][nt][0] = ex2(kt[mi][nt][0] - m0); kt[mi][nt][1] = ex2(kt[mi][nt][1] - m0);
          kt[mi][nt][2] = ex2(kt[mi][nt][2] - m1); kt[mi][nt][3] = ex2(kt[mi][nt][3] - m1);
          s0 += kt[mi][nt][0] + kt[mi][nt][1]; s1 += kt[mi][nt][2] + kt[mi][nt][3];
        }
        lrow[mi][0] = lrow[mi][0] * c0 + s0;
        lrow[mi][1] = lrow[mi][1] * c1 + s1;
#pragma unroll
        for (int j = 0; j < 4; ++j) { ctx[mi][j][0] *= c0; ctx[mi][j][1] *= c0; ctx[mi][j][2] *= c1; ctx[mi][j][3] *= c1; }
        // accumulator tiles (pixel n-tiles 0, 1) == A fragment (rows d, k = 16 pixels)
        split_f16x2_trunc(kt[mi][0][0], kt[mi][0][1], ph[mi][0], pl[mi][0]);
        split_f16x2_trunc(kt[mi][0][2], kt[mi][0][3], ph[mi][1], pl[mi][1]);
        split_f16x2_trunc(kt[mi][1][0], kt[mi][1][1], ph[mi][2], pl[mi][2]);
        split_f16x2_trunc(kt[mi][1][2], kt[mi][1][3], ph[mi][3], pl[mi][3]);
      }
      // ------------------------------------------------------------ ctx[d][e] += sum_px p[d][px] * v[e][px]
#pragma unroll
      for (int j = 0; j < 4; ++j) {                     // e tile j = rows 8j..8j+7 of V^T: row tile j>>1, half j&1
        const int vi = j >> 1, hf = (j & 1) * 2;
        uint32_t b[4];                                  // {hi k0-7, hi k8-15, lo k0-7, lo k8-15}, k = pixel
        split_f16x2_trunc(vt[vi][0][hf] * a.inv_wscale, vt[vi][0][hf + 1] * a.inv_wscale, b[0], b[2]);
        split_f16x2_trunc(vt[vi][1][hf] * a.inv_wscale, vt[vi][1][hf + 1] * a.inv_wscale, b[1], b[3]);
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
          float acc[4] = {0.f, 0.f, 0.f, 0.f};          // RN accumulation across pixel groups outside the tensor core
          mma3(acc, ph[mi], pl[mi], b);
          ctx[mi][j][0] += acc[0]; ctx[mi][j][1] += acc[1]; ctx[mi][j][2] += acc[2]; ctx[mi][j][3] += acc[3];
        }
      }
    }
  }

  // ------------------------------------------------------------------ partial (m, l, ctx) of this (frame, split, head)
  float* part = a.part + (((size_t)f * gridDim.x + split) * 8 + head) * PART;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float l = lrow[mi][hr];
      l += __shfl_xor_sync(0xffffffffu, l, 1); l += __shfl_xor_sync(0xffffffffu, l, 2);
      const int d = mi * 16 + hr * 8 + g;
      if (t == 0) { part[d] = mrow[mi][hr]; part[32 + d] = l; }
#pragma unroll
      for (int j = 0; j < 4; ++j)
        *reinterpret_cast<float2*>(part + 64 + d * 32 + j * 8 + 2 * t) = make_float2(ctx[mi][j][2 * hr], ctx[mi][j][2 * hr + 1]);
    }
  }
}

// per (frame, head): merge the splits' partials, normalise, compose with the out-projection:
//   Bf[h*32 + d][c] = sum_e ctx[d][e] * WoutT[h*32 + e][c]        (U:619-626)
__global__ void __launch_bounds__(256) sla_merge_kernel(const float* __restrict__ part, int nsplit, const float* __restrict__ WoutT,
                                                        int Cout, float* __restrict__ Bf, int ldb) {
  __shared__ float s_scale[16][32];
  __shared__ float s_inv[32];
  __shared__ float s_ctx[32][33];
  const int f = blockIdx.x, h = blockIdx.y, tid = threadIdx.x;
  const float* base = part + ((size_t)f * nsplit * 8 + h) * PART;
  const size_t sstride = (size_t)8 * PART;
  if (tid < 32) {
    float m = -1e30f;
    for (int s = 0; s < nsplit; ++s) m = fmaxf(m, base[s * sstride + tid]);
    float l = 0.f;
    for (int s = 0; s < nsplit; ++s) {
      const float sc = exp2f(base[s * sstride + tid] - m);
      s_scale[s][tid] = sc;
      l += base[s * sstride + 32 + tid] * sc;
    }
    s_inv[tid] = 1.0f / l;
  }
  __syncthreads();
  for (int idx = tid; idx < 1024; idx += 256) {
    const int d = idx >> 5, e = idx & 31;
    float acc = 0.f;
    for (int s = 0; s < nsplit; ++s) acc += base[s * sstride + 64 + idx] * s_scale[s][d];
    s_ctx[d][e] = acc * s_inv[d];
  }
  __syncthreads();
  float* bf = Bf + (size_t)f * 256 * ldb + (size_t)(h * 32) * ldb;
  const float* wt = WoutT + (size_t)(h * 32) * Cout;
  for (int idx = tid; idx < 32 * Cout; idx += 256) {
    const int dd = idx / Cout, c = idx - dd * Cout;
    float s = 0.f;
#pragma unroll 8
    for (int e = 0; e < 32; ++e) s += s_ctx[dd][e] * wt[(size_t)e * Cout + c];
    bf[(size_t)dd * ldb + c] = s;
  }
}

// ------------------------------------------------------------------------------------------------------------------------------
// out = x + bias + sum_h softmax_d(W_q,h x^) * 32^-1/2 * Bf_f[h]     (q projection, softmax over the head dim, context/out-projection)
// One warp owns 16 pixels: q_h comes out of mma.sync as accumulator fragments, is normalised in registers and re-used as the A operand
// of the product with the frame's composed matrix Bf_f (256 x 64, fp16 hi|lo in shared memory).  q never reaches HBM (the unfused
// path wrote and re-read 840 MB of it per level-0 layer).
constexpr int OCH = 128;               // pixels staged per iteration (one 16-pixel group per warp)
constexpr int BLD = 256 + 8;           // halfs per Bf^T row

__global__ void __launch_bounds__(NTH, 1) sla_out_kernel(SlaOutArgs a) {
  extern __shared__ __align__(16) unsigned char sla_smem[];
  __half* Wh = reinterpret_cast<__half*>(sla_smem);     // [256][LD] q weights, hi
  __half* Wl = Wh + 256 * LD;
  __half* Bh = Wl + 256 * LD;                           // [64 channels][BLD] Bf_f^T, hi
  __half* Bl = Bh + C * BLD;
  __half* Xh = Bl + C * BLD;                            // [OCH][LD]
  __half* Xl = Xh + OCH * LD;
  float* s_bias = reinterpret_cast<float*>(Xl + OCH * LD);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3, lm = lane >> 3, lr = lane & 7;
  const int f = blockIdx.y;
  const int px_lo = blockIdx.x * a.px_per_cta, px_hi = min(a.P, px_lo + a.px_per_cta);
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.Wq);
    for (int i = tid; i < 2 * 256 * C / 8; i += NTH) {
      const int r = i / (C / 8), c8 = i - r * (C / 8);              // r in [0, 512): hi rows then lo rows
      cp_async16(Wh + r * LD + c8 * 8, src + i);
    }
    cp_async_commit();
    const float* Bf = a.Bf + (size_t)f * 256 * a.ldb;
    for (int i = tid; i < 256 * C; i += NTH) {
      const int k = i >> 6, c = i & 63;
      split_f16_trunc(Bf[(size_t)k * a.ldb + c], Bh[c * BLD + k], Bl[c * BLD + k]);
    }
    if (tid < C) s_bias[tid] = a.bias[tid];
  }
  const int l16 = tid & 15;
  float4 xin[OCH / (NTH / 16)];
  auto fetch = [&](int p0) {
#pragma unroll
    for (int i = 0; i < OCH / (NTH / 16); ++i) {
      const int px = p0 + i * (NTH / 16) + (tid >> 4);
      xin[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (px < px_hi) xin[i] = __ldg(reinterpret_cast<const float4*>(a.x + ((size_t)f * a.P + px) * a.ldx) + l16);
    }
  };
  fetch(px_lo);
  const float qscale = a.inv_wscale * LOG2E;

  for (int p0 = px_lo; p0 < px_hi; p0 += OCH) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < OCH / (NTH / 16); ++i) {
      const int r = i * (NTH / 16) + (tid >> 4);
      const float4 v = xin[i];
      const float2 st = row_ln_stats<16, C>(v);
      const float mu = st.x, rs = st.y;
      uint32_t h0, l0, h1, l1;
      split_f16x2_trunc((v.x - mu) * rs, (v.y - mu) * rs, h0, l0); split_f16x2_trunc((v.z - mu) * rs, (v.w - mu) * rs, h1, l1);
      *reinterpret_cast<uint2*>(&Xh[r * LD + l16 * 4]) = make_uint2(h0, h1);
      *reinterpret_cast<uint2*>(&Xl[r * LD + l16 * 4]) = make_uint2(l0, l1);
    }
    cp_async_wait<0>();
    __syncthreads();
    if (p0 + OCH < px_hi) fetch(p0 + OCH);

    const int grp0 = p0 + warp * 16;
    if (grp0 >= px_hi) continue;
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int aoff = (warp * 16 + (lm & 1) * 8 + lr) * LD + ks * 16 + (lm >> 1) * 8;
      ldsm4(ah[ks], Xh + aoff);
      ldsm4(al[ks], Xl + aoff);
    }
    float y[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int c = 0; c < 4; ++c) y[n][c] = 0.f;
#pragma unroll 1
    for (int head = 0; head < 8; ++head) {
      float q[4][4];
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int c = 0; c < 4; ++c) q[n][c] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          uint32_t b[4];
          ldsm4(b, ((lm & 2) ? Wl : Wh) + (head * 32 + n * 8 + lr) * LD + ks * 16 + (lm & 1) * 8);
          mma3(q[n], ah[ks], al[ks], b);
        }
      // softmax over the 32 head dims of each row (log2 domain), times 32^-1/2
      float m0 = -1e30f, m1 = -1e30f;
#pragma unroll
      for (int n = 0; n < 4; ++n) {
#pragma unroll
        for (int c = 0; c < 4; ++c) q[n][c] *= qscale;
        m0 = fmaxf(m0, fmaxf(q[n][0], q[n][1])); m1 = fmaxf(m1, fmaxf(q[n][2], q[n][3]));
      }
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        q[n][0] = ex2(q[n][0] - m0); q[n][1] = ex2(q[n][1] - m0); q[n][2] = ex2(q[n][2] - m1); q[n][3] = ex2(q[n][3] - m1);
        s0 += q[n][0] + q[n][1]; s1 += q[n][2] + q[n][3];
      }
      s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
      const float i0 = 0.17677669529663687f / s0, i1 = 0.17677669529663687f / s1;
      uint32_t ph[2][4], pl[2][4];
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        split_f16x2_trunc(q[2 * ks][0] * i0, q[2 * ks][1] * i0, ph[ks][0], pl[ks][0]);
        split_f16x2_trunc(q[2 * ks][2] * i1, q[2 * ks][3] * i1, ph[ks][1], pl[ks][1]);
        split_f16x2_trunc(q[2 * ks + 1][0] * i0, q[2 * ks + 1][1] * i0, ph[ks][2], pl[ks][2]);
        split_f16x2_trunc(q[2 * ks + 1][2] * i1, q[2 * ks + 1][3] * i1, ph[ks][3], pl[ks][3]);
      }
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
          uint32_t b[4];
          ldsm4(b, ((lm & 2) ? Bl : Bh) + (n * 8 + lr) * BLD + head * 32 + ks * 16 + (lm & 1) * 8);
          mma3(acc, ph[ks], pl[ks], b);
        }
        y[n][0] += acc[0]; y[n][1] += acc[1]; y[n][2] += acc[2]; y[n][3] += acc[3];
      }
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const size_t row = (size_t)f * a.P + grp0 + g + 8 * hr;
      const float* xr = a.x + row * a.ldx;
      float* dst = a.out + row * a.ldo;
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const int c = n * 8 + 2 * t;
        const float2 r = *reinterpret_cast<const float2*>(xr + c);
        *reinterpret_cast<float2*>(dst + c) = make_float2(r.x + s_bias[c] + y[n][2 * hr], r.y + s_bias[c + 1] + y[n][2 * hr + 1]);
      }
    }
  }
}

constexpr size_t kSmem = (size_t)(2 * 512 * LD + 2 * CHUNK * LD) * 2;
constexpr size_t kSmemOut = (size_t)(2 * 256 * LD + 2 * C * BLD + 2 * OCH * LD) * 2 + C * 4;

}  // namespace

// Pixels per context CTA: the largest power of two from 512 down to 64 that divides P (64 if none does), or -1 when that needs
// more than 16 splits.  The kernel only consumes whole 16-pixel groups, so every split but the last must be a multiple of 16:
// ceil(P / nsplit) is not (P = 80 would give splits of 40 and drop 16 pixels).
int sla_fused_run(int P) {
  int px = 512;
  while (px > 64 && P % px != 0) px >>= 1;
  return (P + px - 1) / px > 16 ? -1 : px;
}
int sla_fused_splits(int P) {
  const int px = sla_fused_run(P);
  return px < 0 ? -1 : (P + px - 1) / px;
}
bool sla_fused_supported(int C_, int P) { return C_ == C && P % 16 == 0 && P >= 64 && sla_fused_run(P) > 0; }
size_t sla_fused_part_floats(int F, int P) { return (size_t)F * std::max(1, sla_fused_splits(P)) * 8 * PART; }

int launch_sla_ctx_fused(const SlaCtxArgs& a_in, const float* WoutT, float* Bf, int ldb, cudaStream_t st) {
  SlaCtxArgs a = a_in;
  const int nsplit = sla_fused_splits(a.P);
  if (!sla_fused_supported(C, a.P) || nsplit < 1) { set_last_error("sla_fused: unsupported shape"); return -1; }
  a.px_per_cta = sla_fused_run(a.P);
  static bool attr = false;
  if (!attr) {
    DAWN_CUDA_OK(cudaFuncSetAttribute(sla_ctx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
    attr = true;
  }
  sla_ctx_kernel<<<dim3(nsplit, a.F), NTH, kSmem, st>>>(a);
  DAWN_LAUNCH_OK();
  sla_merge_kernel<<<dim3(a.F, 8), 256, 0, st>>>(a.part, nsplit, WoutT, C, Bf, ldb);
  DAWN_LAUNCH_OK();
  return 0;
}

int launch_sla_out_fused(const SlaOutArgs& a_in, cudaStream_t st) {
  SlaOutArgs a = a_in;
  if (!sla_fused_supported(C, a.P)) { set_last_error("sla_out: unsupported shape"); return -1; }
  static bool attr = false;
  if (!attr) {
    DAWN_CUDA_OK(cudaFuncSetAttribute(sla_out_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemOut));
    attr = true;
  }
  int px = 512;
  while (px > OCH && a.P % px != 0) px >>= 1;
  a.px_per_cta = px;
  sla_out_kernel<<<dim3((a.P + px - 1) / px, a.F), NTH, kSmemOut, st>>>(a);
  DAWN_LAUNCH_OK();
  return 0;
}

// wq: rows 0..255 of the gamma-folded to_qkv weight -> [hi|lo][256][64] fp16 with a power-of-two pre-scale
void sla_out_pack(const float* wqkv, std::vector<uint16_t>& W, float* inv_wscale) {
  float mx = 0.f;
  for (size_t i = 0; i < (size_t)256 * C; ++i) mx = std::max(mx, std::fabs(wqkv[i]));
  const float sc = f16_prescale(mx);
  *inv_wscale = 1.0f / sc;
  W.assign((size_t)2 * 256 * C, 0);
  for (int r = 0; r < 256; ++r)
    for (int k = 0; k < C; ++k) split_f16_host(wqkv[(size_t)r * C + k] * sc, W[(size_t)r * C + k], W[((size_t)256 + r) * C + k]);
}

// wkv: rows 256..767 of the gamma-folded to_qkv weight ([768][64]); output [hi|lo][8 heads x (k 32 | v 32)][64] fp16, power-of-two pre-scale
void sla_fused_pack(const float* wqkv, std::vector<uint16_t>& W, float* inv_wscale) {
  float mx = 0.f;
  for (size_t i = (size_t)256 * C; i < (size_t)768 * C; ++i) mx = std::max(mx, std::fabs(wqkv[i]));
  const float sc = f16_prescale(mx);
  *inv_wscale = 1.0f / sc;
  W.assign((size_t)2 * 512 * C, 0);
  for (int h = 0; h < 8; ++h)
    for (int part = 0; part < 2; ++part)
      for (int r = 0; r < 32; ++r)
        for (int k = 0; k < C; ++k) {
          const size_t row = (size_t)h * 64 + part * 32 + r;
          split_f16_host(wqkv[(size_t)(256 + part * 256 + h * 32 + r) * C + k] * sc, W[row * C + k], W[((size_t)512 + row) * C + k]);
        }
}

}  // namespace dawn
