// Spatial linear attention context for 64-channel levels (reference U:602-627), fused:
//
//   per frame f, head h:  ctx[d][e] = sum_n softmax_n(k)[d, n] * v[e, n]      k, v = W_k x^, W_v x^  (x^ = channel LayerNorm of x)
//
// The unfused path wrote k and v (512 of the 768 qkv columns, 1.7 GB per level-0 layer) to HBM and read them back twice.  Here a CTA
// owns a run of pixels of one frame and every warp owns ONE HEAD.  The two warpgroups project K^T and V^T of 64 pixels at a time with
// warpgroup MMAs (m64n64k16, 3-term FP16 split, fp32 accumulate), the weights as the M operand: warpgroup g's four 64-row tiles hold
// rows 0-15, 16-31 of k and of v of heads 4g .. 4g+3, warp w of the warpgroup getting head 4g + w, so that each warp's accumulator
// fragments of exp(K^T - m) are already the A operand and those of V^T the B operand of the mma.sync context product -- k and v never
// leave registers.  The softmax over pixels is the FlashAttention recurrence with the roles transposed (rows = head dims d, "keys" =
// pixels): running row maximum m[d], running sum l[d], rescaled ctx rows.  Each CTA writes its partial (m, l, ctx) per head;
// sla_merge_kernel combines the partials of a frame, normalises, and composes the context with the out-projection into the per-frame
// 256 x C matrix the output GEMM consumes (as sla_context_kernel did).
#include <cuda_fp16.h>
#include <algorithm>
#include <cmath>
#include <vector>
#include "common.cuh"
#include "f16x3.cuh"
#include "kernels.cuh"
#include "sla_fused.cuh"
#include "tc_common.cuh"

namespace dawn {
namespace {

constexpr int C = 64;
constexpr int CHUNK = 64;              // pixels per context MMA step (the N of every projection MMA)
constexpr int NTH = 256;               // 8 warps = 8 heads = 2 warpgroups
constexpr int PART = 64 + 32 * 32;     // floats per partial: m[32], l[32], ctx[32][32]
constexpr float LOG2E = 1.4426950408889634f;
constexpr int W_IMG = 512 * 128;       // bytes of one swizzled [512][64] fp16 K/V weight image (hi or lo)
constexpr int X_PANEL = CHUNK * 128;   // bytes of one swizzled [64 pixels][64] fp16 x^ panel (hi or lo)
constexpr size_t kSmem = 1024 + 2 * W_IMG + 2 * 2 * X_PANEL;   // alignment slack, weights, two stages of x^ hi | lo

// D (64 x 64) = sum over 4 k-steps of (A_lo B_hi + A_hi B_lo + A_hi B_hi), the split terms in mma3's order
__device__ __forceinline__ void proj_ss(float (&d)[32], uint64_t ahi, uint64_t alo, uint64_t bhi, uint64_t blo) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const uint64_t o = (uint64_t)(ks * 2);              // +32 bytes per k-step, in 16-byte units
    tc::wgmma_m64n64k16(d, alo + o, bhi + o, ks == 0 ? 0u : 1u);
    tc::wgmma_m64n64k16(d, ahi + o, blo + o, 1u);
    tc::wgmma_m64n64k16(d, ahi + o, bhi + o, 1u);
  }
}

__global__ void __launch_bounds__(NTH, 1) sla_ctx_kernel(SlaCtxArgs a) {
  extern __shared__ __align__(16) unsigned char sla_smem[];
  uint8_t* Ws = tc::smem_align1024(sla_smem);           // K/V weights: hi image, lo image at + W_IMG; tile i = rows 64i .. 64i+63
  uint8_t* Xs = Ws + 2 * W_IMG;                         // two stages of [x^ hi | x^ lo] panels

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int g = lane >> 2, t = lane & 3;
  const int f = blockIdx.y, split = blockIdx.x;
  const int px_lo = split * a.px_per_cta, px_hi = min(a.P, px_lo + a.px_per_cta);

  // all heads' K/V weights: dense [hi|lo][8 heads x (k 32 | v 32)][64] fp16 in global; packed row h*64 + r lands in row
  // (4 (h/4) + r/16) * 64 + 16 (h%4) + r%16 of its swizzled image: tile 4 (h/4) + i, rows of warp h%4
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.Wkv);
    for (int i = tid; i < 2 * 512 * C / 8; i += NTH) {
      const int s = i >> 3, img = s >> 9, h = (s >> 6) & 7, r = s & 63;
      const int row = ((h >> 2) * 4 + (r >> 4)) * 64 + (h & 3) * 16 + (r & 15);
      cp_async16(Ws + img * W_IMG + tc::swz(row, i & 7), src + i);
    }
    cp_async_commit();
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
  // LayerNorm over channels, fp16 hi/lo into one stage (pixels past the split are zero rows)
  auto stage = [&](uint8_t* X) {
#pragma unroll
    for (int i = 0; i < CHUNK / (NTH / 16); ++i) {
      const int r = i * (NTH / 16) + (tid >> 4);
      const float4 v = xin[i];
      const float2 st = row_ln_stats<16, C>(v);
      const float mu = st.x, rs = st.y;
      uint32_t h0, l0, h1, l1;
      split_f16x2_trunc((v.x - mu) * rs, (v.y - mu) * rs, h0, l0); split_f16x2_trunc((v.z - mu) * rs, (v.w - mu) * rs, h1, l1);
      const uint32_t off = tc::swz(r, l16 >> 1) + (l16 & 1) * 8;
      *reinterpret_cast<uint2*>(X + off) = make_uint2(h0, h1);
      *reinterpret_cast<uint2*>(X + X_PANEL + off) = make_uint2(l0, l1);
    }
  };
  fetch(px_lo);
  stage(Xs);
  if (px_lo + CHUNK < px_hi) fetch(px_lo + CHUNK);
  cp_async_wait<0>();
  tc::fence_proxy_async();                              // generic-proxy writes (weights, first stage) -> wgmma reads
  __syncthreads();

  const int head = warp;                                // = 4 wg + warp within the warpgroup
  const float kscale = a.inv_wscale * LOG2E;            // k lives in the log2 domain (softmax through ex2)
  const uint64_t whi = tc::make_desc(tc::smem_u32(Ws + wg * 4 * 64 * 128)), wlo = whi + (W_IMG >> 4);
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

  int stg = 0;
  for (int p0 = px_lo; p0 < px_hi; p0 += CHUNK, stg ^= 1) {
    // -------------------------------------------------------------- K^T, V^T (32 x 64 each per warp) = W_{k,v}[head] * x^ chunk^T
    const uint64_t xhi = tc::make_desc(tc::smem_u32(Xs + stg * 2 * X_PANEL)), xlo = xhi + (X_PANEL >> 4);
    float kt[2][32], vt[2][32];                         // accumulator n-tile j = pixels 8j .. 8j+7 of the chunk
    tc::wgmma_fence();
    proj_ss(kt[0], whi, wlo, xhi, xlo);
    proj_ss(kt[1], whi + 512, wlo + 512, xhi, xlo);     // + 64 rows x 128 B per tile
    tc::wgmma_commit();
    proj_ss(vt[0], whi + 1024, wlo + 1024, xhi, xlo);
    proj_ss(vt[1], whi + 1536, wlo + 1536, xhi, xlo);
    tc::wgmma_commit();
    // the next chunk goes into the other stage while the MMAs run (its last readers finished before the previous barrier)
    if (p0 + CHUNK < px_hi) {
      stage(Xs + (stg ^ 1) * 2 * X_PANEL);
      if (p0 + 2 * CHUNK < px_hi) fetch(p0 + 2 * CHUNK);
    }
    const int ngrp = min(CHUNK, px_hi - p0) >> 4;       // valid 16-pixel groups (P is a multiple of 16)

    // -------------------------------------------------------------- online softmax over pixels (rows = head dims)
    tc::wgmma_wait<1>();
    tc::wgmma_fence_acc(kt[0]);
    tc::wgmma_fence_acc(kt[1]);
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) {
      float mx0 = -1e30f, mx1 = -1e30f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float* k = kt[mi] + 4 * j;
        const bool ok = (j >> 1) < ngrp;                // pixels past the split add exactly zero: ex2(-1e30 - m) = 0
#pragma unroll
        for (int c = 0; c < 4; ++c) k[c] = ok ? k[c] * kscale : -1e30f;
        mx0 = fmaxf(mx0, fmaxf(k[0], k[1]));
        mx1 = fmaxf(mx1, fmaxf(k[2], k[3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float m0 = fmaxf(mrow[mi][0], mx0), m1 = fmaxf(mrow[mi][1], mx1);
      const float c0 = ex2(mrow[mi][0] - m0), c1 = ex2(mrow[mi][1] - m1);
      mrow[mi][0] = m0; mrow[mi][1] = m1;
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float* k = kt[mi] + 4 * j;
        k[0] = ex2(k[0] - m0); k[1] = ex2(k[1] - m0);
        k[2] = ex2(k[2] - m1); k[3] = ex2(k[3] - m1);
        s0 += k[0] + k[1]; s1 += k[2] + k[3];
      }
      lrow[mi][0] = lrow[mi][0] * c0 + s0;
      lrow[mi][1] = lrow[mi][1] * c1 + s1;
#pragma unroll
      for (int j = 0; j < 4; ++j) { ctx[mi][j][0] *= c0; ctx[mi][j][1] *= c0; ctx[mi][j][2] *= c1; ctx[mi][j][3] *= c1; }
    }
    tc::wgmma_wait<0>();
    tc::wgmma_fence_acc(vt[0]);
    tc::wgmma_fence_acc(vt[1]);

    // -------------------------------------------------------------- ctx[d][e] += sum_px p[d][px] * v[e][px], 16 pixels per product
#pragma unroll
    for (int grp = 0; grp < CHUNK / 16; ++grp) {
      if (grp >= ngrp) break;
      const int n0 = 8 * grp;                           // accumulator index of n-tile 2 grp
      uint32_t ph[2][4], pl[2][4];                      // accumulator tiles (n-tiles 2grp, 2grp+1) == A fragment (rows d, k = 16 pixels)
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        split_f16x2_trunc(kt[mi][n0 + 0], kt[mi][n0 + 1], ph[mi][0], pl[mi][0]);
        split_f16x2_trunc(kt[mi][n0 + 2], kt[mi][n0 + 3], ph[mi][1], pl[mi][1]);
        split_f16x2_trunc(kt[mi][n0 + 4], kt[mi][n0 + 5], ph[mi][2], pl[mi][2]);
        split_f16x2_trunc(kt[mi][n0 + 6], kt[mi][n0 + 7], ph[mi][3], pl[mi][3]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {                     // e tile j = rows 8j..8j+7 of V^T: row tile j>>1, half j&1
        const float* v = vt[j >> 1] + n0 + (j & 1) * 2;
        uint32_t b[4];                                  // {hi k0-7, hi k8-15, lo k0-7, lo k8-15}, k = pixel
        split_f16x2_trunc(v[0] * a.inv_wscale, v[1] * a.inv_wscale, b[0], b[2]);
        split_f16x2_trunc(v[4] * a.inv_wscale, v[5] * a.inv_wscale, b[1], b[3]);
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
          float acc[4] = {0.f, 0.f, 0.f, 0.f};          // RN accumulation across pixel groups outside the tensor core
          mma3(acc, ph[mi], pl[mi], b);
          ctx[mi][j][0] += acc[0]; ctx[mi][j][1] += acc[1]; ctx[mi][j][2] += acc[2]; ctx[mi][j][3] += acc[3];
        }
      }
    }
    tc::fence_proxy_async();                            // the staged next chunk -> wgmma reads
    __syncthreads();                                    // next chunk staged; this chunk's stage is free
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
// Each warpgroup owns 64 pixels at a time, warp w rows 16w .. 16w+15.  x^ is built in registers straight in the A-fragment layout
// and is the register A operand of the q projection of all four head pairs (m64n64k16, B = W_q rows of the pair from a swizzled
// image); each head's q is normalised in registers and is the register A operand of the product with the frame's composed matrix
// Bf_f (256 x 64, fp16 hi|lo, transposed into swizzled panels), a fresh accumulator per head added into y with round-to-nearest
// fp32 adds.  q never reaches HBM (the unfused path wrote and re-read 840 MB of it per level-0 layer).  The two warpgroups share
// nothing after the prologue, so one's softmax overlaps the other's MMAs.
constexpr int OCH = 128;               // pixels per CTA iteration (two warpgroups x 64)
constexpr int WQ_IMG = 256 * 128;      // bytes of the swizzled [256][64] fp16 q weight image (hi or lo)
constexpr int BF_PANEL = 64 * 128;     // bytes of one swizzled [64 channels][64 k] fp16 panel of Bf_f^T; four cover k = 0..255
constexpr size_t kSmemOut = 1024 + 2 * WQ_IMG + 2 * 4 * BF_PANEL + C * 4;

__global__ void __launch_bounds__(NTH, 1) sla_out_kernel(SlaOutArgs a) {
  extern __shared__ __align__(16) unsigned char sla_smem[];
  uint8_t* Wq = tc::smem_align1024(sla_smem);           // q weights: hi image, lo image at + WQ_IMG
  uint8_t* Bs = Wq + 2 * WQ_IMG;                        // Bf_f^T: hi panels, lo panels at + 4 BF_PANEL
  float* s_bias = reinterpret_cast<float*>(Bs + 8 * BF_PANEL);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int g = lane >> 2, t = lane & 3;
  const int f = blockIdx.y;
  const int px_lo = blockIdx.x * a.px_per_cta, px_hi = min(a.P, px_lo + a.px_per_cta);
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.Wq);
    for (int i = tid; i < 2 * 256 * C / 8; i += NTH) cp_async16(Wq + tc::swz(i >> 3, i & 7), src + i);   // lo image = rows 256..
    cp_async_commit();
    const float* Bf = a.Bf + (size_t)f * 256 * a.ldb;
    for (int i = tid; i < 128 * C; i += NTH) {          // k pairs (2 k2, 2 k2 + 1) of channel c
      const int k = (i >> 6) * 2, c = i & 63;
      uint32_t h, l;
      split_f16x2_trunc(Bf[(size_t)k * a.ldb + c], Bf[(size_t)(k + 1) * a.ldb + c], h, l);
      const uint32_t off = (k >> 6) * BF_PANEL + tc::swz(c, (k & 63) >> 3) + (k & 7) * 2;
      *reinterpret_cast<uint32_t*>(Bs + off) = h;
      *reinterpret_cast<uint32_t*>(Bs + 4 * BF_PANEL + off) = l;
    }
    if (tid < C) s_bias[tid] = a.bias[tid];
    cp_async_wait<0>();
    tc::fence_proxy_async();                            // generic-proxy writes (weights, Bf panels) -> wgmma reads
    __syncthreads();
  }
  const float qscale = a.inv_wscale * LOG2E;
  const uint64_t wqhi = tc::make_desc(tc::smem_u32(Wq)), wqlo = wqhi + (WQ_IMG >> 4);
  const uint64_t bfhi = tc::make_desc(tc::smem_u32(Bs)), bflo = bfhi + (4 * BF_PANEL >> 4);

  for (int p0 = px_lo + wg * 64; p0 < px_hi; p0 += OCH) {        // warpgroup-uniform
    const bool rows_ok = p0 + (warp & 3) * 16 < px_hi;          // warp-uniform: the split ends on a 16-pixel boundary
    const size_t row0 = (size_t)f * a.P + p0 + (warp & 3) * 16 + g;
    // x rows g, g+8 of the warp's 16 at channels 8j + 2t, 8j + 2t + 1 (j = 0..7): the A-fragment columns of k-step j/2, and
    // the accumulator columns of n-tile j
    float2 xv[2][8];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr)
#pragma unroll
      for (int j = 0; j < 8; ++j)
        xv[hr][j] = rows_ok ? __ldg(reinterpret_cast<const float2*>(a.x + (row0 + 8 * hr) * a.ldx + 8 * j + 2 * t))
                            : make_float2(0.f, 0.f);
    uint32_t xh[4][4], xl[4][4];                        // x^ as A fragments of the four k-steps
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {                    // LayerNorm over the row's 64 channels, held by the lane quad
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += xv[hr][j].x + xv[hr][j].y;
      s += __shfl_xor_sync(0xffffffffu, s, 1); s += __shfl_xor_sync(0xffffffffu, s, 2);
      const float mu = s * (1.0f / C);
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d0 = xv[hr][j].x - mu, d1 = xv[hr][j].y - mu;
        ss += d0 * d0 + d1 * d1;
      }
      ss += __shfl_xor_sync(0xffffffffu, ss, 1); ss += __shfl_xor_sync(0xffffffffu, ss, 2);
      const float rs = 1.0f / sqrtf(ss * (1.0f / C) + 1e-5f);
#pragma unroll
      for (int j = 0; j < 8; ++j)                       // fragment register hr + 2 (j & 1) of k-step j / 2
        split_f16x2_trunc((xv[hr][j].x - mu) * rs, (xv[hr][j].y - mu) * rs, xh[j >> 1][hr + 2 * (j & 1)], xl[j >> 1][hr + 2 * (j & 1)]);
    }

    // q of heads 2hp, 2hp+1 (n-tiles 0-3, 4-7) = x^ * W_q[rows 64hp..]^T
    float q[32];
    auto issue_q = [&](int hp) {
      const uint64_t bh = wqhi + hp * 512, bl = wqlo + hp * 512;   // + 64 rows x 128 B per head pair
      tc::wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        tc::wgmma_m64n64k16_rs(q, xl[ks], bh + ks * 2, ks == 0 ? 0u : 1u);
        tc::wgmma_m64n64k16_rs(q, xh[ks], bl + ks * 2, 1u);
        tc::wgmma_m64n64k16_rs(q, xh[ks], bh + ks * 2, 1u);
      }
      tc::wgmma_commit();
    };
    // softmax over the 32 dims of head hh of the pair in q (log2 domain), times 32^-1/2, as A fragments of the two k-steps
    auto softmax = [&](int hh, uint32_t (&ph)[2][4], uint32_t (&pl)[2][4]) {
      float* qh = q + 16 * hh;
      float m0 = -1e30f, m1 = -1e30f;
#pragma unroll
      for (int n = 0; n < 4; ++n) {
#pragma unroll
        for (int c = 0; c < 4; ++c) qh[4 * n + c] *= qscale;
        m0 = fmaxf(m0, fmaxf(qh[4 * n], qh[4 * n + 1])); m1 = fmaxf(m1, fmaxf(qh[4 * n + 2], qh[4 * n + 3]));
      }
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        qh[4 * n] = ex2(qh[4 * n] - m0); qh[4 * n + 1] = ex2(qh[4 * n + 1] - m0);
        qh[4 * n + 2] = ex2(qh[4 * n + 2] - m1); qh[4 * n + 3] = ex2(qh[4 * n + 3] - m1);
        s0 += qh[4 * n] + qh[4 * n + 1]; s1 += qh[4 * n + 2] + qh[4 * n + 3];
      }
      s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
      const float i0 = 0.17677669529663687f / s0, i1 = 0.17677669529663687f / s1;
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {                  // accumulator tiles (2ks, 2ks+1) == A fragment of k-step ks
        const float* p = qh + 8 * ks;
        split_f16x2_trunc(p[0] * i0, p[1] * i0, ph[ks][0], pl[ks][0]);
        split_f16x2_trunc(p[2] * i1, p[3] * i1, ph[ks][1], pl[ks][1]);
        split_f16x2_trunc(p[4] * i0, p[5] * i0, ph[ks][2], pl[ks][2]);
        split_f16x2_trunc(p[6] * i1, p[7] * i1, ph[ks][3], pl[ks][3]);
      }
    };
    // acc = p_h (64 x 32) * Bf_f[h] (32 x 64), a fresh accumulator per head: RN accumulation over heads outside the tensor core
    float acc[32], y[32];
    auto issue_bf = [&](int head, const uint32_t (&ph)[2][4], const uint32_t (&pl)[2][4]) {
      const uint64_t o = (uint64_t)((head >> 1) * (BF_PANEL >> 4) + (head & 1) * 4);   // panel, then + 64 B for the odd head
      tc::wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        tc::wgmma_m64n64k16_rs(acc, pl[ks], bfhi + o + ks * 2, ks == 0 ? 0u : 1u);
        tc::wgmma_m64n64k16_rs(acc, ph[ks], bflo + o + ks * 2, 1u);
        tc::wgmma_m64n64k16_rs(acc, ph[ks], bfhi + o + ks * 2, 1u);
      }
      tc::wgmma_commit();
    };
    auto add_acc = [&](bool first) {
      tc::wgmma_fence_acc(acc);
#pragma unroll
      for (int i = 0; i < 32; ++i) y[i] = first ? acc[i] : y[i] + acc[i];
    };
    // Software pipeline over the head pairs: head 2hp+1's softmax runs under head 2hp's Bf product, the next pair's q projection
    // under the adds, and head 2hp+2's softmax under head 2hp+1's Bf product.  Commit groups complete in order.
    issue_q(0);
#pragma unroll
    for (int hp = 0; hp < 4; ++hp) {
      uint32_t ph0[2][4], pl0[2][4], ph1[2][4], pl1[2][4];
      if (hp == 0) tc::wgmma_wait<0>(); else tc::wgmma_wait<1>();   // q of this pair (the previous Bf product may still run)
      tc::wgmma_fence_acc(q);
      softmax(0, ph0, pl0);
      if (hp > 0) {
        tc::wgmma_wait<0>();
        add_acc(false);
      }
      issue_bf(2 * hp, ph0, pl0);
      softmax(1, ph1, pl1);
      if (hp < 3) {
        issue_q(hp + 1);
        tc::wgmma_wait<1>();
      } else {
        tc::wgmma_wait<0>();
      }
      add_acc(hp == 0);
      issue_bf(2 * hp + 1, ph1, pl1);
    }
    tc::wgmma_wait<0>();
    add_acc(false);
    if (rows_ok) {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        float* dst = a.out + (row0 + 8 * hr) * a.ldo;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = 8 * j + 2 * t;
          *reinterpret_cast<float2*>(dst + c) =
              make_float2(xv[hr][j].x + s_bias[c] + y[4 * j + 2 * hr], xv[hr][j].y + s_bias[c + 1] + y[4 * j + 2 * hr + 1]);
        }
      }
    }
  }
}

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
