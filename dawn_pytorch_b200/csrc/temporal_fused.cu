// Fused temporal attention for 64-channel levels (reference U:648-725 == LA:275-342 wrapped in Residual(PreNorm(...)),
// U:763-765): one CTA owns ONE PIXEL's whole frame sequence and does everything on chip:
//
//   x[:, p, :] (F x 64 fp32) -> LayerNorm statistics -> fp16 hi/lo split in shared memory
//   per head h:   K_h, V_h, Q_h = LN-folded projections (mma.sync m16n8k16, 3-term FP16 split, fp32 accumulate)
//                 rotary on q, k (registers)  ->  K_h (row-major) and V_h^T to shared memory as fp16 hi/lo; Q_h stays in registers
//                 banded (+-band, + relative bias) softmax attention (FlashAttention-2 style, as attn_tc.cu)
//                 y += O_h * Wout_h            (accumulator layout of O == A-operand layout of the next MMA)
//   out[:, p, :] = x + y
//
// q/k/v and the attention output never reach HBM (the unfused path wrote 2.5 GB of q|k|v per level-0 layer and read it back),
// the three launches (qkv GEMM, attention, out-projection GEMM) become one.  16 warps: every warp projects K/V of the 16-frame tiles
// w, w+16, ... and owns ONE query tile whose Q fragments and y accumulators live in registers across the whole head loop.  All
// operand fragments come from shared memory through ldmatrix.x4 (hi and lo halves of a B fragment in one instruction).
#include <cuda_fp16.h>
#include <cmath>
#include <cstring>
#include <vector>
#include <algorithm>
#include "common.cuh"
#include "kernels.cuh"
#include "tc_common.cuh"
#include "temporal_fused.cuh"

namespace dawn {
namespace {

constexpr int C = 64;                 // channels of the levels this kernel serves
constexpr int X_LD = C + 8;           // halfs per x row      (conflict-free A-fragment reads)
constexpr int W_LD = C + 8;           // halfs per W_h row    (B-fragment reads)
constexpr int K_LD = 40;              // halfs per K row
constexpr int WO_LD = 40;             // halfs per Wout_h row ([n = channel][k = head dim])
constexpr int NTH = 512;
constexpr int NWARP = NTH / 32;
constexpr int W_STAGE = 2 * 96 * W_LD + 2 * 64 * WO_LD;      // halfs per weight stage
constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
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
__device__ __forceinline__ void cp_async_16(void* dst, const void* src) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"(d), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
  return y;
}
// x = hi + lo with hi the leading 11 significant bits (truncated, exact in fp16) and lo the fp16-rounded remainder
__device__ __forceinline__ void split2h(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const float h0 = __uint_as_float(__float_as_uint(x0) & 0xFFFFE000u);
  const float h1 = __uint_as_float(__float_as_uint(x1) & 0xFFFFE000u);
  const __half2 h = __floats2half2_rn(h0, h1);
  const __half2 l = __floats2half2_rn(x0 - h0, x1 - h1);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
// 3-term split product: acc += a_lo*b_hi + a_hi*b_lo + a_hi*b_hi, b = {hi k0-7, hi k8-15, lo k0-7, lo k8-15}
__device__ __forceinline__ void mma3(float (&acc)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], const uint32_t (&b)[4]) {
  mma16816(acc, al, b[0], b[1]);
  mma16816(acc, ah, b[2], b[3]);
  mma16816(acc, ah, b[0], b[1]);
}

// Banded (+-band, + relative bias) softmax attention of the 16-query tile i0 .. i0+15 of one warp against K_h and V_h in shared
// memory (FlashAttention-2 style, as attn_tc.cu): scores in the log2 domain, 32-key blocks, each block's P*V added to the output
// with round-to-nearest fp32 adds.  Returns the normalised output split into hi / lo A fragments of the two k16 steps of the
// out-projection.
__device__ __forceinline__ void banded_attention(const uint32_t (&qh)[2][4], const uint32_t (&ql)[2][4], const __half* Kh,
                                                 const __half* Kl, const __half* Vh, const __half* Vl, const float* bias, int i0,
                                                 int band, int F, int lane, uint32_t (&oh)[2][4], uint32_t (&ol)[2][4]) {
  const int g = lane >> 2, t = lane & 3, lm = lane >> 3, lr = lane & 7;
  float o[4][4], mrow[2] = {-1e30f, -1e30f}, lrow[2] = {0.f, 0.f};
#pragma unroll
  for (int n = 0; n < 4; ++n)
#pragma unroll
    for (int c = 0; c < 4; ++c) o[n][c] = 0.f;
  const int kr_lo = max(0, i0 - band) & ~7, kr_hi = min(F, i0 + 16 + band);
  for (int kr0 = kr_lo; kr0 < kr_hi; kr0 += 32) {
    float s[4][4];
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int c = 0; c < 4; ++c) s[n][c] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        uint32_t b[4];
        ldsm4(b, ((lm & 2) ? Kl : Kh) + (kr0 + n * 8 + lr) * K_LD + ks * 16 + (lm & 1) * 8);
        mma3(s[n], qh[ks], ql[ks], b);
      }
    // relative position bias (+ band / sequence-end mask on the edge blocks only); every real row has a valid key in its first
    // block, so a masked score of -1e30 always meets a finite running maximum
    float mnew[2] = {mrow[0], mrow[1]};
    const int rel0 = kr0 - i0 + 2 * t - g;             // rel of element (n = 0, c = 0)
    const bool edge = (kr0 + 31 - i0 > band) || (kr0 - i0 - 15 < -band) || (kr0 + 32 > F);
    if (edge) {
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int rel = rel0 + n * 8 + (c & 1) - ((c & 2) ? 8 : 0);
          const bool v = ((unsigned)(rel + band) <= (unsigned)(2 * band)) && (kr0 + n * 8 + 2 * t + (c & 1) < F);
          s[n][c] = v ? s[n][c] + bias[v ? rel : 0] : -1e30f;
          mnew[c >> 1] = fmaxf(mnew[c >> 1], s[n][c]);
        }
    } else {
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          s[n][c] += bias[rel0 + n * 8 + (c & 1) - ((c & 2) ? 8 : 0)];
          mnew[c >> 1] = fmaxf(mnew[c >> 1], s[n][c]);
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mnew[r] = fmaxf(mnew[r], __shfl_xor_sync(0xffffffffu, mnew[r], 1));
      mnew[r] = fmaxf(mnew[r], __shfl_xor_sync(0xffffffffu, mnew[r], 2));
    }
    const float corr0 = ex2(mrow[0] - mnew[0]), corr1 = ex2(mrow[1] - mnew[1]);
    mrow[0] = mnew[0]; mrow[1] = mnew[1];
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      s[n][0] = ex2(s[n][0] - mnew[0]); s[n][1] = ex2(s[n][1] - mnew[0]);
      s[n][2] = ex2(s[n][2] - mnew[1]); s[n][3] = ex2(s[n][3] - mnew[1]);
      ps0 += s[n][0] + s[n][1]; ps1 += s[n][2] + s[n][3];
    }
    lrow[0] = lrow[0] * corr0 + ps0;
    lrow[1] = lrow[1] * corr1 + ps1;
#pragma unroll
    for (int n = 0; n < 4; ++n) { o[n][0] *= corr0; o[n][1] *= corr0; o[n][2] *= corr1; o[n][3] *= corr1; }
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      uint32_t ph[4], pl[4];                            // P's accumulator tiles (2ks, 2ks+1) == A fragment of k16 step ks
      split2h(s[2 * ks][0], s[2 * ks][1], ph[0], pl[0]);
      split2h(s[2 * ks][2], s[2 * ks][3], ph[1], pl[1]);
      split2h(s[2 * ks + 1][0], s[2 * ks + 1][1], ph[2], pl[2]);
      split2h(s[2 * ks + 1][2], s[2 * ks + 1][3], ph[3], pl[3]);
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        uint32_t b[4];
        ldsm4_trans(b, ((lm & 2) ? Vl : Vh) + (kr0 + ks * 16 + (lm & 1) * 8 + lr) * K_LD + n * 8);
        float acc[4] = {0.f, 0.f, 0.f, 0.f};            // RN accumulation across key blocks outside the tensor core
        mma3(acc, ph, pl, b);
        o[n][0] += acc[0]; o[n][1] += acc[1]; o[n][2] += acc[2]; o[n][3] += acc[3];
      }
    }
  }
  float l0 = lrow[0], l1 = lrow[1];
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    split2h(o[2 * ks][0] * inv0, o[2 * ks][1] * inv0, oh[ks][0], ol[ks][0]);
    split2h(o[2 * ks][2] * inv1, o[2 * ks][3] * inv1, oh[ks][1], ol[ks][1]);
    split2h(o[2 * ks + 1][0] * inv0, o[2 * ks + 1][1] * inv0, oh[ks][2], ol[ks][2]);
    split2h(o[2 * ks + 1][2] * inv1, o[2 * ks + 1][3] * inv1, oh[ks][3], ol[ks][3]);
  }
}

// out = residual + y for the frames of query tile qtile that this call owns
__device__ __forceinline__ void store_rows(const TemporalFusedArgs& a, int pix, int qtile, const float (&y)[8][4], int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int hrow = 0; hrow < 2; ++hrow) {
    const int f = qtile * 16 + g + 8 * hrow;
    if (f < a.q_lo || f >= a.q_hi) continue;
    const size_t orow = (size_t)(f - a.q_lo) * a.P + pix;
    const float* res = a.res + orow * a.ldr;
    float* dst = a.out + orow * a.ldo;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const float2 r = *reinterpret_cast<const float2*>(res + n * 8 + 2 * t);
      *reinterpret_cast<float2*>(dst + n * 8 + 2 * t) = make_float2(r.x + y[n][2 * hrow], r.y + y[n][2 * hrow + 1]);
    }
  }
}

__global__ void __launch_bounds__(NTH, 1) temporal_fused_kernel(TemporalFusedArgs a) {
  extern __shared__ __align__(16) unsigned char tf_smem[];
  const int F = a.F;                                   // sequence length held on chip (incl. halo frames when sharded)
  const int Fp = (F + 15) & ~15;                       // padded to whole 16-frame tiles
  const int KROWS = Fp + 32;                           // key rows incl. zero rows read by the last 32-key block
  const int nbuf = a.nbuf;                             // weight stages: 2 = next head's weights stream in behind the attention
  __half* Xh = reinterpret_cast<__half*>(tf_smem);
  __half* Xl = Xh + Fp * X_LD;
  __half* Kh = Xl + Fp * X_LD;
  __half* Kl = Kh + KROWS * K_LD;
  __half* Vh = Kl + KROWS * K_LD;                      // V_h row-major like K_h (B operand of P*V through ldmatrix.trans)
  __half* Vl = Vh + KROWS * K_LD;
  __half* Wst = Vl + KROWS * K_LD;                     // weight stages: [W'_h hi | lo : 2 x 96 x W_LD][Wout_h hi | lo : 2 x 64 x WO_LD]
  float* s_stat = reinterpret_cast<float*>(Wst + nbuf * W_STAGE);  // [Fp][2]  (mu, rstd)
  float* s_bias = s_stat + 2 * Fp;                                 // [8][2*band+1], pre-multiplied by log2(e)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int lm = lane >> 3, lr = lane & 7;             // ldmatrix: matrix index / row supplied by this lane
  const int pix = blockIdx.x;
  const int band = a.band;
  const int nbias = 2 * band + 1;

  // ------------------------------------------------------------------ phase 0: x rows of this pixel, LN statistics, fp16 split
  for (int i = tid; i < 8 * nbias; i += NTH) s_bias[i] = a.bias[i] * LOG2E;
  {
    const int l16 = tid & 15;                           // 16 lanes x float4 = one 64-channel row
    for (int f0 = 0; f0 < Fp; f0 += NTH / 16) {
      const int f = f0 + (tid >> 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f < F) v = __ldg(reinterpret_cast<const float4*>(a.x + ((size_t)f * a.P + pix) * a.ldx) + l16);
      float s = (v.x + v.y) + (v.z + v.w);
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mu = s * (1.0f / C);
      const float d0 = v.x - mu, d1 = v.y - mu, d2 = v.z - mu, d3 = v.w - mu;
      float ss = (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      if (f < Fp) {
        if (l16 == 0) { s_stat[2 * f] = mu; s_stat[2 * f + 1] = 1.0f / sqrtf(ss * (1.0f / C) + 1e-5f); }
        uint32_t h0, l0, h1, l1;
        split2h(v.x, v.y, h0, l0); split2h(v.z, v.w, h1, l1);
        *reinterpret_cast<uint2*>(&Xh[f * X_LD + l16 * 4]) = make_uint2(h0, h1);
        *reinterpret_cast<uint2*>(&Xl[f * X_LD + l16 * 4]) = make_uint2(l0, l1);
      }
    }
    // zero the key rows / value columns beyond the sequence once (masked lanes must multiply finite numbers)
    for (int i = tid; i < (KROWS - F) * K_LD; i += NTH) {
      Kh[F * K_LD + i] = __float2half(0.f); Kl[F * K_LD + i] = __float2half(0.f);
      Vh[F * K_LD + i] = __float2half(0.f); Vl[F * K_LD + i] = __float2half(0.f);
    }
  }

  const int ntiles = Fp >> 4;
  const int qtile = (a.q_lo >> 4) + warp;               // the 16-frame query tile this warp owns (if it holds an owned frame)
  const bool has_q = qtile * 16 < a.q_hi;
  float y[8][4];                                        // out-projection accumulators of the query tile: 8 n-tiles of 8 channels
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int c = 0; c < 4; ++c) y[n][c] = 0.f;

  // One projection part (0: q, 1: k, 2: v) of one 16-frame tile: acc = x_tile (16 x 64) * W'_h[part]^T (64 x 32), LayerNorm folded,
  // rotary applied to q and k.  Four independent accumulator chains (n-tiles) per k16 step.
  int head_off = 0;                                     // head * 32: column offset inside the q | k | v blocks of wsum
  const __half* Wh = Wst;                               // current stage (set per head)
  // stream one head's weights into a stage (fp16 hi | lo images, dense in global, padded rows in shared memory)
  auto stage_weights = [&](int head, __half* dst) {
    const uint4* src = reinterpret_cast<const uint4*>(a.Wqkv + (size_t)head * 2 * 96 * C);       // hi then lo, dense [96][64]
    for (int i = tid; i < 2 * 96 * C / 8; i += NTH) {
      const int r = i / (C / 8), c8 = i - r * (C / 8);                                             // r in [0, 192): hi rows then lo rows
      cp_async_16(dst + r * W_LD + c8 * 8, src + i);
    }
    const uint4* so = reinterpret_cast<const uint4*>(a.Wout + (size_t)head * 2 * 64 * 32);        // hi then lo, dense [64][32]
    __half* od = dst + 2 * 96 * W_LD;
    for (int i = tid; i < 2 * 64 * 32 / 8; i += NTH) {
      const int r = i >> 2, c8 = i & 3;                                                            // r in [0, 128)
      cp_async_16(od + r * WO_LD + c8 * 8, so + i);
    }
    cp_async_commit();
  };
  auto project = [&](int f0, int part, float (&acc)[4][4]) {
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[n][c] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint32_t ah[4], al[4];
      const int aoff = (f0 + (lm & 1) * 8 + lr) * X_LD + ks * 16 + (lm >> 1) * 8;
      ldsm4(ah, Xh + aoff);
      ldsm4(al, Xl + aoff);
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        uint32_t b[4];
        ldsm4(b, Wh + ((lm >> 1) * 96 + part * 32 + n * 8 + lr) * W_LD + ks * 16 + (lm & 1) * 8);
        mma3(acc[n], ah, al, b);
      }
    }
    const float mu0 = s_stat[2 * (f0 + g)], rs0 = s_stat[2 * (f0 + g) + 1];
    const float mu1 = s_stat[2 * (f0 + g + 8)], rs1 = s_stat[2 * (f0 + g + 8) + 1];
    const int fr0 = min(f0 + g, F - 1), fr1 = min(f0 + g + 8, F - 1);
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      const float2 w = __ldg(reinterpret_cast<const float2*>(a.wsum + part * 256 + head_off + n * 8 + 2 * t));
      acc[n][0] = rs0 * (acc[n][0] * a.inv_wscale - mu0 * w.x);
      acc[n][1] = rs0 * (acc[n][1] * a.inv_wscale - mu0 * w.y);
      acc[n][2] = rs1 * (acc[n][2] * a.inv_wscale - mu1 * w.x);
      acc[n][3] = rs1 * (acc[n][3] * a.inv_wscale - mu1 * w.y);
      if (part < 2) {                                    // rotary: interleaved pair (2i, 2i+1), pair index = n*4 + t
        const float2 cs0 = __ldg(reinterpret_cast<const float2*>(a.rot) + (size_t)fr0 * 16 + n * 4 + t);
        const float2 cs1 = __ldg(reinterpret_cast<const float2*>(a.rot) + (size_t)fr1 * 16 + n * 4 + t);
        const float x0 = acc[n][0], x1 = acc[n][1], x2 = acc[n][2], x3 = acc[n][3];
        acc[n][0] = x0 * cs0.x - x1 * cs0.y; acc[n][1] = x1 * cs0.x + x0 * cs0.y;
        acc[n][2] = x2 * cs1.x - x3 * cs1.y; acc[n][3] = x3 * cs1.x + x2 * cs1.y;
      }
    }
  };

  if (nbuf == 2) stage_weights(0, Wst);
  for (int head = 0; head < 8; ++head) {
    if (nbuf == 2) {
      cp_async_wait_all();
      __syncthreads();                                  // this head's weights landed; previous head's K/V and other stage are free
      Wh = Wst + (head & 1) * W_STAGE;
      if (head + 1 < 8) stage_weights(head + 1, Wst + ((head + 1) & 1) * W_STAGE);
    } else {
      __syncthreads();
      stage_weights(head, Wst);
      cp_async_wait_all();
      __syncthreads();
    }
    const __half* Oh = Wh + 2 * 96 * W_LD;              // Wout_h: hi rows [0, 64), lo rows [64, 128)
    head_off = head * 32;

    // ---------------------------------------------------------------- (b) K_h, V_h of every 16-frame tile (rotary on k)
    for (int tile = warp; tile < ntiles; tile += NWARP) {
      const int f0 = tile * 16, fr0 = f0 + g, fr1 = f0 + g + 8;
      float acc[4][4];
      project(f0, 1, acc);
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        uint32_t h0, l0, h1, l1;
        split2h(acc[n][0], acc[n][1], h0, l0); split2h(acc[n][2], acc[n][3], h1, l1);
        *reinterpret_cast<uint32_t*>(&Kh[fr0 * K_LD + n * 8 + 2 * t]) = h0;
        *reinterpret_cast<uint32_t*>(&Kl[fr0 * K_LD + n * 8 + 2 * t]) = l0;
        *reinterpret_cast<uint32_t*>(&Kh[fr1 * K_LD + n * 8 + 2 * t]) = h1;
        *reinterpret_cast<uint32_t*>(&Kl[fr1 * K_LD + n * 8 + 2 * t]) = l1;
      }
      project(f0, 2, acc);
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        uint32_t h0, l0, h1, l1;
        split2h(acc[n][0], acc[n][1], h0, l0); split2h(acc[n][2], acc[n][3], h1, l1);
        *reinterpret_cast<uint32_t*>(&Vh[fr0 * K_LD + n * 8 + 2 * t]) = h0;
        *reinterpret_cast<uint32_t*>(&Vl[fr0 * K_LD + n * 8 + 2 * t]) = l0;
        *reinterpret_cast<uint32_t*>(&Vh[fr1 * K_LD + n * 8 + 2 * t]) = h1;
        *reinterpret_cast<uint32_t*>(&Vl[fr1 * K_LD + n * 8 + 2 * t]) = l1;
      }
    }
    // ---------------------------------------------------------------- (c) Q_h of the owned query tile -> A fragments in registers
    uint32_t qh[2][4], ql[2][4];
    if (has_q) {
      float acc[4][4];
      project(qtile * 16, 0, acc);
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[n][c] *= LOG2E;   // scores live in the log2 domain: softmax through ex2
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {                    // accumulator tiles (2ks, 2ks+1) == A fragment of k16 step ks
        split2h(acc[2 * ks][0], acc[2 * ks][1], qh[ks][0], ql[ks][0]);
        split2h(acc[2 * ks][2], acc[2 * ks][3], qh[ks][1], ql[ks][1]);
        split2h(acc[2 * ks + 1][0], acc[2 * ks + 1][1], qh[ks][2], ql[ks][2]);
        split2h(acc[2 * ks + 1][2], acc[2 * ks + 1][3], qh[ks][3], ql[ks][3]);
      }
    }
    __syncthreads();                                    // K_h, V_h^T of every frame are in shared memory
    if (!has_q) continue;

    // ---------------------------------------------------------------- (d) banded attention of the query tile
    uint32_t oh[2][4], ol[2][4];
    banded_attention(qh, ql, Kh, Kl, Vh, Vl, s_bias + head * nbias + band, qtile * 16, band, F, lane, oh, ol);
    // ---------------------------------------------------------------- (e) y_tile += O_h (16 x 32) * Wout_h^T (32 x 64)
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        uint32_t b[4];
        ldsm4(b, Oh + ((lm >> 1) * 64 + n * 8 + lr) * WO_LD + ks * 16 + (lm & 1) * 8);
        mma3(acc, oh[ks], ol[ks], b);
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) y[n][c] += acc[c] * a.inv_oscale;           // RN accumulation over heads outside the tensor core
    }
  }

  // ------------------------------------------------------------------ out = residual + y for the frames this call owns
  if (has_q) store_rows(a, pix, qtile, y, lane);
}

// ==================================================================== the same operation with the dense GEMMs on warpgroup MMAs
// For sequences of at most 256 frames.  Warpgroup g projects frames 64g .. 64g+63 of head h with one m64n96k16 chain (q | k | v),
// both operands read from 128-byte-swizzled shared-memory panels by descriptor, and adds O_h * Wout_h^T with m64n64k16 whose A
// operand is the attention output in registers.  Warp w of warpgroup g owns query tile 4g + w: rows 16w .. 16w+15 of the
// warpgroup's accumulator, in the m16n8 layout the QK^T A fragments need, so Q never leaves registers.  The banded attention is
// the mma.sync code above.  Accumulator chains are as long as in temporal_fused_kernel (K 64 in the projection, 32 per head in the
// out-projection) and the split terms run in the same order, lo*hi, hi*lo, hi*hi.
constexpr int WG_ROWS = 256;                    // frames on chip: 4 warpgroups x 64 rows of X panels and LayerNorm statistics
constexpr int WG_WQ = 96 * 128;                 // bytes of one swizzled [96][64] fp16 panel of W'_h (hi or lo)
constexpr int WG_WO = 64 * 128;                 // bytes of the swizzled Wout_h panel: [64 channels][hi d 0-31 | lo d 0-31]
constexpr int WG_STAGE = 2 * WG_WQ + WG_WO;     // one head's weights; two stages, the next head streams in behind this one
constexpr int WG_KROWS = WG_ROWS + 32;          // key rows incl. zero rows read by the last 32-key block
// Fixed layout for every F (one CTA per SM at any size), so every shared-memory address is the aligned base plus a constant:
// 1024 B of alignment slack, X hi | lo, two weight stages, K_h / V_h hi | lo (rows of K_LD halfs, as temporal_fused_kernel),
// LayerNorm statistics, relative bias at the largest band (64)
constexpr int WG_OFF_K = 2 * WG_ROWS * 128 + 2 * WG_STAGE;
constexpr int WG_OFF_STAT = WG_OFF_K + 4 * WG_KROWS * K_LD * 2;
constexpr int WG_SMEM = 1024 + WG_OFF_STAT + (2 * WG_ROWS + 8 * (2 * 64 + 1)) * 4;
static_assert(WG_SMEM == 230432 && WG_SMEM <= 227 * 1024, "225.0 KB: within the H100's 227 KB per-block opt-in limit");

__global__ void __launch_bounds__(NTH, 1) temporal_fused_wg_kernel(TemporalFusedArgs a) {
  extern __shared__ __align__(16) unsigned char tf_smem[];
  const int F = a.F, Fp = (F + 15) & ~15;
  uint8_t* Xh = tc::smem_align1024(tf_smem);            // [256][64] fp16 K-major panels, 128-byte swizzle
  uint8_t* Xl = Xh + WG_ROWS * 128;
  uint8_t* Wst = Xl + WG_ROWS * 128;                    // stage: [W'_h hi][W'_h lo][Wout_h hi | lo]
  __half* Kh = reinterpret_cast<__half*>(Xh + WG_OFF_K);
  __half* Kl = Kh + WG_KROWS * K_LD;
  __half* Vh = Kl + WG_KROWS * K_LD;
  __half* Vl = Vh + WG_KROWS * K_LD;
  float* s_stat = reinterpret_cast<float*>(Xh + WG_OFF_STAT);     // [256][2] (mu, rstd); (0, 0) past the sequence
  float* s_bias = s_stat + 2 * WG_ROWS;                           // [8][2*band+1], pre-multiplied by log2(e)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int g = lane >> 2, t = lane & 3;
  const int pix = blockIdx.x;
  const int band = a.band;
  const int nbias = 2 * band + 1;

  // ------------------------------------------------------------------ phase 0: x rows of this pixel, LN statistics, fp16 split
  for (int i = tid; i < 8 * nbias; i += NTH) s_bias[i] = a.bias[i] * LOG2E;
  {
    const int l16 = tid & 15;                           // 16 lanes x float4 = one 64-channel row
    for (int f0 = 0; f0 < WG_ROWS; f0 += NTH / 16) {    // rows F .. 255 are zero with zero statistics: they project to zeros
      const int f = f0 + (tid >> 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f < F) v = __ldg(reinterpret_cast<const float4*>(a.x + ((size_t)f * a.P + pix) * a.ldx) + l16);
      float s = (v.x + v.y) + (v.z + v.w);
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mu = s * (1.0f / C);
      const float d0 = v.x - mu, d1 = v.y - mu, d2 = v.z - mu, d3 = v.w - mu;
      float ss = (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      if (l16 == 0) { s_stat[2 * f] = mu; s_stat[2 * f + 1] = f < F ? 1.0f / sqrtf(ss * (1.0f / C) + 1e-5f) : 0.f; }
      uint32_t h0, l0, h1, l1;
      split2h(v.x, v.y, h0, l0); split2h(v.z, v.w, h1, l1);
      const uint32_t off = tc::swz(f, l16 >> 1) + (l16 & 1) * 8;
      *reinterpret_cast<uint2*>(Xh + off) = make_uint2(h0, h1);
      *reinterpret_cast<uint2*>(Xl + off) = make_uint2(l0, l1);
    }
    // zero the key rows / value columns beyond the sequence once (masked lanes must multiply finite numbers)
    for (int i = tid; i < (Fp + 32 - F) * K_LD; i += NTH) {
      Kh[F * K_LD + i] = __float2half(0.f); Kl[F * K_LD + i] = __float2half(0.f);
      Vh[F * K_LD + i] = __float2half(0.f); Vl[F * K_LD + i] = __float2half(0.f);
    }
  }

  const int qtile = warp;                               // the 16-frame query tile this warp owns (if it holds an owned frame)
  const bool has_q = qtile * 16 < a.q_hi && qtile * 16 + 16 > a.q_lo;
  const bool projects = wg * 64 < Fp;                   // warpgroup-uniform: its 64 rows reach into the sequence
  float y[8][4];                                        // out-projection accumulators of the query tile: 8 n-tiles of 8 channels
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int c = 0; c < 4; ++c) y[n][c] = 0.f;

  // stream one head's weights into a stage: the packed dense images (as temporal_fused_kernel reads them) land in swizzled panels
  auto stage_weights = [&](int head, uint8_t* dst) {
    const uint4* src = reinterpret_cast<const uint4*>(a.Wqkv + (size_t)head * 2 * 96 * C);       // hi then lo, dense [96][64]
    for (int i = tid; i < 2 * 96 * C / 8; i += NTH) cp_async_16(dst + tc::swz(i >> 3, i & 7), src + i);   // lo panel = rows 96..
    const uint4* so = reinterpret_cast<const uint4*>(a.Wout + (size_t)head * 2 * 64 * 32);        // hi then lo, dense [64][32]
    for (int i = tid; i < 2 * 64 * 32 / 8; i += NTH)
      cp_async_16(dst + 2 * WG_WQ + tc::swz((i >> 2) & 63, (i >> 8) * 4 + (i & 3)), so + i);
    cp_async_commit();
  };

  stage_weights(0, Wst);
  for (int head = 0; head < 8; ++head) {
    cp_async_wait_all();
    tc::fence_proxy_async();                            // generic-proxy writes (X panels, this head's weights) -> wgmma reads
    __syncthreads();                                    // this head's weights landed; previous head's K/V and other stage are free
    const uint8_t* Ws = Wst + (head & 1) * WG_STAGE;
    if (head + 1 < 8) stage_weights(head + 1, Wst + ((head + 1) & 1) * WG_STAGE);

    // ---------------------------------------------------------------- (b) q | k | v of the warpgroup's 64 frames
    uint32_t qh[2][4], ql[2][4];
    if (projects) {
      float d[48];                                      // n-tile j: q (0-3), k (4-7), v (8-11) of 8 head dims each
      const uint64_t ahi = tc::make_desc(tc::smem_u32(Xh + wg * 64 * 128)), alo = tc::make_desc(tc::smem_u32(Xl + wg * 64 * 128));
      const uint64_t bhi = tc::make_desc(tc::smem_u32(Ws)), blo = tc::make_desc(tc::smem_u32(Ws + WG_WQ));
      tc::wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t o = (uint64_t)(ks * 2);          // +32 bytes per k-step, in 16-byte units
        tc::wgmma_m64n96k16(d, alo + o, bhi + o, ks == 0 ? 0u : 1u);
        tc::wgmma_m64n96k16(d, ahi + o, blo + o, 1u);
        tc::wgmma_m64n96k16(d, ahi + o, bhi + o, 1u);
      }
      tc::wgmma_commit();
      tc::wgmma_wait<0>();
      tc::wgmma_fence_acc(d);
      // LayerNorm fold, rotary on q and k (interleaved pair (2i, 2i+1), pair index = n*4 + t)
      const int f0 = warp * 16;
      const float mu0 = s_stat[2 * (f0 + g)], rs0 = s_stat[2 * (f0 + g) + 1];
      const float mu1 = s_stat[2 * (f0 + g + 8)], rs1 = s_stat[2 * (f0 + g + 8) + 1];
      const int fr0 = min(f0 + g, F - 1), fr1 = min(f0 + g + 8, F - 1);
#pragma unroll
      for (int j = 0; j < 12; ++j) {
        const int part = j >> 2, n = j & 3;
        float* acc = d + 4 * j;
        const float2 w = __ldg(reinterpret_cast<const float2*>(a.wsum + part * 256 + head * 32 + n * 8 + 2 * t));
        acc[0] = rs0 * (acc[0] * a.inv_wscale - mu0 * w.x);
        acc[1] = rs0 * (acc[1] * a.inv_wscale - mu0 * w.y);
        acc[2] = rs1 * (acc[2] * a.inv_wscale - mu1 * w.x);
        acc[3] = rs1 * (acc[3] * a.inv_wscale - mu1 * w.y);
        if (part < 2) {
          const float2 cs0 = __ldg(reinterpret_cast<const float2*>(a.rot) + (size_t)fr0 * 16 + n * 4 + t);
          const float2 cs1 = __ldg(reinterpret_cast<const float2*>(a.rot) + (size_t)fr1 * 16 + n * 4 + t);
          const float x0 = acc[0], x1 = acc[1], x2 = acc[2], x3 = acc[3];
          acc[0] = x0 * cs0.x - x1 * cs0.y; acc[1] = x1 * cs0.x + x0 * cs0.y;
          acc[2] = x2 * cs1.x - x3 * cs1.y; acc[3] = x3 * cs1.x + x2 * cs1.y;
        }
      }
      if (f0 < Fp) {                                    // K_h, V_h of the warp's tile to shared memory as fp16 hi / lo
        const int r0 = f0 + g, r1 = f0 + g + 8;
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          uint32_t h0, l0, h1, l1;
          split2h(d[16 + 4 * n], d[16 + 4 * n + 1], h0, l0); split2h(d[16 + 4 * n + 2], d[16 + 4 * n + 3], h1, l1);
          *reinterpret_cast<uint32_t*>(&Kh[r0 * K_LD + n * 8 + 2 * t]) = h0;
          *reinterpret_cast<uint32_t*>(&Kl[r0 * K_LD + n * 8 + 2 * t]) = l0;
          *reinterpret_cast<uint32_t*>(&Kh[r1 * K_LD + n * 8 + 2 * t]) = h1;
          *reinterpret_cast<uint32_t*>(&Kl[r1 * K_LD + n * 8 + 2 * t]) = l1;
          split2h(d[32 + 4 * n], d[32 + 4 * n + 1], h0, l0); split2h(d[32 + 4 * n + 2], d[32 + 4 * n + 3], h1, l1);
          *reinterpret_cast<uint32_t*>(&Vh[r0 * K_LD + n * 8 + 2 * t]) = h0;
          *reinterpret_cast<uint32_t*>(&Vl[r0 * K_LD + n * 8 + 2 * t]) = l0;
          *reinterpret_cast<uint32_t*>(&Vh[r1 * K_LD + n * 8 + 2 * t]) = h1;
          *reinterpret_cast<uint32_t*>(&Vl[r1 * K_LD + n * 8 + 2 * t]) = l1;
        }
      }
      if (has_q) {                                      // Q_h stays in registers as the A fragments of Q K^T
#pragma unroll
        for (int i = 0; i < 16; ++i) d[i] *= LOG2E;     // scores live in the log2 domain: softmax through ex2
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {                // accumulator tiles (2ks, 2ks+1) == A fragment of k16 step ks
          split2h(d[8 * ks], d[8 * ks + 1], qh[ks][0], ql[ks][0]);
          split2h(d[8 * ks + 2], d[8 * ks + 3], qh[ks][1], ql[ks][1]);
          split2h(d[8 * ks + 4], d[8 * ks + 5], qh[ks][2], ql[ks][2]);
          split2h(d[8 * ks + 6], d[8 * ks + 7], qh[ks][3], ql[ks][3]);
        }
      }
    }
    __syncthreads();                                    // K_h, V_h of every frame are in shared memory

    // ---------------------------------------------------------------- (d) banded attention of the query tile
    uint32_t oh[2][4] = {}, ol[2][4] = {};              // warps without an owned frame join the out-projection with zeros
    if (has_q) banded_attention(qh, ql, Kh, Kl, Vh, Vl, s_bias + head * nbias + band, qtile * 16, band, F, lane, oh, ol);
    // ---------------------------------------------------------------- (e) y_tile += O_h (16 x 32) * Wout_h^T (32 x 64)
    float acc[32];                                      // fresh per head: RN accumulation over heads outside the tensor core
    const uint64_t bo = tc::make_desc(tc::smem_u32(Ws + 2 * WG_WQ));   // hi k16 steps at +0 / +32 B, lo at +64 / +96 B
    tc::wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      tc::wgmma_m64n64k16_rs(acc, ol[ks], bo + ks * 2, ks == 0 ? 0u : 1u);
      tc::wgmma_m64n64k16_rs(acc, oh[ks], bo + 4 + ks * 2, 1u);
      tc::wgmma_m64n64k16_rs(acc, oh[ks], bo + ks * 2, 1u);
    }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::wgmma_fence_acc(acc);
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int c = 0; c < 4; ++c) y[n][c] += acc[4 * n + c] * a.inv_oscale;
  }

  // ------------------------------------------------------------------ out = residual + y for the frames this call owns
  if (has_q) store_rows(a, pix, qtile, y, lane);
}

size_t smem_bytes(int F, int band, int nbuf) {
  const int Fp = (F + 15) & ~15, KROWS = Fp + 32;
  size_t halfs = (size_t)2 * Fp * X_LD + 4 * KROWS * K_LD + (size_t)nbuf * W_STAGE;
  return halfs * 2 + (size_t)(2 * Fp + 8 * (2 * band + 1)) * 4;
}
constexpr size_t kSmemMax = 225 * 1024;

}  // namespace

bool temporal_fused_supported(int C_, int F, int band, int q_lo, int q_hi) {
  if (C_ != C || band < 1 || band > 64 || F < 1 || q_lo < 0 || q_hi > F || q_lo >= q_hi) return false;
  if (((q_hi + 15) >> 4) - (q_lo >> 4) > NWARP) return false;   // one 16-frame query tile per warp
  return smem_bytes(F, band, 1) <= kSmemMax;
}

// every shape temporal_fused_supported takes; all of them pass the mma.sync kernel's checks above too
bool temporal_fused_wg_supported(int C_, int F, int band, int q_lo, int q_hi) {
  return C_ == C && band >= 1 && band <= 64 && F >= 1 && F <= WG_ROWS && q_lo >= 0 && q_hi <= F && q_lo < q_hi;
}

int launch_temporal_fused(const TemporalFusedArgs& a_in, cudaStream_t st, bool mma_sync_only) {
  if (!temporal_fused_supported(C, a_in.F, a_in.band, a_in.q_lo, a_in.q_hi)) { set_last_error("temporal_fused: unsupported shape"); return -1; }
  if (!mma_sync_only && temporal_fused_wg_supported(C, a_in.F, a_in.band, a_in.q_lo, a_in.q_hi)) {
    static bool attr_set = false;
    if (!attr_set) {
      DAWN_CUDA_OK(cudaFuncSetAttribute(temporal_fused_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM));
      attr_set = true;
    }
    temporal_fused_wg_kernel<<<a_in.P, NTH, WG_SMEM, st>>>(a_in);
    DAWN_LAUNCH_OK();
    return 0;
  }
  static size_t attr_bytes = 0;
  TemporalFusedArgs a = a_in;
  a.nbuf = smem_bytes(a.F, a.band, 2) <= kSmemMax ? 2 : 1;
  const size_t smem = smem_bytes(a.F, a.band, a.nbuf);
  if (smem > attr_bytes) {
    DAWN_CUDA_OK(cudaFuncSetAttribute(temporal_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_bytes = smem;
  }
  temporal_fused_kernel<<<a.P, NTH, smem, st>>>(a);
  DAWN_LAUNCH_OK();
  return 0;
}

// Host packing.  wqkv: [768][64] fp32 rows = output columns (q | k | v blocks of 256, gamma and q-scale folded), wout: [64][256].
// Produces per head: W'_h [96][64] fp16 hi then lo (rows: q 32, k 32, v 32), Wout_h [64][32] fp16 hi then lo; both pre-scaled by exact
// powers of two (returned as inverse scales).
void temporal_fused_pack(const float* wqkv, const float* wout, std::vector<uint16_t>& Wq, std::vector<uint16_t>& Wo, float* inv_wscale,
                         float* inv_oscale) {
  auto pow2scale = [](const float* p, size_t n) {
    float mx = 0.f;
    for (size_t i = 0; i < n; ++i) mx = std::max(mx, std::fabs(p[i]));
    int e = 0;
    if (mx > 0.f) std::frexp(mx, &e);
    return std::ldexp(1.0f, 11 - e);
  };
  const float sq = pow2scale(wqkv, (size_t)768 * 64), so = pow2scale(wout, (size_t)64 * 256);
  *inv_wscale = 1.0f / sq; *inv_oscale = 1.0f / so;
  auto put = [](uint16_t* hi, uint16_t* lo, float v) {
    const __half h = __float2half_rn(v);
    const __half l = __float2half_rn(v - __half2float(h));
    memcpy(hi, &h, 2); memcpy(lo, &l, 2);
  };
  Wq.assign((size_t)8 * 2 * 96 * 64, 0);
  Wo.assign((size_t)8 * 2 * 64 * 32, 0);
  for (int h = 0; h < 8; ++h) {
    uint16_t* qh = Wq.data() + (size_t)h * 2 * 96 * 64; uint16_t* ql = qh + 96 * 64;
    for (int part = 0; part < 3; ++part)
      for (int r = 0; r < 32; ++r)
        for (int k = 0; k < 64; ++k)
          put(qh + (part * 32 + r) * 64 + k, ql + (part * 32 + r) * 64 + k, wqkv[(size_t)(part * 256 + h * 32 + r) * 64 + k] * sq);
    uint16_t* oh = Wo.data() + (size_t)h * 2 * 64 * 32; uint16_t* ol = oh + 64 * 32;
    for (int c = 0; c < 64; ++c)
      for (int d = 0; d < 32; ++d) put(oh + c * 32 + d, ol + c * 32 + d, wout[(size_t)c * 256 + h * 32 + d] * so);
  }
}

}  // namespace dawn
