// Cross-attention gate weights of a conditioned ResnetBlock (reference U:454-463, 505-560), fused for ci <= 128:
//
//   x (block input, M x ci)  ->  LayerNorm_img  ->  q = x^ Wq (3 cross-attentions x 8 heads x 8 dims)
//      ->  per head: cosine-similarity logits against the frame's key and the null key, 2-way softmax  ->  gate
//      ->  per cross-attention: rstd of the LayerNorm'd to_out output from the 9x9 Gram form  ->  Wt (M x 32)
//
// Every frame has exactly two keys per cross-attention (its conditioning token and the learned null token), so the attention output
// is an affine function of one gate per head; unet.cu folds to_out / LayerNorm into per-frame tables (T, G) and the block only needs
// Wt = rstd * [1, gate_0..7] per cross-attention.  The unfused path ran a wgmma GEMM with N = 192 (three 64-column tiles, each
// re-gathering and re-splitting the A rows; gates through HBM) plus ca_rstd_kernel.  Here a warp owns 16 pixels: q comes out of
// mma.sync (3-term FP16 split, fp32 accumulate) 64 columns at a time, the accumulator layout gives each quad one head per n-tile, and
// the gates never leave the SM.
#include <cuda_fp16.h>
#include <algorithm>
#include <cmath>
#include <vector>
#include "common.cuh"
#include "f16x3.cuh"
#include "kernels.cuh"
#include "ca_fused.cuh"

namespace dawn {
namespace {

constexpr int NTH = 256;
constexpr int CHUNK = 128;             // pixels staged per iteration: one 16-pixel group per warp
constexpr int WT_LD = 36;              // floats per row of a warp's gate / Wt patch (bank-conflict-free column writes)

template <int CI>
__global__ void __launch_bounds__(NTH, (CI == 64) ? 2 : 1) ca_wt_kernel(CaFusedArgs a) {
  constexpr int LD = CI + 8;                            // halfs per shared-memory row
  constexpr int LPR = CI / 4;                           // lanes (float4 each) per pixel row
  constexpr int RPP = NTH / LPR;                        // rows per staging pass
  constexpr int NPASS = CHUNK / RPP;
  constexpr int KS = CI / 16;
  extern __shared__ __align__(16) unsigned char ca_smem[];
  __half* Wh = reinterpret_cast<__half*>(ca_smem);      // [192][LD] hi
  __half* Wl = Wh + 192 * LD;
  __half* Xh = Wl + 192 * LD;                           // [CHUNK][LD]
  __half* Xl = Xh + CHUNK * LD;
  float* s_kq = reinterpret_cast<float*>(Xl + CHUNK * LD);   // [3][64] this frame's projected keys (q/k scales folded)
  float* s_nk = s_kq + 192;                             // [3][8] null keys
  float* s_G = s_nk + 24;                               // [3][81] Gram forms
  float* s_wt = s_G + 244;                              // [8 warps][16][WT_LD] gate / Wt patch

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3, lm = lane >> 3, lr = lane & 7;
  const int f = blockIdx.y, split = blockIdx.x;
  const int px_lo = split * a.px_per_cta, px_hi = min(a.P, px_lo + a.px_per_cta);

  {
    const uint4* src = reinterpret_cast<const uint4*>(a.Wq);      // dense [hi|lo][192][CI] fp16
    for (int i = tid; i < 2 * 192 * CI / 8; i += NTH) {
      const int r = i / (CI / 8), c8 = i - r * (CI / 8);
      cp_async16(Wh + r * LD + c8 * 8, src + i);
    }
    cp_async_commit();
    for (int i = tid; i < 192; i += NTH) s_kq[i] = a.kq[(size_t)f * 192 + i];
    if (tid < 24) s_nk[tid] = a.nkq[tid];
    for (int i = tid; i < 243; i += NTH) s_G[i] = a.G[(size_t)f * 243 + i];
  }

  const int lrow = tid % LPR;
  float4 xin[NPASS];
  auto fetch = [&](int p0) {
#pragma unroll
    for (int i = 0; i < NPASS; ++i) {
      const int px = p0 + i * RPP + tid / LPR;
      xin[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (px < px_hi) xin[i] = __ldg(reinterpret_cast<const float4*>(a.x + ((size_t)f * a.P + px) * a.ldx) + lrow);
    }
  };
  fetch(px_lo);
  float* wt = s_wt + warp * 16 * WT_LD;

  for (int p0 = px_lo; p0 < px_hi; p0 += CHUNK) {
    __syncthreads();
    // ---------------------------------------------------------------- stage CHUNK pixels: LayerNorm_img, fp16 hi/lo
#pragma unroll
    for (int i = 0; i < NPASS; ++i) {
      const int r = i * RPP + tid / LPR;
      const float4 v = xin[i];
      const float2 st = row_ln_stats<LPR, CI>(v);
      const float mu = st.x, rs = st.y;
      uint32_t h0, l0, h1, l1;
      split_f16x2_trunc((v.x - mu) * rs, (v.y - mu) * rs, h0, l0); split_f16x2_trunc((v.z - mu) * rs, (v.w - mu) * rs, h1, l1);
      *reinterpret_cast<uint2*>(&Xh[r * LD + lrow * 4]) = make_uint2(h0, h1);
      *reinterpret_cast<uint2*>(&Xl[r * LD + lrow * 4]) = make_uint2(l0, l1);
    }
    cp_async_wait<0>();
    __syncthreads();
    if (p0 + CHUNK < px_hi) fetch(p0 + CHUNK);

    const int grp0 = p0 + warp * 16;                    // this warp's 16 pixels
    if (grp0 >= px_hi) continue;
    // A fragments of the 16 x CI pixel tile
    uint32_t ah[KS][4], al[KS][4];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const int aoff = (warp * 16 + (lm & 1) * 8 + lr) * LD + ks * 16 + (lm >> 1) * 8;
      ldsm4(ah[ks], Xh + aoff);
      ldsm4(al[ks], Xl + aoff);
    }
#pragma unroll 1
    for (int ca = 0; ca < 3; ++ca) {
      float q[8][4];                                    // n-tile = head, columns 2t, 2t+1 = head dims
#pragma unroll
      for (int n = 0; n < 8; ++n)
#pragma unroll
        for (int c = 0; c < 4; ++c) q[n][c] = 0.f;
#pragma unroll
      for (int ks = 0; ks < KS; ++ks)
#pragma unroll
        for (int n = 0; n < 8; ++n) {
          uint32_t b[4];
          ldsm4(b, ((lm & 2) ? Wl : Wh) + (ca * 64 + n * 8 + lr) * LD + ks * 16 + (lm & 1) * 8);
          mma3(q[n], ah[ks], al[ks], b);
        }
      // per-lane partial sums over its two head dims: |q|^2, q.k, q.k_null for rows g (a) and g+8 (b) of every head
      const float2 nk = *reinterpret_cast<const float2*>(s_nk + ca * 8 + 2 * t);
      float v[8][6];
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const float2 k = *reinterpret_cast<const float2*>(s_kq + ca * 64 + n * 8 + 2 * t);
        const float q0 = q[n][0] * a.inv_wscale, q1 = q[n][1] * a.inv_wscale, q2 = q[n][2] * a.inv_wscale, q3 = q[n][3] * a.inv_wscale;
        v[n][0] = q0 * q0 + q1 * q1; v[n][1] = q0 * k.x + q1 * k.y; v[n][2] = q0 * nk.x + q1 * nk.y;
        v[n][3] = q2 * q2 + q3 * q3; v[n][4] = q2 * k.x + q3 * k.y; v[n][5] = q2 * nk.x + q3 * nk.y;
      }
      // reduce-scatter over the quad: lane t ends up with the complete sums of heads t and t + 4
      float w[4][6], u[2][6];
      const bool odd = t & 1, hi2 = t & 2;
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 6; ++e) {
          const float send = odd ? v[2 * j][e] : v[2 * j + 1][e];
          const float keep = odd ? v[2 * j + 1][e] : v[2 * j][e];
          w[j][e] = keep + __shfl_xor_sync(0xffffffffu, send, 1);          // head 2j + (t & 1)
        }
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 6; ++e) {
          const float send = hi2 ? w[2 * j][e] : w[2 * j + 1][e];
          const float keep = hi2 ? w[2 * j + 1][e] : w[2 * j][e];
          u[j][e] = keep + __shfl_xor_sync(0xffffffffu, send, 2);          // head 4j + t
        }
      // l2-normalised q (F.normalize, eps 1e-12) x scale 8; two-way softmax over {key, null key} = sigmoid(s_key - s_null)
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float n2 = u[j][3 * r], dr = u[j][3 * r + 1], dn = u[j][3 * r + 2];
          const float inv = 8.0f * rsqrtf(fmaxf(n2, 1e-24f));
          const float gate = __fdividef(1.0f, 1.0f + __expf((dn - dr) * inv));
          wt[(g + 8 * r) * WT_LD + ca * 8 + 4 * j + t] = gate;
        }
    }
    __syncwarp();
    // ---------------------------------------------------------------- rstd from the Gram form; Wt row = [rs*[1, gates] x 3, 0 x 5]
    float outv[2][9];
    float rsv[2];
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int item = lane + 32 * it;                  // (row, ca): 48 items
      const int row = item / 3, ca = item - row * 3;
      if (item < 48) {
        float c[9];
        c[0] = 1.f;
#pragma unroll
        for (int hd = 0; hd < 8; ++hd) c[hd + 1] = wt[row * WT_LD + ca * 8 + hd];
        const float* G = s_G + ca * 81;
        float var = 0.f;
#pragma unroll
        for (int i = 0; i < 9; ++i) {
          float rowv = 0.f;
#pragma unroll
          for (int j = 0; j < 9; ++j) rowv += G[i * 9 + j] * c[j];
          var += c[i] * rowv;
        }
        rsv[it] = rsqrtf(fmaxf(var, 0.f) + 1e-5f);
#pragma unroll
        for (int i = 0; i < 9; ++i) outv[it][i] = rsv[it] * c[i];
      }
    }
    __syncwarp();                                       // all gates read before the patch is overwritten
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int item = lane + 32 * it;
      const int row = item / 3, ca = item - row * 3;
      if (item < 48) {
#pragma unroll
        for (int i = 0; i < 9; ++i) wt[row * WT_LD + ca * 9 + i] = outv[it][i];
      }
    }
    if (lane < 16) {
#pragma unroll
      for (int k = 27; k < 32; ++k) wt[lane * WT_LD + k] = 0.f;
    }
    __syncwarp();
    // 16 rows x 128 B are contiguous in Wt (ld 32): coalesced float4 stores
    float4* dst = reinterpret_cast<float4*>(a.Wt + ((size_t)f * a.P + grp0) * 32);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = lane + 32 * i;                    // float4 index in the dense 16 x 32 tile
      dst[idx] = *reinterpret_cast<const float4*>(wt + (idx >> 3) * WT_LD + (idx & 7) * 4);
    }
    __syncwarp();
  }
}

template <int CI>
constexpr size_t smem_bytes() { return (size_t)(2 * 192 * (CI + 8) + 2 * CHUNK * (CI + 8)) * 2 + (size_t)(192 + 24 + 244 + 8 * 16 * WT_LD) * 4; }

template <int CI>
int launch_ci(CaFusedArgs a, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    DAWN_CUDA_OK(cudaFuncSetAttribute(ca_wt_kernel<CI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<CI>()));
    attr = true;
  }
  // pixel runs of 512 (fewer for small frames): F * splits CTAs
  int px = 512;
  while (px > CHUNK && a.P % px != 0) px >>= 1;
  a.px_per_cta = px;
  const int nsplit = (a.P + px - 1) / px;
  ca_wt_kernel<CI><<<dim3(nsplit, a.F), NTH, smem_bytes<CI>(), st>>>(a);
  DAWN_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------------------
// a1 = SiLU(FiLM(GroupNorm(y))) + Wt (M x 32) * T_f (32 x co)      (first half of a conditioned ResnetBlock, U:366-380, 454-463)
// A streaming kernel: Wt rows arrive straight in A-fragment order from global memory, the frame's table T_f sits in shared memory as
// fp16 hi|lo, the K = 32 product is 6 mma.sync per 8 channels, and the epilogue reads y / writes a1 in 32-byte quad segments.
// transpose the 4 x 4 matrix M[lane t of the quad][i] in place: afterwards v[j] = what lane j held in its v[t]
__device__ __forceinline__ void quad_transpose(uint32_t (&v)[4], int t) {
  {   // exchange 2 x 2 blocks with the lane two away
    const bool up = (t & 2) != 0;
    const uint32_t s0 = up ? v[0] : v[2], s1 = up ? v[1] : v[3];
    const uint32_t r0 = __shfl_xor_sync(0xffffffffu, s0, 2), r1 = __shfl_xor_sync(0xffffffffu, s1, 2);
    if (up) { v[0] = r0; v[1] = r1; } else { v[2] = r0; v[3] = r1; }
  }
  {   // exchange single elements with the neighbouring lane
    const bool up = (t & 1) != 0;
    const uint32_t s0 = up ? v[0] : v[1], s1 = up ? v[2] : v[3];
    const uint32_t r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
    if (up) { v[0] = r0; v[2] = r1; } else { v[1] = r0; v[3] = r1; }
  }
}

template <bool SPLIT>
__global__ void __launch_bounds__(NTH, 3) gn_hcond_kernel(GnHcondArgs a) {
  constexpr int TLD = 40;
  extern __shared__ __align__(16) unsigned char gh_smem[];
  __half* Th = reinterpret_cast<__half*>(gh_smem);      // [co][TLD]  B operand: rows = output channel, k = table row
  __half* Tl = Th + a.co * TLD;
  float* s_al = reinterpret_cast<float*>(Tl + a.co * TLD);     // per channel: t = y * al + be
  float* s_be = s_al + a.co;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3, lm = lane >> 3, lr = lane & 7;
  const int f = blockIdx.y;
  const int px_lo = blockIdx.x * a.px_per_cta, px_hi = min(a.P, px_lo + a.px_per_cta);
  const int co = a.co;

  {
    const float* T = a.T + (size_t)f * 32 * a.ldbT;
    for (int i = tid; i < 32 * co; i += NTH) {
      const int k = i / co, c = i - k * co;
      split_f16_trunc(T[(size_t)k * a.ldbT + c], Th[c * TLD + k], Tl[c * TLD + k]);
    }
    const int clip = a.clips > 1 ? f % a.clips : 0;
    const double* gs = a.gn_stats + 16 * clip;
    const float* film = a.film ? a.film + (size_t)clip * 2 * co : nullptr;
    for (int c = tid; c < co; c += NTH) {
      const int grp = c / a.cpg;
      const double sm = gs[2 * grp], ss = gs[2 * grp + 1];
      const double mean = sm / a.gn_count;
      const double var = ss / a.gn_count - mean * mean;
      const float rstd = (float)(1.0 / sqrt(var + 1e-5));
      float al = rstd * a.gn_w[c], be = a.gn_b[c] - (float)mean * al;
      if (film) { const float sc = film[c] + 1.f; al *= sc; be = be * sc + film[co + c]; }
      s_al[c] = al; s_be[c] = be;
    }
  }
  __syncthreads();

  for (int p0 = px_lo + warp * 16; p0 < px_hi; p0 += 16 * (NTH / 32)) {
    const size_t row0 = (size_t)f * a.P + p0 + g, row1 = row0 + 8;
    // Wt rows in A-fragment order: (row g | g+8) x (k = ks*16 + {0, 8} + 2t, 2t+1)
    uint32_t ah[2][4], al[2][4];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const float2 v0 = __ldg(reinterpret_cast<const float2*>(a.Wt + row0 * 32 + ks * 16 + 2 * t));
      const float2 v1 = __ldg(reinterpret_cast<const float2*>(a.Wt + row1 * 32 + ks * 16 + 2 * t));
      const float2 v2 = __ldg(reinterpret_cast<const float2*>(a.Wt + row0 * 32 + ks * 16 + 8 + 2 * t));
      const float2 v3 = __ldg(reinterpret_cast<const float2*>(a.Wt + row1 * 32 + ks * 16 + 8 + 2 * t));
      split_f16x2_trunc(v0.x, v0.y, ah[ks][0], al[ks][0]); split_f16x2_trunc(v1.x, v1.y, ah[ks][1], al[ks][1]);
      split_f16x2_trunc(v2.x, v2.y, ah[ks][2], al[ks][2]); split_f16x2_trunc(v3.x, v3.y, ah[ks][3], al[ks][3]);
    }
    const float* y0 = a.Y + row0 * a.ldy;
    const float* y1 = a.Y + row1 * a.ldy;
    float* o0 = a.Out + row0 * a.ldo;
    float* o1 = a.Out + row1 * a.ldo;
    for (int n0 = 0; n0 < co; n0 += 32) {
      float2 yv[4][2];
#pragma unroll
      for (int n = 0; n < 4; ++n) {                     // issue the y loads ahead of the tensor-core work
        yv[n][0] = __ldg(reinterpret_cast<const float2*>(y0 + n0 + n * 8 + 2 * t));
        yv[n][1] = __ldg(reinterpret_cast<const float2*>(y1 + n0 + n * 8 + 2 * t));
      }
      uint32_t sh[2][4], sl[2][4];                      // split-output mode: packed (c, c+1) pairs per n-block, rows g / g+8
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
          uint32_t b[4];
          ldsm4(b, ((lm & 2) ? Tl : Th) + (n0 + n * 8 + lr) * TLD + ks * 16 + (lm & 1) * 8);
          mma3(acc, ah[ks], al[ks], b);
        }
        const int c = n0 + n * 8 + 2 * t;
        const float2 al2 = *reinterpret_cast<const float2*>(s_al + c), be2 = *reinterpret_cast<const float2*>(s_be + c);
        const float t00 = yv[n][0].x * al2.x + be2.x, t01 = yv[n][0].y * al2.y + be2.y;
        const float t10 = yv[n][1].x * al2.x + be2.x, t11 = yv[n][1].y * al2.y + be2.y;
        const float r00 = silu(t00) + acc[0], r01 = silu(t01) + acc[1], r10 = silu(t10) + acc[2], r11 = silu(t11) + acc[3];
        if (!SPLIT) {
          *reinterpret_cast<float2*>(o0 + c) = make_float2(r00, r01);
          *reinterpret_cast<float2*>(o1 + c) = make_float2(r10, r11);
        } else {                                         // the wgmma GEMM reads these planes in place of its producers' split
          split_f16x2_rn(r00, r01, sh[0][n], sl[0][n]);
          split_f16x2_rn(r10, r11, sh[1][n], sl[1][n]);
        }
      }
      if (SPLIT) {
        // 4 x 4 transpose inside the quad (lane t holds the column pairs 2t, 2t+1 of the four 8-column blocks; afterwards it holds the
        // whole block t): every lane then writes 16 contiguous bytes per row and plane, a full 64-byte run per quad
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          quad_transpose(sh[r], t);
          quad_transpose(sl[r], t);
          const size_t row = (r ? row1 : row0);
          const size_t off = row * (size_t)co + n0 + 8 * t;
          *reinterpret_cast<uint4*>(a.Out16h + off) = make_uint4(sh[r][0], sh[r][1], sh[r][2], sh[r][3]);
          *reinterpret_cast<uint4*>(a.Out16l + off) = make_uint4(sl[r][0], sl[r][1], sl[r][2], sl[r][3]);
        }
      }
    }
  }
}

}  // namespace

bool gn_hcond_supported(int co, int P) { return co % 32 == 0 && co <= 512 && P % 16 == 0; }

int launch_gn_hcond(const GnHcondArgs& a_in, cudaStream_t st) {
  GnHcondArgs a = a_in;
  if (!gn_hcond_supported(a.co, a.P)) { set_last_error("gn_hcond: unsupported shape"); return -1; }
  const size_t smem = (size_t)2 * a.co * 40 * 2 + (size_t)2 * a.co * 4;
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    DAWN_CUDA_OK(cudaFuncSetAttribute(gn_hcond_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DAWN_CUDA_OK(cudaFuncSetAttribute(gn_hcond_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  int px = 512;
  while (px > 128 && a.F * ((a.P + px - 1) / px) < 2 * 148) px >>= 1;     // enough CTAs to fill the SMs on the small levels
  a.px_per_cta = px;
  if (a.Out16h != nullptr) gn_hcond_kernel<true><<<dim3((a.P + px - 1) / px, a.F), NTH, smem, st>>>(a);
  else gn_hcond_kernel<false><<<dim3((a.P + px - 1) / px, a.F), NTH, smem, st>>>(a);
  DAWN_LAUNCH_OK();
  return 0;
}

bool ca_fused_supported(int ci, int P) { return (ci == 64 || ci == 128) && P % 16 == 0 && P >= CHUNK; }

int launch_ca_fused(const CaFusedArgs& a, int ci, cudaStream_t st) {
  if (!ca_fused_supported(ci, a.P)) { set_last_error("ca_fused: unsupported shape"); return -1; }
  return ci == 64 ? launch_ci<64>(a, st) : launch_ci<128>(a, st);
}

// wq: [ci][192] folded projection (k-major, as the GEMM path packs it) -> [hi|lo][192][ci] fp16 with a power-of-two pre-scale
void ca_fused_pack(const float* wq, int ci, std::vector<uint16_t>& W, float* inv_wscale) {
  float mx = 0.f;
  for (size_t i = 0; i < (size_t)ci * 192; ++i) mx = std::max(mx, std::fabs(wq[i]));
  const float sc = f16_prescale(mx);
  *inv_wscale = 1.0f / sc;
  W.assign((size_t)2 * 192 * ci, 0);
  for (int n = 0; n < 192; ++n)
    for (int k = 0; k < ci; ++k) split_f16_host(wq[(size_t)k * 192 + n] * sc, W[(size_t)n * ci + k], W[((size_t)192 + n) * ci + k]);
}

}  // namespace dawn
