// Tensor-core softmax attention for the DAWN UNet (temporal band attention U:697-725 == LA:71-99, and the mid
// block's full spatial attention U:841-843): FlashAttention-2 style, warp-level mma.sync m16n8k16 with the same
// 3-term split as the contraction kernels (fp16 hi/lo pieces, fp32 accumulate) so that scores and outputs keep
// fp32-level parity.
//   CTA = (sequence, head, span of 128 queries); 8 warps, each owns one 16-query block.
//   Keys/values of the span (banded: 128 + 2*band <= 208 keys; full: streamed in chunks of 192) are split once into
//   fp16 hi/lo in shared memory: K row-major [key][d], V transposed [d][key] (B-operand layouts, padded against bank
//   conflicts).  S = Q K^T per 32-key block -> + bias, band mask -> online softmax (fp32) -> P (accumulator layout
//   == A-operand layout of the next MMA) -> O = O*corr + P V.
#include "common.cuh"
#include "f16x3.cuh"
#include "kernels.cuh"

namespace dawn {
namespace {

constexpr int QSPAN = 128;            // queries per CTA
constexpr int KCAP = 208;             // key rows a banded span needs (128 + 2*40)
constexpr int KROWS = 224;            // rows staged (7 blocks of 32; rows past the chunk are zero-filled so masked lanes multiply 0 x 0)
constexpr int KFULL = 192;            // chunk length in full-attention mode
constexpr int K_LD = 40;              // halfs per K row (32 + 8 pad): conflict-free B-fragment reads
constexpr int V_LD = KROWS + 8;       // halfs per V^T row: (V_LD/2) mod 32 == 20 -> conflict-free

constexpr int ATHREADS = 256;

__global__ void __launch_bounds__(ATHREADS) attention_tc_kernel(AttnArgs a) {
  extern __shared__ __align__(16) unsigned char att_smem[];
  __half* sKh = reinterpret_cast<__half*>(att_smem);
  __half* sKl = sKh + KROWS * K_LD;
  __half* sVh = sKl + KROWS * K_LD;
  __half* sVl = sVh + 32 * V_LD;
  float* s_bias = reinterpret_cast<float*>(sVl + 32 * V_LD);

  // heads are the fastest grid dimension: the 8 CTAs of one pixel run together and sweep whole 3 KB q|k|v rows
  // (one 128-byte line per row per CTA otherwise -> one DRAM row activation per line)
  const int head = blockIdx.x, seq = blockIdx.y;
  const int q0 = a.q_lo + blockIdx.z * QSPAN;
  const int q1 = min(q0 + QSPAN, a.q_hi);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const long long base = attn_seq_base(a, seq);
  const long long estride = attn_elem_stride(a);
  const int band = a.band;
  const bool banded = band < a.L;

  if (a.bias != nullptr) {
    for (int i = tid; i < 2 * band + 1 && i < 256; i += ATHREADS) s_bias[i] = a.bias[head * (2 * band + 1) + i];
  }

  // this warp's query block(s): qb = warp + 8 b (16 queries each)
  constexpr int NQB = QSPAN / 16 / (ATHREADS / 32);    // 1 per warp
  uint32_t qh[NQB][2][4], ql[NQB][2][4];
  float o[NQB][4][4], mrow[NQB][2], lrow[NQB][2];
#pragma unroll
  for (int b = 0; b < NQB; ++b) {
    const int i0 = q0 + (warp + (ATHREADS / 32) * b) * 16;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        // a0: (row g, cols 2t..), a1: (row g+8), a2: (row g, cols 2t+8..), a3: (row g+8, cols 2t+8..)
        const int row = i0 + g + ((r & 1) ? 8 : 0);
        const int col = ks * 16 + 2 * t + ((r & 2) ? 8 : 0);
        float2 v = make_float2(0.f, 0.f);
        if (row < q1)
          v = *reinterpret_cast<const float2*>(a.qkv + (size_t)(base + (long long)row * estride) * a.ld + head * 32 + col);
        split_f16x2_rn(v.x, v.y, qh[b][ks][r], ql[b][ks][r]);
      }
    }
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int c = 0; c < 4; ++c) o[b][n][c] = 0.f;
    mrow[b][0] = mrow[b][1] = -1e30f;
    lrow[b][0] = lrow[b][1] = 0.f;
  }

  // key range of this CTA
  const int klo_all = banded ? (q0 - band) : 0;                    // may be negative (rows zero-filled)
  const int khi_all = banded ? (q0 + QSPAN + band) : a.L;
  const int kstep = banded ? KCAP : KFULL;

  for (int kc0 = klo_all; kc0 < khi_all; kc0 += kstep) {
    const int nk = min(kstep, khi_all - kc0);                      // key rows of this chunk (multiple of 16 when banded)
    __syncthreads();
    // ---- stage K (row-major) and V (transposed), split into fp16 hi/lo; global loads issued in batches of 7
    constexpr int ITEMS = KROWS * 16, BATCH = 14;      // every load of the chunk in flight at once (ncu: staging was latency-bound)
    static_assert(ITEMS % (ATHREADS * BATCH) == 0, "staging loop assumes full batches");
    for (int it0 = 0; it0 < ITEMS; it0 += ATHREADS * BATCH) {
      float4 vb[BATCH];
#pragma unroll
      for (int u = 0; u < BATCH; ++u) {
        const int idx = it0 + u * ATHREADS + tid;
        const int r = idx >> 4, c = idx & 15;                      // c < 8: K float4 #c, else V float4 #(c-8)
        const int key = kc0 + r;
        vb[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < nk && key >= 0 && key < a.L)
          vb[u] = __ldg(reinterpret_cast<const float4*>(a.qkv + (size_t)(base + (long long)key * estride) * a.ld + 256 + (c >> 3) * 256 +
                                                        head * 32 + (c & 7) * 4));
      }
#pragma unroll
      for (int u = 0; u < BATCH; ++u) {
        const int idx = it0 + u * ATHREADS + tid;
        const int r = idx >> 4, c = idx & 15;
        const float4 v = vb[u];
        if (c < 8) {
          uint32_t h0, l0, h1, l1;
          split_f16x2_rn(v.x, v.y, h0, l0); split_f16x2_rn(v.z, v.w, h1, l1);
          *reinterpret_cast<uint2*>(&sKh[r * K_LD + c * 4]) = make_uint2(h0, h1);
          *reinterpret_cast<uint2*>(&sKl[r * K_LD + c * 4]) = make_uint2(l0, l1);
        } else {
          const int d = (c - 8) * 4;
          const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            __half hh, ll;
            split_f16_rn(vv[i], hh, ll);
            sVh[(d + i) * V_LD + r] = hh;
            sVl[(d + i) * V_LD + r] = ll;
          }
        }
      }
    }
    __syncthreads();

#pragma unroll
    for (int b = 0; b < NQB; ++b) {
      const int i0 = q0 + (warp + (ATHREADS / 32) * b) * 16;
      if (i0 >= q1) continue;
      // 32-key blocks this query block needs inside the chunk.  Banded: its 16 queries see keys [i0-band, i0+15+band],
      // i.e. chunk rows [i0-q0, i0-q0+16+2*band): start exactly there (rows need no alignment) -> 3 blocks instead of 4.
      int kr_lo = 0, kr_hi = nk;
      if (banded) { kr_lo = i0 - q0; kr_hi = min(nk, i0 - q0 + 16 + 2 * band); }
      for (int kr0 = kr_lo; kr0 < kr_hi; kr0 += 32) {
        // ---------------- S = Q K^T  (4 n-tiles of 8 keys, k = 32 dims in 2 steps, 3-term split)
        float s[4][4];
#pragma unroll
        for (int n = 0; n < 4; ++n) {
#pragma unroll
          for (int c = 0; c < 4; ++c) s[n][c] = 0.f;
          const int krow = kr0 + n * 8 + g;
#pragma unroll
          for (int ks = 0; ks < 2; ++ks) {
            const int off = krow * K_LD + ks * 16 + 2 * t;
            const uint32_t bk[4] = {*reinterpret_cast<const uint32_t*>(&sKh[off]), *reinterpret_cast<const uint32_t*>(&sKh[off + 8]),
                                    *reinterpret_cast<const uint32_t*>(&sKl[off]), *reinterpret_cast<const uint32_t*>(&sKl[off + 8])};
            mma3(s[n], qh[b][ks], ql[b][ks], bk);
          }
        }
        // ---------------- bias, mask, online softmax (rows g and g+8 of the block)
        float mnew[2] = {mrow[b][0], mrow[b][1]};
        bool ok[4][4];
#pragma unroll
        for (int n = 0; n < 4; ++n)
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int i = i0 + g + ((c & 2) ? 8 : 0);
            const int j = kc0 + kr0 + n * 8 + 2 * t + (c & 1);
            const int rel = j - i;
            // banded: |rel| <= band already implies the row lies inside the staged chunk
            const bool v = banded ? ((unsigned)(rel + band) <= (unsigned)(2 * band)) && ((unsigned)j < (unsigned)a.L)
                                  : ((j < a.L) && (kr0 + n * 8 + 2 * t + (c & 1) < nk));
            ok[n][c] = v;
            if (v) {
              if (a.bias != nullptr) s[n][c] += s_bias[rel + band];
              mnew[c >> 1] = fmaxf(mnew[c >> 1], s[n][c]);
            }
          }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          mnew[r] = fmaxf(mnew[r], __shfl_xor_sync(0xffffffffu, mnew[r], 1));
          mnew[r] = fmaxf(mnew[r], __shfl_xor_sync(0xffffffffu, mnew[r], 2));
        }
        const float corr0 = __expf(mrow[b][0] - mnew[0]), corr1 = __expf(mrow[b][1] - mnew[1]);
        mrow[b][0] = mnew[0]; mrow[b][1] = mnew[1];
        float psum0 = 0.f, psum1 = 0.f;
#pragma unroll
        for (int n = 0; n < 4; ++n)
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float pv = ok[n][c] ? __expf(s[n][c] - mnew[c >> 1]) : 0.f;
            s[n][c] = pv;
            if (c & 2) psum1 += pv; else psum0 += pv;
          }
        lrow[b][0] = lrow[b][0] * corr0 + psum0;                   // per-thread partial sums; quad-reduced at the end
        lrow[b][1] = lrow[b][1] * corr1 + psum1;
        // ---------------- O = O*corr + P V   (P: accumulator layout of two n-tiles == A fragment of one k16 step)
        uint32_t ph[2][4], pl[2][4];
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
          split_f16x2_rn(s[2 * ks][0], s[2 * ks][1], ph[ks][0], pl[ks][0]);
          split_f16x2_rn(s[2 * ks][2], s[2 * ks][3], ph[ks][1], pl[ks][1]);
          split_f16x2_rn(s[2 * ks + 1][0], s[2 * ks + 1][1], ph[ks][2], pl[ks][2]);
          split_f16x2_rn(s[2 * ks + 1][2], s[2 * ks + 1][3], ph[ks][3], pl[ks][3]);
        }
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          float acc[4] = {0.f, 0.f, 0.f, 0.f};
          const int drow = (n * 8 + g) * V_LD;
#pragma unroll
          for (int ks = 0; ks < 2; ++ks) {
            const int off = drow + kr0 + ks * 16 + 2 * t;
            const uint32_t bv[4] = {*reinterpret_cast<const uint32_t*>(&sVh[off]), *reinterpret_cast<const uint32_t*>(&sVh[off + 8]),
                                    *reinterpret_cast<const uint32_t*>(&sVl[off]), *reinterpret_cast<const uint32_t*>(&sVl[off + 8])};
            mma3(acc, ph[ks], pl[ks], bv);
          }
          o[b][n][0] = o[b][n][0] * corr0 + acc[0];
          o[b][n][1] = o[b][n][1] * corr0 + acc[1];
          o[b][n][2] = o[b][n][2] * corr1 + acc[2];
          o[b][n][3] = o[b][n][3] * corr1 + acc[3];
        }
      }
    }
  }

  // ---- normalise and store
#pragma unroll
  for (int b = 0; b < NQB; ++b) {
    const int i0 = q0 + (warp + (ATHREADS / 32) * b) * 16;
    float l0 = lrow[b][0], l1 = lrow[b][1];
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    const int r0 = i0 + g, r1 = i0 + g + 8;
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      const int col = head * 32 + n * 8 + 2 * t;
      if (r0 < q1)
        *reinterpret_cast<float2*>(a.out + (size_t)(base + (long long)r0 * estride) * a.ldo + col) =
            make_float2(o[b][n][0] * inv0, o[b][n][1] * inv0);
      if (r1 < q1)
        *reinterpret_cast<float2*>(a.out + (size_t)(base + (long long)r1 * estride) * a.ldo + col) =
            make_float2(o[b][n][2] * inv1, o[b][n][3] * inv1);
    }
  }
}

}  // namespace

bool attention_tc_supported(const AttnArgs& a) {
  if (a.band < a.L && a.band > 40) return false;       // shared-memory key window sized for band <= 40
  if ((a.ld & 3) || (a.ldo & 1)) return false;
  return true;
}

int launch_attention_tc(const AttnArgs& a, cudaStream_t st) {
  if (a.q_hi <= a.q_lo || a.nseq <= 0) return 0;
  constexpr int SMEM = (2 * KROWS * K_LD + 2 * 32 * V_LD) * 2 + 256 * 4;
  static bool attr = false;
  if (!attr) {
    DAWN_CUDA_OK(cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr = true;
  }
  dim3 grid(8, a.nseq, (a.q_hi - a.q_lo + QSPAN - 1) / QSPAN);
  attention_tc_kernel<<<grid, ATHREADS, SMEM, st>>>(a);
  DAWN_LAUNCH_OK();
  return 0;
}

}  // namespace dawn
