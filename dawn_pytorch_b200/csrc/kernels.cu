// Non-GEMM kernels of the DAWN denoising UNet: norms, conditioning tables, attention cores, layout.
#include <algorithm>
#include "common.cuh"
#include "f16x3.cuh"
#include "kernels.cuh"

namespace dawn {

// =========================================================================== row LayerNorm statistics
// one warp per pixel row; C <= 128 * NV (NV float4 per lane), C % 4 == 0.  biased variance, two-pass from registers
// (U:186-188, 201-203).  NV = 16 serves the 2048-channel inputs of the first up block below a 1024-channel level.
template <int NV>
__global__ void rowstats_kernel(const float* __restrict__ x, int ld, int C, int M, float eps,
                                float* __restrict__ out) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * ld);
  const int nvec = C >> 2;
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i = lane + 32 * k;
    v[k] = (i < nvec) ? xr[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
  }
  const float mu = warp_sum(s) / (float)C;
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i = lane + 32 * k;
    if (i < nvec) {
      const float a = v[k].x - mu, b = v[k].y - mu, c = v[k].z - mu, d = v[k].w - mu;
      ss += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float var = warp_sum(ss) / (float)C;
  if (lane == 0) {
    out[2 * (size_t)row] = mu;
    out[2 * (size_t)row + 1] = 1.0f / sqrtf(var + eps);
  }
}

int launch_rowstats(const float* x, int ld, int C, int M, float eps, float* out, cudaStream_t st) {
  if (C > 2048 || (C & 3) || (ld & 3)) { set_last_error("rowstats: C must be <= 2048 and a multiple of 4"); return -1; }
  const int wpb = 8;
  if (C <= 1024) rowstats_kernel<8><<<(M + wpb - 1) / wpb, wpb * 32, 0, st>>>(x, ld, C, M, eps, out);
  else rowstats_kernel<16><<<(M + wpb - 1) / wpb, wpb * 32, 0, st>>>(x, ld, C, M, eps, out);
  DAWN_LAUNCH_OK();
  return 0;
}

// =========================================================================== GroupNorm apply (elementwise)
__global__ void gn_apply_kernel(const float* __restrict__ Y, int ldy, int C, long long nvec_total,
                                const double* __restrict__ stats, double count, int cpg, int P, int clips,
                                const float* __restrict__ gw, const float* __restrict__ gb,
                                const float* __restrict__ film, const float* Res, int ldr,
                                float* Out, int ldo) {
  __shared__ float s_gn[16 * kMaxClips];
  if (threadIdx.x < 8 * clips) {                 // (mean, rstd) of every clip's 8 groups
    const double s = stats[2 * threadIdx.x], ss = stats[2 * threadIdx.x + 1];
    const double mean = s / count;
    const double var = ss / count - mean * mean;
    s_gn[2 * threadIdx.x] = (float)mean;
    s_gn[2 * threadIdx.x + 1] = (float)(1.0 / sqrt(var + 1e-5));
  }
  __syncthreads();
  const int vpr = C >> 2;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < nvec_total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / vpr;
    const int c = (int)(idx - row * vpr) * 4;
    const int clip = clips > 1 ? (int)((row / P) % clips) : 0;
    const float4 y = *reinterpret_cast<const float4*>(Y + row * ldy + c);
    const int grp = c / cpg;
    const float mean = s_gn[16 * clip + 2 * grp], rstd = s_gn[16 * clip + 2 * grp + 1];
    const float4 w = *reinterpret_cast<const float4*>(gw + c);
    const float4 b = *reinterpret_cast<const float4*>(gb + c);
    float t0 = (y.x - mean) * rstd * w.x + b.x;
    float t1 = (y.y - mean) * rstd * w.y + b.y;
    float t2 = (y.z - mean) * rstd * w.z + b.z;
    float t3 = (y.w - mean) * rstd * w.w + b.w;
    if (film) {
      const float* fc = film + (size_t)clip * 2 * C;
      const float4 sc = *reinterpret_cast<const float4*>(fc + c);
      const float4 sh = *reinterpret_cast<const float4*>(fc + C + c);
      t0 = t0 * (sc.x + 1.f) + sh.x; t1 = t1 * (sc.y + 1.f) + sh.y;
      t2 = t2 * (sc.z + 1.f) + sh.z; t3 = t3 * (sc.w + 1.f) + sh.w;
    }
    float4 o = make_float4(silu(t0), silu(t1), silu(t2), silu(t3));
    if (Res) {
      const float4 r = *reinterpret_cast<const float4*>(Res + row * ldr + c);
      o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
    }
    *reinterpret_cast<float4*>(Out + row * ldo + c) = o;
  }
}

int launch_gn_apply(const float* Y, int ldy, int C, int M, const double* stats, double count, int cpg, int P, int clips,
                    const float* gw, const float* gb, const float* film, const float* Res, int ldr,
                    float* Out, int ldo, cudaStream_t st) {
  if (clips < 1 || clips > kMaxClips || P < 1) { set_last_error("gn_apply: bad clip geometry"); return -1; }
  const long long nvec = (long long)M * (C >> 2);
  const int threads = 256;
  long long blocks = (nvec + threads - 1) / threads;
  if (blocks > 148LL * 16) blocks = 148LL * 16;
  gn_apply_kernel<<<(int)blocks, threads, 0, st>>>(Y, ldy, C, nvec, stats, count, cpg, P, clips, gw, gb, film, Res, ldr, Out, ldo);
  DAWN_LAUNCH_OK();
  return 0;
}

// =========================================================================== small dense layers (per frame GEMV)
// out[f][j] = b[j] + sum_i W[j][i] act(x[f][off + i]), act = SiLU when ACT = 1 (cond MLPs U:371-384, 440-442; to_kv U:524).
// A block owns FL_JT*8 = 32 outputs x FL_FT = 8 frames, so every weight row is read once per 8 frames and act(x) is evaluated
// once per 32 outputs; a warp computes FL_JT outputs with lane-strided partial sums and a butterfly reduction.
constexpr int FL_FT = 8, FL_JT = 4;
// Output row i (table order: frame f of clip b is i = f * clips + b) reads input row b * (F / clips) + f (clips back to back).
template <int ACT>
__device__ __forceinline__ void frame_linear_tiled_body(const float* __restrict__ x, int ldx, int off, int K,
                                                        const float* __restrict__ W, const float* __restrict__ b, int Nout,
                                                        float* __restrict__ out, int F, int clips) {
  extern __shared__ float sx[];                 // [FL_FT][K]
  const int f0 = blockIdx.y * FL_FT;
  for (int i = threadIdx.x; i < FL_FT * K; i += blockDim.x) {
    const int ft = i / K, k = i - ft * K;
    float v = 0.f;
    if (f0 + ft < F) {
      const int ti = f0 + ft, src = (ti % clips) * (F / clips) + ti / clips;
      v = x[(size_t)src * ldx + off + k]; v = ACT ? silu(v) : v;
    }
    sx[i] = v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j0 = (blockIdx.x * (blockDim.x >> 5) + warp) * FL_JT;
  if (j0 >= Nout) return;
  float acc[FL_JT][FL_FT];
#pragma unroll
  for (int jj = 0; jj < FL_JT; ++jj)
#pragma unroll
    for (int ft = 0; ft < FL_FT; ++ft) acc[jj][ft] = 0.f;
  for (int i = lane; i < K; i += 32) {
    float wv[FL_JT];
#pragma unroll
    for (int jj = 0; jj < FL_JT; ++jj) wv[jj] = (j0 + jj < Nout) ? W[(size_t)(j0 + jj) * K + i] : 0.f;
#pragma unroll
    for (int ft = 0; ft < FL_FT; ++ft) {
      const float xv = sx[ft * K + i];
#pragma unroll
      for (int jj = 0; jj < FL_JT; ++jj) acc[jj][ft] += wv[jj] * xv;
    }
  }
#pragma unroll
  for (int jj = 0; jj < FL_JT; ++jj)
#pragma unroll
    for (int ft = 0; ft < FL_FT; ++ft) {
      const float r = warp_sum(acc[jj][ft]);
      if (lane == 0 && j0 + jj < Nout && f0 + ft < F) out[(size_t)(f0 + ft) * Nout + j0 + jj] = r + (b ? b[j0 + jj] : 0.f);
    }
}
__global__ void __launch_bounds__(256) cond_mlp_tiled_kernel(const float* __restrict__ cond, int cond_ld, const CondDesc* __restrict__ descs, int F,
                                                             int clips) {
  const CondDesc d = descs[blockIdx.z];
  if ((int)blockIdx.x * 8 * FL_JT >= d.n1) return;
  frame_linear_tiled_body<1>(cond, cond_ld, d.off, d.K, d.mW, d.mB, d.n1, d.ctx, F, clips);
}
__global__ void __launch_bounds__(256) cond_kv_tiled_kernel(const CondDesc* __restrict__ descs, int F) {
  const CondDesc d = descs[blockIdx.z];
  frame_linear_tiled_body<0>(d.ctx, d.n1, 0, d.n1, d.Wkv, nullptr, 128, d.kv, F, 1);
}

// =========================================================================== cross-attention per-frame tables
// With exactly two keys (null, real) per query the attention output of head h is
//   o_h = nv + w_h (v_h - nv),  so  to_out(o) = u_0 + sum_h w_h u_h  with per-frame vectors
//   u_0 = Wout * rep(nv),  u_h = Wout[:, h] (v_h - nv)   (U:530-559).
// The output LayerNorm (U:511-514) of that combination needs only the centred vectors and their Gram matrix.
__device__ __forceinline__ void ca_tables_body(const CaTableArgs& a, int f) {
  extern __shared__ float sm[];
  float* u = sm;                       // [9][co]
  __shared__ float s_kv[128];
  __shared__ float s_red[9];
  __shared__ float s_nk[8], s_nv[8];
  const int tid = threadIdx.x;
  const int co = a.co;
  if (tid < 128) s_kv[tid] = a.kv[(size_t)f * 128 + tid];
  if (tid < 8) { s_nk[tid] = a.nkv[tid]; s_nv[tid] = a.nkv[8 + tid]; }
  __syncthreads();
  // normalised keys folded with q_scale * k_scale  (U:537-539)
  if (tid < 64) {
    const int h = tid >> 3, d = tid & 7;
    float n2 = 0.f;
    for (int e = 0; e < 8; ++e) n2 += s_kv[h * 8 + e] * s_kv[h * 8 + e];
    const float inv = 1.0f / fmaxf(sqrtf(n2), 1e-12f);
    a.kq[((size_t)f * 3 + a.ca) * 64 + tid] = s_kv[tid] * inv * a.ks[d] * a.qs[d];
  }
  if (f == 0 && tid < 8) {
    float n2 = 0.f;
    for (int e = 0; e < 8; ++e) n2 += s_nk[e] * s_nk[e];
    const float inv = 1.0f / fmaxf(sqrtf(n2), 1e-12f);
    a.nkq[a.ca * 8 + tid] = s_nk[tid] * inv * a.ks[tid] * a.qs[tid];
  }
  // u vectors: a thread owns output channel c, reads its 64-float Wout row once (16 x LDG.128) and forms all nine
  // combinations from registers
  for (int c = tid; c < co; c += blockDim.x) {
    float w[64];
    const float4* wr = reinterpret_cast<const float4*>(a.Wout + (size_t)c * 64);
#pragma unroll
    for (int i = 0; i < 16; ++i) { const float4 t = __ldg(wr + i); w[4 * i] = t.x; w[4 * i + 1] = t.y; w[4 * i + 2] = t.z; w[4 * i + 3] = t.w; }
    float acc0 = 0.f;
#pragma unroll
    for (int h = 0; h < 8; ++h)
#pragma unroll
      for (int d = 0; d < 8; ++d) acc0 += w[h * 8 + d] * s_nv[d];
    u[c] = acc0;
#pragma unroll
    for (int h = 0; h < 8; ++h) {
      float acc = 0.f;
#pragma unroll
      for (int d = 0; d < 8; ++d) acc += w[h * 8 + d] * (s_kv[64 + h * 8 + d] - s_nv[d]);
      u[(h + 1) * co + c] = acc;
    }
  }
  __syncthreads();
  // centre each vector over channels
  const int warp = tid >> 5, lane = tid & 31, nwarp = blockDim.x >> 5;
  for (int r = warp; r < 9; r += nwarp) {
    float s = 0.f;
    for (int c = lane; c < co; c += 32) s += u[r * co + c];
    s = warp_sum(s);
    if (lane == 0) s_red[r] = s / (float)co;
  }
  __syncthreads();
  for (int idx = tid; idx < 9 * co; idx += blockDim.x) u[idx] -= s_red[idx / co];
  __syncthreads();
  // Gram matrix (1/co) <u_a, u_b>
  for (int pr = warp; pr < 81; pr += nwarp) {
    const int ra = pr / 9, rb = pr - ra * 9;
    float s = 0.f;
    for (int c = lane; c < co; c += 32) s += u[ra * co + c] * u[rb * co + c];
    s = warp_sum(s);
    if (lane == 0) a.G[((size_t)f * 3 + a.ca) * 81 + pr] = s / (float)co;
  }
  // gain-folded table rows
  float* T = a.T + (size_t)f * 32 * a.ldbT + (size_t)(a.ca * 9) * a.ldbT;
  for (int idx = tid; idx < 9 * co; idx += blockDim.x) {
    const int r = idx / co, c = idx - r * co;
    T[(size_t)r * a.ldbT + c] = u[idx] * a.gout[c];
  }
}

// grid (F, descriptors): one block per (frame, conditioned block x cross-attention)
__global__ void __launch_bounds__(256) ca_tables_batched_kernel(const CondDesc* __restrict__ descs) { ca_tables_body(descs[blockIdx.y].t, blockIdx.x); }

int launch_cond_batched(const float* cond, int cond_ld, const CondDesc* descs_dev, int ndesc, int max_n1, int max_k, int max_co, int F,
                        int clips, cudaStream_t st) {
  if (clips < 1 || F % clips != 0) { set_last_error("cond tables: frames must be a multiple of the clip count"); return -1; }
  const size_t sm1 = (size_t)FL_FT * max_k * sizeof(float), sm2 = (size_t)FL_FT * max_n1 * sizeof(float);
  const size_t smem_t = (size_t)9 * max_co * sizeof(float);
  static size_t attr = 0;
  if (std::max({sm1, sm2, smem_t}) > 48 * 1024 && std::max({sm1, sm2, smem_t}) > attr) {
    attr = std::max({sm1, sm2, smem_t});
    DAWN_CUDA_OK(cudaFuncSetAttribute(cond_mlp_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attr));
    DAWN_CUDA_OK(cudaFuncSetAttribute(cond_kv_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attr));
    DAWN_CUDA_OK(cudaFuncSetAttribute(ca_tables_batched_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attr));
  }
  const int ft = (F + FL_FT - 1) / FL_FT, jb = 8 * FL_JT;
  cond_mlp_tiled_kernel<<<dim3((max_n1 + jb - 1) / jb, ft, ndesc), 256, sm1, st>>>(cond, cond_ld, descs_dev, F, clips);
  DAWN_LAUNCH_OK();
  cond_kv_tiled_kernel<<<dim3((128 + jb - 1) / jb, ft, ndesc), 256, sm2, st>>>(descs_dev, F);
  DAWN_LAUNCH_OK();
  ca_tables_batched_kernel<<<dim3(F, ndesc), 256, smem_t, st>>>(descs_dev);
  DAWN_LAUNCH_OK();
  return 0;
}

// one thread per (token, ca): rstd of the LayerNorm'd to_out output from the Gram quadratic form
__global__ void ca_rstd_kernel(const float* __restrict__ gates, const float* __restrict__ G, int M, int P,
                               float* __restrict__ Wt) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)M * 4) return;
  const int m = (int)(idx >> 2), ca = (int)(idx & 3);
  float* wt = Wt + (size_t)m * 32;
  if (ca == 3) {
#pragma unroll
    for (int k = 27; k < 32; ++k) wt[k] = 0.f;
    return;
  }
  const int f = m / P;
  const float* g = G + ((size_t)f * 3 + ca) * 81;
  float c[9];
  c[0] = 1.f;
#pragma unroll
  for (int h = 0; h < 8; ++h) c[h + 1] = gates[(size_t)m * 24 + ca * 8 + h];
  float var = 0.f;
#pragma unroll
  for (int a = 0; a < 9; ++a) {
    float row = 0.f;
#pragma unroll
    for (int b = 0; b < 9; ++b) row += g[a * 9 + b] * c[b];
    var += c[a] * row;
  }
  const float rs = rsqrtf(fmaxf(var, 0.f) + 1e-5f);
#pragma unroll
  for (int a = 0; a < 9; ++a) wt[ca * 9 + a] = rs * c[a];
}

int launch_ca_rstd(const float* gates, const float* G, int M, int P, float* Wt, cudaStream_t st) {
  const long long n = (long long)M * 4;
  ca_rstd_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(gates, G, M, P, Wt);
  DAWN_LAUNCH_OK();
  return 0;
}

// =========================================================================== fp16 hi | lo copy of an activation
// x (M rows, C channels, row stride ld) -> dense hi[M][C], lo[M][C]: the round-to-nearest split the wgmma GEMM producers apply on the fly
__global__ void split_rows_kernel(const float* __restrict__ x, int ld, int C, long long M, uint2* __restrict__ hi,
                                  uint2* __restrict__ lo) {
  const int c4n = C >> 2;
  const long long total = M * c4n;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / c4n;
    const int c4 = (int)(idx - row * c4n);
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + (size_t)row * ld) + c4);
    uint32_t h0, l0, h1, l1;
    split_f16x2_rn(v.x, v.y, h0, l0);
    split_f16x2_rn(v.z, v.w, h1, l1);
    hi[idx] = make_uint2(h0, h1);
    lo[idx] = make_uint2(l0, l1);
  }
}
int launch_split_rows(const float* x, int ld, int C, long long M, void* hi, void* lo, cudaStream_t st) {
  const long long total = M * (C >> 2);
  const int blocks = (int)std::min<long long>((total + 255) / 256, 148LL * 16);
  split_rows_kernel<<<blocks, 256, 0, st>>>(x, ld, C, M, (uint2*)hi, (uint2*)lo);
  DAWN_LAUNCH_OK();
  return 0;
}

// =========================================================================== one-pixel border of the upconv input
// x (frames, H, W, C) rows of stride ld -> dense out (frames, H + 2, W + 2, C): the interior is x, border row / column -1 and H / W
// read x at the clamped (wrap = 0) or wrapped (wrap = 1) index
__global__ void pad_border_kernel(const float* __restrict__ x, int ld, int C, int frames, int H, int W, int wrap,
                                  float4* __restrict__ out) {
  const int c4n = C >> 2, PW = W + 2, PH = H + 2;
  const long long total = (long long)frames * PH * PW * c4n;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx / c4n;
    const int c4 = (int)(idx - r * c4n);
    const int px = (int)(r % PW) - 1; r /= PW;
    const int py = (int)(r % PH) - 1;
    const long long f = r / PH;
    const int sy = wrap ? (py + H) % H : min(max(py, 0), H - 1);
    const int sx = wrap ? (px + W) % W : min(max(px, 0), W - 1);
    out[idx] = __ldg(reinterpret_cast<const float4*>(x + ((size_t)(f * H + sy) * W + sx) * ld) + c4);
  }
}
int launch_pad_border(const float* x, int ld, int C, int frames, int H, int W, int wrap, float* out, cudaStream_t st) {
  DAWN_CHECK(C % 4 == 0 && ld % 4 == 0, "launch_pad_border: channels and row stride must be multiples of 4");
  const long long total = (long long)frames * (H + 2) * (W + 2) * (C >> 2);
  const int blocks = (int)std::min<long long>((total + 255) / 256, 148LL * 16);
  pad_border_kernel<<<blocks, 256, 0, st>>>(x, ld, C, frames, H, W, wrap, reinterpret_cast<float4*>(out));
  DAWN_LAUNCH_OK();
  return 0;
}

// =========================================================================== time embedding
__global__ void time_mlp_kernel(const int64_t* __restrict__ t, const float* __restrict__ freqs, int dim,
                                const float* __restrict__ W1, const float* __restrict__ b1,
                                const float* __restrict__ W2, const float* __restrict__ b2,
                                float* __restrict__ t_silu, int t_stride) {
  extern __shared__ float sm[];
  float* emb = sm;             // [dim]
  float* hid = sm + dim;       // [4 dim]
  const int tdim = 4 * dim, half = dim / 2;
  const float tv = (float)t[(size_t)blockIdx.x * t_stride];     // block = clip
  t_silu += (size_t)blockIdx.x * tdim;
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    const float a = tv * freqs[i];
    emb[i] = sinf(a);
    emb[half + i] = cosf(a);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < tdim; j += blockDim.x) {
    float acc = b1[j];
    for (int i = 0; i < dim; ++i) acc += W1[(size_t)j * dim + i] * emb[i];
    hid[j] = 0.5f * acc * (1.0f + erff(acc * 0.70710678118654752440f));     // exact GELU (U:792)
  }
  __syncthreads();
  for (int j = threadIdx.x; j < tdim; j += blockDim.x) {
    float acc = b2[j];
    for (int i = 0; i < tdim; ++i) acc += W2[(size_t)j * tdim + i] * hid[i];
    t_silu[j] = silu(acc);                                                  // every consumer applies SiLU first (U:366-369)
  }
}

int launch_time_mlp(const int64_t* t_dev, int t_stride, int clips, const float* freqs, int dim, const float* W1, const float* b1,
                    const float* W2, const float* b2, float* t_silu, cudaStream_t st) {
  time_mlp_kernel<<<clips, 256, 5 * dim * sizeof(float), st>>>(t_dev, freqs, dim, W1, b1, W2, b2, t_silu, t_stride);
  DAWN_LAUNCH_OK();
  return 0;
}

__global__ void film_kernel(const FilmDesc* __restrict__ descs, const float* __restrict__ t_silu, int tdim) {
  const FilmDesc d = descs[blockIdx.y];
  const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31, clip = blockIdx.z;
  if (j >= d.n) return;
  t_silu += (size_t)clip * tdim;
  float acc = 0.f;
  for (int i = lane; i < tdim; i += 32) acc += d.W[(size_t)j * tdim + i] * t_silu[i];
  acc = warp_sum(acc);
  if (lane == 0) d.out[(size_t)clip * d.n + j] = acc + d.b[j];
}

// max_n: the largest descriptor n (2 x the widest conditioned block's channels); one warp per output
int launch_film(const FilmDesc* descs_dev, int ndesc, int max_n, int clips, const float* t_silu, int tdim, cudaStream_t st) {
  dim3 grid((max_n + 7) / 8, ndesc, clips);
  film_kernel<<<grid, 256, 0, st>>>(descs_dev, t_silu, tdim);
  DAWN_LAUNCH_OK();
  return 0;
}

__global__ void rotary_table_kernel(const float* __restrict__ freqs, int F, int pos0, float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= F * 16) return;
  const int f = idx >> 4, i = idx & 15;
  const float a = (float)(pos0 + f) * freqs[i];
  out[2 * idx] = cosf(a);
  out[2 * idx + 1] = sinf(a);
}
int launch_rotary_table(const float* freqs, int F, int pos0, float* out, cudaStream_t st) {
  rotary_table_kernel<<<(F * 16 + 255) / 256, 256, 0, st>>>(freqs, F, pos0, out);
  DAWN_LAUNCH_OK();
  return 0;
}

// =========================================================================== attention core
// grid (nseq, 8 heads, query blocks of 128); 4 warps, lane = query, keys broadcast from shared memory.
constexpr int ATT_QB = 128;
constexpr int ATT_KC = 128;

__global__ void __launch_bounds__(128) attention_kernel(AttnArgs a) {
  __shared__ __align__(16) float Ks[ATT_KC][32];
  __shared__ __align__(16) float Vs[ATT_KC][32];
  const int seq = blockIdx.x, head = blockIdx.y;
  const int q0 = a.q_lo + blockIdx.z * ATT_QB;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int iq = q0 + warp * 32 + lane;
  const bool qv = iq < a.q_hi;
  const long long base = attn_seq_base(a, seq);
  const long long estride = attn_elem_stride(a);
  const int band = a.band;
  const bool banded = band < a.L;

  float q[32], o[32];
  {
    const int ic = qv ? iq : a.q_lo;
    const float4* qp = reinterpret_cast<const float4*>(a.qkv + (size_t)(base + (long long)ic * estride) * a.ld + head * 32);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float4 t = qp[k];
      q[4 * k] = t.x; q[4 * k + 1] = t.y; q[4 * k + 2] = t.z; q[4 * k + 3] = t.w;
    }
  }
#pragma unroll
  for (int k = 0; k < 32; ++k) o[k] = 0.f;
  float mrun = -1e30f, lrun = 0.f;

  const int q_last = min(q0 + ATT_QB, a.q_hi) - 1;
  const int klo = banded ? max(0, q0 - band) : 0;
  const int khi = banded ? min(a.L, q_last + band + 1) : a.L;
  const int wq0 = q0 + warp * 32;                  // this warp's first / last query
  const int wq1 = min(wq0 + 31, a.q_hi - 1);
  const float* bias = a.bias ? a.bias + head * (2 * band + 1) + band : nullptr;

  for (int kc0 = klo; kc0 < khi; kc0 += ATT_KC) {
    const int nk = min(ATT_KC, khi - kc0);
    __syncthreads();
    for (int idx = threadIdx.x; idx < nk * 16; idx += blockDim.x) {
      const int r = idx >> 4, c = idx & 15;      // c < 8: K, else V
      const float* src = a.qkv + (size_t)(base + (long long)(kc0 + r) * estride) * a.ld + 256 + (c >> 3) * 256 + head * 32 + (c & 7) * 4;
      const float4 t = *reinterpret_cast<const float4*>(src);
      float* dst = (c < 8) ? &Ks[r][(c & 7) * 4] : &Vs[r][(c & 7) * 4];
      *reinterpret_cast<float4*>(dst) = t;
    }
    __syncthreads();
    int j0 = kc0, j1 = kc0 + nk;                   // keys this warp needs from the chunk
    if (banded) { j0 = max(j0, wq0 - band); j1 = min(j1, wq1 + band + 1); }
    if (wq0 > wq1) { j0 = 0; j1 = 0; }
    for (int j = j0; j < j1; j += 4) {
      float s[4];
      bool ok[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int jj = j + u;
        const int rel = jj - iq;
        ok[u] = qv && (jj < j1) && (!banded || (rel <= band && rel >= -band));
        const int r = min(jj, kc0 + nk - 1) - kc0;
        const float4* kr = reinterpret_cast<const float4*>(&Ks[r][0]);
        float d = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float4 t = kr[k];
          d += q[4 * k] * t.x + q[4 * k + 1] * t.y + q[4 * k + 2] * t.z + q[4 * k + 3] * t.w;
        }
        if (bias && ok[u]) d += bias[rel];
        s[u] = ok[u] ? d : -1e30f;
      }
      const float mnew = fmaxf(fmaxf(fmaxf(s[0], s[1]), fmaxf(s[2], s[3])), mrun);
      const float corr = expf(mrun - mnew);
      float pw[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) pw[u] = ok[u] ? expf(s[u] - mnew) : 0.f;
      lrun = lrun * corr + ((pw[0] + pw[1]) + (pw[2] + pw[3]));
      mrun = mnew;
#pragma unroll
      for (int k = 0; k < 32; ++k) o[k] *= corr;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int r = min(j + u, kc0 + nk - 1) - kc0;
        const float4* vr = reinterpret_cast<const float4*>(&Vs[r][0]);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float4 t = vr[k];
          o[4 * k] += pw[u] * t.x; o[4 * k + 1] += pw[u] * t.y;
          o[4 * k + 2] += pw[u] * t.z; o[4 * k + 3] += pw[u] * t.w;
        }
      }
    }
  }
  if (qv) {
    const float inv = 1.0f / lrun;
    float4* op = reinterpret_cast<float4*>(a.out + (size_t)(base + (long long)iq * estride) * a.ldo + head * 32);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      op[k] = make_float4(o[4 * k] * inv, o[4 * k + 1] * inv, o[4 * k + 2] * inv, o[4 * k + 3] * inv);
  }
}

int launch_attention(const AttnArgs& a, cudaStream_t st) {
  if (a.q_hi <= a.q_lo || a.nseq <= 0) return 0;
  dim3 grid(a.nseq, 8, (a.q_hi - a.q_lo + ATT_QB - 1) / ATT_QB);
  attention_kernel<<<grid, 128, 0, st>>>(a);
  DAWN_LAUNCH_OK();
  return 0;
}

// =========================================================================== spatial linear attention context
// per (frame, head): ctx[d][e] = sum_n softmax_n(k)[d,n] v[e,n]; then Bf rows = ctx * Wout slice   (U:619-626)
__global__ void __launch_bounds__(256) sla_context_kernel(const float* __restrict__ qkv, int ld, int P,
                                                          const float* __restrict__ WoutT, int C,
                                                          float* __restrict__ Bf, int ldb) {
  __shared__ float s_ek[64][32];
  __shared__ float s_v[64][33];
  __shared__ float s_max[8][32];
  __shared__ float s_ctx[32][33];
  __shared__ float s_sum[32];
  const int f = blockIdx.x, h = blockIdx.y, tid = threadIdx.x;
  const float* kbase = qkv + (size_t)f * P * ld + 256 + h * 32;
  const float* vbase = qkv + (size_t)f * P * ld + 512 + h * 32;
  // pass 1: column max over positions
  {
    const int d = tid & 31, r = tid >> 5;
    float mx = -3.0e38f;
    for (int n = r; n < P; n += 8) mx = fmaxf(mx, kbase[(size_t)n * ld + d]);
    s_max[r][d] = mx;
  }
  __syncthreads();
  if (tid < 32) {
    float mx = s_max[0][tid];
#pragma unroll
    for (int r = 1; r < 8; ++r) mx = fmaxf(mx, s_max[r][tid]);
    s_max[0][tid] = mx;
  }
  __syncthreads();
  // pass 2: thread owns ctx[d][e0..e0+3]
  const int d = tid >> 3, e0 = (tid & 7) * 4;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  float ssum = 0.f;
  for (int n0 = 0; n0 < P; n0 += 64) {
    const int nn = min(64, P - n0);
    __syncthreads();
    for (int idx = tid; idx < 64 * 32; idx += 256) {
      const int r = idx >> 5, c = idx & 31;
      float ek = 0.f, vv = 0.f;
      if (r < nn) {
        ek = expf(kbase[(size_t)(n0 + r) * ld + c] - s_max[0][c]);
        vv = vbase[(size_t)(n0 + r) * ld + c];
      }
      s_ek[r][c] = ek;
      s_v[r][c] = vv;
    }
    __syncthreads();
#pragma unroll 8
    for (int r = 0; r < 64; ++r) {
      const float ek = s_ek[r][d];
      ssum += ek;
      acc[0] += ek * s_v[r][e0]; acc[1] += ek * s_v[r][e0 + 1];
      acc[2] += ek * s_v[r][e0 + 2]; acc[3] += ek * s_v[r][e0 + 3];
    }
  }
  if ((tid & 7) == 0) s_sum[d] = ssum;
  __syncthreads();
  {
    const float inv = 1.0f / s_sum[d];
#pragma unroll
    for (int u = 0; u < 4; ++u) s_ctx[d][e0 + u] = acc[u] * inv;
  }
  __syncthreads();
  // compose with the out-projection: Bf[h*32+dd][c] = sum_e ctx[dd][e] * WoutT[h*32+e][c]
  float* bf = Bf + (size_t)f * 256 * ldb + (size_t)(h * 32) * ldb;
  const float* wt = WoutT + (size_t)(h * 32) * C;
  for (int idx = tid; idx < 32 * C; idx += 256) {
    const int dd = idx / C, c = idx - dd * C;
    float s = 0.f;
#pragma unroll 8
    for (int e = 0; e < 32; ++e) s += s_ctx[dd][e] * wt[(size_t)e * C + c];
    bf[(size_t)dd * ldb + c] = s;
  }
}

int launch_sla_context(const float* qkv, int ld, int F, int P, const float* WoutT, int C, float* Bf, int ldb,
                       cudaStream_t st) {
  dim3 grid(F, 8);
  sla_context_kernel<<<grid, 256, 0, st>>>(qkv, ld, P, WoutT, C, Bf, ldb);
  DAWN_LAUNCH_OK();
  return 0;
}

// =========================================================================== layout transforms / init conv / heads
// x[c][f][p] -> out[f][p][c_dst0 + c] (Cpad channels per pixel).  Channels outside [c_dst0, c_dst0+C) are zeroed.
// x holds `clips` such tensors back to back; output frame f * clips + b is frame f of clip b
__global__ void ncf_to_nhwc_kernel(const float* __restrict__ x, int C, int F, int HW, int Cpad, int c_dst0,
                                   float* __restrict__ out, const int* __restrict__ skip_flag, int skip_if, int clips) {
  __shared__ float tile[32][33];
  if (skip_flag && *skip_flag == skip_if) return;
  const int fo = blockIdx.z, f = fo / clips;
  x += (size_t)(fo % clips) * C * F * HW;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;       // c0 indexes destination channels
  const int tx = threadIdx.x, ty = threadIdx.y;               // (32, 8)
  for (int k = ty; k < 32; k += 8) {
    const int cd = c0 + k, cs = cd - c_dst0, p = p0 + tx;
    float v = 0.f;
    if (cs >= 0 && cs < C && p < HW) v = x[((size_t)cs * F + f) * HW + p];
    tile[k][tx] = v;
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    const int p = p0 + k, cd = c0 + tx;
    if (p < HW && cd < Cpad) out[((size_t)fo * HW + p) * Cpad + cd] = tile[tx][k];
  }
}
int launch_ncf_to_nhwc(const float* x, int C, int F, int HW, int Cpad, int c_dst0, float* out, cudaStream_t st,
                       const int* skip_flag, int skip_if, int clips) {
  dim3 grid((HW + 31) / 32, (Cpad + 31) / 32, F * clips);
  ncf_to_nhwc_kernel<<<grid, dim3(32, 8), 0, st>>>(x, C, F, HW, Cpad, c_dst0, out, skip_flag, skip_if, clips);
  DAWN_LAUNCH_OK();
  return 0;
}

// Per-clip constant part of the k x k init conv as k row-convolutions that run side by side: copy s of the feature frame is
// the frame shifted by (s - pad) rows (zero outside), so row ky of the kernel becomes a 1 x k conv over copy ky and the k
// partial maps only need adding.  One frame of 64x64 pixels is 32 row tiles of the contraction kernel: k copies = k x 32 CTAs.
// x[c][p] -> out[s][p][c_dst0 + c], Cpad channels per pixel, other channels zero.  With several clips (clip b's frame at
// x + b * clip_stride) copy s of clip b is out[s * clips + b].
__global__ void fea_shift_nhwc_kernel(const float* __restrict__ x, long long cstride, long long clip_stride, int clips, int C, int H, int W,
                                      int Cpad, int c_dst0, int pad, float* __restrict__ out, const int* __restrict__ skip_flag, int skip_if) {
  __shared__ float tile[32][33];
  if (skip_flag && *skip_flag == skip_if) return;
  const int so = blockIdx.z, s = so / clips, HW = H * W, shift = (s - pad) * W;
  x += (size_t)(so % clips) * clip_stride;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;               // (32, 8)
  for (int k = ty; k < 32; k += 8) {
    const int cd = c0 + k, cs = cd - c_dst0, p = p0 + tx, ps = p + shift;
    float v = 0.f;
    if (cs >= 0 && cs < C && p < HW && ps >= 0 && ps < HW) v = x[(size_t)cs * cstride + ps];
    tile[k][tx] = v;
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    const int p = p0 + k, cd = c0 + tx;
    if (p < HW && cd < Cpad) out[((size_t)so * HW + p) * Cpad + cd] = tile[tx][k];
  }
}
int launch_fea_shift_nhwc(const float* x, long long cstride, long long clip_stride, int clips, int C, int H, int W, int Cpad, int c_dst0,
                          int k, float* out, cudaStream_t st, const int* skip_flag, int skip_if) {
  dim3 grid((H * W + 31) / 32, (Cpad + 31) / 32, k * clips);
  fea_shift_nhwc_kernel<<<grid, dim3(32, 8), 0, st>>>(x, cstride, clip_stride, clips, C, H, W, Cpad, c_dst0, k / 2, out, skip_flag, skip_if);
  DAWN_LAUNCH_OK();
  return 0;
}
// map[i] = bias[i % Co] + sum_s part[s][i]   (fixed order: deterministic)
__global__ void map_reduce_kernel(const float* __restrict__ part, int nsplit, long long n, const float* __restrict__ bias, int Co,
                                  float* __restrict__ map, const int* __restrict__ skip_flag, int skip_if) {
  if (skip_flag && *skip_flag == skip_if) return;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float acc = bias ? bias[(int)(i % Co)] : 0.f;
  for (int s = 0; s < nsplit; ++s) acc += part[(size_t)s * n + i];
  map[i] = acc;
}
int launch_map_reduce(const float* part, int nsplit, long long n, const float* bias, int Co, float* map, cudaStream_t st,
                      const int* skip_flag, int skip_if) {
  map_reduce_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(part, nsplit, n, bias, Co, map, skip_flag, skip_if);
  DAWN_LAUNCH_OK();
  return 0;
}

// flag = 1 iff some channel c in [c0, C) of x (C, F, HW) differs between frame 0 and any other frame (bit compare: NaNs and
// signed zeros count as different -> the general path).  The reference's sampler tiles the per-clip features over the frames
// (U:1167 `fea.repeat`), so the general entry can take the hoisted init conv whenever this finds no difference.
// Per clip (x holds `clips` (C, F, HW) tensors back to back): flag[b] for clip b, and flag[clips] counts the clips whose flag is set.
__global__ void frame_invariance_kernel(const float* __restrict__ x, int c0, int C, int F, int HW, int clips, int* __restrict__ flag) {
  const long long per_c = (long long)(F - 1) * HW, per_clip = (long long)(C - c0) * per_c, total = per_clip * clips;
  unsigned int diff = 0;                         // bit b: clip b differs
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / per_clip);
    const long long ic = i - (long long)b * per_clip;
    const int c = c0 + (int)(ic / per_c);
    const long long r = ic - (long long)(c - c0) * per_c;
    const int p = (int)(r % HW);
    const float* base = x + ((size_t)b * C + c) * F * HW;
    if (__float_as_uint(base[HW + r]) != __float_as_uint(base[p])) diff |= 1u << b;
  }
  diff = __reduce_or_sync(0xffffffffu, diff);
  if ((threadIdx.x & 31) == 0)
    for (int b = 0; b < clips; ++b)
      if (((diff >> b) & 1u) && atomicOr(flag + b, 1) == 0) atomicAdd(flag + clips, 1);
}
int launch_frame_invariance(const float* x, int c0, int C, int F, int HW, int clips, int* flag, cudaStream_t st) {
  DAWN_CUDA_OK(cudaMemsetAsync(flag, 0, sizeof(int) * (clips + 1), st));
  if (F > 1 && C > c0) {
    frame_invariance_kernel<<<148 * 8, 256, 0, st>>>(x, c0, C, F, HW, clips, flag);
    DAWN_LAUNCH_OK();
  }
  return 0;
}

// hoisted init conv: only the 3 noisy channels change per step; the 272 feature channels are a per-clip map.
// Clip b's channels 0..2 start at xt + b * clip_stride, map holds one (H, W, Co) map per clip; output frame f * clips + b is frame f
// of clip b, and skip_flag (optional) is per clip: clip b is left alone when skip_flag[b] == skip_if.
__global__ void init_conv_x3_kernel(const float* __restrict__ xt, long long clip_stride, int F, int H, int W, int clips,
                                    const float* __restrict__ w3, const float* __restrict__ map, int Co,
                                    float* __restrict__ out, int ldo, int ksz, const int* __restrict__ skip_flag, int skip_if) {
  extern __shared__ float sw[];                 // [ksz*ksz*3][Co]
  const int ntap = ksz * ksz * 3;
  for (int i = threadIdx.x; i < ntap * Co; i += blockDim.x) sw[i] = w3[i];
  __syncthreads();
  const int cg = Co >> 2;                       // float4 groups per pixel
  const long long total = (long long)F * clips * H * W * cg;
  const int pad = ksz / 2;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(idx % cg) * 4;
    const long long pix = idx / cg;
    const int x0 = (int)(pix % W);
    const int y0 = (int)((pix / W) % H);
    const int fo = (int)(pix / ((long long)W * H)), f = fo / clips, b = fo % clips;
    if (skip_flag && skip_flag[b] == skip_if) continue;
    const float* xc = xt + (size_t)b * clip_stride;
    float4 acc = *reinterpret_cast<const float4*>(map + (((size_t)b * H + y0) * W + x0) * Co + c4);
    for (int ky = 0; ky < ksz; ++ky) {
      const int iy = y0 + ky - pad;
      if (iy < 0 || iy >= H) continue;
      for (int kx = 0; kx < ksz; ++kx) {
        const int ix = x0 + kx - pad;
        if (ix < 0 || ix >= W) continue;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float xv = xc[(((size_t)c * F + f) * H + iy) * W + ix];
          const float4 wv = *reinterpret_cast<const float4*>(&sw[((ky * ksz + kx) * 3 + c) * Co + c4]);
          acc.x += xv * wv.x; acc.y += xv * wv.y; acc.z += xv * wv.z; acc.w += xv * wv.w;
        }
      }
    }
    *reinterpret_cast<float4*>(out + (size_t)pix * ldo + c4) = acc;
  }
}
// register-tiled variant for the 64-channel model family: a block owns 8 output rows x 64 columns of one frame, a thread 4 pixels x 8
// channels (32 accumulators).  One (channel, ky) input row segment of 4 + KS - 1 values feeds KS x 32 FMAs, so shared-memory traffic
// per FMA drops ~4x against the one-pixel-per-thread kernel above, which was bound by its weight reads.
template <int KS>
__global__ void __launch_bounds__(128) init_conv_x3_tiled_kernel(const float* __restrict__ xt, long long clip_stride, int F, int H, int W,
                                                                 int clips,
                                                                 const float* __restrict__ w3, const float* __restrict__ map,
                                                                 float* __restrict__ out, int ldo, const int* __restrict__ skip_flag,
                                                                 int skip_if) {
  constexpr int PAD = KS / 2, TW = 64, TR = 8, IR = TR + KS - 1, ILD = 72, NW = KS * KS * 3 * 64;
  extern __shared__ __align__(16) float sm_ic[];
  const int fo = blockIdx.z, f = fo / clips, b = fo % clips;
  if (skip_flag && skip_flag[b] == skip_if) return;
  float* sw = sm_ic;                            // [KS*KS*3][64]
  float* sx = sm_ic + NW;                       // [3][IR][ILD]
  const int tid = threadIdx.x;
  const int y0 = blockIdx.y * TR, x0 = blockIdx.x * TW;
  xt += (size_t)b * clip_stride;
  map += (size_t)b * H * W * 64;
  for (int i = tid; i < NW / 4; i += 128) reinterpret_cast<float4*>(sw)[i] = __ldg(reinterpret_cast<const float4*>(w3) + i);
  for (int i = tid; i < 3 * IR * ILD; i += 128) {
    const int c = i / (IR * ILD), rem = i - c * IR * ILD, r = rem / ILD, col = rem - r * ILD;
    const int iy = y0 + r - PAD, ix = x0 + col - PAD;
    float v = 0.f;
    if (col < TW + KS - 1 && iy >= 0 && iy < H && ix >= 0 && ix < W) v = xt[(((size_t)c * F + f) * H + iy) * W + ix];
    sx[i] = v;
  }
  __syncthreads();
  const int pxg = tid >> 3, cg = tid & 7;
  for (int r = 0; r < TR; ++r) {
    const int y = y0 + r;
    if (y >= H) break;
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int x = x0 + pxg * 4 + i;
      if (x < W) {
        const float4 m0 = __ldg(reinterpret_cast<const float4*>(map + ((size_t)y * W + x) * 64 + cg * 8));
        const float4 m1 = __ldg(reinterpret_cast<const float4*>(map + ((size_t)y * W + x) * 64 + cg * 8 + 4));
        acc[i][0] = m0.x; acc[i][1] = m0.y; acc[i][2] = m0.z; acc[i][3] = m0.w;
        acc[i][4] = m1.x; acc[i][5] = m1.y; acc[i][6] = m1.z; acc[i][7] = m1.w;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
      }
    }
#pragma unroll 1
    for (int c = 0; c < 3; ++c)
#pragma unroll 1
      for (int ky = 0; ky < KS; ++ky) {
        const float* row = sx + (c * IR + r + ky) * ILD + pxg * 4;
        float xv[12];
        *reinterpret_cast<float4*>(xv) = *reinterpret_cast<const float4*>(row);
        *reinterpret_cast<float4*>(xv + 4) = *reinterpret_cast<const float4*>(row + 4);
        *reinterpret_cast<float4*>(xv + 8) = *reinterpret_cast<const float4*>(row + 8);
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
          const float* wp = sw + ((ky * KS + kx) * 3 + c) * 64 + cg * 8;
          const float4 w0 = *reinterpret_cast<const float4*>(wp), w1 = *reinterpret_cast<const float4*>(wp + 4);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float xx = xv[i + kx];
            acc[i][0] += xx * w0.x; acc[i][1] += xx * w0.y; acc[i][2] += xx * w0.z; acc[i][3] += xx * w0.w;
            acc[i][4] += xx * w1.x; acc[i][5] += xx * w1.y; acc[i][6] += xx * w1.z; acc[i][7] += xx * w1.w;
          }
        }
      }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int x = x0 + pxg * 4 + i;
      if (x < W) {
        float* dst = out + ((size_t)fo * H * W + (size_t)y * W + x) * ldo + cg * 8;
        *reinterpret_cast<float4*>(dst) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
        *reinterpret_cast<float4*>(dst + 4) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
      }
    }
  }
}

int launch_init_conv_x3(const float* xt, long long clip_stride, int F, int H, int W, int clips, const float* w3, const float* map, int Co,
                        float* out, int ldo, int ksz, cudaStream_t st, const int* skip_flag, int skip_if) {
  if (ksz == 7 && Co == 64) {
    constexpr size_t smem_t = (size_t)(7 * 7 * 3 * 64 + 3 * (8 + 6) * 72) * sizeof(float);
    static bool attr_t = false;
    if (!attr_t) {
      DAWN_CUDA_OK(cudaFuncSetAttribute(init_conv_x3_tiled_kernel<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_t));
      attr_t = true;
    }
    init_conv_x3_tiled_kernel<7><<<dim3((W + 63) / 64, (H + 7) / 8, F * clips), 128, smem_t, st>>>(xt, clip_stride, F, H, W, clips, w3, map, out, ldo,
                                                                                                  skip_flag, skip_if);
    DAWN_LAUNCH_OK();
    return 0;
  }
  const size_t smem = (size_t)ksz * ksz * 3 * Co * sizeof(float);
  static bool attr = false;
  if (!attr) {
    DAWN_CUDA_OK(cudaFuncSetAttribute(init_conv_x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    attr = true;
  }
  if (smem > 100 * 1024) { set_last_error("init_conv_x3: kernel too large for shared memory"); return -1; }
  const long long total = (long long)F * clips * H * W * (Co >> 2);
  long long blocks = (total + 255) / 256;
  if (blocks > 148 * 8) blocks = 148 * 8;
  init_conv_x3_kernel<<<(int)blocks, 256, smem, st>>>(xt, clip_stride, F, H, W, clips, w3, map, Co, out, ldo, ksz, skip_flag, skip_if);
  DAWN_LAUNCH_OK();
  return 0;
}

// final 1x1 convs of both heads, written channel-major (the module's NCFHW output), clip by clip: row m is pixel p of frame
// fo = f * clips + b, written to out[b][j][f][p]
__global__ void heads_out_kernel(const float* __restrict__ hf, const float* __restrict__ ho, int C, int M, int HW, int clips,
                                 const float* __restrict__ Wf, const float* __restrict__ bf, int ng,
                                 const float* __restrict__ Wo, const float* __restrict__ bo, int nc,
                                 float* __restrict__ out) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  size_t mc = m, Mc = M;                                       // row within the clip, rows per clip
  if (clips > 1) {
    const int fo = m / HW, b = fo % clips;
    Mc = M / clips;
    mc = (size_t)(fo / clips) * HW + (m - fo * HW);
    out += (size_t)b * (ng + nc) * Mc;
  }
  for (int j = 0; j < ng + nc; ++j) {
    const float* src = (j < ng ? hf : ho) + (size_t)m * C;
    const float* w = (j < ng) ? Wf + (size_t)j * C : Wo + (size_t)(j - ng) * C;
    float acc = (j < ng) ? bf[j] : bo[j - ng];
    for (int c = 0; c < C; c += 4) {
      const float4 a = *reinterpret_cast<const float4*>(src + c);
      const float4 b = *reinterpret_cast<const float4*>(w + c);
      acc += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
    }
    out[j * Mc + mc] = acc;
  }
}
int launch_heads_out(const float* hf, const float* ho, int C, int M, int HW, int clips, const float* Wf, const float* bf, int ng,
                     const float* Wo, const float* bo, int nc, float* out, cudaStream_t st) {
  heads_out_kernel<<<(M + 127) / 128, 128, 0, st>>>(hf, ho, C, M, HW, clips, Wf, bf, ng, Wo, bo, nc, out);
  DAWN_LAUNCH_OK();
  return 0;
}

}  // namespace dawn
