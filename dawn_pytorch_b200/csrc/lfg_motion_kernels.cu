// Non-GEMM kernels of the LFG motion estimator: the anti-aliased 1/4 downsample, the region softmax and moments, the flow
// predictor's input assembly and output combine, the background head and its input packing.  The convolutions run on the shared
// contraction kernels and the pooling on the decoder's (lfg_motion.cu).  Reference: LFG/modules/region_predictor.py, bg_motion_predictor.py,
// pixelwise_flow_predictor.py, util.py:22-67 (region2gaussian, make_coordinate_grid), :217-275 (AntiAliasInterpolation2d).
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "lfg_kernels.cuh"
#include "lfg_motion_kernels.cuh"

namespace dawn {
namespace {

// make_coordinate_grid (util.py:51-67) as torch evaluates it in fp32: 2 * (i / (n - 1)) - 1
__device__ __forceinline__ float grid_coord(int i, int n) { return 2.f * ((float)i / (float)(n - 1)) - 1.f; }

inline int grid_for(long long n, int threads, int cap) {
  const long long b = (n + threads - 1) / threads;
  return (int)std::max<long long>(1, std::min<long long>(b, cap));
}

// sum over a 256-thread block; every thread gets the result
__device__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double t = 0.0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
  return t;
}
__device__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) t = fmaxf(t, red[i]);
  return t;
}

// --------------------------------------------------------------------------------------------- 1. anti-aliased downsample
// one thread = one kept pixel (every 4th row and column) x 3 channels; the 13x13 taps of each channel live in shared memory
__global__ void __launch_bounds__(256) aa_down_kernel(const float* __restrict__ img, int N, int H, int W, const float* __restrict__ wt,
                                                      float* __restrict__ out, int ld, int off, int cw) {
  __shared__ float s_w[3 * kAAK * kAAK];
  for (int i = threadIdx.x; i < 3 * kAAK * kAAK; i += blockDim.x) s_w[i] = wt[i];
  __syncthreads();
  const int h = H >> 2, w = W >> 2, ka = kAAK / 2;
  const long long total = (long long)N * h * w;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % w), y = (int)((idx / w) % h), n = (int)(idx / ((long long)w * h));
    float acc[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* plane = img + ((size_t)n * 3 + c) * H * W;
      float a = 0.f;
      for (int i = 0; i < kAAK; ++i) {
        const int iy = 4 * y + i - ka;
        if (iy < 0 || iy >= H) continue;
        const float* row = plane + (size_t)iy * W;
#pragma unroll
        for (int j = 0; j < kAAK; ++j) {
          const int ix = 4 * x + j - ka;
          if (ix >= 0 && ix < W) a += s_w[(c * kAAK + i) * kAAK + j] * __ldg(row + ix);
        }
      }
      acc[c] = a;
    }
    float* o = out + (size_t)idx * ld + off;
    o[0] = acc[0]; o[1] = acc[1]; o[2] = acc[2];
    for (int c = 3; c < cw; ++c) o[c] = 0.f;
  }
}

// --------------------------------------------------------------------------------------------- 2. region softmax and moments
// one CTA = one (frame, region); three sweeps over the h w logits: max, then exp sums with the first moments, then the second
// moments about the mean (as region2affine subtracts the mean before the products)
__global__ void __launch_bounds__(256) region_moments_kernel(const float* __restrict__ logits, int ldl, int h, int w, int R, float temp,
                                                             float* __restrict__ shift, float* __restrict__ covar, float* __restrict__ heat) {
  __shared__ double red_d[8];
  __shared__ float red_f[8];
  const int n = blockIdx.x / R, r = blockIdx.x - n * R, P = h * w;
  const float* lg = logits + (size_t)n * P * ldl + r;
  float m = -INFINITY;
  for (int p = threadIdx.x; p < P; p += blockDim.x) m = fmaxf(m, __ldg(lg + (size_t)p * ldl) / temp);
  m = block_max(m, red_f);
  double s0 = 0.0, sx = 0.0, sy = 0.0;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const double e = (double)expf(__ldg(lg + (size_t)p * ldl) / temp - m);
    s0 += e; sx += e * grid_coord(p % w, w); sy += e * grid_coord(p / w, h);
  }
  s0 = block_sum(s0, red_d); sx = block_sum(sx, red_d); sy = block_sum(sy, red_d);
  const double mx = sx / s0, my = sy / s0;
  double cxx = 0.0, cxy = 0.0, cyy = 0.0;
  float* hm = heat ? heat + ((size_t)n * R + r) * P : nullptr;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const double e = (double)expf(__ldg(lg + (size_t)p * ldl) / temp - m) / s0;
    const double dx = grid_coord(p % w, w) - mx, dy = grid_coord(p / w, h) - my;
    cxx += e * dx * dx; cxy += e * dx * dy; cyy += e * dy * dy;
    if (hm) hm[p] = (float)e;
  }
  cxx = block_sum(cxx, red_d); cxy = block_sum(cxy, red_d); cyy = block_sum(cyy, red_d);
  if (threadIdx.x == 0) {
    const size_t b = (size_t)n * R + r;
    shift[2 * b] = (float)mx; shift[2 * b + 1] = (float)my;
    covar[4 * b] = (float)cxx; covar[4 * b + 1] = (float)cxy; covar[4 * b + 2] = (float)cxy; covar[4 * b + 3] = (float)cyy;
  }
}

// --------------------------------------------------------------------------------------------- 3. flow-predictor input
struct RegionAlgebra { float inv_d[4], inv_s[4], A[4], mu_d[2], mu_s[2]; };

__device__ void inverse2(const float* m, double* o) {
  const double a = m[0], b = m[1], c = m[2], d = m[3], det = a * d - b * c;
  o[0] = d / det; o[1] = -b / det; o[2] = -c / det; o[3] = a / det;
}
// exp(-0.5 (g - mu)^T inv (g - mu)) in region2gaussian's order (util.py:44-46)
__device__ __forceinline__ float gaussian(float gx, float gy, const float* mu, const float* inv) {
  const float sx = gx - mu[0], sy = gy - mu[1];
  const float e = (sx * inv[0] + sy * inv[2]) * sx + (sx * inv[1] + sy * inv[3]) * sy;
  return expf(-0.5f * e);
}

__global__ void __launch_bounds__(256) flow_input_kernel(const float4* __restrict__ src4, int h, int w, int R,
                                                         const float* __restrict__ src_shift, const float* __restrict__ src_covar,
                                                         const float* __restrict__ src_affine, const float* __restrict__ drv_shift,
                                                         const float* __restrict__ drv_covar, const float* __restrict__ drv_affine,
                                                         const float* __restrict__ bg, int revert, float* __restrict__ out, int ld,
                                                         int off, int cw, float* __restrict__ motion) {
  __shared__ RegionAlgebra s_r[kMotionMaxRegions];
  __shared__ float s_bg[9];
  const int n = blockIdx.y, P = h * w;
  if (threadIdx.x < R) {
    const int r = threadIdx.x;
    const size_t b = (size_t)n * R + r;
    RegionAlgebra a;
    double id[4], is[4], iad[4];
    inverse2(drv_covar + 4 * b, id);
    inverse2(src_covar + 4 * b, is);
    inverse2(drv_affine + 4 * b, iad);                                   // torch.inverse(driving affine), :76
    const float* as = src_affine + 4 * b;
    double A[4] = {as[0] * iad[0] + as[1] * iad[2], as[0] * iad[1] + as[1] * iad[3],
                   as[2] * iad[0] + as[3] * iad[2], as[2] * iad[1] + as[3] * iad[3]};
    if (revert) {                                                        // :77-78: affine * sign(affine[0, 0])
      const double sg = (double)((A[0] > 0.0) - (A[0] < 0.0));
      for (int i = 0; i < 4; ++i) A[i] *= sg;
    }
    for (int i = 0; i < 4; ++i) { a.inv_d[i] = (float)id[i]; a.inv_s[i] = (float)is[i]; a.A[i] = (float)A[i]; }
    a.mu_d[0] = drv_shift[2 * b]; a.mu_d[1] = drv_shift[2 * b + 1];
    a.mu_s[0] = src_shift[2 * b]; a.mu_s[1] = src_shift[2 * b + 1];
    s_r[r] = a;
  }
  if (threadIdx.x < 9) s_bg[threadIdx.x] = bg ? bg[(size_t)n * 9 + threadIdx.x] : (float)(threadIdx.x % 4 == 0);
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const float gx = grid_coord(p % w, w), gy = grid_coord(p / w, h);
  float* o = out + ((size_t)n * P + p) * ld + off;
  float* mo = motion + ((size_t)n * P + p) * 2 * (R + 1);
  for (int k = 0; k <= R; ++k) {
    float mx, my, heat;
    if (k == 0) {                                                        // background grid (:87-95), zero heatmap (:63-65)
      mx = gx; my = gy; heat = 0.f;
      if (bg) {
        const float hx = s_bg[0] * gx + s_bg[1] * gy + s_bg[2], hy = s_bg[3] * gx + s_bg[4] * gy + s_bg[5];
        const float hz = s_bg[6] * gx + s_bg[7] * gy + s_bg[8];
        mx = hx / hz; my = hy / hz;
      }
    } else {
      const RegionAlgebra& a = s_r[k - 1];
      heat = gaussian(gx, gy, a.mu_d, a.inv_d) - gaussian(gx, gy, a.mu_s, a.inv_s);   // :56-61
      const float cx = gx - a.mu_d[0], cy = gy - a.mu_d[1];              // :72-84
      mx = (a.A[0] * cx + a.A[1] * cy) + a.mu_s[0];
      my = (a.A[2] * cx + a.A[3] * cy) + a.mu_s[1];
    }
    mo[2 * k] = mx; mo[2 * k + 1] = my;
    const Corners c = grid_corners(mx, my, h, w);                        // :99-109, grid_sample defaults
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c.vnw) { const float4 v = __ldg(src4 + (size_t)c.y0 * w + c.x0); s.x += v.x * c.wnw; s.y += v.y * c.wnw; s.z += v.z * c.wnw; }
    if (c.vne) { const float4 v = __ldg(src4 + (size_t)c.y0 * w + c.x0 + 1); s.x += v.x * c.wne; s.y += v.y * c.wne; s.z += v.z * c.wne; }
    if (c.vsw) { const float4 v = __ldg(src4 + (size_t)(c.y0 + 1) * w + c.x0); s.x += v.x * c.wsw; s.y += v.y * c.wsw; s.z += v.z * c.wsw; }
    if (c.vse) { const float4 v = __ldg(src4 + (size_t)(c.y0 + 1) * w + c.x0 + 1); s.x += v.x * c.wse; s.y += v.y * c.wse; s.z += v.z * c.wse; }
    o[4 * k] = heat; o[4 * k + 1] = s.x; o[4 * k + 2] = s.y; o[4 * k + 3] = s.z;   // (R + 1, 1 + 3) order, :117-121
  }
  for (int c = 4 * (R + 1); c < cw; ++c) o[c] = 0.f;
}

// --------------------------------------------------------------------------------------------- 4. mask, flow and occlusion
__global__ void __launch_bounds__(256) flow_combine_kernel(const float* __restrict__ logits, int ldl, const float* __restrict__ motion,
                                                           long long M, int R, float* __restrict__ flow, float* __restrict__ occ) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const float* lg = logits + (size_t)i * ldl;
  const float* mo = motion + (size_t)i * 2 * (R + 1);
  float mx = -INFINITY;
  for (int k = 0; k <= R; ++k) mx = fmaxf(mx, lg[k]);
  float s = 0.f;
  for (int k = 0; k <= R; ++k) s += expf(lg[k] - mx);
  float fx = 0.f, fy = 0.f;
  for (int k = 0; k <= R; ++k) {
    const float mk = expf(lg[k] - mx) / s;
    fx += mo[2 * k] * mk; fy += mo[2 * k + 1] * mk;
  }
  flow[2 * i] = fx; flow[2 * i + 1] = fy;
  occ[i] = 1.0f / (1.0f + expf(-lg[R + 1]));
}

// --------------------------------------------------------------------------------------------- 5. background head
__global__ void __launch_bounds__(256) bg_head_kernel(const float* __restrict__ x, int ld, int C, int P, const float* __restrict__ fc_w,
                                                      const float* __restrict__ fc_b, float* __restrict__ bg) {
  extern __shared__ float s_mean[];
  const int n = blockIdx.x;
  float* o = bg + (size_t)n * 9;
  if (!fc_w) {
    if (threadIdx.x < 9) o[threadIdx.x] = (float)(threadIdx.x % 4 == 0);
    return;
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double s = 0.0;
    for (int p = 0; p < P; ++p) s += x[((size_t)n * P + p) * ld + c];
    s_mean[c] = (float)(s / P);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < 6) {
    double s = 0.0;
    for (int c = lane; c < C; c += 32) s += (double)fc_w[(size_t)warp * C + c] * s_mean[c];
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
    if (lane == 0) o[warp] = (float)(s + fc_b[warp]);                   // out[:, :2, :] = prediction.view(bs, 2, 3)
  }
  if (threadIdx.x < 3) o[6 + threadIdx.x] = (float)(threadIdx.x == 2);
}

// --------------------------------------------------------------------------------------------- layout pass
__global__ void pack_pair_kernel(const float* __restrict__ source, int n_source, const float* __restrict__ driving, int HW, long long total,
                                 float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = (int)(idx & 31);
  const long long pix = idx >> 5;
  const int p = (int)(pix % HW), n = (int)(pix / HW);
  float v = 0.f;
  if (c < 3) v = source[((size_t)(n_source == 1 ? 0 : n) * 3 + c) * HW + p];
  else if (c < 6) v = driving[((size_t)n * 3 + c - 3) * HW + p];
  out[idx] = v;
}

}  // namespace

int launch_lfgm_aa_down(const float* images, int N, int H, int W, const float* weight, float* out, int ld, int off, int cw,
                        cudaStream_t st) {
  const long long n = (long long)N * (H >> 2) * (W >> 2);
  aa_down_kernel<<<grid_for(n, 256, 148 * 16), 256, 0, st>>>(images, N, H, W, weight, out, ld, off, cw);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_lfgm_region_moments(const float* logits, int ldl, int N, int h, int w, int R, float temperature, float* shift,
                               float* covar, float* heatmap, cudaStream_t st) {
  region_moments_kernel<<<N * R, 256, 0, st>>>(logits, ldl, h, w, R, temperature, shift, covar, heatmap);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_lfgm_flow_input(const float* source4, int N, int h, int w, int R, const float* src_shift, const float* src_covar,
                           const float* src_affine, const float* drv_shift, const float* drv_covar, const float* drv_affine,
                           const float* bg, int revert, float* out, int ld, int off, int cw, float* motion, cudaStream_t st) {
  dim3 grid((h * w + 255) / 256, N);
  flow_input_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const float4*>(source4), h, w, R, src_shift, src_covar, src_affine,
                                          drv_shift, drv_covar, drv_affine, bg, revert, out, ld, off, cw, motion);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_lfgm_flow_combine(const float* logits, int ldl, const float* motion, int N, int h, int w, int R, float* flow,
                             float* occlusion, cudaStream_t st) {
  const long long M = (long long)N * h * w;
  flow_combine_kernel<<<(int)((M + 255) / 256), 256, 0, st>>>(logits, ldl, motion, M, R, flow, occlusion);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_lfgm_bg_head(const float* x, int ld, int C, int N, int P, const float* fc_w, const float* fc_b, float* bg, cudaStream_t st) {
  bg_head_kernel<<<N, 256, (size_t)C * sizeof(float), st>>>(x, ld, C, P, fc_w, fc_b, bg);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_lfgm_pack_pair(const float* source, int n_source, const float* driving, int N, int HW, float* out, cudaStream_t st) {
  const long long total = (long long)N * HW * 32;
  pack_pair_kernel<<<(int)((total + 255) / 256), 256, 0, st>>>(source, n_source, driving, HW, total, out);
  DAWN_LAUNCH_OK();
  return 0;
}

}  // namespace dawn
