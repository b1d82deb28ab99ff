// Non-GEMM kernels of the LFG flow decoder: motion packing, warp + occlusion blend (apply_optical), BatchNorm/ReLU passes,
// pooling, layout transforms and the final 7x7 conv + sigmoid + source-image blend.
// Reference: LFG/modules/generator.py:59-90 (deform_input / apply_optical), :138-171 (forward_with_flow); util.py:70-150 (blocks).
#include <algorithm>
#include "common.cuh"
#include "lfg_kernels.cuh"

namespace dawn {
namespace {

// F.interpolate(mode='bilinear', align_corners=False) source taps of output index `dst` (ATen area_pixel_compute_source_index +
// guard_index_and_lambda): src = scale * (dst + 0.5) - 0.5 clamped at 0, i0 = floor(src), i1 = i0 + (i0 < in - 1), l1 = src - i0.
struct Lerp { int i0, i1; float l0, l1; };
__device__ __forceinline__ Lerp lerp_taps(int dst, int in_size, int out_size) {
  Lerp r;
  if (in_size == out_size) { r.i0 = r.i1 = dst; r.l0 = 1.f; r.l1 = 0.f; return r; }
  const float scale = (float)in_size / (float)out_size;
  float src = scale * ((float)dst + 0.5f) - 0.5f;
  src = fmaxf(src, 0.f);
  r.i0 = min((int)floorf(src), in_size - 1);
  r.i1 = r.i0 + ((r.i0 < in_size - 1) ? 1 : 0);
  r.l1 = fminf(fmaxf(src - (float)r.i0, 0.f), 1.f);
  r.l0 = 1.f - r.l1;
  return r;
}
// (grid_x, grid_y, occlusion) of frame f at pixel (y, x) of an (Ho, Wo) level, resized from the (h, w) motion field
__device__ __forceinline__ float3 motion_at(const float4* __restrict__ motion, int f, int h, int w, int y, int x, int Ho, int Wo) {
  const float4* m = motion + (size_t)f * h * w;
  if (Ho == h && Wo == w) { const float4 v = __ldg(m + y * w + x); return make_float3(v.x, v.y, v.z); }
  const Lerp ly = lerp_taps(y, h, Ho), lx = lerp_taps(x, w, Wo);
  const float4 v00 = __ldg(m + ly.i0 * w + lx.i0), v01 = __ldg(m + ly.i0 * w + lx.i1);
  const float4 v10 = __ldg(m + ly.i1 * w + lx.i0), v11 = __ldg(m + ly.i1 * w + lx.i1);
  float3 r;
  r.x = ly.l0 * (lx.l0 * v00.x + lx.l1 * v01.x) + ly.l1 * (lx.l0 * v10.x + lx.l1 * v11.x);
  r.y = ly.l0 * (lx.l0 * v00.y + lx.l1 * v01.y) + ly.l1 * (lx.l0 * v10.y + lx.l1 * v11.y);
  r.z = ly.l0 * (lx.l0 * v00.z + lx.l1 * v01.z) + ly.l1 * (lx.l0 * v10.z + lx.l1 * v11.z);
  return r;
}
__global__ void motion_pack_kernel(const float* __restrict__ flow, const float* __restrict__ occ, int layout, int F, int hw,
                                   float4* __restrict__ motion) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * hw) return;
  float gx, gy, oc;
  if (layout == 0) {
    gx = flow[2 * i]; gy = flow[2 * i + 1]; oc = occ[i];
  } else {
    const long long n = (long long)F * hw;
    gx = flow[i]; gy = flow[n + i]; oc = (flow[2 * n + i] + 1.f) * 0.5f;       // FD:369: (pred[:, 2] + 1) * 0.5
  }
  motion[i] = make_float4(gx, gy, oc, 0.f);
}

// one thread = one output pixel x 4 channels; consecutive threads = consecutive channel groups of the same pixel
__global__ void __launch_bounds__(256) warp_blend_kernel(const float* __restrict__ skip, int C, int Hs, int Ws,
                                                         const float4* __restrict__ motion, int F, int h, int w,
                                                         const float* __restrict__ prev, int ldp, float* __restrict__ out, int ldo) {
  const int cg = C >> 2;
  const long long total = (long long)F * Hs * Ws * cg;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(idx % cg) * 4;
    const long long pix = idx / cg;
    const int x = (int)(pix % Ws), y = (int)((pix / Ws) % Hs), f = (int)(pix / ((long long)Ws * Hs));
    const float3 m = motion_at(motion, f, h, w, y, x, Hs, Ws);
    const Corners c = grid_corners(m.x, m.y, Hs, Ws);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const float* base = skip + c4;
    if (c.vnw) { const float4 v = __ldg(reinterpret_cast<const float4*>(base + ((size_t)c.y0 * Ws + c.x0) * C));
                 acc.x += v.x * c.wnw; acc.y += v.y * c.wnw; acc.z += v.z * c.wnw; acc.w += v.w * c.wnw; }
    if (c.vne) { const float4 v = __ldg(reinterpret_cast<const float4*>(base + ((size_t)c.y0 * Ws + c.x0 + 1) * C));
                 acc.x += v.x * c.wne; acc.y += v.y * c.wne; acc.z += v.z * c.wne; acc.w += v.w * c.wne; }
    if (c.vsw) { const float4 v = __ldg(reinterpret_cast<const float4*>(base + ((size_t)(c.y0 + 1) * Ws + c.x0) * C));
                 acc.x += v.x * c.wsw; acc.y += v.y * c.wsw; acc.z += v.z * c.wsw; acc.w += v.w * c.wsw; }
    if (c.vse) { const float4 v = __ldg(reinterpret_cast<const float4*>(base + ((size_t)(c.y0 + 1) * Ws + c.x0 + 1) * C));
                 acc.x += v.x * c.wse; acc.y += v.y * c.wse; acc.z += v.z * c.wse; acc.w += v.w * c.wse; }
    const float oc = m.z;
    float4 o = make_float4(acc.x * oc, acc.y * oc, acc.z * oc, acc.w * oc);
    if (prev) {
      const float4 p = *reinterpret_cast<const float4*>(prev + (size_t)pix * ldp + c4);
      const float k = 1.f - oc;
      o.x += p.x * k; o.y += p.y * k; o.z += p.z * k; o.w += p.w * k;
    }
    *reinterpret_cast<float4*>(out + (size_t)pix * ldo + c4) = o;
  }
}

__global__ void __launch_bounds__(256) affine_relu_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ scale,
                                                          const float* __restrict__ shift, int C, long long nvec,
                                                          float* __restrict__ z, int ldz) {
  const int cg = C >> 2;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < nvec; idx += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(idx % cg) * 4;
    const long long row = idx / cg;
    float4 v = *reinterpret_cast<const float4*>(x + (size_t)row * ldx + c4);
    if (scale) {
      const float4 s = __ldg(reinterpret_cast<const float4*>(scale + c4)), t = __ldg(reinterpret_cast<const float4*>(shift + c4));
      v.x = v.x * s.x + t.x; v.y = v.y * s.y + t.y; v.z = v.z * s.z + t.z; v.w = v.w * s.w + t.w;
    }
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    *reinterpret_cast<float4*>(z + (size_t)row * ldz + c4) = v;
  }
}

__global__ void __launch_bounds__(256) residual_bn_relu_kernel(const float* __restrict__ y, const float* __restrict__ x, int C, long long nvec,
                                                               float* __restrict__ xnew, const float* __restrict__ scale,
                                                               const float* __restrict__ shift, float* __restrict__ z) {
  const int cg = C >> 2;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < nvec; idx += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(idx % cg) * 4;
    const float4 a = reinterpret_cast<const float4*>(y)[idx], b = reinterpret_cast<const float4*>(x)[idx];
    float4 v = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    reinterpret_cast<float4*>(xnew)[idx] = v;
    if (z) {
      const float4 s = __ldg(reinterpret_cast<const float4*>(scale + c4)), t = __ldg(reinterpret_cast<const float4*>(shift + c4));
      v.x = fmaxf(v.x * s.x + t.x, 0.f); v.y = fmaxf(v.y * s.y + t.y, 0.f);
      v.z = fmaxf(v.z * s.z + t.z, 0.f); v.w = fmaxf(v.w * s.w + t.w, 0.f);
      reinterpret_cast<float4*>(z)[idx] = v;
    }
  }
}

__global__ void relu_avgpool2_kernel(const float* __restrict__ x, int H, int W, int C, float* __restrict__ out) {
  const int cg = C >> 2, Ho = H >> 1, Wo = W >> 1;
  const long long total = (long long)Ho * Wo * cg;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c4 = (int)(idx % cg) * 4;
  const long long pix = idx / cg;
  const int xo = (int)(pix % Wo), yo = (int)(pix / Wo);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const float4 v = *reinterpret_cast<const float4*>(x + ((size_t)(2 * yo + dy) * W + 2 * xo + dx) * C + c4);
      acc.x += fmaxf(v.x, 0.f); acc.y += fmaxf(v.y, 0.f); acc.z += fmaxf(v.z, 0.f); acc.w += fmaxf(v.w, 0.f);
    }
  *reinterpret_cast<float4*>(out + (size_t)pix * C + c4) = make_float4(acc.x * 0.25f, acc.y * 0.25f, acc.z * 0.25f, acc.w * 0.25f);
}

__global__ void chw_to_hwc_kernel(const float* __restrict__ x, int C, int HW, int Cpad, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)HW * Cpad) return;
  const int c = (int)(idx % Cpad);
  const long long p = idx / Cpad;
  out[idx] = (c < C) ? x[(size_t)c * HW + p] : 0.f;
}
__global__ void hwc_to_chw_kernel(const float* __restrict__ x, int ld, int C, long long M, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * C) return;
  const int c = (int)(idx / M);
  const long long m = idx - (long long)c * M;
  out[idx] = x[(size_t)m * ld + c];
}

// final 7x7 conv (Cin -> 3) + sigmoid + source blend.  Block = 16 x 16 output pixels of one frame, thread = one pixel.
// Input channels go through shared memory 8 at a time: halo tile [22][22][8] floats (15.5 KB) + weight slice [49][8][4] (6.3 KB).
constexpr int FT = 16, FK = 7, FP = 3, FH = FT + FK - 1, FC = 8;
__global__ void __launch_bounds__(FT * FT) final_conv_kernel(const float* __restrict__ x, int ldx, int Cin, int F, int H, int W,
                                                             const float* __restrict__ wpack, const float* __restrict__ bias3,
                                                             const float* __restrict__ source, const float4* __restrict__ motion,
                                                             int h, int w, int blend, float* __restrict__ prediction,
                                                             float* __restrict__ deformed) {
  __shared__ __align__(16) float s_in[FH * FH * FC];
  __shared__ __align__(16) float s_w[FK * FK * FC * 4];
  const int tx = threadIdx.x % FT, ty = threadIdx.x / FT;
  const int f = blockIdx.z, y0 = blockIdx.y * FT, x0 = blockIdx.x * FT;
  const int oy = y0 + ty, ox = x0 + tx;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  const float* img = x + (size_t)f * H * W * ldx;
  for (int c0 = 0; c0 < Cin; c0 += FC) {
    __syncthreads();
    // halo tile of FC channels: 2 float4 per halo pixel
    for (int i = threadIdx.x; i < FH * FH * (FC / 4); i += FT * FT) {
      const int q = i % (FC / 4), hp = i / (FC / 4);
      const int hy = hp / FH, hx = hp - hy * FH;
      const int iy = y0 + hy - FP, ix = x0 + hx - FP;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = *reinterpret_cast<const float4*>(img + ((size_t)iy * W + ix) * ldx + c0 + 4 * q);
      *reinterpret_cast<float4*>(&s_in[hp * FC + 4 * q]) = v;
    }
    for (int i = threadIdx.x; i < FK * FK * FC; i += FT * FT) {
      const int tap = i / FC, c = i - tap * FC;
      *reinterpret_cast<float4*>(&s_w[i * 4]) = __ldg(reinterpret_cast<const float4*>(wpack + ((size_t)tap * Cin + c0 + c) * 4));
    }
    __syncthreads();
#pragma unroll 1
    for (int ky = 0; ky < FK; ++ky)
#pragma unroll
      for (int kx = 0; kx < FK; ++kx) {
        const float* pin = &s_in[((ty + ky) * FH + tx + kx) * FC];
        const float* pw = &s_w[(ky * FK + kx) * FC * 4];
#pragma unroll
        for (int c = 0; c < FC; ++c) {
          const float v = pin[c];
          const float4 wv = *reinterpret_cast<const float4*>(pw + 4 * c);
          a0 += v * wv.x; a1 += v * wv.y; a2 += v * wv.z;
        }
      }
  }
  if (oy >= H || ox >= W) return;
  float o[3] = {a0 + bias3[0], a1 + bias3[1], a2 + bias3[2]};
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = 1.0f / (1.0f + expf(-o[c]));                          // torch.sigmoid (generator.py:164)
  const size_t HWs = (size_t)H * W;
  const size_t obase = (size_t)f * 3 * HWs + (size_t)oy * W + ox;
  if (blend || deformed) {
    const float3 m = motion_at(motion, f, h, w, oy, ox, H, W);
    const Corners cn = grid_corners(m.x, m.y, H, W);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* sp = source + (size_t)c * HWs;
      float s = 0.f;
      if (cn.vnw) s += __ldg(sp + (size_t)cn.y0 * W + cn.x0) * cn.wnw;
      if (cn.vne) s += __ldg(sp + (size_t)cn.y0 * W + cn.x0 + 1) * cn.wne;
      if (cn.vsw) s += __ldg(sp + (size_t)(cn.y0 + 1) * W + cn.x0) * cn.wsw;
      if (cn.vse) s += __ldg(sp + (size_t)(cn.y0 + 1) * W + cn.x0 + 1) * cn.wse;
      if (deformed) deformed[obase + c * HWs] = s;
      if (blend) o[c] = s * m.z + o[c] * (1.f - m.z);                                       // generator.py:166-167
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) prediction[obase + c * HWs] = o[c];
}

// Face_loc_Encoder layer (FD:39-50): out = relu(conv3x3 stride 2, pad 1 (x) + b), planar (C, H, W) tensors, a handful of channels.
// One thread per output element; runs twice per clip on a (1, H, W) mask.
__global__ void conv3x3_s2_relu_kernel(const float* __restrict__ x, int Ci, int H, int W, const float* __restrict__ wgt,
                                       const float* __restrict__ bias, int Co, float* __restrict__ out) {
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;                     // floor((H + 2 - 3) / 2) + 1
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)Co * Ho * Wo) return;
  const int xo = (int)(idx % Wo), yo = (int)((idx / Wo) % Ho), co = (int)(idx / ((long long)Wo * Ho));
  float acc = bias[co];
  for (int ci = 0; ci < Ci; ++ci)
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = 2 * yo + ky - 1;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = 2 * xo + kx - 1;
        if (ix < 0 || ix >= W) continue;
        acc += x[((size_t)ci * H + iy) * W + ix] * wgt[((co * Ci + ci) * 3 + ky) * 3 + kx];
      }
    }
  out[idx] = fmaxf(acc, 0.f);
}

inline int grid_for(long long n, int threads, int cap) {
  long long b = (n + threads - 1) / threads;
  return (int)std::max<long long>(1, std::min<long long>(b, cap));
}

}  // namespace

int launch_lfg_motion_pack(const float* flow, const float* occ, int layout, int F, int h, int w, float4* motion, cudaStream_t st) {
  const long long n = (long long)F * h * w;
  motion_pack_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(flow, occ, layout, F, h * w, motion);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_lfg_warp_blend(const float* skip, int C, int Hs, int Ws, const float4* motion, int F, int h, int w,
                          const float* prev, int ldp, float* out, int ldo, cudaStream_t st) {
  const long long n = (long long)F * Hs * Ws * (C >> 2);
  warp_blend_kernel<<<grid_for(n, 256, 148 * 16), 256, 0, st>>>(skip, C, Hs, Ws, motion, F, h, w, prev, ldp, out, ldo);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_lfg_affine_relu(const float* x, int ldx, const float* scale, const float* shift, int C, long long M, float* z, int ldz,
                           cudaStream_t st) {
  const long long n = M * (C >> 2);
  affine_relu_kernel<<<grid_for(n, 256, 148 * 16), 256, 0, st>>>(x, ldx, scale, shift, C, n, z, ldz);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_lfg_residual_bn_relu(const float* y, const float* x, int C, long long M, float* xnew, const float* scale,
                                const float* shift, float* z, cudaStream_t st) {
  const long long n = M * (C >> 2);
  residual_bn_relu_kernel<<<grid_for(n, 256, 148 * 16), 256, 0, st>>>(y, x, C, n, xnew, scale, shift, z);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_lfg_relu_avgpool2(const float* x, int H, int W, int C, float* out, cudaStream_t st) {
  const long long n = (long long)(H >> 1) * (W >> 1) * (C >> 2);
  relu_avgpool2_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(x, H, W, C, out);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_lfg_chw_to_hwc(const float* x, int C, int HW, int Cpad, float* out, cudaStream_t st) {
  const long long n = (long long)HW * Cpad;
  chw_to_hwc_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(x, C, HW, Cpad, out);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_lfg_hwc_to_chw(const float* x, int ld, int C, long long M, float* out, cudaStream_t st) {
  const long long n = M * C;
  hwc_to_chw_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(x, ld, C, M, out);
  DAWN_LAUNCH_OK();
  return 0;
}
int launch_conv3x3_s2_relu(const float* x, int Ci, int H, int W, const float* wgt, const float* bias, int Co, float* out, cudaStream_t st) {
  const long long n = (long long)Co * ((H + 1) / 2) * ((W + 1) / 2);
  conv3x3_s2_relu_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(x, Ci, H, W, wgt, bias, Co, out);
  DAWN_LAUNCH_OK();
  return 0;
}
std::vector<float> lfg_final_pack(const float* weight, int Cin) {
  std::vector<float> wp((size_t)FK * FK * Cin * 4, 0.f);
  for (int o = 0; o < 3; ++o)
    for (int c = 0; c < Cin; ++c)
      for (int t = 0; t < FK * FK; ++t) wp[((size_t)t * Cin + c) * 4 + o] = weight[((size_t)o * Cin + c) * FK * FK + t];
  return wp;
}
int launch_lfg_final(const float* x, int ldx, int Cin, int F, int H, int W, const float* wpack, const float* bias3,
                     const float* source, const float4* motion, int h, int w, int blend, float* prediction, float* deformed,
                     cudaStream_t st) {
  if (Cin % FC != 0 || (ldx & 3)) { set_last_error("lfg final conv: Cin must be a multiple of 8"); return -1; }
  dim3 grid((W + FT - 1) / FT, (H + FT - 1) / FT, F);
  final_conv_kernel<<<grid, FT * FT, 0, st>>>(x, ldx, Cin, F, H, W, wpack, bias3, source, motion, h, w, blend, prediction, deformed);
  DAWN_LAUNCH_OK();
  return 0;
}

}  // namespace dawn
