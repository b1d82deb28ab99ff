// Non-GEMM kernels of the LFG flow decoder (reference LFG/modules/generator.py:59-90, 138-171; util.py:70-150) — see lfg_kernels.cu.
// All activations are channels-last fp32 (frames, H, W, C); the per-clip source features are one frame (H, W, C).
#pragma once
#include <cuda_runtime.h>
#include <vector>

namespace dawn {

// F.grid_sample(mode='bilinear', padding_mode='zeros', align_corners=False): corner indices, weights and validity (shared with
// the motion estimator's sparse-motion sampling, lfg_motion_kernels.cu)
struct Corners { int x0, y0; float wnw, wne, wsw, wse; bool vnw, vne, vsw, vse; };
__device__ __forceinline__ Corners grid_corners(float gx, float gy, int H, int W) {
  const float ix = ((gx + 1.f) * (float)W - 1.f) * 0.5f;
  const float iy = ((gy + 1.f) * (float)H - 1.f) * 0.5f;
  const float fx = floorf(ix), fy = floorf(iy);
  Corners c;
  // float -> int conversion saturates; far-away samples are simply invalid
  c.x0 = (int)fminf(fmaxf(fx, -2.f), (float)W + 1.f);
  c.y0 = (int)fminf(fmaxf(fy, -2.f), (float)H + 1.f);
  const float ex = (fx + 1.f) - ix, ey = (fy + 1.f) - iy;        // (ix_se - ix), (iy_se - iy)
  const float dx = ix - fx, dy = iy - fy;
  c.wnw = ex * ey; c.wne = dx * ey; c.wsw = ex * dy; c.wse = dx * dy;
  const bool inx0 = (fx >= 0.f) && (fx <= (float)(W - 1)), inx1 = (fx + 1.f >= 0.f) && (fx + 1.f <= (float)(W - 1));
  const bool iny0 = (fy >= 0.f) && (fy <= (float)(H - 1)), iny1 = (fy + 1.f >= 0.f) && (fy + 1.f <= (float)(H - 1));
  c.vnw = inx0 && iny0; c.vne = inx1 && iny0; c.vsw = inx0 && iny1; c.vse = inx1 && iny1;
  return c;
}

// motion[f][y][x] = (grid_x, grid_y, occlusion, 0).
// layout 0: flow (F, h, w, 2) + occ (F, 1, h, w)                              (forward_with_flow's arguments, generator.py:138)
// layout 1: sample (3, F, h, w) = [grid_x, grid_y, conf]; occlusion = (conf + 1) / 2   (sample_one_video, FD:366-369)
int launch_lfg_motion_pack(const float* flow, const float* occ, int layout, int F, int h, int w, float4* motion, cudaStream_t st);

// apply_optical (generator.py:71-90) on a C-channel level of size (Hs, Ws):
//   out[f] = grid_sample(skip, resize(flow_f)) * resize(occ_f) + prev[f] * (1 - resize(occ_f))      (prev may be null)
// resize = bilinear, align_corners=False (identity when the sizes match); grid_sample = bilinear, zeros, align_corners=False.
int launch_lfg_warp_blend(const float* skip, int C, int Hs, int Ws, const float4* motion, int F, int h, int w,
                          const float* prev, int ldp, float* out, int ldo, cudaStream_t st);

// z = relu(x * scale[c] + shift[c])  (eval-mode BatchNorm + ReLU, util.py:86-87); scale == null: z = relu(x).  In place allowed.
int launch_lfg_affine_relu(const float* x, int ldx, const float* scale, const float* shift, int C, long long M, float* z, int ldz,
                           cudaStream_t st);
// xnew = y + x (ResBlock2d's `out += x`, util.py:92) and, when z != null, z = relu(xnew * scale + shift) for the next block
int launch_lfg_residual_bn_relu(const float* y, const float* x, int C, long long M, float* xnew, const float* scale,
                                const float* shift, float* z, cudaStream_t st);
// 2x2 average pooling (util.py:124, 131) with ReLU applied to the inputs first: out = avgpool(relu(x)); one frame
int launch_lfg_relu_avgpool2(const float* x, int H, int W, int C, float* out, cudaStream_t st);
// (C, H, W) -> (H, W, Cpad) channels-last, zero padded; and back: (M, C) rows -> (C, M)
int launch_lfg_chw_to_hwc(const float* x, int C, int HW, int Cpad, float* out, cudaStream_t st);
int launch_lfg_hwc_to_chw(const float* x, int ld, int C, long long M, float* out, cudaStream_t st);

// out (Co, ceil(H/2), ceil(W/2)) = relu(conv3x3 stride 2 pad 1 of x (Ci, H, W) + bias); wgt (Co, Ci, 3, 3) as nn.Conv2d stores it
int launch_conv3x3_s2_relu(const float* x, int Ci, int H, int W, const float* wgt, const float* bias, int Co, float* out, cudaStream_t st);

// final 7x7 conv (Cin -> 3) + sigmoid + the last apply_optical with the source image (generator.py:163-167):
//   prediction[f] = grid_sample(source, flow_f^) * occ_f^ + sigmoid(conv(x_f)) * (1 - occ_f^)     written as (F, 3, H, W)
//   deformed[f]   = grid_sample(source, flow_f^)                                                  (optional, generator.py:152)
// x: (F, H, W, Cin) channels-last; wpack: [49][Cin][4] (3 outputs + pad), lfg_final_pack of the (3, Cin, 7, 7) Conv2d weight;
// source: (3, H, W) planar.
std::vector<float> lfg_final_pack(const float* weight, int Cin);
int launch_lfg_final(const float* x, int ldx, int Cin, int F, int H, int W, const float* wpack, const float* bias3,
                     const float* source, const float4* motion, int h, int w, int blend, float* prediction, float* deformed,
                     cudaStream_t st);

}  // namespace dawn
