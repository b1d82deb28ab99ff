// Non-GEMM kernels of the LFG motion estimator (RegionPredictor, BGMotionPredictor, PixelwiseFlowPredictor) — see
// lfg_motion_kernels.cu.  Activations are channels-last fp32 (frames, h, w, ld); R = num_regions.
#pragma once
#include <cuda_runtime.h>

namespace dawn {

constexpr int kMotionMaxRegions = 16;
constexpr int kAAK = 13;                 // AntiAliasInterpolation2d kernel at scale 0.25 (sigma 1.5): 13 x 13, zero pad 6

// AntiAliasInterpolation2d (util.py:254-264) at scale 1/4, evaluated only at the kept pixels: images (N, 3, H, W) planar ->
// out (N, H/4, W/4, ld) channels [off, off + cw): the 3 filtered channels, then zeros.  weight (3, 13, 13).
int launch_lfgm_aa_down(const float* images, int N, int H, int W, const float* weight, float* out, int ld, int off, int cw,
                        cudaStream_t st);
// region_predictor.py:97-104 + region2affine (:60-75): one CTA per (frame, region).  softmax over h w of logits / temperature,
// then shift = sum heat g and covar = sum heat (g - shift)(g - shift)^T (fp64 sums).  logits (N, h, w, ldl), first R columns.
int launch_lfgm_region_moments(const float* logits, int ldl, int N, int h, int w, int R, float temperature, float* shift,
                               float* covar, float* heatmap, cudaStream_t st);
// the flow predictor's input (pixelwise_flow_predictor.py:51-109, 116-121) in one pass: per (frame, region) the 2x2 algebra
// (covariance inverses, A_s inv(A_d), axis-swap sign), per pixel the Gaussian differences, the R + 1 sparse-motion grids and
// bilinear samples of source4 (h, w, 4).  out (N, h, w, ld) channels [off, off + cw) in the reference's (R + 1, 1 + 3) order,
// zero padded; motion (N, h, w, 2 (R + 1)), background grid first.  bg (N, 3, 3) or null (identity background grid).
int launch_lfgm_flow_input(const float* source4, int N, int h, int w, int R, const float* src_shift, const float* src_covar,
                           const float* src_affine, const float* drv_shift, const float* drv_covar, const float* drv_affine,
                           const float* bg, int revert, float* out, int ld, int off, int cw, float* motion, cudaStream_t st);
// pixelwise_flow_predictor.py:125-135: columns 0..R of logits = mask, column R + 1 = occlusion:
// flow = sum_k softmax(mask)_k motion_k -> (N, h, w, 2); occlusion = sigmoid -> (N, 1, h, w)
int launch_lfgm_flow_combine(const float* logits, int ldl, const float* motion, int N, int h, int w, int R, float* flow,
                             float* occlusion, cudaStream_t st);
// bg_motion_predictor.py:49-55: spatial mean of x (N, P, ld) over P, fc (6, C) -> rows 0-1 of bg (N, 3, 3), row 2 = (0, 0, 1);
// fc_w == null: identity ('zero')
int launch_lfgm_bg_head(const float* x, int ld, int C, int N, int P, const float* fc_w, const float* fc_b, float* bg, cudaStream_t st);

// BGMotionPredictor's input cat([source, driving]) (N, 6, H, W) as (N, H, W, 32) zero padded; n_source 1 shares one source
int launch_lfgm_pack_pair(const float* source, int n_source, const float* driving, int N, int HW, float* out, cudaStream_t st);

}  // namespace dawn
