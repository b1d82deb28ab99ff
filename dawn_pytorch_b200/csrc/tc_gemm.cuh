// wgmma (Hopper warpgroup MMA) implicit GEMM — see tc_gemm.cu
#pragma once
#include <cuda_runtime.h>
#include <vector>
#include "gemm.cuh"

namespace dawn {

// true when launch_tc_gemm can run this problem (regular shapes, static weights); otherwise use launch_gemm
int tc_tile_n(int N);
bool tc_gemm_supported(const GemmParams& p, int epi);
// host: [K][ldb] fp32 -> pre-scaled, pre-split (fp16 hi | lo), pre-swizzled shared-memory images per (n-tile, k-panel)
size_t tc_pack_weights(const float* Bkn, int K, int N, int ldb, std::vector<float>& out, float* scale);
int launch_tc_gemm(const GemmParams& p, const float* Bimg, int epi, cudaStream_t st);
// halo-tile 3x3 convolution (tc_conv3.cu): same weight image, activations staged once per 64-channel chunk
bool tc_conv3_supported(const GemmParams& p, int epi);
int launch_tc_conv3(const GemmParams& p, const float* Bimg, cudaStream_t st);

}  // namespace dawn
