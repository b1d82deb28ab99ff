// Host side of every contraction of the UNet and the LFG decoder (contraction.cu): the host-parameter store and device
// allocations, packed weight matrices with their wgmma images, GemmParams builders, the choice among the kernel paths
// (DAWN_PATH_* in include/dawn_unet.h) and their launch, and the 2x upsampling conv.
#pragma once
#include <cstdint>
#include <functional>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/dawn_unet.h"
#include "gemm.cuh"

namespace dawn {

// ---------------------------------------------------------------- host parameters and device allocations
struct HostParam {
  std::vector<float> data;
  std::vector<int64_t> shape;
};
struct HostParams {
  std::unordered_map<std::string, HostParam> map;
  std::string prefix;          // starts every error message
  void set(const std::string& name, const float* data, const int64_t* shape, int ndim);
  // *out = the parameter `name`; -1 when it is missing or its shape is not `shape`
  int need(const std::string& name, const std::vector<int64_t>& shape, const HostParam** out) const;
};

int dev_alloc(std::vector<void*>& owner, size_t nfloats, float** out, int64_t* counter = nullptr);
int dev_upload(std::vector<void*>& owner, const std::vector<float>& v, float** out);
int dev_upload(std::vector<void*>& owner, const std::vector<uint16_t>& v, uint16_t** out);   // fp16 images of the fused kernels
void free_all(std::vector<void*>& v);
inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// ---------------------------------------------------------------- packed weights
// B operand of a contraction: fp32 [K][ldb] (ldb a multiple of 64, zero padded), optional bias [ldb], and when N and K are
// multiples of 64 the wgmma image (tc_pack_weights) with the power-of-two scale it was built with
struct PackedWeight {
  float* w = nullptr; float* b = nullptr; float* img = nullptr; float img_scale = 1.f;
  int K = 0, N = 0, ldb = 0;
};
int upload_weight(std::vector<void*>& owner, const std::vector<float>& m, int K, int N, int ldb, const std::vector<float>& bias,
                  PackedWeight* out);

// ---------------------------------------------------------------- GemmParams
// 1x1 contraction of (frames, H, W, Cin) rows of stride lda onto the same grid
void base_params(GemmParams& p, const float* A, int lda, int Cin, int frames, int H, int W);
void set_weights(GemmParams& p, const PackedWeight& w);       // the only place that sets B, Bimg, tc_scale, ldb, N, K, bias
void set_square_taps(GemmParams& p, int k, int pad);

// ---------------------------------------------------------------- kernel paths
// can `path` run p?  scratch_bytes: room for the fp16 planes of A when the path needs a split pass (A16h not set by a producer)
bool path_ok(const GemmParams& p, int epi, int path, size_t scratch_bytes);
// the path the networks take: halo conv, else wgmma GEMM (pre-split when it pays and the planes fit), else mma.sync
int choose_path(const GemmParams& p, int epi, size_t scratch_bytes);
// enqueues `path` (the split pass first when it needs one, into scratch); *kernels = kernels enqueued (1, or 2 with the split)
int launch_path(const GemmParams& p, int epi, int path, void* scratch, cudaStream_t st, int* kernels = nullptr);

// ---------------------------------------------------------------- 2x upsampling conv
// On the low-resolution grid, output pixel (2y + py, 2x + px) is a 2x2 conv of parity class (py, px): tap (ty, tx) reads input
// offset (off[py][ty], off[px][tx]).  When co == 64 and ci % 64 == 0, `all` holds the four classes as one 3x3 conv with 4 x co
// output columns (the halo conv's up2 epilogue); taps a class does not use stay zero.
struct UpConv {
  PackedWeight cls[4], all;
  int off[2][2];
};
using UpWeight = std::function<float(int py, int px, int ty, int tx, int c, int n)>;   // weight of class tap (ty, tx), c -> n
int pack_up(std::vector<void*>& owner, int ci, int co, const int (&off)[2][2], const std::vector<float>& bias, const UpWeight& weight,
            UpConv* u);
// in: base_params of the low-resolution input; out: (frames, 2H, 2W) rows of stride ldo.  run launches one contraction: once with
// the up2 halo conv when that path takes it, otherwise once per parity class.
int run_up(const GemmParams& in, const UpConv& u, float* out, int ldo, const std::function<int(const GemmParams&)>& run);

}  // namespace dawn
