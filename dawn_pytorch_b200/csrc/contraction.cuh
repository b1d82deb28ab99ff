// Host side of every contraction of the UNet and the LFG networks (contraction.cu): the host-parameter store and device
// allocations, packed weight matrices with their wgmma images, the linear, BatchNorm and conv weight folds, GemmParams builders,
// the choice among the kernel paths (DAWN_PATH_* in include/dawn_unet.h) and their launch, and the 2x upsampling conv with the
// nearest-upsample fold.
#pragma once
#include <cstdint>
#include <functional>
#include <memory>
#include <string>
#include <unordered_map>
#include <utility>
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

// Owner of device allocations: every block is its own cudaMalloc of at least 16 bytes, freed by release() or the destructor.
// bytes() counts this arena's blocks; live_bytes() counts the blocks of every arena in the process.
class DeviceArena {
 public:
  DeviceArena() = default;
  DeviceArena(const DeviceArena&) = delete;
  DeviceArena& operator=(const DeviceArena&) = delete;
  ~DeviceArena() { release(); }

  template <class T>
  int alloc(size_t count, T** out) {
    void* p = nullptr;
    const int rc = alloc_bytes(count * sizeof(T), &p);
    *out = static_cast<T*>(p);
    return rc;
  }
  // a block holding v (fp32 weights, fp16 images of the fused kernels)
  template <class T>
  int upload(const std::vector<T>& v, T** out) {
    const int rc = alloc(v.size(), out);
    return rc != 0 ? rc : copy_in(*out, v.data(), v.size() * sizeof(T));
  }
  void release();
  int64_t bytes() const { return bytes_; }
  static int64_t live_bytes();

 private:
  struct Free { void operator()(void* p) const { cudaFree(p); } };
  int alloc_bytes(size_t bytes, void** out);
  static int copy_in(void* dst, const void* src, size_t bytes);
  std::vector<std::unique_ptr<void, Free>> blocks_;
  int64_t bytes_ = 0;
};
inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// ---------------------------------------------------------------- packed weights
// B operand of a contraction: fp32 [K][ldb] (ldb a multiple of 64, zero padded), optional bias [ldb], and when N and K are
// multiples of 64 the wgmma image (tc_pack_weights) with the power-of-two scale it was built with
struct PackedWeight {
  float* w = nullptr; float* b = nullptr; float* img = nullptr; float img_scale = 1.f;
  int K = 0, N = 0, ldb = 0;
};
int upload_weight(DeviceArena& arena, const std::vector<float>& m, int K, int N, int ldb, const std::vector<float>& bias,
                  PackedWeight* out);

// Folds shared by the network's weight upload and dawn_test_fused.  Linear weight w [N][K] (row-major) with a per-input gain
// (a LayerNorm gamma, may be null) folded into its columns and rows [0, nscale) scaled by qscale: (w[n][k] * gain[k]) * sc.
std::vector<float> fold_linear(const float* w, int N, int K, const float* gain, float qscale, int nscale);
// per-row sums of a folded [N][K] matrix (fp64 accumulation): the column sums of B that the LayerNorm fold subtracts
std::vector<float> row_sums(const std::vector<float>& w, int N, int K);
// the three cross-attentions' to_q [64][ci] with their LayerNorm_img gains folded, as one k-major [ci][192] matrix and its wsum
void fold_ca_q(const float* const to_q[3], const float* const gain[3], int ci, std::vector<float>& wq, std::vector<float>& wsum);

// eval-mode BatchNorm `prefix` (weight, bias, running_mean, running_var; c channels) as y = x s + t with eps 1e-5, in fp64
// (LFG sync_batchnorm/batchnorm.py:50-53: F.batch_norm with the running statistics)
int bn_affine(const HostParams& raw, const std::string& prefix, int c, std::vector<double>& s, std::vector<double>& t);
// conv weight w (co, ci, taps) -> m[(tap ci_pad + c) ldb + n0 + n] = w[n][c][tap] * scale[n], rounded once (scale null: a copy)
void pack_conv_taps(const float* w, int co, int ci, int taps, int ci_pad, int ldb, int n0, const double* scale, std::vector<float>& m);
// The LFG networks' Conv2d weights (co_j, ci, k, k) and biases of `convs` (state_dict prefix, co_j), side by side in the output
// columns, with the BatchNorm `bn_after` (none when empty) folded in: W' = W s, b' = b s + t.  Input channels ci..ci_pad stay zero.
int pack_lfg_conv(const HostParams& raw, DeviceArena& arena, const std::vector<std::pair<std::string, int>>& convs,
                  const std::string& bn_after, int ci, int k, int ci_pad, PackedWeight* out);

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
// Nearest x2 followed by a 3x3 conv (padding 1) on the low-resolution grid: parity p's tap t reads offset kUpOff[p][t] and its
// weight is the sum of the kernel indices k with up_in_set(p, t, k), i.e. p = 0: {-1 <- k0, 0 <- k1 + k2}, p = 1: {0 <- k0 + k1,
// +1 <- k2}.  Zero padding is the same on both grids (upsampled index -1 / 2H <-> low-resolution index -1 / H).
constexpr int kUpOff[2][2] = {{-1, 0}, {0, 1}};
inline bool up_in_set(int parity, int tap, int k) { return parity == 0 ? (tap == 0 ? k == 0 : k >= 1) : (tap == 0 ? k <= 1 : k == 2); }
int pack_up(DeviceArena& arena, int ci, int co, const int (&off)[2][2], const std::vector<float>& bias, const UpWeight& weight,
            UpConv* u);
// nearest x2 -> 3x3 conv with weight w (co, ci, 3, 3) [times scale[n]] as the parity classes above: each class tap is the sum of
// the 3x3 taps it covers, summed in fp64 and rounded once (scale null: no scale)
int pack_up_nearest(DeviceArena& arena, const float* w, int ci, int co, const double* scale, const std::vector<float>& bias,
                    UpConv* u);
// the LFG networks' UpBlock2d `name` (util.py:106-111): nearest x2 -> conv3x3 (name.conv) -> BatchNorm (name.norm) folded
int pack_lfg_up(const HostParams& raw, DeviceArena& arena, const std::string& name, int co, int ci, UpConv* u);
// in: base_params of the low-resolution input; out: (frames, 2H, 2W) rows of stride ldo.  run launches one contraction: once with
// the up2 halo conv when that path takes it, otherwise once per parity class.  border = 1: `in` reads a grid that carries a
// one-pixel border (IH = OHs + 2, IW = OWs + 2); the classes then run as valid 2x2 convs over it, so no tap leaves the grid.
int run_up(const GemmParams& in, const UpConv& u, float* out, int ldo, const std::function<int(const GemmParams&)>& run,
           int border = 0);

}  // namespace dawn
