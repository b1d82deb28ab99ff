// Pixel stages of the video generator outside the networks (include/dawn_video.h): the portrait resize of
// unified_video_generator.py:320-325, 372 as Pillow's 8-bit bilinear resampler computes it, fused with ToTensor / * 255 / / 255.
#include <cmath>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/dawn_video.h"
#include "common.cuh"

namespace dawn {
namespace {

constexpr int kPrecisionBits = 32 - 8 - 2;      // Pillow's fixed-point coefficients for 8-bit images
constexpr int kMaxSide = 8192;

// One axis of Pillow's bilinear resampling from `in` to `out` samples (support 1, widened by the reduction factor when
// downscaling): for each output sample the first input sample `bounds[2 i]`, the tap count `bounds[2 i + 1]`, and `ksize`
// normalised weights in int32 fixed point with kPrecisionBits fractional bits, rounded half away from zero.
struct AxisCoeffs {
  int ksize = 0;
  std::vector<int> bounds, k;
};

AxisCoeffs axis_coeffs(int in, int out) {
  AxisCoeffs a;
  const double scale = (double)in / out;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 1.0 * filterscale;
  a.ksize = (int)std::ceil(support) * 2 + 1;
  a.bounds.assign(2 * (size_t)out, 0);
  a.k.assign((size_t)out * a.ksize, 0);
  std::vector<double> w(a.ksize);
  for (int i = 0; i < out; ++i) {
    const double center = (i + 0.5) * scale, ss = 1.0 / filterscale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in) xmax = in;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      double t = std::fabs((x + xmin - center + 0.5) * ss);
      w[x] = t < 1.0 ? 1.0 - t : 0.0;
      ww += w[x];
    }
    for (int x = 0; x < xmax; ++x) {
      const double v = ww != 0.0 ? w[x] / ww : w[x];
      a.k[(size_t)i * a.ksize + x] = v < 0 ? (int)(-0.5 + v * (1 << kPrecisionBits)) : (int)(0.5 + v * (1 << kPrecisionBits));
    }
    a.bounds[2 * i] = xmin;
    a.bounds[2 * i + 1] = xmax;
  }
  return a;
}

__device__ __forceinline__ uint8_t clip8(int v) {
  return v <= 0 ? 0 : (v >> kPrecisionBits) >= 255 ? 255 : (uint8_t)(v >> kPrecisionBits);
}

// horizontal pass over input rows [row0, row0 + rows): (rows, S, 3) uint8, one thread per output pixel
__global__ void resize_h_kernel(const uint8_t* __restrict__ img, int W0, int row0, int rows, int S, const int* __restrict__ bounds,
                                const int* __restrict__ k, int ksize, uint8_t* __restrict__ tmp) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)rows * S) return;
  const int xx = (int)(idx % S), r = (int)(idx / S);
  const int xmin = bounds[2 * xx], n = bounds[2 * xx + 1];
  const int* kk = k + (size_t)xx * ksize;
  const uint8_t* src = img + ((size_t)(row0 + r) * W0 + xmin) * 3;
  int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
  for (int x = 0; x < n; ++x) {
    const int w = kk[x];
    s0 += src[3 * x] * w; s1 += src[3 * x + 1] * w; s2 += src[3 * x + 2] * w;
  }
  uint8_t* o = tmp + (size_t)idx * 3;
  o[0] = clip8(s0); o[1] = clip8(s1); o[2] = clip8(s2);
}

// vertical pass (bounds == null: the axis keeps its size, u = tmp) fused with ToTensor, * 255 and / 255 (UVG:323-325, 372):
// tmp (rows, S, 3) uint8 -> source (3, S, S) fp32 and resized (S, S, 3) uint8 (or null)
__global__ void resize_v_scale_kernel(const uint8_t* __restrict__ tmp, int S, const int* __restrict__ bounds, const int* __restrict__ k,
                                      int ksize, float* __restrict__ source, uint8_t* __restrict__ resized) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)S * S) return;
  const int xx = (int)(idx % S), yy = (int)(idx / S);
  uint8_t u[3];
  if (bounds) {
    const int ymin = bounds[2 * yy], n = bounds[2 * yy + 1];
    const int* kk = k + (size_t)yy * ksize;
    int s[3] = {1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1)};
    for (int y = 0; y < n; ++y) {
      const uint8_t* p = tmp + ((size_t)(ymin + y) * S + xx) * 3;
      const int w = kk[y];
      s[0] += p[0] * w; s[1] += p[1] * w; s[2] += p[2] * w;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) u[c] = clip8(s[c]);
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) u[c] = tmp[(size_t)idx * 3 + c];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    // ToTensor: float(u).div(255); UVG:325: * 255; UVG:372: / 255. — three fp32 roundings, none contracted
    source[(size_t)c * S * S + idx] = __fdiv_rn(__fmul_rn(__fdiv_rn((float)u[c], 255.f), 255.f), 255.f);
    if (resized) resized[(size_t)idx * 3 + c] = u[c];
  }
}

int blocks_for(long long n) { return (int)((n + 255) / 256); }

}  // namespace
}  // namespace dawn

using namespace dawn;

extern "C" int dawn_portrait_resize(const uint8_t* img, int H0, int W0, int S, float* source, uint8_t* resized, void* stream) {
  DAWN_CHECK(H0 >= 1 && W0 >= 1 && H0 <= kMaxSide && W0 <= kMaxSide,
             "dawn_portrait_resize: the image must be 1 to 8192 pixels on a side, got " + std::to_string(H0) + "x" + std::to_string(W0));
  DAWN_CHECK(S >= 1 && S <= kMaxSide, "dawn_portrait_resize: the output side must be 1 to 8192, got " + std::to_string(S));
  DAWN_CHECK(img && source, "dawn_portrait_resize: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const bool need_h = W0 != S, need_v = H0 != S;
  AxisCoeffs ch, cv;
  int row0 = 0, rows = H0;
  if (need_h) ch = axis_coeffs(W0, S);
  if (need_v) {
    cv = axis_coeffs(H0, S);
    row0 = cv.bounds[0];                                                // first and last input rows the vertical pass reads
    rows = cv.bounds[2 * (S - 1)] + cv.bounds[2 * (S - 1) + 1] - row0;
    if (need_h)
      for (int i = 0; i < S; ++i) cv.bounds[2 * i] -= row0;             // it reads the horizontal pass's rows
  }
  // one table: horizontal bounds + weights, vertical bounds + weights
  std::vector<int> table;
  table.insert(table.end(), ch.bounds.begin(), ch.bounds.end());
  table.insert(table.end(), ch.k.begin(), ch.k.end());
  table.insert(table.end(), cv.bounds.begin(), cv.bounds.end());
  table.insert(table.end(), cv.k.begin(), cv.k.end());
  int* dtab = nullptr;
  uint8_t* tmp = nullptr;
  if (!table.empty()) {
    DAWN_CUDA_OK(cudaMallocAsync((void**)&dtab, table.size() * sizeof(int), st));
    // pageable source: the call returns once the table is staged, so `table` may go out of scope
    const cudaError_t e = cudaMemcpyAsync(dtab, table.data(), table.size() * sizeof(int), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) { cudaFreeAsync(dtab, st); DAWN_CUDA_OK(e); }
  }
  const int* hb = dtab;
  const int* hk = hb + ch.bounds.size();
  const int* vb = hk + ch.k.size();
  const int* vk = vb + cv.bounds.size();
  int rc = 0;
  const uint8_t* vin = img;
  if (need_h) {
    cudaError_t e = cudaMallocAsync((void**)&tmp, (size_t)rows * S * 3, st);
    if (e == cudaSuccess) {
      resize_h_kernel<<<blocks_for((long long)rows * S), 256, 0, st>>>(img, W0, row0, rows, S, hb, hk, ch.ksize, tmp);
      e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_last_error(std::string("dawn_portrait_resize: ") + cudaGetErrorString(e)); rc = -2; }
    vin = tmp;
  }
  if (rc == 0) {
    resize_v_scale_kernel<<<blocks_for((long long)S * S), 256, 0, st>>>(vin, S, need_v ? vb : nullptr, vk, cv.ksize, source, resized);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_last_error(std::string("dawn_portrait_resize: ") + cudaGetErrorString(e)); rc = -2; }
  }
  if (tmp) cudaFreeAsync(tmp, st);
  if (dtab) cudaFreeAsync(dtab, st);
  return rc;
}
