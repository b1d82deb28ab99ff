// dawn_lfg_test_kernel (include/dawn_lfg.h): one non-GEMM kernel of the LFG flow decoder on caller-owned buffers, for per-kernel
// tests against a high-precision reference.  The final conv's weight goes through lfg_final_pack, as dawn_lfg_commit_params does.
#include <string>
#include <vector>

#include "../../include/dawn_lfg.h"
#include "common.cuh"
#include "contraction.cuh"
#include "lfg_kernels.cuh"

namespace dawn {
namespace {

int refuse(const char* why) {
  set_last_error(std::string("dawn_lfg_test_kernel: ") + why);
  return -1;
}

struct Owned {
  std::vector<void*> v;
  ~Owned() { free_all(v); }
};

// a channels-last row stride the float4 kernels can take
bool row_ok(int ld, int C) { return C >= 4 && (C & 3) == 0 && ld >= C && (ld & 3) == 0; }

int test_kernel(const dawn_lfg_kernel_case& c, Owned& own, cudaStream_t st) {
  const float4* motion = reinterpret_cast<const float4*>(c.motion);
  switch (c.kernel) {
    case DAWN_LFG_MOTION_PACK:
      if (!c.flow || !c.out || (c.layout == 0 && !c.occ)) return refuse("missing pointer");
      if (c.F < 1 || c.h < 1 || c.w < 1 || (c.layout != 0 && c.layout != 1)) return refuse("bad geometry");
      return launch_lfg_motion_pack(c.flow, c.occ, c.layout, c.F, c.h, c.w, reinterpret_cast<float4*>(c.out), st);
    case DAWN_LFG_WARP_BLEND:
      if (!c.x || !c.motion || !c.out) return refuse("missing pointer");
      if (c.F < 1 || c.H < 1 || c.W < 1 || c.h < 1 || c.w < 1 || !row_ok(c.ldo, c.C) || (c.prev && !row_ok(c.ldp, c.C)))
        return refuse("bad geometry");
      return launch_lfg_warp_blend(c.x, c.C, c.H, c.W, motion, c.F, c.h, c.w, c.prev, c.ldp, c.out, c.ldo, st);
    case DAWN_LFG_AFFINE_RELU:
      if (!c.x || !c.out || (c.scale == nullptr) != (c.shift == nullptr)) return refuse("missing pointer");
      if (c.M < 1 || !row_ok(c.ldx, c.C) || !row_ok(c.ldo, c.C)) return refuse("bad geometry");
      return launch_lfg_affine_relu(c.x, c.ldx, c.scale, c.shift, c.C, c.M, c.out, c.ldo, st);
    case DAWN_LFG_RESIDUAL_BN_RELU:
      if (!c.x || !c.y || !c.out || (c.out2 && (!c.scale || !c.shift))) return refuse("missing pointer");
      if (c.M < 1 || !row_ok(c.C, c.C)) return refuse("bad geometry");
      return launch_lfg_residual_bn_relu(c.y, c.x, c.C, c.M, c.out, c.scale, c.shift, c.out2, st);
    case DAWN_LFG_RELU_AVGPOOL2:
      if (!c.x || !c.out) return refuse("missing pointer");
      if (c.H < 2 || c.W < 2 || !row_ok(c.C, c.C)) return refuse("bad geometry");
      return launch_lfg_relu_avgpool2(c.x, c.H, c.W, c.C, c.out, st);
    case DAWN_LFG_CHW_TO_HWC:
      if (!c.x || !c.out) return refuse("missing pointer");
      if (c.C < 1 || c.H < 1 || c.W < 1 || c.Cpad < c.C) return refuse("bad geometry");
      return launch_lfg_chw_to_hwc(c.x, c.C, c.H * c.W, c.Cpad, c.out, st);
    case DAWN_LFG_HWC_TO_CHW:
      if (!c.x || !c.out) return refuse("missing pointer");
      if (c.C < 1 || c.M < 1 || c.ldx < c.C) return refuse("bad geometry");
      return launch_lfg_hwc_to_chw(c.x, c.ldx, c.C, c.M, c.out, st);
    case DAWN_LFG_FINAL_CONV: {
      if (!c.x || !c.weight || !c.bias || !c.out || ((c.blend || c.out2) && (!c.source || !c.motion))) return refuse("missing pointer");
      if (c.F < 1 || c.H < 1 || c.W < 1 || c.h < 1 || c.w < 1 || c.C % 8 != 0 || !row_ok(c.ldx, c.C)) return refuse("bad geometry");
      std::vector<float> w((size_t)3 * c.C * 49);
      DAWN_CUDA_OK(cudaMemcpy(w.data(), c.weight, w.size() * sizeof(float), cudaMemcpyDeviceToHost));
      float* wp;
      DAWN_TRY(dev_upload(own.v, lfg_final_pack(w.data(), c.C), &wp));
      return launch_lfg_final(c.x, c.ldx, c.C, c.F, c.H, c.W, wp, c.bias, c.source, motion, c.h, c.w, c.blend, c.out, c.out2, st);
    }
  }
  return refuse("unknown kernel");
}

}  // namespace
}  // namespace dawn

extern "C" int dawn_lfg_test_kernel(const dawn_lfg_kernel_case* c, void* stream) {
  if (!c) return dawn::refuse("null case");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  dawn::Owned own;
  const int rc = dawn::test_kernel(*c, own, st);
  if (rc != 0) return rc;
  DAWN_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}
