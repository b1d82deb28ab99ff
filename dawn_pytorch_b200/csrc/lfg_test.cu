// dawn_lfg_test_kernel and dawn_lfg_motion_test_kernel (include/dawn_lfg.h): one non-GEMM kernel of the LFG flow decoder or of
// the motion estimator on caller-owned buffers, for per-kernel tests against a high-precision reference.  The final conv's weight
// goes through lfg_final_pack, as dawn_lfg_commit_params does.
#include <string>
#include <vector>

#include "../../include/dawn_lfg.h"
#include "common.cuh"
#include "contraction.cuh"
#include "lfg_kernels.cuh"
#include "lfg_motion_kernels.cuh"

namespace dawn {
namespace {

constexpr const char* kLfg = "dawn_lfg_test_kernel";
constexpr const char* kMotion = "dawn_lfg_motion_test_kernel";

int refuse(const char* entry, const char* why) {
  set_last_error(std::string(entry) + ": " + why);
  return -1;
}

// a channels-last row stride the float4 kernels can take
bool row_ok(int ld, int C) { return C >= 4 && (C & 3) == 0 && ld >= C && (ld & 3) == 0; }

int test_kernel(const dawn_lfg_kernel_case& c, DeviceArena& arena, cudaStream_t st) {
  const float4* motion = reinterpret_cast<const float4*>(c.motion);
  switch (c.kernel) {
    case DAWN_LFG_MOTION_PACK:
      if (!c.flow || !c.out || (c.layout == 0 && !c.occ)) return refuse(kLfg, "missing pointer");
      if (c.F < 1 || c.h < 1 || c.w < 1 || (c.layout != 0 && c.layout != 1)) return refuse(kLfg, "bad geometry");
      return launch_lfg_motion_pack(c.flow, c.occ, c.layout, c.F, c.h, c.w, reinterpret_cast<float4*>(c.out), st);
    case DAWN_LFG_WARP_BLEND:
      if (!c.x || !c.motion || !c.out) return refuse(kLfg, "missing pointer");
      if (c.F < 1 || c.H < 1 || c.W < 1 || c.h < 1 || c.w < 1 || !row_ok(c.ldo, c.C) || (c.prev && !row_ok(c.ldp, c.C)))
        return refuse(kLfg, "bad geometry");
      return launch_lfg_warp_blend(c.x, c.C, c.H, c.W, motion, c.F, c.h, c.w, c.prev, c.ldp, c.out, c.ldo, st);
    case DAWN_LFG_AFFINE_RELU:
      if (!c.x || !c.out || (c.scale == nullptr) != (c.shift == nullptr)) return refuse(kLfg, "missing pointer");
      if (c.M < 1 || !row_ok(c.ldx, c.C) || !row_ok(c.ldo, c.C)) return refuse(kLfg, "bad geometry");
      return launch_lfg_affine_relu(c.x, c.ldx, c.scale, c.shift, c.C, c.M, c.out, c.ldo, st);
    case DAWN_LFG_RESIDUAL_BN_RELU:
      if (!c.x || !c.y || !c.out || (c.out2 && (!c.scale || !c.shift))) return refuse(kLfg, "missing pointer");
      if (c.M < 1 || !row_ok(c.C, c.C)) return refuse(kLfg, "bad geometry");
      return launch_lfg_residual_bn_relu(c.y, c.x, c.C, c.M, c.out, c.scale, c.shift, c.out2, st);
    case DAWN_LFG_RELU_AVGPOOL2: {
      const int ldo = c.ldo ? c.ldo : c.C;                                   // 0: dense output rows
      if (!c.x || !c.out) return refuse(kLfg, "missing pointer");
      if (c.H < 2 || c.W < 2 || !row_ok(ldo, c.C)) return refuse(kLfg, "bad geometry");
      return launch_lfg_relu_avgpool2(c.x, c.H, c.W, c.C, c.out, ldo, st);
    }
    case DAWN_LFG_CHW_TO_HWC:
      if (!c.x || !c.out) return refuse(kLfg, "missing pointer");
      if (c.C < 1 || c.H < 1 || c.W < 1 || c.Cpad < c.C) return refuse(kLfg, "bad geometry");
      return launch_lfg_chw_to_hwc(c.x, c.C, c.H * c.W, c.Cpad, c.out, st);
    case DAWN_LFG_HWC_TO_CHW:
      if (!c.x || !c.out) return refuse(kLfg, "missing pointer");
      if (c.C < 1 || c.M < 1 || c.ldx < c.C) return refuse(kLfg, "bad geometry");
      return launch_lfg_hwc_to_chw(c.x, c.ldx, c.C, c.M, c.out, st);
    case DAWN_LFG_FINAL_CONV: {
      if (!c.x || !c.weight || !c.bias || !c.out || ((c.blend || c.out2) && (!c.source || !c.motion))) return refuse(kLfg, "missing pointer");
      if (c.F < 1 || c.H < 1 || c.W < 1 || c.h < 1 || c.w < 1 || c.C % 8 != 0 || !row_ok(c.ldx, c.C)) return refuse(kLfg, "bad geometry");
      std::vector<float> w((size_t)3 * c.C * 49);
      DAWN_CUDA_OK(cudaMemcpy(w.data(), c.weight, w.size() * sizeof(float), cudaMemcpyDeviceToHost));
      float* wp;
      DAWN_TRY(arena.upload(lfg_final_pack(w.data(), c.C), &wp));
      return launch_lfg_final(c.x, c.ldx, c.C, c.F, c.H, c.W, wp, c.bias, c.source, motion, c.h, c.w, c.blend, c.out, c.out2, st);
    }
  }
  return refuse(kLfg, "unknown kernel");
}

int test_motion_kernel(const dawn_lfg_motion_kernel_case& c, cudaStream_t st) {
  const bool geo = c.N >= 1 && c.N <= 65535;
  switch (c.kernel) {
    case DAWN_LFG_MOTION_AA_DOWN:
      if (!c.x || !c.weight || !c.out) return refuse(kMotion, "missing pointer");
      if (!geo || c.H < 4 || c.W < 4 || c.H % 4 != 0 || c.W % 4 != 0 || c.cw < 3 || c.off < 0 || c.off + c.cw > c.ld)
        return refuse(kMotion, "bad geometry");
      return launch_lfgm_aa_down(c.x, c.N, c.H, c.W, c.weight, c.out, c.ld, c.off, c.cw, st);
    case DAWN_LFG_MOTION_REGION_MOMENTS:
      if (!c.logits || !c.out || !c.out2) return refuse(kMotion, "missing pointer");
      if (!geo || c.h < 2 || c.w < 2 || c.R < 1 || c.ldl < c.R || !(c.temperature > 0.f)) return refuse(kMotion, "bad geometry");
      return launch_lfgm_region_moments(c.logits, c.ldl, c.N, c.h, c.w, c.R, c.temperature, c.out, c.out2, c.out3, st);
    case DAWN_LFG_MOTION_FLOW_INPUT:
      if (!c.source || !c.src_shift || !c.src_covar || !c.src_affine || !c.drv_shift || !c.drv_covar || !c.drv_affine || !c.out || !c.out2)
        return refuse(kMotion, "missing pointer");
      if (!geo || c.h < 2 || c.w < 2 || c.R < 1 || c.R > kMotionMaxRegions || c.off < 0 || c.cw < 4 * (c.R + 1) || c.off + c.cw > c.ld)
        return refuse(kMotion, "bad geometry");
      return launch_lfgm_flow_input(c.source, c.N, c.h, c.w, c.R, c.src_shift, c.src_covar, c.src_affine, c.drv_shift, c.drv_covar,
                                    c.drv_affine, c.bg, c.revert, c.out, c.ld, c.off, c.cw, c.out2, st);
    case DAWN_LFG_MOTION_FLOW_COMBINE:
      if (!c.logits || !c.motion || !c.out || !c.out2) return refuse(kMotion, "missing pointer");
      if (!geo || c.h < 1 || c.w < 1 || c.R < 1 || c.R > kMotionMaxRegions || c.ldl < c.R + 2) return refuse(kMotion, "bad geometry");
      return launch_lfgm_flow_combine(c.logits, c.ldl, c.motion, c.N, c.h, c.w, c.R, c.out, c.out2, st);
    case DAWN_LFG_MOTION_BG_HEAD:
      if (!c.out || (c.fc_w == nullptr) != (c.fc_b == nullptr) || (!c.x && c.fc_w)) return refuse(kMotion, "missing pointer");
      if (!geo || (c.fc_w && (c.cw < 1 || c.cw > 8192 || c.ld < c.cw || c.h * c.w < 1))) return refuse(kMotion, "bad geometry");
      return launch_lfgm_bg_head(c.x, c.ld, c.cw, c.N, c.h * c.w, c.fc_w, c.fc_b, c.out, st);
  }
  return refuse(kMotion, "unknown kernel");
}

int synchronize(int rc, cudaStream_t st) {
  if (rc != 0) return rc;
  DAWN_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace
}  // namespace dawn

extern "C" int dawn_lfg_test_kernel(const dawn_lfg_kernel_case* c, void* stream) {
  if (!c) return dawn::refuse(dawn::kLfg, "null case");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  dawn::DeviceArena arena;
  return dawn::synchronize(dawn::test_kernel(*c, arena, st), st);
}

extern "C" int dawn_lfg_motion_test_kernel(const dawn_lfg_motion_kernel_case* c, void* stream) {
  if (!c) return dawn::refuse(dawn::kMotion, "null case");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return dawn::synchronize(dawn::test_motion_kernel(*c, st), st);
}
