// Fused temporal attention (LayerNorm-folded QKV projection + rotary + banded attention + out-projection + residual) for the
// 64-channel levels; see temporal_fused.cu.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <vector>

namespace dawn {

struct TemporalFusedArgs {
  const float* x; int ldx;        // layer input over F frames (own frames + neighbour halos when sharded): rows f*P + pixel
  const float* res; int ldr;      // residual rows of the owned frames: (f - q_lo)*P + pixel
  float* out; int ldo;            // output rows, same indexing as res (may alias res)
  int F, P;                       // sequence length on chip, pixels per frame
  int q_lo, q_hi;                 // frames [q_lo, q_hi) produce output
  const uint16_t* Wqkv;           // [8 heads][hi|lo][96][64] fp16, LayerNorm gain and q scale folded, pre-scaled by 1/inv_wscale
  const uint16_t* Wout;           // [8 heads][hi|lo][64][32] fp16, pre-scaled by 1/inv_oscale
  const float* wsum;              // [768] fp32 column sums of the folded QKV weight
  const float* rot;               // [F][16][2] cos/sin per frame (rotary_table)
  const float* bias;              // [8][2*band+1] relative position bias
  int band;
  float inv_wscale, inv_oscale;
  int nbuf;                       // weight stages in shared memory (set by the launcher)
};

// one of the two kernels takes the shape: temporal_fused_wg_kernel (warpgroup MMAs, F <= 256) or temporal_fused_kernel (mma.sync)
bool temporal_fused_supported(int C, int F, int band, int q_lo, int q_hi);
bool temporal_fused_wg_supported(int C, int F, int band, int q_lo, int q_hi);
// runs temporal_fused_wg_kernel where it takes the shape, else temporal_fused_kernel; mma_sync_only forces the latter (tests)
int launch_temporal_fused(const TemporalFusedArgs& a, cudaStream_t st, bool mma_sync_only = false);
void temporal_fused_pack(const float* wqkv, const float* wout, std::vector<uint16_t>& Wq, std::vector<uint16_t>& Wo, float* inv_wscale,
                         float* inv_oscale);

}  // namespace dawn
