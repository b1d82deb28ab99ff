// Fused cross-attention gate weights (LayerNorm_img + q projection + 2-key softmax gates + Gram-form rstd); see ca_fused.cu.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <vector>

namespace dawn {

struct CaFusedArgs {
  const float* x; int ldx;        // block input, rows f*P + pixel, ci channels
  int F, P;
  const uint16_t* Wq;             // [hi|lo][192][ci] fp16, LayerNorm gain folded, pre-scaled by 1/inv_wscale
  float inv_wscale;
  const float* kq;                // [F][3][64] projected keys of the frame's conditioning tokens
  const float* nkq;               // [3][8] null keys
  const float* G;                 // [F][3][81] Gram forms of the folded to_out / LayerNorm
  float* Wt;                      // [F*P][32] output: rstd * [1, gate_0..7] per cross-attention, 5 zero columns
  int px_per_cta;                 // set by the launcher
};

struct GnHcondArgs {
  const float* Wt;                // [F*P][32] gate weights (ca_fused / ca_rstd)
  const float* T; int ldbT;       // [F][32][ldbT] per-frame tables
  const float* Y; int ldy;        // conv1 output
  float* Out; int ldo;            // a1 (fp32), or
  unsigned short *Out16h, *Out16l; // a1 as two dense fp16 planes [F*P][co] (hi | lo of the wgmma-kernel split): the consuming 3x3 conv then
                                  // fetches its halo tiles by TMA with no conversion pass; same bytes as the fp32 row
  int F, P, co;
  const double* gn_stats; double gn_count; int cpg;     // clip-wide GroupNorm sums (sum, sumsq per group), [clips][16]
  const float *gn_w, *gn_b, *film;                     // film: [clips][2*co] (scale | shift) or nullptr
  int px_per_cta;                 // set by the launcher
  int clips = 1;                  // frame f belongs to clip f % clips
};
bool gn_hcond_supported(int co, int P);
int launch_gn_hcond(const GnHcondArgs& a, cudaStream_t st);

bool ca_fused_supported(int ci, int P);
int launch_ca_fused(const CaFusedArgs& a, int ci, cudaStream_t st);
void ca_fused_pack(const float* wq_kmajor, int ci, std::vector<uint16_t>& W, float* inv_wscale);

}  // namespace dawn
