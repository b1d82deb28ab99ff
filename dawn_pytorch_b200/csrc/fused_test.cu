// dawn_test_fused (include/dawn_unet.h): one fused attention / cross-attention kernel with the weight folds and packers the
// network's upload runs, for per-kernel tests against a high-precision reference.
#include <cmath>
#include <string>
#include <vector>

#include "ca_fused.cuh"
#include "common.cuh"
#include "contraction.cuh"
#include "kernels.cuh"
#include "sla_fused.cuh"
#include "temporal_fused.cuh"

namespace dawn {
namespace {

int refuse(const char* why) {
  set_last_error(std::string("dawn_test_fused: ") + why);
  return -1;
}

int to_host(const float* d, size_t n, std::vector<float>& h) {
  h.resize(n);
  DAWN_CUDA_OK(cudaMemcpy(h.data(), d, n * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

AttnArgs attn_args(const dawn_fused_case& c) {
  AttnArgs a{};
  a.qkv = c.qkv; a.ld = c.ld; a.out = c.out; a.ldo = c.ldo;
  a.nseq = c.nseq; a.L = c.L; a.seq_base_stride = c.seq_base_stride; a.elem_stride = c.elem_stride;
  a.band = c.band; a.bias = c.bias; a.q_lo = c.q_lo; a.q_hi = c.q_hi; a.pb = c.pb;
  return a;
}

int test_fused(const dawn_fused_case& c, DeviceArena& arena, cudaStream_t st) {
  switch (c.kernel) {
    case DAWN_FUSED_TEMPORAL:
    case DAWN_FUSED_TEMPORAL_MMA_SYNC: {
      if (!c.x || !c.res || !c.out || !c.gamma || !c.w_qkv || !c.w_out || !c.rot || !c.bias) return refuse("missing pointer");
      if (c.P < 1 || c.ldx < 64 || c.ldr < 64 || c.ldo < 64 || (c.ldx | c.ldr | c.ldo) & 3) return refuse("bad geometry");
      if (!temporal_fused_supported(c.C, c.F, c.band, c.q_lo, c.q_hi)) return refuse("temporal_fused_supported refuses the geometry");
      std::vector<float> g, wqkv, wout;
      DAWN_TRY(to_host(c.gamma, 64, g)); DAWN_TRY(to_host(c.w_qkv, 768 * 64, wqkv)); DAWN_TRY(to_host(c.w_out, 64 * 256, wout));
      const std::vector<float> wf = fold_linear(wqkv.data(), 768, 64, g.data(), 1.0f / sqrtf(32.0f), 256);
      TemporalFusedArgs a{};
      std::vector<uint16_t> Wq, Wo;
      temporal_fused_pack(wf.data(), wout.data(), Wq, Wo, &a.inv_wscale, &a.inv_oscale);
      uint16_t *dq, *dwo;
      float* wsum;
      DAWN_TRY(arena.upload(Wq, &dq)); DAWN_TRY(arena.upload(Wo, &dwo));
      DAWN_TRY(arena.upload(row_sums(wf, 768, 64), &wsum));
      a.x = c.x; a.ldx = c.ldx; a.res = c.res; a.ldr = c.ldr; a.out = c.out; a.ldo = c.ldo;
      a.F = c.F; a.P = c.P; a.q_lo = c.q_lo; a.q_hi = c.q_hi;
      a.Wqkv = dq; a.Wout = dwo; a.wsum = wsum; a.rot = c.rot; a.bias = c.bias; a.band = c.band;
      return launch_temporal_fused(a, st, c.kernel == DAWN_FUSED_TEMPORAL_MMA_SYNC);
    }
    case DAWN_FUSED_ATTN_TC:
    case DAWN_FUSED_ATTN_SIMT: {
      if (!c.qkv || !c.out) return refuse("missing pointer");
      if (c.nseq < 1 || c.L < 1 || c.band < 1 || c.q_lo < 0 || c.q_hi > c.L || c.q_lo >= c.q_hi || c.ld < 768 || c.ldo < 256 ||
          ((c.ld | c.ldo) & 3) ||                                        // float4 rows in both kernels
          c.pb < 0 || (c.pb > 0 && c.nseq % c.pb))                       // sequence blocks must tile the rows
        return refuse("bad geometry");
      const AttnArgs a = attn_args(c);
      if (c.kernel == DAWN_FUSED_ATTN_SIMT) return launch_attention(a, st);
      if (!attention_tc_supported(a)) return refuse("attention_tc_supported refuses the geometry");
      return launch_attention_tc(a, st);
    }
    case DAWN_FUSED_SLA_CTX:
    case DAWN_FUSED_SLA_OUT: {
      if (!c.x || !c.gamma || !c.w_qkv || !c.Bf) return refuse("missing pointer");
      if (c.F < 1 || c.ldx < 64 || (c.ldx & 3) || c.ldb < 64) return refuse("bad geometry");
      if (!sla_fused_supported(c.C, c.P)) return refuse("sla_fused_supported refuses the geometry");
      std::vector<float> g, wqkv;
      DAWN_TRY(to_host(c.gamma, 64, g)); DAWN_TRY(to_host(c.w_qkv, 768 * 64, wqkv));
      const std::vector<float> wf = fold_linear(wqkv.data(), 768, 64, g.data(), 1.f, 0);
      std::vector<uint16_t> W;
      if (c.kernel == DAWN_FUSED_SLA_CTX) {
        if (!c.w_out) return refuse("missing pointer");
        std::vector<float> wout, wt((size_t)256 * 64);
        DAWN_TRY(to_host(c.w_out, 64 * 256, wout));
        for (int ch = 0; ch < 64; ++ch)
          for (int k = 0; k < 256; ++k) wt[(size_t)k * 64 + ch] = wout[(size_t)ch * 256 + k];
        SlaCtxArgs a{};
        sla_fused_pack(wf.data(), W, &a.inv_wscale);
        uint16_t* dw;
        float *dwt, *part;
        DAWN_TRY(arena.upload(W, &dw)); DAWN_TRY(arena.upload(wt, &dwt));
        DAWN_TRY(arena.alloc(sla_fused_part_floats(c.F, c.P), &part));
        a.x = c.x; a.ldx = c.ldx; a.F = c.F; a.P = c.P; a.Wkv = dw; a.part = part;
        return launch_sla_ctx_fused(a, dwt, c.Bf, c.ldb, st);
      }
      if (!c.out || !c.out_bias || c.ldo < 64 || (c.ldo & 1)) return refuse("bad output");
      SlaOutArgs o{};
      sla_out_pack(wf.data(), W, &o.inv_wscale);
      uint16_t* dw;
      DAWN_TRY(arena.upload(W, &dw));
      o.x = c.x; o.ldx = c.ldx; o.out = c.out; o.ldo = c.ldo; o.F = c.F; o.P = c.P; o.Wq = dw;
      o.Bf = c.Bf; o.ldb = c.ldb; o.bias = c.out_bias;
      return launch_sla_out_fused(o, st);
    }
    case DAWN_FUSED_SLA_CTX_UNFUSED: {
      if (!c.qkv || !c.w_out || !c.Bf) return refuse("missing pointer");
      if (c.F < 1 || c.P < 1 || c.C < 1 || c.ld < 768 || c.ldb < c.C) return refuse("bad geometry");
      std::vector<float> wout, wt((size_t)256 * c.C);
      DAWN_TRY(to_host(c.w_out, (size_t)c.C * 256, wout));
      for (int ch = 0; ch < c.C; ++ch)
        for (int k = 0; k < 256; ++k) wt[(size_t)k * c.C + ch] = wout[(size_t)ch * 256 + k];
      float* dwt;
      DAWN_TRY(arena.upload(wt, &dwt));
      return launch_sla_context(c.qkv, c.ld, c.F, c.P, dwt, c.C, c.Bf, c.ldb, st);
    }
    case DAWN_FUSED_CA_WT: {
      if (!c.x || !c.gamma || !c.w_qkv || !c.kq || !c.nkq || !c.G || !c.Wt) return refuse("missing pointer");
      if (c.F < 1 || c.ldx < c.C || (c.ldx & 3)) return refuse("bad geometry");
      if (!ca_fused_supported(c.C, c.P)) return refuse("ca_fused_supported refuses the geometry");
      std::vector<float> g, q;
      DAWN_TRY(to_host(c.gamma, (size_t)3 * c.C, g)); DAWN_TRY(to_host(c.w_qkv, (size_t)3 * 64 * c.C, q));
      const float* to_q[3] = {q.data(), q.data() + (size_t)64 * c.C, q.data() + (size_t)128 * c.C};
      const float* gain[3] = {g.data(), g.data() + c.C, g.data() + 2 * c.C};
      std::vector<float> wq, wsum;
      fold_ca_q(to_q, gain, c.C, wq, wsum);
      CaFusedArgs a{};
      std::vector<uint16_t> W;
      ca_fused_pack(wq.data(), c.C, W, &a.inv_wscale);
      uint16_t* dw;
      DAWN_TRY(arena.upload(W, &dw));
      a.x = c.x; a.ldx = c.ldx; a.F = c.F; a.P = c.P; a.Wq = dw; a.kq = c.kq; a.nkq = c.nkq; a.G = c.G; a.Wt = c.Wt;
      return launch_ca_fused(a, c.C, st);
    }
    case DAWN_FUSED_CA_RSTD:
      if (!c.gates || !c.G || !c.Wt) return refuse("missing pointer");
      if (c.F < 1 || c.P < 1) return refuse("bad geometry");
      return launch_ca_rstd(c.gates, c.G, c.F * c.P, c.P, c.Wt, st);
    case DAWN_FUSED_GN_HCOND: {
      if (!c.Wt || !c.T || !c.Y || !c.gn_stats || !c.gn_w || !c.gn_b) return refuse("missing pointer");
      if ((c.out16h == nullptr) != (c.out16l == nullptr) || (!c.out16h && !c.out)) return refuse("no output buffer");
      if (c.F < 1 || c.cpg < 1 || c.C % c.cpg || c.C / c.cpg > 8 || c.ldbT < c.C || c.ldy < c.C || (c.ldy & 1) ||
          (c.out && (c.ldo < c.C || (c.ldo & 1))))
        return refuse("bad geometry");
      if (!gn_hcond_supported(c.C, c.P)) return refuse("gn_hcond_supported refuses the geometry");
      GnHcondArgs a{};
      a.Wt = c.Wt; a.T = c.T; a.ldbT = c.ldbT; a.Y = c.Y; a.ldy = c.ldy;
      a.Out = c.out; a.ldo = c.ldo; a.Out16h = c.out16h; a.Out16l = c.out16l;
      a.F = c.F; a.P = c.P; a.co = c.C;
      a.gn_stats = c.gn_stats; a.gn_count = c.gn_count; a.cpg = c.cpg; a.gn_w = c.gn_w; a.gn_b = c.gn_b; a.film = c.film;
      return launch_gn_hcond(a, st);
    }
  }
  return refuse("unknown kernel");
}

}  // namespace
}  // namespace dawn

extern "C" int dawn_test_fused(const dawn_fused_case* c, void* stream) {
  if (!c) return dawn::refuse("null case");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  dawn::DeviceArena arena;
  const int rc = dawn::test_fused(*c, arena, st);
  if (rc != 0) return rc;
  DAWN_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}
