// dawn_test_contraction (include/dawn_unet.h): one contraction through exactly one kernel path, with the GemmParams, weight
// image and accumulator scale built the way the network builds them (unet.cu: base_params / set_weights / upload_tc_image /
// Ctx::gemm).  A path that refuses the geometry returns -1 before anything is launched; there is no fallback to another kernel.
#include <cstring>
#include <vector>
#include "../../include/dawn_unet.h"
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.cuh"
#include "tc_gemm.cuh"

namespace dawn {
namespace {

int refuse(const char* why) {
  set_last_error(std::string("dawn_test_contraction: ") + why);
  return -1;
}

struct DevBufs {
  std::vector<void*> v;
  ~DevBufs() { for (void* p : v) cudaFree(p); }
  int alloc(size_t bytes, void** out) {
    DAWN_CUDA_OK(cudaMalloc(out, bytes < 16 ? 16 : bytes));
    v.push_back(*out);
    return 0;
  }
};

int run(const dawn_contraction_case& c, cudaStream_t st) {
  if (c.path < DAWN_PATH_MMA_SYNC || c.path > DAWN_PATH_TC_CONV3_TMA) return refuse("unknown path");
  if (c.epi < EPI_PLAIN || c.epi > EPI_GN_APPLY) return refuse("unknown epilogue");
  if (c.ntaps < 1 || c.ntaps > 52 || c.F < 1 || c.N < 1 || c.ldb < c.N || c.lda < c.Cin) return refuse("bad geometry");
  if (!c.A || !c.B) return refuse("A and B are required");
  if (c.epi == EPI_CA_GATE ? !c.gates : !c.Out) return refuse("no output buffer");

  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.A = c.A; p.lda = c.lda; p.Cin = c.Cin;
  p.up2 = c.up2;
  p.IH = c.IH; p.IW = c.IW; p.OHs = c.OHs; p.OWs = c.OWs; p.in_stride = c.in_stride;
  p.ntaps = c.ntaps;
  for (int t = 0; t < c.ntaps; ++t) { p.dy[t] = (signed char)c.dy[t]; p.dx[t] = (signed char)c.dx[t]; }
  p.M = c.F * c.OHs * c.OWs; p.N = c.N; p.K = c.ntaps * c.Cin;
  p.rows_per_batch = c.rows_per_batch > 0 ? c.rows_per_batch : p.M;
  p.perm_pb = c.perm_pb; p.perm_F = c.perm_F; p.perm_in = c.perm_in; p.perm_out = c.perm_out;
  p.perm_f_lo = c.perm_f_lo; p.perm_f_hi = c.perm_f_hi;
  p.B = c.B; p.ldb = c.ldb; p.b_batch_stride = c.b_batch_stride;
  p.Out = c.Out; p.ldo = c.ldo; p.OH = c.OH; p.OW = c.OW; p.out_stride = c.out_stride; p.oy0 = c.oy0; p.ox0 = c.ox0;
  p.bias = c.bias; p.Res = c.Res; p.ldr = c.ldr;
  p.stats = c.stats; p.cpg = c.cpg;
  p.rowstats = c.rowstats; p.ln_inline = c.ln_inline; p.wsum = c.wsum; p.rot = c.rot; p.P = c.P;
  p.q_post_scale = c.q_post_scale;
  p.kq = c.kq; p.nkq = c.nkq; p.gates = c.gates;
  p.Y = c.Y; p.ldy = c.ldy; p.gn_stats = c.gn_stats; p.gn_w = c.gn_w; p.gn_b = c.gn_b; p.film = c.film; p.gn_count = c.gn_count;
  p.drain = c.drain;

  const bool ln = c.epi >= EPI_QKV_TEMPORAL && c.epi <= EPI_CA_GATE;
  if (p.ln_inline && (c.path != DAWN_PATH_TC_GEMM || p.ntaps != 1)) return refuse("inline LayerNorm statistics need the gather-producer wgmma GEMM and one tap");
  if (ln && !p.ln_inline && !p.rowstats) return refuse("LayerNorm epilogue without row statistics");
  if (ln && !p.wsum) return refuse("LayerNorm epilogue without wsum");
  if (c.epi == EPI_PLAIN && p.stats && (p.cpg <= 0 || p.N / p.cpg > 8)) return refuse("GroupNorm statistics need 8 groups");

  if (c.path == DAWN_PATH_MMA_SYNC) {
    const int rc = launch_gemm(p, c.epi, st);
    if (rc != 0) return rc;
    DAWN_CUDA_OK(cudaStreamSynchronize(st));
    return 0;
  }

  // wgmma paths: the chosen kernel must accept the geometry as given
  const bool conv3 = c.path == DAWN_PATH_TC_CONV3 || c.path == DAWN_PATH_TC_CONV3_TMA;
  if (conv3 ? !tc_conv3_supported(p, c.epi) : !tc_gemm_supported(p, c.epi)) return refuse("the path does not accept this geometry");
  if (p.N % 64 != 0 || p.K % 64 != 0) return refuse("the path does not accept this geometry");
  const bool presplit = c.path == DAWN_PATH_TC_GEMM_PRESPLIT || c.path == DAWN_PATH_TC_CONV3_TMA;
  if (c.path == DAWN_PATH_TC_CONV3_TMA && p.lda != p.Cin) return refuse("the TMA halo conv reads dense fp16 planes (lda == Cin)");

  // weight image and scale exactly as the network's upload (upload_tc_image + set_weights)
  std::vector<float> hB((size_t)p.K * p.ldb);
  DAWN_CUDA_OK(cudaMemcpy(hB.data(), p.B, hB.size() * sizeof(float), cudaMemcpyDeviceToHost));
  std::vector<float> img;
  float img_scale = 1.f;
  tc_pack_weights(hB.data(), p.K, p.N, p.ldb, img, &img_scale);
  p.tc_scale = 1.0f / (kTcActScale * img_scale);
  DevBufs bufs;
  void* dimg = nullptr;
  if (bufs.alloc(img.size() * sizeof(float), &dimg)) return -2;
  DAWN_CUDA_OK(cudaMemcpyAsync(dimg, img.data(), img.size() * sizeof(float), cudaMemcpyHostToDevice, st));
  p.Bimg = static_cast<const float*>(dimg);

  if (presplit) {
    // the split pass writes dense rows of Cin fp16 values per input pixel (Ctx::gemm)
    const long long in_rows = (long long)(p.M / (p.OHs * p.OWs)) * p.IH * p.IW;
    void* planes = nullptr;
    if (bufs.alloc((size_t)in_rows * p.Cin * 4, &planes)) return -2;
    unsigned short* hi = static_cast<unsigned short*>(planes);
    p.A16h = hi; p.A16l = hi + (size_t)in_rows * p.Cin;
    const int rc = launch_split_rows(p.A, p.lda, p.Cin, in_rows, (void*)p.A16h, (void*)p.A16l, st);
    if (rc != 0) return rc;
  }
  const int rc = conv3 ? launch_tc_conv3(p, p.Bimg, st) : launch_tc_gemm(p, p.Bimg, c.epi, st);
  if (rc != 0) return rc;
  DAWN_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace
}  // namespace dawn

extern "C" int dawn_test_contraction(const dawn_contraction_case* c, void* stream) {
  if (!c) return dawn::refuse("null case");
  return dawn::run(*c, static_cast<cudaStream_t>(stream));
}
