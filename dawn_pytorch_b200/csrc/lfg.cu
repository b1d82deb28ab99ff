// Host-side orchestration + C-ABI of the LFG flow decoder (include/dawn_lfg.h; reference LFG/modules/generator.py:132-171).
// One handle = one GPU.  The source-image encoder runs once per clip (dawn_lfg_set_source); dawn_lfg_decode turns a batch of
// frames' (flow, occlusion) maps into images: warp + blend (apply_optical) -> 6 pre-activation ResBlocks -> 2 up blocks with
// warped skips -> 7x7 conv + sigmoid -> blend with the warped source image.  Convolutions run on the wgmma kernels of the
// UNet (tc_conv3.cu / tc_gemm.cu, FP16x3 split precision, fp32 accumulation); eval-mode BatchNorms are folded into the conv
// that precedes them (conv -> BN) or applied as a per-channel affine in the elementwise pass (BN -> ReLU -> conv).
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/dawn_lfg.h"
#include "common.cuh"
#include "contraction.cuh"
#include "gemm.cuh"
#include "lfg_kernels.cuh"

namespace dawn {
namespace {

struct ResPack { PackedWeight c1, c2; float *s1 = nullptr, *t1 = nullptr; };   // norm1 as affine; norm2 folded into conv1

}  // namespace
}  // namespace dawn

using namespace dawn;

struct dawn_lfg {
  dawn_lfg_cfg cfg{};
  int n = 0;                                   // down/up blocks
  std::vector<int> C;                          // channels per level 0..n
  HostParams raw{{}, "lfg: "};
  bool committed = false;
  DeviceArena weights, workspace;
  int64_t launches = 0;
  // packed weights
  PackedWeight first;
  std::vector<PackedWeight> down;
  std::vector<ResPack> res;
  std::vector<UpConv> up;
  float *final_w = nullptr, *final_b = nullptr;
  // geometry / workspace
  int F = 0, H = 0, W = 0, fh = 0, fw = 0;
  std::vector<int> lH, lW;
  float *SRC = nullptr, *SRC_HWC = nullptr, *TMP = nullptr;
  std::vector<float*> SKIP, UP, BL;
  float *X = nullptr, *Y = nullptr, *Z = nullptr;
  float4* MOTION = nullptr;
  bool have_source = false, decoded = false;
};

namespace {

// ------------------------------------------------------------------------------------------ contraction dispatch
int run_conv(dawn_lfg* h, const GemmParams& p, cudaStream_t st) {
  // 14 convolutions without a normalisation in between: the tensor core's round-toward-zero accumulation is a systematic bias that
  // compounds through the stack, so the register accumulators are drained into the RN fp32 tile every 3 taps / K panels (K = 192) instead
  // of every 9 / 4.
  GemmParams q = p;
  q.drain = 3;
  int kernels = 0;
  const int rc = launch_path(q, EPI_PLAIN, choose_path(q, EPI_PLAIN, 0), nullptr, st, &kernels);
  h->launches += kernels;
  return rc;
}
// out (frames, Hh, Ww, w.N) = conv kxk (same padding) of in (frames, Hh, Ww, Cin) + bias
int conv_same(dawn_lfg* h, const PackedWeight& w, int k, const float* in, int Cin, int frames, int Hh, int Ww, float* out, cudaStream_t st) {
  GemmParams p; base_params(p, in, Cin, Cin, frames, Hh, Ww);
  set_weights(p, w); set_square_taps(p, k, k / 2);
  p.Out = out; p.ldo = w.N;
  return run_conv(h, p, st);
}
// out (frames, 2Hh, 2Ww, co) = conv3x3(nearest_upsample_2x(in)) + bias (BatchNorm folded)
int conv_up(dawn_lfg* h, const UpConv& u, const float* in, int Cin, int frames, int Hh, int Ww, float* out, int co, cudaStream_t st) {
  GemmParams p; base_params(p, in, Cin, Cin, frames, Hh, Ww);
  return run_up(p, u, out, co, [&](const GemmParams& q) { return run_conv(h, q, st); });
}

// prediction (F, 3, H, W) fp32 [+ deformed], or with rgb8 != null 8-bit RGB frames (F, H, W, 3) offset by mean (launch_lfg_final_rgb8)
int decode_core(dawn_lfg* h, float* prediction, float* deformed, uint8_t* rgb8, const double* mean, cudaStream_t st) {
  const int n = h->n, F = h->F;
  const int Cb = h->C[n], Hn = h->lH[n], Wn = h->lW[n];
  const long long Mn = (long long)F * Hn * Wn;
  // generator.py:154: out = warp(skip_n) * occ
  h->launches++;
  DAWN_TRY(launch_lfg_warp_blend(h->SKIP[n], Cb, Hn, Wn, h->MOTION, F, h->fh, h->fw, nullptr, 0, h->X, Cb, st));
  // generator.py:156: bottleneck of pre-activation ResBlocks (util.py:85-93)
  const int nres = (int)h->res.size();
  if (nres > 0) {
    h->launches++;
    DAWN_TRY(launch_lfg_affine_relu(h->X, Cb, h->res[0].s1, h->res[0].t1, Cb, Mn, h->Z, Cb, st));
  }
  for (int r = 0; r < nres; ++r) {
    DAWN_TRY(conv_same(h, h->res[r].c1, 3, h->Z, Cb, F, Hn, Wn, h->Y, st));            // conv1 (+ norm2 folded)
    h->launches++;
    DAWN_TRY(launch_lfg_affine_relu(h->Y, Cb, nullptr, nullptr, Cb, Mn, h->Y, Cb, st)); // relu
    DAWN_TRY(conv_same(h, h->res[r].c2, 3, h->Y, Cb, F, Hn, Wn, h->Z, st));            // conv2
    const bool more = r + 1 < nres;
    h->launches++;
    DAWN_TRY(launch_lfg_residual_bn_relu(h->Z, h->X, Cb, Mn, h->X, more ? h->res[r + 1].s1 : nullptr, more ? h->res[r + 1].t1 : nullptr,
                                        more ? h->Z : nullptr, st));                  // out += x; next block's relu(norm1(.))
  }
  // generator.py:157-160: up blocks, each fed by the occlusion blend of the warped skip and the running output
  const float* prev = h->X;
  for (int i = 0; i < n; ++i) {
    const int l = n - i, Cl = h->C[l], Hl = h->lH[l], Wl = h->lW[l], Co = h->C[l - 1];
    const float* in = prev;
    if (h->cfg.skips) {
      float* bl = (i == 0) ? h->Y : h->BL[l];
      h->launches++;
      DAWN_TRY(launch_lfg_warp_blend(h->SKIP[l], Cl, Hl, Wl, h->MOTION, F, h->fh, h->fw, prev, Cl, bl, Cl, st));
      in = bl;
    }
    DAWN_TRY(conv_up(h, h->up[i], in, Cl, F, Hl, Wl, h->UP[l - 1], Co, st));
    h->launches++;
    DAWN_TRY(launch_lfg_affine_relu(h->UP[l - 1], Co, nullptr, nullptr, Co, (long long)F * h->lH[l - 1] * h->lW[l - 1], h->UP[l - 1], Co, st));
    prev = h->UP[l - 1];
  }
  // generator.py:161-167: last skip blend, 7x7 conv + sigmoid, blend with the warped source image
  const float* fin = prev;
  if (h->cfg.skips) {
    h->launches++;
    DAWN_TRY(launch_lfg_warp_blend(h->SKIP[0], h->C[0], h->H, h->W, h->MOTION, F, h->fh, h->fw, prev, h->C[0], h->BL[0], h->C[0], st));
    fin = h->BL[0];
  }
  h->launches++;
  if (rgb8)
    DAWN_TRY(launch_lfg_final_rgb8(fin, h->C[0], h->C[0], F, h->H, h->W, h->final_w, h->final_b, h->SRC, h->MOTION, h->fh, h->fw,
                                   h->cfg.skips ? 1 : 0, mean, rgb8, st));
  else
    DAWN_TRY(launch_lfg_final(fin, h->C[0], h->C[0], F, h->H, h->W, h->final_w, h->final_b, h->SRC, h->MOTION, h->fh, h->fw,
                              h->cfg.skips ? 1 : 0, prediction, deformed, st));
  h->decoded = true;
  return 0;
}

}  // namespace

extern "C" {

int dawn_lfg_create(const dawn_lfg_cfg* cfg, dawn_lfg** out) {
  DAWN_CHECK(cfg && out, "null argument");
  DAWN_TRY(dawn_check_single_device());
  DAWN_CHECK(cfg->num_channels == 3, "lfg: num_channels must be 3");
  DAWN_CHECK(cfg->block_expansion % 64 == 0 && cfg->block_expansion <= 128, "lfg: block_expansion must be 64 or 128");
  DAWN_CHECK(cfg->num_down_blocks >= 1 && cfg->num_down_blocks <= 4, "lfg: num_down_blocks out of range");
  DAWN_CHECK(cfg->num_bottleneck_blocks >= 0 && cfg->num_bottleneck_blocks <= 32, "lfg: num_bottleneck_blocks out of range");
  // the last up block yields min(max_features, block_expansion) channels and the final conv takes block_expansion (generator.py:59)
  DAWN_CHECK(cfg->max_features >= cfg->block_expansion, "lfg: max_features must be at least block_expansion");
  std::vector<int> C;
  for (int i = 0; i <= cfg->num_down_blocks; ++i) {
    C.push_back(std::min(cfg->max_features, cfg->block_expansion << i));                                        // generator.py:40-50
    DAWN_CHECK(C.back() % 32 == 0, "lfg: every level width min(max_features, block_expansion * 2^i) must be a multiple of 32, got " +
                                       std::to_string(C.back()));                                               // launch_gemm's n-tiles
  }
  dawn_lfg* h = new dawn_lfg();
  h->cfg = *cfg;
  h->n = cfg->num_down_blocks;
  h->C = C;
  *out = h;
  return 0;
}

void dawn_lfg_destroy(dawn_lfg* h) {
  delete h;
}

int dawn_lfg_set_param(dawn_lfg* h, const char* name, const float* host, const int64_t* shape, int ndim) {
  DAWN_CHECK(h && name && (shape || ndim == 0), "null argument");
  const std::string n(name);
  if (n.rfind("pixelwise_flow_predictor.", 0) == 0) return 0;                     // never read by forward_with_flow (generator.py:138-171)
  if (n.size() >= 19 && n.compare(n.size() - 19, 19, "num_batches_tracked") == 0) return 0;
  DAWN_CHECK(host, "null argument");
  h->raw.set(n, host, shape, ndim);
  h->committed = false;
  return 0;
}

int dawn_lfg_commit_params(dawn_lfg* h) {
  DAWN_CHECK(h, "null handle");
  h->weights.release();
  h->down.clear(); h->res.clear(); h->up.clear();
  const int n = h->n;
  const HostParams& raw = h->raw;
  auto& arena = h->weights;
  DAWN_TRY(pack_lfg_conv(raw, arena, {{"first.conv", h->C[0]}}, "first.norm", h->cfg.num_channels, 7, 32, &h->first));    // generator.py:36
  for (int i = 0; i < n; ++i) {
    PackedWeight d;
    const std::string p = "down_blocks." + std::to_string(i);
    DAWN_TRY(pack_lfg_conv(raw, arena, {{p + ".conv", h->C[i + 1]}}, p + ".norm", h->C[i], 3, h->C[i], &d));                 // :38-44
    h->down.push_back(d);
  }
  const int Cb = h->C[n];
  for (int r = 0; r < h->cfg.num_bottleneck_blocks; ++r) {
    ResPack rp;
    const std::string p = "bottleneck.r" + std::to_string(r);
    DAWN_TRY(pack_lfg_conv(raw, arena, {{p + ".conv1", Cb}}, p + ".norm2", Cb, 3, Cb, &rp.c1));   // util.py:88-89: conv1 -> norm2 folded
    DAWN_TRY(pack_lfg_conv(raw, arena, {{p + ".conv2", Cb}}, "", Cb, 3, Cb, &rp.c2));
    std::vector<double> s, t;
    DAWN_TRY(bn_affine(raw, p + ".norm1", Cb, s, t));
    std::vector<float> sf(s.begin(), s.end()), tf(t.begin(), t.end());
    DAWN_TRY(arena.upload(sf, &rp.s1));
    DAWN_TRY(arena.upload(tf, &rp.t1));
    h->res.push_back(rp);
  }
  for (int i = 0; i < n; ++i) {
    UpConv u;
    DAWN_TRY(pack_lfg_up(raw, arena, "up_blocks." + std::to_string(i), h->C[n - i - 1], h->C[n - i], &u));            // generator.py:46-52
    h->up.push_back(u);
  }
  {
    const HostParam *w, *b;
    DAWN_TRY(h->raw.need("final.weight", {3, h->C[0], 7, 7}, &w));
    DAWN_TRY(h->raw.need("final.bias", {3}, &b));
    std::vector<float> bp(4, 0.f);
    for (int o = 0; o < 3; ++o) bp[o] = b->data[o];
    DAWN_TRY(h->weights.upload(lfg_final_pack(w->data.data(), h->C[0]), &h->final_w));
    DAWN_TRY(h->weights.upload(bp, &h->final_b));
  }
  h->committed = true;
  h->have_source = false;
  return 0;
}

int dawn_lfg_set_geometry(dawn_lfg* h, int frames, int H, int W, int flow_h, int flow_w) {
  DAWN_CHECK(h, "null handle");
  DAWN_CHECK(h->committed, "lfg: commit_params must precede set_geometry");
  DAWN_CHECK(frames >= 1 && frames <= 65535, "lfg: frames out of range");
  const int n = h->n, div = 1 << n;
  DAWN_CHECK(H >= div && W >= div && H % div == 0 && W % div == 0, "lfg: image height/width must be divisible by 2^num_down_blocks");
  DAWN_CHECK(flow_h >= 1 && flow_w >= 1, "lfg: bad flow size");
  h->workspace.release();
  h->F = frames; h->H = H; h->W = W; h->fh = flow_h; h->fw = flow_w;
  h->lH.assign(n + 1, 0); h->lW.assign(n + 1, 0);
  for (int l = 0; l <= n; ++l) { h->lH[l] = H >> l; h->lW[l] = W >> l; }
  auto& ws = h->workspace;
  const size_t P0 = (size_t)H * W;
  DAWN_TRY(ws.alloc(3 * P0, &h->SRC));
  DAWN_TRY(ws.alloc(32 * P0, &h->SRC_HWC));
  size_t tmp = 0;
  for (int l = 0; l < n; ++l) tmp = std::max(tmp, (size_t)h->lH[l] * h->lW[l] * h->C[l + 1]);
  DAWN_TRY(ws.alloc(tmp, &h->TMP));
  h->SKIP.assign(n + 1, nullptr); h->UP.assign(n + 1, nullptr); h->BL.assign(n + 1, nullptr);
  for (int l = 0; l <= n; ++l) DAWN_TRY(ws.alloc((size_t)h->lH[l] * h->lW[l] * h->C[l], &h->SKIP[l]));
  for (int l = 0; l < n; ++l) {
    const size_t e = (size_t)frames * h->lH[l] * h->lW[l] * h->C[l];
    DAWN_TRY(ws.alloc(e, &h->UP[l]));
    if (h->cfg.skips) DAWN_TRY(ws.alloc(e, &h->BL[l]));
  }
  const size_t eb = (size_t)frames * h->lH[n] * h->lW[n] * h->C[n];
  DAWN_TRY(ws.alloc(eb, &h->X));
  DAWN_TRY(ws.alloc(eb, &h->Y));
  DAWN_TRY(ws.alloc(eb, &h->Z));
  DAWN_TRY(ws.alloc((size_t)frames * flow_h * flow_w, &h->MOTION));
  h->have_source = false; h->decoded = false;
  return 0;
}

int dawn_lfg_set_source(dawn_lfg* h, const float* source, void* stream) {
  DAWN_CHECK(h && source, "null argument");
  DAWN_CHECK(h->F > 0, "lfg: set_geometry must precede set_source");
  cudaStream_t st = (cudaStream_t)stream;
  const int n = h->n, H = h->H, W = h->W;
  h->launches = 0;
  DAWN_CUDA_OK(cudaMemcpyAsync(h->SRC, source, (size_t)3 * H * W * sizeof(float), cudaMemcpyDeviceToDevice, st));
  h->launches++;
  DAWN_TRY(launch_lfg_chw_to_hwc(source, 3, H * W, 32, h->SRC_HWC, st));
  // first: conv7x7 -> BN -> ReLU (util.py:147-150), BN folded
  DAWN_TRY(conv_same(h, h->first, 7, h->SRC_HWC, 32, 1, H, W, h->SKIP[0], st));
  h->launches++;
  DAWN_TRY(launch_lfg_affine_relu(h->SKIP[0], h->C[0], nullptr, nullptr, h->C[0], (long long)H * W, h->SKIP[0], h->C[0], st));
  // down blocks: conv3x3 -> BN -> ReLU -> avgpool 2x2 (util.py:126-131)
  for (int i = 0; i < n; ++i) {
    DAWN_TRY(conv_same(h, h->down[i], 3, h->SKIP[i], h->C[i], 1, h->lH[i], h->lW[i], h->TMP, st));
    h->launches++;
    DAWN_TRY(launch_lfg_relu_avgpool2(h->TMP, h->lH[i], h->lW[i], h->C[i + 1], h->SKIP[i + 1], h->C[i + 1], st));
  }
  h->have_source = true;
  return 0;
}

int dawn_lfg_get_fea(dawn_lfg* h, float* fea, void* stream) {
  DAWN_CHECK(h && fea, "null argument");
  DAWN_CHECK(h->have_source, "lfg: set_source must precede get_fea");
  const int n = h->n;
  return launch_lfg_hwc_to_chw(h->SKIP[n], h->C[n], h->C[n], (long long)h->lH[n] * h->lW[n], fea, (cudaStream_t)stream);
}

int dawn_lfg_decode(dawn_lfg* h, const float* flow, const float* occ, float* prediction, float* deformed, void* stream) {
  DAWN_CHECK(h && flow && occ && prediction, "null argument");
  DAWN_CHECK(h->have_source, "lfg: set_source must precede decode");
  cudaStream_t st = (cudaStream_t)stream;
  h->launches = 1;
  DAWN_TRY(launch_lfg_motion_pack(flow, occ, 0, h->F, h->fh, h->fw, h->MOTION, st));
  return decode_core(h, prediction, deformed, nullptr, nullptr, st);
}

int dawn_lfg_decode_sample(dawn_lfg* h, const float* sample, float* prediction, float* deformed, void* stream) {
  DAWN_CHECK(h && sample && prediction, "null argument");
  DAWN_CHECK(h->have_source, "lfg: set_source must precede decode");
  cudaStream_t st = (cudaStream_t)stream;
  h->launches = 1;
  DAWN_TRY(launch_lfg_motion_pack(sample, nullptr, 1, h->F, h->fh, h->fw, h->MOTION, st));
  return decode_core(h, prediction, deformed, nullptr, nullptr, st);
}

int dawn_lfg_decode_sample_rgb8(dawn_lfg* h, const float* sample, const double mean[3], uint8_t* frames, void* stream) {
  DAWN_CHECK(h && sample && mean && frames, "null argument");
  DAWN_CHECK(h->have_source, "lfg: set_source must precede decode");
  cudaStream_t st = (cudaStream_t)stream;
  h->launches = 1;
  DAWN_TRY(launch_lfg_motion_pack(sample, nullptr, 1, h->F, h->fh, h->fw, h->MOTION, st));
  return decode_core(h, nullptr, nullptr, frames, mean, st);
}

int dawn_lfg_read_tap(dawn_lfg* h, const char* name, float* dst, int* C, int* Hl, int* Wl, void* stream) {
  DAWN_CHECK(h && name && C && Hl && Wl, "null argument");
  DAWN_CHECK(h->F > 0, "lfg: set_geometry first");
  const std::string nm(name);
  const int n = h->n;
  const float* src = nullptr;
  int level = -1;
  if (nm == "bottleneck") { src = h->X; level = n; }
  else if (nm.rfind("up", 0) == 0 && nm.size() == 3 && nm[2] >= '0' && nm[2] < '0' + n) { level = n - 1 - (nm[2] - '0'); src = h->UP[level]; }
  DAWN_CHECK(src != nullptr, "lfg: unknown tap " + nm);
  *C = h->C[level]; *Hl = h->lH[level]; *Wl = h->lW[level];
  if (!dst) return 0;
  DAWN_CHECK(h->decoded, "lfg: decode must precede read_tap");
  return launch_lfg_hwc_to_chw(src, *C, *C, (long long)h->F * *Hl * *Wl, dst, (cudaStream_t)stream);
}

// one layer of Face_loc_Encoder (FD:39-50): relu(conv3x3 stride 2 pad 1); all device pointers, weights as nn.Conv2d stores them
int dawn_conv3x3_s2_relu(const float* x, int Ci, int H, int W, const float* weight, const float* bias, int Co, float* out, void* stream) {
  DAWN_CHECK(x && weight && bias && out && Ci >= 1 && Co >= 1 && H >= 1 && W >= 1, "dawn_conv3x3_s2_relu: bad argument");
  return launch_conv3x3_s2_relu(x, Ci, H, W, weight, bias, Co, out, (cudaStream_t)stream);
}

int64_t dawn_lfg_last_launch_count(dawn_lfg* h) { return h ? h->launches : 0; }
int64_t dawn_lfg_workspace_bytes(dawn_lfg* h) { return h ? h->workspace.bytes() : 0; }

}  // extern "C"
