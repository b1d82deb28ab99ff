// Host-side orchestration + C-ABI of the LFG motion estimator (include/dawn_lfg.h, dawn_lfg_motion_*): RegionPredictor,
// BGMotionPredictor and the Generator's PixelwiseFlowPredictor (LFG/modules/region_predictor.py, bg_motion_predictor.py,
// pixelwise_flow_predictor.py).  Every convolution goes through the shared contraction dispatcher (contraction.cuh) with the
// eval-mode BatchNorm folded in; the UpBlocks run as parity-class 2x2 convs (run_up).  An Hourglass decoder level is one buffer
// [up-block output | encoder skip] with the concatenation formed through the row stride; level 0 holds [up | input | zeros]
// so that the input conv and the 7x7 output conv both read 32- / 64-channel aligned rows.
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/dawn_lfg.h"
#include "common.cuh"
#include "contraction.cuh"
#include "gemm.cuh"
#include "lfg_kernels.cuh"
#include "lfg_motion_kernels.cuh"

namespace dawn {
namespace {

// Encoder (util.py:153-169) and, with `decoder`, Hourglass (util.py:172-215) on channels-last activations
struct Net {
  std::string prefix;                  // state_dict prefix of the module holding `encoder` (and `decoder`)
  bool decoder = false;
  int nb = 0, be = 0, mx = 0, cin = 0, cpad = 0;
  std::vector<int> Ce;                 // channels of encoder level i (Ce[0] = cin)
  std::vector<PackedWeight> down;
  std::vector<UpConv> up;
  std::vector<int> upco;               // output channels of up block j
  // workspace at the handle's frame count
  int H0 = 0, W0 = 0;
  std::vector<float*> L;               // encoder: level i buffer; hourglass: concatenation of level i (i < nb), L[nb] = bottom
  std::vector<int> ld;                 // row stride of L[i]
  int last_n = 0;
  int width(int i) const { return std::min(mx, be << i); }
  // encoder level i >= 1 is written to (and read from) here
  float* enc_ptr(int i) const { return (decoder && i < nb) ? L[i] + width(i) : L[i]; }
};

}  // namespace
}  // namespace dawn

using namespace dawn;

struct dawn_lfg_motion {
  dawn_lfg_motion_cfg cfg{};
  HostParams raw{{}, "lfg_motion: "};
  bool committed = false, have_rp = false, have_pw = false, have_bg = false;
  DeviceArena weights, workspace;
  int64_t launches = 0;
  Net rp, bg, pw;
  PackedWeight regions, mask_occ;
  float *rp_aa = nullptr, *pw_aa = nullptr, *fc_w = nullptr, *fc_b = nullptr;
  int F = 0, H = 0, W = 0, h = 0, w = 0;
  float *TMP = nullptr, *LOGITS = nullptr, *SRC4 = nullptr, *MOTION = nullptr;
};

namespace {

constexpr int kLdLogits = 16;

void init_net(Net& net, const std::string& prefix, bool decoder, int nb, int be, int mx, int cin, int cpad) {
  net = Net();
  net.prefix = prefix; net.decoder = decoder; net.nb = nb; net.be = be; net.mx = mx; net.cin = cin; net.cpad = cpad;
  net.Ce.push_back(cin);
  for (int i = 1; i <= nb; ++i) net.Ce.push_back(net.width(i));                    // util.py:159-163
}

int pack_net(dawn_lfg_motion* h, Net& net) {
  net.down.clear(); net.up.clear(); net.upco.clear();
  for (int i = 0; i < net.nb; ++i) {
    const std::string p = net.prefix + ".encoder.down_blocks." + std::to_string(i);
    PackedWeight d;
    DAWN_TRY(pack_lfg_conv(h->raw, h->weights, {{p + ".conv", net.Ce[i + 1]}}, p + ".norm", net.Ce[i], 3, i == 0 ? net.cpad : net.Ce[i],
                           &d));
    net.down.push_back(d);
  }
  if (!net.decoder) return 0;
  for (int j = 0; j < net.nb; ++j) {                                                // util.py:183-186
    const int i = net.nb - 1 - j;
    const int ci = (i == net.nb - 1 ? 1 : 2) * net.width(i + 1), co = net.width(i);
    UpConv u;
    DAWN_TRY(pack_lfg_up(h->raw, h->weights, net.prefix + ".decoder.up_blocks." + std::to_string(j), co, ci, &u));
    net.up.push_back(u);
    net.upco.push_back(co);
  }
  return 0;
}

int alloc_net(dawn_lfg_motion* h, Net& net, int H0, int W0) {
  net.H0 = H0; net.W0 = W0;
  net.L.assign(net.nb + 1, nullptr); net.ld.assign(net.nb + 1, 0);
  for (int i = 0; i <= net.nb; ++i) {
    int ld;
    if (!net.decoder) ld = (i == 0) ? net.cpad : net.Ce[i];
    else if (i == net.nb) ld = net.Ce[i];
    else if (i == 0) ld = round_up(net.width(0) + net.cpad, 64);                    // [up | input, zero padded | zeros]
    else ld = 2 * net.width(i);                                                     // [up | skip]
    net.ld[i] = ld;
    DAWN_TRY(h->workspace.alloc((size_t)h->F * (H0 >> i) * (W0 >> i) * ld, &net.L[i]));
    if (i == 0) DAWN_CUDA_OK(cudaMemset(net.L[0], 0, (size_t)h->F * H0 * W0 * ld * sizeof(float)));
  }
  return 0;
}

// ------------------------------------------------------------------------------------------ contraction dispatch
int run_conv(dawn_lfg_motion* h, const GemmParams& p, cudaStream_t st) {
  // no normalisation between these convolutions either: drain the wgmma accumulators every 3 taps / K panels, as the decoder does
  GemmParams q = p;
  q.drain = 3;
  int kernels = 0;
  // a level with fewer pixels per frame than one wgmma row tile (128) would switch between the mma.sync and wgmma paths with the
  // frame count: keep it on mma.sync so that a frame's result does not depend on the batch it runs in
  const bool small = !q.up2 && (long long)q.OHs * q.OWs < 128;
  const int rc = launch_path(q, EPI_PLAIN, small ? DAWN_PATH_MMA_SYNC : choose_path(q, EPI_PLAIN, 0), nullptr, st, &kernels);
  h->launches += kernels;
  return rc;
}
int conv_same(dawn_lfg_motion* h, const PackedWeight& w, int k, const float* in, int lda, int Cin, int frames, int Hh, int Ww, float* out,
              int ldo, cudaStream_t st) {
  GemmParams p; base_params(p, in, lda, Cin, frames, Hh, Ww);
  set_weights(p, w); set_square_taps(p, k, k / 2);
  p.Out = out; p.ldo = ldo;
  return run_conv(h, p, st);
}

// the Encoder's down blocks over net.L[0] (its input, already written), then for an Hourglass the decoder
int run_net(dawn_lfg_motion* h, Net& net, int n, cudaStream_t st) {
  for (int i = 0; i < net.nb; ++i) {                                                // DownBlock2d: conv -> BN -> ReLU -> pool
    const int Hi = net.H0 >> i, Wi = net.W0 >> i, co = net.Ce[i + 1];
    const float* in = (i == 0) ? (net.decoder ? net.L[0] + net.width(0) : net.L[0]) : net.enc_ptr(i);
    DAWN_TRY(conv_same(h, net.down[i], 3, in, net.ld[i], i == 0 ? net.cpad : net.Ce[i], n, Hi, Wi, h->TMP, co, st));
    h->launches++;
    DAWN_TRY(launch_lfg_relu_avgpool2(h->TMP, n * Hi, Wi, co, net.enc_ptr(i + 1), net.ld[i + 1], st));
  }
  if (net.decoder) {
    for (int j = 0; j < net.nb; ++j) {                                              // UpBlock2d, then cat([out, skip]) in place
      const int i = net.nb - 1 - j, co = net.upco[j];
      const int Hs = net.H0 >> (i + 1), Ws = net.W0 >> (i + 1);
      const int Cin = (j == 0) ? net.Ce[net.nb] : net.ld[i + 1];
      GemmParams p; base_params(p, net.L[i + 1], net.ld[i + 1], Cin, n, Hs, Ws);
      DAWN_TRY(run_up(p, net.up[j], net.L[i], net.ld[i], [&](const GemmParams& q) { return run_conv(h, q, st); }));
      h->launches++;
      DAWN_TRY(launch_lfg_affine_relu(net.L[i], net.ld[i], nullptr, nullptr, co, (long long)n * (net.H0 >> i) * (net.W0 >> i), net.L[i],
                                      net.ld[i], st));
    }
  }
  net.last_n = n;
  return 0;
}

int check_n(dawn_lfg_motion* h, int n, bool part, const char* what) {
  DAWN_CHECK(h->committed && h->F > 0, "lfg_motion: commit_params and set_geometry must precede the stage calls");
  DAWN_CHECK(part, std::string("lfg_motion: no ") + what + " parameters were committed");
  DAWN_CHECK(n >= 1 && n <= h->F, "lfg_motion: n must be in [1, frames of set_geometry]");
  return 0;
}

}  // namespace

extern "C" {

int dawn_lfg_motion_create(const dawn_lfg_motion_cfg* cfg, dawn_lfg_motion** out) {
  DAWN_CHECK(cfg && out, "null argument");
  DAWN_TRY(dawn_check_single_device());
  const dawn_lfg_motion_cfg& c = *cfg;
  DAWN_CHECK(c.num_regions == 10, "lfg_motion: num_regions must be 10");
  DAWN_CHECK(c.num_channels == 3, "lfg_motion: num_channels must be 3");
  DAWN_CHECK(c.estimate_affine == 1 && c.pca_based == 1, "lfg_motion: only the PCA-based affine estimate is supported (estimate_affine, pca_based)");
  DAWN_CHECK(c.fast_svd == 0, "lfg_motion: fast_svd is not supported");
  DAWN_CHECK(c.rp_block_expansion == 32 && c.rp_max_features == 1024 && c.rp_num_blocks == 5,
             "lfg_motion: region predictor must have block_expansion 32, max_features 1024, num_blocks 5");
  DAWN_CHECK(c.rp_temperature == 0.1f && c.rp_scale_factor == 0.25f, "lfg_motion: region predictor must have temperature 0.1, scale_factor 0.25");
  DAWN_CHECK(c.bg_type == DAWN_LFG_BG_AFFINE || c.bg_type == DAWN_LFG_BG_ZERO, "lfg_motion: bg_type must be 'affine' or 'zero'");
  DAWN_CHECK(c.bg_type == DAWN_LFG_BG_ZERO || (c.bg_block_expansion == 32 && c.bg_max_features == 1024 && c.bg_num_blocks == 5),
             "lfg_motion: bg predictor must have block_expansion 32, max_features 1024, num_blocks 5");
  DAWN_CHECK(c.pw_block_expansion == 64 && c.pw_max_features == 1024 && c.pw_num_blocks == 5 && c.pw_scale_factor == 0.25f,
             "lfg_motion: flow predictor must have block_expansion 64, max_features 1024, num_blocks 5, scale_factor 0.25");
  DAWN_CHECK(c.use_covar_heatmap == 1 && c.use_deformed_source == 1 && c.estimate_occlusion_map == 1,
             "lfg_motion: use_covar_heatmap, use_deformed_source and estimate_occlusion_map must be true");
  DAWN_CHECK(c.revert_axis_swap == 0 || c.revert_axis_swap == 1, "lfg_motion: revert_axis_swap must be 0 or 1");
  dawn_lfg_motion* h = new dawn_lfg_motion();
  h->cfg = c;
  init_net(h->rp, "region_predictor.predictor", true, 5, 32, 1024, 3, 32);
  init_net(h->bg, "bg_predictor", false, 5, 32, 1024, 6, 32);
  init_net(h->pw, "pixelwise_flow_predictor.hourglass", true, 5, 64, 1024, (c.num_regions + 1) * (c.num_channels + 1), 64);
  *out = h;
  return 0;
}

void dawn_lfg_motion_destroy(dawn_lfg_motion* h) {
  delete h;
}

int dawn_lfg_motion_set_param(dawn_lfg_motion* h, const char* name, const float* host, const int64_t* shape, int ndim) {
  DAWN_CHECK(h && name && (shape || ndim == 0), "null argument");
  const std::string n(name);
  if (n.size() >= 19 && n.compare(n.size() - 19, 19, "num_batches_tracked") == 0) return 0;
  DAWN_CHECK(n.rfind("region_predictor.", 0) == 0 || n.rfind("bg_predictor.", 0) == 0 || n.rfind("pixelwise_flow_predictor.", 0) == 0,
             "lfg_motion: unexpected parameter " + n);
  DAWN_CHECK(host, "null argument");
  h->raw.set(n, host, shape, ndim);
  h->committed = false;
  return 0;
}

int dawn_lfg_motion_commit_params(dawn_lfg_motion* h) {
  DAWN_CHECK(h, "null handle");
  h->weights.release();
  // each module may hold only its own part (RegionPredictor, BGMotionPredictor, the Generator's flow predictor): a part is
  // packed when any of its parameters was set, and its stage refuses to run otherwise
  auto has = [&](const char* prefix) {
    for (auto& kv : h->raw.map) if (kv.first.rfind(prefix, 0) == 0) return true;
    return false;
  };
  h->have_rp = has("region_predictor.");
  h->have_pw = has("pixelwise_flow_predictor.");
  h->have_bg = has("bg_predictor.") || h->cfg.bg_type == DAWN_LFG_BG_ZERO;
  DAWN_CHECK(h->have_rp || h->have_pw || h->have_bg, "lfg_motion: no parameters set");
  const int R = h->cfg.num_regions;
  if (h->have_rp) {
    DAWN_TRY(pack_net(h, h->rp));
    DAWN_TRY(pack_lfg_conv(h->raw, h->weights, {{"region_predictor.regions", R}}, "", h->rp.be + h->rp.cin, 7,
                           round_up(h->rp.be + h->rp.cpad, 64), &h->regions));                 // region_predictor.py:39-40
    const HostParam* g;
    DAWN_TRY(h->raw.need("region_predictor.down.weight", {3, 1, kAAK, kAAK}, &g));
    DAWN_TRY(h->weights.upload(g->data, &h->rp_aa));
  }
  if (h->have_pw) {
    DAWN_TRY(pack_net(h, h->pw));
    DAWN_TRY(pack_lfg_conv(h->raw, h->weights, {{"pixelwise_flow_predictor.mask", R + 1}, {"pixelwise_flow_predictor.occlusion", 1}}, "",
                           h->pw.be + h->pw.cin, 7, round_up(h->pw.be + h->pw.cpad, 64), &h->mask_occ));   // pixelwise_flow_predictor.py:32-37
    const HostParam* g;
    DAWN_TRY(h->raw.need("pixelwise_flow_predictor.down.weight", {3, 1, kAAK, kAAK}, &g));
    DAWN_TRY(h->weights.upload(g->data, &h->pw_aa));
  }
  h->fc_w = h->fc_b = nullptr;
  if (h->cfg.bg_type == DAWN_LFG_BG_AFFINE && h->have_bg) {
    DAWN_TRY(pack_net(h, h->bg));
    const HostParam *w, *b;
    DAWN_TRY(h->raw.need("bg_predictor.fc.weight", {6, h->bg.Ce[h->bg.nb]}, &w));
    DAWN_TRY(h->raw.need("bg_predictor.fc.bias", {6}, &b));
    DAWN_TRY(h->weights.upload(w->data, &h->fc_w));
    DAWN_TRY(h->weights.upload(b->data, &h->fc_b));
  }
  h->committed = true;
  h->F = 0;
  return 0;
}

int dawn_lfg_motion_set_geometry(dawn_lfg_motion* h, int frames, int H, int W) {
  DAWN_CHECK(h, "null handle");
  DAWN_CHECK(h->committed, "lfg_motion: commit_params must precede set_geometry");
  DAWN_CHECK(frames >= 1 && frames <= 1024, "lfg_motion: frames out of range [1, 1024]");
  DAWN_CHECK(H >= 128 && W >= 128 && H % 128 == 0 && W % 128 == 0, "lfg_motion: H and W must be multiples of 128");
  DAWN_CHECK((long long)frames * H * W * 64 < (1LL << 31), "lfg_motion: frames x H x W too large for one call; use fewer frames per call");
  h->workspace.release();
  h->F = frames; h->H = H; h->W = W; h->h = H / 4; h->w = W / 4;
  const int hh = h->h, ww = h->w;
  const bool bg_net = h->have_bg && h->cfg.bg_type == DAWN_LFG_BG_AFFINE;
  if (h->have_rp) DAWN_TRY(alloc_net(h, h->rp, hh, ww));
  if (h->have_pw) DAWN_TRY(alloc_net(h, h->pw, hh, ww));
  if (bg_net) DAWN_TRY(alloc_net(h, h->bg, H, W));
  size_t tmp = 0;
  for (Net* net : {&h->rp, &h->pw, &h->bg}) {
    if (net->L.empty()) continue;
    for (int i = 0; i < net->nb; ++i) tmp = std::max(tmp, (size_t)(net->H0 >> i) * (net->W0 >> i) * net->Ce[i + 1]);
  }
  DAWN_TRY(h->workspace.alloc(tmp * frames, &h->TMP));
  DAWN_TRY(h->workspace.alloc((size_t)frames * hh * ww * kLdLogits, &h->LOGITS));
  DAWN_TRY(h->workspace.alloc((size_t)hh * ww * 4, &h->SRC4));
  DAWN_TRY(h->workspace.alloc((size_t)frames * hh * ww * 2 * (h->cfg.num_regions + 1), &h->MOTION));
  return 0;
}

int dawn_lfg_motion_regions(dawn_lfg_motion* h, const float* images, int n, float* shift, float* covar, float* heatmap, void* stream) {
  DAWN_CHECK(h && images && shift && covar, "null argument");
  DAWN_TRY(check_n(h, n, h->have_rp, "region_predictor"));
  cudaStream_t st = (cudaStream_t)stream;
  Net& net = h->rp;
  h->launches = 1;
  DAWN_TRY(launch_lfgm_aa_down(images, n, h->H, h->W, h->rp_aa, net.L[0], net.ld[0], net.width(0), net.cpad, st));   // :79-80
  DAWN_TRY(run_net(h, net, n, st));                                                                                 // :82
  DAWN_TRY(conv_same(h, h->regions, 7, net.L[0], net.ld[0], net.ld[0], n, h->h, h->w, h->LOGITS, kLdLogits, st));   // :83
  h->launches++;
  return launch_lfgm_region_moments(h->LOGITS, kLdLogits, n, h->h, h->w, h->cfg.num_regions, h->cfg.rp_temperature, shift, covar,
                                    heatmap, st);                                                                    // :85-91
}

int dawn_lfg_motion_bg(dawn_lfg_motion* h, const float* source, int n_source, const float* driving, int n, float* bg, void* stream) {
  DAWN_CHECK(h && bg, "null argument");
  DAWN_TRY(check_n(h, n, h->have_bg, "bg_predictor"));
  cudaStream_t st = (cudaStream_t)stream;
  h->launches = 1;
  if (h->cfg.bg_type == DAWN_LFG_BG_ZERO) return launch_lfgm_bg_head(nullptr, 0, 0, n, 0, nullptr, nullptr, bg, st);
  DAWN_CHECK(source && driving && (n_source == 1 || n_source == n), "lfg_motion: bg needs source (1 or n frames) and driving");
  Net& net = h->bg;
  DAWN_TRY(launch_lfgm_pack_pair(source, n_source, driving, n, h->H * h->W, net.L[0], st));                       // :49
  DAWN_TRY(run_net(h, net, n, st));
  h->launches++;
  const int P = (h->H >> net.nb) * (h->W >> net.nb), C = net.Ce[net.nb];
  return launch_lfgm_bg_head(net.L[net.nb], C, C, n, P, h->fc_w, h->fc_b, bg, st);                                  // :50-55
}

int dawn_lfg_motion_flow(dawn_lfg_motion* h, const float* source, int n, const float* src_shift, const float* src_covar,
                         const float* src_affine, const float* drv_shift, const float* drv_covar, const float* drv_affine,
                         const float* bg, float* flow, float* occlusion, void* stream) {
  DAWN_CHECK(h && source && src_shift && src_covar && src_affine && drv_shift && drv_covar && drv_affine && flow && occlusion,
             "null argument");
  DAWN_TRY(check_n(h, n, h->have_pw, "pixelwise_flow_predictor"));
  cudaStream_t st = (cudaStream_t)stream;
  Net& net = h->pw;
  const int R = h->cfg.num_regions;
  h->launches = 2;
  DAWN_TRY(launch_lfgm_aa_down(source, 1, h->H, h->W, h->pw_aa, h->SRC4, 4, 0, 4, st));                            // :112-113
  DAWN_TRY(launch_lfgm_flow_input(h->SRC4, n, h->h, h->w, R, src_shift, src_covar, src_affine, drv_shift, drv_covar, drv_affine, bg,
                                  h->cfg.revert_axis_swap, net.L[0] + net.width(0), net.ld[0], 0, net.cpad, h->MOTION, st));   // :118-121
  DAWN_TRY(run_net(h, net, n, st));                                                                                  // :123
  DAWN_TRY(conv_same(h, h->mask_occ, 7, net.L[0], net.ld[0], net.ld[0], n, h->h, h->w, h->LOGITS, kLdLogits, st));   // :125, :134
  h->launches++;
  return launch_lfgm_flow_combine(h->LOGITS, kLdLogits, h->MOTION, n, h->h, h->w, R, flow, occlusion, st);           // :126-135
}

int dawn_lfg_motion_read_tap(dawn_lfg_motion* h, const char* name, float* dst, int* C, int* n, int* Hl, int* Wl, void* stream) {
  DAWN_CHECK(h && name && C && n && Hl && Wl, "null argument");
  DAWN_CHECK(h->F > 0, "lfg_motion: set_geometry first");
  const std::string nm(name);
  const Net* net = nullptr;
  if (nm == "region_predictor") net = &h->rp;
  else if (nm == "flow_hourglass") net = &h->pw;
  else if (nm == "bg_encoder" && h->cfg.bg_type == DAWN_LFG_BG_AFFINE) net = &h->bg;
  DAWN_CHECK(net != nullptr && !net->L.empty(), "lfg_motion: unknown tap " + nm);
  const int lvl = net->decoder ? 0 : net->nb;
  *C = net->decoder ? net->be + net->cin : net->Ce[lvl];
  *n = net->last_n; *Hl = net->H0 >> lvl; *Wl = net->W0 >> lvl;
  if (!dst) return 0;
  DAWN_CHECK(net->last_n > 0, "lfg_motion: run the stage before read_tap");
  return launch_lfg_hwc_to_chw(net->L[lvl], net->ld[lvl], *C, (long long)*n * *Hl * *Wl, dst, (cudaStream_t)stream);
}

int64_t dawn_lfg_motion_last_launch_count(dawn_lfg_motion* h) { return h ? h->launches : 0; }
int64_t dawn_lfg_motion_workspace_bytes(dawn_lfg_motion* h) { return h ? h->workspace.bytes() : 0; }

}  // extern "C"
