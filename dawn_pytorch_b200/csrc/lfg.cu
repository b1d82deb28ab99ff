// Host-side orchestration + C-ABI of the LFG flow decoder (include/dawn_lfg.h; reference LFG/modules/generator.py:132-171).
// One handle = one GPU.  The source-image encoder runs once per clip (dawn_lfg_set_source); dawn_lfg_decode turns a batch of
// frames' (flow, occlusion) maps into images: warp + blend (apply_optical) -> 6 pre-activation ResBlocks -> 2 up blocks with
// warped skips -> 7x7 conv + sigmoid -> blend with the warped source image.  Convolutions run on the wgmma kernels of the
// UNet (tc_conv3.cu / tc_gemm.cu, FP16x3 split precision, fp32 accumulation); eval-mode BatchNorms are folded into the conv
// that precedes them (conv -> BN) or applied as a per-channel affine in the elementwise pass (BN -> ReLU -> conv).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/dawn_lfg.h"
#include "common.cuh"
#include "gemm.cuh"
#include "tc_gemm.cuh"
#include "lfg_kernels.cuh"

namespace dawn {
namespace {

#define LFG_CHECK(cond, msg)                  \
  do {                                        \
    if (!(cond)) {                            \
      ::dawn::set_last_error(msg);            \
      return -1;                              \
    }                                         \
  } while (0)
#define LFG_TRY(expr)            \
  do {                           \
    int _rc = (expr);            \
    if (_rc != 0) return _rc;    \
  } while (0)

struct HostParam {
  std::vector<float> data;
  std::vector<int64_t> shape;
};
struct ConvPack {            // [tap * ci_pad + c][ldb] fp32 (+ wgmma weight image), bias [ldb]
  float* w = nullptr; float* img = nullptr; float img_scale = 1.f; float* b = nullptr;
  int K = 0, N = 0, ldb = 0, ci_pad = 0;
};
struct UpPack {              // nearest-2x upsample + 3x3 conv as output-parity classes over the low-resolution grid
  ConvPack cls[4];           // 2x2-tap conv per class (py, px)
  ConvPack all;              // Cout == 64: one 3x3 conv with 4 x 64 output columns (tc_conv3 `up2` epilogue)
  bool has_all = false;
};
struct ResPack { ConvPack c1, c2; float *s1 = nullptr, *t1 = nullptr; };   // norm1 as affine; norm2 folded into conv1

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

}  // namespace
}  // namespace dawn

using namespace dawn;

struct dawn_lfg {
  dawn_lfg_cfg cfg{};
  int n = 0;                                   // down/up blocks
  std::vector<int> C;                          // channels per level 0..n
  std::unordered_map<std::string, HostParam> raw;
  bool committed = false;
  std::vector<void*> owned, ws_owned;
  int64_t ws_bytes = 0, launches = 0;
  // packed weights
  ConvPack first;
  std::vector<ConvPack> down;
  std::vector<ResPack> res;
  std::vector<UpPack> up;
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

int dev_alloc(std::vector<void*>& owner, size_t nfloats, float** out, int64_t* counter = nullptr) {
  void* p = nullptr;
  const size_t bytes = std::max<size_t>(nfloats, 4) * sizeof(float);
  DAWN_CUDA_OK(cudaMalloc(&p, bytes));
  owner.push_back(p);
  if (counter) *counter += (int64_t)bytes;
  *out = (float*)p;
  return 0;
}
int dev_upload(dawn_lfg* h, const std::vector<float>& v, float** out) {
  LFG_TRY(dev_alloc(h->owned, v.size(), out));
  DAWN_CUDA_OK(cudaMemcpy(*out, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}
void free_all(std::vector<void*>& v) {
  for (void* p : v) cudaFree(p);
  v.clear();
}
int need(dawn_lfg* h, const std::string& name, std::vector<int64_t> shape, const HostParam** out) {
  auto it = h->raw.find(name);
  if (it == h->raw.end()) { set_last_error("lfg: missing parameter " + name); return -1; }
  if (it->second.shape != shape) { set_last_error("lfg: parameter " + name + " has an unexpected shape"); return -1; }
  *out = &it->second;
  return 0;
}
// eval-mode BatchNorm as y = x * s + t   (LFG/sync_batchnorm/batchnorm.py:50-53: F.batch_norm with running statistics, eps 1e-5)
int bn_affine(dawn_lfg* h, const std::string& p, int c, std::vector<double>& s, std::vector<double>& t) {
  const HostParam *g, *b, *rm, *rv;
  LFG_TRY(need(h, p + ".weight", {c}, &g));
  LFG_TRY(need(h, p + ".bias", {c}, &b));
  LFG_TRY(need(h, p + ".running_mean", {c}, &rm));
  LFG_TRY(need(h, p + ".running_var", {c}, &rv));
  s.resize(c); t.resize(c);
  for (int i = 0; i < c; ++i) {
    s[i] = (double)g->data[i] / std::sqrt((double)rv->data[i] + 1e-5);
    t[i] = (double)b->data[i] - (double)rm->data[i] * s[i];
  }
  return 0;
}
int upload_matrix(dawn_lfg* h, const std::vector<float>& m, const std::vector<float>& bias, int K, int N, int ldb, int ci_pad, ConvPack* out) {
  LFG_TRY(dev_upload(h, m, &out->w));
  out->img = nullptr; out->img_scale = 1.f;
  if (N % 64 == 0 && K % 64 == 0) {
    std::vector<float> im;
    tc_pack_weights(m.data(), K, N, ldb, im, &out->img_scale);
    LFG_TRY(dev_upload(h, im, &out->img));
  }
  std::vector<float> bb(ldb, 0.f);
  std::copy(bias.begin(), bias.end(), bb.begin());
  LFG_TRY(dev_upload(h, bb, &out->b));
  out->K = K; out->N = N; out->ldb = ldb; out->ci_pad = ci_pad;
  return 0;
}
// Conv2d weight (co, ci, k, k) [+ a following BatchNorm folded: W' = W * s[co], b' = b * s + t] -> [(ky*k + kx)*ci_pad + c][ldb]
int pack_conv(dawn_lfg* h, const std::string& conv, const std::string& bn_after, int co, int ci, int k, int ci_pad, ConvPack* out) {
  const HostParam *w, *b;
  LFG_TRY(need(h, conv + ".weight", {co, ci, k, k}, &w));
  LFG_TRY(need(h, conv + ".bias", {co}, &b));
  std::vector<double> s(co, 1.0), t(co, 0.0);
  if (!bn_after.empty()) LFG_TRY(bn_affine(h, bn_after, co, s, t));
  const int ldb = round_up(co, 64), K = k * k * ci_pad;
  std::vector<float> m((size_t)K * ldb, 0.f), bias(co);
  for (int n = 0; n < co; ++n) {
    bias[n] = (float)((double)b->data[n] * s[n] + t[n]);
    for (int c = 0; c < ci; ++c)
      for (int tp = 0; tp < k * k; ++tp)
        m[((size_t)tp * ci_pad + c) * ldb + n] = (float)((double)w->data[((size_t)n * ci + c) * k * k + tp] * s[n]);
  }
  return upload_matrix(h, m, bias, K, co, ldb, ci_pad, out);
}
// UpBlock2d (util.py:106-111): F.interpolate(scale_factor=2) [nearest] -> conv3x3 -> BN -> ReLU.  On the LOW-resolution grid the
// output pixel (2y+py, 2x+px) sees rows {y-1 (ky=0), y (ky=1,2)} for py=0 and {y (ky=0,1), y+1 (ky=2)} for py=1 (same for columns):
// each output-parity class is a 2x2 conv whose taps are sums of the 3x3 kernel's taps — 2.25x fewer MACs and the upsampled
// tensor never exists.  Zero padding is the same on both grids (upsampled index -1 / 2H <-> low-res index -1 / H).
const int kUpOff[2][2] = {{-1, 0}, {0, 1}};                     // [parity][tap] -> low-res offset
inline bool up_in_set(int parity, int tap, int k) {             // does kernel index k feed (parity, tap)?
  return parity == 0 ? (tap == 0 ? k == 0 : k >= 1) : (tap == 0 ? k <= 1 : k == 2);
}
int pack_up(dawn_lfg* h, const std::string& name, int co, int ci, UpPack* u) {
  const HostParam *w, *b;
  LFG_TRY(need(h, name + ".conv.weight", {co, ci, 3, 3}, &w));
  LFG_TRY(need(h, name + ".conv.bias", {co}, &b));
  std::vector<double> s, t;
  LFG_TRY(bn_affine(h, name + ".norm", co, s, t));
  std::vector<float> bias(co);
  for (int n = 0; n < co; ++n) bias[n] = (float)((double)b->data[n] * s[n] + t[n]);
  auto wsum = [&](int n, int c, int py, int ty, int px, int tx) {
    double acc = 0.0;
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx)
        if (up_in_set(py, ty, ky) && up_in_set(px, tx, kx)) acc += (double)w->data[(((size_t)n * ci + c) * 3 + ky) * 3 + kx];
    return (float)(acc * s[n]);
  };
  const int ldb = round_up(co, 64);
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      std::vector<float> m((size_t)4 * ci * ldb, 0.f);
      for (int ty = 0; ty < 2; ++ty)
        for (int tx = 0; tx < 2; ++tx)
          for (int c = 0; c < ci; ++c)
            for (int n = 0; n < co; ++n) m[((size_t)(ty * 2 + tx) * ci + c) * ldb + n] = wsum(n, c, py, ty, px, tx);
      LFG_TRY(upload_matrix(h, m, bias, 4 * ci, co, ldb, ci, &u->cls[py * 2 + px]));
    }
  u->has_all = (co == 64 && ci % 64 == 0);
  if (u->has_all) {
    const int N4 = 4 * co;
    std::vector<float> m((size_t)9 * ci * N4, 0.f), b4(N4);
    for (int py = 0; py < 2; ++py)
      for (int px = 0; px < 2; ++px) {
        const int cls = py * 2 + px;
        for (int n = 0; n < co; ++n) b4[cls * co + n] = bias[n];
        for (int ty = 0; ty < 2; ++ty)
          for (int tx = 0; tx < 2; ++tx) {
            const int tap = (kUpOff[py][ty] + 1) * 3 + (kUpOff[px][tx] + 1);
            for (int c = 0; c < ci; ++c)
              for (int n = 0; n < co; ++n) m[((size_t)tap * ci + c) * N4 + cls * co + n] = wsum(n, c, py, ty, px, tx);
          }
      }
    LFG_TRY(upload_matrix(h, m, b4, 9 * ci, N4, N4, ci, &u->all));
  }
  return 0;
}

// ------------------------------------------------------------------------------------------ contraction dispatch
void base_params(GemmParams& p, const float* A, int lda, int Cin, int frames, int Hh, int Ww) {
  memset(&p, 0, sizeof(p));
  p.A = A; p.lda = lda; p.Cin = Cin;
  p.IH = Hh; p.IW = Ww; p.OHs = Hh; p.OWs = Ww; p.in_stride = 1;
  p.ntaps = 1;
  p.M = frames * Hh * Ww; p.rows_per_batch = p.M;
  p.OH = Hh; p.OW = Ww; p.out_stride = 1;
  p.P = Hh * Ww;
  p.q_post_scale = 1.f;
  // 14 convolutions without a normalisation in between: the tensor core's round-toward-zero accumulation is a systematic bias that
  // compounds through the stack, so the register accumulators are drained into the RN fp32 tile every 3 taps / K panels (K = 192) instead
  // of every 9 / 4.
  p.drain = 3;
}
void set_weights(GemmParams& p, const ConvPack& w) {
  p.B = w.w; p.Bimg = w.img; p.tc_scale = 1.0f / (kTcActScale * w.img_scale); p.ldb = w.ldb; p.N = w.N; p.K = w.K; p.bias = w.b;
}
void set_square_taps(GemmParams& p, int k) {
  p.ntaps = k * k;
  for (int ky = 0; ky < k; ++ky)
    for (int kx = 0; kx < k; ++kx) { p.dy[ky * k + kx] = (signed char)(ky - k / 2); p.dx[ky * k + kx] = (signed char)(kx - k / 2); }
}
int run_conv(dawn_lfg* h, const GemmParams& p, cudaStream_t st) {
  h->launches++;
  if (p.Bimg != nullptr && tc_conv3_supported(p, EPI_PLAIN)) return launch_tc_conv3(p, p.Bimg, st);
  if (p.Bimg != nullptr && tc_gemm_supported(p, EPI_PLAIN)) return launch_tc_gemm(p, p.Bimg, EPI_PLAIN, st);
  return launch_gemm(p, EPI_PLAIN, st);
}
// out (frames, Hh, Ww, w.N) = conv kxk (same padding) of in (frames, Hh, Ww, Cin) + bias
int conv_same(dawn_lfg* h, const ConvPack& w, int k, const float* in, int Cin, int frames, int Hh, int Ww, float* out, cudaStream_t st) {
  GemmParams p; base_params(p, in, Cin, Cin, frames, Hh, Ww);
  set_weights(p, w); set_square_taps(p, k);
  p.Out = out; p.ldo = w.N;
  return run_conv(h, p, st);
}
// out (frames, 2Hh, 2Ww, co) = conv3x3(nearest_upsample_2x(in)) + bias (BatchNorm folded)
int conv_up(dawn_lfg* h, const UpPack& u, const float* in, int Cin, int frames, int Hh, int Ww, float* out, int co, cudaStream_t st) {
  if (u.has_all) {
    GemmParams p; base_params(p, in, Cin, Cin, frames, Hh, Ww);
    set_weights(p, u.all); set_square_taps(p, 3);
    p.up2 = 1; p.Out = out; p.ldo = co;
    if (p.Bimg != nullptr && tc_conv3_supported(p, EPI_PLAIN)) { h->launches++; return launch_tc_conv3(p, p.Bimg, st); }
  }
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      GemmParams p; base_params(p, in, Cin, Cin, frames, Hh, Ww);
      set_weights(p, u.cls[py * 2 + px]);
      p.ntaps = 4;
      for (int ty = 0; ty < 2; ++ty)
        for (int tx = 0; tx < 2; ++tx) { p.dy[ty * 2 + tx] = (signed char)kUpOff[py][ty]; p.dx[ty * 2 + tx] = (signed char)kUpOff[px][tx]; }
      p.OH = 2 * Hh; p.OW = 2 * Ww; p.out_stride = 2; p.oy0 = py; p.ox0 = px;
      p.Out = out; p.ldo = co;
      LFG_TRY(run_conv(h, p, st));
    }
  return 0;
}

int decode_core(dawn_lfg* h, float* prediction, float* deformed, cudaStream_t st) {
  const int n = h->n, F = h->F;
  const int Cb = h->C[n], Hn = h->lH[n], Wn = h->lW[n];
  const long long Mn = (long long)F * Hn * Wn;
  // generator.py:154: out = warp(skip_n) * occ
  h->launches++;
  LFG_TRY(launch_lfg_warp_blend(h->SKIP[n], Cb, Hn, Wn, h->MOTION, F, h->fh, h->fw, nullptr, 0, h->X, Cb, st));
  // generator.py:156: bottleneck of pre-activation ResBlocks (util.py:85-93)
  const int nres = (int)h->res.size();
  if (nres > 0) {
    h->launches++;
    LFG_TRY(launch_lfg_affine_relu(h->X, Cb, h->res[0].s1, h->res[0].t1, Cb, Mn, h->Z, Cb, st));
  }
  for (int r = 0; r < nres; ++r) {
    LFG_TRY(conv_same(h, h->res[r].c1, 3, h->Z, Cb, F, Hn, Wn, h->Y, st));            // conv1 (+ norm2 folded)
    h->launches++;
    LFG_TRY(launch_lfg_affine_relu(h->Y, Cb, nullptr, nullptr, Cb, Mn, h->Y, Cb, st)); // relu
    LFG_TRY(conv_same(h, h->res[r].c2, 3, h->Y, Cb, F, Hn, Wn, h->Z, st));            // conv2
    const bool more = r + 1 < nres;
    h->launches++;
    LFG_TRY(launch_lfg_residual_bn_relu(h->Z, h->X, Cb, Mn, h->X, more ? h->res[r + 1].s1 : nullptr, more ? h->res[r + 1].t1 : nullptr,
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
      LFG_TRY(launch_lfg_warp_blend(h->SKIP[l], Cl, Hl, Wl, h->MOTION, F, h->fh, h->fw, prev, Cl, bl, Cl, st));
      in = bl;
    }
    LFG_TRY(conv_up(h, h->up[i], in, Cl, F, Hl, Wl, h->UP[l - 1], Co, st));
    h->launches++;
    LFG_TRY(launch_lfg_affine_relu(h->UP[l - 1], Co, nullptr, nullptr, Co, (long long)F * h->lH[l - 1] * h->lW[l - 1], h->UP[l - 1], Co, st));
    prev = h->UP[l - 1];
  }
  // generator.py:161-167: last skip blend, 7x7 conv + sigmoid, blend with the warped source image
  const float* fin = prev;
  if (h->cfg.skips) {
    h->launches++;
    LFG_TRY(launch_lfg_warp_blend(h->SKIP[0], h->C[0], h->H, h->W, h->MOTION, F, h->fh, h->fw, prev, h->C[0], h->BL[0], h->C[0], st));
    fin = h->BL[0];
  }
  h->launches++;
  LFG_TRY(launch_lfg_final(fin, h->C[0], h->C[0], F, h->H, h->W, h->final_w, h->final_b, h->SRC, h->MOTION, h->fh, h->fw,
                           h->cfg.skips ? 1 : 0, prediction, deformed, st));
  h->decoded = true;
  return 0;
}

}  // namespace

extern "C" {

int dawn_check_single_device(void);          // unet.cu: one GPU per process

int dawn_lfg_create(const dawn_lfg_cfg* cfg, dawn_lfg** out) {
  LFG_CHECK(cfg && out, "null argument");
  LFG_TRY(dawn_check_single_device());
  LFG_CHECK(cfg->num_channels == 3, "lfg: num_channels must be 3");
  LFG_CHECK(cfg->block_expansion % 64 == 0 && cfg->block_expansion <= 128, "lfg: block_expansion must be 64 or 128");
  LFG_CHECK(cfg->num_down_blocks >= 1 && cfg->num_down_blocks <= 4, "lfg: num_down_blocks out of range");
  LFG_CHECK(cfg->num_bottleneck_blocks >= 0 && cfg->num_bottleneck_blocks <= 32, "lfg: num_bottleneck_blocks out of range");
  dawn_lfg* h = new dawn_lfg();
  h->cfg = *cfg;
  h->n = cfg->num_down_blocks;
  for (int i = 0; i <= h->n; ++i) h->C.push_back(std::min(cfg->max_features, cfg->block_expansion << i));     // generator.py:40-50
  *out = h;
  return 0;
}

void dawn_lfg_destroy(dawn_lfg* h) {
  if (!h) return;
  free_all(h->owned);
  free_all(h->ws_owned);
  delete h;
}

int dawn_lfg_set_param(dawn_lfg* h, const char* name, const float* host, const int64_t* shape, int ndim) {
  LFG_CHECK(h && name && (shape || ndim == 0), "null argument");
  const std::string n(name);
  if (n.rfind("pixelwise_flow_predictor.", 0) == 0) return 0;                     // never read by forward_with_flow (generator.py:138-171)
  if (n.size() >= 19 && n.compare(n.size() - 19, 19, "num_batches_tracked") == 0) return 0;
  LFG_CHECK(host, "null argument");
  HostParam p;
  p.shape.assign(shape, shape + ndim);
  int64_t numel = 1;
  for (int i = 0; i < ndim; ++i) numel *= shape[i];
  p.data.assign(host, host + numel);
  h->raw[n] = std::move(p);
  h->committed = false;
  return 0;
}

int dawn_lfg_commit_params(dawn_lfg* h) {
  LFG_CHECK(h, "null handle");
  free_all(h->owned);
  h->down.clear(); h->res.clear(); h->up.clear();
  const int n = h->n;
  LFG_TRY(pack_conv(h, "first.conv", "first.norm", h->C[0], h->cfg.num_channels, 7, 32, &h->first));           // generator.py:36
  for (int i = 0; i < n; ++i) {
    ConvPack d;
    const std::string p = "down_blocks." + std::to_string(i);
    LFG_TRY(pack_conv(h, p + ".conv", p + ".norm", h->C[i + 1], h->C[i], 3, h->C[i], &d));                       // generator.py:38-44
    h->down.push_back(d);
  }
  const int Cb = h->C[n];
  for (int r = 0; r < h->cfg.num_bottleneck_blocks; ++r) {
    ResPack rp;
    const std::string p = "bottleneck.r" + std::to_string(r);
    LFG_TRY(pack_conv(h, p + ".conv1", p + ".norm2", Cb, Cb, 3, Cb, &rp.c1));      // util.py:88-89: conv1 -> norm2 folded
    LFG_TRY(pack_conv(h, p + ".conv2", "", Cb, Cb, 3, Cb, &rp.c2));
    std::vector<double> s, t;
    LFG_TRY(bn_affine(h, p + ".norm1", Cb, s, t));
    std::vector<float> sf(s.begin(), s.end()), tf(t.begin(), t.end());
    LFG_TRY(dev_upload(h, sf, &rp.s1));
    LFG_TRY(dev_upload(h, tf, &rp.t1));
    h->res.push_back(rp);
  }
  for (int i = 0; i < n; ++i) {
    UpPack u;
    LFG_TRY(pack_up(h, "up_blocks." + std::to_string(i), h->C[n - i - 1], h->C[n - i], &u));                     // generator.py:46-52
    h->up.push_back(u);
  }
  {
    const HostParam *w, *b;
    LFG_TRY(need(h, "final.weight", {3, h->C[0], 7, 7}, &w));
    LFG_TRY(need(h, "final.bias", {3}, &b));
    std::vector<float> wp((size_t)49 * h->C[0] * 4, 0.f), bp(4, 0.f);
    for (int o = 0; o < 3; ++o) {
      bp[o] = b->data[o];
      for (int c = 0; c < h->C[0]; ++c)
        for (int t = 0; t < 49; ++t) wp[((size_t)t * h->C[0] + c) * 4 + o] = w->data[((size_t)o * h->C[0] + c) * 49 + t];
    }
    LFG_TRY(dev_upload(h, wp, &h->final_w));
    LFG_TRY(dev_upload(h, bp, &h->final_b));
  }
  h->committed = true;
  h->have_source = false;
  return 0;
}

int dawn_lfg_set_geometry(dawn_lfg* h, int frames, int H, int W, int flow_h, int flow_w) {
  LFG_CHECK(h, "null handle");
  LFG_CHECK(h->committed, "lfg: commit_params must precede set_geometry");
  LFG_CHECK(frames >= 1 && frames <= 65535, "lfg: frames out of range");
  const int n = h->n, div = 1 << n;
  LFG_CHECK(H >= div && W >= div && H % div == 0 && W % div == 0, "lfg: image height/width must be divisible by 2^num_down_blocks");
  LFG_CHECK(flow_h >= 1 && flow_w >= 1, "lfg: bad flow size");
  free_all(h->ws_owned);
  h->ws_bytes = 0;
  h->F = frames; h->H = H; h->W = W; h->fh = flow_h; h->fw = flow_w;
  h->lH.assign(n + 1, 0); h->lW.assign(n + 1, 0);
  for (int l = 0; l <= n; ++l) { h->lH[l] = H >> l; h->lW[l] = W >> l; }
  auto& own = h->ws_owned;
  int64_t* cnt = &h->ws_bytes;
  const size_t P0 = (size_t)H * W;
  LFG_TRY(dev_alloc(own, 3 * P0, &h->SRC, cnt));
  LFG_TRY(dev_alloc(own, 32 * P0, &h->SRC_HWC, cnt));
  size_t tmp = 0;
  for (int l = 0; l < n; ++l) tmp = std::max(tmp, (size_t)h->lH[l] * h->lW[l] * h->C[l + 1]);
  LFG_TRY(dev_alloc(own, tmp, &h->TMP, cnt));
  h->SKIP.assign(n + 1, nullptr); h->UP.assign(n + 1, nullptr); h->BL.assign(n + 1, nullptr);
  for (int l = 0; l <= n; ++l) LFG_TRY(dev_alloc(own, (size_t)h->lH[l] * h->lW[l] * h->C[l], &h->SKIP[l], cnt));
  for (int l = 0; l < n; ++l) {
    const size_t e = (size_t)frames * h->lH[l] * h->lW[l] * h->C[l];
    LFG_TRY(dev_alloc(own, e, &h->UP[l], cnt));
    if (h->cfg.skips) LFG_TRY(dev_alloc(own, e, &h->BL[l], cnt));
  }
  const size_t eb = (size_t)frames * h->lH[n] * h->lW[n] * h->C[n];
  LFG_TRY(dev_alloc(own, eb, &h->X, cnt));
  LFG_TRY(dev_alloc(own, eb, &h->Y, cnt));
  LFG_TRY(dev_alloc(own, eb, &h->Z, cnt));
  { float* m; LFG_TRY(dev_alloc(own, (size_t)frames * flow_h * flow_w * 4, &m, cnt)); h->MOTION = (float4*)m; }
  h->have_source = false; h->decoded = false;
  return 0;
}

int dawn_lfg_set_source(dawn_lfg* h, const float* source, void* stream) {
  LFG_CHECK(h && source, "null argument");
  LFG_CHECK(h->F > 0, "lfg: set_geometry must precede set_source");
  cudaStream_t st = (cudaStream_t)stream;
  const int n = h->n, H = h->H, W = h->W;
  h->launches = 0;
  DAWN_CUDA_OK(cudaMemcpyAsync(h->SRC, source, (size_t)3 * H * W * sizeof(float), cudaMemcpyDeviceToDevice, st));
  h->launches++;
  LFG_TRY(launch_lfg_chw_to_hwc(source, 3, H * W, 32, h->SRC_HWC, st));
  // first: conv7x7 -> BN -> ReLU (util.py:147-150), BN folded
  LFG_TRY(conv_same(h, h->first, 7, h->SRC_HWC, 32, 1, H, W, h->SKIP[0], st));
  h->launches++;
  LFG_TRY(launch_lfg_affine_relu(h->SKIP[0], h->C[0], nullptr, nullptr, h->C[0], (long long)H * W, h->SKIP[0], h->C[0], st));
  // down blocks: conv3x3 -> BN -> ReLU -> avgpool 2x2 (util.py:126-131)
  for (int i = 0; i < n; ++i) {
    LFG_TRY(conv_same(h, h->down[i], 3, h->SKIP[i], h->C[i], 1, h->lH[i], h->lW[i], h->TMP, st));
    h->launches++;
    LFG_TRY(launch_lfg_relu_avgpool2(h->TMP, h->lH[i], h->lW[i], h->C[i + 1], h->SKIP[i + 1], st));
  }
  h->have_source = true;
  return 0;
}

int dawn_lfg_get_fea(dawn_lfg* h, float* fea, void* stream) {
  LFG_CHECK(h && fea, "null argument");
  LFG_CHECK(h->have_source, "lfg: set_source must precede get_fea");
  const int n = h->n;
  return launch_lfg_hwc_to_chw(h->SKIP[n], h->C[n], h->C[n], (long long)h->lH[n] * h->lW[n], fea, (cudaStream_t)stream);
}

int dawn_lfg_decode(dawn_lfg* h, const float* flow, const float* occ, float* prediction, float* deformed, void* stream) {
  LFG_CHECK(h && flow && occ && prediction, "null argument");
  LFG_CHECK(h->have_source, "lfg: set_source must precede decode");
  cudaStream_t st = (cudaStream_t)stream;
  h->launches = 1;
  LFG_TRY(launch_lfg_motion_pack(flow, occ, 0, h->F, h->fh, h->fw, h->MOTION, st));
  return decode_core(h, prediction, deformed, st);
}

int dawn_lfg_decode_sample(dawn_lfg* h, const float* sample, float* prediction, float* deformed, void* stream) {
  LFG_CHECK(h && sample && prediction, "null argument");
  LFG_CHECK(h->have_source, "lfg: set_source must precede decode");
  cudaStream_t st = (cudaStream_t)stream;
  h->launches = 1;
  LFG_TRY(launch_lfg_motion_pack(sample, nullptr, 1, h->F, h->fh, h->fw, h->MOTION, st));
  return decode_core(h, prediction, deformed, st);
}

int dawn_lfg_read_tap(dawn_lfg* h, const char* name, float* dst, int* C, int* Hl, int* Wl, void* stream) {
  LFG_CHECK(h && name && C && Hl && Wl, "null argument");
  LFG_CHECK(h->F > 0, "lfg: set_geometry first");
  const std::string nm(name);
  const int n = h->n;
  const float* src = nullptr;
  int level = -1;
  if (nm == "bottleneck") { src = h->X; level = n; }
  else if (nm.rfind("up", 0) == 0 && nm.size() == 3 && nm[2] >= '0' && nm[2] < '0' + n) { level = n - 1 - (nm[2] - '0'); src = h->UP[level]; }
  LFG_CHECK(src != nullptr, "lfg: unknown tap " + nm);
  *C = h->C[level]; *Hl = h->lH[level]; *Wl = h->lW[level];
  if (!dst) return 0;
  LFG_CHECK(h->decoded, "lfg: decode must precede read_tap");
  return launch_lfg_hwc_to_chw(src, *C, *C, (long long)h->F * *Hl * *Wl, dst, (cudaStream_t)stream);
}

// one layer of Face_loc_Encoder (FD:39-50): relu(conv3x3 stride 2 pad 1); all device pointers, weights as nn.Conv2d stores them
int dawn_conv3x3_s2_relu(const float* x, int Ci, int H, int W, const float* weight, const float* bias, int Co, float* out, void* stream) {
  LFG_CHECK(x && weight && bias && out && Ci >= 1 && Co >= 1 && H >= 1 && W >= 1, "dawn_conv3x3_s2_relu: bad argument");
  return launch_conv3x3_s2_relu(x, Ci, H, W, weight, bias, Co, out, (cudaStream_t)stream);
}

int64_t dawn_lfg_last_launch_count(dawn_lfg* h) { return h ? h->launches : 0; }
int64_t dawn_lfg_workspace_bytes(dawn_lfg* h) { return h ? h->ws_bytes : 0; }

}  // extern "C"
