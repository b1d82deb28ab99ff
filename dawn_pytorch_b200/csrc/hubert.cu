// Host-side folds, orchestration and C-ABI of the HuBERT audio encoder (include/dawn_hubert.h): the eval forward of
// transformers' HubertModel with feat_extract_norm "layer" and do_stable_layer_norm (hubert-large-ls960-ft).
//
// One forward, for a feature extractor of n convs and L encoder layers, is 2 n + G + 7 L + 3 launches (no split passes):
//   conv 0 + LayerNorm + GELU | per conv i >= 1: strided conv (contraction), LayerNorm + GELU | row statistics, feature
//   projection (LayerNorm folded) | grouped re-layout, one contraction per positional-conv group (GELU + residual epilogue) |
//   per layer: row statistics, q|k|v (LayerNorm folded), attention, out_proj + residual, row statistics, fc1 (final_layer_norm
//   folded, GELU), fc2 + residual | the encoder's LayerNorm into the output.
// The strided convs are implicit GEMMs over channels-last rows: output t of a kernel-k stride-s conv gathers taps t s + j,
// j < k, through the contraction's tap offsets (in_stride = s), so neither an im2col copy nor overlapping row windows are
// needed.  The positional conv's groups are re-laid out as padded 64-channel planes: the 64 x k window of output t is then one
// contiguous run, read as a 1x1 contraction with K = 64 k over rows of stride 64.
#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "../../include/dawn_hubert.h"
#include "common.cuh"
#include "contraction.cuh"
#include "gemm.cuh"
#include "hubert_kernels.cuh"
#include "kernels.cuh"

using namespace dawn;

namespace {

constexpr float kConvLnEps = 1e-5f;      // the feature extractor's nn.LayerNorm keeps torch's default eps

struct LnLinear {                        // a Linear with the LayerNorm before it folded in: W' = W diag(gamma), b' = b + W beta
  PackedWeight w;
  float* wsum = nullptr;                 // [ldb] column sums of W'
};

struct LayerPack {
  LnLinear qkv, fc1;
  PackedWeight out, fc2;
};

}  // namespace

struct dawn_hubert {
  dawn_hubert_cfg cfg{};
  HostParams raw{{}, "hubert: "};
  bool committed = false;
  DeviceArena weights, workspace;
  int64_t launches = 0;
  // packed parameters
  float *w0 = nullptr, *b0 = nullptr;                       // conv 0 (k0, C0) k-major, bias
  PackedWeight conv[DAWN_HUBERT_MAX_CONV];                  // convs >= 1: (k Cin, Cout), tap-major rows
  float *conv_ln[DAWN_HUBERT_MAX_CONV][2] = {};
  LnLinear proj;
  std::vector<PackedWeight> pos;                            // one (64 k, 64) matrix per group, bias slice
  std::vector<LayerPack> layers;
  float *enc_ln[2] = {};
  // workspace
  long long cap_fe[2] = {0, 0}, cap_T = 0, cap_xg = 0;
  float *FE[2] = {}, *H = nullptr, *QKV = nullptr, *O = nullptr, *F1 = nullptr, *RS = nullptr, *XG = nullptr;
};

namespace {

int out_len(int L, int k, int s) { return L < k ? 0 : (L - k) / s + 1; }

int upload_vec(dawn_hubert* h, const std::string& name, int n, float** out) {
  const HostParam* p;
  DAWN_TRY(h->raw.need(name, {n}, &p));
  return h->weights.upload(p->data, out);
}

struct LinearPart {                     // one nn.Linear of a LayerNorm-folded projection: W (Nj, K), b (Nj), output scale
  const float* w;
  const float* b;
  float scale;
};

// nn.Linear weights (N_j, K) of `parts` side by side in the output columns, k-major (K, sum N_j), each scaled by its factor
// (an exact power of two), with the LayerNorm (gamma, beta over K) folded in, in fp64:
//   W'[k][n] = W[n][k] gamma[k] sc,  b'[n] = (b[n] + sum_k W[n][k] beta[k]) sc,  wsum[n] = sum_k W'[k][n]
int pack_ln_linear(DeviceArena& arena, const std::vector<LinearPart>& parts, int Nj, int K, const float* gamma, const float* beta,
                   LnLinear* out) {
  const int N = Nj * (int)parts.size(), ldb = round_up(N, 64);
  std::vector<float> m((size_t)K * ldb, 0.f), bias(N), wsum(ldb, 0.f);
  for (size_t j = 0; j < parts.size(); ++j) {
    const double sc = parts[j].scale;
    for (int n = 0; n < Nj; ++n) {
      const float* wr = parts[j].w + (size_t)n * K;
      const int col = (int)j * Nj + n;
      double bb = parts[j].b[n], ws = 0.0;
      for (int k = 0; k < K; ++k) {
        const float v = (float)((double)wr[k] * (double)gamma[k] * sc);
        m[(size_t)k * ldb + col] = v;
        ws += v;
        bb += (double)wr[k] * (double)beta[k];
      }
      bias[col] = (float)(bb * sc);
      wsum[col] = (float)ws;
    }
  }
  DAWN_TRY(upload_weight(arena, m, K, N, ldb, bias, &out->w));
  return arena.upload(wsum, &out->wsum);
}

// the same from the handle's parameters: (Linear name, scale) per part, the LayerNorm's name
int pack_ln_linear(dawn_hubert* h, const std::vector<std::pair<std::string, float>>& names, int Nj, int K, const std::string& ln,
                   LnLinear* out) {
  const HostParam *g, *be;
  DAWN_TRY(h->raw.need(ln + ".weight", {K}, &g));
  DAWN_TRY(h->raw.need(ln + ".bias", {K}, &be));
  std::vector<LinearPart> parts;
  for (const auto& nm : names) {
    const HostParam *w, *b;
    DAWN_TRY(h->raw.need(nm.first + ".weight", {Nj, K}, &w));
    DAWN_TRY(h->raw.need(nm.first + ".bias", {Nj}, &b));
    parts.push_back({w->data.data(), b->data.data(), nm.second});
  }
  return pack_ln_linear(h->weights, parts, Nj, K, g->data.data(), be->data.data(), out);
}

// feature-extractor conv >= 1: Conv1d weight (co, ci, k) -> tap-major (k ci, co) rows, bias (co) or null (conv_bias false)
int pack_fe_conv(DeviceArena& arena, const float* w, const float* bias, int co, int ci, int k, PackedWeight* out) {
  std::vector<float> m((size_t)k * ci * co);
  pack_conv_taps(w, co, ci, k, ci, co, 0, nullptr, m);
  return upload_weight(arena, m, k * ci, co, co, bias ? std::vector<float>(bias, bias + co) : std::vector<float>(co, 0.f), out);
}

// nn.Linear (N, K) + bias -> k-major packed weight
int pack_linear(dawn_hubert* h, const std::string& name, int N, int K, PackedWeight* out) {
  const HostParam *w, *b;
  DAWN_TRY(h->raw.need(name + ".weight", {N, K}, &w));
  DAWN_TRY(h->raw.need(name + ".bias", {N}, &b));
  const int ldb = round_up(N, 64);
  std::vector<float> m((size_t)K * ldb, 0.f);
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) m[(size_t)k * ldb + n] = w->data[(size_t)n * K + k];
  return upload_weight(h->weights, m, K, N, ldb, b->data, out);
}

// positional conv: weight_norm over dim 2 (w[o][i][t] = g[t] v[o][i][t] / ||v[:, :, t]||, fp64), then per group gi the
// (64 k, 64) matrix whose row t 64 + i is input channel i of window row t, and the group's bias slice
int pack_pos_conv(DeviceArena& arena, const float* g, const float* v, const float* bias, int D, int k, int G,
                  std::vector<PackedWeight>& out) {
  std::vector<double> inv(k, 0.0);
  for (size_t e = 0; e < (size_t)D * 64 * k; ++e) inv[e % k] += (double)v[e] * (double)v[e];
  for (int t = 0; t < k; ++t) inv[t] = (double)g[t] / std::sqrt(inv[t]);
  out.assign(G, PackedWeight{});
  for (int gi = 0; gi < G; ++gi) {
    std::vector<float> m((size_t)k * 64 * 64);
    for (int o = 0; o < 64; ++o)
      for (int i = 0; i < 64; ++i)
        for (int t = 0; t < k; ++t)
          m[((size_t)t * 64 + i) * 64 + o] = (float)((double)v[((size_t)(gi * 64 + o) * 64 + i) * k + t] * inv[t]);
    DAWN_TRY(upload_weight(arena, m, 64 * k, 64, 64, std::vector<float>(bias + gi * 64, bias + gi * 64 + 64), &out[gi]));
  }
  return 0;
}

int run(const GemmParams& p, int epi, cudaStream_t st, int64_t* launches) {
  int kernels = 0;
  DAWN_TRY(launch_path(p, epi, choose_path(p, epi, 0), nullptr, st, &kernels));
  *launches += kernels;
  return 0;
}

// h (B * T, 64 G) += GELU(conv(h)): xg holds the padded group planes
int run_pos_conv(const std::vector<PackedWeight>& pos, const float* h, int B, int T, int k, float* xg, float* out, cudaStream_t st,
                 int64_t* launches) {
  const int G = (int)pos.size(), pad = k / 2, Tp = T + 2 * pad, D = 64 * G;
  DAWN_TRY(launch_hb_group_pad(h, B, T, G, pad, xg, st));
  ++*launches;
  for (int gi = 0; gi < G; ++gi) {
    GemmParams p;
    base_params(p, xg + (size_t)gi * B * Tp * 64, 64, 64 * k, B, 1, Tp);
    p.OWs = p.OW = T; p.M = p.rows_per_batch = B * T; p.P = T;
    set_weights(p, pos[gi]);
    p.Out = out + gi * 64; p.ldo = D;
    p.Res = h + gi * 64; p.ldr = D;
    DAWN_TRY(run(p, EPI_GELU, st, launches));
  }
  return 0;
}

// feature-extractor conv >= 1 of B sequences, Tin -> Tout rows: dst (B Tout, co) = GELU(LayerNorm(conv(in))), gamma / beta = ln[0 / 1]
int run_fe_conv(const PackedWeight& w, const float* const ln[2], const float* in, int B, int Tin, int Tout, int ci, int co, int k, int s,
                float* dst, cudaStream_t st, int64_t* launches) {
  GemmParams p;
  base_params(p, in, ci, ci, B, 1, Tin);
  p.OWs = p.OW = Tout; p.M = p.rows_per_batch = B * Tout; p.P = Tout;
  p.in_stride = s;
  p.ntaps = k;
  for (int t = 0; t < p.ntaps; ++t) { p.dy[t] = 0; p.dx[t] = (signed char)t; }
  set_weights(p, w);
  p.Out = dst; p.ldo = co;
  DAWN_TRY(run(p, EPI_PLAIN, st, launches));
  DAWN_TRY(launch_hb_row_ln(dst, co, B * Tout, co, ln[0], ln[1], kConvLnEps, 1, dst, co, st));
  ++*launches;
  return 0;
}

// a pre-LN projection of `rows` dense rows of K: the rows' (mu, rstd) into rs, then the contraction through the fold
int run_ln_linear(const LnLinear& w, const float* A, int K, int rows, float eps, int epi, float* rs, float* dst, cudaStream_t st,
                  int64_t* launches) {
  DAWN_TRY(launch_rowstats(A, K, K, rows, eps, rs, st));
  ++*launches;
  GemmParams p;
  base_params(p, A, K, K, 1, 1, rows);
  set_weights(p, w.w);
  p.rowstats = rs; p.wsum = w.wsum;
  p.Out = dst; p.ldo = w.w.N;
  return run(p, epi, st, launches);
}

int ensure_workspace(dawn_hubert* h, long long fe0, long long fe1, long long BT, long long xg) {
  if (fe0 <= h->cap_fe[0] && fe1 <= h->cap_fe[1] && BT <= h->cap_T && xg <= h->cap_xg) return 0;
  h->workspace.release();
  const long long c0 = std::max(fe0, h->cap_fe[0]), c1 = std::max(fe1, h->cap_fe[1]), cT = std::max(BT, h->cap_T),
                  cx = std::max(xg, h->cap_xg);
  const dawn_hubert_cfg& c = h->cfg;
  auto& ws = h->workspace;
  auto alloc = [&]() -> int {
    DAWN_TRY(ws.alloc((size_t)c0, &h->FE[0]));
    DAWN_TRY(ws.alloc((size_t)c1, &h->FE[1]));
    DAWN_TRY(ws.alloc((size_t)cT * c.hidden_size, &h->H));
    DAWN_TRY(ws.alloc((size_t)cT * 3 * c.hidden_size, &h->QKV));
    DAWN_TRY(ws.alloc((size_t)cT * c.hidden_size, &h->O));
    DAWN_TRY(ws.alloc((size_t)cT * c.intermediate_size, &h->F1));
    DAWN_TRY(ws.alloc((size_t)cT * 2, &h->RS));
    DAWN_TRY(ws.alloc((size_t)cx, &h->XG));
    return 0;
  };
  const int rc = alloc();
  if (rc != 0) {
    h->workspace.release();
    h->cap_fe[0] = h->cap_fe[1] = h->cap_T = h->cap_xg = 0;
    return rc;
  }
  h->cap_fe[0] = c0; h->cap_fe[1] = c1; h->cap_T = cT; h->cap_xg = cx;
  return 0;
}

std::string conv_prefix(int i) { return "feature_extractor.conv_layers." + std::to_string(i) + "."; }
std::string layer_prefix(int l) { return "encoder.layers." + std::to_string(l) + "."; }

int refuse_case(const char* why) {
  set_last_error(std::string("hubert test: ") + why);
  return -1;
}

}  // namespace

extern "C" {

int dawn_hubert_create(const dawn_hubert_cfg* cfg, dawn_hubert** out) {
  DAWN_CHECK(cfg && out, "null argument");
  DAWN_TRY(dawn_check_single_device());
  const dawn_hubert_cfg& c = *cfg;
  DAWN_CHECK(c.num_heads >= 1 && c.hidden_size == kHbHeadDim * c.num_heads,
             "hubert: hidden_size must be 64 x num_attention_heads (heads 64 wide)");
  DAWN_CHECK(c.hidden_size <= kHbMaxC, "hubert: hidden_size must be at most " + std::to_string(kHbMaxC));
  DAWN_CHECK(c.intermediate_size >= 64 && c.intermediate_size % 64 == 0, "hubert: intermediate_size must be a positive multiple of 64");
  DAWN_CHECK(c.num_layers >= 1 && c.num_layers <= 64, "hubert: num_hidden_layers must be 1 to 64");
  DAWN_CHECK(c.num_conv >= 1 && c.num_conv <= DAWN_HUBERT_MAX_CONV,
             "hubert: the feature extractor must have 1 to " + std::to_string(DAWN_HUBERT_MAX_CONV) + " conv layers");
  for (int i = 0; i < c.num_conv; ++i) {
    DAWN_CHECK(c.conv_dim[i] >= 64 && c.conv_dim[i] % 64 == 0 && c.conv_dim[i] <= kHbMaxC,
               "hubert: conv_dim must be multiples of 64 up to " + std::to_string(kHbMaxC));
    DAWN_CHECK(c.conv_kernel[i] >= 1 && c.conv_kernel[i] <= (i == 0 ? 64 : 52) && c.conv_stride[i] >= 1,
               "hubert: conv_kernel must be 1 to 64 (layer 0) or 52 (later layers), conv_stride positive");
  }
  DAWN_CHECK(c.pos_kernel >= 1 && c.pos_kernel <= 1024, "hubert: num_conv_pos_embeddings must be 1 to 1024");
  DAWN_CHECK(c.pos_groups >= 1 && c.hidden_size == 64 * c.pos_groups,
             "hubert: num_conv_pos_embedding_groups must be hidden_size / 64 (64-channel groups)");
  DAWN_CHECK(c.layer_norm_eps > 0.f, "hubert: layer_norm_eps must be positive");
  dawn_hubert* h = new dawn_hubert();
  h->cfg = c;
  *out = h;
  return 0;
}

void dawn_hubert_destroy(dawn_hubert* h) { delete h; }

int dawn_hubert_set_param(dawn_hubert* h, const char* name, const float* host, const int64_t* shape, int ndim) {
  DAWN_CHECK(h && name && host && (shape || ndim == 0), "null argument");
  h->raw.set(name, host, shape, ndim);
  h->committed = false;
  return 0;
}

int dawn_hubert_commit_params(dawn_hubert* h) {
  DAWN_CHECK(h, "null handle");
  h->weights.release();
  h->layers.clear();
  h->pos.clear();
  h->committed = false;
  const dawn_hubert_cfg& c = h->cfg;
  const int D = c.hidden_size, I = c.intermediate_size;
  const HostParams& raw = h->raw;
  // ---- feature extractor
  for (int i = 0; i < c.num_conv; ++i) {
    const std::string p = conv_prefix(i);
    const int co = c.conv_dim[i], ci = i == 0 ? 1 : c.conv_dim[i - 1], k = c.conv_kernel[i];
    const HostParam *w, *b = nullptr;
    DAWN_TRY(raw.need(p + "conv.weight", {co, ci, k}, &w));
    if (c.conv_bias) DAWN_TRY(raw.need(p + "conv.bias", {co}, &b));
    if (i == 0) {
      std::vector<float> m((size_t)k * co);
      for (int n = 0; n < co; ++n)
        for (int t = 0; t < k; ++t) m[(size_t)t * co + n] = w->data[(size_t)n * k + t];
      DAWN_TRY(h->weights.upload(m, &h->w0));
      if (b) DAWN_TRY(h->weights.upload(b->data, &h->b0));
    } else {
      DAWN_TRY(pack_fe_conv(h->weights, w->data.data(), b ? b->data.data() : nullptr, co, ci, k, &h->conv[i]));
    }
    DAWN_TRY(upload_vec(h, p + "layer_norm.weight", co, &h->conv_ln[i][0]));
    DAWN_TRY(upload_vec(h, p + "layer_norm.bias", co, &h->conv_ln[i][1]));
  }
  const int Cl = c.conv_dim[c.num_conv - 1];
  DAWN_TRY(pack_ln_linear(h, {{"feature_projection.projection", 1.f}}, D, Cl, "feature_projection.layer_norm", &h->proj));
  // ---- positional conv
  {
    const HostParam *g, *v, *b;
    DAWN_TRY(raw.need("encoder.pos_conv_embed.conv.weight_g", {1, 1, c.pos_kernel}, &g));
    DAWN_TRY(raw.need("encoder.pos_conv_embed.conv.weight_v", {D, 64, c.pos_kernel}, &v));
    DAWN_TRY(raw.need("encoder.pos_conv_embed.conv.bias", {D}, &b));
    DAWN_TRY(pack_pos_conv(h->weights, g->data.data(), v->data.data(), b->data.data(), D, c.pos_kernel, c.pos_groups, h->pos));
  }
  // ---- encoder layers
  const float qscale = 1.0f / std::sqrt((float)kHbHeadDim);        // head_dim ** -0.5 = 1/8, exact
  for (int l = 0; l < c.num_layers; ++l) {
    const std::string p = layer_prefix(l);
    LayerPack lp;
    DAWN_TRY(pack_ln_linear(h, {{p + "attention.q_proj", qscale}, {p + "attention.k_proj", 1.f}, {p + "attention.v_proj", 1.f}}, D, D,
                            p + "layer_norm", &lp.qkv));
    DAWN_TRY(pack_linear(h, p + "attention.out_proj", D, D, &lp.out));
    DAWN_TRY(pack_ln_linear(h, {{p + "feed_forward.intermediate_dense", 1.f}}, I, D, p + "final_layer_norm", &lp.fc1));
    DAWN_TRY(pack_linear(h, p + "feed_forward.output_dense", D, I, &lp.fc2));
    h->layers.push_back(lp);
  }
  DAWN_TRY(upload_vec(h, "encoder.layer_norm.weight", D, &h->enc_ln[0]));
  DAWN_TRY(upload_vec(h, "encoder.layer_norm.bias", D, &h->enc_ln[1]));
  h->committed = true;
  return 0;
}

int dawn_hubert_output_length(const dawn_hubert* h, int L) {
  if (!h) return 0;
  for (int i = 0; i < h->cfg.num_conv; ++i) L = out_len(L, h->cfg.conv_kernel[i], h->cfg.conv_stride[i]);
  return L;
}

}  // extern "C"

namespace {

// the forward through the first `layers` encoder layers; final_ln: then the encoder's LayerNorm into out, else the hidden state
int run_forward(dawn_hubert* h, const float* input, int B, int L, int layers, bool final_ln, float* out, cudaStream_t st) {
  DAWN_CHECK(h && input && out, "null argument");
  DAWN_CHECK(h->committed, "hubert: commit_params must precede forward");
  const dawn_hubert_cfg& c = h->cfg;
  DAWN_CHECK(B >= 1 && B <= 65535 && L >= 1, "hubert: B must be 1 to 65535 and L positive");
  int Ts[DAWN_HUBERT_MAX_CONV];
  long long fe[2] = {0, 0};
  {
    int len = L;
    for (int i = 0; i < c.num_conv; ++i) {
      len = Ts[i] = out_len(len, c.conv_kernel[i], c.conv_stride[i]);
      DAWN_CHECK(len >= 1, "hubert: the input is shorter than the feature extractor's receptive field");
      fe[i & 1] = std::max(fe[i & 1], (long long)B * len * c.conv_dim[i]);
    }
  }
  const int T = Ts[c.num_conv - 1], D = c.hidden_size, k = c.pos_kernel;
  DAWN_CHECK((long long)B * T * c.intermediate_size < (1LL << 31) && fe[0] < (1LL << 31), "hubert: B x L too large for one call");
  const long long BT = (long long)B * T;
  DAWN_TRY(ensure_workspace(h, fe[0], fe[1], BT, (long long)c.pos_groups * B * (T + 2 * (k / 2)) * 64));
  h->launches = 0;
  // ---- feature extractor
  DAWN_TRY(launch_hb_conv0(input, B, L, h->w0, h->b0, c.conv_kernel[0], c.conv_stride[0], c.conv_dim[0], h->conv_ln[0][0],
                           h->conv_ln[0][1], kConvLnEps, h->FE[0], st));
  h->launches++;
  for (int i = 1; i < c.num_conv; ++i)
    DAWN_TRY(run_fe_conv(h->conv[i], h->conv_ln[i], h->FE[(i - 1) & 1], B, Ts[i - 1], Ts[i], c.conv_dim[i - 1], c.conv_dim[i],
                         c.conv_kernel[i], c.conv_stride[i], h->FE[i & 1], st, &h->launches));
  const float* feat = h->FE[(c.num_conv - 1) & 1];
  const int Cl = c.conv_dim[c.num_conv - 1];
  // pre-LN projections: row statistics, then the LayerNorm folded into the Linear
  auto ln_gemm = [&](const float* A, int K, const LnLinear& w, int epi, float* dst) -> int {
    return run_ln_linear(w, A, K, (int)BT, c.layer_norm_eps, epi, h->RS, dst, st, &h->launches);
  };
  auto res_gemm = [&](const float* A, int K, const PackedWeight& w, float* hid) -> int {
    GemmParams p;
    base_params(p, A, K, K, 1, 1, (int)BT);
    set_weights(p, w);
    p.Out = hid; p.ldo = D; p.Res = hid; p.ldr = D;
    return run(p, EPI_PLAIN, st, &h->launches);
  };
  DAWN_TRY(ln_gemm(feat, Cl, h->proj, EPI_LN_BIAS, h->H));
  // ---- positional conv: h += GELU(conv(h))
  DAWN_TRY(run_pos_conv(h->pos, h->H, B, T, k, h->XG, h->H, st, &h->launches));
  // ---- encoder layers
  for (int l = 0; l < layers; ++l) {
    const LayerPack& lp = h->layers[l];
    DAWN_TRY(ln_gemm(h->H, D, lp.qkv, EPI_LN_BIAS, h->QKV));
    DAWN_TRY(launch_hb_attention(h->QKV, h->QKV + D, h->QKV + 2 * D, 3 * D, B, T, c.num_heads, h->O, D, st));
    h->launches++;
    DAWN_TRY(res_gemm(h->O, D, lp.out, h->H));
    DAWN_TRY(ln_gemm(h->H, D, lp.fc1, EPI_LN_BIAS_GELU, h->F1));
    DAWN_TRY(res_gemm(h->F1, c.intermediate_size, lp.fc2, h->H));
  }
  if (final_ln) {
    DAWN_TRY(launch_hb_row_ln(h->H, D, (int)BT, D, h->enc_ln[0], h->enc_ln[1], c.layer_norm_eps, 0, out, D, st));
    h->launches++;
  } else {
    DAWN_CUDA_OK(cudaMemcpyAsync(out, h->H, (size_t)BT * D * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  return 0;
}

}  // namespace

extern "C" {

int dawn_hubert_forward(dawn_hubert* h, const float* input, int B, int L, float* out, void* stream) {
  DAWN_CHECK(h, "null handle");
  return run_forward(h, input, B, L, h->cfg.num_layers, true, out, (cudaStream_t)stream);
}

int dawn_hubert_hidden(dawn_hubert* h, const float* input, int B, int L, int layers, float* out, void* stream) {
  DAWN_CHECK(h, "null handle");
  DAWN_CHECK(layers >= 0 && layers <= h->cfg.num_layers, "hubert: layers must be 0 to num_hidden_layers");
  return run_forward(h, input, B, L, layers, false, out, (cudaStream_t)stream);
}

int64_t dawn_hubert_last_launch_count(dawn_hubert* h) { return h ? h->launches : 0; }
int64_t dawn_hubert_workspace_bytes(dawn_hubert* h) { return h ? h->workspace.bytes() : 0; }

int dawn_hubert_test_kernel(const dawn_hubert_kernel_case* c, void* stream) {
  if (!c || !c->out) return refuse_case("null case or output");
  cudaStream_t st = (cudaStream_t)stream;
  switch (c->kernel) {
    case DAWN_HUBERT_ATTENTION:
      if (!c->q || !c->kk || !c->v) return refuse_case("attention needs q, k and v");
      if (c->ldo != 0 && c->ldo < kHbHeadDim * c->H) return refuse_case("attention ldo must be 0 or at least 64 H");
      DAWN_TRY(launch_hb_attention(c->q, c->kk, c->v, c->ld, c->B, c->T, c->H, c->out, c->ldo ? c->ldo : kHbHeadDim * c->H, st));
      break;
    case DAWN_HUBERT_ROW_LN:
      if (!c->x || !c->gamma || !c->beta) return refuse_case("row LayerNorm needs x, gamma and beta");
      if (c->ld < c->C || c->ldo < c->C) return refuse_case("row LayerNorm strides must be at least C");
      DAWN_TRY(launch_hb_row_ln(c->x, c->ld, c->M, c->C, c->gamma, c->beta, c->eps, c->gelu, c->out, c->ldo, st));
      break;
    case DAWN_HUBERT_FE_CONV: {
      if (!c->x || !c->w || !c->gamma || !c->beta) return refuse_case("feature-extractor conv needs x, w, gamma and beta");
      if (c->B < 1 || c->k < 1 || c->k > 52 || c->s < 1 || c->L < c->k || c->C < 64 || c->C % 64 || c->N < 64 || c->N % 64 ||
          c->N > kHbMaxC)
        return refuse_case("bad feature-extractor conv geometry");
      std::vector<float> hw((size_t)c->N * c->C * c->k), hb;
      DAWN_CUDA_OK(cudaMemcpy(hw.data(), c->w, hw.size() * sizeof(float), cudaMemcpyDeviceToHost));
      if (c->bias) {
        hb.resize(c->N);
        DAWN_CUDA_OK(cudaMemcpy(hb.data(), c->bias, hb.size() * sizeof(float), cudaMemcpyDeviceToHost));
      }
      DeviceArena arena;
      PackedWeight w;
      DAWN_TRY(pack_fe_conv(arena, hw.data(), c->bias ? hb.data() : nullptr, c->N, c->C, c->k, &w));
      const float* ln[2] = {c->gamma, c->beta};
      int64_t launches = 0;
      DAWN_TRY(run_fe_conv(w, ln, c->x, c->B, c->L, out_len(c->L, c->k, c->s), c->C, c->N, c->k, c->s, c->out, st, &launches));
      DAWN_CUDA_OK(cudaStreamSynchronize(st));
      break;
    }
    case DAWN_HUBERT_LN_LINEAR: {
      if (!c->x || !c->w || !c->bias || !c->gamma || !c->beta) return refuse_case("LayerNorm + Linear needs x, w, bias, gamma and beta");
      if (c->M < 1 || c->C < 64 || c->C % 64 || c->C > kHbMaxC || c->N < 1 || c->parts < 1 || c->parts > 3)
        return refuse_case("bad LayerNorm + Linear geometry");
      const int N = c->parts * c->N;
      std::vector<float> hw((size_t)N * c->C), hb(N), hg(c->C), hbe(c->C);
      DAWN_CUDA_OK(cudaMemcpy(hw.data(), c->w, hw.size() * sizeof(float), cudaMemcpyDeviceToHost));
      DAWN_CUDA_OK(cudaMemcpy(hb.data(), c->bias, hb.size() * sizeof(float), cudaMemcpyDeviceToHost));
      DAWN_CUDA_OK(cudaMemcpy(hg.data(), c->gamma, hg.size() * sizeof(float), cudaMemcpyDeviceToHost));
      DAWN_CUDA_OK(cudaMemcpy(hbe.data(), c->beta, hbe.size() * sizeof(float), cudaMemcpyDeviceToHost));
      std::vector<LinearPart> parts;
      for (int j = 0; j < c->parts; ++j)
        parts.push_back({hw.data() + (size_t)j * c->N * c->C, hb.data() + (size_t)j * c->N, j == 0 ? c->qscale : 1.f});
      DeviceArena arena;
      LnLinear lin;
      DAWN_TRY(pack_ln_linear(arena, parts, c->N, c->C, hg.data(), hbe.data(), &lin));
      float* rs;
      DAWN_TRY(arena.alloc((size_t)c->M * 2, &rs));
      int64_t launches = 0;
      DAWN_TRY(run_ln_linear(lin, c->x, c->C, c->M, c->eps, c->gelu ? EPI_LN_BIAS_GELU : EPI_LN_BIAS, rs, c->out, st, &launches));
      DAWN_CUDA_OK(cudaStreamSynchronize(st));
      break;
    }
    case DAWN_HUBERT_CONV0:
      if (!c->x || !c->w || !c->gamma || !c->beta) return refuse_case("conv0 needs x, w, gamma and beta");
      if (c->k < 1 || c->k > 64) return refuse_case("conv0 kernel must be 1 to 64");
      {
        // (C, 1, k) -> (k, C) k-major, as commit_params packs it
        std::vector<float> hw((size_t)c->C * c->k), m(hw.size());
        DAWN_CUDA_OK(cudaMemcpy(hw.data(), c->w, hw.size() * sizeof(float), cudaMemcpyDeviceToHost));
        for (int n = 0; n < c->C; ++n)
          for (int t = 0; t < c->k; ++t) m[(size_t)t * c->C + n] = hw[(size_t)n * c->k + t];
        DeviceArena arena;
        float* w0;
        DAWN_TRY(arena.upload(m, &w0));
        DAWN_TRY(launch_hb_conv0(c->x, c->B, c->L, w0, c->bias, c->k, c->s, c->C, c->gamma, c->beta, c->eps, c->out, st));
        DAWN_CUDA_OK(cudaStreamSynchronize(st));
      }
      break;
    case DAWN_HUBERT_POS_CONV: {
      if (!c->x || !c->w || !c->g || !c->bias) return refuse_case("pos conv needs x, w, g and bias");
      if (c->G < 1 || c->k < 1 || c->k > 1024 || c->B < 1 || c->T < 1) return refuse_case("bad pos conv geometry");
      const int D = 64 * c->G;
      std::vector<float> hg(c->k), hv((size_t)D * 64 * c->k), hb(D);
      DAWN_CUDA_OK(cudaMemcpy(hg.data(), c->g, hg.size() * sizeof(float), cudaMemcpyDeviceToHost));
      DAWN_CUDA_OK(cudaMemcpy(hv.data(), c->w, hv.size() * sizeof(float), cudaMemcpyDeviceToHost));
      DAWN_CUDA_OK(cudaMemcpy(hb.data(), c->bias, hb.size() * sizeof(float), cudaMemcpyDeviceToHost));
      DeviceArena arena;
      std::vector<PackedWeight> pos;
      DAWN_TRY(pack_pos_conv(arena, hg.data(), hv.data(), hb.data(), D, c->k, c->G, pos));
      float* xg;
      DAWN_TRY(arena.alloc((size_t)c->G * c->B * (c->T + 2 * (c->k / 2)) * 64, &xg));
      int64_t launches = 0;
      DAWN_TRY(run_pos_conv(pos, c->x, c->B, c->T, c->k, xg, c->out, st, &launches));
      DAWN_CUDA_OK(cudaStreamSynchronize(st));
      break;
    }
    default:
      return refuse_case("unknown kernel");
  }
  DAWN_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
