// Host-side packing, orchestration and C-ABI of the PBnet pose / blink decoder (include/dawn_pbnet.h; reference
// PBnet/src/models/architectures/transformerreemb5.py:311-378, transformerdecoder4.py:24-221).
//
// One generate, for L layers, is 7 L + 1 launches:
//   rotary table | audio contraction (audioEmbedding with ztimelinear's audio slice folded in) | memory rows | k, v of the
//   memory for every layer's cross-attention | layer 0: q, cross-attention, to_out + LN2, FFN + LN3 | layers 1..L-1: q k v,
//   self-attention, to_out + LN1, q, cross-attention, to_out + LN2, FFN + LN3 (the last one also runs finallayer + mask).
// The queries entering the decoder are init_proj(0), one row for every frame.  init_temporal_attn and the first layer's
// self-attention then average identical value rows with softmax weights that sum to 1, so their result is that same row: it is
// evaluated once per commit on the host (fp64) and the first layer starts at its cross-attention.
#include <algorithm>
#include <cmath>
#include <initializer_list>
#include <string>
#include <vector>

#include "../../include/dawn_pbnet.h"
#include "common.cuh"
#include "contraction.cuh"
#include "gemm.cuh"
#include "kernels.cuh"
#include "pbnet_kernels.cuh"

using namespace dawn;

namespace {

struct LayerPack {
  float *w_qkv = nullptr, *w_out_self = nullptr;          // self-attention (layers >= 1)
  float *w_q = nullptr, *w_out_cross = nullptr;           // cross-attention
  float *w1 = nullptr, *b1 = nullptr, *w2 = nullptr, *b2 = nullptr;
  float *ln[3][2] = {};                                   // layer_norm1..3 weight, bias
};

}  // namespace

struct dawn_pbnet {
  dawn_pbnet_cfg cfg{};
  int D = 0, hid = 0, npairs = 0, nout = 0;
  HostParams raw{{}, "pbnet: "};
  bool committed = false;
  DeviceArena weights, workspace;
  int64_t launches = 0;
  // packed parameters
  PackedWeight aud;                                       // (audio_dim, D): audioEmbedding folded through ztimelinear
  float *wz = nullptr, *wp = nullptr;                     // ztimelinear's z slice (Lz, D); first-pose slice folded (pose_dim, D)
  float *w_kv = nullptr;                                  // (D, 2 hid L): k_l | v_l of every layer's cross-attention
  float *c0 = nullptr;                                    // (D): the frame-invariant row entering layer 0's cross-attention
  float *freqs = nullptr, *bias_tgt = nullptr, *bias_mem = nullptr;
  float *wf = nullptr, *bf = nullptr;
  std::vector<LayerPack> layers;
  // workspace
  int cap_T = 0, cap_F = 0;
  float *AUD = nullptr, *MEM = nullptr, *X = nullptr, *KV = nullptr, *QKV = nullptr, *O = nullptr, *ROT = nullptr;
};

namespace {

// nn.Linear weight (N, K) -> k-major (K, N), optionally into columns [n0, n0 + N) of a (K, ldn) matrix
void transpose_into(const float* w, int N, int K, std::vector<float>& m, int ldn, int n0) {
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) m[(size_t)k * ldn + n0 + n] = w[(size_t)n * K + k];
}

int upload_linear_t(dawn_pbnet* h, const std::string& name, int N, int K, float** out) {
  const HostParam* w;
  DAWN_TRY(h->raw.need(name, {N, K}, &w));
  std::vector<float> m((size_t)K * N);
  transpose_into(w->data.data(), N, K, m, N, 0);
  return h->weights.upload(m, out);
}

int upload_vec(dawn_pbnet* h, const std::string& name, const std::vector<int64_t>& shape, float** out) {
  const HostParam* p;
  DAWN_TRY(h->raw.need(name, shape, &p));
  return h->weights.upload(p->data, out);
}

// y = W x (+ b), W (N, K) row-major fp32, in fp64
std::vector<double> matvec(const HostParam& w, const std::vector<double>& x, const HostParam* b) {
  const int N = (int)w.shape[0], K = (int)w.shape[1];
  std::vector<double> y(N);
  for (int n = 0; n < N; ++n) {
    double a = b ? (double)b->data[n] : 0.0;
    for (int k = 0; k < K; ++k) a += (double)w.data[(size_t)n * K + k] * x[k];
    y[n] = a;
  }
  return y;
}
// rows [r0, r0 + n) of W as their own (n, K) parameter
HostParam row_slice(const HostParam& w, int r0, int n) {
  HostParam s;
  const int K = (int)w.shape[1];
  s.shape = {n, K};
  s.data.assign(w.data.begin() + (size_t)r0 * K, w.data.begin() + (size_t)(r0 + n) * K);
  return s;
}
// (x - mean) / sqrt(var + 1e-5) * gamma (+ beta), biased variance (reemb5:16-25 with gamma only; nn.LayerNorm with beta)
std::vector<double> layer_norm(const std::vector<double>& x, const float* gamma, const float* beta) {
  const size_t n = x.size();
  double mean = 0.0, var = 0.0;
  for (double v : x) mean += v;
  mean /= (double)n;
  for (double v : x) var += (v - mean) * (v - mean);
  var /= (double)n;
  const double rstd = 1.0 / std::sqrt(var + 1e-5);
  std::vector<double> y(n);
  for (size_t i = 0; i < n; ++i) y[i] = (x[i] - mean) * rstd * gamma[i] + (beta ? beta[i] : 0.0);
  return y;
}

std::string layer_prefix(int l) { return "seqTransDecoder.decoder_layers." + std::to_string(l) + "."; }

// the frame-invariant prefix of the decoder, in fp64: init_proj(0) -> Residual(PreNorm(Attention)) -> layer 0's
// self-attention + layer_norm1.  Attention over identical rows returns to_out(v) of that row.
int frame_invariant_row(const dawn_pbnet* h, std::vector<double>& row) {
  const int D = h->D, hid = h->hid;
  const HostParam *b0, *g, *qkv, *out, *qkv0, *out0, *ln_w, *ln_b;
  DAWN_TRY(h->raw.need("init_proj.bias", {D}, &b0));
  DAWN_TRY(h->raw.need("init_proj.weight", {D, D}, &g));                        // multiplies zeros: only its shape is checked
  DAWN_TRY(h->raw.need("init_temporal_attn.fn.norm.gamma", {1, 1, D}, &g));
  DAWN_TRY(h->raw.need("init_temporal_attn.fn.fn.to_qkv.weight", {3 * hid, D}, &qkv));
  DAWN_TRY(h->raw.need("init_temporal_attn.fn.fn.to_out.weight", {D, hid}, &out));
  const std::string p = layer_prefix(0);
  DAWN_TRY(h->raw.need(p + "self_attn.to_qkv.weight", {3 * hid, D}, &qkv0));
  DAWN_TRY(h->raw.need(p + "self_attn.to_out.weight", {D, hid}, &out0));
  DAWN_TRY(h->raw.need(p + "layer_norm1.weight", {D}, &ln_w));
  DAWN_TRY(h->raw.need(p + "layer_norm1.bias", {D}, &ln_b));
  std::vector<double> t0(b0->data.begin(), b0->data.end());
  const std::vector<double> n0 = layer_norm(t0, g->data.data(), nullptr);
  const std::vector<double> a0 = matvec(*out, matvec(row_slice(*qkv, 2 * hid, hid), n0, nullptr), nullptr);
  std::vector<double> t1(D);
  for (int c = 0; c < D; ++c) t1[c] = a0[c] + t0[c];
  const std::vector<double> a1 = matvec(*out0, matvec(row_slice(*qkv0, 2 * hid, hid), t1, nullptr), nullptr);
  for (int c = 0; c < D; ++c) t1[c] += a1[c];
  row = layer_norm(t1, ln_w->data.data(), ln_b->data.data());
  return 0;
}

int ensure_workspace(dawn_pbnet* h, int T, int F) {
  if (T <= h->cap_T && F <= h->cap_F) return 0;
  h->workspace.release();
  const int D = h->D, hid = h->hid, L = h->cfg.num_layers;
  const int cT = std::max(T, h->cap_T), cF = std::max(F, h->cap_F);
  auto& ws = h->workspace;
  auto alloc = [&]() -> int {
    DAWN_TRY(ws.alloc((size_t)cT * D, &h->AUD));
    DAWN_TRY(ws.alloc((size_t)cT * D, &h->MEM));
    DAWN_TRY(ws.alloc((size_t)cT * D, &h->X));
    DAWN_TRY(ws.alloc((size_t)cT * 2 * hid * L, &h->KV));
    DAWN_TRY(ws.alloc((size_t)cT * 3 * hid, &h->QKV));
    DAWN_TRY(ws.alloc((size_t)cT * hid, &h->O));
    DAWN_TRY(ws.alloc((size_t)cF * h->npairs * 2, &h->ROT));
    return 0;
  };
  const int rc = alloc();
  if (rc != 0) {
    h->workspace.release();
    h->cap_T = h->cap_F = 0;
    return rc;
  }
  h->cap_T = cT; h->cap_F = cF;
  return 0;
}

PbProjGroups groups_of(std::initializer_list<int> flags) {
  PbProjGroups g{};
  int i = 0;
  for (int f : flags) g.flags[i++] = f;
  return g;
}

}  // namespace

extern "C" {

int dawn_pbnet_create(const dawn_pbnet_cfg* cfg, dawn_pbnet** out) {
  DAWN_CHECK(cfg && out, "null argument");
  DAWN_TRY(dawn_check_single_device());
  const dawn_pbnet_cfg& c = *cfg;
  DAWN_CHECK(c.band == 200 || c.band == 100, "pbnet: band must be 200 (transformerreemb5) or 100 (transformerreemb6)");
  DAWN_CHECK(c.pose_dim >= 1 && c.pose_dim <= kPbMaxOut, "pbnet: pos_dim + eye_dim must be 1 to " + std::to_string(kPbMaxOut));
  DAWN_CHECK(c.audio_dim >= 64 && c.audio_dim % 64 == 0, "pbnet: audio_dim must be a positive multiple of 64");
  DAWN_CHECK(c.audio_latent_dim >= 1 && c.latent_dim == c.audio_latent_dim,
             "pbnet: latent_dim must equal audio_latent_dim (z is concatenated as an audio_latent_dim-wide slice, reemb5:326)");
  DAWN_CHECK(c.pose_latent_dim >= 32 && c.pose_latent_dim <= kPbMaxD && c.pose_latent_dim % 32 == 0,
             "pbnet: pose_latent_dim must be a multiple of 32 from 32 to " + std::to_string(kPbMaxD));
  DAWN_CHECK(c.ff_size >= 1 && c.ff_size <= kPbMaxFF, "pbnet: ff_size must be 1 to " + std::to_string(kPbMaxFF));
  DAWN_CHECK(c.num_layers >= 1 && 2 * c.num_layers <= kPbMaxGroups, "pbnet: num_layers must be 1 to " + std::to_string(kPbMaxGroups / 2));
  DAWN_CHECK(c.num_heads >= 2 && c.num_heads <= kPbMaxHeads && c.num_heads % 2 == 0,
             "pbnet: num_heads must be even and at most " + std::to_string(kPbMaxHeads));
  dawn_pbnet* h = new dawn_pbnet();
  h->cfg = c;
  h->D = c.pose_latent_dim;
  h->hid = 32 * c.num_heads;
  h->npairs = std::min(32, c.num_heads) / 2;
  h->nout = c.pose_dim;
  *out = h;
  return 0;
}

void dawn_pbnet_destroy(dawn_pbnet* h) {
  delete h;
}

int dawn_pbnet_set_param(dawn_pbnet* h, const char* name, const float* host, const int64_t* shape, int ndim) {
  DAWN_CHECK(h && name && host && (shape || ndim == 0), "null argument");
  h->raw.set(name, host, shape, ndim);
  h->committed = false;
  return 0;
}

int dawn_pbnet_commit_params(dawn_pbnet* h) {
  DAWN_CHECK(h, "null handle");
  h->weights.release();
  h->layers.clear();
  h->committed = false;
  const dawn_pbnet_cfg& c = h->cfg;
  const int D = h->D, hid = h->hid, L = c.num_layers, P = c.pose_dim, A = c.audio_latent_dim, K = c.audio_dim;
  const HostParams& raw = h->raw;
  // ---- memory rows: ztimelinear(cat[firstposeEmbedding(x0), z, audioEmbedding(y)]) (reemb5:321-327), folded in fp64
  const HostParam *wzt, *bzt, *wa, *ba, *wfp, *bfp;
  DAWN_TRY(raw.need("ztimelinear.weight", {D, D + 2 * A}, &wzt));
  DAWN_TRY(raw.need("ztimelinear.bias", {D}, &bzt));
  DAWN_TRY(raw.need("audioEmbedding.weight", {A, K}, &wa));
  DAWN_TRY(raw.need("audioEmbedding.bias", {A}, &ba));
  DAWN_TRY(raw.need("firstposeEmbedding.weight", {D, P}, &wfp));
  DAWN_TRY(raw.need("firstposeEmbedding.bias", {D}, &bfp));
  const int ldz = D + 2 * A;
  auto zt = [&](int n, int col) { return (double)wzt->data[(size_t)n * ldz + col]; };
  {
    std::vector<double> acc((size_t)K * D, 0.0);                 // k-major (K, D): sum_j Wzt[n][D + A + j] Wa[j][k]
    for (int n = 0; n < D; ++n)
      for (int j = 0; j < A; ++j) {
        const double s = zt(n, D + A + j);
        const float* war = wa->data.data() + (size_t)j * K;
        for (int k = 0; k < K; ++k) acc[(size_t)k * D + n] += s * (double)war[k];
      }
    const int ldb = round_up(D, 64);
    std::vector<float> m((size_t)K * ldb, 0.f), bias(D);
    for (int k = 0; k < K; ++k)
      for (int n = 0; n < D; ++n) m[(size_t)k * ldb + n] = (float)acc[(size_t)k * D + n];
    for (int n = 0; n < D; ++n) {
      double b = (double)bzt->data[n];
      for (int j = 0; j < A; ++j) b += zt(n, D + A + j) * (double)ba->data[j];
      for (int j = 0; j < D; ++j) b += zt(n, j) * (double)bfp->data[j];
      bias[n] = (float)b;
    }
    DAWN_TRY(upload_weight(h->weights, m, K, D, ldb, bias, &h->aud));
    std::vector<float> wz((size_t)A * D), wp((size_t)P * D);
    for (int k = 0; k < A; ++k)
      for (int n = 0; n < D; ++n) wz[(size_t)k * D + n] = wzt->data[(size_t)n * ldz + D + k];
    for (int p = 0; p < P; ++p)
      for (int n = 0; n < D; ++n) {
        double s = 0.0;
        for (int j = 0; j < D; ++j) s += zt(n, j) * (double)wfp->data[(size_t)j * P + p];
        wp[(size_t)p * D + n] = (float)s;
      }
    DAWN_TRY(h->weights.upload(wz, &h->wz));
    DAWN_TRY(h->weights.upload(wp, &h->wp));
  }
  // ---- frame-invariant prefix
  {
    std::vector<double> row;
    DAWN_TRY(frame_invariant_row(h, row));
    DAWN_TRY(h->weights.upload(std::vector<float>(row.begin(), row.end()), &h->c0));
  }
  // ---- layers
  std::vector<float> kv((size_t)D * 2 * hid * L);
  for (int l = 0; l < L; ++l) {
    const std::string p = layer_prefix(l);
    LayerPack lp;
    if (l > 0) {
      DAWN_TRY(upload_linear_t(h, p + "self_attn.to_qkv.weight", 3 * hid, D, &lp.w_qkv));
      DAWN_TRY(upload_linear_t(h, p + "self_attn.to_out.weight", D, hid, &lp.w_out_self));
    }
    DAWN_TRY(upload_linear_t(h, p + "multihead_attn.to_q.weight", hid, D, &lp.w_q));
    DAWN_TRY(upload_linear_t(h, p + "multihead_attn.to_out.weight", D, hid, &lp.w_out_cross));
    const HostParam *wk, *wv;
    DAWN_TRY(raw.need(p + "multihead_attn.to_k.weight", {hid, D}, &wk));
    DAWN_TRY(raw.need(p + "multihead_attn.to_v.weight", {hid, D}, &wv));
    transpose_into(wk->data.data(), hid, D, kv, 2 * hid * L, 2 * hid * l);
    transpose_into(wv->data.data(), hid, D, kv, 2 * hid * L, 2 * hid * l + hid);
    DAWN_TRY(upload_linear_t(h, p + "ffn.linear1.weight", c.ff_size, D, &lp.w1));
    DAWN_TRY(upload_vec(h, p + "ffn.linear1.bias", {c.ff_size}, &lp.b1));
    DAWN_TRY(upload_linear_t(h, p + "ffn.linear2.weight", D, c.ff_size, &lp.w2));
    DAWN_TRY(upload_vec(h, p + "ffn.linear2.bias", {D}, &lp.b2));
    for (int i = 0; i < 3; ++i) {
      const std::string ln = p + "layer_norm" + std::to_string(i + 1);
      DAWN_TRY(upload_vec(h, ln + ".weight", {D}, &lp.ln[i][0]));
      DAWN_TRY(upload_vec(h, ln + ".bias", {D}, &lp.ln[i][1]));
    }
    h->layers.push_back(lp);
  }
  DAWN_TRY(h->weights.upload(kv, &h->w_kv));
  DAWN_TRY(upload_linear_t(h, "finallayer.weight", P, D, &h->wf));
  DAWN_TRY(upload_vec(h, "finallayer.bias", {P}, &h->bf));
  DAWN_TRY(upload_vec(h, layer_prefix(L - 1) + "multihead_attn.rotary_emb.freqs", {h->npairs}, &h->freqs));
  DAWN_TRY(upload_vec(h, "aux.bias_tgt", {c.num_heads, 2 * c.band + 1}, &h->bias_tgt));
  DAWN_TRY(upload_vec(h, "aux.bias_mem", {c.num_heads, 2 * c.band + 1}, &h->bias_mem));
  h->committed = true;
  return 0;
}

int dawn_pbnet_generate(dawn_pbnet* h, const float* audio, const float* z, const float* first_pose, const unsigned char* mask,
                        int bs, int F, float* out, void* stream) {
  DAWN_CHECK(h && audio && z && first_pose && mask && out, "null argument");
  DAWN_CHECK(h->committed, "pbnet: commit_params must precede generate");
  DAWN_CHECK(bs >= 1 && F >= 1 && (long long)bs * F <= (1 << 24), "pbnet: bs x F out of range");
  cudaStream_t st = (cudaStream_t)stream;
  const dawn_pbnet_cfg& c = h->cfg;
  const int T = bs * F, D = h->D, hid = h->hid, L = c.num_layers, H = c.num_heads, band = c.band;
  const int ldkv = 2 * hid * L;
  const float qscale = 1.0f / std::sqrt(32.0f);                  // dim_head ** -0.5 (transformerdecoder4.py:33)
  DAWN_TRY(ensure_workspace(h, T, F));
  h->launches = 0;
  DAWN_TRY(launch_rotary_table(h->freqs, h->npairs, F, 0, h->ROT, st));
  h->launches++;
  {
    GemmParams p; base_params(p, audio, c.audio_dim, c.audio_dim, 1, 1, T);
    set_weights(p, h->aud);
    p.Out = h->AUD; p.ldo = D;
    int kernels = 0;
    DAWN_TRY(launch_path(p, EPI_PLAIN, choose_path(p, EPI_PLAIN, 0), nullptr, st, &kernels));
    h->launches += kernels;
  }
  DAWN_TRY(launch_pb_memory(h->AUD, z, c.latent_dim, h->wz, first_pose, c.pose_dim, h->wp, bs, F, D, h->MEM, st));
  h->launches++;
  {
    PbProjGroups g{};
    for (int l = 0; l < L; ++l) g.flags[2 * l] = PB_ROTARY;        // k rotated, v not (transformerdecoder4.py:146-148)
    DAWN_TRY(launch_pb_proj(h->MEM, D, T, F, D, h->w_kv, hid, 2 * L, g, 1.f, h->ROT, h->npairs, h->KV, st));
    h->launches++;
  }
  int attn = 0;                                                    // attention launches: one per 65 535 clips per site
  for (int l = 0; l < L; ++l) {
    const LayerPack& lp = h->layers[l];
    const float* xin = h->c0;
    int ldx = 0;
    if (l > 0) {                                                   // self-attention + layer_norm1 (transformerdecoder4.py:202)
      DAWN_TRY(launch_pb_proj(h->X, D, T, F, D, lp.w_qkv, hid, 3, groups_of({PB_SCALE | PB_ROTARY, PB_ROTARY, 0}), qscale, h->ROT,
                              h->npairs, h->QKV, st));
      DAWN_TRY(launch_pb_attention(h->QKV, 3 * hid, h->QKV + hid, 3 * hid, h->QKV + 2 * hid, 3 * hid, h->bias_tgt, band, bs, F, H,
                                   h->O, st, &attn));
      DAWN_TRY(launch_pb_out_ln(h->O, hid, lp.w_out_self, h->X, D, lp.ln[0][0], lp.ln[0][1], T, D, h->X, st));
      h->launches += 2;
      xin = h->X; ldx = D;
    }
    // cross-attention over the memory + layer_norm2 (:203)
    DAWN_TRY(launch_pb_proj(xin, ldx, T, F, D, lp.w_q, hid, 1, groups_of({PB_SCALE | PB_ROTARY}), qscale, h->ROT, h->npairs, h->QKV, st));
    DAWN_TRY(launch_pb_attention(h->QKV, hid, h->KV + 2 * hid * l, ldkv, h->KV + 2 * hid * l + hid, ldkv, h->bias_mem, band, bs, F, H,
                                 h->O, st, &attn));
    DAWN_TRY(launch_pb_out_ln(h->O, hid, lp.w_out_cross, xin, ldx, lp.ln[1][0], lp.ln[1][1], T, D, h->X, st));
    // FFN + layer_norm3 (:204); after the last layer finallayer + the length mask (reemb5:370-374)
    const bool last = l + 1 == L;
    DAWN_TRY(launch_pb_ffn_ln(h->X, T, D, lp.w1, lp.b1, c.ff_size, lp.w2, lp.b2, lp.ln[2][0], lp.ln[2][1], last ? h->wf : nullptr,
                              last ? h->bf : nullptr, h->nout, mask, out, st));
    h->launches += 3;
  }
  h->launches += attn;
  return 0;
}

int64_t dawn_pbnet_last_launch_count(dawn_pbnet* h) { return h ? h->launches : 0; }
int64_t dawn_pbnet_workspace_bytes(dawn_pbnet* h) { return h ? h->workspace.bytes() : 0; }

int dawn_pbnet_test_attention(const dawn_pbnet_attention_case* c, void* stream) {
  DAWN_CHECK(c && c->x_q && c->x_kv && c->wq && c->wk && c->wv && c->freqs && c->bias && c->out, "pbnet test: missing pointer");
  DAWN_CHECK(c->bs >= 1 && c->F >= 1 && c->D >= 32 && c->D <= kPbMaxD && c->D % 32 == 0 && c->H >= 1 && c->H <= kPbMaxHeads &&
                 c->band >= 0 && c->npairs >= 0 && c->npairs <= 16,
             "pbnet test: bad geometry");
  cudaStream_t st = (cudaStream_t)stream;
  const int T = c->bs * c->F, hid = 32 * c->H;
  DeviceArena arena;
  float *rot, *q, *k, *v;
  DAWN_TRY(arena.alloc((size_t)c->F * std::max(c->npairs, 1) * 2, &rot));
  DAWN_TRY(arena.alloc((size_t)T * hid, &q));
  DAWN_TRY(arena.alloc((size_t)T * hid, &k));
  DAWN_TRY(arena.alloc((size_t)T * hid, &v));
  if (c->npairs > 0) DAWN_TRY(launch_rotary_table(c->freqs, c->npairs, c->F, 0, rot, st));
  DAWN_TRY(launch_pb_proj(c->x_q, c->D, T, c->F, c->D, c->wq, hid, 1, groups_of({PB_SCALE | PB_ROTARY}), c->qscale, rot, c->npairs, q, st));
  DAWN_TRY(launch_pb_proj(c->x_kv, c->D, T, c->F, c->D, c->wk, hid, 1, groups_of({PB_ROTARY}), 1.f, rot, c->npairs, k, st));
  DAWN_TRY(launch_pb_proj(c->x_kv, c->D, T, c->F, c->D, c->wv, hid, 1, groups_of({0}), 1.f, rot, c->npairs, v, st));
  DAWN_TRY(launch_pb_attention(q, hid, k, hid, v, hid, c->bias, c->band, c->bs, c->F, c->H, c->out, st));
  DAWN_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
