// Host side of every contraction (contraction.cuh), and dawn_test_contraction (include/dawn_unet.h), which runs one
// contraction through the same weight upload and path launcher as the networks.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>

#include "common.cuh"
#include "contraction.cuh"
#include "kernels.cuh"
#include "tc_gemm.cuh"

namespace dawn {

// ------------------------------------------------------------------------------------------ host parameters, allocations
void HostParams::set(const std::string& name, const float* data, const int64_t* shape, int ndim) {
  HostParam p;
  p.shape.assign(shape, shape + ndim);
  int64_t numel = 1;
  for (int64_t s : p.shape) numel *= s;
  p.data.assign(data, data + numel);
  map[name] = std::move(p);
}

int HostParams::need(const std::string& name, const std::vector<int64_t>& shape, const HostParam** out) const {
  auto it = map.find(name);
  if (it == map.end()) { set_last_error(prefix + "missing parameter: " + name); return -1; }
  const HostParam& p = it->second;
  if (p.shape != shape) {
    std::string s = prefix + "parameter " + name + " has shape (";
    for (auto d : p.shape) s += std::to_string(d) + ",";
    s += ") expected (";
    for (auto d : shape) s += std::to_string(d) + ",";
    set_last_error(s + ")");
    return -1;
  }
  *out = &p;
  return 0;
}

namespace {
std::atomic<int64_t> g_arena_bytes{0};     // blocks of every DeviceArena
}  // namespace

int DeviceArena::alloc_bytes(size_t bytes, void** out) {
  *out = nullptr;
  bytes = std::max<size_t>(bytes, 16);
  DAWN_CUDA_OK(cudaMalloc(out, bytes));
  blocks_.emplace_back(*out);
  bytes_ += (int64_t)bytes;
  g_arena_bytes += (int64_t)bytes;
  return 0;
}
int DeviceArena::copy_in(void* dst, const void* src, size_t bytes) {
  DAWN_CUDA_OK(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
  return 0;
}
void DeviceArena::release() {
  blocks_.clear();
  g_arena_bytes -= bytes_;
  bytes_ = 0;
}
int64_t DeviceArena::live_bytes() { return g_arena_bytes.load(); }

// ------------------------------------------------------------------------------------------ packed weights
int upload_weight(DeviceArena& arena, const std::vector<float>& m, int K, int N, int ldb, const std::vector<float>& bias,
                  PackedWeight* out) {
  *out = PackedWeight{};
  DAWN_TRY(arena.upload(m, &out->w));
  if (N % 64 == 0 && K % 64 == 0) {             // the shapes the wgmma kernels can take
    std::vector<float> img;
    tc_pack_weights(m.data(), K, N, ldb, img, &out->img_scale);
    DAWN_TRY(arena.upload(img, &out->img));
  }
  if (!bias.empty()) {
    std::vector<float> b(ldb, 0.f);
    std::copy(bias.begin(), bias.end(), b.begin());
    DAWN_TRY(arena.upload(b, &out->b));
  }
  out->K = K; out->N = N; out->ldb = ldb;
  return 0;
}

std::vector<float> fold_linear(const float* w, int N, int K, const float* gain, float qscale, int nscale) {
  std::vector<float> m((size_t)N * K);
  for (int n = 0; n < N; ++n) {
    const float sc = (n < nscale) ? qscale : 1.0f;
    for (int k = 0; k < K; ++k) {
      float v = w[(size_t)n * K + k];
      if (gain) v *= gain[k];
      m[(size_t)n * K + k] = v * sc;
    }
  }
  return m;
}

std::vector<float> row_sums(const std::vector<float>& w, int N, int K) {
  std::vector<float> s(N);
  for (int n = 0; n < N; ++n) {
    double acc = 0.0;
    for (int k = 0; k < K; ++k) acc += w[(size_t)n * K + k];
    s[n] = (float)acc;
  }
  return s;
}

void fold_ca_q(const float* const to_q[3], const float* const gain[3], int ci, std::vector<float>& wq, std::vector<float>& wsum) {
  wq.assign((size_t)ci * 192, 0.f);
  wsum.assign(192, 0.f);
  for (int a = 0; a < 3; ++a) {
    const std::vector<float> m = fold_linear(to_q[a], 64, ci, gain[a], 1.f, 0);
    const std::vector<float> s = row_sums(m, 64, ci);
    for (int j = 0; j < 64; ++j) {
      for (int k = 0; k < ci; ++k) wq[(size_t)k * 192 + a * 64 + j] = m[(size_t)j * ci + k];
      wsum[a * 64 + j] = s[j];
    }
  }
}

int bn_affine(const HostParams& raw, const std::string& prefix, int c, std::vector<double>& s, std::vector<double>& t) {
  const HostParam *g, *b, *rm, *rv;
  DAWN_TRY(raw.need(prefix + ".weight", {c}, &g));
  DAWN_TRY(raw.need(prefix + ".bias", {c}, &b));
  DAWN_TRY(raw.need(prefix + ".running_mean", {c}, &rm));
  DAWN_TRY(raw.need(prefix + ".running_var", {c}, &rv));
  s.resize(c); t.resize(c);
  for (int i = 0; i < c; ++i) {
    s[i] = (double)g->data[i] / std::sqrt((double)rv->data[i] + 1e-5);
    t[i] = (double)b->data[i] - (double)rm->data[i] * s[i];
  }
  return 0;
}

void pack_conv_taps(const float* w, int co, int ci, int taps, int ci_pad, int ldb, int n0, const double* scale, std::vector<float>& m) {
  for (int n = 0; n < co; ++n) {
    const double sn = scale ? scale[n] : 1.0;            // (float)((double)w * 1.0) == w: no scale is an exact copy
    for (int c = 0; c < ci; ++c)
      for (int tp = 0; tp < taps; ++tp)
        m[((size_t)tp * ci_pad + c) * ldb + n0 + n] = (float)((double)w[((size_t)n * ci + c) * taps + tp] * sn);
  }
}

int pack_lfg_conv(const HostParams& raw, DeviceArena& arena, const std::vector<std::pair<std::string, int>>& convs,
                  const std::string& bn_after, int ci, int k, int ci_pad, PackedWeight* out) {
  int N = 0;
  for (auto& c : convs) N += c.second;
  const int ldb = round_up(N, 64), K = k * k * ci_pad;
  std::vector<float> m((size_t)K * ldb, 0.f), bias(N);
  int n0 = 0;
  for (auto& cv : convs) {
    const int co = cv.second;
    const HostParam *w, *b;
    DAWN_TRY(raw.need(cv.first + ".weight", {co, ci, k, k}, &w));
    DAWN_TRY(raw.need(cv.first + ".bias", {co}, &b));
    std::vector<double> s(co, 1.0), t(co, 0.0);
    if (!bn_after.empty()) DAWN_TRY(bn_affine(raw, bn_after, co, s, t));
    for (int n = 0; n < co; ++n) bias[n0 + n] = (float)((double)b->data[n] * s[n] + t[n]);
    pack_conv_taps(w->data.data(), co, ci, k * k, ci_pad, ldb, n0, s.data(), m);
    n0 += co;
  }
  return upload_weight(arena, m, K, N, ldb, bias, out);
}

// ------------------------------------------------------------------------------------------ GemmParams
void base_params(GemmParams& p, const float* A, int lda, int Cin, int frames, int H, int W) {
  memset(&p, 0, sizeof(p));
  p.A = A; p.lda = lda; p.Cin = Cin;
  p.IH = H; p.IW = W; p.OHs = H; p.OWs = W; p.in_stride = 1;
  p.ntaps = 1;
  p.M = frames * H * W; p.rows_per_batch = p.M;
  p.OH = H; p.OW = W; p.out_stride = 1;
  p.P = H * W;
  p.q_post_scale = 1.f;
  p.clips = 1;
}
void set_weights(GemmParams& p, const PackedWeight& w) {
  p.B = w.w; p.Bimg = w.img; p.tc_scale = 1.0f / w.img_scale; p.ldb = w.ldb; p.N = w.N; p.K = w.K; p.bias = w.b;
}
void set_square_taps(GemmParams& p, int k, int pad) {
  p.ntaps = k * k;
  for (int ky = 0; ky < k; ++ky)
    for (int kx = 0; kx < k; ++kx) { p.dy[ky * k + kx] = (signed char)(ky - pad); p.dx[ky * k + kx] = (signed char)(kx - pad); }
}

// ------------------------------------------------------------------------------------------ kernel paths
namespace {
// the split pass writes dense rows of Cin fp16 values per input pixel: the hi plane, then the lo plane
long long split_rows(const GemmParams& p) { return (long long)(p.M / (p.OHs * p.OWs)) * p.IH * p.IW; }
}  // namespace

bool path_ok(const GemmParams& p, int epi, int path, size_t scratch_bytes) {
  const bool planes = p.A16h != nullptr || (p.Cin % 64 == 0 && (size_t)split_rows(p) * p.Cin * 4 <= scratch_bytes);
  switch (path) {
    case DAWN_PATH_MMA_SYNC: return true;
    case DAWN_PATH_TC_GEMM: return p.Bimg && tc_gemm_supported(p, epi);
    case DAWN_PATH_TC_GEMM_PRESPLIT: return p.Bimg && tc_gemm_supported(p, epi) && planes;
    case DAWN_PATH_TC_CONV3: return p.Bimg && tc_conv3_supported(p, epi);
    case DAWN_PATH_TC_CONV3_TMA: return p.Bimg && tc_conv3_supported(p, epi) && p.lda == p.Cin && planes;   // TMA reads dense planes
  }
  return false;
}

int choose_path(const GemmParams& p, int epi, size_t scratch_bytes) {
  // A16h set: the producing kernel wrote the input as fp16 hi | lo planes (and not as fp32), so the halo conv fetches them by TMA
  if (path_ok(p, epi, DAWN_PATH_TC_CONV3, 0)) return p.A16h ? DAWN_PATH_TC_CONV3_TMA : DAWN_PATH_TC_CONV3;
  if (!path_ok(p, epi, DAWN_PATH_TC_GEMM, 0)) return DAWN_PATH_MMA_SYNC;
  // several n-tiles re-convert the same A panels (per-tap gather of the small levels' 3x3 convolutions): split once instead
  const bool split = (p.ntaps == 9 && p.N >= 256 && !p.perm_in) || p.want_split;
  return split && path_ok(p, epi, DAWN_PATH_TC_GEMM_PRESPLIT, scratch_bytes) ? DAWN_PATH_TC_GEMM_PRESPLIT : DAWN_PATH_TC_GEMM;
}

int launch_path(const GemmParams& p, int epi, int path, void* scratch, cudaStream_t st, int* kernels) {
  if (kernels) *kernels = 1;
  if (path == DAWN_PATH_MMA_SYNC) return launch_gemm(p, epi, st);
  GemmParams q = p;
  if ((path == DAWN_PATH_TC_GEMM_PRESPLIT || path == DAWN_PATH_TC_CONV3_TMA) && p.A16h == nullptr) {
    const long long rows = split_rows(p);
    unsigned short* hi = static_cast<unsigned short*>(scratch);
    q.A16h = hi; q.A16l = hi + (size_t)rows * p.Cin;
    DAWN_TRY(launch_split_rows(p.A, p.lda, p.Cin, rows, (void*)q.A16h, (void*)q.A16l, st));
    if (kernels) *kernels = 2;
  }
  if (path == DAWN_PATH_TC_CONV3 || path == DAWN_PATH_TC_CONV3_TMA) return launch_tc_conv3(q, q.Bimg, st);
  return launch_tc_gemm(q, q.Bimg, epi, st);
}

// ------------------------------------------------------------------------------------------ 2x upsampling conv
int pack_up(DeviceArena& arena, int ci, int co, const int (&off)[2][2], const std::vector<float>& bias, const UpWeight& weight,
            UpConv* u) {
  memcpy(u->off, off, sizeof(u->off));
  const int ldb = round_up(co, 64);
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      std::vector<float> m((size_t)4 * ci * ldb, 0.f);
      for (int ty = 0; ty < 2; ++ty)
        for (int tx = 0; tx < 2; ++tx)
          for (int c = 0; c < ci; ++c)
            for (int n = 0; n < co; ++n) m[((size_t)(ty * 2 + tx) * ci + c) * ldb + n] = weight(py, px, ty, tx, c, n);
      DAWN_TRY(upload_weight(arena, m, 4 * ci, co, ldb, bias, &u->cls[py * 2 + px]));
    }
  if (co == 64 && ci % 64 == 0) {
    // one 3x3 conv over the input grid: weight rows (tap, cin), columns (class, cout); 2.25x the MACs of the four class convs,
    // one launch of the halo-tile kernel instead of four gather GEMMs
    const int N4 = 4 * co;
    std::vector<float> m((size_t)9 * ci * N4, 0.f), b4(N4, 0.f);
    for (int py = 0; py < 2; ++py)
      for (int px = 0; px < 2; ++px) {
        const int cls = py * 2 + px;
        for (int n = 0; n < co; ++n) b4[cls * co + n] = bias[n];
        for (int ty = 0; ty < 2; ++ty)
          for (int tx = 0; tx < 2; ++tx) {
            const int tap = (off[py][ty] + 1) * 3 + (off[px][tx] + 1);
            for (int c = 0; c < ci; ++c)
              for (int n = 0; n < co; ++n) m[((size_t)tap * ci + c) * N4 + cls * co + n] = weight(py, px, ty, tx, c, n);
          }
      }
    DAWN_TRY(upload_weight(arena, m, 9 * ci, N4, N4, b4, &u->all));
  }
  return 0;
}

int pack_up_nearest(DeviceArena& arena, const float* w, int ci, int co, const double* scale, const std::vector<float>& bias,
                    UpConv* u) {
  return pack_up(arena, ci, co, kUpOff, bias, [&](int py, int px, int ty, int tx, int c, int n) {
    double acc = 0.0;
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx)
        if (up_in_set(py, ty, ky) && up_in_set(px, tx, kx)) acc += (double)w[(((size_t)n * ci + c) * 3 + ky) * 3 + kx];
    return (float)(scale ? acc * scale[n] : acc);
  }, u);
}

int pack_lfg_up(const HostParams& raw, DeviceArena& arena, const std::string& name, int co, int ci, UpConv* u) {
  // on the low-resolution grid each output-parity class is a 2x2 conv: 2.25x fewer MACs, and the upsampled tensor never exists
  const HostParam *w, *b;
  DAWN_TRY(raw.need(name + ".conv.weight", {co, ci, 3, 3}, &w));
  DAWN_TRY(raw.need(name + ".conv.bias", {co}, &b));
  std::vector<double> s, t;
  DAWN_TRY(bn_affine(raw, name + ".norm", co, s, t));
  std::vector<float> bias(co);
  for (int n = 0; n < co; ++n) bias[n] = (float)((double)b->data[n] * s[n] + t[n]);
  return pack_up_nearest(arena, w->data.data(), ci, co, s.data(), bias, u);
}

int run_up(const GemmParams& in, const UpConv& u, float* out, int ldo, const std::function<int(const GemmParams&)>& run, int border) {
  if (!border) {
    GemmParams p = in;
    set_weights(p, u.all); set_square_taps(p, 3, 1);
    p.up2 = 1; p.Out = out; p.ldo = ldo;
    if (path_ok(p, EPI_PLAIN, DAWN_PATH_TC_CONV3, 0)) return run(p);
  }
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      GemmParams q = in;
      set_weights(q, u.cls[py * 2 + px]);
      q.ntaps = 4;
      for (int ty = 0; ty < 2; ++ty)
        for (int tx = 0; tx < 2; ++tx) {
          q.dy[ty * 2 + tx] = (signed char)(u.off[py][ty] + border); q.dx[ty * 2 + tx] = (signed char)(u.off[px][tx] + border);
        }
      q.OH = 2 * in.OHs; q.OW = 2 * in.OWs; q.out_stride = 2; q.oy0 = py; q.ox0 = px;
      q.Out = out; q.ldo = ldo;
      DAWN_TRY(run(q));
    }
  return 0;
}

// ------------------------------------------------------------------------------------------ dawn_test_contraction
namespace {

int refuse(const char* why) {
  set_last_error(std::string("dawn_test_contraction: ") + why);
  return -1;
}

int test_contraction(const dawn_contraction_case& c, cudaStream_t st) {
  if (c.path < DAWN_PATH_MMA_SYNC || c.path > DAWN_PATH_TC_CONV3_TMA) return refuse("unknown path");
  if (c.epi < EPI_PLAIN || c.epi > EPI_LN_BIAS_GELU) return refuse("unknown epilogue");
  // one tap may read overlapping rows (lda < Cin): the positional conv's 64 x k windows over a 64-channel plane
  if (c.ntaps < 1 || c.ntaps > 52 || c.F < 1 || c.N < 1 || c.ldb < c.N || c.lda < 1 || (c.ntaps > 1 && c.lda < c.Cin))
    return refuse("bad geometry");
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
  p.stats = c.stats; p.cpg = c.cpg; p.clips = 1;
  p.rowstats = c.rowstats; p.ln_inline = c.ln_inline; p.wsum = c.wsum; p.rot = c.rot; p.P = c.P;
  p.q_post_scale = c.q_post_scale;
  p.kq = c.kq; p.nkq = c.nkq; p.gates = c.gates;
  p.Y = c.Y; p.ldy = c.ldy; p.gn_stats = c.gn_stats; p.gn_w = c.gn_w; p.gn_b = c.gn_b; p.film = c.film; p.gn_count = c.gn_count;
  p.drain = c.drain;

  const bool ln_bias = c.epi == EPI_LN_BIAS || c.epi == EPI_LN_BIAS_GELU;
  const bool ln = (c.epi >= EPI_QKV_TEMPORAL && c.epi <= EPI_CA_GATE) || ln_bias;
  if (p.ln_inline && (c.path != DAWN_PATH_TC_GEMM || p.ntaps != 1)) return refuse("inline LayerNorm statistics need the gather-producer wgmma GEMM and one tap");
  if (ln && !p.ln_inline && !p.rowstats) return refuse("LayerNorm epilogue without row statistics");
  if (ln && !p.wsum) return refuse("LayerNorm epilogue without wsum");
  if (ln_bias && !p.bias) return refuse("LayerNorm + bias epilogue without a bias");          // both kernels read bias[n] unguarded
  // the plain epilogue is the only one whose partial sums both kernels accumulate (the wgmma GEMM would also sum GELU outputs,
  // the mma.sync kernel would not)
  if (p.stats && c.epi != EPI_PLAIN) return refuse("GroupNorm statistics with an epilogue other than the plain one");
  if (c.epi == EPI_PLAIN && p.stats && (p.cpg <= 0 || p.N / p.cpg > 8)) return refuse("GroupNorm statistics need 8 groups");

  DeviceArena arena;
  if (c.path != DAWN_PATH_MMA_SYNC) {
    // the wgmma paths read the weight image the network's upload builds from the same fp32 matrix
    std::vector<float> hB((size_t)p.K * p.ldb);
    DAWN_CUDA_OK(cudaMemcpy(hB.data(), p.B, hB.size() * sizeof(float), cudaMemcpyDeviceToHost));
    PackedWeight w;
    DAWN_TRY(upload_weight(arena, hB, p.K, p.N, p.ldb, {}, &w));
    set_weights(p, w);
    p.bias = c.bias;
  }
  const bool split = c.path == DAWN_PATH_TC_GEMM_PRESPLIT || c.path == DAWN_PATH_TC_CONV3_TMA;
  const size_t scratch_bytes = split ? (size_t)split_rows(p) * p.Cin * 4 : 0;
  if (!path_ok(p, c.epi, c.path, scratch_bytes)) return refuse("the path does not accept this geometry");
  unsigned short* scratch = nullptr;                     // the fp16 hi | lo planes of A
  if (split) DAWN_TRY(arena.alloc(scratch_bytes / sizeof(unsigned short), &scratch));
  DAWN_TRY(launch_path(p, c.epi, c.path, scratch, st));
  DAWN_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace
}  // namespace dawn

extern "C" int dawn_test_contraction(const dawn_contraction_case* c, void* stream) {
  if (!c) return dawn::refuse("null case");
  return dawn::test_contraction(*c, static_cast<cudaStream_t>(stream));
}
