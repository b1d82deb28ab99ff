// dawn_test_kernel (include/dawn_unet.h): one per-clip or per-step glue kernel of the UNet through the launcher unet.cu calls, or
// one sampler update through the step functions of sampler.cu, on caller-owned buffers, for per-kernel tests against a
// high-precision reference.  Every geometry is checked here, before any CUDA call, so a refused case launches nothing.
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/dawn_unet.h"
#include "common.cuh"
#include "contraction.cuh"
#include "kernels.cuh"
#include "sampler.cuh"

namespace dawn {
namespace {

int refuse(const char* why) {
  set_last_error(std::string("dawn_test_kernel: ") + why);
  return -1;
}

// a row stride the float4 kernels can take
bool row_ok(int ld, int C) { return C >= 4 && (C & 3) == 0 && ld >= C && (ld & 3) == 0; }
bool clips_ok(int clips) { return clips >= 1 && clips <= kMaxClips; }

int cond_tables(const dawn_kernel_case& c, DeviceArena& arena, cudaStream_t st) {
  if (!c.x) return refuse("missing pointer");
  if (c.ndesc < 1 || c.ndesc > DAWN_KERNEL_MAX_DESC || c.F < 1 || !clips_ok(c.clips) || c.F % c.clips) return refuse("bad geometry");
  std::vector<CondDesc> cd;
  int max_n1 = 0, max_k = 0, max_co = 0;
  for (int i = 0; i < c.ndesc; ++i) {
    const dawn_kernel_desc& e = c.desc[i];
    if (!e.mW || !e.mB || !e.Wkv || !e.nkv || !e.qs || !e.ks || !e.Wout || !e.gout || !e.ctx || !e.kv || !e.kq || !e.nkq || !e.T || !e.G)
      return refuse("missing descriptor pointer");
    if (e.K < 1 || e.off < 0 || e.off + e.K > c.cond_ld || e.co < 4 || (e.co & 3) || e.ldbT < e.co || e.ca < 0 || e.ca > 2)
      return refuse("bad descriptor geometry");
    CondDesc d{};
    d.mW = e.mW; d.mB = e.mB; d.off = e.off; d.K = e.K; d.n1 = 2 * e.co; d.Wkv = e.Wkv; d.ctx = e.ctx; d.kv = e.kv;
    d.t.kv = e.kv; d.t.nkv = e.nkv; d.t.qs = e.qs; d.t.ks = e.ks; d.t.Wout = e.Wout; d.t.gout = e.gout;
    d.t.co = e.co; d.t.ldbT = e.ldbT; d.t.ca = e.ca; d.t.kq = e.kq; d.t.nkq = e.nkq; d.t.T = e.T; d.t.G = e.G;
    cd.push_back(d);
    max_n1 = std::max(max_n1, d.n1); max_k = std::max(max_k, d.K); max_co = std::max(max_co, e.co);
  }
  // every stage's dynamic shared memory must fit the opt-in limit of one block
  if ((size_t)8 * std::max(max_k, max_n1) * sizeof(float) > 227 * 1024 || (size_t)9 * max_co * sizeof(float) > 227 * 1024)
    return refuse("tables too wide for shared memory");
  CondDesc* dd;
  DAWN_TRY(arena.upload(cd, &dd));
  return launch_cond_batched(c.x, c.cond_ld, dd, c.ndesc, max_n1, max_k, max_co, c.F, c.clips, st);
}

int film(const dawn_kernel_case& c, DeviceArena& arena, cudaStream_t st) {
  if (!c.x) return refuse("missing pointer");
  if (c.ndesc < 1 || c.ndesc > DAWN_KERNEL_MAX_DESC || c.C < 1 || !clips_ok(c.clips)) return refuse("bad geometry");
  std::vector<FilmDesc> fd;
  int max_n = 0;
  for (int i = 0; i < c.ndesc; ++i) {
    const dawn_kernel_desc& e = c.desc[i];
    if (!e.W || !e.b || !e.out) return refuse("missing descriptor pointer");
    if (e.n < 1) return refuse("bad descriptor geometry");
    fd.push_back(FilmDesc{e.W, e.b, e.out, e.n});
    max_n = std::max(max_n, e.n);
  }
  FilmDesc* dd;
  DAWN_TRY(arena.upload(fd, &dd));
  return launch_film(dd, c.ndesc, max_n, c.clips, c.x, c.C, st);
}

// The cross-rank reductions of W ranks that all hold the caller's keys: every sum is W times the own value and every min the
// own value, so one GPU runs the frame-sharded select and its result is known from the local keys alone.
template <class T>
__global__ void times_kernel(T* b, size_t n, T w) {
  for (size_t i = threadIdx.x; i < n; i += blockDim.x) b[i] *= w;
}
int replica_sum_u32(void* ctx, unsigned int* b, size_t n, cudaStream_t st) {
  times_kernel<<<1, 256, 0, st>>>(b, n, (unsigned int)*static_cast<const int*>(ctx));
  DAWN_LAUNCH_OK();
  return 0;
}
int replica_sum_u64(void* ctx, unsigned long long* b, size_t n, cudaStream_t st) {
  times_kernel<<<1, 256, 0, st>>>(b, n, (unsigned long long)*static_cast<const int*>(ctx));
  DAWN_LAUNCH_OK();
  return 0;
}
int replica_min_u32(void*, unsigned int*, size_t, cudaStream_t) { return 0; }

int sampler_step(const dawn_kernel_case& c, cudaStream_t st) {
  const DdpmCoef* tab = c.kernel == DAWN_KERNEL_DDPM_STEP ? reinterpret_cast<const DdpmCoef*>(c.tab) : nullptr;
  if (!c.xs || !c.e || !c.scratch || (tab && !c.t_slot)) return refuse("missing pointer");
  // every digit bin and count_le of W replicas stays below 2^32 when W n does
  if (c.n < 1 || c.replicas < 0 || (long long)c.replicas * c.n >= (1LL << 32) || (tab && c.num_t < 1)) return refuse("bad geometry");
  int w = c.replicas;
  const DdimReduce rep{&w, replica_sum_u32, replica_sum_u64, replica_min_u32};
  const DdimReduce* red = w > 0 ? &rep : nullptr;
  const int64_t n_global = c.n * (w > 0 ? w : 1);
  const float* k = c.coef;
  if (c.kernel == DAWN_KERNEL_DDIM_STEP)
    return ddim_step_impl(c.xs, c.e, c.noise, c.n, n_global, k[0], k[1], k[2], k[3], k[4], c.q, c.scratch, st, red);
  return ddpm_step_impl(c.xs, c.e, c.noise, c.n, n_global, DdpmCoef{k[0], k[1], k[2], k[3], k[4]}, tab, c.t_slot, c.num_t, c.q,
                        c.scratch, st, red);
}

int test_kernel(const dawn_kernel_case& c, DeviceArena& arena, cudaStream_t st) {
  switch (c.kernel) {
    case DAWN_KERNEL_ROWSTATS:
      if (!c.x || !c.out) return refuse("missing pointer");
      if (c.M < 1 || c.C > 2048 || !row_ok(c.ld, c.C)) return refuse("bad geometry");
      return launch_rowstats(c.x, c.ld, c.C, c.M, c.eps, c.out, st);
    case DAWN_KERNEL_GN_APPLY:
      if (!c.y || !c.stats || !c.w || !c.b || !c.out) return refuse("missing pointer");
      // 8 groups, and a float4 never straddles two groups
      if (c.M < 1 || c.P < 1 || !clips_ok(c.clips) || c.cpg < 4 || (c.cpg & 3) || c.C != 8 * c.cpg || !(c.count > 0) ||
          !row_ok(c.ldy, c.C) || !row_ok(c.ldo, c.C) || (c.res && !row_ok(c.ldr, c.C)))
        return refuse("bad geometry");
      return launch_gn_apply(c.y, c.ldy, c.C, c.M, c.stats, c.count, c.cpg, c.P, c.clips, c.w, c.b, nullptr, c.res, c.ldr, c.out,
                             c.ldo, st);
    case DAWN_KERNEL_COND_TABLES:
      return cond_tables(c, arena, st);
    case DAWN_KERNEL_TIME_MLP:
      if (!c.t || !c.freqs || !c.w || !c.b || !c.w2 || !c.b2 || !c.out) return refuse("missing pointer");
      if (c.dim < 2 || (c.dim & 1) || (size_t)5 * c.dim * sizeof(float) > 48 * 1024 || !clips_ok(c.clips) ||
          (c.t_stride != 0 && c.t_stride != 1))
        return refuse("bad geometry");
      return launch_time_mlp(c.t, c.t_stride, c.clips, c.freqs, c.dim, c.w, c.b, c.w2, c.b2, c.out, st);
    case DAWN_KERNEL_FILM:
      return film(c, arena, st);
    case DAWN_KERNEL_ROTARY:
      if (!c.freqs || !c.out) return refuse("missing pointer");
      if (c.F < 1 || c.pos0 < 0 || c.F > (1 << 20)) return refuse("bad geometry");
      return launch_rotary_table(c.freqs, 16, c.F, c.pos0, c.out, st);
    case DAWN_KERNEL_SPLIT_ROWS:
      if (!c.x || !c.out_hi || !c.out_lo) return refuse("missing pointer");
      if (c.M < 1 || !row_ok(c.ld, c.C)) return refuse("bad geometry");
      return launch_split_rows(c.x, c.ld, c.C, c.M, c.out_hi, c.out_lo, st);
    case DAWN_KERNEL_NCF_TO_NHWC:
      if (!c.x || !c.out) return refuse("missing pointer");
      if (c.C < 1 || c.F < 1 || c.P < 1 || c.c0 < 0 || c.Cpad < c.c0 + c.C || !clips_ok(c.clips) || c.F * c.clips > 65535)
        return refuse("bad geometry");
      return launch_ncf_to_nhwc(c.x, c.C, c.F, c.P, c.Cpad, c.c0, c.out, st, c.skip_flag, c.skip_if, c.clips);
    case DAWN_KERNEL_FRAME_INVARIANCE:
      if (!c.x || !c.flag) return refuse("missing pointer");
      if (c.C < 1 || c.F < 1 || c.P < 1 || c.c0 < 0 || c.c0 > c.C || !clips_ok(c.clips)) return refuse("bad geometry");
      return launch_frame_invariance(c.x, c.c0, c.C, c.F, c.P, c.clips, c.flag, st);
    case DAWN_KERNEL_FEA_SHIFT:
      if (!c.x || !c.out) return refuse("missing pointer");
      if (c.C < 1 || c.H < 1 || c.W < 1 || c.k < 1 || !(c.k & 1) || c.c0 < 0 || c.Cpad < c.c0 + c.C || !clips_ok(c.clips) ||
          c.cstride < (long long)c.H * c.W || (c.clips > 1 && c.clip_stride < (c.C - 1) * c.cstride + (long long)c.H * c.W))
        return refuse("bad geometry");
      return launch_fea_shift_nhwc(c.x, c.cstride, c.clip_stride, c.clips, c.C, c.H, c.W, c.Cpad, c.c0, c.k, c.out, st, c.skip_flag,
                                   c.skip_if);
    case DAWN_KERNEL_MAP_REDUCE:
      if (!c.x || !c.out) return refuse("missing pointer");
      if (c.k < 1 || c.n < 1 || c.C < 1 || (c.n + 255) / 256 > 0x7fffffffLL) return refuse("bad geometry");
      return launch_map_reduce(c.x, c.k, c.n, c.b, c.C, c.out, st, c.skip_flag, c.skip_if);
    case DAWN_KERNEL_INIT_CONV_X3:
      if (!c.x || !c.w || !c.map || !c.out) return refuse("missing pointer");
      if (c.F < 1 || c.H < 1 || c.W < 1 || !clips_ok(c.clips) || c.k < 1 || !(c.k & 1) || !row_ok(c.ldo, c.C) ||
          c.clip_stride < 3LL * c.F * c.H * c.W || (size_t)c.k * c.k * 3 * c.C * sizeof(float) > 100 * 1024)
        return refuse("bad geometry");
      return launch_init_conv_x3(c.x, c.clip_stride, c.F, c.H, c.W, c.clips, c.w, c.map, c.C, c.out, c.ldo, c.k, st, c.skip_flag,
                                 c.skip_if);
    case DAWN_KERNEL_HEADS_OUT:
      if (!c.x || !c.y || !c.w || !c.b || !c.out || (c.nc > 0 && (!c.w2 || !c.b2))) return refuse("missing pointer");
      if (c.C < 4 || (c.C & 3) || c.M < 1 || c.P < 1 || !clips_ok(c.clips) || c.M % ((long long)c.P * c.clips) || c.ng < 0 ||
          c.nc < 0 || c.ng + c.nc < 1)
        return refuse("bad geometry");
      return launch_heads_out(c.x, c.y, c.C, c.M, c.P, c.clips, c.w, c.b, c.ng, c.w2, c.b2, c.nc, c.out, st);
    case DAWN_KERNEL_DDIM_STEP:
    case DAWN_KERNEL_DDPM_STEP:
      return sampler_step(c, st);
    case DAWN_KERNEL_Q_SAMPLE:
      if (!c.x || !c.noise || !c.t || !c.w || !c.b || !c.out) return refuse("missing pointer");
      if (c.n < 1 || c.num_t < 1 || c.clips < 1 || c.clips > 65535) return refuse("bad geometry");
      return q_sample_impl(c.x, c.noise, c.t, c.w, c.b, c.num_t, c.clips, c.n, c.out, st);
    case DAWN_KERNEL_MOTION_TO_LATENT:
      if (!c.x || !c.y || !c.out || (c.t && (!c.noise || !c.w || !c.b))) return refuse("missing pointer");
      if (c.F < 1 || c.H < 1 || c.W < 1 || c.clips < 1 || c.clips > 65535 || (c.t && c.num_t < 1)) return refuse("bad geometry");
      return motion_to_latent_impl(c.x, c.y, c.clips, c.F, c.H, c.W, c.t, c.noise, c.w, c.b, c.num_t, c.out, st);
  }
  return refuse("unknown kernel");
}

}  // namespace
}  // namespace dawn

extern "C" int dawn_test_kernel(const dawn_kernel_case* c, void* stream) {
  if (!c) return dawn::refuse("null case");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  dawn::DeviceArena arena;
  const int rc = dawn::test_kernel(*c, arena, st);
  if (rc != 0) return rc;
  DAWN_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}
