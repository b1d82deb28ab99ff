// DDIM update around the denoising UNet (reference U:1169-1205): x0 prediction, dynamic thresholding with the exact
// 0.9-quantile of |x0| over the whole clip (torch.quantile semantics, linear interpolation), and the eta-noise update.
// The ancestral (DDPM) update of p_sample (U:1087-1121) shares the same threshold.  q_sample (U:1226-1232) and the motion
// estimator's output -> latent pass (FD:248-262, 280-282) start a sampler from a real clip.
// Everything stays on the device: no host synchronisation inside a sampling step.
#include "common.cuh"
#include "sampler.cuh"
#include "../../include/dawn_unet.h"

namespace dawn {
namespace {

// classifier-free guidance (reference forward_with_cond_scale U:879-890): null + (cond - null) * s, rounded as its three fp32
// torch ops (no fused multiply-add)
__device__ __forceinline__ float guided_eps(float e_cond, float e_null, float s) {
  return __fadd_rn(e_null, __fmul_rn(__fsub_rn(e_cond, e_null), s));
}

// eps of a DDIM update: eps[i], or with guidance (eps_n != nullptr) the guided eps of eps[i] and eps_n[i] at scale g, which is
// formed here and never stored
__device__ __forceinline__ float update_eps(const float* __restrict__ eps, const float* __restrict__ eps_n, float g, long long i) {
  return eps_n ? guided_eps(eps[i], eps_n[i], g) : eps[i];
}

// x0 = ca * x - cb * e rounded like the reference's two products and one difference (U:1072-1076).  A fused multiply-add
// would keep ca * x unrounded: near t = 999 both products are ~3e4 times x and cancel, so that moved the sample by 1e-5.
__device__ __forceinline__ float ddim_x0(float ca, float x, float cb, float e) { return __fsub_rn(__fmul_rn(ca, x), __fmul_rn(cb, e)); }

// keys[i] = |x0|, e = update_eps  (x0 magnitude; non-negative floats order like their bit patterns)
__global__ void x0_abs_kernel(const float* __restrict__ x, const float* __restrict__ eps, const float* __restrict__ eps_n,
                              const float* __restrict__ scale, float ca, float cb, long long n, uint32_t* __restrict__ keys) {
  const float g = eps_n ? *scale : 0.0f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    keys[i] = __float_as_uint(fabsf(ddim_x0(ca, x[i], cb, update_eps(eps, eps_n, g, i))));
}

// clamp(x0, -s, s) / s as torch evaluates it (U:1107, 1196): a NaN x0 stays NaN, where fmaxf / fminf would return a bound,
// and a NaN s makes the quotient NaN
__device__ __forceinline__ float clip_x0(float x0, float s) {
  return __fdiv_rn(isnan(x0) ? x0 : fminf(fmaxf(x0, -s), s), s);
}

// one launch instead of a pageable-host memcpy + four memsets (keeps the step capturable in a CUDA graph)
__global__ void select_init_kernel(uint32_t* state, unsigned int* hist, unsigned long long* count_le, unsigned int* min_gt,
                                   unsigned int* any_nan, unsigned long long lo) {
  hist[threadIdx.x] = 0;
  if (threadIdx.x == 0) {
    state[0] = 0u; state[1] = 0u; state[2] = (uint32_t)(lo & 0xFFFFFFFFull); state[3] = (uint32_t)(lo >> 32);
    *count_le = 0ull; *min_gt = 0xFFFFFFFFu; *any_nan = 0u;
  }
}

// state[0] = prefix value, state[1] = prefix mask, state[2..3] = remaining rank (64-bit), hist[256]
__global__ void radix_hist_kernel(const uint32_t* __restrict__ keys, long long n, const uint32_t* __restrict__ state, int shift,
                                  unsigned int* __restrict__ hist) {
  __shared__ unsigned int sh[256];
  sh[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t pv = state[0], pm = state[1];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t k = keys[i];
    if ((k & pm) == pv) atomicAdd(&sh[(k >> shift) & 255u], 1u);
  }
  __syncthreads();
  if (sh[threadIdx.x]) atomicAdd(&hist[threadIdx.x], sh[threadIdx.x]);
}

__global__ void radix_pick_kernel(uint32_t* state, int shift, unsigned int* hist) {
  if (threadIdx.x != 0) return;
  unsigned long long rank = ((unsigned long long)state[3] << 32) | state[2];
  unsigned long long cum = 0;
  int b = 0;
  for (; b < 256; ++b) {
    if (cum + hist[b] > rank) break;
    cum += hist[b];
  }
  if (b > 255) b = 255;
  rank -= cum;
  state[0] |= (uint32_t)b << shift;
  state[1] |= 255u << shift;
  state[2] = (uint32_t)rank; state[3] = (uint32_t)(rank >> 32);
  for (int i = 0; i < 256; ++i) hist[i] = 0;
}

// after the 4 digit passes state[0] is the key of order statistic `lo`: count_le = #keys <= it, min_gt = min key above it,
// any_nan != 0 when a key is NaN (a bit pattern above +inf's)
__global__ void next_stat_kernel(const uint32_t* __restrict__ keys, long long n, const uint32_t* __restrict__ state,
                                 unsigned long long* __restrict__ count_le, unsigned int* __restrict__ min_gt,
                                 unsigned int* __restrict__ any_nan) {
  const uint32_t v = state[0];
  unsigned long long c = 0;
  unsigned int m = 0xFFFFFFFFu;
  bool nan = false;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t k = keys[i];
    if (k <= v) ++c; else m = min(m, k);
    nan |= k > 0x7F800000u;
  }
  for (int o = 16; o > 0; o >>= 1) {
    c += __shfl_xor_sync(0xffffffffu, c, o);
    m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
  }
  nan = __any_sync(0xffffffffu, nan);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(count_le, c);
    atomicMin(min_gt, m);
    if (nan) atomicOr(any_nan, 1u);
  }
}

// s = max(1, lerp(v[lo], v[hi], w)) exactly as torch.quantile + clamp_(min=1)  (U:1186-1193).  Both give NaN when a key is NaN
// (torch.quantile moves every rank onto the NaN the sort put last) or when the lerp does (inf - inf), and clamp_ keeps it.
__global__ void threshold_kernel(const uint32_t* state, const unsigned long long* count_le, const unsigned int* min_gt,
                                 const unsigned int* any_nan, long long lo, long long hi, float w, float* s_out) {
  const float vlo = __uint_as_float(state[0]);
  float vhi = vlo;
  if (hi > lo && *count_le < (unsigned long long)(lo + 2)) vhi = __uint_as_float(*min_gt);
  const float d = vhi - vlo;
  const float q = (w < 0.5f) ? (vlo + w * d) : (vhi - d * (1.0f - w));     // at::lerp
  *s_out = (*any_nan || isnan(q)) ? __uint_as_float(0x7FC00000u) : fmaxf(q, 1.0f);
}

// img = clamp(x0, -s, s)/s * sqrt(a_next) + c * e + sigma * noise, e = update_eps, each product and sum rounded as the
// reference's fp32 ops (U:1203-1205; fused multiply-adds moved about one element in four by an ulp).  noise == nullptr is the
// last step, where the reference adds sigma * 0. (U:1201): that add turns a -0 sum into +0.  clamp == 0: x0 is used as
// predicted (clip_denoised=False, U:1183).  x_n != nullptr (guidance): the new x also goes to the null slot, so the next
// forward sees the same x_t in both
__global__ void ddim_update_kernel(float* __restrict__ x, float* __restrict__ x_n, const float* __restrict__ eps,
                                   const float* __restrict__ eps_n, const float* __restrict__ scale, const float* __restrict__ noise,
                                   const float* __restrict__ s_ptr, float ca, float cb, float sqrt_an, float c, float sigma,
                                   long long n, int clamp) {
  const float s = s_ptr ? *s_ptr : 1.0f;
  const float g = eps_n ? *scale : 0.0f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float e = update_eps(eps, eps_n, g, i);
    float x0 = ddim_x0(ca, x[i], cb, e);
    if (clamp) x0 = clip_x0(x0, s);
    float v = __fadd_rn(__fmul_rn(x0, sqrt_an), __fmul_rn(c, e));
    v = __fadd_rn(v, __fmul_rn(sigma, noise ? noise[i] : 0.0f));
    x[i] = v;
    if (x_n) x_n[i] = v;
  }
}

// coefficients of this launch: the by-value set, or the table row of the timestep in the device slot (step graph)
__device__ __forceinline__ DdpmCoef ddpm_coef(const DdpmCoef& c, const DdpmCoef* tab, const int64_t* t_slot, int num_t) {
  if (!tab) return c;
  const long long t = *t_slot;
  return tab[t < 0 ? 0 : (t >= num_t ? num_t - 1 : t)];
}

// keys[i] = |x0| rounded like the reference's two products and one difference (U:1072-1076; no fused multiply-add: at
// t = 999 the products are ~6e4 times x, so a contraction would move x0 by far more than an ulp of it)
__global__ void ddpm_x0_abs_kernel(const float* __restrict__ x, const float* __restrict__ eps, DdpmCoef c,
                                   const DdpmCoef* __restrict__ tab, const int64_t* __restrict__ t_slot, int num_t, long long n,
                                   uint32_t* __restrict__ keys) {
  const DdpmCoef k = ddpm_coef(c, tab, t_slot, num_t);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    keys[i] = __float_as_uint(fabsf(__fsub_rn(__fmul_rn(k.ca, x[i]), __fmul_rn(k.cb, eps[i]))));
}

// x = c1 * clamp(x0, -s, s)/s + c2 * x + sigma * noise  (U:1078-1085, 1107, 1118-1121), each operation rounded as torch does;
// clamp == 0: x0 is used as predicted (clip_denoised=False)
__global__ void ddpm_update_kernel(float* __restrict__ x, const float* __restrict__ eps, const float* __restrict__ noise,
                                   const float* __restrict__ s_ptr, DdpmCoef c, const DdpmCoef* __restrict__ tab,
                                   const int64_t* __restrict__ t_slot, int num_t, long long n, int clamp) {
  const DdpmCoef k = ddpm_coef(c, tab, t_slot, num_t);
  const float s = s_ptr ? *s_ptr : 1.0f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float xi = x[i];
    float x0 = __fsub_rn(__fmul_rn(k.ca, xi), __fmul_rn(k.cb, eps[i]));
    if (clamp) x0 = clip_x0(x0, s);
    float v = __fadd_rn(__fmul_rn(k.c1, x0), __fmul_rn(k.c2, xi));
    if (noise) v = __fadd_rn(v, __fmul_rn(k.sigma, noise[i]));
    x[i] = v;
  }
}

// the step graph's last node: the next replay runs timestep t - 1
__global__ void ddpm_advance_kernel(int64_t* t_slot) { *t_slot -= 1; }

// launch shape of the grid-stride key, statistics and update kernels: kThreads per block, at most 148 x 8 blocks
constexpr int kThreads = 256;
int update_blocks(long long n) { return (int)std::min<long long>((n + kThreads - 1) / kThreads, 148LL * 8); }

// s = max(1, q-quantile of the n_global keys) by exact radix select, written to scratch word 263 (*s_ptr points there).
// write_keys(keys) enqueues the kernel that fills this rank's n keys at scratch word 512 once the select state is reset.
// scratch layout (32-bit words): [0,4) select state | [4,260) histogram | [260,262) count_le (u64) | 262 min_gt | 263 s |
// 264 any_nan | [512, 512+n) keys
template <class WriteKeys>
int clip_threshold(void* scratch, long long n, int64_t n_global, float q, int blocks, cudaStream_t st, const DdimReduce* red,
                   float** s_ptr, WriteKeys write_keys) {
  uint32_t* base = (uint32_t*)scratch;
  uint32_t* state = base;
  unsigned int* hist = base + 4;
  unsigned long long* count_le = (unsigned long long*)(base + 260);
  unsigned int* min_gt = base + 262;
  float* s_out = (float*)(base + 263);
  unsigned int* any_nan = base + 264;
  uint32_t* keys = base + 512;
  // torch.quantile: ranks = q * (n - 1) evaluated in fp32 (ATen quantile_compute), lerp between floor and ceil
  const float rank_f = q * (float)(n_global - 1);
  const long long lo = (long long)floorf(rank_f), hi = (long long)ceilf(rank_f);
  const float w = rank_f - floorf(rank_f);
  select_init_kernel<<<1, 256, 0, st>>>(state, hist, count_le, min_gt, any_nan, (unsigned long long)lo);
  write_keys(keys);
  for (int shift = 24; shift >= 0; shift -= 8) {
    radix_hist_kernel<<<blocks, 256, 0, st>>>(keys, n, state, shift, hist);
    if (red) DAWN_TRY(red->sum_u32(red->ctx, hist, 256, st));
    radix_pick_kernel<<<1, 32, 0, st>>>(state, shift, hist);
  }
  next_stat_kernel<<<blocks, kThreads, 0, st>>>(keys, n, state, count_le, min_gt, any_nan);
  if (red) {
    DAWN_TRY(red->sum_u64(red->ctx, count_le, 1, st));
    DAWN_TRY(red->min_u32(red->ctx, min_gt, 1, st));
    DAWN_TRY(red->sum_u32(red->ctx, any_nan, 1, st));
  }
  threshold_kernel<<<1, 1, 0, st>>>(state, count_le, min_gt, any_nan, lo, hi, w, s_out);
  *s_ptr = s_out;
  return 0;
}

// the DDIM update behind both entries below; eps_n / scale / x_n are nullptr without guidance
int ddim_update(float* x, float* x_n, const float* eps, const float* eps_n, const float* scale, const float* noise, int64_t n_local,
                int64_t n_global, float ca, float cb, float sqrt_an, float c, float sigma, float q, void* scratch, cudaStream_t st,
                const DdimReduce* red) {
  const long long n = n_local;
  const int blocks = update_blocks(n);
  float* s_ptr = nullptr;
  if (q > 0.f)
    DAWN_TRY(clip_threshold(scratch, n, n_global, q, blocks, st, red, &s_ptr, [&](uint32_t* keys) {
      x0_abs_kernel<<<blocks, kThreads, 0, st>>>(x, eps, eps_n, scale, ca, cb, n, keys);
    }));
  ddim_update_kernel<<<blocks, kThreads, 0, st>>>(x, x_n, eps, eps_n, scale, noise, s_ptr, ca, cb, sqrt_an, c, sigma, n,
                                                  q < 0.f ? 0 : 1);
  DAWN_LAUNCH_OK();
  return 0;
}

}  // namespace

// One DDIM update in place on x (n_local floats of this rank's frames of the (3, F, h, w) latent).  The dynamic threshold
// is the q-quantile of |x0| over the n_global values of the WHOLE clip: with a frame-sharded clip every rank histograms
// its own keys and the 256-bin digit histograms (4 passes), the count <= v and the min key above v are all-reduced through
// `red`, so every rank walks the identical radix-select and ends with the bit-identical threshold (SURVEY 8e-iii).
int ddim_step_impl(float* x, const float* eps, const float* noise, int64_t n_local, int64_t n_global, float ca, float cb,
                   float sqrt_an, float c, float sigma, float q, void* scratch, cudaStream_t st, const DdimReduce* red) {
  if (!x || !eps || !scratch || n_local <= 0 || n_global < n_local) { set_last_error("dawn_ddim_step: bad argument"); return -1; }
  return ddim_update(x, nullptr, eps, nullptr, nullptr, noise, n_local, n_global, ca, cb, sqrt_an, c, sigma, q, scratch, st, red);
}

// One guided DDIM update of one conditioned / null pair (n values each): the eps of the update is
// eps_n + (eps_c - eps_n) * *scale, formed inside the key and update kernels; the quantile is over this pair's n values.
int ddim_guided_step_impl(float* x_c, float* x_n, const float* eps_c, const float* eps_n, const float* noise, int64_t n_clip,
                          const float* scale, float ca, float cb, float sqrt_an, float c, float sigma, float q, void* scratch,
                          cudaStream_t st) {
  if (!x_c || !x_n || !eps_c || !eps_n || !scale || !scratch || n_clip <= 0) {
    set_last_error("dawn_ddim_step_guided: bad argument");
    return -1;
  }
  return ddim_update(x_c, x_n, eps_c, eps_n, scale, noise, n_clip, n_clip, ca, cb, sqrt_an, c, sigma, q, scratch, st, nullptr);
}

// One ancestral update in place on x, same threshold and sharding as ddim_step_impl; the step graph passes `tab` and `t_slot`
// so that one captured step serves every timestep.
int ddpm_step_impl(float* x, const float* eps, const float* noise, int64_t n_local, int64_t n_global, DdpmCoef c,
                   const DdpmCoef* tab, const int64_t* t_slot, int num_t, float q, void* scratch, cudaStream_t st,
                   const DdimReduce* red) {
  if (!x || !eps || !scratch || n_local <= 0 || n_global < n_local || (tab && (!t_slot || num_t < 1))) {
    set_last_error("dawn_ddpm_step: bad argument");
    return -1;
  }
  const long long n = n_local;
  const int blocks = update_blocks(n);
  float* s_ptr = nullptr;
  if (q > 0.f)
    DAWN_TRY(clip_threshold(scratch, n, n_global, q, blocks, st, red, &s_ptr, [&](uint32_t* keys) {
      ddpm_x0_abs_kernel<<<blocks, kThreads, 0, st>>>(x, eps, c, tab, t_slot, num_t, n, keys);
    }));
  ddpm_update_kernel<<<blocks, kThreads, 0, st>>>(x, eps, noise, s_ptr, c, tab, t_slot, num_t, n, q < 0.f ? 0 : 1);
  DAWN_LAUNCH_OK();
  return 0;
}

int ddpm_advance_slot(int64_t* t_slot, cudaStream_t st) {
  ddpm_advance_kernel<<<1, 1, 0, st>>>(t_slot);
  DAWN_LAUNCH_OK();
  return 0;
}

namespace {

// the schedule row of clip b's timestep, clamped into the table (the host wrappers check the range where t is on the host)
__device__ __forceinline__ int q_row(const int64_t* __restrict__ t, long long b, int num_t) {
  const long long v = t[b];
  return (int)(v < 0 ? 0 : (v >= num_t ? num_t - 1 : v));
}

// a[t] * x0 + b[t] * noise rounded as the reference's two fp32 products and one sum (U:1226-1232; no fused multiply-add)
__device__ __forceinline__ float q_mix(float ca, float x0, float cb, float z) { return __fadd_rn(__fmul_rn(ca, x0), __fmul_rn(cb, z)); }

// x_t = a[t_c] x0 + b[t_c] noise over B clips of n values: blockIdx.y is the clip
__global__ void q_sample_kernel(const float* __restrict__ x0, const float* __restrict__ noise, const int64_t* __restrict__ t,
                                const float* __restrict__ a, const float* __restrict__ b, int num_t, long long n,
                                float* __restrict__ out) {
  const long long c = blockIdx.y;
  const int r = q_row(t, c, num_t);
  const float ca = a[r], cb = b[r];
  const long long base = c * n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[base + i] = q_mix(ca, x0[base + i], cb, noise[base + i]);
}

// the motion estimator's flow (F, h, w, 2) and occlusion (F, 1, h, w) of clip blockIdx.y -> its latent (3, F, h, w) =
// [grid_x, grid_y, occ * 2 - 1] (FD:259-260, 281-282); with t != nullptr the latent is noised to x_t on the way out
__global__ void motion_to_latent_kernel(const float* __restrict__ flow, const float* __restrict__ occ, int F, int hw,
                                        const int64_t* __restrict__ t, const float* __restrict__ noise, const float* __restrict__ a,
                                        const float* __restrict__ b, int num_t, float* __restrict__ out) {
  const long long c = blockIdx.y;
  const long long m = (long long)F * hw;                 // pixels of one clip
  float ca = 0.f, cb = 0.f;
  if (t) {
    const int r = q_row(t, c, num_t);
    ca = a[r]; cb = b[r];
  }
  const float2* fl = reinterpret_cast<const float2*>(flow) + c * m;
  const float* oc = occ + c * m;
  float* o = out + c * 3 * m;
  const float* z = t ? noise + c * 3 * m : nullptr;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < m; p += (long long)gridDim.x * blockDim.x) {
    const float2 g = fl[p];
    float v[3] = {g.x, g.y, __fsub_rn(__fmul_rn(oc[p], 2.0f), 1.0f)};
#pragma unroll
    for (int j = 0; j < 3; ++j) o[j * m + p] = z ? q_mix(ca, v[j], cb, z[j * m + p]) : v[j];
  }
}

// grid of a per-clip elementwise pass over n values of each of B clips
dim3 clip_grid(long long n, int64_t B) {
  return dim3((unsigned)std::min<long long>((n + kThreads - 1) / kThreads, 148LL * 8 / std::max<int64_t>(1, std::min<int64_t>(B, 8))),
              (unsigned)B);
}

}  // namespace

int q_sample_impl(const float* x0, const float* noise, const int64_t* t, const float* a, const float* b, int num_t, int64_t B,
                  int64_t n, float* out, cudaStream_t st) {
  if (!x0 || !noise || !t || !a || !b || !out || num_t < 1 || B < 1 || B > 65535 || n < 1) {
    set_last_error("dawn_q_sample: bad argument");
    return -1;
  }
  q_sample_kernel<<<clip_grid(n, B), kThreads, 0, st>>>(x0, noise, t, a, b, num_t, n, out);
  DAWN_LAUNCH_OK();
  return 0;
}

int motion_to_latent_impl(const float* flow, const float* occ, int64_t B, int F, int h, int w, const int64_t* t, const float* noise,
                          const float* a, const float* b, int num_t, float* out, cudaStream_t st) {
  if (!flow || !occ || !out || B < 1 || B > 65535 || F < 1 || h < 1 || w < 1 || (t && (!noise || !a || !b || num_t < 1))) {
    set_last_error("dawn_motion_to_latent: bad argument");
    return -1;
  }
  if (reinterpret_cast<uintptr_t>(flow) % sizeof(float2)) {
    set_last_error("dawn_motion_to_latent: flow must be 8-byte aligned");
    return -1;
  }
  const int hw = h * w;
  motion_to_latent_kernel<<<clip_grid((long long)F * hw, B), kThreads, 0, st>>>(flow, occ, F, hw, t, noise, a, b, num_t, out);
  DAWN_LAUNCH_OK();
  return 0;
}

}  // namespace dawn

using namespace dawn;

extern "C" {

// single-GPU entry (see include/dawn_unet.h); dawn_unet_ddim_step in unet.cu is the frame-sharded one
int dawn_ddim_step(float* x, const float* eps, const float* noise, int64_t n, float ca, float cb, float sqrt_an, float c,
                   float sigma, float q, void* scratch, void* stream) {
  return ddim_step_impl(x, eps, noise, n, n, ca, cb, sqrt_an, c, sigma, q, scratch, (cudaStream_t)stream, nullptr);
}

// single-GPU entry (see include/dawn_unet.h); dawn_unet_ddpm_step in unet.cu is the frame-sharded one
int dawn_ddpm_step(float* x, const float* eps, const float* noise, int64_t n, float ca, float cb, float c1, float c2, float sigma,
                   float q, void* scratch, void* stream) {
  return ddpm_step_impl(x, eps, noise, n, n, DdpmCoef{ca, cb, c1, c2, sigma}, nullptr, nullptr, 0, q, scratch,
                        (cudaStream_t)stream, nullptr);
}

int dawn_q_sample(const float* x0, const float* noise, const int64_t* t, const float* sqrt_acp, const float* sqrt_1m_acp, int num_t,
                  int64_t B, int64_t n, float* out, void* stream) {
  return q_sample_impl(x0, noise, t, sqrt_acp, sqrt_1m_acp, num_t, B, n, out, (cudaStream_t)stream);
}

int dawn_motion_to_latent(const float* flow, const float* occlusion, int64_t B, int F, int h, int w, const int64_t* t,
                          const float* noise, const float* sqrt_acp, const float* sqrt_1m_acp, int num_t, float* out, void* stream) {
  return motion_to_latent_impl(flow, occlusion, B, F, h, w, t, noise, sqrt_acp, sqrt_1m_acp, num_t, out, (cudaStream_t)stream);
}

}  // extern "C"
