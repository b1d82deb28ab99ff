// DDIM and ancestral (DDPM) updates around the UNet (sampler.cu): shared between the single-GPU C entry and the frame-sharded one in unet.cu.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

namespace dawn {

// cross-rank reductions of the exact radix-select (in place, stream-ordered); ctx is the caller's communicator
struct DdimReduce {
  void* ctx;
  int (*sum_u32)(void* ctx, unsigned int* buf, size_t n, cudaStream_t st);
  int (*sum_u64)(void* ctx, unsigned long long* buf, size_t n, cudaStream_t st);
  int (*min_u32)(void* ctx, unsigned int* buf, size_t n, cudaStream_t st);
};

int ddim_step_impl(float* x, const float* eps, const float* noise, int64_t n_local, int64_t n_global, float ca, float cb,
                   float sqrt_an, float c, float sigma, float q, void* scratch, cudaStream_t st, const DdimReduce* red);

// One classifier-free-guided DDIM update of a conditioned / null pair of one clip each (n_clip floats): the update of
// ddim_step_impl with eps = eps_n + (eps_c - eps_n) * (*scale) (device float), written to both x_c and x_n.  Unsharded only.
int ddim_guided_step_impl(float* x_c, float* x_n, const float* eps_c, const float* eps_n, const float* noise, int64_t n_clip,
                          const float* scale, float ca, float cb, float sqrt_an, float c, float sigma, float q, void* scratch,
                          cudaStream_t st);

// coefficients of one ancestral (DDPM) step at timestep t; layout of a row of the step graph's device table
struct DdpmCoef {
  float ca, cb;      // sqrt_recip_alphas_cumprod[t], sqrt_recipm1_alphas_cumprod[t]
  float c1, c2;      // posterior_mean_coef1[t], posterior_mean_coef2[t]
  float sigma;       // [t > 0] * exp(0.5 * posterior_log_variance_clipped[t])
};

// One DDPM update in place on x.  tab == nullptr: the coefficients are `c`.  Otherwise they are row
// clamp(*t_slot, 0, num_t - 1) of the device table tab (num_t rows), read on the device (graph replays).
int ddpm_step_impl(float* x, const float* eps, const float* noise, int64_t n_local, int64_t n_global, DdpmCoef c,
                   const DdpmCoef* tab, const int64_t* t_slot, int num_t, float q, void* scratch, cudaStream_t st,
                   const DdimReduce* red);
// *t_slot -= 1 on the stream (one thread; the last node of the ancestral step graph)
int ddpm_advance_slot(int64_t* t_slot, cudaStream_t st);

// x_t = a[t[c]] x0 + b[t[c]] noise for B clips of n values (dawn_q_sample)
int q_sample_impl(const float* x0, const float* noise, const int64_t* t, const float* a, const float* b, int num_t, int64_t B,
                  int64_t n, float* out, cudaStream_t st);
// flow (B*F, h, w, 2) and occlusion (B*F, 1, h, w) -> (B, 3, F, h, w) latent, noised when t != nullptr (dawn_motion_to_latent)
int motion_to_latent_impl(const float* flow, const float* occ, int64_t B, int F, int h, int w, const int64_t* t, const float* noise,
                          const float* a, const float* b, int num_t, float* out, cudaStream_t st);

}  // namespace dawn
