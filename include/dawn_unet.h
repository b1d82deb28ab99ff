/* dawn_unet.h — C-ABI of the H100-native DAWN denoising UNet (one "denoising step").
 *
 * The reference has no FFI layer: its seam is the Python nn.Module `DynamicNfUnet3D`
 * (DM_3/modules/video_flow_diffusion_multiGPU_v0_crema_plus_faceemb_ca_multi_test.py:728-965) held by
 * `GaussianDiffusion.denoise_fn` (same file :1010) and `FlowDiffusion.unet`
 * (..._flow_fast_init_cond_test.py:140).  The entry points below are what a binding for that seam needs;
 * dawn_pytorch_b200/unet.py is the ctypes binding that keeps the reference's Python signature on top of them.
 * Plain pointers and sizes only; no torch types.  One handle per GPU, not thread-safe, stream-ordered,
 * no hidden host synchronisation inside forward calls.  All tensors are fp32.  A handle runs a batch of B clips (batch
 * elements) per call, B = 1 unless dawn_unet_set_geometry says otherwise; every per-clip tensor below then holds the B clips
 * back to back (a leading batch dimension of B) and each clip is computed as it would be on its own.
 *
 * Return value: 0 ok; -1 bad argument / unsupported configuration / wrong call order; -2 CUDA error.
 * dawn_last_error() returns a human-readable description of the last failure on this thread.
 */
#ifndef DAWN_UNET_H_
#define DAWN_UNET_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dawn_unet dawn_unet;

/* Constructor arguments of Unet3D.__init__ (reference :729-753) that change the network's shape. */
typedef struct {
  int dim;              /* 64 */
  int n_levels;         /* len(dim_mults) = 4 */
  int dim_mults[8];     /* (1,2,4,8) */
  int channels;         /* 275 = 3 + 256 + 16 */
  int cond_aud;         /* 1024 */
  int cond_pose;        /* 6 */
  int cond_eye;         /* 2 */
  int out_grid_dim;     /* 2 */
  int out_conf_dim;     /* 1 */
  int attn_heads;       /* 8  (only 8 supported) */
  int attn_dim_head;    /* 32 (only 32 supported) */
  int resnet_groups;    /* 8  (only 8 supported) */
  int init_kernel_size; /* 7 */
  int win_width;        /* 40: temporal attention attends |i-j| <= win_width (reference :117) */
  /* Fields below are zero for DAWN's own network. */
  int upconv;           /* 0: up path ConvTranspose3d (1,4,4)/(1,2,2) (use_deconv=True); 1: nearest x2 + Conv3d (1,3,3) (U:165-172) */
  int pad_mode;         /* upconv only, the Conv3d's padding_mode on H and W: 0 zeros, 1 reflect, 2 replicate, 3 circular */
  int no_sla;           /* 1: no spatial linear attention in the down and up blocks (use_sparse_linear_attn=False, U:833, 855) */
} dawn_unet_cfg;

/* replaces Unet3D.__init__ / DynamicNfUnet3D.__init__ (reference :728-877, 959-963) */
int dawn_unet_create(const dawn_unet_cfg* cfg, dawn_unet** out);
void dawn_unet_destroy(dawn_unet* h);

/* replaces nn.Module.load_state_dict (unified_video_generator.py:527-528): `name` is the reference
 * state_dict key (SURVEY Appendix B), `host` a host pointer to the fp32 values, row-major in `shape`.
 * Two auxiliary host-computed tables use the same call:
 *   "aux.time_freqs"  (dim/2,)      SinusoidalPosEmb frequencies (reference :157-159)
 *   "aux.rel_bias"    (heads, 2w+1) RelativePositionBias values for rel = -w..w (reference :111-119)  */
int dawn_unet_set_param(dawn_unet* h, const char* name, const float* host, const int64_t* shape, int ndim);
/* repack all parameters into kernel layouts and upload; must follow the last set_param */
int dawn_unet_commit_params(dawn_unet* h);

/* replaces DynamicNfUnet3D.update_num_frames (reference :964-965) and fixes the latent size.
 * For a frame-sharded clip F is the LOCAL frame count of this rank. */
int dawn_unet_set_num_frames(dawn_unet* h, int F, int height, int width);
/* B clips of F frames each in one pass (reference batch dimension, U:892-956); set_num_frames(F, h, w) is set_geometry(1, F, h, w).
 * Sizes the workspace for B*F frames and one GroupNorm statistics / FiLM / init-conv map / cross-attention table slice per clip;
 * drops every captured sampler graph.  1 <= B <= 16.  B > 1 is refused (-1) on a frame-sharded handle, with debugging taps set,
 * by init_shard (with more than one rank), forward_host and set_tap. */
int dawn_unet_set_geometry(dawn_unet* h, int B, int F, int height, int width);

/* Exact frame sharding of ONE clip over `nranks` GPUs (no reference counterpart; SURVEY 8e): rank r owns the contiguous
 * global frames [r*F, (r+1)*F).  Every temporal attention exchanges its +-win_width boundary frames with the adjacent
 * ranks (ncclSend/ncclRecv) and every GroupNorm all-reduces its 16 partial sums (fp64), so the sharded forward equals the
 * single-GPU forward.  dawn_nccl_unique_id: call on one rank, broadcast the 128 bytes, then init_shard on every rank
 * (after set_num_frames with the local F).  All inputs/outputs of forward* are then the LOCAL frames. */
int dawn_nccl_unique_id(char* out128);
int dawn_unet_init_shard(dawn_unet* h, const char* id128, int nranks, int rank, int F_global);
/* Optional, after init_shard (one process per GPU on ONE node, 2..8 ranks): GroupNorm statistics are then all-reduced by a single
 * kernel over NVLink peer memory (every rank stores its 16 partial sums into every peer's mailbox and adds the mailboxes in rank
 * order: bit-identical on all ranks) instead of ncclAllReduce.  export: this rank's mailbox as a 64-byte cudaIpc handle; exchange the
 * handles (any host channel), then import all of them (nranks x 64 bytes, rank order) and put a barrier before the next forward. */
int dawn_unet_shard_ipc_export(dawn_unet* h, char* out64);
int dawn_unet_shard_ipc_import(dawn_unet* h, const char* handles);

/* Clip invariants (SURVEY §8 a2/a5): the 272 feature channels are identical for every frame and every
 * DDIM step (reference :1167 `fea.repeat`), and cross-attention keys/values depend only on `cond`.
 * fea: device (B, channels-3, height, width); cond: device (B, F, cond_dim).  Needed by dawn_unet_forward_x3. */
int dawn_unet_set_clip_invariants(dawn_unet* h, const float* fea, const float* cond, void* stream);

/* replaces Unet3D.forward / forward_with_cond_scale(cond_scale=1) (reference :879-956) for one clip:
 * x: device (B, channels, F, height, width); t: device int64[B]; cond: device (B, F, cond_dim);
 * out: device (B, out_grid_dim + out_conf_dim, F, height, width).  The frame-invariant path of the init conv is chosen per
 * clip on the device. */
int dawn_unet_forward(dawn_unet* h, const float* x, const int64_t* t, const float* cond, float* out, void* stream);

/* same function when the caller knows the clip invariants: x_t: device (B, 3, F, height, width), t: device int64[B] */
int dawn_unet_forward_x3(dawn_unet* h, const float* x_t, const int64_t* t, float* out, void* stream);

/* end-to-end entry with HOST buffers (pinned recommended): copies x_t, fea, cond, t to the device,
 * runs set_clip_invariants + forward_x3 and copies the result back; returns after the stream is synchronised. */
int dawn_unet_forward_host(dawn_unet* h, const float* x_t, const float* fea, const float* cond, int64_t t, float* out);

/* debugging / sub-module parity: request a copy of an internal activation (names as in oracle/unet_oracle.py
 * taps, e.g. "downs.1.0") into dst (device, (C, F, h_l, w_l)) during the next forward calls; dst = NULL clears. */
int dawn_unet_set_tap(dawn_unet* h, const char* name, float* dst);
/* channels and spatial size of a tap for the current set_num_frames: writes C, h_l, w_l */
int dawn_unet_tap_shape(dawn_unet* h, const char* name, int* C, int* hl, int* wl);

/* Per-kernel-category timing with CUDA events on the launching stream (bench.py's roofline object).
 * enable(1) clears the counters and brackets every launch of the following forward calls with events;
 * read() synchronises on the last event and returns, per category, accumulated milliseconds, algorithmic
 * flops (2*MAC, counted once — not the 3 split-precision passes), algorithmic bytes and launch counts.
 * Arrays must hold DAWN_PROF_NCAT entries.  Category order: conv3x3, conv_other, qkv_proj, out_proj,
 * ca_gate, gn_hcond, attn_core, sla_context, gn_apply, rowstats, ca_rstd, misc, prep, temporal_fused_l0 (the fused
 * temporal attention launches at level 0, not counted in attn_core), conv3x3_l0 (dim -> dim 3x3 convs at level 0, not
 * counted in conv3x3). */
#define DAWN_PROF_NCAT 20
int dawn_unet_profile_enable(dawn_unet* h, int on);
int dawn_unet_profile_read(dawn_unet* h, double* ms, double* flops, double* bytes, int64_t* count);

/* number of kernels launched by the last forward on this handle (bench.py's gpu_launches) */
int64_t dawn_unet_last_launch_count(dawn_unet* h);
/* bytes of device workspace currently held */
int64_t dawn_unet_workspace_bytes(dawn_unet* h);

/* One DDIM update around the UNet (reference GaussianDiffusion.ddim_sample :1169-1205), in place on x (device, n floats):
 *   x0 = ca*x - cb*eps;  s = max(1, quantile_q(|x0|)) over all n values (torch.quantile semantics) if q > 0, else 1;
 *   q < 0: x0 is neither clamped nor divided (the reference's clip_denoised=False, U:1183);
 *   x = clamp(x0,-s,s)/s * sqrt_an + c*eps + sigma*noise      (noise = NULL for the last step: sigma*0 is added, as there)
 * every operation rounded as the reference's fp32 torch op, so the result is bit-identical to it.  As torch.quantile and clamp,
 * s is NaN when an |x0| is NaN or the quantile's lerp is inf - inf, and a NaN x0 or s gives a NaN element.
 * scratch: device buffer of n + 512 32-bit words.  No host synchronisation. */
int dawn_ddim_step(float* x, const float* eps, const float* noise, int64_t n, float ca, float cb, float sqrt_an, float c,
                   float sigma, float q, void* scratch, void* stream);

/* The same update for the frames a handle owns.  Unsharded handle: x, eps, noise hold the B clips back to back (n = B * per-clip
 * size) and each clip is updated as dawn_ddim_step would update it alone (its own quantile).  After dawn_unet_init_shard
 * the quantile spans the whole clip (n_local * nranks values): the radix-select's four 256-bin histograms, its two tail
 * statistics and its NaN flag are all-reduced (NCCL, on `stream`), so every rank applies the bit-identical threshold.  Every rank must call
 * it with the same coefficients; `noise` is this rank's slice of the clip's noise. */
int dawn_unet_ddim_step(dawn_unet* h, float* x, const float* eps, const float* noise, int64_t n_local, float ca, float cb,
                        float sqrt_an, float c, float sigma, float q, void* scratch, void* stream);

/* The whole sampling loop of one clip (reference ddim_sample :1156-1208: 20 x [UNet forward + DDIM update]) captured
 * once into ONE CUDA graph and replayed per clip with a single launch: no host work between steps.  All addresses are
 * fixed at capture: x (B,3,F,h,w) start noise in / sample out, eps (B,3,F,h,w) scratch, noise_all ((nsteps-1) x B*3*F*h*w,
 * slice k feeds step k; the last step adds none), t_all (nsteps int64, device; every clip runs step k at t_all[k]), scratch
 * (as dawn_ddim_step).
 * coef (host): nsteps x {ca, cb, sqrt_alpha_next, c, sigma}.  Per clip: fill x / noise_all, call
 * dawn_unet_set_clip_invariants (rewrites the same tables), then dawn_unet_sampler_launch(stream).
 * set_num_frames / commit_params / init_shard drop the graph. */
int dawn_unet_sampler_capture(dawn_unet* h, float* x, float* eps, const float* noise_all, const int64_t* t_all,
                              const float* coef, int nsteps, float q, void* scratch);
int dawn_unet_sampler_launch(dawn_unet* h, void* stream);

/* Classifier-free-guided DDIM update (reference forward_with_cond_scale :879-890 inside ddim_sample :1169-1205) on an
 * unsharded handle whose geometry holds B = 2b clips: clips 0..b-1 are the conditioned clips, clips b..2b-1 their null twins
 * (all-zero cond), clip i pairing with clip b+i.  x, eps: device (2b, 3, F, h, w); noise: device (b, 3, F, h, w) or NULL for
 * the last step; n_clip = 3*F*h*w.  Per pair, with s = *cond_scale_dev (a device float, so one captured graph serves every
 * scale):
 *   e = e_null + (e_cond - e_null) * s    (rounded as the reference's three fp32 ops, no fused multiply-add)
 * then the update of dawn_ddim_step with that e and the pair's own quantile; the combined e is never stored.  The new x is
 * written to BOTH the conditioned and the null slot.  scratch: n_clip + 512 32-bit words.  Returns -1 on a frame-sharded
 * handle or an odd B. */
int dawn_unet_ddim_step_guided(dawn_unet* h, float* x, const float* eps, const float* noise, int64_t n_clip, const float* cond_scale_dev,
                               float ca, float cb, float sqrt_an, float c, float sigma, float q, void* scratch, void* stream);

/* The guided sampling loop captured as one CUDA graph: nsteps x [forward_x3 over the 2b clips + dawn_unet_ddim_step_guided].
 * All addresses are fixed at capture: x (2b,3,F,h,w) start noise in both halves / sample out (both halves equal), eps
 * (2b,3,F,h,w) scratch, noise_all ((nsteps-1) x b*3*F*h*w, slice k feeds step k), t_all (nsteps int64, device),
 * cond_scale_dev (one float, device; read at every replay), scratch (as dawn_unet_ddim_step_guided), coef (host, as
 * dawn_unet_sampler_capture).  Per launch: dawn_unet_set_clip_invariants with fea (2b, ...) = [fea; fea] and cond
 * (2b, F, cond_dim) = [cond; 0], fill both halves of x, noise_all and *cond_scale_dev, then dawn_unet_sampler_launch_guided.
 * The graph has its own slot: capturing it leaves the dawn_unet_sampler_capture and dawn_unet_ddpm_capture graphs in place,
 * and capturing either of those leaves it in place.  set_geometry / commit_params / init_shard drop all three. */
int dawn_unet_sampler_capture_guided(dawn_unet* h, float* x, float* eps, const float* noise_all, const int64_t* t_all,
                                     const float* cond_scale_dev, const float* coef, int nsteps, float q, void* scratch);
int dawn_unet_sampler_launch_guided(dawn_unet* h, void* stream);

/* One ancestral (DDPM) update around the UNet (reference GaussianDiffusion.p_sample :1087-1121), in place on x (device,
 * n floats), each operation rounded as the reference's fp32 torch arithmetic (no fused multiply-add):
 *   x0 = ca*x - cb*eps;  s and the clamp exactly as dawn_ddim_step (q > 0 dynamic threshold, q = 0 clamp to [-1, 1],
 *   q < 0 no clip: the reference's clip_denoised=False);
 *   x = c1*(clamp(x0,-s,s)/s) + c2*x + sigma*noise      (noise may be NULL)
 * with ca = sqrt_recip_alphas_cumprod[t], cb = sqrt_recipm1_alphas_cumprod[t], c1/c2 = posterior_mean_coef1/2[t] and
 * sigma = [t > 0] * exp(0.5 * posterior_log_variance_clipped[t]).  scratch as dawn_ddim_step.  No host synchronisation. */
int dawn_ddpm_step(float* x, const float* eps, const float* noise, int64_t n, float ca, float cb, float c1, float c2,
                   float sigma, float q, void* scratch, void* stream);

/* The same update for the frames a handle owns.  Unsharded handle: B clips back to back, each updated as dawn_ddpm_step would
 * update it alone.  After dawn_unet_init_shard
 * the quantile spans the whole clip, as in dawn_unet_ddim_step; every rank passes the same coefficients and its slice of
 * the clip's noise. */
int dawn_unet_ddpm_step(dawn_unet* h, float* x, const float* eps, const float* noise, int64_t n_local, float ca, float cb,
                        float c1, float c2, float sigma, float q, void* scratch, void* stream);

/* One step of the ancestral loop (reference p_sample_loop :1123-1134) captured as a CUDA graph and replayed once per
 * timestep: forward_x3(x, t = *t_slot) -> eps, the DDPM update with row *t_slot of coef, then *t_slot -= 1.  All
 * addresses are fixed at capture: x (B,3,F,h,w) in/out, eps (B,3,F,h,w) scratch, noise (B,3,F,h,w; refill it on the stream
 * before every replay), t_slot (one int64, device, shared by every clip), coef (device, num_timesteps x {ca, cb, c1, c2, sigma}; the slot is
 * clamped to [0, num_timesteps) when the row is read), scratch (as dawn_ddim_step).  Per clip: fill x, set *t_slot =
 * num_timesteps - 1, call dawn_unet_set_clip_invariants, then dawn_unet_ddpm_launch(stream) num_timesteps times.
 * set_num_frames / commit_params / init_shard drop the graph.  It is held beside the dawn_unet_sampler_capture graph:
 * capturing either one leaves the other in place. */
int dawn_unet_ddpm_capture(dawn_unet* h, float* x, float* eps, const float* noise, int64_t* t_slot, const float* coef,
                           int num_timesteps, float q, void* scratch);
int dawn_unet_ddpm_launch(dawn_unet* h, void* stream);

/* Forward noising of a clean latent (reference GaussianDiffusion.q_sample U:1226-1232) for B clips of n floats each:
 *   out[c] = sqrt_acp[t[c]] * x0[c] + sqrt_1m_acp[t[c]] * noise[c]
 * rounded as the reference's two fp32 products and one sum (no fused multiply-add), so the result is bit-identical to torch.
 * x0, noise, out: device (B, n); t: device int64[B], one timestep per clip; sqrt_acp / sqrt_1m_acp: device fp32 tables of
 * num_t entries (the schedule's sqrt_alphas_cumprod and sqrt_one_minus_alphas_cumprod).  A timestep outside [0, num_t) reads
 * the nearest table row: range checks belong to the caller, where t is known on the host.  out must not overlap x0 or noise.
 * 1 <= B <= 65535.  No host synchronisation: it may be captured into a CUDA graph. */
int dawn_q_sample(const float* x0, const float* noise, const int64_t* t, const float* sqrt_acp, const float* sqrt_1m_acp, int num_t,
                  int64_t B, int64_t n, float* out, void* stream);

/* The LFG motion estimator's output as the sampler's latent (FD:248-262, 280-282): for each of B clips of F frames, flow
 * (F, h, w, 2) and occlusion (F, 1, h, w), as dawn_lfg_motion_flow writes them (clips back to back), become
 *   out (B, 3, F, h, w) = [flow_x, flow_y, occlusion * 2 - 1]      (the product and difference rounded as fp32 torch ops)
 * t == NULL: out is that x0.  t != NULL: out is dawn_q_sample of it with noise (B, 3, F, h, w) and the tables, in the same
 * pass; bit-identical to the two calls.  flow 8-byte aligned; out must not overlap the inputs.  No host synchronisation. */
int dawn_motion_to_latent(const float* flow, const float* occlusion, int64_t B, int F, int h, int w, const int64_t* t,
                          const float* noise, const float* sqrt_acp, const float* sqrt_1m_acp, int num_t, float* out, void* stream);

/* One contraction through exactly one kernel path, for per-kernel tests against a high-precision reference.
 * Out[m, n] = epilogue( sum_{tap, c} A[pixel(m, tap), c] * B[tap*Cin + c, n] ) with the product's GemmParams semantics
 * (dawn_pytorch_b200/csrc/gemm.cuh): rows m = (f, i, j) over an F x OHs x OWs output sub-grid (M = F*OHs*OWs), input pixel
 * (i*in_stride + dy[t], j*in_stride + dx[t]) of an F x IH x IW image with row stride lda (one tap: lda < Cin reads
 * overlapping rows), output pixel
 * (f*OH + i*out_stride + oy0) * OW + j*out_stride + ox0 with row stride ldo.  B is fp32 [K][ldb], K = ntaps*Cin.
 * The wgmma paths build their weight image and accumulator scale from B the way the network's weight upload does.
 * Returns -1 and launches nothing when the chosen path does not accept the geometry (it never falls back to
 * another kernel), -2 on a CUDA error; synchronises the stream before it returns. */
enum {
  DAWN_PATH_MMA_SYNC = 0,          /* mma.sync 3xTF32 implicit GEMM (every epilogue, per-frame B) */
  DAWN_PATH_TC_GEMM = 1,           /* wgmma implicit GEMM, fp32 gather producers */
  DAWN_PATH_TC_GEMM_PRESPLIT = 2,  /* wgmma implicit GEMM, A pre-split into fp16 hi | lo planes, cp.async producers */
  DAWN_PATH_TC_CONV3 = 3,          /* wgmma 3x3 halo-tile conv, fp32 gather producers */
  DAWN_PATH_TC_CONV3_TMA = 4       /* wgmma 3x3 halo-tile conv, A pre-split, halo tiles fetched by TMA */
};
typedef struct {
  int path, epi;                   /* DAWN_PATH_*; epilogue: 0 plain, 1 qkv+rotary, 2 qkv+SLA softmax, 3 qkv, 4 cross-attn gate, 5 GN apply,
                                      6 bias + erf GELU (+ residual), 7 LayerNorm fold + bias, 8 LayerNorm fold + bias + erf GELU;
                                      7 and 8 need a bias, GroupNorm stats only the plain epilogue */
  int F, IH, IW, Cin, lda;
  int ntaps; int dy[52]; int dx[52]; int in_stride;
  int OHs, OWs, OH, OW, out_stride, oy0, ox0;
  int up2;                         /* halo conv: 64-column block j of the output is parity class j of the 2x grid */
  int perm_pb, perm_F, perm_in, perm_out, perm_f_lo, perm_f_hi;
  int P;                           /* rows per frame (rotary / gate frame index, sequence-blocked order) */
  int N, ldb, ldo, ldr, drain, ln_inline;
  int rows_per_batch;              /* 0 = M */
  long long b_batch_stride;        /* floats between per-batch B matrices (mma.sync only) */
  int cpg;                         /* GroupNorm channels per group */
  float q_post_scale;
  /* device pointers owned by the caller */
  const float* A; const float* B; const float* bias; const float* Res; float* Out;
  double* stats;                   /* [16] GroupNorm partial sums, accumulated into */
  const float* rowstats;           /* [rows][2] (mu, rstd) */
  const float* wsum;               /* [N] column sums of B */
  const float* rot;                /* [frames][16][2] */
  const float* kq; const float* nkq; float* gates;
  const float* Y; int ldy; const double* gn_stats; const float* gn_w; const float* gn_b; const float* film; double gn_count;
} dawn_contraction_case;
int dawn_test_contraction(const dawn_contraction_case* c, void* stream);

/* One fused attention / cross-attention kernel, for per-kernel tests against a high-precision reference.  Weights arrive
 * as fp32 device matrices in the reference's layout; the harness builds the fp16 hi|lo images, scales and column sums with
 * the host code the network's weight upload runs.  Rows are f*P + pixel (channels last).  Every table (rotary, relative
 * bias, cross-attention keys and Gram forms, GroupNorm sums, FiLM) is a caller input.  Returns -1 and launches nothing
 * when the kernel's own shape predicate refuses the geometry (it never falls back to another kernel), -2 on a CUDA error;
 * synchronises the stream before it returns. */
enum {
  DAWN_FUSED_TEMPORAL = 0,         /* temporal_fused_(wg_)kernel: out = res + to_out(banded attention(rotary(LN-folded q|k|v of x)))
                                      over an on-chip sequence of F frames; rows [q_lo, q_hi) of it are written to out / read
                                      from res at row (f - q_lo)*P + pixel */
  DAWN_FUSED_ATTN_TC = 1,          /* attention_tc_kernel: softmax attention core over qkv rows [q | k | v] (256 each) */
  DAWN_FUSED_ATTN_SIMT = 2,        /* attention_kernel: the same operation on the fp32 SIMT kernel */
  DAWN_FUSED_SLA_CTX = 3,          /* sla_ctx_kernel + sla_merge_kernel: Bf[f] = per-head softmax_px(k) v^T composed with to_out */
  DAWN_FUSED_SLA_OUT = 4,          /* sla_out_kernel: out = x + out_bias + sum_h softmax_d(q_h) 32^-1/2 Bf[f][h] */
  DAWN_FUSED_SLA_CTX_UNFUSED = 5,  /* sla_context_kernel: Bf from a qkv buffer (ld 768) */
  DAWN_FUSED_CA_WT = 6,            /* ca_wt_kernel<C>: Wt = rstd * [1, gates] of the three cross-attentions */
  DAWN_FUSED_CA_RSTD = 7,          /* ca_rstd_kernel: Wt from given gates [F*P][24] */
  DAWN_FUSED_GN_HCOND = 8,         /* gn_hcond_kernel: SiLU(FiLM(GN(Y))) + Wt T_f, fp32 rows, or fp16 hi|lo planes if out16h */
  DAWN_FUSED_TEMPORAL_MMA_SYNC = 9 /* DAWN_FUSED_TEMPORAL on temporal_fused_kernel (mma.sync) also where the warpgroup-MMA
                                      kernel temporal_fused_wg_kernel would take the shape (F <= 256) */
};
typedef struct {
  int kernel;                      /* DAWN_FUSED_* */
  int F, P, C;                     /* frames, pixels per frame, channels (ca: ci; gn_hcond: co) */
  int band, q_lo, q_hi;            /* temporal and attention cores: |key - query| <= band attend (attention: band >= L is full) */
  int nseq, L, pb;                 /* attention cores: element e of sequence s is row ((s / pb) * L + e) * pb + s % pb if pb > 0, */
  long long seq_base_stride, elem_stride;   /* else s * seq_base_stride + e * elem_stride */
  int ldx, ldr, ldo, ld, ldb, ldy, ldbT;
  /* device pointers owned by the caller */
  const float* x; const float* res; float* out;
  const float* gamma;              /* [C] PreNorm gamma; ca: [3][C] LayerNorm_img gains */
  const float* w_qkv;              /* [768][C] to_qkv; ca: [3][64][C] to_q */
  const float* w_out;              /* [C][256] to_out */
  const float* rot;                /* [F][16][2] (cos, sin) */
  const float* bias;               /* [8][2*band+1] relative bias, rel = key - query; NULL for none (attention cores) */
  const float* qkv;                /* attention cores, unfused SLA context */
  float* Bf;                       /* [F][256][ldb] SLA context output / SLA output input */
  const float* out_bias;           /* [C] SLA to_out bias */
  const float* kq; const float* nkq; const float* G; const float* gates; float* Wt;
  const float* T; const float* Y; unsigned short* out16h; unsigned short* out16l;
  const double* gn_stats; double gn_count; int cpg; const float* gn_w; const float* gn_b; const float* film;
} dawn_fused_case;
int dawn_test_fused(const dawn_fused_case* c, void* stream);

/* One per-clip or per-step glue kernel of the UNet (csrc/kernels.cu), through the launcher the network calls, on caller-owned
 * buffers, for per-kernel tests against a high-precision reference.  The COND_TABLES and FILM descriptor arrays are built
 * on the device from `desc`.  Returns -1 and launches nothing when the geometry is refused, -2 on a CUDA error; synchronises
 * the stream before it returns.  Fields a kernel does not name are ignored. */
enum {
  DAWN_KERNEL_ROWSTATS = 0,        /* out[m] = (mean, 1/sqrt(biased var + eps)) of x row m (C channels, stride ld), m < M */
  DAWN_KERNEL_GN_APPLY = 1,        /* out = SiLU(GN(y) w + b) (+ res) from stats [clips][8][2] (fp64 sum, sum of squares over count
                                      values), cpg channels per group; row r is in clip (r / P) % clips */
  DAWN_KERNEL_COND_TABLES = 2,     /* desc[0..ndesc): ctx = Linear(SiLU(x[:, off:off+K])) (x = cond, row stride cond_ld), kv = ctx Wkv^T,
                                      then kq, nkq, G, T of slot ca; F table frames of `clips` clips */
  DAWN_KERNEL_TIME_MLP = 3,        /* out[clip] = SiLU(Linear2(GELU(Linear1(sinusoidal(t[clip * t_stride]))))), freqs [dim/2] */
  DAWN_KERNEL_FILM = 4,            /* desc[d].out[clip][j] = desc[d].W[j] . x[clip] + desc[d].b[j], x = t_silu [clips][C] */
  DAWN_KERNEL_ROTARY = 5,          /* out[f][i] = (cos, sin)((pos0 + f) freqs[i]), f < F, i < 16 */
  DAWN_KERNEL_SPLIT_ROWS = 6,      /* out_hi / out_lo = fp16 hi | lo planes [M][C] of x (row stride ld) */
  DAWN_KERNEL_NCF_TO_NHWC = 7,     /* x (clips, C, F, P) -> out (F * clips, P, Cpad) at channel c0, other channels zero */
  DAWN_KERNEL_FRAME_INVARIANCE = 8,/* flag[b] = channels [c0, C) of clip b of x (clips, C, F, P) differ between frames; flag[clips] counts */
  DAWN_KERNEL_FEA_SHIFT = 9,       /* k row-shifted channels-last copies (Cpad, at channel c0) of one (C, H, W) frame per clip */
  DAWN_KERNEL_MAP_REDUCE = 10,     /* out[i] = b[i % C] + sum_{s < k} x[s * n + i], i < n */
  DAWN_KERNEL_INIT_CONV_X3 = 11,   /* out[f * clips + b][p][0, C) (row stride ldo) = map[b][p] + k x k conv of x (clip b at
                                      x + b * clip_stride, (3, F, H, W)) with w [k * k * 3][C] */
  DAWN_KERNEL_HEADS_OUT = 12,      /* out[b][j][f][p] = 1x1 heads of x (j < ng: w, b) and y (j >= ng: w2, b2), C channels, P = H*W */
  DAWN_KERNEL_DDIM_STEP = 13,      /* the DDIM update of dawn_ddim_step on xs (n values, in place) with eps e, noise (may be NULL),
                                      coef {ca, cb, sqrt_alpha_next, c, sigma}, q and scratch (n + 512 words); see `replicas` */
  DAWN_KERNEL_DDPM_STEP = 14,      /* the ancestral update of dawn_ddpm_step, coef {ca, cb, c1, c2, sigma}; with tab (num_t rows of
                                      those five) the coefficients are row clamp(*t_slot, 0, num_t - 1), read on the device */
  DAWN_KERNEL_Q_SAMPLE = 15,       /* dawn_q_sample: out (clips, n) from x = x0, noise, t [clips], w / b = the two num_t-entry tables */
  DAWN_KERNEL_MOTION_TO_LATENT = 16 /* dawn_motion_to_latent: x = flow (clips*F, H, W, 2), y = occlusion (clips*F, 1, H, W) ->
                                      out (clips, 3, F, H, W); with t the fused noising (noise, w, b, num_t as Q_SAMPLE) */
};
#define DAWN_KERNEL_MAX_DESC 16
typedef struct {
  int off, K, co, ldbT, ca;        /* COND_TABLES: cond columns [off, off + K), block width co (MLP width 2 co), T row stride, slot */
  const float* mW; const float* mB;/* [2 co][K], [2 co] */
  const float* Wkv;                /* [128][2 co] */
  const float* nkv; const float* qs; const float* ks;   /* [2][8], [8], [8] */
  const float* Wout; const float* gout;                 /* [co][64], [co] */
  float* ctx; float* kv;           /* [F][2 co], [F][128] (table order) */
  float* kq; float* nkq; float* T; float* G;            /* [F][3][64], [3][8], [F][32][ldbT], [F][3][81] */
  const float* W; const float* b; float* out; int n;    /* FILM: [n][C], [n], [clips][n] */
} dawn_kernel_desc;
typedef struct {
  int kernel;                      /* DAWN_KERNEL_* */
  int M, C, ld, ldy, ldr, ldo;
  int F, H, W, P, clips;
  int Cpad, c0, k, skip_if, cpg, t_stride, pos0, dim, ng, nc, cond_ld, ndesc;
  long long n, cstride, clip_stride;
  double count; float eps;
  /* device pointers owned by the caller */
  const float* x; const float* y; const float* res;
  const float* w; const float* b; const float* w2; const float* b2;
  const float* map; const float* freqs; const double* stats; const int64_t* t; const int* skip_flag;
  float* out; void* out_hi; void* out_lo; int* flag;
  dawn_kernel_desc desc[DAWN_KERNEL_MAX_DESC];
  /* DDIM_STEP / DDPM_STEP.  replicas W >= 1 runs the frame-sharded select as one of W ranks that each hold these n values:
   * n_global = W n, and the cross-rank reductions are replaced by sum = W x own value, min = own value (needs W n < 2^32, the
   * range of a histogram count).  replicas = 0: the unsharded select. */
  float* xs; const float* e; const float* noise; void* scratch;
  const float* tab; const int64_t* t_slot; int num_t;
  int replicas;
  float coef[5]; float q;
} dawn_kernel_case;
int dawn_test_kernel(const dawn_kernel_case* c, void* stream);

const char* dawn_last_error(void);
/* device bytes the library holds in the process: the packed parameters and workspaces of every live handle of include/dawn_unet.h,
   include/dawn_lfg.h and include/dawn_pbnet.h */
int64_t dawn_live_bytes(void);
const char* dawn_build_info(void);

#ifdef __cplusplus
}
#endif
#endif /* DAWN_UNET_H_ */
