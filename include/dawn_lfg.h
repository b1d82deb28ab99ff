/* dawn_lfg.h — C-ABI of the H100-native LFG flow decoder (SURVEY.md §8f N1): the stage of DAWN that turns the sampled latent
 * flow / occlusion maps into video frames.
 *
 * Reference seam: `Generator.compute_fea` and `Generator.forward_with_flow` (LFG/modules/generator.py:132-171), called by
 * `FlowDiffusion.sample_one_video` once per clip and once per FRAME respectively, batch 1, in a Python loop
 * (DM_3/modules/video_flow_diffusion_model_multiGPU_v0_crema_vgg_floss_plus_faceemb_flow_fast_init_cond_test.py:327, 375-383).
 * Here the source-image encoder (first + down blocks, generator.py:140-146) runs once per clip and all frames are decoded as
 * one batch.  Plain pointers and sizes; one handle per GPU, not thread-safe, stream-ordered, no host synchronisation inside
 * set_source / decode.  All tensors fp32.  Return: 0 ok, -1 bad argument / order / unsupported configuration, -2 CUDA error;
 * text through dawn_last_error, declared in include/dawn_unet.h.
 */
#ifndef DAWN_LFG_H_
#define DAWN_LFG_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dawn_lfg dawn_lfg;

/* generator_params of config/hdtf128.yaml:82-93 (Generator.__init__, generator.py:25-57) */
typedef struct {
  int num_channels;          /* 3 */
  int block_expansion;       /* 64 */
  int max_features;          /* 512 */
  int num_down_blocks;       /* 2 */
  int num_bottleneck_blocks; /* 6 */
  int skips;                 /* 1 */
} dawn_lfg_cfg;

int dawn_lfg_create(const dawn_lfg_cfg* cfg, dawn_lfg** out);
void dawn_lfg_destroy(dawn_lfg* h);

/* replaces generator.load_state_dict(checkpoint['generator']) (FD:120): `name` is the reference state_dict key
 * (first.conv.weight, bottleneck.r0.norm1.running_var, ...); entries under pixelwise_flow_predictor.* and
 * *.num_batches_tracked are accepted and ignored (never read by the decode path).  host: fp32 values, row-major in `shape`. */
int dawn_lfg_set_param(dawn_lfg* h, const char* name, const float* host, const int64_t* shape, int ndim);
/* fold the eval-mode BatchNorms into the convolutions where a conv precedes them, repack and upload */
int dawn_lfg_commit_params(dawn_lfg* h);

/* frames per decode call, image size (H, W: multiples of 2^num_down_blocks * 16 / 8 so every level tiles), flow size (h, w) */
int dawn_lfg_set_geometry(dawn_lfg* h, int frames, int H, int W, int flow_h, int flow_w);

/* per clip: source image (3, H, W) in [0, 1] on the device -> skip features of every level (generator.py:140-146) */
int dawn_lfg_set_source(dawn_lfg* h, const float* source, void* stream);
/* replaces Generator.compute_fea (generator.py:132-136): fea (C_bottleneck, H/2^n, W/2^n) of the current source, device */
int dawn_lfg_get_fea(dawn_lfg* h, float* fea, void* stream);

/* replaces the per-frame loop over Generator.forward_with_flow (FD:375-383) for `frames` frames at once:
 *   flow (frames, h, w, 2) sampling grid in [-1, 1] (x, y), occ (frames, 1, h, w)  ->  prediction (frames, 3, H, W),
 *   deformed (frames, 3, H, W) or NULL.  All device pointers. */
int dawn_lfg_decode(dawn_lfg* h, const float* flow, const float* occ, float* prediction, float* deformed, void* stream);
/* same from the sampler's output: sample (3, frames, h, w) = [grid_x, grid_y, conf], occlusion = (conf + 1) / 2 (FD:366-369) */
int dawn_lfg_decode_sample(dawn_lfg* h, const float* sample, float* prediction, float* deformed, void* stream);
/* dawn_lfg_decode_sample with deformed == NULL, storing the frames as 8-bit RGB instead of fp32: frames (frames, H, W, 3) uint8 on
 * the device, frames[f, y, x, c] = (uint8) trunc(fl32(clamp(fl32((double) prediction[f, c, y, x] + mean[c] / 255.0), 0, 1) * 255f)),
 * the conversion unified_video_generator.py:544-548 applies to each frame (channels in RGB order) */
int dawn_lfg_decode_sample_rgb8(dawn_lfg* h, const float* sample, const double mean[3], uint8_t* frames, void* stream);

/* debugging / sub-module parity: copy of an internal activation of the last decode as (C, frames, Hl, Wl):
 * "bottleneck", "up0", "up1" (names as in oracle/lfg_oracle.py taps).  Writes C, Hl, Wl; dst may be NULL to query the shape. */
int dawn_lfg_read_tap(dawn_lfg* h, const char* name, float* dst, int* C, int* Hl, int* Wl, void* stream);

/* one layer of Face_loc_Encoder (FD:39-50), the per-clip face-box embedding fed to the UNet next to the source features:
 * out (Co, ceil(H/2), ceil(W/2)) = relu(conv3x3 stride 2 pad 1 of x (Ci, H, W) + bias).  All device pointers; weight (Co, Ci, 3, 3). */
int dawn_conv3x3_s2_relu(const float* x, int Ci, int H, int W, const float* weight, const float* bias, int Co, float* out, void* stream);

int64_t dawn_lfg_last_launch_count(dawn_lfg* h);
int64_t dawn_lfg_workspace_bytes(dawn_lfg* h);

/* Per-kernel tests: one decoder kernel on caller-owned device buffers, then a stream synchronise.  Channels-last tensors are
 * (rows, ld) fp32 with the channels first in each row; motion is (F, h, w, 4) = (grid_x, grid_y, occlusion, unused).
 *   MOTION_PACK       flow, occ (layout 0) or flow = sample (layout 1), F, h, w            -> out = motion
 *   WARP_BLEND        x = skip (H, W, C), motion, F, h, w, prev / ldp (may be NULL)       -> out (F, H, W, ldo)
 *   AFFINE_RELU       x (M, ldx), scale / shift (C, both NULL: plain ReLU), C, M           -> out (M, ldo); out may be x
 *   RESIDUAL_BN_RELU  y, x (M, C), scale / shift, C, M                                    -> out = y + x, out2 (or NULL)
 *   RELU_AVGPOOL2     x (H, W, C), H = rows (frames x an even height), ldo (0: C)        -> out (H/2, W/2, ldo)
 *   CHW_TO_HWC        x (C, H, W), Cpad                                                   -> out (H, W, Cpad)
 *   HWC_TO_CHW        x (M, ldx), C, M                                                    -> out (C, M)
 *   FINAL_CONV        x (F, H, W, ldx), C = Cin, weight (3, Cin, 7, 7), bias (3), source (3, H, W), motion, h, w,
 *                     blend                                                               -> out = prediction, out2 = deformed
 *                                                                                            (F, 3, H, W; out2 may be NULL)
 * Returns -1 with a message for a missing pointer or a geometry the kernel does not take. */
enum { DAWN_LFG_MOTION_PACK, DAWN_LFG_WARP_BLEND, DAWN_LFG_AFFINE_RELU, DAWN_LFG_RESIDUAL_BN_RELU, DAWN_LFG_RELU_AVGPOOL2,
       DAWN_LFG_CHW_TO_HWC, DAWN_LFG_HWC_TO_CHW, DAWN_LFG_FINAL_CONV };
typedef struct {
  int kernel;
  int F, H, W, h, w, C, Cpad, layout, blend;
  int ldx, ldp, ldo;
  long long M;
  const float *x, *y, *flow, *occ, *motion, *prev, *scale, *shift, *weight, *bias, *source;
  float *out, *out2;
} dawn_lfg_kernel_case;
int dawn_lfg_test_kernel(const dawn_lfg_kernel_case* c, void* stream);

/* ================================================================================================================================
 * dawn_lfg_motion — the motion estimator of the LFG autoencoder: RegionPredictor (LFG/modules/region_predictor.py),
 * BGMotionPredictor (bg_motion_predictor.py) and the Generator's PixelwiseFlowPredictor (pixelwise_flow_predictor.py), which
 * FlowAE (flow_autoenc.py) runs before the decoder above.  Same conventions as dawn_lfg: one handle per GPU, not thread-safe,
 * stream-ordered, no host synchronisation inside the three stage entries, fp32 device tensors, 0 / -1 / -2 returns.
 * The 2x2 SVD of the region covariances (region_predictor.py:16-25) is not here: the reference runs it on the host.
 */
typedef struct dawn_lfg_motion dawn_lfg_motion;

enum { DAWN_LFG_BG_ZERO = 0, DAWN_LFG_BG_AFFINE = 1 };

/* model_params of config/hdtf128.yaml / hdtf256.yaml; create accepts exactly DAWN's shipped values (in the comments), except
 * bg_type (zero or affine) and revert_axis_swap (either) */
typedef struct {
  int num_regions, num_channels;                                 /* 10, 3 */
  int estimate_affine, pca_based, fast_svd;                      /* 1, 1, 0 */
  int rp_block_expansion, rp_max_features, rp_num_blocks;        /* 32, 1024, 5 */
  float rp_temperature, rp_scale_factor;                         /* 0.1, 0.25 */
  int bg_block_expansion, bg_max_features, bg_num_blocks;        /* 32, 1024, 5 */
  int bg_type;                                                   /* DAWN_LFG_BG_AFFINE or DAWN_LFG_BG_ZERO */
  int pw_block_expansion, pw_max_features, pw_num_blocks;        /* 64, 1024, 5 */
  float pw_scale_factor;                                         /* 0.25 */
  int use_covar_heatmap, use_deformed_source, estimate_occlusion_map;   /* 1, 1, 1 */
  int revert_axis_swap;                                          /* 0 or 1 */
} dawn_lfg_motion_cfg;

int dawn_lfg_motion_create(const dawn_lfg_motion_cfg* cfg, dawn_lfg_motion** out);
void dawn_lfg_motion_destroy(dawn_lfg_motion* h);
/* reference state_dict keys: region_predictor.* / bg_predictor.* entries as those modules name them, prefixed "region_predictor."
 * and "bg_predictor.", and the generator's "pixelwise_flow_predictor.*" (including each down.weight Gaussian buffer);
 * *.num_batches_tracked is accepted and ignored */
int dawn_lfg_motion_set_param(dawn_lfg_motion* h, const char* name, const float* host, const int64_t* shape, int ndim);
/* fold the eval-mode BatchNorms into the convolutions that precede them, repack and upload */
int dawn_lfg_motion_commit_params(dawn_lfg_motion* h);
/* at most `frames` frames per stage call; H, W multiples of 128 */
int dawn_lfg_motion_set_geometry(dawn_lfg_motion* h, int frames, int H, int W);

/* RegionPredictor.forward up to the SVD (region_predictor.py:77-104): images (n, 3, H, W) -> shift (n, R, 2), covar (n, R, 2, 2),
 * heatmap (n, R, H/4, W/4) or NULL */
int dawn_lfg_motion_regions(dawn_lfg_motion* h, const float* images, int n, float* shift, float* covar, float* heatmap, void* stream);
/* BGMotionPredictor.forward: source (n_source = 1 or n, 3, H, W), driving (n, 3, H, W) -> bg (n, 3, 3) */
int dawn_lfg_motion_bg(dawn_lfg_motion* h, const float* source, int n_source, const float* driving, int n, float* bg, void* stream);
/* PixelwiseFlowPredictor.forward for n frames of one source image (3, H, W): region parameters (n, R, 2) / (n, R, 2, 2) of the
 * source and of the driving frames, bg (n, 3, 3) or NULL -> flow (n, H/4, W/4, 2) and occlusion (n, 1, H/4, W/4), the layout
 * dawn_lfg_decode takes */
int dawn_lfg_motion_flow(dawn_lfg_motion* h, const float* source, int n, const float* src_shift, const float* src_covar,
                         const float* src_affine, const float* drv_shift, const float* drv_covar, const float* drv_affine,
                         const float* bg, float* flow, float* occlusion, void* stream);
/* sub-module parity: the last call's "region_predictor" (Hourglass output, 35 channels), "bg_encoder" (last Encoder level) or
 * "flow_hourglass" (108 channels) as (C, n, Hl, Wl); *n is the frame count of that call.  dst may be NULL to query the shape. */
int dawn_lfg_motion_read_tap(dawn_lfg_motion* h, const char* name, float* dst, int* C, int* n, int* Hl, int* Wl, void* stream);
int64_t dawn_lfg_motion_last_launch_count(dawn_lfg_motion* h);
int64_t dawn_lfg_motion_workspace_bytes(dawn_lfg_motion* h);

/* Per-kernel tests: one motion-estimator kernel on caller-owned device buffers, then a stream synchronise.
 *   AA_DOWN         x = images (N, 3, H, W), weight (3, 13, 13)      -> out (N, H/4, W/4, ld): channels [off, off + cw), 3 real
 *   REGION_MOMENTS  logits (N, h, w, ldl) first R columns, temperature -> out = shift (N, R, 2), out2 = covar (N, R, 2, 2),
 *                                                                         out3 = heatmap (N, R, h, w) or NULL
 *   FLOW_INPUT      source (h, w, 4) channels-last, src_/drv_ shift / covar / affine (N, R, ...), bg (N, 3, 3) or NULL, revert
 *                                                                      -> out (N, h, w, ld) channels [off, off + cw), 4 (R + 1) real;
 *                                                                         out2 = motion (N, h, w, 2 (R + 1))
 *   FLOW_COMBINE    logits (N, h, w, ldl) R + 2 columns, motion (N, h, w, 2 (R + 1)) -> out = flow (N, h, w, 2), out2 = occ (N, 1, h, w)
 *   BG_HEAD         x (N, P = h w, ld) C = cw channels, fc_w (6, C) / fc_b (6) or both NULL -> out (N, 3, 3) */
enum { DAWN_LFG_MOTION_AA_DOWN, DAWN_LFG_MOTION_REGION_MOMENTS, DAWN_LFG_MOTION_FLOW_INPUT, DAWN_LFG_MOTION_FLOW_COMBINE,
       DAWN_LFG_MOTION_BG_HEAD };
typedef struct {
  int kernel;
  int N, H, W, h, w, R, ld, off, cw, ldl, revert;
  float temperature;
  const float *x, *weight, *logits, *motion, *source, *bg, *fc_w, *fc_b;
  const float *src_shift, *src_covar, *src_affine, *drv_shift, *drv_covar, *drv_affine;
  float *out, *out2, *out3;
} dawn_lfg_motion_kernel_case;
int dawn_lfg_motion_test_kernel(const dawn_lfg_motion_kernel_case* c, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DAWN_LFG_H_ */
