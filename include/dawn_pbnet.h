/* dawn_pbnet.h — C-ABI of the H100-native PBnet pose / blink generator: the decoder of DAWN's CVAE, which turns a clip's audio
 * features, a first pose and a noise sequence into a pose (or blink) sequence for every frame of the audio.
 *
 * Reference seam: `CAE.generate` (PBnet/src/models/modeltype/cae.py:112-172) with the decoder of transformerreemb5 / reemb6
 * (architectures/transformerreemb5.py:311-378, transformerdecoder4.py:24-221), as unified_video_generator.py:290-291 calls it.
 * Only the decoder runs at inference; the encoder is training-only.  Same conventions as include/dawn_lfg.h: plain pointers and
 * sizes, one handle per GPU, not thread-safe, stream-ordered, no host synchronisation inside generate.  All tensors fp32.
 * Return: 0 ok, -1 bad argument / order / unsupported configuration, -2 CUDA error; text through dawn_last_error, declared in
 * include/dawn_unet.h.
 */
#ifndef DAWN_PBNET_H_
#define DAWN_PBNET_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dawn_pbnet dawn_pbnet;

/* DAWN's values in the comments (PBnet/src/parser/model.py defaults; UVG:80-92).  band: the eval-mode attention window, 200 for
 * transformerreemb5 and 100 for transformerreemb6 (reemb5:119-123): keys with |j - i| > band get -1e8 and weigh exactly 0. */
typedef struct {
  int band;                  /* 200 or 100 */
  int pose_dim;              /* pos_dim + eye_dim: 6 (pose) or 2 (blink); at most 32 */
  int audio_dim;             /* 1024 */
  int latent_dim;            /* 256: width of the noise z, equal to audio_latent_dim */
  int audio_latent_dim;      /* 256 */
  int pose_latent_dim;       /* 64: d_model, a multiple of 32, at most 256 */
  int ff_size;               /* 128: at most 2048 */
  int num_layers;            /* 2: 1 to 8 */
  int num_heads;             /* 4: even, at most 32; heads are 32 wide and the rotary covers min(32, num_heads) features */
} dawn_pbnet_cfg;

int dawn_pbnet_create(const dawn_pbnet_cfg* cfg, dawn_pbnet** out);
void dawn_pbnet_destroy(dawn_pbnet* h);

/* the decoder's state_dict entries under their Decoder_TRANSFORMERREEMB5 names (firstposeEmbedding.weight,
 * seqTransDecoder.decoder_layers.0.self_attn.to_qkv.weight, ...), plus the two relative-position bias tables the caller builds
 * with the reference's bucket function: "aux.bias_tgt" and "aux.bias_mem", each (num_heads, 2 band + 1), entry [h][j - i + band].
 * The rotary frequencies are read from seqTransDecoder.decoder_layers.<num_layers - 1>.multihead_attn.rotary_emb.freqs, the
 * entry that loads last into the rotary module every layer shares.  host: fp32 values, row-major in `shape`. */
int dawn_pbnet_set_param(dawn_pbnet* h, const char* name, const float* host, const int64_t* shape, int ndim);
/* fold ztimelinear's audio and first-pose slices into audioEmbedding / firstposeEmbedding (fp64), evaluate the frame-invariant
 * prefix (init_proj of zeros, init_temporal_attn, the first layer's self-attention: one row for every frame), repack, upload */
int dawn_pbnet_commit_params(dawn_pbnet* h);

/* Decoder_TRANSFORMERREEMB5.forward for bs clips of F frames, all device pointers:
 *   audio (bs, F, audio_dim), z (F, bs, latent_dim) as CAE.generate draws it, first_pose (bs, pose_dim) = x[:, 0, :],
 *   mask (bs, F) bytes (lengths_to_mask)  ->  out (bs, F, pose_dim), zero where mask is 0.
 * Padded frames take part in every attention, as in the reference. */
int dawn_pbnet_generate(dawn_pbnet* h, const float* audio, const float* z, const float* first_pose, const unsigned char* mask,
                        int bs, int F, float* out, void* stream);

int64_t dawn_pbnet_last_launch_count(dawn_pbnet* h);
/* device bytes of the handle's activation workspace (grows to the largest bs x F generated) */
int64_t dawn_pbnet_workspace_bytes(dawn_pbnet* h);

/* Kernel test: the banded attention of one site on caller-owned device buffers, then a stream synchronise.
 *   q = (x_q @ wq) * qscale, k = x_kv @ wk, v = x_kv @ wv, rotary (freqs, npairs) on q and k by frame, then
 *   out[b, i] = softmax_j(q_i . k_j + bias[h][j - i + band]) v_j over |j - i| <= band, per 32-wide head.
 *   x_q, x_kv (bs * F, D); wq, wk, wv (D, 32 H) k-major; bias (H, 2 band + 1); out (bs * F, 32 H). */
typedef struct {
  int bs, F, D, H, band, npairs;
  float qscale;
  const float *x_q, *x_kv, *wq, *wk, *wv, *freqs, *bias;
  float* out;
} dawn_pbnet_attention_case;
int dawn_pbnet_test_attention(const dawn_pbnet_attention_case* c, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DAWN_PBNET_H_ */
