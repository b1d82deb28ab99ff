/* dawn_hubert.h — C-ABI of the H100-native HuBERT audio encoder: the stable-layer-norm HuBERT (hubert-large-ls960-ft) that turns
 * 16 kHz speech into the (frames, 1024) audio condition of every other DAWN stage, as transformers' HubertModel computes it in
 * eval mode (unified_video_generator.py:71, 433-501).
 *
 * Same conventions as include/dawn_pbnet.h: plain pointers and sizes, one handle per GPU, not thread-safe, stream-ordered, no
 * host synchronisation inside forward.  All tensors fp32.  Return: 0 ok, -1 bad argument / order / unsupported configuration,
 * -2 CUDA error; text through dawn_last_error, declared in include/dawn_unet.h.
 */
#ifndef DAWN_HUBERT_H_
#define DAWN_HUBERT_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dawn_hubert dawn_hubert;

#define DAWN_HUBERT_MAX_CONV 8

/* HubertConfig fields (hubert-large-ls960-ft values in the comments).  The feature extractor is the "layer" variant (Conv1d ->
 * LayerNorm over channels, eps 1e-5 -> GELU per layer) and the encoder the stable-layer-norm one (pre-LN layers, LayerNorm after
 * the last).  Heads are 64 wide; widths are multiples of 64; the positional conv's groups are 64 channels wide. */
typedef struct {
  int hidden_size;                          /* 1024 = 64 num_heads */
  int num_layers;                           /* 24 */
  int num_heads;                            /* 16 */
  int intermediate_size;                    /* 4096 */
  int num_conv;                             /* 7 */
  int conv_dim[DAWN_HUBERT_MAX_CONV];       /* 512 x 7, at most 2048 */
  int conv_kernel[DAWN_HUBERT_MAX_CONV];    /* 10, 3, 3, 3, 3, 2, 2: layer 0 at most 64, the others at most 52 */
  int conv_stride[DAWN_HUBERT_MAX_CONV];    /* 5, 2, 2, 2, 2, 2, 2 */
  int conv_bias;                            /* 1 */
  int pos_kernel;                           /* num_conv_pos_embeddings, 128 */
  int pos_groups;                           /* num_conv_pos_embedding_groups, 16 = hidden_size / 64 */
  float layer_norm_eps;                     /* 1e-5: feature projection and encoder LayerNorms */
} dawn_hubert_cfg;

int dawn_hubert_create(const dawn_hubert_cfg* cfg, dawn_hubert** out);
void dawn_hubert_destroy(dawn_hubert* h);

/* HubertModel's state_dict entries under their transformers names (feature_extractor.conv_layers.0.conv.weight, ...,
 * encoder.layers.0.attention.q_proj.weight, ...).  The positional conv's weight norm goes as
 * encoder.pos_conv_embed.conv.weight_g (1, 1, pos_kernel) and .weight_v (hidden, 64, pos_kernel).  masked_spec_embed is not
 * taken (SpecAugment is a no-op in eval).  host: fp32 values, row-major in `shape`. */
int dawn_hubert_set_param(dawn_hubert* h, const char* name, const float* host, const int64_t* shape, int ndim);
/* fold every pre-contraction LayerNorm's gamma / beta into the following projection and q's 1/8 into q_proj, evaluate the weight
 * norm (fp64), pack and upload */
int dawn_hubert_commit_params(dawn_hubert* h);

/* last_hidden_state of B waveforms of L samples each: input (B, L) -> out (B, T, hidden_size), all device pointers, T the
 * feature extractor's output length (T = (L_i - k_i) / s_i + 1 per layer); L must give T >= 1. */
int dawn_hubert_forward(dawn_hubert* h, const float* input, int B, int L, float* out, void* stream);
int dawn_hubert_output_length(const dawn_hubert* h, int L);
/* the encoder's hidden state after its first `layers` layers (0: after the positional conv), before the final LayerNorm: the
 * boundaries the per-layer parity tests compare.  out (B, T, hidden_size). */
int dawn_hubert_hidden(dawn_hubert* h, const float* input, int B, int L, int layers, float* out, void* stream);

int64_t dawn_hubert_last_launch_count(dawn_hubert* h);
/* device bytes of the handle's activation workspace (grows to the largest B x L run) */
int64_t dawn_hubert_workspace_bytes(dawn_hubert* h);

/* Kernel test: one kernel on caller-owned device buffers, then a stream synchronise.
 *   DAWN_HUBERT_ATTENTION: out (B * T, 64 H) = softmax(q k^T) v per 64-wide head; q, k, v (B * T, ld) rows, q pre-scaled.
 *   DAWN_HUBERT_CONV0:     out (B * T0, C) = GELU(LayerNorm(Conv1d(x (B, L); w (C, 1, k), bias, stride s); gamma, beta, eps)).
 *   DAWN_HUBERT_POS_CONV:  out (B, T, 64 G) = x + GELU(SamePad(Conv1d(x; weight_norm(g (1, 1, k), w (64 G, 64, k)), bias,
 *                          padding k / 2, G groups))), through the same fold and contractions as the network (w is weight_v). */
enum { DAWN_HUBERT_ATTENTION = 0, DAWN_HUBERT_CONV0 = 1, DAWN_HUBERT_POS_CONV = 2 };
typedef struct {
  int kernel;
  int B, T, L, H, ld, C, k, s, G;
  float eps;
  const float *q, *kk, *v, *x, *w, *bias, *gamma, *beta, *g;
  float* out;
} dawn_hubert_kernel_case;
int dawn_hubert_test_kernel(const dawn_hubert_kernel_case* c, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DAWN_HUBERT_H_ */
