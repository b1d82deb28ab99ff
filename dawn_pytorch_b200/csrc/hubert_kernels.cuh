// Kernels of the HuBERT audio encoder (stable-layer-norm HuBERT, as transformers' HubertModel computes it in eval mode) that
// are not contractions — see hubert_kernels.cu.  Activations are channels-last fp32 rows: row m = b * T + t.
#pragma once
#include <cuda_runtime.h>

namespace dawn {

constexpr int kHbHeadDim = 64;        // every head of the encoder's self-attention is 64 wide
constexpr int kHbMaxC = 2048;         // widest row the row kernels take

// Feature-extractor layer 0: Conv1d(1 -> C, kernel k, stride s, bias) over each of B waveforms of L samples, then LayerNorm over
// the C channels (weight gamma, bias beta, eps) and erf GELU.  w (k, C) k-major, bias (C) or null; out (B * T0, C) with
// T0 = (L - k) / s + 1.
int launch_hb_conv0(const float* x, int B, int L, const float* w, const float* bias, int k, int s, int C, const float* gamma,
                    const float* beta, float eps, float* out, cudaStream_t st);

// y[m] = LayerNorm(x[m]) * gamma + beta over C channels (two-pass variance), then erf GELU when gelu; rows of stride ld (x) and
// ldo (y), C a multiple of 64.  In place when y == x.
int launch_hb_row_ln(const float* x, int ld, int M, int C, const float* gamma, const float* beta, float eps, int gelu, float* y,
                     int ldo, cudaStream_t st);

// Positional-conv input: h (B * T, G * 64) -> xg (G, B, T + 2 pad, 64), the G groups of 64 channels as separate planes, each
// sequence zero padded by `pad` rows on both sides.  Output t of group g then reads the 64 x k window that starts at row t of
// its plane: one contiguous run of k * 64 floats.
int launch_hb_group_pad(const float* h, int B, int T, int G, int pad, float* xg, cudaStream_t st);

// Full softmax attention of B sequences of T rows, H heads of 64: out[b, i, h] = softmax_j(q_i . k_j) v_j, keys streamed in
// blocks of 64 (memory O(T d) for any T), FP16x3 split products, fp32 online softmax.  q, k, v: rows of stride ld, head h at
// columns [64 h, 64 h + 64) of each; q carries its 1/sqrt(64) already.  out (B * T, 64 H) rows of stride ldo.
int launch_hb_attention(const float* q, const float* k, const float* v, int ld, int B, int T, int H, float* out, int ldo,
                        cudaStream_t st);

}  // namespace dawn
