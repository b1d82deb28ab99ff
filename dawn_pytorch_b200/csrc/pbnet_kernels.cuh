// Kernels of PBnet's transformer decoder (reference PBnet/src/models/architectures/transformerreemb5.py:311-378,
// transformerdecoder4.py:24-206) — see pbnet_kernels.cu.  Rows are (clip, frame) pairs, row m = b * F + f; every row is
// d_model = D fp32 values.  Weights are k-major: W[k][n] is input k -> output n.
#pragma once
#include <cuda_runtime.h>

namespace dawn {

// Limits of the row kernels: one warp per row, each lane holding D / 32 outputs and the FFN's hidden row in shared memory.
constexpr int kPbMaxD = 256;          // pose_latent_dim (d_model): a multiple of 32
constexpr int kPbMaxFF = 2048;        // ff_size
constexpr int kPbMaxHeads = 32;       // heads of 32 features each
constexpr int kPbMaxOut = 32;         // pos_dim + eye_dim
constexpr int kPbMaxGroups = 8;       // column groups of one projection

// memory rows (reemb5:321-327): mem[m] = aud[m] + z[f][b] @ wz + xref[b] @ wp, for m = b * F + f.  aud (T, D) already holds the
// folded audio term and every bias; z (F, bs, Lz) as CAE.generate draws it; xref (bs, PE) the first pose of each clip.
int launch_pb_memory(const float* aud, const float* z, int Lz, const float* wz, const float* xref, int PE, const float* wp,
                     int bs, int F, int D, float* mem, cudaStream_t st);

// out[m][g * hid + c] = (x[m] @ w)[g * hid + c], for column groups g < ngroups of width hid (a multiple of 32).  Group flags:
// PB_SCALE multiplies by qscale, then PB_ROTARY rotates the interleaved pairs (2i, 2i + 1), i < npairs, of every 32-wide head
// by the angle of row m's frame: rot[f][i] = (cos, sin).  ldx = 0 reads one row for every m.  out is (T, ngroups * hid).
enum { PB_SCALE = 1, PB_ROTARY = 2 };
struct PbProjGroups { int flags[kPbMaxGroups]; };
int launch_pb_proj(const float* x, int ldx, int T, int F, int D, const float* w, int hid, int ngroups, PbProjGroups groups,
                   float qscale, const float* rot, int npairs, float* out, cudaStream_t st);

// banded multi-head attention of (bs clips) x (F frames): out[b, i, h] = softmax_j(q_i . k_j + bias[h][j - i + band]) v_j over
// |j - i| <= band, online softmax.  q, k, v: (bs * F, ld*) rows, head h at columns [32 h, 32 h + 32); bias (H, 2 band + 1);
// out (bs * F, 32 H).  One launch per 65 535 clips (gridDim.z); each launch adds 1 to *launches when it is not null.
int launch_pb_attention(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* bias, int band,
                        int bs, int F, int H, float* out, cudaStream_t st, int* launches = nullptr);

// x_out[m] = LayerNorm(res[m] + o[m] @ wo) with weight / bias (nn.LayerNorm, eps 1e-5); o (T, hid); ldr = 0: one residual row
int launch_pb_out_ln(const float* o, int hid, const float* wo, const float* res, int ldr, const float* gamma, const float* beta,
                     int T, int D, float* x_out, cudaStream_t st);

// x = LayerNorm(x + gelu(x @ w1 + b1) @ w2 + b2) (PositionwiseFeedforwardLayer + layer_norm3, erf GELU); in place.  When wf is
// not null the row goes on through finallayer instead of back to x: out[m] = mask[m] ? x @ wf + bf : 0, out (T, nout).
int launch_pb_ffn_ln(float* x, int T, int D, const float* w1, const float* b1, int ff, const float* w2, const float* b2,
                     const float* gamma, const float* beta, const float* wf, const float* bf, int nout, const unsigned char* mask,
                     float* out, cudaStream_t st);

}  // namespace dawn
