// Launchers for the non-GEMM kernels of the DAWN denoising UNet (all fp32, channels-last).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace dawn {

// per-row LayerNorm statistics (mu, rstd) over C channels; rows = pixels with stride ld.  U:179-203
int launch_rowstats(const float* x, int ld, int C, int M, float eps, float* out_mu_rstd, cudaStream_t st);

// Out = SiLU(FiLM(GroupNorm(Y))) (+ Res).  U:235-248, 478-479
// Per clip (row r is in frame r / P, clip (r / P) % clips): stats [clips][16], film [clips][2C].
int launch_gn_apply(const float* Y, int ldy, int C, int M, const double* stats, double count, int cpg, int P, int clips,
                    const float* gw, const float* gb, const float* film /*[clips][2C] or null*/,
                    const float* Res, int ldr, float* Out, int ldo, cudaStream_t st);

// ---------------------------------------------------------------- conditioning tables (clip invariants)
struct CaTableArgs {
  const float* kv;     // [F][128]  (k | v) of this cross-attention
  const float* nkv;    // [2][8] null key / value
  const float* qs;     // [8] q_scale
  const float* ks;     // [8] k_scale
  const float* Wout;   // [co][64]
  const float* gout;   // [co]
  int co; int ldbT;    // table row stride (co padded to 64)
  int ca;              // 0..2 slot
  float* kq;           // [F][3][64]
  float* nkq;          // [3][8]
  float* T;            // [F][32][ldbT]
  float* G;            // [F][3][81]
};
// one (conditioned block, cross-attention) pair of the per-clip conditioning pipeline: cond slice -> MLP -> (k | v) -> tables
struct CondDesc {
  const float* mW; const float* mB; int off, K, n1;   // Linear(SiLU(cond[:, off:off+K])) -> n1 = 2*co features
  const float* Wkv;                                   // [128][n1]
  float* ctx; float* kv;                              // scratch [F][n1], [F][128]
  CaTableArgs t;
};
// F table frames of `clips` clips: table frame f * clips + b is built from cond row b * (F / clips) + f
int launch_cond_batched(const float* cond, int cond_ld, const CondDesc* descs_dev, int ndesc, int max_n1, int max_k, int max_co, int F,
                        int clips, cudaStream_t st);

// Wt[m][ca*9 + {0, 1+h}] = rstd_ca(m) * {1, gate(m,ca,h)}           U:511-514 (to_out LayerNorm) via Gram form
int launch_ca_rstd(const float* gates, const float* G, int M, int P, float* Wt /*[M][32]*/, cudaStream_t st);

// ---------------------------------------------------------------- time embedding  U:150-162, 788-794, 366-369
// one timestep per clip: clip b uses t_dev[b * t_stride] (t_stride 0: one shared timestep) and writes t_silu[b], out[b]
struct FilmDesc { const float* W; const float* b; float* out; int n; };   // out[clip][n] = W[n][tdim] silu(t[clip]) + b
int launch_time_mlp(const int64_t* t_dev, int t_stride, int clips, const float* freqs /*[dim/2]*/, int dim, const float* W1, const float* b1,
                    const float* W2, const float* b2, float* t_silu /*[clips][4*dim]*/, cudaStream_t st);
// max_n >= every descriptor's n: all outputs of every descriptor are written
int launch_film(const FilmDesc* descs_dev, int ndesc, int max_n, int clips, const float* t_silu, int tdim, cudaStream_t st);

// rotary cos/sin table [F][16][2] from freqs[16], position = pos0 + f
int launch_rotary_table(const float* freqs, int F, int pos0, float* out, cudaStream_t st);

// ---------------------------------------------------------------- attention cores
// banded / full softmax attention over strided sequences; qkv rows are [q(256) | k(256) | v(256)], head = 32 dims
struct AttnArgs {
  const float* qkv; int ld;      // row stride (768)
  float* out; int ldo;           // [rows][256]
  int nseq; int L;               // number of sequences, sequence length
  long long seq_base_stride;     // first row of sequence s = s * seq_base_stride
  long long elem_stride;         // row step between consecutive sequence elements
  int band;                      // |i-j| <= band attend; >= L means full
  const float* bias;             // [8][2*band+1] or null
  int q_lo, q_hi;                // only queries in [q_lo, q_hi) are computed (frame sharding); keys span [0, L)
  int pb;                        // > 0: sequence-blocked rows: element e of sequence s is row ((s / pb) * L + e) * pb + s % pb
};
__host__ __device__ inline long long attn_seq_base(const AttnArgs& a, int s) {
  return a.pb > 0 ? (long long)(s / a.pb) * a.L * a.pb + (s % a.pb) : (long long)s * a.seq_base_stride;
}
__host__ __device__ inline long long attn_elem_stride(const AttnArgs& a) { return a.pb > 0 ? a.pb : a.elem_stride; }
int launch_attention(const AttnArgs& a, cudaStream_t st);          // SIMT fp32 reference kernel
bool attention_tc_supported(const AttnArgs& a);
int launch_attention_tc(const AttnArgs& a, cudaStream_t st);       // tensor-core (mma.sync fp16x3) kernel, attn_tc.cu

// spatial linear attention: per (frame, head) context + composed out-projection  U:618-626
//   Bf[f][h*32+d][c] = sum_e ctx[f,h][d][e] * WoutT[h*32+e][c]
int launch_split_rows(const float* x, int ld, int C, long long M, void* hi, void* lo, cudaStream_t st);
int launch_sla_context(const float* qkv, int ld, int F, int P, const float* WoutT /*[256][C]*/, int C,
                       float* Bf, int ldb, cudaStream_t st);

// x (frames, H, W, C) rows of stride ld -> dense (frames, H + 2, W + 2, C) with a one-pixel border at the clamped (wrap = 0) or
// wrapped (wrap = 1) index: the upconv's reflect / replicate / circular padding seen on the low-resolution grid (unet.cu)
int launch_pad_border(const float* x, int ld, int C, int frames, int H, int W, int wrap, float* out, cudaStream_t st);

// ---------------------------------------------------------------- layout / heads / init conv
// x (clips, C, F, H*W) channel-major -> (F * clips, H*W, Cpad) channels-last (frame f of clip b at f * clips + b), zero padding
// channels [C, Cpad).  skip_flag (device int, optional): the kernel returns at once when *skip_flag == skip_if (device-side path
// selection)
int launch_ncf_to_nhwc(const float* x, int C, int F, int HW, int Cpad, int c_dst0, float* out, cudaStream_t st,
                       const int* skip_flag = nullptr, int skip_if = 0, int clips = 1);
// x (clips, C, F, HW): flag[b] = 1 iff channels [c0, C) of clip b are not identical in every frame; flag[clips] = number of such clips
int launch_frame_invariance(const float* x, int c0, int C, int F, int HW, int clips, int* flag, cudaStream_t st);
// k vertically shifted channels-last copies of one (C, H, W) frame per clip (clip b's frame at x + b * clip_stride; copy s of clip b
// is output frame s * clips + b) and the reduction of the k partial maps (per-clip init-conv maps)
int launch_fea_shift_nhwc(const float* x, long long cstride, long long clip_stride, int clips, int C, int H, int W, int Cpad, int c_dst0,
                          int k, float* out, cudaStream_t st, const int* skip_flag = nullptr, int skip_if = 0);
int launch_map_reduce(const float* part, int nsplit, long long n, const float* bias, int Co, float* map, cudaStream_t st,
                      const int* skip_flag = nullptr, int skip_if = 0);
// out[f*clips+b][p][co0..] = map[b][p][:] + conv7x7(x_t[b][3][F][H][W]; w3[49*3][64])   (hoisted init conv, SURVEY a2), clip b's
// channels 0..2 at xt + b * clip_stride; skip_flag (optional) per clip: clip b is skipped when skip_flag[b] == skip_if
int launch_init_conv_x3(const float* xt, long long clip_stride, int F, int H, int W, int clips, const float* w3, const float* map, int Co,
                        float* out, int ldo, int ksz, cudaStream_t st, const int* skip_flag = nullptr, int skip_if = 0);
// eps[b][c][f][p] = head 1x1 convs of row (f*clips+b)*HW + p: c<ng from flow features, else occlusion features   U:863, 876, 956
int launch_heads_out(const float* hf, const float* ho, int C, int M, int HW, int clips, const float* Wf, const float* bf, int ng,
                     const float* Wo, const float* bo, int nc, float* out /*[clips][(ng+nc)][M/clips]*/, cudaStream_t st);

}  // namespace dawn
