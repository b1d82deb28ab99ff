// Universal implicit-GEMM for the channels-last (F,H,W,C) activations of the DAWN UNet.
//   Out[m, n] = epilogue( sum_{tap, c} A[pixel(m, tap), c] * B[tap*Cin + c, n] )
// rows m enumerate (frame, i, j) over an output sub-grid; `taps` give the input offsets, so the
// same kernel serves 3x3 / 7x7 convs, 4x4 stride-2 down convs, the 4 parity classes of the 4x4
// stride-2 transposed conv, 1x1 convs and Linear layers (reference U:165-176, 229, 417, 608-609, 662-663).
#pragma once
#include <cuda_runtime.h>

namespace dawn {

enum Epi : int {
  EPI_PLAIN = 0,         // acc + bias (+ residual), optional GroupNorm partial statistics
  EPI_QKV_TEMPORAL = 1,  // LayerNorm fold + rotary on q,k            (U:179-188, 673-693)
  EPI_QKV_SLA = 2,       // LayerNorm fold + softmax over head dim of q, * d^-0.5   (U:615-621)
  EPI_QKV_MID = 3,       // LayerNorm fold only                        (U:841-843)
  EPI_CA_GATE = 4,       // LayerNorm_img fold + cosine-sim 2-key softmax -> gate  (U:519-555)
  EPI_GN_APPLY = 5,      // Out = SiLU(FiLM(GroupNorm(Y))) + acc       (U:235-248, 473-476)
  EPI_GELU = 6,          // gelu(acc + bias) (+ residual), erf GELU     (HuBERT positional conv)
  EPI_LN_BIAS = 7,       // LayerNorm fold + bias                       (HuBERT q|k|v, feature projection)
  EPI_LN_BIAS_GELU = 8,  // LayerNorm fold + bias, then erf GELU        (HuBERT fc1)
};

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

struct GemmParams {
  // A operand (gathered)
  const float* A; int lda; int Cin;
  // optional pre-split copy of A (fp16 hi and lo planes, dense rows of Cin halfs): the wgmma-kernel producers then only copy
  const unsigned short* A16h = nullptr; const unsigned short* A16l = nullptr;
  int want_split = 0;      // host side: ask choose_path (contraction.cuh) for the pre-split copy
  int up2 = 0;             // halo conv3 kernel only: 64-column block j of the output is parity class j of a 2x upsampled grid
  int IH, IW;              // input frame dims
  int OHs, OWs;            // output sub-grid dims; rows m = (f, i, j)
  int in_stride;           // input pixel = (i*in_stride + dy, j*in_stride + dx)
  int ntaps; signed char dy[52]; signed char dx[52];
  int M, N, K;             // K = ntaps * Cin (multiple of 32)
  int rows_per_batch;      // rows sharing one B matrix (P for per-frame weights, else M)
  // sequence-blocked row order for temporal attention (1x1 problems only): row m = ((p / pb) * F + f) * pb + p % pb
  // stands for pixel f * P + p.  perm_in: the A operand / LayerNorm statistics / rotary frame of row m come from that
  // pixel; perm_out: output and residual of row m go to that pixel.  pb = 0 disables.
  int perm_pb, perm_F, perm_in, perm_out;
  int perm_f_lo, perm_f_hi;  // perm_out only: rows whose frame f lies outside [f_lo, f_hi) are dropped, the rest go to frame f - f_lo
  // B operand [K][ldb] (ldb multiple of 64, zero padded)
  const float* B; int ldb; long long b_batch_stride;
  const float* Bimg;       // optional wgmma image of B (tc_pack_weights), or null
  float tc_scale;          // accumulator rescale of the wgmma path: 1 / (activation scale * weight image scale)
  // output
  float* Out; int ldo; int OH, OW, out_stride, oy0, ox0;
  const float* bias;
  const float* Res; int ldr;
  double* stats; int cpg;  // GroupNorm accumulators [groups][2], channels per group
  int clips;               // >= 1 clips interleaved by frame (frame index = f * clips + clip): stats and gn_stats are [clips][16], film [clips][2N]
  // LayerNorm fold
  const float* rowstats;   // [M][2] (mu, rstd); null on the wgmma path when ln_inline is set
  int ln_inline;           // wgmma 1x1 GEMMs: the producers accumulate each row's sum / sum of squares while they stream it
  const float* wsum;       // [N]  sum_k B[k][n]
  const float* rot;        // [F][16][2] (cos, sin)
  int P;                   // positions per frame (row -> frame index)
  float q_post_scale;
  // cross-attention gate
  const float* kq;         // [F][3][64]
  const float* nkq;        // [3][8]
  float* gates;            // [M][24]
  // GroupNorm apply
  const float* Y; int ldy; const double* gn_stats; const float* gn_w; const float* gn_b;
  const float* film;       // [2N] scale | shift, or null
  double gn_count;         // elements per group
  const int* skip_flag; int skip_if;   // mma.sync kernel only: return at once when *skip_flag == skip_if (device-side path selection)
  int drain;                   // wgmma kernels: K panels (tc_gemm) / taps (tc_conv3) accumulated in registers before the fp32 drain; 0 = default
                               // (4 panels = K 256 / 9 taps = K 576).  The tensor core adds with round-toward-zero: un-normalised conv stacks
                               // (LFG decoder) drain every panel / tap to keep the bias below the fp32 tolerance.
};

// pixel index (f * P + p) of row m in sequence-blocked order
__host__ __device__ inline int seq_blocked_pixel(int m, int pb, int F, int P) {
  const int blk = m / (F * pb), rem = m - blk * F * pb;
  const int f = rem / pb, pi = rem - f * pb;
  return f * P + blk * pb + pi;
}
// same, for an output restricted to frames [f_lo, f_hi): returns -1 for rows of other (halo) frames
__host__ __device__ inline int seq_blocked_out_pixel(int m, int pb, int F, int P, int f_lo, int f_hi) {
  const int blk = m / (F * pb), rem = m - blk * F * pb;
  const int f = rem / pb, pi = rem - f * pb;
  if (f < f_lo || f >= f_hi) return -1;
  return (f - f_lo) * P + blk * pb + pi;
}

int launch_gemm(const GemmParams& p, int epi, cudaStream_t st);

}  // namespace dawn
