// Universal implicit GEMM, warp-level mma.sync m16n8k8 with 3xTF32 split precision
// (hi*hi + hi*lo + lo*hi, fp32 accumulate): SURVEY Appendix D shows single-pass TF32/BF16 break the
// rtol 1e-3 / atol 1e-4 parity bar, the 3-term split sits at the fp32 re-association floor.
// This is the robust baseline contraction path; the wgmma path (tc_gemm.cu) takes over the
// large regular contractions.
#include "common.cuh"
#include "gemm.cuh"

namespace dawn {

namespace {

constexpr int BM = 128;
constexpr int BN = 64;
constexpr int BK = 32;
constexpr int STAGES = 3;
constexpr int A_LD = BK + 4;   // 36: conflict-free fragment reads (bank = 4*g + t)
constexpr int B_LD = BN + 8;   // 72: bank = 8*t + g
constexpr int THREADS = 256;
constexpr int SMEM_BYTES = STAGES * (BM * A_LD + BK * B_LD) * 4;

template <int EPI>
__global__ void __launch_bounds__(THREADS, 2) gemm_kernel(const GemmParams p) {
  extern __shared__ __align__(16) float smem[];
  float* As = smem;
  float* Bs = smem + STAGES * BM * A_LD;
  __shared__ float s_stat[16];
  __shared__ float s_gn[16 * kMaxClips];

  if (p.skip_flag && *p.skip_flag == p.skip_if) return;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int wm = warp & 3, wn = warp >> 2;
  const int g = lane >> 2, t4 = lane & 3;

  // ---- tile coordinates (rows are grouped by batch so that a tile never mixes B matrices)
  const int tiles_per_batch = (p.rows_per_batch + BM - 1) / BM;
  const int batch = blockIdx.x / tiles_per_batch;
  const int tile = blockIdx.x - batch * tiles_per_batch;
  const int m0 = batch * p.rows_per_batch + tile * BM;
  const int m_end = min(p.M, (batch + 1) * p.rows_per_batch);
  const int n0 = blockIdx.y * BN;
  const float* Bmat = p.B + (long long)batch * p.b_batch_stride;

  if (tid < 16) s_stat[tid] = 0.f;
  if (EPI == EPI_GN_APPLY && tid < 8 * p.clips) {     // (mean, rstd) of every clip's 8 groups
    double s = p.gn_stats[2 * tid], ss = p.gn_stats[2 * tid + 1];
    double mean = s / p.gn_count;
    double var = ss / p.gn_count - mean * mean;
    s_gn[2 * tid] = (float)mean;
    s_gn[2 * tid + 1] = (float)(1.0 / sqrt(var + 1e-5));
  }

  // ---- A gather bookkeeping: thread loads rows (tid/8 + 32q), 16-byte column tid%8
  const int Ps = p.OHs * p.OWs;
  const int a_c4 = (tid & 7) * 4;
  int a_pix[4], a_iy[4], a_ix[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    int m = m0 + (tid >> 3) + 32 * q;
    if (m < m_end && p.perm_in) {
      a_pix[q] = seq_blocked_pixel(m, p.perm_pb, p.perm_F, p.P); a_iy[q] = 0; a_ix[q] = 0;
    } else if (m < m_end) {
      int f = m / Ps, rem = m - f * Ps;
      int i = rem / p.OWs, j = rem - i * p.OWs;
      a_pix[q] = f * p.IH * p.IW;
      a_iy[q] = i * p.in_stride;
      a_ix[q] = j * p.in_stride;
    } else {
      a_pix[q] = -1; a_iy[q] = 0; a_ix[q] = 0;
    }
  }
  const int chunks_per_tap = p.Cin / BK;
  const int KC = p.K / BK;

  auto load_stage = [&](int kc, int stage) {
    int tap = kc / chunks_per_tap;
    int c0 = (kc - tap * chunks_per_tap) * BK;
    int dy = p.dy[tap], dx = p.dx[tap];
    float* as = As + stage * BM * A_LD;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      int iy = a_iy[q] + dy, ix = a_ix[q] + dx;
      bool ok = (a_pix[q] >= 0) && (iy >= 0) && (iy < p.IH) && (ix >= 0) && (ix < p.IW);
      const float* src = ok ? p.A + (size_t)(a_pix[q] + iy * p.IW + ix) * p.lda + c0 + a_c4 : p.A;
      cp_async16_zfill(as + ((tid >> 3) + 32 * q) * A_LD + a_c4, src, ok);
    }
    float* bs = Bs + stage * BK * B_LD;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      int idx = tid + q * THREADS;          // 0..511 : 32 rows x 16 float4
      int r = idx >> 4, c4 = (idx & 15) * 4;
      cp_async16_zfill(bs + r * B_LD + c4, Bmat + (size_t)(kc * BK + r) * p.ldb + n0 + c4, true);
    }
  };

  float acc[2][4][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < KC) load_stage(s, s);
    cp_async_commit();
  }

  for (int kc = 0; kc < KC; ++kc) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    {
      int nk = kc + STAGES - 1;
      if (nk < KC) load_stage(nk, nk % STAGES);
      cp_async_commit();
    }
    const float* as = As + (kc % STAGES) * BM * A_LD + (wm * 32) * A_LD;
    const float* bs = Bs + (kc % STAGES) * BK * B_LD + wn * 32;
#pragma unroll
    for (int ks = 0; ks < BK / 8; ++ks) {
      uint32_t ahi[2][4], alo[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const float* a = as + (mt * 16 + g) * A_LD + ks * 8 + t4;
        split_tf32(a[0], ahi[mt][0], alo[mt][0]);
        split_tf32(a[8 * A_LD], ahi[mt][1], alo[mt][1]);
        split_tf32(a[4], ahi[mt][2], alo[mt][2]);
        split_tf32(a[8 * A_LD + 4], ahi[mt][3], alo[mt][3]);
      }
      // The tensor core accumulates with round-toward-zero; chained over K that bias grows ~K*2^-24
      // (1.4e-4 at K=14112).  So each k-step's 3-term product lands in a zeroed
      // fragment and is added to the running sum with an ordinary round-to-nearest FADD.
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        uint32_t bhi[2], blo[2];
        const float* b = bs + (ks * 8 + t4) * B_LD + nt * 8 + g;
        split_tf32(b[0], bhi[0], blo[0]);
        split_tf32(b[4 * B_LD], bhi[1], blo[1]);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          float d[4] = {0.f, 0.f, 0.f, 0.f};
          mma_tf32(d, alo[mt], bhi);
          mma_tf32(d, ahi[mt], blo);
          mma_tf32(d, ahi[mt], bhi);
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[mt][nt][i] += d[i];
        }
      }
    }
  }
  cp_async_wait<0>();

  // ------------------------------------------------------------------ epilogue
  // thread owns rows r(mt,h) = m0 + wm*32 + mt*16 + g + 8h, cols n0 + wn*32 + nt*8 + 2*t4 (+1)
  const int ncol0 = n0 + wn * 32 + 2 * t4;
  float st_s[4] = {0.f, 0.f, 0.f, 0.f}, st_ss[4] = {0.f, 0.f, 0.f, 0.f};
  // GroupNorm statistics are per clip: a tile whose rows span frames of several clips adds each row's sums to its own clip's slot
  const bool mixed_clips = p.clips > 1 && m0 / Ps != (min(m0 + BM, m_end) - 1) / Ps;

#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + wm * 32 + mt * 16 + g + 8 * h;
      bool rv = m < m_end;
      const int mc = rv ? m : m0;     // clamp for address math; stores are predicated
      int opx = 0;
      if (p.perm_out) {
        opx = seq_blocked_out_pixel(mc, p.perm_pb, p.perm_F, p.P, p.perm_f_lo, p.perm_f_hi);
        if (opx < 0) { rv = false; opx = 0; }
      }
      const int f = mc / Ps;
      const int rem = mc - f * Ps;
      const int oi = rem / p.OWs, oj = rem - oi * p.OWs;
      const size_t opix = p.perm_out ? (size_t)opx
                                     : (size_t)(f * p.OH + oi * p.out_stride + p.oy0) * p.OW + oj * p.out_stride + p.ox0;
      const int srow = p.perm_in ? seq_blocked_pixel(mc, p.perm_pb, p.perm_F, p.P) : mc;   // pixel behind this row
      float v[4][2];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        v[nt][0] = acc[mt][nt][2 * h];
        v[nt][1] = acc[mt][nt][2 * h + 1];
      }

      if (EPI == EPI_PLAIN || EPI == EPI_GELU) {
        float rs_[4] = {0.f, 0.f, 0.f, 0.f}, rss_[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int n = ncol0 + nt * 8;
          if (n < p.N) {
            float b0 = 0.f, b1 = 0.f;
            if (p.bias) { b0 = p.bias[n]; b1 = p.bias[n + 1]; }
            float x0 = v[nt][0] + b0, x1 = v[nt][1] + b1;
            if (EPI == EPI_GELU) { x0 = gelu_erf(x0); x1 = gelu_erf(x1); }
            if (rv) {
              if (p.Res) {
                const float2 r = *reinterpret_cast<const float2*>(p.Res + opix * p.ldr + n);
                x0 += r.x; x1 += r.y;
              }
              *reinterpret_cast<float2*>(p.Out + opix * p.ldo + n) = make_float2(x0, x1);
              rs_[nt] = x0 + x1;
              rss_[nt] = x0 * x0 + x1 * x1;
              st_s[nt] += rs_[nt];
              st_ss[nt] += rss_[nt];
            }
          }
        }
        if (p.stats != nullptr && mixed_clips) {
          double* cs = p.stats + 16 * (f % p.clips);
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            const float s = quad_sum(rs_[nt]), ss = quad_sum(rss_[nt]);
            const int n = n0 + wn * 32 + nt * 8;
            if (t4 == 0 && rv && n < p.N) {
              const int grp = n / p.cpg;
              atomicAdd(&cs[2 * grp], (double)s);
              atomicAdd(&cs[2 * grp + 1], (double)ss);
            }
          }
        }
      } else if (EPI == EPI_GN_APPLY) {
        const int clip = p.clips > 1 ? f % p.clips : 0;
        const float* gn = s_gn + 16 * clip;
        const float* film = p.film ? p.film + (size_t)clip * 2 * p.N : nullptr;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int n = ncol0 + nt * 8;
          if (n < p.N && rv) {
            const float2 y = *reinterpret_cast<const float2*>(p.Y + opix * p.ldy + n);
            const int grp = n / p.cpg;
            const float mean = gn[2 * grp], rstd = gn[2 * grp + 1];
            float t0 = (y.x - mean) * rstd * p.gn_w[n] + p.gn_b[n];
            float t1 = (y.y - mean) * rstd * p.gn_w[n + 1] + p.gn_b[n + 1];
            if (film) {
              t0 = t0 * (film[n] + 1.f) + film[p.N + n];
              t1 = t1 * (film[n + 1] + 1.f) + film[p.N + n + 1];
            }
            *reinterpret_cast<float2*>(p.Out + opix * p.ldo + n) =
                make_float2(silu(t0) + v[nt][0], silu(t1) + v[nt][1]);
          }
        }
      } else {
        // LayerNorm fold: W(gamma .* (x-mu)*rstd) = rstd * (W' x - mu * rowsum(W'))
        const float mu = p.rowstats[2 * (size_t)srow], rs = p.rowstats[2 * (size_t)srow + 1];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int n = ncol0 + nt * 8;
          v[nt][0] = rs * (v[nt][0] - mu * p.wsum[n]);
          v[nt][1] = rs * (v[nt][1] - mu * p.wsum[n + 1]);
          if (EPI == EPI_LN_BIAS || EPI == EPI_LN_BIAS_GELU) {      // the folded LayerNorm beta and the Linear bias
            v[nt][0] += p.bias[n]; v[nt][1] += p.bias[n + 1];
          }
          if (EPI == EPI_LN_BIAS_GELU) { v[nt][0] = gelu_erf(v[nt][0]); v[nt][1] = gelu_erf(v[nt][1]); }
        }
        if (EPI == EPI_QKV_TEMPORAL) {
          const int fr = srow / p.P;
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            const int n = ncol0 + nt * 8;
            if (n < 512) {   // q and k blocks: interleaved-pair rotary, position = frame index
              const int pi = (n & 31) >> 1;
              const float2 cs = *reinterpret_cast<const float2*>(p.rot + (size_t)(fr * 16 + pi) * 2);
              const float x0 = v[nt][0], x1 = v[nt][1];
              v[nt][0] = x0 * cs.x - x1 * cs.y;
              v[nt][1] = x1 * cs.x + x0 * cs.y;
            }
          }
        } else if (EPI == EPI_QKV_SLA) {
          if (n0 + wn * 32 < 256) {   // q block: softmax over the 32 dims of this head (= this warp's columns)
            float mx = v[0][0];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) mx = fmaxf(mx, fmaxf(v[nt][0], v[nt][1]));
            mx = quad_max(mx);
            float sum = 0.f;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
              v[nt][0] = expf(v[nt][0] - mx);
              v[nt][1] = expf(v[nt][1] - mx);
              sum += v[nt][0] + v[nt][1];
            }
            sum = quad_sum(sum);
            const float inv = p.q_post_scale / sum;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) { v[nt][0] *= inv; v[nt][1] *= inv; }
          }
        }
        if (EPI == EPI_CA_GATE) {
          const int fr = mc / p.P;
          const int ca = n0 >> 6;
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            const int head = wn * 4 + nt;
            const int d0 = 2 * t4;
            const float* kq = p.kq + ((size_t)fr * 3 + ca) * 64 + head * 8 + d0;
            const float* nk = p.nkq + ca * 8 + d0;
            const float q0 = v[nt][0], q1 = v[nt][1];
            const float nrm2 = quad_sum(q0 * q0 + q1 * q1);
            const float dr = quad_sum(q0 * kq[0] + q1 * kq[1]);
            const float dn = quad_sum(q0 * nk[0] + q1 * nk[1]);
            const float inv = 8.0f / fmaxf(sqrtf(nrm2), 1e-12f);
            const float sr = dr * inv, sn = dn * inv;
            const float mx = fmaxf(sr, sn);
            const float er = expf(sr - mx), en = expf(sn - mx);
            if (t4 == 0 && rv) p.gates[(size_t)m * 24 + ca * 8 + head] = er / (er + en);
          }
        } else {
          if (rv) {
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
              const int n = ncol0 + nt * 8;
              if (n < p.N)
                *reinterpret_cast<float2*>(p.Out + opix * p.ldo + n) = make_float2(v[nt][0], v[nt][1]);
            }
          }
        }
      }
    }

  if (EPI == EPI_PLAIN && p.stats != nullptr && !mixed_clips) {
    // GroupNorm partial statistics of the values just written (U:230: statistics span the clip)
    double* cs = p.clips > 1 ? p.stats + 16 * ((m0 / Ps) % p.clips) : p.stats;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      float s = warp_sum(st_s[nt]), ss = warp_sum(st_ss[nt]);
      const int n = n0 + wn * 32 + nt * 8;
      if (lane == 0 && n < p.N) {
        const int grp = n / p.cpg;
        atomicAdd(&s_stat[2 * grp], s);
        atomicAdd(&s_stat[2 * grp + 1], ss);
      }
    }
    __syncthreads();
    if (tid < 16) {
      const int grp = tid >> 1;
      const int glo = n0 / p.cpg, ghi = (min(n0 + BN, p.N) - 1) / p.cpg;
      if (grp >= glo && grp <= ghi) atomicAdd(&cs[tid], (double)s_stat[tid]);
    }
  }
}

template <int EPI>
int launch_t(const GemmParams& p, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    DAWN_CUDA_OK(cudaFuncSetAttribute(gemm_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    attr_set = true;
  }
  const int tiles_per_batch = (p.rows_per_batch + BM - 1) / BM;
  const int nbatch = (p.M + p.rows_per_batch - 1) / p.rows_per_batch;
  dim3 grid(nbatch * tiles_per_batch, (p.N + BN - 1) / BN);
  gemm_kernel<EPI><<<grid, THREADS, SMEM_BYTES, st>>>(p);
  DAWN_LAUNCH_OK();
  return 0;
}

}  // namespace

int launch_gemm(const GemmParams& p, int epi, cudaStream_t st) {
  if (p.K % BK != 0 || p.Cin % BK != 0 || p.ldb % BN != 0 || p.ntaps > 52 || (p.lda & 3) || (p.ldo & 1)) {
    set_last_error("launch_gemm: unsupported geometry (K/Cin must be multiples of 32, ldb of 64)");
    return -1;
  }
  if (p.M <= 0) return 0;
  switch (epi) {
    case EPI_PLAIN: return launch_t<EPI_PLAIN>(p, st);
    case EPI_QKV_TEMPORAL: return launch_t<EPI_QKV_TEMPORAL>(p, st);
    case EPI_QKV_SLA: return launch_t<EPI_QKV_SLA>(p, st);
    case EPI_QKV_MID: return launch_t<EPI_QKV_MID>(p, st);
    case EPI_CA_GATE: return launch_t<EPI_CA_GATE>(p, st);
    case EPI_GN_APPLY: return launch_t<EPI_GN_APPLY>(p, st);
    case EPI_GELU: return launch_t<EPI_GELU>(p, st);
    case EPI_LN_BIAS: return launch_t<EPI_LN_BIAS>(p, st);
    case EPI_LN_BIAS_GELU: return launch_t<EPI_LN_BIAS_GELU>(p, st);
  }
  set_last_error("launch_gemm: bad epilogue id");
  return -1;
}

}  // namespace dawn
