// wgmma implicit GEMM for the DAWN UNet contractions (sm_90a): Out = epilogue(A (gathered, fp32) x B (weights)).
//
//   * 128-row position tile x 64/128-column output tile, K streamed in 64-element panels (= one 128-byte swizzle row of fp16).
//   * fp32-level parity needs the 3-term split  hi*hi + hi*lo + lo*hi  (SURVEY App. D).  The pieces are FP16
//     (K = 16 per instruction): an fp16 piece carries the same 11-bit significand as a TF32 piece, so hi+lo keeps
//     ~22 bits like 3xTF32, but every MMA does twice the work of a K = 8 TF32 one and reads half the bytes.
//     fp16's narrow exponent is handled with an exact power-of-two pre-scale of each weight matrix (undone in the
//     epilogue); activations stay unscaled (|x| < 65504; tiny lo pieces go subnormal, abs error <= 2^-25).  A is split on the fly by the producer warps, B is pre-split and pre-swizzled on the
//     host into ready-to-copy shared-memory images (1-D bulk copies, no tensor maps).
//   * The tensor core adds into its accumulator with truncation; chained over a long K that is a biased error
//     (1.4e-4 at K=14112).  So the register accumulator only spans CHUNK panels (first MMA overwrites) and is then
//     added into an fp32 tile in shared memory with ordinary round-to-nearest adds.
//   * persistent CTAs of whole warpgroups: 0-1 A producers (gather + split + swizzled st.shared, global loads prefetched
//     two panels ahead in registers for BN = 64, one for BN = 128), then BN/64 consumer warpgroups (wgmma on 128 rows x 64
//     columns each, then the epilogue with one output row per thread, read back from the staged tile), last the weight
//     loader (one thread; the other three warps exit).  setmaxnreg moves registers from the loader warpgroup to the
//     consumers (budgets in Cfg), so the consumers' accumulators and the producers' prefetch do not spill.
//   * each chunk of CHUNK (or `drain`) panels is expanded at compile time: wait_group 1 between panels keeps one panel's
//     MMAs in flight while the next is issued, wait_group 0 comes only before the drain.
#include <cuda_fp16.h>
#include "common.cuh"
#include "f16x3.cuh"
#include "gemm.cuh"
#include "tc_common.cuh"
#include "tc_gemm.cuh"

namespace dawn {
namespace {

constexpr int BM = 128;
constexpr int BKP = 64;                 // K elements per panel row (64 fp16 = 128 bytes)
constexpr int CHUNK = 4;                // panels accumulated in the register accumulator before a drain (K = 256)
constexpr int A_PANEL_MIN = BM * 128;    // 16 KB
constexpr int NPROD = 256;              // producer threads (warps 0-7)

// BN = 64: one consumer warpgroup, 3 stages of 48 KB.  BN = 128: two consumer warpgroups (64 columns each), 2 stages of 64 KB.
// Each consumer warpgroup also owns a 128 x 64 fp32 staging tile (34 KB); the stage counts are what fits next to it in 227 KB.
template <int BN>
struct Cfg {
  static constexpr int NWG = BN / 64;                        // consumer warpgroups
  static constexpr int A_PANEL = A_PANEL_MIN;
  static constexpr int B_PANEL = BN * 128;
  static constexpr int STAGE_BYTES = 2 * A_PANEL + 2 * B_PANEL;
  static constexpr int STAGES = (BN == 64) ? 3 : 2;
  static constexpr int LOAD_WARP = (NPROD + 128 * NWG) / 32;
  static constexpr int NTHREADS = 32 * LOAD_WARP + 128;      // producers | consumers | loader warpgroup (one thread works)
  // registers per thread by warpgroup.  Every warp starts with what NTHREADS allows (BN = 64: 128, BN = 128: 96), and
  // setmaxnreg.inc can only take what other warpgroups of the CTA released: the producers keep their count, the loader gives
  // all but 24 back and the consumers take them.  BN = 64: 2 x 128 + 24 + 232 = 512, BN = 128: 2 x 96 + 24 + 2 x 128 = 472 (of 480)
  static constexpr uint32_t REG_LAUNCH = (65536 / NTHREADS) & ~7u;
  static constexpr uint32_t REG_LOAD = 24, REG_MMA = (BN == 64) ? 232 : 128;
  // setmaxnreg.dec may only lower a warp's count and setmaxnreg.inc only raise it
  static_assert(REG_LOAD < REG_LAUNCH && REG_MMA > REG_LAUNCH, "register budgets");
  static_assert(2 * REG_LAUNCH + REG_LOAD + NWG * REG_MMA <= NTHREADS / 128 * REG_LAUNCH, "CTA register pool");
  static constexpr int ACC_STAGE = NWG * BM * tc::kStageLd * 4;
  static constexpr int SMEM_DYN = STAGES * STAGE_BYTES + ACC_STAGE + 1024;
};

using namespace tc;

struct RowInfo { int pix; int iy, ix; };     // per tile row: input frame base pixel, top-left input coordinate

template <int EPI, int BN>
__global__ void __launch_bounds__(Cfg<BN>::NTHREADS, 1) tc_gemm_kernel(const GemmParams p, const float* __restrict__ Bimg, int KC,
                                                                       int tiles_m, int tiles_n) {
  using C = Cfg<BN>;
  constexpr int STAGES = C::STAGES, STAGE_BYTES = C::STAGE_BYTES, B_PANEL = C::B_PANEL, A_PANEL = C::A_PANEL;
  constexpr int LOAD_WARP = C::LOAD_WARP, NWG = C::NWG;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t a_full[STAGES], b_full[STAGES], slot_free[STAGES];
  __shared__ RowInfo s_rows[3][BM];
  __shared__ float2 s_ln[8][BM];              // (mu, rstd) per tile row, ring over this CTA's tiles (producers run ahead of the epilogue)
  __shared__ float s_stat[NWG][16];
  __shared__ __align__(16) float s_biasv[1024];  // the whole bias vector, fetched once per CTA (the per-tile __ldg round trip was 1-3k cycles of an epilogue-bound tile)

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);          // warp-uniform by construction
  uint8_t* smem = smem_align1024(smem_raw);

  if (tid == 0) {
    // slot_free: one arrive per consumer warp once its MMAs on the slot have completed
    for (int s = 0; s < STAGES; ++s) { mbar_init(&a_full[s], NPROD); mbar_init(&b_full[s], 1); mbar_init(&slot_free[s], 4 * NWG); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int total_tiles = tiles_m * tiles_n;
  const int Ps = p.OHs * p.OWs;
  const int chunks_per_tap = p.Cin / BKP;

  if (warp < 8) {
    // =============================================================== A producers (keep the launch register budget)
    // Work items are (tile, k-panel) pairs flattened over this CTA's tiles, so the register prefetch keeps running
    // across tile boundaries (with K = 64 a tile is a single panel: per-tile prologues exposed the full load latency).
    const int c16 = tid & 7;            // 16-byte chunk inside the 128-byte row
    const int r0 = tid >> 3;            // rows r0 + 32 q, q = 0..3
    const int my_tiles = (total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int n_items = my_tiles * KC;
    int last_table = -1;
    float ln_s[4] = {0.f, 0.f, 0.f, 0.f}, ln_ss[4] = {0.f, 0.f, 0.f, 0.f};   // LayerNorm partial sums of this thread's 4 rows
    float ln_pv[4] = {0.f, 0.f, 0.f, 0.f};                                    // per-row shift (the row's first element)
    uint32_t it = 0;

    // row table of this CTA's T-th tile (ring of 3: prefetch runs at most 2 items = 2 tiles ahead of the stores)
    auto ensure_table = [&](int T) {
      if (T <= last_table) return;
      const int tile = blockIdx.x + T * gridDim.x;
      const int m0 = (tile / tiles_n) * BM;
      if (tid < BM) {
        const int m = m0 + tid;
        RowInfo ri;
        if (m < p.M && p.perm_in) {
          ri.pix = seq_blocked_pixel(m, p.perm_pb, p.perm_F, p.P); ri.iy = 0; ri.ix = 0;
        } else if (m < p.M) {
          const int f = m / Ps, rem = m - f * Ps;
          const int i = rem / p.OWs, j = rem - i * p.OWs;
          ri.pix = f * p.IH * p.IW; ri.iy = i * p.in_stride; ri.ix = j * p.in_stride;
        } else {
          ri.pix = -1; ri.iy = 0; ri.ix = 0;
        }
        s_rows[T % 3][tid] = ri;
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      last_table = T;
    };
    auto load_item = [&](float4 (&v)[8], int g) {
      const int T = g / KC, kc = g - T * KC;
      ensure_table(T);
      const RowInfo* rows = s_rows[T % 3];
      const int tap = kc / chunks_per_tap;
      const int c0 = (kc - tap * chunks_per_tap) * BKP;
      const int dy = p.dy[tap], dx = p.dx[tap];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const RowInfo ri = rows[r0 + 32 * q];
        const int iy = ri.iy + dy, ix = ri.ix + dx;
        const bool ok = (ri.pix >= 0) && (iy >= 0) && (iy < p.IH) && (ix >= 0) && (ix < p.IW);
        if (ok) {
          const float4* src = reinterpret_cast<const float4*>(p.A + (size_t)(ri.pix + iy * p.IW + ix) * p.lda + c0) + 2 * c16;
          v[2 * q] = __ldg(src);
          v[2 * q + 1] = __ldg(src + 1);
        } else {
          v[2 * q] = make_float4(0.f, 0.f, 0.f, 0.f);
          v[2 * q + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    };
    auto store_item = [&](const float4 (&v)[8]) {
      const int s = it % STAGES;
      const uint32_t round = it / STAGES;
      mbar_wait(&slot_free[s], (round & 1) ^ 1);
      uint8_t* a_hi = smem + s * STAGE_BYTES;
      uint8_t* a_lo = a_hi + A_PANEL;
      const int Ts = (int)(it / (uint32_t)KC), kcs = (int)(it - (uint32_t)Ts * KC);
      if (p.ln_inline && kcs == 0) {
        // shift each row by its first element before summing: one-pass E[x^2] - mu^2 in fp32 cancels catastrophically when
        // |mu| >> sigma (a row at mu = 100 sigma lost ~1e-3 of its rstd); the lane holding chunk 0 of the row broadcasts it
#pragma unroll
        for (int q = 0; q < 4; ++q) ln_pv[q] = __shfl_sync(0xffffffffu, v[2 * q].x, lane & ~7);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        uint32_t h[4], l[4];
        split_f16x2_rn(v[2 * q].x, v[2 * q].y, h[0], l[0]);
        split_f16x2_rn(v[2 * q].z, v[2 * q].w, h[1], l[1]);
        split_f16x2_rn(v[2 * q + 1].x, v[2 * q + 1].y, h[2], l[2]);
        split_f16x2_rn(v[2 * q + 1].z, v[2 * q + 1].w, h[3], l[3]);
        const uint32_t off = swz(r0 + 32 * q, c16);
        *reinterpret_cast<uint4*>(a_hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(a_lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
        if (p.ln_inline) {
          const float pv = ln_pv[q];
          const float4 a = make_float4(v[2 * q].x - pv, v[2 * q].y - pv, v[2 * q].z - pv, v[2 * q].w - pv);
          const float4 b = make_float4(v[2 * q + 1].x - pv, v[2 * q + 1].y - pv, v[2 * q + 1].z - pv, v[2 * q + 1].w - pv);
          ln_s[q] += ((a.x + a.y) + (a.z + a.w)) + ((b.x + b.y) + (b.z + b.w));
          ln_ss[q] += ((a.x * a.x + a.y * a.y) + (a.z * a.z + a.w * a.w)) + ((b.x * b.x + b.y * b.y) + (b.z * b.z + b.w * b.w));
        }
      }
      if (p.ln_inline) {
        if (kcs == KC - 1) {                                   // the row is complete: reduce over the 8 lanes that share it
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float sx = ln_s[q], sxx = ln_ss[q];
#pragma unroll
            for (int o = 1; o < 8; o <<= 1) { sx += __shfl_xor_sync(0xffffffffu, sx, o); sxx += __shfl_xor_sync(0xffffffffu, sxx, o); }
            if (c16 == 0) {
              const float inv = 1.0f / (float)p.K;
              const float dm = sx * inv;                       // mean of the shifted row
              const float var = fmaxf(sxx * inv - dm * dm, 0.f);
              s_ln[Ts & 7][r0 + 32 * q] = make_float2(ln_pv[q] + dm, 1.0f / sqrtf(var + 1e-5f));
            }
            ln_s[q] = 0.f; ln_ss[q] = 0.f;
          }
        }
      }
      // no proxy fence here: fence.proxy.async compiles to MEMBAR.ALL.CTA + FENCE.VIEW.ASYNC and would make every
      // producer thread drain its outstanding prefetch loads once per panel.  The st.shared above and this arrive
      // retire in order through the same shared-memory pipe; the consumers run the proxy fence after acquiring a_full
      // (they have no loads in flight), before the async-proxy reads of wgmma.
      mbar_arrive_relaxed(&a_full[s]);
      ++it;
    };

    // Pre-split A (fp16 hi | lo planes written by split_rows_kernel): the panel rows are copied global -> shared with cp.async, no
    // register staging and no conversion.  Each thread's copies of a stage signal a_full through cp.async.mbarrier.arrive.noinc, so
    // the producers run up to STAGES panels ahead.  Used where one A panel feeds several n-tiles and the conversion was the
    // bottleneck (the 8x8-level 3x3 convolutions: 4 n-tiles, producers at ~4.5k cycles per panel against ~0.85k of MMA issue).
    if (p.A16h != nullptr) {
      for (int gi = 0; gi < n_items; ++gi, ++it) {
        const int T = gi / KC, kc = gi - T * KC;
        ensure_table(T);
        const RowInfo* rows = s_rows[T % 3];
        const int tap = kc / chunks_per_tap;
        const int c0 = (kc - tap * chunks_per_tap) * BKP;
        const int dy = p.dy[tap], dx = p.dx[tap];
        const int s = it % STAGES;
        mbar_wait(&slot_free[s], ((it / STAGES) & 1) ^ 1);
        const uint32_t a_hi = smem_u32(smem + s * STAGE_BYTES), a_lo = a_hi + A_PANEL;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const RowInfo ri = rows[r0 + 32 * q];
          const int iy = ri.iy + dy, ix = ri.ix + dx;
          const bool ok = (ri.pix >= 0) && (iy >= 0) && (iy < p.IH) && (ix >= 0) && (ix < p.IW);
          const size_t e = ok ? (size_t)(ri.pix + iy * p.IW + ix) * p.Cin + c0 + 8 * c16 : 0;
          const uint32_t off = swz(r0 + 32 * q, c16), nbytes = ok ? 16u : 0u;        // src-size 0: zero fill
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(a_hi + off), "l"(p.A16h + e), "r"(nbytes) : "memory");
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(a_lo + off), "l"(p.A16l + e), "r"(nbytes) : "memory");
        }
        asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(&a_full[s])) : "memory");
      }
    } else
    // global loads run ahead of the split/store in statically indexed register buffers:
    // two items ahead (3 buffers) for BN = 64, one item ahead (2 buffers) for BN = 128 (96-register budget)
    if constexpr (BN == 64) {
      float4 v0[8], v1[8], v2[8];
      if (n_items > 0) load_item(v0, 0);
      if (n_items > 1) load_item(v1, 1);
      for (int g = 0; g < n_items; g += 3) {
        if (g + 2 < n_items) load_item(v2, g + 2);
        store_item(v0);
        if (g + 1 < n_items) {
          if (g + 3 < n_items) load_item(v0, g + 3);
          store_item(v1);
        }
        if (g + 2 < n_items) {
          if (g + 4 < n_items) load_item(v1, g + 4);
          store_item(v2);
        }
      }
    } else {
      float4 v0[8], v1[8];
      if (n_items > 0) load_item(v0, 0);
      for (int g = 0; g < n_items; g += 2) {
        if (g + 1 < n_items) load_item(v1, g + 1);
        store_item(v0);
        if (g + 1 < n_items) {
          if (g + 2 < n_items) load_item(v0, g + 2);
          store_item(v1);
        }
      }
    }
  } else if (warp >= LOAD_WARP) {
    // =============================================================== weight loader (pre-swizzled hi|lo images)
    setmaxnreg_dec<C::REG_LOAD>();
    if (warp == LOAD_WARP && lane == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = tile % tiles_n;
        const uint8_t* src = reinterpret_cast<const uint8_t*>(Bimg) + (size_t)nt * KC * (2 * B_PANEL);
        for (int kc = 0; kc < KC; ++kc, ++it) {
          const int s = it % STAGES;
          const uint32_t round = it / STAGES;
          mbar_wait(&slot_free[s], (round & 1) ^ 1);
          mbar_arrive_expect_tx(&b_full[s], 2 * B_PANEL);
          bulk_copy_g2s(smem + s * STAGE_BYTES + 2 * A_PANEL, src + (size_t)kc * (2 * B_PANEL), 2 * B_PANEL, &b_full[s]);
        }
      }
    }
  } else {
    // =============================================================== consumers (warps 8 .. 8+4*NWG-1): MMA + epilogue
    // warpgroup wg owns output columns [64 wg, 64 wg + 64) of the tile (two m64n64 MMAs per k-step: rows 0-63 and 64-127);
    // in the epilogue thread etid owns tile row etid (row-per-thread layout, read back from the staged fp32 tile)
    setmaxnreg_inc<C::REG_MMA>();
    const int wg = (warp - 8) >> 2;
    const int ew = (warp - 8) & 3;
    const int row_in_tile = ew * 32 + lane;
    const int etid = (tid - NPROD) & 127;
    float* s_st = s_stat[wg];
    const int bar_id = 2 + wg;
    constexpr int EN = 64;                                 // columns per epilogue thread
    float* stage = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES) + wg * BM * kStageLd;
    float* wbuf = stage + ew * 32 * kStageLd;              // this warp's own staged rows, free once they are read back
    int Te = -1;
    const bool bias_s = (p.bias != nullptr) && p.N <= 1024;
    if (bias_s) {
      for (int i = (tid - NPROD); i < p.N; i += 128 * NWG) s_biasv[i] = __ldg(p.bias + i);
      asm volatile("bar.sync 4, %0;" ::"n"(128 * NWG) : "memory");
    }
    const int CH = (p.drain > 0 && p.drain < CHUNK) ? p.drain : CHUNK;
    // NP consecutive K panels into the register accumulator, then one drain into the staged tile (`first`: the tile's first
    // chunk stores, later chunks add).  The panels are expanded at compile time, so the only waits are the wait_group 1 that
    // keeps one panel's MMAs in flight and the wait_group 0 before the drain.
    auto mma_chunk = [&](auto NPc, float* stage, uint32_t& it, bool first) {
      constexpr int NP = decltype(NPc)::value;
      float d0[32], d1[32];
      static_for<0, NP>([&](auto Ic) {
        constexpr int i = decltype(Ic)::value;
        const int s = it % STAGES;
        const int sprev = (it + STAGES - 1) % STAGES;        // previous panel's stage, released once its MMAs completed
        const uint32_t round = it / STAGES;
        mbar_wait(&a_full[s], round & 1);
        mbar_wait(&b_full[s], round & 1);
        fence_proxy_async();          // generic-proxy operand writes of the producers -> async proxy (see store_item)
        const uint32_t sa = smem_u32(smem + s * STAGE_BYTES);
        const uint64_t ahi = make_desc(sa), alo = make_desc(sa + A_PANEL);
        const uint64_t bhi = make_desc(sa + 2 * A_PANEL + wg * 64 * 128), blo = make_desc(sa + 2 * A_PANEL + B_PANEL + wg * 64 * 128);
        constexpr uint64_t H2 = 64 * 128 / 16;                // rows 64-127 of the A panel
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < BKP / 16; ++j) {
          const uint64_t o = (uint64_t)(j * 2);               // +32 bytes per k-step, in 16-byte units
          const uint32_t acc = (i == 0 && j == 0) ? 0u : 1u;
          wgmma_m64n64k16(d0, alo + o, bhi + o, acc);
          wgmma_m64n64k16(d1, alo + H2 + o, bhi + o, acc);
          wgmma_m64n64k16(d0, ahi + o, blo + o, 1u);
          wgmma_m64n64k16(d1, ahi + H2 + o, blo + o, 1u);
          wgmma_m64n64k16(d0, ahi + o, bhi + o, 1u);
          wgmma_m64n64k16(d1, ahi + H2 + o, bhi + o, 1u);
        }
        wgmma_commit();
        if constexpr (i == NP - 1) {
          wgmma_wait<0>();
          wgmma_fence_acc(d0); wgmma_fence_acc(d1);
          if (lane == 0) { if (i > 0) mbar_arrive(&slot_free[sprev]); mbar_arrive(&slot_free[s]); }
          stage_fragment(stage, 0, d0, first, etid);
          stage_fragment(stage, 64, d1, first, etid);
        } else {
          wgmma_wait<1>();
          wgmma_fence_acc(d0); wgmma_fence_acc(d1);
          if (lane == 0 && i > 0) mbar_arrive(&slot_free[sprev]);
        }
        ++it;
      });
    };
    static_assert(CHUNK == 4, "the chunk dispatch below expands 1 .. 4 panels");
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      ++Te;
      const int m0 = (tile / tiles_n) * BM, n0 = (tile % tiles_n) * BN + wg * EN;
      for (int kc = 0; kc < KC; kc += CH) {                 // chunks of CH panels, the last one possibly shorter
        const int np = min(CH, KC - kc);
        if (np == 4) mma_chunk(std::integral_constant<int, 4>{}, stage, it, kc == 0);
        else if (np == 3) mma_chunk(std::integral_constant<int, 3>{}, stage, it, kc == 0);
        else if (np == 2) mma_chunk(std::integral_constant<int, 2>{}, stage, it, kc == 0);
        else mma_chunk(std::integral_constant<int, 1>{}, stage, it, kc == 0);
      }
      asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
      float acc[EN];
      {
        const float4* src = reinterpret_cast<const float4*>(stage + row_in_tile * kStageLd);
#pragma unroll
        for (int i = 0; i < EN / 4; ++i) {
          const float4 v = src[i];
          acc[4 * i] = v.x; acc[4 * i + 1] = v.y; acc[4 * i + 2] = v.z; acc[4 * i + 3] = v.w;
        }
      }
      __syncwarp();

      // ---------------------------------------------------------- final epilogue: this thread owns row m
      const int m = m0 + row_in_tile;
      bool rv = m < p.M;
      const int mc = rv ? m : (p.M - 1);
      int opx = 0;
      if (p.perm_out) {
        opx = seq_blocked_out_pixel(mc, p.perm_pb, p.perm_F, p.P, p.perm_f_lo, p.perm_f_hi);
        if (opx < 0) { rv = false; opx = 0; }
      }
      const int f = mc / Ps, rem = mc - f * Ps;
      const int oi = rem / p.OWs, oj = rem - oi * p.OWs;
      const size_t opix = p.perm_out ? (size_t)opx
                                     : (size_t)(f * p.OH + oi * p.out_stride + p.oy0) * p.OW + oj * p.out_stride + p.ox0;
      const int srow = p.perm_in ? seq_blocked_pixel(mc, p.perm_pb, p.perm_F, p.P) : mc;     // pixel behind this row

      if (EPI == EPI_PLAIN || EPI == EPI_GELU) {
        const float sc = p.tc_scale;                          // undoes the exact power-of-two weight pre-scale
        if (bias_s) {
          const float4* bp = reinterpret_cast<const float4*>(s_biasv + n0);
#pragma unroll
          for (int i = 0; i < EN / 4; ++i) {
            const float4 b = bp[i];
            acc[4 * i] = fmaf(acc[4 * i], sc, b.x); acc[4 * i + 1] = fmaf(acc[4 * i + 1], sc, b.y);
            acc[4 * i + 2] = fmaf(acc[4 * i + 2], sc, b.z); acc[4 * i + 3] = fmaf(acc[4 * i + 3], sc, b.w);
          }
        } else if (p.bias) {
          const float4* bp = reinterpret_cast<const float4*>(p.bias + n0);
#pragma unroll
          for (int i = 0; i < EN / 4; ++i) {
            const float4 b = __ldg(bp + i);
            acc[4 * i] = fmaf(acc[4 * i], sc, b.x); acc[4 * i + 1] = fmaf(acc[4 * i + 1], sc, b.y);
            acc[4 * i + 2] = fmaf(acc[4 * i + 2], sc, b.z); acc[4 * i + 3] = fmaf(acc[4 * i + 3], sc, b.w);
          }
        } else {
#pragma unroll
          for (int i = 0; i < EN; ++i) acc[i] *= sc;
        }
        if (EPI == EPI_GELU) {
#pragma unroll
          for (int i = 0; i < EN; ++i) acc[i] = gelu_erf(acc[i]);
        }
        if (rv && p.Res) {
          const float4* rp = reinterpret_cast<const float4*>(p.Res + opix * p.ldr + n0);
#pragma unroll
          for (int i = 0; i < EN / 4; ++i) {
            const float4 r = rp[i];
            acc[4 * i] += r.x; acc[4 * i + 1] += r.y; acc[4 * i + 2] += r.z; acc[4 * i + 3] += r.w;
          }
        }
        store_rows_coalesced(wbuf, acc, p.Out, opix, p.ldo, n0, rv, lane);
        if (p.stats != nullptr && p.clips > 1 && m0 / Ps != (min(m0 + BM, p.M) - 1) / Ps) {
          // the tile's rows belong to several clips (small levels of a batched pass): the warp reduces its 32 rows once per clip
          // present among them and adds each clip's sums to that clip's slot
          const int clip = f % p.clips;
          unsigned rest = 0xffffffffu;
          while (rest) {
            const int c = __shfl_sync(0xffffffffu, clip, __ffs(rest) - 1);
            rest &= ~__ballot_sync(0xffffffffu, clip == c);
            const bool mine = rv && clip == c;
            double* cs = p.stats + 16 * c;
#pragma unroll
            for (int b8 = 0; b8 < EN / 8; ++b8) {
              float s = 0.f, ss = 0.f;
              if (mine) {
#pragma unroll
                for (int i = 0; i < 8; ++i) { const float x = acc[b8 * 8 + i]; s += x; ss += x * x; }
              }
              s = warp_sum(s); ss = warp_sum(ss);
              if (lane == 0) {
                const int grp = (n0 + b8 * 8) / p.cpg;
                atomicAdd(&cs[2 * grp], (double)s);
                atomicAdd(&cs[2 * grp + 1], (double)ss);
              }
            }
          }
        } else if (p.stats != nullptr) {
          // GroupNorm partial statistics (U:230): per 8-column sub-block, reduced over the warp's 32 rows
          double* cs = p.clips > 1 ? p.stats + 16 * ((m0 / Ps) % p.clips) : p.stats;
          if (etid < 16) s_st[etid] = 0.f;
          asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
#pragma unroll
          for (int b8 = 0; b8 < EN / 8; ++b8) {
            float s = 0.f, ss = 0.f;
            if (rv) {
#pragma unroll
              for (int i = 0; i < 8; ++i) { const float x = acc[b8 * 8 + i]; s += x; ss += x * x; }
            }
            s = warp_sum(s); ss = warp_sum(ss);
            if (lane == 0) {
              const int grp = (n0 + b8 * 8) / p.cpg;
              atomicAdd(&s_st[2 * grp], s);
              atomicAdd(&s_st[2 * grp + 1], ss);
            }
          }
          asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
          if (etid < 16) {
            const int grp = etid >> 1;
            const int glo = n0 / p.cpg, ghi = (n0 + EN - 1) / p.cpg;
            if (grp >= glo && grp <= ghi) atomicAdd(&cs[etid], (double)s_st[etid]);
          }
        }
      } else {
        // LayerNorm fold (see gemm.cu): v = rstd * (acc - mu * colsum)
        float mu, rs;
        if (p.ln_inline) { const float2 st = s_ln[Te & 7][row_in_tile]; mu = st.x; rs = st.y; }
        else { mu = p.rowstats[2 * (size_t)srow]; rs = p.rowstats[2 * (size_t)srow + 1]; }
        {
          const float fa = rs * p.tc_scale, fb = -rs * mu;     // rstd * (scale*acc - mu*colsum)
          const float4* wp = reinterpret_cast<const float4*>(p.wsum + n0);
#pragma unroll
          for (int i = 0; i < EN / 4; ++i) {
            const float4 w = __ldg(wp + i);
            acc[4 * i] = fmaf(fb, w.x, fa * acc[4 * i]); acc[4 * i + 1] = fmaf(fb, w.y, fa * acc[4 * i + 1]);
            acc[4 * i + 2] = fmaf(fb, w.z, fa * acc[4 * i + 2]); acc[4 * i + 3] = fmaf(fb, w.w, fa * acc[4 * i + 3]);
          }
        }
        if (EPI == EPI_LN_BIAS || EPI == EPI_LN_BIAS_GELU) {   // the folded LayerNorm beta and the Linear bias
          const float4* bp = reinterpret_cast<const float4*>(p.bias + n0);
#pragma unroll
          for (int i = 0; i < EN / 4; ++i) {
            const float4 b = __ldg(bp + i);
            acc[4 * i] += b.x; acc[4 * i + 1] += b.y; acc[4 * i + 2] += b.z; acc[4 * i + 3] += b.w;
          }
        }
        if (EPI == EPI_LN_BIAS_GELU) {
#pragma unroll
          for (int i = 0; i < EN; ++i) acc[i] = gelu_erf(acc[i]);
        }
        if (EPI == EPI_QKV_TEMPORAL) {
          if (n0 < 512) {
            const int fr = srow / p.P;
            // this row's 16 (cos, sin) pairs serve both heads of the 64-column slice
            const float4* rp = reinterpret_cast<const float4*>(p.rot + (size_t)fr * 32);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float4 cs = __ldg(rp + j);                    // pairs 2j, 2j+1
#pragma unroll
              for (int hd = 0; hd < EN / 32; ++hd) {
                const int i = hd * 32 + 4 * j;
                const float x0 = acc[i], x1 = acc[i + 1], x2 = acc[i + 2], x3 = acc[i + 3];
                acc[i] = x0 * cs.x - x1 * cs.y; acc[i + 1] = x1 * cs.x + x0 * cs.y;
                acc[i + 2] = x2 * cs.z - x3 * cs.w; acc[i + 3] = x3 * cs.z + x2 * cs.w;
              }
            }
          }
        } else if (EPI == EPI_QKV_SLA) {
          if (n0 < 256) {
#pragma unroll
            for (int hd = 0; hd < EN / 32; ++hd) {
              float mx = acc[hd * 32];
#pragma unroll
              for (int i = 1; i < 32; ++i) mx = fmaxf(mx, acc[hd * 32 + i]);
              float sum = 0.f;
#pragma unroll
              for (int i = 0; i < 32; ++i) { acc[hd * 32 + i] = expf(acc[hd * 32 + i] - mx); sum += acc[hd * 32 + i]; }
              const float inv = p.q_post_scale / sum;
#pragma unroll
              for (int i = 0; i < 32; ++i) acc[hd * 32 + i] *= inv;
            }
          }
        }
        if (EPI == EPI_CA_GATE) {
          const int fr = mc / p.P;
          const int ca = n0 >> 6;
          const float* kq = p.kq + ((size_t)fr * 3 + ca) * 64;
          const float* nk = p.nkq + ca * 8;
#pragma unroll
          for (int hd = 0; hd < 8; ++hd) {
            float nrm2 = 0.f, dr = 0.f, dn = 0.f;
#pragma unroll
            for (int d = 0; d < 8; ++d) {
              const float q = acc[hd * 8 + d];
              nrm2 += q * q; dr += q * kq[hd * 8 + d]; dn += q * nk[d];
            }
            const float inv = 8.0f / fmaxf(sqrtf(nrm2), 1e-12f);
            const float sr = dr * inv, sn = dn * inv;
            const float mx = fmaxf(sr, sn);
            const float er = expf(sr - mx), en = expf(sn - mx);
            if (rv) p.gates[(size_t)m * 24 + ca * 8 + hd] = er / (er + en);
          }
        } else {
          store_rows_coalesced(wbuf, acc, p.Out, opix, p.ldo, n0, rv, lane);
        }
      }
      asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");     // the staged tile is rewritten by the next tile's first drain
    }
  }
}

template <int EPI, int BN>
int launch_t(const GemmParams& p, const float* Bimg, cudaStream_t st) {
  using C = Cfg<BN>;
  static bool attr_set = false;
  static int num_sms = 0;
  if (!attr_set) {
    DAWN_CUDA_OK(cudaFuncSetAttribute(tc_gemm_kernel<EPI, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_DYN));
    int dev = 0;
    DAWN_CUDA_OK(cudaGetDevice(&dev));
    DAWN_CUDA_OK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    attr_set = true;
  }
  const int tiles_m = (p.M + BM - 1) / BM, tiles_n = p.N / BN;
  const int KC = p.K / BKP;
  const int grid = std::min(tiles_m * tiles_n, num_sms);
  tc_gemm_kernel<EPI, BN><<<grid, C::NTHREADS, C::SMEM_DYN, st>>>(p, Bimg, KC, tiles_m, tiles_n);
  DAWN_LAUNCH_OK();
  return 0;
}

template <int EPI>
int launch_bn(const GemmParams& p, const float* Bimg, cudaStream_t st) {
  return tc_tile_n(p.N) == 128 ? launch_t<EPI, 128>(p, Bimg, st) : launch_t<EPI, 64>(p, Bimg, st);
}

}  // namespace

// output-tile width used for a problem with N columns (also decides the weight image layout)
int tc_tile_n(int N) { return (N % 128 == 0) ? 128 : 64; }

bool tc_gemm_supported(const GemmParams& p, int epi) {
  if (epi == EPI_GN_APPLY) return false;
  if (p.b_batch_stride != 0 || p.rows_per_batch != p.M) return false;
  if (p.N % 64 != 0 || p.K % BKP != 0 || p.Cin % BKP != 0) return false;      // 64-channel panels
  if ((p.lda & 3) || (p.ldo & 3) || (p.Res && (p.ldr & 3))) return false;
  if (p.M < BM) return false;
  if (epi == EPI_PLAIN && p.stats && (p.cpg % 8 != 0)) return false;
  return true;
}

// Host: [K][ldb] fp32 weights -> per (n-tile, k-panel) shared-memory images: hi panel (BN rows x 64 fp16, 128-byte
// swizzled) | lo panel.  Weights are multiplied by the exact power of two `*scale` first so that the lo pieces
// stay fp16-normal; returns the image size in floats.
size_t tc_pack_weights(const float* Bkn, int K, int N, int ldb, std::vector<float>& out, float* scale) {
  const int BN = tc_tile_n(N);
  const int KC = K / BKP, NT = N / BN, PH = BN * 64;           // panel size in fp16 elements
  float mx = 0.f;
  for (int k = 0; k < K; ++k)
    for (int n = 0; n < N; ++n) mx = std::max(mx, std::fabs(Bkn[(size_t)k * ldb + n]));
  const float sc = f16_prescale(mx);
  *scale = sc;
  out.assign(((size_t)NT * KC * 2 * PH + 1) / 2, 0.f);
  uint16_t* base = reinterpret_cast<uint16_t*>(out.data());
  for (int nt = 0; nt < NT; ++nt)
    for (int kc = 0; kc < KC; ++kc) {
      uint16_t* hi = base + ((size_t)nt * KC + kc) * 2 * PH;
      uint16_t* lo = hi + PH;
      for (int n = 0; n < BN; ++n)
        for (int k = 0; k < BKP; ++k) {
          const int off = (n >> 3) * 512 + (n & 7) * 64 + (((k >> 3) ^ (n & 7)) << 3) + (k & 7);   // in fp16 elements
          split_f16_host(Bkn[(size_t)(kc * BKP + k) * ldb + nt * BN + n] * sc, hi[off], lo[off]);
        }
    }
  return out.size();
}

int launch_tc_gemm(const GemmParams& p, const float* Bimg, int epi, cudaStream_t st) {
  if (!tc_gemm_supported(p, epi)) { set_last_error("launch_tc_gemm: unsupported geometry"); return -1; }
  switch (epi) {
    case EPI_PLAIN: return launch_bn<EPI_PLAIN>(p, Bimg, st);
    case EPI_QKV_TEMPORAL: return launch_bn<EPI_QKV_TEMPORAL>(p, Bimg, st);
    case EPI_QKV_SLA: return launch_bn<EPI_QKV_SLA>(p, Bimg, st);
    case EPI_QKV_MID: return launch_bn<EPI_QKV_MID>(p, Bimg, st);
    case EPI_CA_GATE: return launch_bn<EPI_CA_GATE>(p, Bimg, st);
    case EPI_GELU: return launch_bn<EPI_GELU>(p, Bimg, st);
    case EPI_LN_BIAS: return launch_bn<EPI_LN_BIAS>(p, Bimg, st);
    case EPI_LN_BIAS_GELU: return launch_bn<EPI_LN_BIAS_GELU>(p, Bimg, st);
  }
  set_last_error("launch_tc_gemm: bad epilogue id");
  return -1;
}

}  // namespace dawn
