// wgmma 3x3 convolution with a shared-memory HALO tile (sm_90a) — the Block.proj of the reference (U:229, 234).
//
// tc_gemm.cu treats a 3x3 conv as 9 independent K panels per 64 channels: the same activations are gathered, split to
// fp16 hi/lo and stored 9 times.  Here a CTA stages the (16+2) x (8+2) pixel halo of its 16x8-pixel output tile ONCE per
// 64-channel chunk (6.3x less gather/convert/store work) and the 9 taps are 9 shifted operand windows over that tile.
// With descriptor base_offset = 0 the 128-byte swizzle follows ABSOLUTE shared-memory address bits, so a K-major operand
// may start at any 128-byte row and use any row-multiple stride between its 8-row groups:
//     window(dy,dx): start = halo + ((dy+1)*10 + (dx+1))*128 B,  stride between 8-pixel rows (SBO) = 10*128 B.
// 8x8 images (the deepest level of a 64x64 latent) run in pair mode (tc_conv3_pair_kernel): a tile is two whole frames of one clip, each
// m64 half one frame with its own 10x10 halo, so only the second half's window offset differs.
// Everything else follows tc_gemm.cu: FP16x3 split precision, register accumulators drained into an RN fp32 tile in shared
// memory (every 9, 3 or 1 taps), row-per-thread epilogue with bias + GroupNorm partial statistics.
//
// Persistent warp-specialised CTA of whole warpgroups, each with its own register budget (setmaxnreg, see CCfg):
//   * warpgroups 0-1: A producers (gather + split + swizzled store of the halo tile), or one TMA thread;
//   * BN = 64: one MMA warpgroup and one epilogue warpgroup.  The MMA warpgroup drains tile t into staging tile t & 1, signals
//     the epilogue warpgroup through an mbarrier and goes on with tile t+1; before its first drain into a staging tile it waits
//     until the epilogue has released that tile.  The tensor cores keep working while the epilogue of the previous tile runs;
//   * BN = 128: two warpgroups, each issuing the MMAs of 64 columns and then running their epilogue from their own staging tile;
//   * last warpgroup: the weight loader (one thread; the other three warps exit).
// The taps of a chunk are expanded at compile time for each drain interval, so the only wgmma waits are wait_group 1 between
// taps (one tap's MMAs stay in flight while the next tap is issued) and wait_group 0 before a drain.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cstdlib>
#include <cstring>
#include <string>
#include <map>
#include <tuple>
#include "common.cuh"
#include "f16x3.cuh"
#include "gemm.cuh"
#include "tc_common.cuh"
#include "tc_gemm.cuh"

namespace dawn {
namespace {

using namespace tc;

constexpr int TH = 16, TW = 8;                 // output tile (pixels) -> M = 128 rows, row m = y*8 + x
constexpr int HH = TH + 2, HW = TW + 2;        // halo tile
constexpr int NPROD = 256;
// Pair mode (8 x 8 images): the 128-row tile is two whole frames of one clip, rows 0-63 frame a and rows 64-127 frame b (row
// 64 * fr + y*8 + x).  The halo stage holds two 10 x 10 halos: frame a from row 0, frame b from row PAIR_ROW_B = 104 rather than
// 100, so that frame b's TMA destination is 1024-byte aligned as the 128-byte swizzle requires; rows 100-103 are never read.
constexpr int PAIR_HH = 8 + 2;
constexpr int PAIR_ROW_B = 104;

// B stages: what fits in 227 KB next to the halo stages and two 128 x 64 fp32 staging tiles (34 KB each).
// BN = 64: one MMA warpgroup and one epilogue warpgroup; the staging tiles are a double buffer between them, so the epilogue
// of tile t runs while the MMAs of tile t+1 are issued.  BN = 128: two warpgroups, each issuing the MMAs of 64 columns and
// then running their epilogue from its own staging tile.
// Warpgroups: 0-1 A producers | MMA (| epilogue) | weight loader.  Registers per thread: every warp starts with the 96 that 640
// threads allow, and setmaxnreg.inc can only take what other warpgroups of the CTA released.  The producers keep 96, the loader
// gives 72 back and the MMA and epilogue warpgroups take them (5 x 96 = 480 at launch):
//   BN =  64: 2 x 96 + 24 + 136 + 128 = 480        BN = 128: 2 x 96 + 24 + 2 x 128 = 472
// Pair mode runs at BN = 64 with three weight stages: its 26 KB halos leave no room for a fourth (or for BN = 128).
template <int BN, bool PAIR = false>
struct CCfg {
  static_assert(!PAIR || BN == 64, "the pair-mode halos fit next to 64-column weight stages only");
  static constexpr int NWG = BN / 64;                          // MMA warpgroups (64 output columns each)
  static constexpr bool SPLIT_EPI = (BN == 64);                // separate epilogue warpgroup
  static constexpr int B_PANEL = BN * 128;                     // one (tap, chunk) weight panel, hi or lo
  static constexpr int FRAME_ROWS = PAIR ? PAIR_HH * HW : HH * HW;       // halo rows of one frame: 100 (pair) or 180
  static constexpr int HALO_ROWS = PAIR ? PAIR_ROW_B + FRAME_ROWS : FRAME_ROWS;   // rows spanned in the stage: 204 or 180
  static constexpr int A_HALO = (HALO_ROWS * 128 + 1023) / 1024 * 1024;  // 26 KB or 23 KB (keeps 1024-byte alignment)
  static constexpr int A_STAGES = 2;
  static constexpr int B_STAGES = PAIR ? 3 : (BN == 64) ? 4 : 2;
  static constexpr int A_BYTES = A_STAGES * 2 * A_HALO;        // hi + lo
  static constexpr int B_BYTES = B_STAGES * 2 * B_PANEL;
  static constexpr int ACC_STAGE = 2 * 128 * kStageLd * 4;
  static constexpr int SMEM_DYN = A_BYTES + B_BYTES + ACC_STAGE + 1024;
  // 227 KB per block, less under 1 KB of static barriers, GroupNorm and bias scratch:
  //   BN =  64:       94 208 (A) + 65 536 (B) + 69 632 (staging) + 1 024 (alignment) = 230 400
  //   BN = 128:       94 208     + 65 536     + 69 632           + 1 024             = 230 400
  //   BN = 64 pair:  106 496     + 49 152     + 69 632           + 1 024             = 226 304
  static_assert(SMEM_DYN + 1024 <= 232448, "shared memory");
  static constexpr int EPI_WARP = NPROD / 32 + 4 * NWG;        // first warp of the epilogue warpgroup (SPLIT_EPI)
  static constexpr int LOAD_WARP = EPI_WARP + (SPLIT_EPI ? 4 : 0);
  static constexpr int NTHREADS = 32 * LOAD_WARP + 128;        // the weight loader is a whole warpgroup (one thread works)
  static constexpr uint32_t REG_LAUNCH = (65536 / NTHREADS) & ~7u;   // what ptxas allots each thread at launch (__launch_bounds__)
  static constexpr uint32_t REG_LOAD = 24, REG_MMA = SPLIT_EPI ? 136 : 128, REG_EPI = 128;
  // setmaxnreg.dec may only lower a warp's count and setmaxnreg.inc only raise it
  static_assert(REG_LOAD < REG_LAUNCH && REG_MMA > REG_LAUNCH && REG_EPI > REG_LAUNCH, "register budgets");
  static_assert(2 * REG_LAUNCH + REG_LOAD + NWG * REG_MMA + (SPLIT_EPI ? REG_EPI : 0) <= NTHREADS / 128 * REG_LAUNCH, "CTA register pool");
};

// A-operand source: TMA = false: fp32 activations, gathered / split / swizzled by the 8 producer warps.  TMA = true: the activation exists as
// two dense fp16 planes (hi | lo, written by the producing kernel's epilogue) and ONE thread fetches the halo tile of a 64-channel chunk with
// two cp.async.bulk.tensor loads (4-D tiled map {C, W, H, F}, box {64, 10, 18, 1}, 128-byte swizzle, out-of-image rows zero-filled by the
// TMA unit): the smem image is byte-identical to what the producers write (row = hy * 10 + hx of 128 B, absolute-address swizzle).
// In pair mode the thread issues two loads per frame (box {64, 10, 10, 1}), frame b's landing at row PAIR_ROW_B.
// img_bn: column width of the weight image's n-tiles (tc_tile_n(N)); the pair kernel's 64-column tiles may be halves of them.
template <int BN, bool TMA, bool PAIR>
__device__ __forceinline__ void tc_conv3_body(const GemmParams& p, const float* __restrict__ Bimg, int tiles_y, int tiles_x, int tiles_n,
                                              int img_bn, const CUtensorMap& tm_hi, const CUtensorMap& tm_lo) {
  using C = CCfg<BN, PAIR>;
  constexpr int B_PANEL = C::B_PANEL, A_STAGES = C::A_STAGES, B_STAGES = C::B_STAGES, NWG = C::NWG;
  constexpr int A_HALO = C::A_HALO, FRAME_ROWS = C::FRAME_ROWS;
  constexpr bool SPLIT = C::SPLIT_EPI;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t a_full[A_STAGES], a_free[A_STAGES], b_full[B_STAGES], b_free[B_STAGES];
  __shared__ uint64_t st_full[2], st_free[2];           // SPLIT: staging tile b handed from the MMA warpgroup to the epilogue and back
  __shared__ float s_stat[NWG][16];
  __shared__ __align__(16) float s_bias[NWG][64];       // bias of this epilogue warpgroup's 64 columns (single n-tile: constant for the whole launch)

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);          // warp-uniform by construction
  uint8_t* smem = smem_align1024(smem_raw);
  uint8_t* smemA = smem;
  uint8_t* smemB = smem + C::A_BYTES;
  float* stage_base = reinterpret_cast<float*>(smemB + C::B_BYTES);   // two [128][kStageLd] fp32 staging tiles

  if (tid == 0) {
    // a_free / b_free: one arrive per MMA warp once its MMAs on the slot have completed; st_full / st_free: one arrive per thread
    for (int s = 0; s < A_STAGES; ++s) { mbar_init(&a_full[s], TMA ? 1 : NPROD); mbar_init(&a_free[s], 4 * NWG); }
    for (int s = 0; s < B_STAGES; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_free[s], 4 * NWG); }
    for (int s = 0; s < 2; ++s) { mbar_init(&st_full[s], 128); mbar_init(&st_free[s], 128); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int H = p.IH, W = p.IW;
  const int F = p.M / (H * W);
  const int NCH = p.Cin / 64;                                  // 64-channel chunks
  const int tiles_sp = tiles_y * tiles_x;
  // Tiles are visited clip by clip (image f * clips + b is the (f, b) frame): a CTA's consecutive tiles then stay in one clip, so the
  // deferred GroupNorm partial sums below are flushed every 8 tiles and not at every change of clip.
  const int fpc = F / p.clips;                                 // frames per clip
  const int ppc = (fpc + 1) / 2;                               // pair mode: tiles per clip; an odd clip ends in a one-frame tile
  const int total_tiles = (PAIR ? p.clips * ppc : F * tiles_sp) * tiles_n;   // n fastest: CTAs of one patch share its activations in L2
  // the tile's first image f, its position (y0, x0) and n-tile nt; nf: frames in the tile (pair mode: images f and f + clips)
  auto decode = [&](int tile, int& f, int& y0, int& x0, int& nt, int& nf) {
    nt = tile % tiles_n;
    const int sp = tile / tiles_n;
    if constexpr (PAIR) {
      const int clip = sp / ppc, fa = 2 * (sp - clip * ppc);
      f = fa * p.clips + clip;
      nf = fa + 1 < fpc ? 2 : 1;
      y0 = 0; x0 = 0;
    } else {
      const int seq = sp / tiles_sp;                           // clip-major image sequence number
      const int r = sp - seq * tiles_sp;
      f = p.clips == 1 ? seq : (seq % fpc) * p.clips + seq / fpc;
      nf = 1;
      y0 = (r / tiles_x) * TH; x0 = (r % tiles_x) * TW;
    }
  };

  if (warp < 8) {                                              // keeps the launch register budget
    if (TMA) {
      // ============================================================= TMA producer: one thread, two tensor loads per (tile, chunk)
      if (tid == 0) {
        const uint64_t mh = reinterpret_cast<uint64_t>(&tm_hi), ml = reinterpret_cast<uint64_t>(&tm_lo);
        uint32_t ait = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
          int f, y0, x0, nt, nf;
          decode(tile, f, y0, x0, nt, nf);
          for (int cc = 0; cc < NCH; ++cc, ++ait) {
            const int s = ait % A_STAGES;
            mbar_wait(&a_free[s], ((ait / A_STAGES) & 1) ^ 1);
            mbar_arrive_expect_tx(&a_full[s], nf * 2 * FRAME_ROWS * 128);
            const uint32_t bar = smem_u32(&a_full[s]);
            const int c0 = cc * 64, c1 = x0 - 1, c2 = y0 - 1;
            for (int fr = 0; fr < nf; ++fr) {                  // a one-frame pair tile leaves rows 64-127 unused (not stored)
              const uint32_t dst = smem_u32(smemA + s * 2 * A_HALO) + fr * PAIR_ROW_B * 128;
              const int c3 = f + fr * p.clips;
              asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                           ::"r"(dst), "l"(mh), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
              asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                           ::"r"(dst + A_HALO), "l"(ml), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
            }
          }
        }
      }
    } else {
      // ============================================================= producers: halo tile of one 64-channel chunk
      // Logical halo row l = r0 + 32 q (< 180, pair mode < 200) is row hl of frame fr's halo, stored at row fr * PAIR_ROW_B + hl.
      constexpr int NQ = (C::FRAME_ROWS * (PAIR ? 2 : 1) + 31) / 32;   // 6 row passes, 7 in pair mode
      const int c16 = tid & 7;
      const int r0 = (tid >> 3) & 31;                          // tid < 256
      uint32_t ait = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int f, y0, x0, nt, nf;
        decode(tile, f, y0, x0, nt, nf);
        const float* img = p.A + (size_t)f * H * W * p.lda;
        const float* img_b = PAIR ? img + (size_t)p.clips * H * W * p.lda : img;   // pair mode: frame b
        for (int cc = 0; cc < NCH; ++cc, ++ait) {
          const int s = ait % A_STAGES;
          const uint32_t round = ait / A_STAGES;
          auto load = [&](int q, float4& a, float4& b) {
            const int l = r0 + 32 * q;
            // frame of the row: known from q alone except in the pass that crosses row FRAME_ROWS
            const int fr = (!PAIR || 32 * q + 31 < FRAME_ROWS) ? 0 : (32 * q >= FRAME_ROWS) ? 1 : (l >= FRAME_ROWS ? 1 : 0);
            const int r = l - fr * FRAME_ROWS;
            const int hy = r / HW, hx = r - hy * HW;
            const int iy = y0 + hy - 1, ix = x0 + hx - 1;
            const bool ok = (r < FRAME_ROWS) && fr < nf && (iy >= 0) && (iy < H) && (ix >= 0) && (ix < W);
            if (ok) {
              const float* fimg = fr ? img_b : img;
              const float4* src = reinterpret_cast<const float4*>(fimg + (size_t)(iy * W + ix) * p.lda + cc * 64) + 2 * c16;
              a = __ldg(src);
              b = __ldg(src + 1);
            } else {
              a = make_float4(0.f, 0.f, 0.f, 0.f);
              b = make_float4(0.f, 0.f, 0.f, 0.f);
            }
          };
          uint8_t* a_hi = smemA + s * 2 * A_HALO;
          uint8_t* a_lo = a_hi + A_HALO;
          auto store = [&](int q, const float4& a, const float4& b) {
            const int lr = r0 + 32 * q;
            const int fr = (!PAIR || 32 * q + 31 < FRAME_ROWS) ? 0 : (32 * q >= FRAME_ROWS) ? 1 : (lr >= FRAME_ROWS ? 1 : 0);
            const int r = lr + fr * (PAIR_ROW_B - FRAME_ROWS);
            if (lr < FRAME_ROWS * (PAIR ? 2 : 1)) {
              uint32_t h[4], l[4];
              split_f16x2_rn(a.x, a.y, h[0], l[0]);
              split_f16x2_rn(a.z, a.w, h[1], l[1]);
              split_f16x2_rn(b.x, b.y, h[2], l[2]);
              split_f16x2_rn(b.z, b.w, h[3], l[3]);
              const uint32_t off = swz(r, c16);                // absolute-row swizzle (halo base is 1024-byte aligned)
              *reinterpret_cast<uint4*>(a_hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
              *reinterpret_cast<uint4*>(a_lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
            }
          };
          // six passes are fetched into registers before the wait for the stage; a seventh would spill at 96 registers, so the pair
          // mode's last pass (rows 192-199) is fetched after it
          constexpr int NPRE = NQ < 6 ? NQ : 6;
          float4 v[2 * NPRE];
#pragma unroll
          for (int q = 0; q < NPRE; ++q) load(q, v[2 * q], v[2 * q + 1]);
          mbar_wait(&a_free[s], (round & 1) ^ 1);
#pragma unroll
          for (int q = 0; q < NPRE; ++q) store(q, v[2 * q], v[2 * q + 1]);
#pragma unroll
          for (int q = NPRE; q < NQ; ++q) {
            float4 a, b;
            load(q, a, b);
            store(q, a, b);
          }
          mbar_arrive_relaxed(&a_full[s]);                     // proxy fence runs on the consumer side (see tc_gemm.cu)
        }
      }
    }
    return;
  }
  if (warp >= C::LOAD_WARP) {
    // =============================================================== weight loader: one (tap, chunk) panel pair per slot
    setmaxnreg_dec<C::REG_LOAD>();
    if (warp == C::LOAD_WARP && lane == 0) {
      uint32_t bit = 0;
      const int KC = 9 * NCH;                                  // panels per n-tile in the weight image: kc = tap*NCH + cc
      // pair mode: the kernel's n-tile is 64-column block nt % sub of image n-tile nt / sub, rows [64 (nt % sub), +64) of each panel
      const int sub = PAIR ? img_bn / BN : 1;
      const size_t ipanel = (size_t)sub * B_PANEL;             // one image panel, hi or lo
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int f, y0, x0, nt, nf;
        decode(tile, f, y0, x0, nt, nf);
        const uint8_t* src = reinterpret_cast<const uint8_t*>(Bimg) + (size_t)(nt / sub) * KC * (2 * ipanel) + (size_t)(nt % sub) * B_PANEL;
        for (int cc = 0; cc < NCH; ++cc)
          for (int tap = 0; tap < 9; ++tap, ++bit) {
            const int s = bit % B_STAGES;
            const uint32_t round = bit / B_STAGES;
            mbar_wait(&b_free[s], (round & 1) ^ 1);
            mbar_arrive_expect_tx(&b_full[s], 2 * B_PANEL);
            const uint8_t* panel = src + (size_t)(tap * NCH + cc) * (2 * ipanel);
            if (PAIR) {
              bulk_copy_g2s(smemB + s * 2 * B_PANEL, panel, B_PANEL, &b_full[s]);
              bulk_copy_g2s(smemB + s * 2 * B_PANEL + B_PANEL, panel + ipanel, B_PANEL, &b_full[s]);
            } else {
              bulk_copy_g2s(smemB + s * 2 * B_PANEL, panel, 2 * B_PANEL, &b_full[s]);
            }
          }
      }
    }
    return;
  }

  // ================================================================= MMA (two m64n64 per k-step: output rows 0-63 and 64-127 of the
  // warpgroup's 64 columns) and row-per-thread epilogue read back from the staged fp32 tile
  const int wg = SPLIT ? 0 : (warp - 8) >> 2;                  // 64-column block of this MMA / epilogue warpgroup
  const int ew = (warp - 8) & 3;
  const int etid = ew * 32 + lane;                             // thread in the warpgroup = its tile row in the epilogue
  const int bar_id = 2 + wg;
  constexpr uint32_t SBO_HALO = HW * 128;                      // 10 pixel rows of 128 B between 8-row groups
  // output rows 64-127 start 8 pixel rows of the halo further down, or (pair mode) at frame b's halo
  constexpr uint32_t H2 = PAIR ? PAIR_ROW_B * 128 : 8 * HW * 128;
  const int dt = (p.drain == 1 || p.drain == 3) ? p.drain : 9; // taps accumulated in registers before a drain

  // All MMAs of one tile into `stage`.  The nine taps of a chunk are expanded at compile time for a drain interval DT of 1, 3
  // or 9 taps, so the only waits are the wait_group 1 that keeps one tap's MMAs in flight and the wait_group 0 before a drain.
  // claim() runs once, before the tile's first drain writes the staging tile.
  auto mma_tile = [&](auto DTc, float* stage, uint32_t& ait, uint32_t& bit, auto&& claim) {
    constexpr int DT = decltype(DTc)::value;
    float d0[32], d1[32];
    bool first_drain = true;
    for (int cc = 0; cc < NCH; ++cc, ++ait) {
      const int sa = ait % A_STAGES;
      mbar_wait(&a_full[sa], (ait / A_STAGES) & 1);
      fence_proxy_async();
      const uint32_t a_hi = smem_u32(smemA + sa * 2 * A_HALO), a_lo = a_hi + A_HALO;
      static_for<0, 9>([&](auto TAPc) {
        constexpr int tap = decltype(TAPc)::value;
        constexpr bool group_first = tap % DT == 0, group_last = tap % DT == DT - 1;
        constexpr uint32_t woff = (uint32_t)(((tap / 3) * HW + tap % 3) * 128);   // window start: halo pixel (ky, kx)
        const int sb = bit % B_STAGES;
        const int sprev = (bit + B_STAGES - 1) % B_STAGES;     // previous tap's B stage, released once its MMAs completed
        mbar_wait(&b_full[sb], (bit / B_STAGES) & 1);
        const uint64_t ahi = make_desc(a_hi + woff, SBO_HALO), alo = make_desc(a_lo + woff, SBO_HALO);
        const uint64_t ahi2 = make_desc(a_hi + woff + H2, SBO_HALO), alo2 = make_desc(a_lo + woff + H2, SBO_HALO);
        const uint32_t sbaddr = smem_u32(smemB + sb * 2 * B_PANEL) + wg * 64 * 128;
        const uint64_t bhi = make_desc(sbaddr), blo = make_desc(sbaddr + B_PANEL);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint64_t o = (uint64_t)(j * 2);
          const uint32_t acc = (group_first && j == 0) ? 0u : 1u;
          wgmma_m64n64k16(d0, alo + o, bhi + o, acc);
          wgmma_m64n64k16(d1, alo2 + o, bhi + o, acc);
          wgmma_m64n64k16(d0, ahi + o, blo + o, 1u);
          wgmma_m64n64k16(d1, ahi2 + o, blo + o, 1u);
          wgmma_m64n64k16(d0, ahi + o, bhi + o, 1u);
          wgmma_m64n64k16(d1, ahi2 + o, bhi + o, 1u);
        }
        wgmma_commit();
        if constexpr (group_last) {
          wgmma_wait<0>();
          wgmma_fence_acc(d0); wgmma_fence_acc(d1);
          if (lane == 0) { if (!group_first) mbar_arrive(&b_free[sprev]); mbar_arrive(&b_free[sb]); }
          if (first_drain) claim();
          stage_fragment(stage, 0, d0, first_drain, etid);
          stage_fragment(stage, 64, d1, first_drain, etid);
          first_drain = false;
        } else {
          wgmma_wait<1>();
          wgmma_fence_acc(d0); wgmma_fence_acc(d1);
          if (lane == 0 && !group_first) mbar_arrive(&b_free[sprev]);
        }
        ++bit;
      });
      if (lane == 0) mbar_arrive(&a_free[sa]);                 // 9 % DT == 0: every MMA of the chunk has completed
    }
  };

  // GroupNorm partial sums (U:230).  Reducing them per tile (16 warp reductions, shared and global atomics, two barriers) costs more
  // than half of a 64 -> 64 tile.  With a single n-tile every epilogue thread owns the same
  // 64 columns for the whole persistent loop, so it keeps fp32 running sums per 8-column block and the warps reduce them (in fp64) only
  // every 8 tiles and at the end: at most 64 values per fp32 partial sum.
  const bool defer_stats = (p.stats != nullptr) && tiles_n == 1;
  // with one n-tile the 64 bias values never change: fetch them once instead of 16 L2 round trips per tile
  const bool bias_smem = (p.bias != nullptr) && tiles_n == 1;
  auto load_bias = [&]() {
    if (bias_smem) {
      if (etid < 64) s_bias[wg][etid] = __ldg(p.bias + wg * 64 + etid);
      asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
    }
  };
  // A tile covers one frame, or two of the same clip, so one clip (frame % clips): the running sums belong to the clip of the tiles they hold and are flushed
  // before a tile of another clip is added.
  auto flush_stats = [&](float (&gs)[8], float (&gss)[8], int clip) {
    const int n0f = wg * 64;                                      // tiles_n == 1: this thread's columns never change
    double* cs = p.stats + 16 * clip;
#pragma unroll
    for (int b8 = 0; b8 < 8; ++b8) {
      double s = (double)gs[b8], ss = (double)gss[b8];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); ss += __shfl_xor_sync(0xffffffffu, ss, o); }
      if (lane == 0) {
        const int grp = (n0f + b8 * 8) / p.cpg;
        atomicAdd(&cs[2 * grp], s);
        atomicAdd(&cs[2 * grp + 1], ss);
      }
      gs[b8] = 0.f; gss[b8] = 0.f;
    }
  };
  // epilogue of one tile: thread etid owns tile row etid; its warp's 32 staged rows serve as the store buffer once read back
  auto epilogue_tile = [&](int tile, float* stage, float (&gs)[8], float (&gss)[8], int& pending, int& pclip) {
    int f, y0, x0, nt, nf;
    decode(tile, f, y0, x0, nt, nf);
    const int clip = p.clips > 1 ? f % p.clips : 0;
    const int n0 = nt * BN + wg * 64;
    const int row_in_tile = etid;
    float* s_st = s_stat[wg];
    float* wbuf = stage + ew * 32 * kStageLd;
    float acc[64];
    {
      const float4* src = reinterpret_cast<const float4*>(stage + row_in_tile * kStageLd);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float4 v = src[i];
        acc[4 * i] = v.x; acc[4 * i + 1] = v.y; acc[4 * i + 2] = v.z; acc[4 * i + 3] = v.w;
      }
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] *= p.tc_scale;
    // pair mode: row 64 fr + y*8 + x of image f + fr * clips; the rows of a one-frame tile's missing frame are not stored or counted
    const int fr = PAIR ? row_in_tile >> 6 : 0;
    const int img = f + fr * p.clips;
    const int oy = y0 + ((row_in_tile >> 3) & (PAIR ? 7 : 15)), ox = x0 + (row_in_tile & 7);
    const bool rv = (oy < H) && (ox < W) && fr < nf;
    size_t opix = (size_t)img * H * W + (size_t)(rv ? oy * W + ox : 0);
    int ocol = n0;
    if (p.up2) {
      // transposed conv as one 3x3 conv with 4 x 64 output columns: column block = output parity class (py, px)
      const int cls = n0 >> 6, py = cls >> 1, px = cls & 1;
      opix = (size_t)img * 4 * H * W + (size_t)(rv ? (2 * oy + py) * 2 * W + 2 * ox + px : 0);
      ocol = n0 & 63;
    }
    if (bias_smem) {
      const float4* bp = reinterpret_cast<const float4*>(s_bias[wg]);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float4 b = bp[i];
        acc[4 * i] += b.x; acc[4 * i + 1] += b.y; acc[4 * i + 2] += b.z; acc[4 * i + 3] += b.w;
      }
    } else if (p.bias) {
      const float4* bp = reinterpret_cast<const float4*>(p.bias + n0);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float4 b = __ldg(bp + i);
        acc[4 * i] += b.x; acc[4 * i + 1] += b.y; acc[4 * i + 2] += b.z; acc[4 * i + 3] += b.w;
      }
    }
    store_rows_coalesced(wbuf, acc, p.Out, opix, p.ldo, ocol, rv, lane);
    if (defer_stats) {
      if (pending > 0 && clip != pclip) { flush_stats(gs, gss, pclip); pending = 0; }
      pclip = clip;
      if (rv) {
#pragma unroll
        for (int b8 = 0; b8 < 8; ++b8) {
          float s = 0.f, ss = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) { const float x = acc[b8 * 8 + i]; s += x; ss += x * x; }
          gs[b8] += s; gss[b8] += ss;
        }
      }
      if (++pending == 8) { flush_stats(gs, gss, clip); pending = 0; }
    } else if (p.stats != nullptr) {
      if (etid < 16) s_st[etid] = 0.f;
      asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
#pragma unroll
      for (int b8 = 0; b8 < 8; ++b8) {
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
        const int glo = n0 / p.cpg, ghi = (n0 + 63) / p.cpg;
        if (grp >= glo && grp <= ghi) atomicAdd(&p.stats[16 * clip + etid], (double)s_st[etid]);
      }
    }
  };
  // the MMA tile loop, expanded once per legal drain interval
  auto with_drain = [&](auto&& run) {
    if (dt == 1) run(std::integral_constant<int, 1>{});
    else if (dt == 3) run(std::integral_constant<int, 3>{});
    else run(std::integral_constant<int, 9>{});
  };

  if (SPLIT && warp >= C::EPI_WARP) {
    // =============================================================== epilogue warpgroup: tile t from staging tile t & 1
    setmaxnreg_inc<C::REG_EPI>();
    float gs[8], gss[8];
    int pending = 0, pclip = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { gs[i] = 0.f; gss[i] = 0.f; }
    load_bias();
    uint32_t lt = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++lt) {
      const int b = lt & 1;
      mbar_wait(&st_full[b], (lt >> 1) & 1);
      epilogue_tile(tile, stage_base + b * 128 * kStageLd, gs, gss, pending, pclip);
      mbar_arrive(&st_free[b]);                                // after the last read and the last store-buffer use of the tile
    }
    if (defer_stats && pending > 0) flush_stats(gs, gss, pclip);
  } else if (SPLIT) {
    // =============================================================== MMA warpgroup: drains tile t into staging tile t & 1, hands it
    // to the epilogue warpgroup and goes on with tile t+1
    setmaxnreg_inc<C::REG_MMA>();
    with_drain([&](auto DTc) {
      uint32_t ait = 0, bit = 0, lt = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++lt) {
        const int b = lt & 1;
        mma_tile(DTc, stage_base + b * 128 * kStageLd, ait, bit, [&]() { mbar_wait(&st_free[b], ((lt >> 1) & 1) ^ 1); });
        mbar_arrive(&st_full[b]);                              // this thread's drained fragments are in the tile
      }
    });
  } else {
    // =============================================================== BN = 128: each warpgroup runs the MMAs and then the epilogue
    // of its 64 columns
    setmaxnreg_inc<C::REG_MMA>();
    float gs[8], gss[8];
    int pending = 0, pclip = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { gs[i] = 0.f; gss[i] = 0.f; }
    load_bias();
    float* stage = stage_base + wg * 128 * kStageLd;
    uint32_t ait = 0, bit = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      with_drain([&](auto DTc) { mma_tile(DTc, stage, ait, bit, []() {}); });
      asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
      epilogue_tile(tile, stage, gs, gss, pending, pclip);
      asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");   // the staged tile is rewritten by the next tile's first drain
    }
    if (defer_stats && pending > 0) flush_stats(gs, gss, pclip);
  }
}

// 16 x 8-pixel tiles of one frame
template <int BN, bool TMA>
__global__ void __launch_bounds__(CCfg<BN>::NTHREADS, 1) tc_conv3_kernel(const GemmParams p, const float* __restrict__ Bimg,
                                                                          int tiles_y, int tiles_x, int tiles_n, int img_bn,
                                                                          const __grid_constant__ CUtensorMap tm_hi,
                                                                          const __grid_constant__ CUtensorMap tm_lo) {
  tc_conv3_body<BN, TMA, false>(p, Bimg, tiles_y, tiles_x, tiles_n, img_bn, tm_hi, tm_lo);
}

// pair mode: 8 x 8 images, two frames of one clip per tile, 64 output columns
template <bool TMA>
__global__ void __launch_bounds__(CCfg<64, true>::NTHREADS, 1) tc_conv3_pair_kernel(const GemmParams p, const float* __restrict__ Bimg,
                                                                                     int tiles_y, int tiles_x, int tiles_n, int img_bn,
                                                                                     const __grid_constant__ CUtensorMap tm_hi,
                                                                                     const __grid_constant__ CUtensorMap tm_lo) {
  tc_conv3_body<64, TMA, true>(p, Bimg, tiles_y, tiles_x, tiles_n, img_bn, tm_hi, tm_lo);
}

template <int BN, bool TMA, bool PAIR>
constexpr auto c3_kernel() {
  if constexpr (PAIR) return tc_conv3_pair_kernel<TMA>;
  else return tc_conv3_kernel<BN, TMA>;
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// box {64 channels, 10, box_h, 1}: box_h = 18 for a 16 x 8 tile's halo, 10 for one frame of a pair tile
int halo_tensor_map(const void* plane, int Cin, int W, int H, int F, int box_h, CUtensorMap* out) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    DAWN_CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q));
    if (q != cudaDriverEntryPointSuccess || !ptr) { set_last_error("cuTensorMapEncodeTiled is not available in this driver"); return -2; }
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  // one map per (plane, geometry): encoding costs microseconds but the activations of a handle live at fixed addresses
  static std::map<std::tuple<const void*, int, int, int, int, int>, CUtensorMap> cache;
  const auto key = std::make_tuple(plane, Cin, W, H, F, box_h);
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return 0; }
  const cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)F};
  const cuuint64_t strides[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)W * Cin * 2, (cuuint64_t)H * W * Cin * 2};
  const cuuint32_t box[4] = {64, (cuuint32_t)HW, (cuuint32_t)box_h, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  CUtensorMap m;
  const CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_UINT16, 4, const_cast<void*>(plane), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r)); return -2; }
  if (cache.size() > 4096) cache.clear();
  cache[key] = m;
  *out = m;
  return 0;
}

template <int BN, bool PAIR>
int launch_c3(const GemmParams& p, const float* Bimg, cudaStream_t st) {
  using C = CCfg<BN, PAIR>;
  static bool attr_set = false;
  static int num_sms = 0;
  if (!attr_set) {
    DAWN_CUDA_OK(cudaFuncSetAttribute(c3_kernel<BN, false, PAIR>(), cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_DYN));
    DAWN_CUDA_OK(cudaFuncSetAttribute(c3_kernel<BN, true, PAIR>(), cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_DYN));
    int dev = 0;
    DAWN_CUDA_OK(cudaGetDevice(&dev));
    DAWN_CUDA_OK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    attr_set = true;
  }
  const int tiles_y = PAIR ? 1 : p.IH / TH, tiles_x = PAIR ? 1 : p.IW / TW, tiles_n = p.N / BN;
  const int F = p.M / (p.IH * p.IW);
  const int seqs = PAIR ? p.clips * ((F / p.clips + 1) / 2) : F;   // pair mode: two frames of a clip per tile
  const int grid = std::min(seqs * tiles_y * tiles_x * tiles_n, num_sms);
  const int img_bn = tc_tile_n(p.N);
  if (p.A16h != nullptr && p.A16l != nullptr) {
    CUtensorMap mh, ml;
    const int box_h = PAIR ? PAIR_HH : HH;
    if (halo_tensor_map(p.A16h, p.Cin, p.IW, p.IH, F, box_h, &mh) != 0 || halo_tensor_map(p.A16l, p.Cin, p.IW, p.IH, F, box_h, &ml) != 0)
      return -2;
    c3_kernel<BN, true, PAIR>()<<<grid, C::NTHREADS, C::SMEM_DYN, st>>>(p, Bimg, tiles_y, tiles_x, tiles_n, img_bn, mh, ml);
  } else {
    CUtensorMap dummy;
    memset(&dummy, 0, sizeof(dummy));
    c3_kernel<BN, false, PAIR>()<<<grid, C::NTHREADS, C::SMEM_DYN, st>>>(p, Bimg, tiles_y, tiles_x, tiles_n, img_bn, dummy, dummy);
  }
  DAWN_LAUNCH_OK();
  return 0;
}

// 8 x 8 images run in pair mode (two frames per tile); other shapes in 16 x 8 tiles
bool pair_mode(const GemmParams& p) { return p.IH == 8 && p.IW == 8; }

}  // namespace

// 3x3, stride 1, same padding, static weights, spatial size a multiple of the 16x8 tile or exactly 8x8 (pair mode), 64-channel
// chunks, EPI_PLAIN without residual
bool tc_conv3_supported(const GemmParams& p, int epi) {
  if (epi != EPI_PLAIN || p.Res != nullptr || p.perm_in || p.perm_out) return false;
  if (p.ntaps != 9 || p.in_stride != 1 || p.out_stride != 1 || p.oy0 != 0 || p.ox0 != 0) return false;
  for (int t = 0; t < 9; ++t)                                  // the kernel's windows are the taps of a same-padded 3x3, in row-major order
    if (p.dy[t] != t / 3 - 1 || p.dx[t] != t % 3 - 1) return false;
  if (p.IH != p.OH || p.IW != p.OW || p.OHs != p.OH || p.OWs != p.OW) return false;
  if ((p.IH % TH != 0 || p.IW % TW != 0) && !pair_mode(p)) return false;
  if (p.Cin % 64 != 0 || p.N % 64 != 0 || p.K != 9 * p.Cin) return false;
  if (p.b_batch_stride != 0 || p.rows_per_batch != p.M) return false;
  if ((p.lda & 3) || (p.ldo & 3)) return false;
  if (p.stats && (p.cpg % 8 != 0)) return false;
  if (p.up2 && (p.stats != nullptr || p.N != 256)) return false;
  return true;
}

int launch_tc_conv3(const GemmParams& p, const float* Bimg, cudaStream_t st) {
  if (!tc_conv3_supported(p, EPI_PLAIN)) { set_last_error("launch_tc_conv3: unsupported geometry"); return -1; }
  if (pair_mode(p)) return launch_c3<64, true>(p, Bimg, st);
  if (tc_tile_n(p.N) == 128) return launch_c3<128, false>(p, Bimg, st);
  return launch_c3<64, false>(p, Bimg, st);
}

}  // namespace dawn
