// wgmma / TMA GEMM and implicit-GEMM 3x3 convolution for sm_90a.
//
// One persistent, warp-specialised kernel of three warpgroups: warpgroup 0 is the TMA producer (one elected thread of
// warp 0 issues the copies; the warpgroup gives most of its registers to the others with setmaxnreg), warpgroups 1 and 2
// are the consumers.  A tile is 128 (M) x BN (N); a ring stage holds its 128 x 64 A box and one BN x 64 weight box, so
// each weight tile is brought into shared memory once per 128 rows.  The consumers issue full-width wgmma.m64nBNk16 on
// the 128-byte-swizzled ring and keep their accumulators in registers; how they share the tiles is fixed by BN:
//  * ping-pong (BN <= 160): the CTA's tiles alternate between the two consumers; a consumer owns the whole 128 x BN tile
//    and issues two m64 MMAs per k16 step (A rows 0-63 and 64-127, the same weight descriptor), BN accumulators a
//    thread.  Two named barriers hand the tensor cores from one consumer to the other once its MMAs are issued, so one
//    consumer's epilogue runs under the other's main loop.
//  * cooperative (BN = 256): both consumers work on every tile, consumer g on rows 64 g .. 64 g + 63 (128 accumulators a
//    thread); a stage is free once all 8 consumer warps have read it.  Epilogues do not overlap MMAs.
// Tiles are (m_tile, n_tile), n fastest, round-robin over the persistent CTAs.  K advances 64 elements (one swizzle row
// of fp16) per ring stage; the producer fills the ring in the order the consumers take the tiles and runs up to STAGES
// k-blocks ahead, across tile boundaries.
// A 3x3 convolution is the same kernel with nine K segments: tap (dy,dx) loads the NHWC activation box shifted by
// (dy,dx) through a 4-D TMA descriptor and the out-of-bounds zero fill of TMA provides the padding; a channel concat
// is two descriptors walked back to back along K.
// Nearest up-sampling + 3x3 conv runs as one launch per output parity on the low-resolution input (pack_conv_subpixel).
// When the target size along an axis is odd (2n - 1, the up-sampler of a level whose size was odd on the way down),
// parity 0 keeps the three row taps apart: its third tap reads the input through a descriptor whose base sits one row
// (column) EARLIER, so coordinate y + 1 of that view is row y of the tensor and the last row falls off the end into the
// zero fill -- which is exactly the padding the up-sampled image has below row 2n - 2.  Only coordinates >= 1 of such a
// view are ever read.  Output pixels beyond the target extent (parity 1 on an odd axis) are never stored.
// A 3x3 conv with stride 2 and right / bottom padding (the VAE encoder's down-samplers) tiles the output pixels and reads
// its taps through four parity views of the input (GemmParamsS2), so no im2col is materialised.
//
// Epilogue (per consumer warp, 16 rows of each 64-row half, one half after the other): registers -> [folded LayerNorm:
// rstd * acc - rstd * mean * u] + bias (+ time-embedding / positional row vector) / GEGLU / quick-GELU / ReLU -> fp16 -> warp-private
// swizzled shared-memory transpose, 32 columns at a time -> (+ fp16 residual) -> coalesced 16-byte global stores.
// Tiny-N or unaligned outputs (conv_out, N = 4) keep a direct-store path with the same rounding order.
// The short-K linears (K <= 640, BN 128 / 160) and GEGLUs (K <= 640, BN 256; GemmParamsEpi) read no global memory in the
// epilogue: warp 1 of the producer warpgroup fetches each tile's bias / LayerNorm / row-vector / residual operands into
// one of two shared-memory slots while the tile's main loop runs (see EpiSlot).
//
// Replaces (reference call sites): InflatedConv3d 3x3 / 1x1 (models/animatediff_models/resnet.py:9-18), every
// nn.Linear / 1x1 conv of Transformer3DModel (attention.py:65-93,174-204) and the motion module
// (motion_module.py:113-136,202-218), GEGLU (diffusers FeedForward).
#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace vs {

namespace {

constexpr int BM = 128;                             // rows of a tile
constexpr int WG_M = 64;                            // rows of one wgmma.m64 (an accumulator half)
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;          // 16 KB
constexpr uint64_t A_HALF_DESC = (WG_M * BK * 2) >> 4;   // descriptor step from A rows 0..63 to rows 64..127 (8 KB)
constexpr int GEMM_THREADS = 384;                   // producer warpgroup + 2 consumer warpgroups
constexpr int SMEM_LIMIT = 227 * 1024;
constexpr int EPI_COLS = 32;                        // output columns per epilogue sub-tile (64 B of fp16)
constexpr int EPI_WARP_BYTES = 16 * 64;             // per consumer warp: [16 rows x 64 B] transpose staging
constexpr int EPI_BYTES = 8 * EPI_WARP_BYTES;
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 64 K registers
enum { EPI_F_GEGLU = 1, EPI_F_RES = 2, EPI_F_RV = 4, EPI_F_LN = 8, EPI_F_LNOUT = 16, EPI_F_QGELU = 32, EPI_F_RELU = 64 };   // compile-time epilogue features

struct GemmParams {
  CUtensorMap tmA, tmA2, tmB;
  int M, N;
  int num_kb;        // total K blocks
  int kb_per_tap;    // K blocks per tap (both concat sources)
  int kb_src1;       // of which from source 1
  int taps;
  int a_rank;        // 2 = plain rows, 4 = NHWC conv
  int nimg, H, W, TH, TW, TN, tiles_x, tiles_y;
  int tap_x0, tap_y0, tap_w;   // conv taps: dy in [tap_y0, tap_y0 + taps / tap_w), dx in [tap_x0, tap_x0 + tap_w)
  int osy, osx, ooy, oox, OH, OW;   // output pixel of input pixel (y, x): (y * osy + ooy, x * osx + oox) in an OH x OW image
  int tw_log, thw_log;   // log2(TW), log2(TH * TW): the conv tile dims are powers of two
  int m_tiles, n_tiles;
  const float* bias;
  const float* rowvec;
  int ldrv;
  int pix_per_batch;
  int rv_mod;        // row-vector index = (pix / pix_per_batch) % rv_mod when > 0 (per-frame vectors)
  const float2* ln_stats;   // folded LayerNorm: per-row (rstd, -mean * rstd)
  const float* ln_u;        // ... and per-column sum of the gamma-scaled weight row
  const float2* ln_parts;   // alternative to ln_stats: [ln_nparts][M] per-row partial (sum, sum of squares) written by the
  int ln_nparts;            // epilogue of the GEMM that PRODUCED this GEMM's A operand (ln_sums_out below)
  float ln_inv_c;           // 1 / (LayerNorm width)
  float2* ln_sums_out;      // EPI_F_LNOUT: [n_tiles][M] per-row (sum, sum of squares) of this tile's stored fp16 outputs
  const __half* residual;
  int ldr;
  __half* out;
  int ldc;
  int staged;        // 1 = smem-transposed coalesced epilogue; 0 = direct stores for tiny / unaligned N
  int stages;        // 0 = all, else limits the smem ring depth (pipeline-depth experiments)
};

// Sub-pixel conv to an odd-sized target (its own kernel instantiations, so every other launch keeps the parameter block
// and the code it had): output extent check and the shifted views of the third tap along an odd axis.
struct GemmParamsSub : GemmParams {
  CUtensorMap tmS[3];    // tmA viewed one row (0), one column (1), one row and one column (2) earlier
  int sub_short;         // bit 0 / 1: the third row / column tap of this parity reads through tmS
};

// 3x3 stride-2 conv of pad(x, (0, 1, 0, 1)) (diffusers Downsample2D(padding=0), the VAE encoder's down-samplers), its own
// instantiations for the same reason.  The input is read through four parity views of the NHWC tensor: view (py, px)
// starts at pixel (py, px) and has doubled pixel strides and dims (W / 2, H / 2), so its element (x', y') is input pixel
// (2 x' + px, 2 y' + py).  tmA is view (0, 0), tmP[k - 1] view k = 2 py + px.  Tap (dy, dx) in {0, 1, 2}^2 of output
// pixel (x, y) reads view (dy & 1, dx & 1) at (x + (dx >> 1), y + (dy >> 1)); at the last output column / row an offset
// of 1 lands on x' = W / 2 (y' = H / 2), outside the view, and the TMA zero fill is exactly the right / bottom padding.
struct GemmParamsS2 : GemmParams {
  CUtensorMap tmP[3];
};

// Short-K linears and GEGLUs (GemmParamsEpi): the producer warpgroup's second warp fetches each tile's epilogue operands
// into a shared-memory slot while the tile's main loop runs; the epilogue then reads shared memory only.  Two slots, each
// guarded by its own full / empty mbarrier pair; tile j of a CTA uses slot j % 2 (ping-pong: the slot of the consumer
// that takes the tile; cooperative GEGLU: both consumers read it, so the next tile's slot fills during this epilogue).
constexpr int LN_MAX_PARTS = 8;                     // LayerNorm partial-sum slices a slot holds
struct GemmParamsEpi : GemmParams {
  CUtensorMap tmR;   // residual [M, N] fp16: boxes of 32 columns x 128 rows, 64-byte swizzle (= the epilogue's sw64_off)
};

template <int BN, int EPI>
struct EpiSlot {
  static constexpr bool RES = (EPI & EPI_F_RES) != 0, LN = (EPI & EPI_F_LN) != 0, RV = (EPI & EPI_F_RV) != 0;
  static constexpr int RES_BYTES = RES ? BM * BN * 2 : 0;              // BN / 32 boxes of [128 rows x 64 B], first
  static constexpr int BIAS_OFF = RES_BYTES;                           // bias[n0, n0 + BN)
  static constexpr int U_OFF = BIAS_OFF + BN * 4;                      // LN: ln_u[n0, n0 + BN)
  static constexpr int RV_OFF = U_OFF + (LN ? BN * 4 : 0);             // RV: the (at most 2) row-vector rows of the tile
  static constexpr int LNR_OFF = RV_OFF + (RV ? 2 * BN * 4 : 0);       // LN: [parts][128 rows] float2 row statistics
  static constexpr int END = LNR_OFF + (LN ? LN_MAX_PARTS * BM * 8 : 0);
  // the residual's swizzle repeats every 512 B, so a slot that holds one starts 1024-aligned
  static constexpr int BYTES = RES ? (END + 1023) / 1024 * 1024 : (END + 127) / 128 * 128;
};

template <int BN, int SLOT_BYTES = 0>
struct Cfg {
  // Cooperative (both consumers on one 128 x BN tile, 64 rows each) for BN = 256: 128 accumulators a thread.  Ping-pong
  // (one consumer owns the whole tile: two m64 halves, BN accumulators a thread) for the narrower tiles.
  static constexpr bool COOP = BN > 160;
  static constexpr int HALVES = COOP ? 1 : 2;       // 64-row accumulator halves per consumer
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  // with epilogue slots the ring gets what the two slots leave (counted without the spare kilobyte of the others)
  static constexpr int STAGES_RAW = SLOT_BYTES ? (SMEM_LIMIT - 1024 - 256 - EPI_BYTES - 2 * SLOT_BYTES) / STAGE_BYTES
                                               : (SMEM_LIMIT - 2048 - EPI_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 12 ? 12 : STAGES_RAW;
  static constexpr int SMEM_BYTES =
      STAGES * STAGE_BYTES + EPI_BYTES + 2 * SLOT_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(B_STAGE_BYTES % 1024 == 0, "B stage must keep 1024-byte alignment for SWIZZLE_128B");
  static_assert(STAGES >= 3, "pipeline too shallow");
  static_assert(SMEM_BYTES <= SMEM_LIMIT, "shared memory");
  static_assert(BN % 32 == 0 && BN <= 256, "wgmma N");
};

__device__ __forceinline__ uint32_t sw64_off(int row, int chunk) {   // byte offset inside a [rows x 64 B] swizzled tile
  return (uint32_t)(row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4));
}

template <int BN, int EPI, typename Params>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tc_kernel(const __grid_constant__ Params p) {
  constexpr bool SUB = std::is_same<Params, GemmParamsSub>::value;
  constexpr bool S2 = std::is_same<Params, GemmParamsS2>::value;
  constexpr bool SLOT = std::is_same<Params, GemmParamsEpi>::value;   // epilogue operands through the slots
  using ES = EpiSlot<BN, EPI>;
  using C = Cfg<BN, SLOT ? ES::BYTES : 0>;
  static_assert(!SLOT || ((C::COOP == ((EPI & EPI_F_GEGLU) != 0)) && (EPI & EPI_F_QGELU) == 0), "epilogue slots: ping-pong linears and cooperative GEGLUs");
  constexpr bool GEGLU = (EPI & EPI_F_GEGLU) != 0, HAS_RES = (EPI & EPI_F_RES) != 0, HAS_RV = (EPI & EPI_F_RV) != 0;
  // LN: the A operand is the RAW input of a LayerNorm whose affine map is folded into the weights:
  //   LN(x) W^T = rstd (x W'^T) - rstd mean u + c,  W' = W * gamma, u[n] = sum_k W'[n,k], c = beta W^T + bias (the `bias`)
  constexpr bool LN = (EPI & EPI_F_LN) != 0;
  // LNOUT: this GEMM's output feeds a LayerNorm (folded into the NEXT GEMM): the row statistics of what is stored -- the
  // fp16-rounded values, after the residual add -- are accumulated here, in the shadow of the store path, and written as
  // one (sum, sum of squares) pair per (column tile, row).  Deterministic (no atomics); replaces a stand-alone statistics
  // pass that would re-read every such tensor from HBM.
  constexpr bool LNOUT = (EPI & EPI_F_LNOUT) != 0;
  constexpr bool QGELU = (EPI & EPI_F_QGELU) != 0;   // quick_gelu(acc + bias) (CLIP's MLP fc1)
  constexpr bool RELU = (EPI & EPI_F_RELU) != 0;     // relu(acc + bias) (the T2I-Adapter's 3x3 block1 convs)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t epi_base = smem_base + C::STAGES * C::STAGE_BYTES;
  const uint32_t slot_base = epi_base + EPI_BYTES;   // SLOT: consumer g's slot at slot_base + g * ES::BYTES
  const uint32_t bar_base = slot_base + (SLOT ? 2 * ES::BYTES : 0);
  // barrier layout: full[S], empty[S], SLOT: slot_full[2], slot_empty[2]
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };
  auto slot_full = [&](int g) { return bar_base + 8u * (2 * C::STAGES + g); };
  auto slot_empty = [&](int g) { return bar_base + 8u * (2 * C::STAGES + 2 + g); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int nst = (p.stages > 0 && p.stages < C::STAGES) ? p.stages : C::STAGES;   // ring depth (debug knob: "gemm_stages")
  // Tile order: tile t = (m_tile, n_tile) = (t / n_tiles, t % n_tiles), n fastest, round-robin over the CTAs (CTAs
  // running at the same time share the A row panel and a few weight tiles in L2).
  const int total_tiles = p.m_tiles * p.n_tiles;

  if (threadIdx.x == 0) {
    prefetch_tmap(&p.tmA);
    prefetch_tmap(&p.tmB);
    if (p.kb_src1 < p.kb_per_tap) prefetch_tmap(&p.tmA2);
    if constexpr (SUB) {
      if (p.sub_short & 1) prefetch_tmap(&p.tmS[0]);
      if (p.sub_short & 2) prefetch_tmap(&p.tmS[1]);
      if (p.sub_short == 3) prefetch_tmap(&p.tmS[2]);
    }
    if constexpr (S2) {
      for (int k = 0; k < 3; ++k) prefetch_tmap(&p.tmP[k]);
    }
    if constexpr (SLOT) {
      if (ES::RES) prefetch_tmap(&p.tmR);
      for (int g = 0; g < 2; ++g) {
        mbar_init(slot_full(g), 1);
        mbar_init(slot_empty(g), C::COOP ? 8 : 4);   // one arrival per warp of the consumer(s) that read the slot
      }
    }
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), C::COOP ? 8 : 4);  // one arrival per warp of the consumer(s) that read the stage
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_trigger();                                 // the next kernel may start its own set-up
  pdl_wait();                                    // everything above overlapped the previous kernel's tail; its data is visible now

  if (wg == 0) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if constexpr (SLOT) {
      if (warp == 1) {
        // ================================================================= epilogue-operand loader (one elected issuer)
        // Fills slot g = j % 2 for tile j of the CTA as soon as the epilogue of tile j - 2 has released it, so the
        // copies land during tile j's main loop (ping-pong: while consumer g waits for the tensor cores and runs it;
        // cooperative: during the epilogue of tile j - 1 and tile j's main loop).  In-place residual (residual == out): a tile's residual block is read here, by this
        // tile only, before its own epilogue writes it; no other tile writes those rows and columns.
        for (int t = blockIdx.x, j = 0; t < total_tiles; t += gridDim.x, ++j) {
          const int g = j & 1;
          mbar_wait(slot_empty(g), ((j >> 1) & 1) ^ 1);
          if (elect_one()) {
            const int m_tile = t / p.n_tiles, n_tile = t % p.n_tiles;
            const int n0 = n_tile * BN, m0 = m_tile * BM;
            const int ncols = p.N - n0 < BN ? p.N - n0 : BN;      // a multiple of 32 (staged epilogue)
            const int parts = p.ln_nparts > 0 ? p.ln_nparts : 1;
            const int rows = p.M - m0 < BM ? p.M - m0 : BM;       // even (the host requires an even M for LN)
            // row-vector rows of the tile's first and last row (the host allows at most two per tile)
            const int last = m0 + rows - 1;
            int rv0 = m0 / p.pix_per_batch, rv1 = last / p.pix_per_batch;
            const int nrv = rv1 != rv0 ? 2 : 1;
            if (p.rv_mod > 0) { rv0 %= p.rv_mod; rv1 %= p.rv_mod; }
            const uint32_t sb = slot_base + (uint32_t)g * ES::BYTES, fb = slot_full(g);
            uint32_t bytes = p.bias != nullptr ? ncols * 4u : 0u;
            if (ES::RES) bytes += (uint32_t)(ncols / EPI_COLS) * (BM * 64);
            if (ES::LN) bytes += ncols * 4u + (uint32_t)(parts * rows) * 8u;
            if (ES::RV) bytes += (uint32_t)nrv * ncols * 4u;
            mbar_expect_tx(fb, bytes);
            if (p.bias != nullptr) bulk_load(sb + ES::BIAS_OFF, p.bias + n0, ncols * 4u, fb);
            if constexpr (ES::RES) {
              for (int c = 0; c < ncols / EPI_COLS; ++c) tma_load_2d(sb + c * (BM * 64), &p.tmR, fb, n0 + c * EPI_COLS, m0);
            }
            if constexpr (ES::LN) {
              bulk_load(sb + ES::U_OFF, p.ln_u + n0, ncols * 4u, fb);
              // the tile's rows of each slice; slot rows past M keep stale values and are never stored
              const float2* src = p.ln_nparts > 0 ? p.ln_parts : p.ln_stats;
              for (int k = 0; k < parts; ++k)
                bulk_load(sb + ES::LNR_OFF + k * (BM * 8), src + (long long)k * p.M + m0, rows * 8u, fb);
            }
            if constexpr (ES::RV) {
              bulk_load(sb + ES::RV_OFF, p.rowvec + (long long)rv0 * p.ldrv + n0, ncols * 4u, fb);
              if (nrv == 2) bulk_load(sb + ES::RV_OFF + BN * 4, p.rowvec + (long long)rv1 * p.ldrv + n0, ncols * 4u, fb);
            }
          }
          __syncwarp();
        }
        return;
      }
    }
    if (warp != 0) return;
    // =================================================================== TMA producer (whole warp, one elected issuer)
    const int num_kb = p.num_kb, kb_per_tap = p.kb_per_tap, kb_src1 = p.kb_src1;
    const bool conv = p.a_rank == 4;
    const int tap_x0 = p.tap_x0, tap_x1 = p.tap_x0 + p.tap_w;
    bool short_y = false, short_x = false;
    if constexpr (SUB) { short_y = (p.sub_short & 1) != 0; short_x = (p.sub_short & 2) != 0; }
    uint32_t pr_s = 0, pr_ph = 0;              // ring stage / phase, carried across tiles
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      const int m_tile = t / p.n_tiles, n_tile = t % p.n_tiles;
      int x0 = 0, y0 = 0, i0 = 0;
      if (conv) {
        x0 = (m_tile % p.tiles_x) * p.TW;
        y0 = ((m_tile / p.tiles_x) % p.tiles_y) * p.TH;
        i0 = (m_tile / (p.tiles_x * p.tiles_y)) * p.TN;
      }
      const int n0 = n_tile * BN;
      const int m0 = m_tile * BM;
      int kcoord = 0;                          // K coordinate into the weight panel (kb * 64)
      int dy = p.tap_y0, dx = tap_x0;          // tap offsets, advanced like an odometer
      int r = 0;                               // k-block inside the tap
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(empty_bar(pr_s), pr_ph ^ 1);
        if (elect_one()) {
          const uint32_t fb = full_bar(pr_s);
          const uint32_t a_dst = smem_base + pr_s * C::STAGE_BYTES;
          const bool first = r < kb_src1;
          const CUtensorMap* tm = first ? &p.tmA : &p.tmA2;
          if constexpr (SUB) {
            const bool sy = short_y && dy == p.tap_y0 + 2, sx = short_x && dx == tap_x0 + 2;   // third tap of an odd axis
            if (sy || sx) tm = sy ? (sx ? &p.tmS[2] : &p.tmS[0]) : &p.tmS[1];
          }
          int ox = dx, oy = dy;                // tap offset in the coordinates of the view `tm`
          if constexpr (S2) {                  // parity view of the tap, offset 0 or 1 inside it
            const int par = ((dy & 1) << 1) | (dx & 1);
            if (par) tm = &p.tmP[par - 1];
            ox = dx >> 1; oy = dy >> 1;
          }
          const int c = (first ? r : r - kb_src1) * BK;
          mbar_expect_tx(fb, C::STAGE_BYTES);
          if (conv) tma_load_4d(a_dst, tm, fb, c, x0 + ox, y0 + oy, i0);
          else tma_load_2d(a_dst, tm, fb, c, m0);
          tma_load_2d(a_dst + A_STAGE_BYTES, &p.tmB, fb, kcoord, n0);
        }
        __syncwarp();
        kcoord += BK;
        if (++r == kb_per_tap) {               // next tap
          r = 0;
          if (++dx == tap_x1) { dx = tap_x0; ++dy; }
        }
        if (++pr_s == (uint32_t)nst) { pr_s = 0; pr_ph ^= 1; }
      }
    }
    return;
  }

  // ===================================================================== consumers: MMA + epilogue
  setmaxnreg_inc<CONSUMER_REGS>();
  const int g = wg - 1;                        // ping-pong: consumer g takes the CTA's tiles j with j % 2 == g;
                                               // cooperative: consumer g takes rows 64 g .. 64 g + 63 of every tile
  const int wq = warp & 3;                     // warp inside the warpgroup: rows 16 wq .. 16 wq + 15 of a 64-row half
  const int q = lane & 3;
  const int rbase = 16 * wq + (lane >> 2);     // this thread's rows of a half: rbase and rbase + 8
  const uint32_t stage_buf = epi_base + (uint32_t)(warp - 4) * EPI_WARP_BYTES;
  const bool has_bias = p.bias != nullptr;
  const bool staged = SLOT || p.staged != 0;
  const int num_kb = p.num_kb;
  // output pixel (row of the GEMM) of tile row `row`, -1 = outside the problem
  auto tile_pixel = [&](int m_tile, int row) -> int {
    if (p.a_rank == 4) {
      const int x0 = (m_tile % p.tiles_x) * p.TW;
      const int y0 = ((m_tile / p.tiles_x) % p.tiles_y) * p.TH;
      const int i0 = (m_tile / (p.tiles_x * p.tiles_y)) * p.TN;
      const int ti = row >> p.thw_log, rem = row & ((1 << p.thw_log) - 1);
      const int y = y0 + (rem >> p.tw_log), x = x0 + (rem & (p.TW - 1)), img = i0 + ti;
      if constexpr (SUB) {                     // parity 1 of an odd axis: its last row / column is not stored
        const int oy = y * p.osy + p.ooy, ox = x * p.osx + p.oox;
        return ((img < p.nimg) && (y < p.H) && (x < p.W) && (oy < p.OH) && (ox < p.OW)) ? (img * p.OH + oy) * p.OW + ox : -1;
      }
      return ((img < p.nimg) && (y < p.H) && (x < p.W)) ? (img * p.OH + y * p.osy + p.ooy) * p.OW + x * p.osx + p.oox : -1;
    }
    const int px = m_tile * BM + row;
    return px < p.M ? px : -1;
  };

  // Ping-pong tensor-core hand-off: consumer g waits on named barrier 1 + g before its main loop and, once all MMAs of
  // its tile are issued, arrives on the other consumer's barrier -- only when the CTA has a next tile, so every arrival
  // is waited for.  The cooperative consumers share every tile and need no hand-off.
  const int bar_mine = 1 + g, bar_other = 2 - g;
  float acc[C::HALVES][BN / 2];
  uint32_t s = 0, ph = 0;                      // ring stage / phase of the next tile's first k-block
  for (int t = blockIdx.x, j = 0; t < total_tiles; t += gridDim.x, ++j) {
    const int m_tile = t / p.n_tiles, n_tile = t % p.n_tiles;
    if (!C::COOP && (j & 1) != g) {            // the other consumer's tile: skip its k-blocks in the ring
      const uint32_t sn = s + (uint32_t)num_kb;
      ph ^= (sn / (uint32_t)nst) & 1u;
      s = sn % (uint32_t)nst;
      continue;
    }
    // ------------------------------------------------------------------ main loop
    if (!C::COOP && j > 0) named_bar_sync(bar_mine, 256);
    uint32_t prev = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(full_bar(s), ph);
      wgmma_fence();
      const uint32_t a_addr = smem_base + s * C::STAGE_BYTES;
      const uint64_t da = gmma_desc_sw128(a_addr) + (C::COOP ? (uint64_t)g * A_HALF_DESC : 0);
      const uint64_t db = gmma_desc_sw128(a_addr + A_STAGE_BYTES);
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
#pragma unroll
        for (int hh = 0; hh < C::HALVES; ++hh)  // both m64 halves read the same weight tile
          wgmma_ss<BN>(acc[hh], da + hh * A_HALF_DESC + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      if (kb > 0) {                            // the MMAs of the previous k-block have read their stage: release it
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(empty_bar(prev));
      }
      prev = s;
      if (++s == (uint32_t)nst) { s = 0; ph ^= 1; }
    }
    if (!C::COOP && t + (int)gridDim.x < total_tiles) named_bar_arrive(bar_other, 256);
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(empty_bar(prev));
    // SLOT: this tile's epilogue operands, read through a generic pointer into the slot (plain shared loads the compiler
    // may schedule freely; the slot is written only by the async proxy, ordered by the mbarrier waits and arrivals)
    const int js = j & 1;                       // this tile's slot (ping-pong: js == g)
    const uint8_t* slot = smem_raw + (slot_base + (uint32_t)js * ES::BYTES - smem_u32(smem_raw));
    if constexpr (SLOT) mbar_wait(slot_full(js), (uint32_t)(j >> 1) & 1u);

    // ------------------------------------------------------------------ epilogue, one 64-row half at a time
    const int n0 = n_tile * BN;
#pragma unroll
    for (int hh = 0; hh < C::HALVES; ++hh) {
      const int r0 = WG_M * (C::COOP ? g : hh) + rbase;   // tile rows of this thread: r0 and r0 + 8
      int pix[2];
      pix[0] = tile_pixel(m_tile, r0);
      pix[1] = tile_pixel(m_tile, r0 + 8);
      const float* rv[2] = {nullptr, nullptr};
      if (SLOT && HAS_RV) {                    // row h's row vector: the slot's first or second row
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int d = pix[h] >= 0 ? pix[h] / p.pix_per_batch - (m_tile * BM) / p.pix_per_batch : 0;
          rv[h] = reinterpret_cast<const float*>(slot + ES::RV_OFF) + d * BN;
        }
      } else if (HAS_RV || !staged) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (p.rowvec != nullptr && pix[h] >= 0) {
            int ri = pix[h] / p.pix_per_batch;
            if (p.rv_mod > 0) ri %= p.rv_mod;
            rv[h] = p.rowvec + (long long)ri * p.ldrv + n0;
          }
        }
      }
      if (staged) {
        constexpr int OC = GEGLU ? BN / 2 : BN;                            // output columns of a full tile
        const int oc0 = n_tile * OC;                                        // first output column of this tile
        const int nsub = (p.N - n0 < BN ? (GEGLU ? (p.N - n0) / 2 : p.N - n0) : OC) / EPI_COLS;
        float la[2] = {1.f, 1.f}, lb[2] = {0.f, 0.f};                      // folded LayerNorm: row scale and shift factor
        if (LN) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (pix[h] < 0) continue;
            const float2* lnr = reinterpret_cast<const float2*>(slot + ES::LNR_OFF) + r0 + 8 * h;   // SLOT: [parts][128]
            if (p.ln_nparts > 0) {            // statistics from the producer GEMM's per-column-tile partial sums
              float S = 0.f, Q = 0.f;
              for (int k = 0; k < p.ln_nparts; ++k) {
                const float2 v = SLOT ? lnr[k * BM] : __ldg(p.ln_parts + (long long)k * p.M + pix[h]);
                S += v.x; Q += v.y;
              }
              const float mean = S * p.ln_inv_c;
              la[h] = rsqrtf(fmaxf(fmaf(-mean, mean, Q * p.ln_inv_c), 0.f) + 1e-5f);
              lb[h] = -mean * la[h];
            } else {
              const float2 st2 = SLOT ? lnr[0] : __ldg(p.ln_stats + pix[h]);
              la[h] = st2.x; lb[h] = st2.y;
            }
          }
        }
        float rs[2] = {0.f, 0.f}, rq[2] = {0.f, 0.f};   // LNOUT: sums of the 2 rows this lane stores
        // After the transpose this lane stores 16-byte chunk q of its own two rows (rbase, rbase + 8).
        __half* orow[2];
        const __half* rrow[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long px = pix[h] >= 0 ? pix[h] : 0;     // rows outside the problem: loads harmless, stores predicated
          orow[h] = p.out + px * p.ldc + oc0 + q * 8;
          rrow[h] = HAS_RES ? p.residual + px * p.ldr + oc0 + q * 8 : nullptr;
        }
#pragma unroll
        for (int sb = 0; sb < OC / EPI_COLS; ++sb) {
          if (sb >= nsub) break;                  // warp-uniform
          uint4 rr[2];
          if (SLOT && HAS_RES) {                  // box sb of the slot, 64-byte swizzled as the staging buffer
#pragma unroll
            for (int h = 0; h < 2; ++h)
              rr[h] = *reinterpret_cast<const uint4*>(slot + sb * (BM * 64) + sw64_off(r0 + 8 * h, q));
          } else if (HAS_RES) {
#pragma unroll
            for (int h = 0; h < 2; ++h) rr[h] = __ldg(reinterpret_cast<const uint4*>(rrow[h] + sb * EPI_COLS));
          }
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * sb + jj;            // n8 block of the (output) tile
            const int c = 8 * j + 2 * q;          // column inside the tile (value column for GEGLU)
            float2 b = make_float2(0.f, 0.f), u = make_float2(0.f, 0.f);
            if constexpr (SLOT) {
              if (has_bias) b = *reinterpret_cast<const float2*>(slot + ES::BIAS_OFF + 4 * c);
              if (LN) u = *reinterpret_cast<const float2*>(slot + ES::U_OFF + 4 * c);
            } else {
              if (has_bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + c));
              if (LN) u = __ldg(reinterpret_cast<const float2*>(p.ln_u + n0 + c));
            }
            float2 bg = make_float2(0.f, 0.f), ug = make_float2(0.f, 0.f);
            if (GEGLU) {                          // gate columns are BN / 2 further on, in the same thread's registers
              if constexpr (SLOT) {
                bg = *reinterpret_cast<const float2*>(slot + ES::BIAS_OFF + 4 * (BN / 2 + c));
                if (LN) ug = *reinterpret_cast<const float2*>(slot + ES::U_OFF + 4 * (BN / 2 + c));
              } else {
                bg = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + BN / 2 + c));
                if (LN) ug = __ldg(reinterpret_cast<const float2*>(p.ln_u + n0 + BN / 2 + c));
              }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float f0 = acc[hh][4 * j + 2 * h], f1 = acc[hh][4 * j + 2 * h + 1];
              if (GEGLU) {
                float g0 = acc[hh][4 * (j + BN / 16) + 2 * h], g1 = acc[hh][4 * (j + BN / 16) + 2 * h + 1];
                float bv0 = b.x, bv1 = b.y, bg0 = bg.x, bg1 = bg.y;
                if (LN) {                         // value / gate pre-activations of the folded LayerNorm
                  bv0 = fmaf(lb[h], u.x, bv0); bv1 = fmaf(lb[h], u.y, bv1);
                  bg0 = fmaf(lb[h], ug.x, bg0); bg1 = fmaf(lb[h], ug.y, bg1);
                  f0 *= la[h]; f1 *= la[h]; g0 *= la[h]; g1 *= la[h];
                }
                f0 = (f0 + bv0) * gelu_sig(g0 + bg0);
                f1 = (f1 + bv1) * gelu_sig(g1 + bg1);
              } else {
                if (LN) {                         // rstd * acc + (-mean rstd) * u + c in two FMAs per element
                  f0 = fmaf(la[h], f0, fmaf(lb[h], u.x, b.x));
                  f1 = fmaf(la[h], f1, fmaf(lb[h], u.y, b.y));
                } else if (has_bias) {
                  f0 += b.x; f1 += b.y;
                }
                if (HAS_RV && rv[h] != nullptr) {
                  const float2 r2 = SLOT ? *reinterpret_cast<const float2*>(rv[h] + c)
                                         : __ldg(reinterpret_cast<const float2*>(rv[h] + c));
                  f0 += r2.x; f1 += r2.y;
                }
                if constexpr (QGELU) {
                  f0 = quick_gelu_f(f0); f1 = quick_gelu_f(f1);
                }
                if constexpr (RELU) {
                  f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f);
                }
              }
              const __half2 hv = __floats2half2_rn(f0, f1);
              const uint32_t sa = stage_buf + sw64_off((lane >> 2) + 8 * h, jj) + 4 * q;
              if constexpr (SLOT)                 // no global loads to order against; the volatile asms keep their order
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sa), "r"(*reinterpret_cast<const uint32_t*>(&hv)));
              else
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sa), "r"(*reinterpret_cast<const uint32_t*>(&hv)) : "memory");
            }
          }
          __syncwarp();
#pragma unroll
          for (int h = 0; h < 2; ++h) {           // 8 rows x 64 contiguous bytes per store instruction
            uint4 o;
            asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w)
                         : "r"(stage_buf + sw64_off((lane >> 2) + 8 * h, q)));
            if (HAS_RES) {                        // fp16 add: the rounding order of the reference's `linear(x) + residual`
              __half2* oh = reinterpret_cast<__half2*>(&o);
              const __half2* rh = reinterpret_cast<const __half2*>(&rr[h]);
#pragma unroll
              for (int t = 0; t < 4; ++t) oh[t] = __hadd2(oh[t], rh[t]);
            }
            if (pix[h] >= 0) *reinterpret_cast<uint4*>(orow[h] + sb * EPI_COLS) = o;
            if (LNOUT) {
              const __half2* oh = reinterpret_cast<const __half2*>(&o);
              const float2 a = __half22float2(oh[0]), b2 = __half22float2(oh[1]), c2 = __half22float2(oh[2]), d2 = __half22float2(oh[3]);
              rs[h] += ((a.x + a.y) + (b2.x + b2.y)) + ((c2.x + c2.y) + (d2.x + d2.y));
              float q0 = fmaf(a.x, a.x, a.y * a.y), q1 = fmaf(b2.x, b2.x, b2.y * b2.y);
              float q2 = fmaf(c2.x, c2.x, c2.y * c2.y), q3 = fmaf(d2.x, d2.x, d2.y * d2.y);
              rq[h] += (q0 + q1) + (q2 + q3);
            }
          }
          __syncwarp();                           // staging buffer free for the next sub-tile
        }
        if (LNOUT) {                              // the 4 column chunks of a row sit in 4 adjacent lanes
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            rs[h] += __shfl_xor_sync(0xffffffffu, rs[h], 1); rq[h] += __shfl_xor_sync(0xffffffffu, rq[h], 1);
            rs[h] += __shfl_xor_sync(0xffffffffu, rs[h], 2); rq[h] += __shfl_xor_sync(0xffffffffu, rq[h], 2);
            if (q == 0 && pix[h] >= 0) p.ln_sums_out[(long long)n_tile * p.M + pix[h]] = make_float2(rs[h], rq[h]);
          }
        }
      } else {
        // -------------------------------------------------------------- direct stores (tiny / unaligned N, linear only)
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int h = e >> 1, c = 8 * j + 2 * q + (e & 1), n = n0 + c;
            if (n < p.N && pix[h] >= 0) {
              float f = acc[hh][4 * j + e];
              if (has_bias) f += p.bias[n];
              if (rv[h]) f += rv[h][c];
              __half y = __float2half_rn(f);
              if (p.residual) y = __hadd(y, p.residual[(long long)pix[h] * p.ldr + n]);   // fp16 add, as the staged path
              p.out[(long long)pix[h] * p.ldc + n] = y;
            }
          }
        }
      }
    }
    if constexpr (SLOT) {                      // every slot value this warp read has gone into a store: release the slot
      __syncwarp();
      if (lane == 0) mbar_arrive(slot_empty(js));
    }
  }
}

struct ConvTile { int tw, th, tn; };

ConvTile pick_conv_tile(int nimg, int H, int W) {   // BM pixels as a TW x TH x TN box with the least padding
  ConvTile best{1, 1, BM};
  long long best_cost = -1;
  for (int tw = 1; tw <= BM; tw *= 2) {
    for (int th = 1; tw * th <= BM; th *= 2) {
      const int tn = BM / (tw * th);
      if (tw > 256 || th > 256 || tn > 256) continue;
      const long long cost = (long long)((W + tw - 1) / tw) * tw * ((H + th - 1) / th) * th * ((nimg + tn - 1) / tn) * tn;
      if (best_cost < 0 || cost < best_cost || (cost == best_cost && tw > best.tw)) {
        best_cost = cost;
        best = ConvTile{tw, th, tn};
      }
    }
  }
  return best;
}

template <int BN, int EPI, typename Params = GemmParams>
int launch(cudaStream_t st, const Params& p) {
  using C = Cfg<BN, std::is_same<Params, GemmParamsEpi>::value ? EpiSlot<BN, EPI>::BYTES : 0>;
  static bool configured = false;
  if (!configured) {
    VS_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, EPI, Params>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    configured = true;
  }
  const int total = p.m_tiles * p.n_tiles;
  int ctas = num_sms();
  const int cap = get_option("gemm_ctas");              // > 0: fewer CTAs, each walking more tiles (another tile schedule)
  if (cap > 0 && cap < ctas) ctas = cap;
  return launch_pdl(gemm_tc_kernel<BN, EPI, Params>, dim3(total < ctas ? total : ctas), dim3(GEMM_THREADS), C::SMEM_BYTES, st, 1, p);
}

template <int BN>
int launch_linear(cudaStream_t st, const GemmParams& p) {
  const int epi = (p.residual ? EPI_F_RES : 0) | (p.rowvec ? EPI_F_RV : 0) | ((p.ln_stats || p.ln_parts) ? EPI_F_LN : 0) |
                  (p.ln_sums_out ? EPI_F_LNOUT : 0);
  switch (epi) {
    case EPI_F_LNOUT: return launch<BN, EPI_F_LNOUT>(st, p);
    case EPI_F_LNOUT | EPI_F_RES: return launch<BN, EPI_F_LNOUT | EPI_F_RES>(st, p);
    case EPI_F_LN: return launch<BN, EPI_F_LN>(st, p);
    case EPI_F_LN | EPI_F_RV: return launch<BN, EPI_F_LN | EPI_F_RV>(st, p);
    case 0: return launch<BN, 0>(st, p);
    case EPI_F_RES: return launch<BN, EPI_F_RES>(st, p);
    case EPI_F_RV: return launch<BN, EPI_F_RV>(st, p);
    case EPI_F_RES | EPI_F_RV: return launch<BN, EPI_F_RES | EPI_F_RV>(st, p);
    default: set_error("gemm_tc: unsupported epilogue combination 0x%x", epi); return 2;
  }
}

// The epilogue-slot launches (GemmParamsEpi); -1 = this launch keeps the parameter block without slots.
// K <= 640 (10 k-blocks); the staged epilogue of a plain linear on a ping-pong tile with one of the transformer's
// epilogue combinations, or of a GEGLU (BN 256, cooperative); operands the bulk copies can fetch: 16-byte aligned
// LayerNorm rows (an even M, so every slice and every tile's rows start 16-byte aligned and span a multiple of 16 bytes)
// of at most LN_MAX_PARTS slices, and at most two row-vector rows per 128-row tile.
template <int BN>
int launch_linear_slot(cudaStream_t st, const GemmParams& p, const GemmArgs& a) {
  const bool geglu = a.mode == EPI_GEGLU;
  if (get_option("gemm_epi_slot") == 0 || a.taps != 1 || (a.mode != EPI_LINEAR && !geglu) || !p.staged || p.num_kb > 10)
    return -1;
  const int epi = (p.residual ? EPI_F_RES : 0) | (p.rowvec ? EPI_F_RV : 0) | ((p.ln_stats || p.ln_parts) ? EPI_F_LN : 0) |
                  (p.ln_sums_out ? EPI_F_LNOUT : 0) | (geglu ? EPI_F_GEGLU : 0);
  if (geglu ? (BN != 256 || (epi & ~EPI_F_LN) != EPI_F_GEGLU)
            : (BN == 256 || (epi != EPI_F_RES && epi != EPI_F_LNOUT && epi != (EPI_F_LNOUT | EPI_F_RES) &&
                             epi != EPI_F_LN && epi != (EPI_F_LN | EPI_F_RV))))
    return -1;
  GemmParamsEpi pe;
  memset(&pe, 0, sizeof(pe));
  static_cast<GemmParams&>(pe) = p;
  if (p.rowvec && !(p.pix_per_batch >= BM || p.pix_per_batch == BM / 2)) return -1;
  if (epi & EPI_F_LN) {
    const void* rows = p.ln_parts ? static_cast<const void*>(p.ln_parts) : static_cast<const void*>(p.ln_stats);
    const int parts = p.ln_parts ? p.ln_nparts : 1;
    if (parts > LN_MAX_PARTS || (reinterpret_cast<uintptr_t>(rows) & 15) != 0 || (p.M & 1) != 0) return -1;
  }
  if (epi & EPI_F_RES) {
    const uint64_t dims[2] = {(uint64_t)p.N, (uint64_t)p.M};
    const uint64_t str[1] = {(uint64_t)p.ldr * 2};
    const uint32_t box[2] = {EPI_COLS, BM};
    if (make_tmap_f16(&pe.tmR, p.residual, 2, dims, str, box, 2)) return 3;
  }
  if constexpr (BN == 256) {
    return epi == EPI_F_GEGLU ? launch<BN, EPI_F_GEGLU>(st, pe) : launch<BN, EPI_F_GEGLU | EPI_F_LN>(st, pe);
  } else {
    switch (epi) {
      case EPI_F_RES: return launch<BN, EPI_F_RES>(st, pe);
      case EPI_F_LNOUT: return launch<BN, EPI_F_LNOUT>(st, pe);
      case EPI_F_LNOUT | EPI_F_RES: return launch<BN, EPI_F_LNOUT | EPI_F_RES>(st, pe);
      case EPI_F_LN: return launch<BN, EPI_F_LN>(st, pe);
      default: return launch<BN, EPI_F_LN | EPI_F_RV>(st, pe);
    }
  }
}

// BLOCK_N by a two-term model: waves of 128 x BN tiles over the persistent grid x operand bytes per k-block of one tile
// (16 KB of A + BN * 128 B of B; wider tiles need fewer bytes per flop).  Ties go to the wider tile only for long K,
// where the main loop -- not the epilogue -- dominates.  Never below 128 for N > 64 (ops.max_column_tiles relies on it).
int pick_bn(int m_tiles, int N, int num_kb) {
  if (N <= 64) return 64;
  int best = 128;
  long long best_cost = -1;
  const int cand[3] = {128, 160, 256};
  for (int i = 0; i < 3; ++i) {
    const int bn = cand[i];
    if (bn != 128 && N % bn != 0) continue;
    const long long tiles = (long long)m_tiles * ((N + bn - 1) / bn);
    const long long waves = (tiles + num_sms() - 1) / num_sms();
    const long long cost = waves * (16 + bn / 8);           // KB per k-block: 16 (A) + bn * 128 B (B)
    if (best_cost < 0 || cost < best_cost || (cost == best_cost && num_kb >= 40)) {
      best_cost = cost;
      best = bn;
    }
  }
  return best;
}

int ilog2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }

}  // namespace

// Column tiles the kernel will use for this problem (= number of LayerNorm partial-sum slices a producer writes).
int gemm_n_tiles(const GemmArgs& a) {
  if (a.taps != 1) return 0;
  int bn = a.force_bn;
  if (a.mode == EPI_GEGLU) bn = 2 * kGegluGranule;
  else if (bn == 0) bn = pick_bn((a.M + BM - 1) / BM, a.N, (a.K1 + BK - 1) / BK + a.K2 / BK);
  return (a.N + bn - 1) / bn;
}

int gemm_tc(cudaStream_t st, const GemmArgs& a) {
  VS_REQUIRE(a.A && a.Bw && a.out, "gemm_tc: null pointer");
  VS_REQUIRE(a.taps == 1 || a.taps == 9 || a.taps == 4, "gemm_tc: taps must be 1, 9 (3x3) or 4 (sub-pixel)");
  VS_REQUIRE(a.K1 % 8 == 0 && a.K2 % 8 == 0, "gemm_tc: K must be a multiple of 8 (TMA 16-byte strides)");
  VS_REQUIRE((long long)a.M * (a.ldc > a.ldr ? a.ldc : a.ldr) < (1LL << 40) && a.M < (1 << 30), "gemm_tc: M too large");
  const bool two = a.A2 != nullptr && a.K2 > 0;
  if (two || a.taps != 1) VS_REQUIRE(a.K1 % BK == 0 && a.K2 % BK == 0, "gemm_tc: concat/conv sources need C %% 64 == 0 (got %d,%d)", a.K1, a.K2);
  GemmParamsSub ps;                            // the GemmParams part is what every launch but an odd-sized sub-pixel one takes
  memset(&ps, 0, sizeof(ps));
  GemmParams& p = ps;
  GemmParamsS2 p2;                             // stride 2: the parity views; its GemmParams part is copied from p at launch
  memset(&p2, 0, sizeof(p2));
  // sub-pixel conv: output extent OH x OW (2H or 2H - 1 rows, 2W or 2W - 1 columns); parity 0 of an odd axis has 3 taps
  const bool sub = a.taps == 4;
  const int OH = sub && a.OH > 0 ? a.OH : 2 * a.H, OW = sub && a.OW > 0 ? a.OW : 2 * a.W;
  const int sub_ty = sub && a.sub_py == 0 && (OH & 1) ? 3 : 2, sub_tx = sub && a.sub_px == 0 && (OW & 1) ? 3 : 2;
  if (sub) VS_REQUIRE((OH == 2 * a.H || OH == 2 * a.H - 1) && (OW == 2 * a.W || OW == 2 * a.W - 1),
                      "gemm_tc: sub-pixel output %dx%d is not 2x (or 2x - 1) of the %dx%d input", OH, OW, a.H, a.W);
  const int ntaps = sub ? sub_ty * sub_tx : a.taps;
  const int Ktap = a.K1 + (two ? a.K2 : 0);
  const int Ktot = Ktap * ntaps;
  p.taps = ntaps;
  p.kb_src1 = (a.K1 + BK - 1) / BK;
  p.kb_per_tap = p.kb_src1 + (two ? a.K2 / BK : 0);
  p.num_kb = p.kb_per_tap * ntaps;
  p.M = a.M;
  p.N = a.N;
  p.bias = a.bias;
  p.rowvec = a.rowvec;
  p.ldrv = a.ldrv > 0 ? a.ldrv : a.N;
  p.pix_per_batch = a.pix_per_batch > 0 ? a.pix_per_batch : 1;
  p.rv_mod = a.rv_mod;
  p.ln_stats = reinterpret_cast<const float2*>(a.ln_stats);
  p.ln_u = a.ln_u;
  p.ln_parts = reinterpret_cast<const float2*>(a.ln_parts);
  p.ln_nparts = a.ln_parts ? a.ln_nparts : 0;
  p.ln_inv_c = 1.f / (float)(a.K1 + a.K2);
  p.ln_sums_out = reinterpret_cast<float2*>(a.ln_sums_out);
  if (a.ln_parts) VS_REQUIRE(a.ln_stats == nullptr && a.ln_nparts >= 1 && a.ln_nparts <= 16 && a.taps == 1, "gemm_tc: bad LayerNorm partial-sum input");
  if (a.ln_stats || a.ln_parts) VS_REQUIRE(a.ln_u != nullptr && a.bias != nullptr && a.residual == nullptr, "gemm_tc: folded LayerNorm needs u and c vectors and no residual");
  if (a.ln_sums_out) VS_REQUIRE(a.taps == 1 && a.mode == EPI_LINEAR && a.rowvec == nullptr && !a.ln_stats && !a.ln_parts,
                                "gemm_tc: row statistics output is implemented for plain linear layers (+ bias / residual)");
  p.residual = a.residual;
  p.ldr = a.ldr;
  p.out = a.out;
  p.ldc = a.ldc;
  p.stages = get_option("gemm_stages");

  // stride 2 (GemmParamsS2): the tiles walk the (H / 2) x (W / 2) output pixels; every other conv tiles its input grid
  const bool s2 = a.stride2 != 0;
  if (s2) VS_REQUIRE(a.taps == 9 && !two && a.H % 2 == 0 && a.W % 2 == 0 && a.lda1 == a.K1 && a.mode == EPI_LINEAR &&
                     !a.ln_stats && !a.ln_parts,
                     "gemm_tc: the stride-2 conv takes one dense NHWC source of even height and width (got %dx%d)", a.H, a.W);
  const int GH = s2 ? a.H / 2 : a.H, GW = s2 ? a.W / 2 : a.W;
  if (a.taps != 1) {
    VS_REQUIRE(a.nimg > 0 && GH > 0 && GW > 0 && a.M == a.nimg * GH * GW, "gemm_tc: bad conv geometry");
    p.a_rank = 4;
    // 3x3: taps (-1..1)^2.  Sub-pixel (one output parity (py, px) of nearest up-sampling + 3x3, see pack_conv_subpixel):
    // taps {py - 1, py} x {px - 1, px}, output pixel (2 y + py, 2 x + px) of the OH x OW image; on an odd axis parity 0
    // has the taps {-1, 0, 0'} with 0' read through the shifted view (tmS).  Stride 2: taps (0..2)^2 on the parity views.
    if (s2) { p.tap_x0 = p.tap_y0 = 0; p.tap_w = 3; p.osy = p.osx = 1; p.ooy = p.oox = 0; p.OH = GH; p.OW = GW; }
    else if (a.taps == 9) { p.tap_x0 = p.tap_y0 = -1; p.tap_w = 3; p.osy = p.osx = 1; p.ooy = p.oox = 0; p.OH = a.H; p.OW = a.W; }
    else {
      VS_REQUIRE((a.sub_py | 1) == 1 && (a.sub_px | 1) == 1, "gemm_tc: sub-pixel parity must be 0 or 1");
      p.tap_y0 = a.sub_py - 1; p.tap_x0 = a.sub_px - 1; p.tap_w = sub_tx;
      ps.sub_short = (sub_ty == 3 ? 1 : 0) | (sub_tx == 3 ? 2 : 0);
      p.osy = p.osx = 2; p.ooy = a.sub_py; p.oox = a.sub_px; p.OH = OH; p.OW = OW;
    }
    const ConvTile t = pick_conv_tile(a.nimg, GH, GW);
    p.nimg = a.nimg; p.H = GH; p.W = GW; p.TW = t.tw; p.TH = t.th; p.TN = t.tn;
    p.tw_log = ilog2(t.tw);
    p.thw_log = ilog2(t.tw * t.th);
    p.tiles_x = (GW + t.tw - 1) / t.tw;
    p.tiles_y = (GH + t.th - 1) / t.th;
    p.m_tiles = p.tiles_x * p.tiles_y * ((a.nimg + t.tn - 1) / t.tn);
    const uint32_t box[4] = {BK, (uint32_t)t.tw, (uint32_t)t.th, (uint32_t)t.tn};
    if (s2) {
      // parity view k = 2 py + px: starts at input pixel (px, py), (W / 2) x (H / 2) pixels at twice the pixel strides
      const uint64_t dims[4] = {(uint64_t)a.K1, (uint64_t)GW, (uint64_t)GH, (uint64_t)a.nimg};
      const uint64_t str[3] = {(uint64_t)a.K1 * 4, (uint64_t)a.K1 * 4 * a.W, (uint64_t)a.K1 * 2 * a.W * a.H};
      if (make_tmap_f16(&p.tmA, a.A, 4, dims, str, box, 1)) return 3;
      for (int k = 1; k < 4; ++k)
        if (make_tmap_f16(&p2.tmP[k - 1], a.A + ((long long)(k >> 1) * a.W + (k & 1)) * a.K1, 4, dims, str, box, 1)) return 3;
    } else {
      const uint64_t dims[4] = {(uint64_t)a.K1, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.nimg};
      const uint64_t str[3] = {(uint64_t)a.lda1 * 2, (uint64_t)a.lda1 * 2 * a.W, (uint64_t)a.lda1 * 2 * a.W * a.H};
      if (make_tmap_f16(&p.tmA, a.A, 4, dims, str, box, 1)) return 3;
      // shifted views for the third tap of an odd axis: element (x, y) of view k is element (x - [k != 0], y - [k != 1])
      // of A; the kernel reads them at coordinates >= 1 only, so no address before A is touched
      const long long shift[3] = {(long long)a.W * a.lda1, (long long)a.lda1, (long long)(a.W + 1) * a.lda1};
      for (int k = 0; k < 3; ++k) {
        const bool used = k == 2 ? ps.sub_short == 3 : ((ps.sub_short >> k) & 1) != 0;
        if (used && make_tmap_f16(&ps.tmS[k], a.A - shift[k], 4, dims, str, box, 1)) return 3;
      }
    }
    if (two) {
      const uint64_t dims[4] = {(uint64_t)a.K2, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.nimg};
      const uint64_t str[3] = {(uint64_t)a.lda2 * 2, (uint64_t)a.lda2 * 2 * a.W, (uint64_t)a.lda2 * 2 * a.W * a.H};
      if (make_tmap_f16(&p.tmA2, a.A2, 4, dims, str, box, 1)) return 3;
    }
  } else {
    p.a_rank = 2;
    p.m_tiles = (a.M + BM - 1) / BM;
    const uint32_t box[2] = {BK, BM};
    {
      const uint64_t dims[2] = {(uint64_t)a.K1, (uint64_t)a.M};
      const uint64_t str[1] = {(uint64_t)a.lda1 * 2};
      if (make_tmap_f16(&p.tmA, a.A, 2, dims, str, box, 1)) return 3;
    }
    if (two) {
      const uint64_t dims[2] = {(uint64_t)a.K2, (uint64_t)a.M};
      const uint64_t str[1] = {(uint64_t)a.lda2 * 2};
      if (make_tmap_f16(&p.tmA2, a.A2, 2, dims, str, box, 1)) return 3;
    }
  }

  int bn = a.force_bn;
  if (a.mode == EPI_GEGLU) {
    bn = 2 * kGegluGranule;
    VS_REQUIRE(a.N % bn == 0, "gemm_tc: GEGLU needs N %% %d == 0 (N=%d)", bn, a.N);
    VS_REQUIRE(a.bias != nullptr && a.residual == nullptr && a.rowvec == nullptr, "gemm_tc: GEGLU takes a bias only");
  } else if (bn == 0) {
    bn = pick_bn(p.m_tiles, a.N, p.num_kb);
  }
  VS_REQUIRE(bn == 64 || bn == 128 || bn == 160 || bn == 256, "gemm_tc: unsupported BLOCK_N %d", bn);
  p.n_tiles = (a.N + bn - 1) / bn;
  {
    const uint64_t dims[2] = {(uint64_t)Ktot, (uint64_t)a.N};
    const uint64_t str[1] = {(uint64_t)Ktot * 2};
    const uint32_t box[2] = {BK, (uint32_t)bn};
    if (make_tmap_f16(&p.tmB, a.Bw, 2, dims, str, box, 1)) return 3;
  }
  // staged (transposed, coalesced) epilogue whenever the output geometry allows it: 16-byte strides, whole 32-column
  // sub-tiles, float4-aligned bias / row vectors
  const int out_cols = (a.mode == EPI_GEGLU) ? a.N / 2 : a.N;
  p.staged = (out_cols % EPI_COLS == 0) && (a.ldc % 8 == 0) && ((reinterpret_cast<uintptr_t>(a.out) & 15) == 0) &&
             (!a.residual || ((a.ldr % 8 == 0) && ((reinterpret_cast<uintptr_t>(a.residual) & 15) == 0))) &&
             (!a.bias || (reinterpret_cast<uintptr_t>(a.bias) & 15) == 0) &&
             (!a.rowvec || ((reinterpret_cast<uintptr_t>(a.rowvec) & 15) == 0 && p.ldrv % 4 == 0));
  if (a.mode == EPI_QUICK_GELU)
    VS_REQUIRE(a.taps == 1 && p.staged && a.residual == nullptr && a.rowvec == nullptr && !a.ln_stats && !a.ln_parts &&
               a.ln_sums_out == nullptr && (bn == 128 || bn == 256),
               "gemm_tc: the quick-GELU epilogue takes a plain GEMM with a bias only, N %% 32 == 0 and BLOCK_N 128 / 256 (got %d)", bn);
  if (a.mode == EPI_RELU)
    VS_REQUIRE(a.taps == 9 && !two && !s2 && p.staged && a.residual == nullptr && a.rowvec == nullptr && !a.ln_stats &&
               a.ln_sums_out == nullptr,
               "gemm_tc: the ReLU epilogue takes a 3x3 conv of one source with a bias only and N %% 32 == 0");
  if (!p.staged) VS_REQUIRE(a.mode == EPI_LINEAR, "gemm_tc: GEGLU output needs 32-column aligned, 16-byte strided rows");
  if (a.ln_stats || a.ln_parts) VS_REQUIRE(p.staged && (reinterpret_cast<uintptr_t>(a.ln_u) & 15) == 0, "gemm_tc: folded LayerNorm needs the staged epilogue");
  if (a.ln_sums_out) VS_REQUIRE(p.staged, "gemm_tc: row statistics output needs the staged epilogue (N %% 32 == 0, aligned rows)");
  ProfScope prof(st, a.taps != 1 ? PC_CONV : PC_GEMM, 2.0 * a.M * (double)a.N * Ktot, 1, a.M, a.N, Ktot);
  if (a.mode == EPI_GEGLU) {
    if (const int e = launch_linear_slot<256>(st, p, a); e >= 0) return e;
    if (p.ln_stats || p.ln_parts) return launch<256, EPI_F_GEGLU | EPI_F_LN>(st, p);
    return launch<256, EPI_F_GEGLU>(st, p);
  }
  if (a.mode == EPI_QUICK_GELU) return bn == 256 ? launch<256, EPI_F_QGELU>(st, p) : launch<128, EPI_F_QGELU>(st, p);
  if (a.mode == EPI_RELU) {
    switch (bn) {
      case 64: return launch<64, EPI_F_RELU>(st, p);
      case 128: return launch<128, EPI_F_RELU>(st, p);
      case 256: return launch<256, EPI_F_RELU>(st, p);
      default: return launch<160, EPI_F_RELU>(st, p);
    }
  }
  if (s2) {
    VS_REQUIRE(a.residual == nullptr && a.rowvec == nullptr && a.ln_sums_out == nullptr && p.staged,
               "gemm_tc: the stride-2 conv takes a bias only and needs N %% 32 == 0");
    static_cast<GemmParams&>(p2) = p;
    switch (bn) {
      case 64: return launch<64, 0, GemmParamsS2>(st, p2);
      case 128: return launch<128, 0, GemmParamsS2>(st, p2);
      case 256: return launch<256, 0, GemmParamsS2>(st, p2);
      default: return launch<160, 0, GemmParamsS2>(st, p2);
    }
  }
  if (sub && ((OH | OW) & 1)) {
    VS_REQUIRE(a.residual == nullptr && a.rowvec == nullptr && p.staged, "gemm_tc: an odd-sized sub-pixel conv takes a bias only");
    switch (bn) {
      case 64: return launch<64, 0, GemmParamsSub>(st, ps);
      case 128: return launch<128, 0, GemmParamsSub>(st, ps);
      case 256: return launch<256, 0, GemmParamsSub>(st, ps);
      default: return launch<160, 0, GemmParamsSub>(st, ps);
    }
  }
  if (bn == 128 || bn == 160) {
    const int e = bn == 128 ? launch_linear_slot<128>(st, p, a) : launch_linear_slot<160>(st, p, a);
    if (e >= 0) return e;
  }
  switch (bn) {
    case 64: return launch_linear<64>(st, p);
    case 128: return launch_linear<128>(st, p);
    case 256: return launch_linear<256>(st, p);
    default: return launch_linear<160>(st, p);
  }
}

// Panel of output parity (py, px) inside the up-sampler weights (see pack_conv_subpixel): the 3x3 panel itself when both
// target axes are odd at parity (0, 0), else one of the panels of `wsub`.
static const __half* subpixel_panel(const __half* w3x3, const __half* wsub, int cout, int cin, int py, int px, bool odd_y,
                                    bool odd_x) {
  const bool ty3 = py == 0 && odd_y, tx3 = px == 0 && odd_x;
  const size_t tap = (size_t)cout * cin;
  if (ty3 && tx3) return w3x3;
  if (ty3) return wsub + (16 + 6 * px) * tap;
  if (tx3) return wsub + (28 + 6 * py) * tap;
  return wsub + (size_t)(2 * py + px) * 4 * tap;
}

int upsample_conv3x3(cudaStream_t st, const __half* x, int nimg, int H, int W, int C, const __half* w3x3, const __half* wsub,
                     const float* bias, int cout, int OH, int OW, __half* out) {
  VS_REQUIRE((OH == 2 * H || OH == 2 * H - 1) && (OW == 2 * W || OW == 2 * W - 1),
             "upsample_conv3x3: output %dx%d is not 2x (or 2x - 1) of the %dx%d input", OH, OW, H, W);
  VS_REQUIRE(w3x3 != nullptr || ((OH & 1) == 0 && (OW & 1) == 0), "upsample_conv3x3: odd output sizes need the 3x3 panel");
  for (int par = 0; par < 4; ++par) {
    GemmArgs g;
    g.A = x; g.K1 = C; g.lda1 = C; g.Bw = subpixel_panel(w3x3, wsub, cout, C, par >> 1, par & 1, OH & 1, OW & 1); g.taps = 4;
    g.sub_py = par >> 1; g.sub_px = par & 1; g.OH = OH; g.OW = OW; g.nimg = nimg; g.H = H; g.W = W; g.M = nimg * H * W;
    g.N = cout; g.bias = bias; g.out = out; g.ldc = cout;
    if (int e = gemm_tc(st, g)) return e;
  }
  return 0;
}

}  // namespace vs
