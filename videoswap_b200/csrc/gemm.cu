// wgmma / TMA GEMM and implicit-GEMM 3x3 convolution for sm_90a.
//
// One persistent, warp-specialised kernel of three warpgroups: warpgroup 0 is the TMA producer (one elected thread of
// warp 0 issues the copies; the warpgroup gives most of its registers to the others with setmaxnreg), warpgroups 1 and 2
// are the consumers: each owns 64 rows of the 128 (M) x BN (N) tile, issues wgmma.m64nNk16 on the 128-byte-swizzled
// operand ring in shared memory and keeps its accumulator in registers.  K advances 64 elements (one swizzle row of
// fp16) per ring stage; the producer runs up to STAGES k-blocks ahead, across tile boundaries, so the next tile's
// operands are in flight while the consumers run the epilogue of the current one.
// A 3x3 convolution is the same kernel with nine K segments: tap (dy,dx) loads the NHWC activation box shifted by
// (dy,dx) through a 4-D TMA descriptor and the out-of-bounds zero fill of TMA provides the padding; a channel concat
// is two descriptors walked back to back along K.
//
// Epilogue (per consumer warp, 16 rows): registers -> [folded LayerNorm: rstd * acc - rstd * mean * u] + bias (+ time-
// embedding / positional row vector) / GEGLU -> fp16 -> warp-private swizzled shared-memory transpose, 32 columns at a
// time -> (+ fp16 residual) -> coalesced 16-byte global stores.  Tiny-N outputs (conv_out, N = 4) keep a direct-store path.
//
// Replaces (reference call sites): InflatedConv3d 3x3 / 1x1 (models/animatediff_models/resnet.py:9-18), every
// nn.Linear / 1x1 conv of Transformer3DModel (attention.py:65-93,174-204) and the motion module
// (motion_module.py:113-136,202-218), GEGLU (diffusers FeedForward).
#include "common.cuh"
#include "kernels.h"

namespace vs {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int GEMM_THREADS = 384;                   // producer warpgroup + 2 consumer warpgroups
constexpr int SMEM_LIMIT = 227 * 1024;
constexpr int EPI_COLS = 32;                        // output columns per epilogue sub-tile (64 B of fp16)
constexpr int EPI_WARP_BYTES = 16 * 64;             // per consumer warp: [16 rows x 64 B] transpose staging
constexpr int EPI_BYTES = 8 * EPI_WARP_BYTES;
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 64 K registers
enum { EPI_F_GEGLU = 1, EPI_F_RES = 2, EPI_F_RV = 4, EPI_F_LN = 8, EPI_F_LNOUT = 16 };   // compile-time epilogue features

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

template <int BN>
struct Cfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STAGES_RAW = (SMEM_LIMIT - 2048 - EPI_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(B_STAGE_BYTES % 1024 == 0, "B stage must keep 1024-byte alignment for SWIZZLE_128B");
  static_assert(STAGES >= 3, "pipeline too shallow");
  static_assert(BN % 32 == 0 && BN <= 256, "wgmma N");
};

__device__ __forceinline__ uint32_t sw64_off(int row, int chunk) {   // byte offset inside a [rows x 64 B] swizzled tile
  return (uint32_t)(row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4));
}

// acc (+)= A[64 rows] B[BN rows]^T over one k16 step: BN / 64 m64n64 instructions and one m64n32 for the rest.
template <int BN>
__device__ __forceinline__ void mma_k16(float* acc, uint64_t da, uint64_t db, uint32_t scale_d) {
#pragma unroll
  for (int c = 0; c < BN / 64; ++c) wgmma_m64n64(acc + 32 * c, da, db + (uint64_t)(c * 64 * 128 / 16), scale_d);
  if (BN % 64) wgmma_m64n32(acc + 32 * (BN / 64), da, db + (uint64_t)((BN / 64) * 64 * 128 / 16), scale_d);
}

template <int BN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
  using C = Cfg<BN>;
  constexpr bool GEGLU = (EPI & EPI_F_GEGLU) != 0, HAS_RES = (EPI & EPI_F_RES) != 0, HAS_RV = (EPI & EPI_F_RV) != 0;
  // LN: the A operand is the RAW input of a LayerNorm whose affine map is folded into the weights:
  //   LN(x) W^T = rstd (x W'^T) - rstd mean u + c,  W' = W * gamma, u[n] = sum_k W'[n,k], c = beta W^T + bias (the `bias`)
  constexpr bool LN = (EPI & EPI_F_LN) != 0;
  // LNOUT: this GEMM's output feeds a LayerNorm (folded into the NEXT GEMM): the row statistics of what is stored -- the
  // fp16-rounded values, after the residual add -- are accumulated here, in the shadow of the store path, and written as
  // one (sum, sum of squares) pair per (column tile, row).  Deterministic (no atomics); replaces a stand-alone statistics
  // pass that would re-read every such tensor from HBM.
  constexpr bool LNOUT = (EPI & EPI_F_LNOUT) != 0;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t epi_base = smem_base + C::STAGES * C::STAGE_BYTES;
  const uint32_t bar_base = epi_base + EPI_BYTES;
  // barrier layout: full[S], empty[S]
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int total_tiles = p.m_tiles * p.n_tiles;
  const int nst = (p.stages > 0 && p.stages < C::STAGES) ? p.stages : C::STAGES;   // ring depth (debug knob: "gemm_stages")
  // Tile order: n fastest, tiles round-robin over the CTAs (CTAs running at the same time share the A row panel and a
  // few weight tiles in L2).
  const int t_begin = blockIdx.x, t_step = gridDim.x;

  if (threadIdx.x == 0) {
    prefetch_tmap(&p.tmA);
    prefetch_tmap(&p.tmB);
    if (p.kb_src1 < p.kb_per_tap) prefetch_tmap(&p.tmA2);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);                // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_trigger();                                 // the next kernel may start its own set-up
  pdl_wait();                                    // everything above overlapped the previous kernel's tail; its data is visible now

  if (wg == 0) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp != 0) return;
    // =================================================================== TMA producer (whole warp, one elected issuer)
    const int num_kb = p.num_kb, kb_per_tap = p.kb_per_tap, kb_src1 = p.kb_src1;
    const bool conv = p.a_rank == 4;
    const int tap_x0 = p.tap_x0, tap_x1 = p.tap_x0 + p.tap_w;
    uint32_t pr_s = 0, pr_ph = 0;              // ring stage / phase, carried across tiles
    for (int tile = t_begin; tile < total_tiles; tile += t_step) {
      const int m_tile = tile / p.n_tiles, n_tile = tile - m_tile * p.n_tiles;
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
          const int c = (first ? r : r - kb_src1) * BK;
          mbar_expect_tx(fb, C::STAGE_BYTES);
          if (conv) tma_load_4d(a_dst, tm, fb, c, x0 + dx, y0 + dy, i0);
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
  const int g = wg - 1;                        // rows [64 g, 64 g + 64) of the tile
  const int wq = warp & 3;                     // warp inside the warpgroup: rows 16 wq .. 16 wq + 15 of those
  const int q = lane & 3;
  const int rbase = 64 * g + 16 * wq + (lane >> 2);   // this thread's tile rows: rbase and rbase + 8
  const uint32_t stage_buf = epi_base + (uint32_t)(warp - 4) * EPI_WARP_BYTES;
  const bool has_bias = p.bias != nullptr;
  const bool staged = p.staged != 0;
  const int num_kb = p.num_kb;
  // output pixel (row of the GEMM) of tile row `row`, -1 = outside the problem
  auto tile_pixel = [&](int m_tile, int row) -> int {
    if (p.a_rank == 4) {
      const int x0 = (m_tile % p.tiles_x) * p.TW;
      const int y0 = ((m_tile / p.tiles_x) % p.tiles_y) * p.TH;
      const int i0 = (m_tile / (p.tiles_x * p.tiles_y)) * p.TN;
      const int ti = row >> p.thw_log, rem = row & ((1 << p.thw_log) - 1);
      const int y = y0 + (rem >> p.tw_log), x = x0 + (rem & (p.TW - 1)), img = i0 + ti;
      return ((img < p.nimg) && (y < p.H) && (x < p.W)) ? (img * p.OH + y * p.osy + p.ooy) * p.OW + x * p.osx + p.oox : -1;
    }
    const int px = m_tile * BM + row;
    return px < p.M ? px : -1;
  };

  float acc[BN / 2];
  uint32_t s = 0, ph = 0;
  for (int tile = t_begin; tile < total_tiles; tile += t_step) {
    // ------------------------------------------------------------------ main loop
    uint32_t prev = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(full_bar(s), ph);
      wgmma_fence();
      const uint32_t a_addr = smem_base + s * C::STAGE_BYTES;
      const uint64_t da = gmma_desc_sw128(a_addr + g * 64 * 128);
      const uint64_t db = gmma_desc_sw128(a_addr + A_STAGE_BYTES);
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) mma_k16<BN>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
      wgmma_commit();
      if (kb > 0) {                            // the MMAs of the previous k-block have read their stage: release it
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(empty_bar(prev));
      }
      prev = s;
      if (++s == (uint32_t)nst) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(empty_bar(prev));

    // ------------------------------------------------------------------ epilogue
    const int m_tile = tile / p.n_tiles, n_tile = tile - m_tile * p.n_tiles;
    const int n0 = n_tile * BN;
    int pix[2];
    pix[0] = tile_pixel(m_tile, rbase);
    pix[1] = tile_pixel(m_tile, rbase + 8);
    const float* rv[2] = {nullptr, nullptr};
    if (HAS_RV || !staged) {
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
          if (p.ln_nparts > 0) {            // statistics from the producer GEMM's per-column-tile partial sums
            float S = 0.f, Q = 0.f;
            for (int k = 0; k < p.ln_nparts; ++k) {
              const float2 v = __ldg(p.ln_parts + (long long)k * p.M + pix[h]);
              S += v.x; Q += v.y;
            }
            const float mean = S * p.ln_inv_c;
            la[h] = rsqrtf(fmaxf(fmaf(-mean, mean, Q * p.ln_inv_c), 0.f) + 1e-5f);
            lb[h] = -mean * la[h];
          } else {
            const float2 st2 = __ldg(p.ln_stats + pix[h]);
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
        if (HAS_RES) {
#pragma unroll
          for (int h = 0; h < 2; ++h) rr[h] = __ldg(reinterpret_cast<const uint4*>(rrow[h] + sb * EPI_COLS));
        }
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = 4 * sb + jj;            // n8 block of the (output) tile
          const int c = 8 * j + 2 * q;          // column inside the tile (value column for GEGLU)
          float2 b = has_bias ? __ldg(reinterpret_cast<const float2*>(p.bias + n0 + c)) : make_float2(0.f, 0.f);
          float2 u = LN ? __ldg(reinterpret_cast<const float2*>(p.ln_u + n0 + c)) : make_float2(0.f, 0.f);
          float2 bg = make_float2(0.f, 0.f), ug = make_float2(0.f, 0.f);
          if (GEGLU) {                          // gate columns are BN / 2 further on, in the same thread's registers
            bg = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + BN / 2 + c));
            if (LN) ug = __ldg(reinterpret_cast<const float2*>(p.ln_u + n0 + BN / 2 + c));
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
            if (GEGLU) {
              float g0 = acc[4 * (j + BN / 16) + 2 * h], g1 = acc[4 * (j + BN / 16) + 2 * h + 1];
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
                const float2 r2 = __ldg(reinterpret_cast<const float2*>(rv[h] + c));
                f0 += r2.x; f1 += r2.y;
              }
            }
            const __half2 hv = __floats2half2_rn(f0, f1);
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(stage_buf + sw64_off((lane >> 2) + 8 * h, jj) + 4 * q),
                         "r"(*reinterpret_cast<const uint32_t*>(&hv)) : "memory");
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
            float f = acc[4 * j + e];
            if (has_bias) f += p.bias[n];
            if (rv[h]) f += rv[h][c];
            if (p.residual) f += __half2float(p.residual[(long long)pix[h] * p.ldr + n]);
            p.out[(long long)pix[h] * p.ldc + n] = __float2half_rn(f);
          }
        }
      }
    }
  }
}

struct ConvTile { int tw, th, tn; };

ConvTile pick_conv_tile(int nimg, int H, int W) {
  ConvTile best{1, 1, 128};
  long long best_cost = -1;
  for (int tw = 1; tw <= 128; tw *= 2) {
    for (int th = 1; tw * th <= 128; th *= 2) {
      const int tn = 128 / (tw * th);
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

template <int BN, int EPI>
int launch(cudaStream_t st, const GemmParams& p) {
  using C = Cfg<BN>;
  static bool configured = false;
  if (!configured) {
    VS_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    configured = true;
  }
  const int total = p.m_tiles * p.n_tiles;
  return launch_pdl(gemm_tc_kernel<BN, EPI>, dim3(total < num_sms() ? total : num_sms()), dim3(GEMM_THREADS), C::SMEM_BYTES,
                    st, 1, p);
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

// BLOCK_N by a two-term model: waves of the persistent grid x shared-memory operand bytes per k-block of one tile
// (16 KB of A + BN * 128 B of B; wider tiles need fewer bytes per flop).  Ties go to the wider tile only for long K,
// where the main loop -- not the epilogue -- dominates.
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
  VS_REQUIRE(a.taps == 1 || a.taps == 9 || a.taps == 4, "gemm_tc: taps must be 1, 9 (3x3) or 4 (2x2 sub-pixel)");
  VS_REQUIRE(a.K1 % 8 == 0 && a.K2 % 8 == 0, "gemm_tc: K must be a multiple of 8 (TMA 16-byte strides)");
  VS_REQUIRE((long long)a.M * (a.ldc > a.ldr ? a.ldc : a.ldr) < (1LL << 40) && a.M < (1 << 30), "gemm_tc: M too large");
  const bool two = a.A2 != nullptr && a.K2 > 0;
  if (two || a.taps != 1) VS_REQUIRE(a.K1 % BK == 0 && a.K2 % BK == 0, "gemm_tc: concat/conv sources need C %% 64 == 0 (got %d,%d)", a.K1, a.K2);
  GemmParams p;
  memset(&p, 0, sizeof(p));
  const int Ktap = a.K1 + (two ? a.K2 : 0);
  const int Ktot = Ktap * a.taps;
  p.taps = a.taps;
  p.kb_src1 = (a.K1 + BK - 1) / BK;
  p.kb_per_tap = p.kb_src1 + (two ? a.K2 / BK : 0);
  p.num_kb = p.kb_per_tap * a.taps;
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

  if (a.taps != 1) {
    VS_REQUIRE(a.nimg > 0 && a.H > 0 && a.W > 0 && a.M == a.nimg * a.H * a.W, "gemm_tc: bad conv geometry");
    p.a_rank = 4;
    // 3x3: taps (-1..1)^2.  2x2 (one output parity (py, px) of nearest-2x + 3x3, see pack_conv_subpixel): taps
    // {py - 1, py} x {px - 1, px}, output pixel (2 y + py, 2 x + px) of the 2H x 2W image.
    if (a.taps == 9) { p.tap_x0 = p.tap_y0 = -1; p.tap_w = 3; p.osy = p.osx = 1; p.ooy = p.oox = 0; p.OH = a.H; p.OW = a.W; }
    else {
      VS_REQUIRE((a.sub_py | 1) == 1 && (a.sub_px | 1) == 1, "gemm_tc: sub-pixel parity must be 0 or 1");
      p.tap_y0 = a.sub_py - 1; p.tap_x0 = a.sub_px - 1; p.tap_w = 2;
      p.osy = p.osx = 2; p.ooy = a.sub_py; p.oox = a.sub_px; p.OH = 2 * a.H; p.OW = 2 * a.W;
    }
    const ConvTile t = pick_conv_tile(a.nimg, a.H, a.W);
    p.nimg = a.nimg; p.H = a.H; p.W = a.W; p.TW = t.tw; p.TH = t.th; p.TN = t.tn;
    p.tw_log = ilog2(t.tw);
    p.thw_log = ilog2(t.tw * t.th);
    p.tiles_x = (a.W + t.tw - 1) / t.tw;
    p.tiles_y = (a.H + t.th - 1) / t.th;
    p.m_tiles = p.tiles_x * p.tiles_y * ((a.nimg + t.tn - 1) / t.tn);
    const uint32_t box[4] = {BK, (uint32_t)t.tw, (uint32_t)t.th, (uint32_t)t.tn};
    {
      const uint64_t dims[4] = {(uint64_t)a.K1, (uint64_t)a.W, (uint64_t)a.H, (uint64_t)a.nimg};
      const uint64_t str[3] = {(uint64_t)a.lda1 * 2, (uint64_t)a.lda1 * 2 * a.W, (uint64_t)a.lda1 * 2 * a.W * a.H};
      if (make_tmap_f16(&p.tmA, a.A, 4, dims, str, box, 1)) return 3;
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
  if (!p.staged) VS_REQUIRE(a.mode == EPI_LINEAR, "gemm_tc: GEGLU output needs 32-column aligned, 16-byte strided rows");
  if (a.ln_stats || a.ln_parts) VS_REQUIRE(p.staged && (reinterpret_cast<uintptr_t>(a.ln_u) & 15) == 0, "gemm_tc: folded LayerNorm needs the staged epilogue");
  if (a.ln_sums_out) VS_REQUIRE(p.staged, "gemm_tc: row statistics output needs the staged epilogue (N %% 32 == 0, aligned rows)");
  ProfScope prof(st, a.taps != 1 ? PC_CONV : PC_GEMM, 2.0 * a.M * (double)a.N * Ktot, 1, a.M, a.N, Ktot);
  if (a.mode == EPI_GEGLU) {
    if (p.ln_stats || p.ln_parts) return launch<256, EPI_F_GEGLU | EPI_F_LN>(st, p);
    return launch<256, EPI_F_GEGLU>(st, p);
  }
  switch (bn) {
    case 64: return launch_linear<64>(st, p);
    case 128: return launch_linear<128>(st, p);
    case 256: return launch_linear<256>(st, p);
    default: return launch_linear<160>(st, p);
  }
}

}  // namespace vs
