// wgmma / TMA flash attention for sm_90a (spatial self-attention N x N and cross-attention N x 77; d = 40 / 80).
//
// One CTA = (batch, head, 128 queries), three warpgroups (FlashAttention-3 structure):
//   warpgroup 0   TMA producer: one elected thread of warp 0 loads Q once, then streams BKV-key K / V tiles into a
//                 STAGES-deep ring guarded by full / empty mbarriers (4-D descriptors [d, head, token, batch] straight from
//                 the fused QKV buffer; head dims are zero-padded to whole 64-column blocks by the TMA out-of-bounds
//                 fill, which also zero-fills keys beyond nk and queries beyond nq).  It gives its registers to the
//                 consumers with setmaxnreg.
//   warpgroups 1-2  consumers, 64 query rows each; every K / V tile in shared memory serves both:
//     S = Q K^T   wgmma.m64nBKVk16, Q and K from 128-byte-swizzled shared memory (both K-major), fp32 in registers
//     softmax     online, per row: max over the warp quad, exp2 of the scaled scores, exact rescale of O and l
//     O += P V    wgmma with the fp16 probabilities as the REGISTER A operand (the S accumulator layout of each warp is
//                 the A-fragment layout), V from shared memory as an MN-major B operand
// Inside a consumer the two products are software-pipelined: Q K^T of tile j and P V of tile j - 1 are issued together,
// the softmax of tile j runs while P V of tile j - 1 is still on the tensor cores (wgmma_wait<1> retires only Q K^T),
// and a stage goes back to the producer once the P V that read it has retired.  Two named barriers hand the tensor cores
// from one consumer to the other once its MMAs are issued (ping-pong), so one consumer's softmax (MUFU + FP32) runs under
// the other's MMAs.
//
// Replaces diffusers AttnProcessor2_0 / EDLoRA_AttnProcessor.__call__ (reference utils/edlora_util.py:47-65,
// models/animatediff_models/attention.py:229-241).
#include "common.cuh"
#include "kernels.h"

namespace vs {
namespace {

constexpr int TQ = 64;                   // queries per consumer warpgroup (= wgmma M); a CTA covers 2 TQ
constexpr int ATT_THREADS = 384;         // producer warpgroup + 2 consumer warpgroups
constexpr int PRODUCER_REGS = 24, CONSUMER_REGS = 240;   // 128 x 24 + 256 x 240 <= 64 K registers

template <int D>
struct TCfg {
  // keys per tile and ring depth, chosen by measurement at the UNet's attention shapes (DESIGN §8.1)
  static constexpr int BKV = 128;
  static constexpr int STAGES = D > 64 ? 3 : 4;
  static constexpr int NCB = (D + 63) / 64;            // 64-wide (128-byte) column blocks of Q/K/V tiles
  static constexpr int DPK = (D + 15) / 16 * 16;       // padded contraction length of Q K^T
  static constexpr int Q_BLOCK = TQ * 128;             // one 64-row x 128-byte swizzled Q block
  static constexpr int KV_BLOCK = BKV * 128;           // one BKV-row x 128-byte swizzled K or V block
  static constexpr int Q_BYTES = NCB * Q_BLOCK;        // one consumer's queries
  static constexpr int KV_STAGE_BYTES = 2 * NCB * KV_BLOCK;         // K then V
  static constexpr int OREG = (D > 64) ? 32 + 8 : 32;               // O accumulator: one n64 block (+ one n16 block)
  static constexpr int SMEM = 2 * Q_BYTES + STAGES * KV_STAGE_BYTES + 1024 + 8 * (1 + 2 * STAGES);
  static_assert(D == 40 || D == 80, "head dims of the tensor-core path");
  static_assert(SMEM <= 227 * 1024, "shared memory");
};

struct TAttnArgs {
  CUtensorMap tmQ, tmK, tmV;
  __half* o;
  int ldo;
  long long o_bs;
  int nq, nk, kv_div;
  float scale_log2;
};

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <int D>
__global__ void __launch_bounds__(ATT_THREADS, 1) attn_tc_kernel(const __grid_constant__ TAttnArgs p) {
  using C = TCfg<D>;
  constexpr int BKV = C::BKV, STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t q_s = base;                                   // [2 consumers][NCB][64 rows x 128 B]
  const uint32_t kv_s = q_s + 2 * C::Q_BYTES;                  // [STAGES][K: NCB blocks | V: NCB blocks]
  const uint32_t bars = kv_s + STAGES * C::KV_STAGE_BYTES;
  const uint32_t q_full = bars;
  auto kv_full = [&](int s) { return bars + 8u * (1 + s); };
  auto kv_empty = [&](int s) { return bars + 8u * (1 + STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int q0 = blockIdx.x * 2 * TQ, head = blockIdx.y, b = blockIdx.z;
  const int nkt = (p.nk + BKV - 1) / BKV;

  if (threadIdx.x == 0) {
    prefetch_tmap(&p.tmQ); prefetch_tmap(&p.tmK); prefetch_tmap(&p.tmV);
    mbar_init(q_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(kv_full(s), 1);
      mbar_init(kv_empty(s), 8);                 // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();                                    // set-up above overlaps the previous kernel's tail

  if (wg == 0) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp != 0) return;
    // ===================================================================== TMA producer (whole warp, one elected issuer)
    const int bk = b / p.kv_div;
    if (elect_one()) {
      mbar_expect_tx(q_full, 2 * C::Q_BYTES);
#pragma unroll
      for (int g = 0; g < 2; ++g)
#pragma unroll
        for (int cb = 0; cb < C::NCB; ++cb)
          tma_load_4d(q_s + g * C::Q_BYTES + cb * C::Q_BLOCK, &p.tmQ, q_full, cb * 64, head, q0 + g * TQ, b);
    }
    __syncwarp();
    for (int j = 0, s = 0, ph = 0; j < nkt; ++j) {
      mbar_wait(kv_empty(s), ph ^ 1);
      if (elect_one()) {
        const uint32_t k_dst = kv_s + s * C::KV_STAGE_BYTES, v_dst = k_dst + C::NCB * C::KV_BLOCK;
        mbar_expect_tx(kv_full(s), C::KV_STAGE_BYTES);
#pragma unroll
        for (int cb = 0; cb < C::NCB; ++cb) {
          tma_load_4d(k_dst + cb * C::KV_BLOCK, &p.tmK, kv_full(s), cb * 64, head, j * BKV, bk);
          tma_load_4d(v_dst + cb * C::KV_BLOCK, &p.tmV, kv_full(s), cb * 64, head, j * BKV, bk);
        }
      }
      __syncwarp();
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    return;
  }

  // ======================================================================= consumers
  setmaxnreg_inc<CONSUMER_REGS>();
  const int g = wg - 1, wq = warp & 3, q4 = lane & 3;
  const uint32_t qg = q_s + g * C::Q_BYTES;
  // Tensor-core hand-off: consumer g waits on named barrier 1 + g before it issues MMAs and arrives on the other's once
  // they are issued.  Consumer 0 goes first; consumer 1 skips its arrival after its last issue, so every arrival is
  // waited for (both issue nkt + 1 times).
  const int bar_mine = 1 + g, bar_other = 2 - g;
  if (g == 1) named_bar_arrive(bar_other, 256);

  const float sc = p.scale_log2;
  float o[C::OREG];
#pragma unroll
  for (int i = 0; i < C::OREG; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};      // rows lane / 4 and lane / 4 + 8 of this warp
  float s[BKV / 2];                                            // S of the newest key tile
  uint32_t pf[BKV / 16][4];                                    // fp16 P of the previous tile, in A-fragment layout

  auto stage_addr = [&](int j) { return kv_s + (uint32_t)(j % STAGES) * C::KV_STAGE_BYTES; };
  auto issue_qk = [&](int j) {
    const uint32_t k_a = stage_addr(j);
#pragma unroll
    for (int k = 0; k < C::DPK / 16; ++k) {
      const uint32_t qoff = (uint32_t)((k * 16) / 64) * C::Q_BLOCK + (uint32_t)((k * 16) % 64) * 2;
      const uint32_t koff = (uint32_t)((k * 16) / 64) * C::KV_BLOCK + (uint32_t)((k * 16) % 64) * 2;
      wgmma_ss<BKV>(s, gmma_desc_sw128(qg + qoff), gmma_desc_sw128(k_a + koff), k != 0 ? 1u : 0u);
    }
  };
  auto issue_pv = [&](int j) {                   // 16 keys per instruction
    const uint32_t v_a = stage_addr(j) + C::NCB * C::KV_BLOCK;
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      const uint32_t v_rows = v_a + kk * 16 * 128;
      wgmma_m64n64_rs<1>(o, pf[kk], gmma_desc_sw128_mn(v_rows, C::KV_BLOCK), 1u);
      if (D > 64) wgmma_m64n16_rs<1>(o + 32, pf[kk], gmma_desc_sw128_mn(v_rows + C::KV_BLOCK, C::KV_BLOCK), 1u);
    }
  };
  // online softmax of S (tile j) in place; returns the rescale factors of O for the two rows of this thread
  auto softmax = [&](int j, float* alpha) {
    const int kbase = j * BKV;
    if (kbase + BKV > p.nk) {                    // keys beyond nk (last tile only)
#pragma unroll
      for (int i = 0; i < BKV / 2; ++i)
        if (kbase + 8 * (i >> 2) + 2 * q4 + (i & 1) >= p.nk) s[i] = -INFINITY;
    }
    // row h = 0: registers with (i >> 1) even, h = 1: odd
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = m[h];
#pragma unroll
      for (int i = 2 * h; i < BKV / 2; i += 4) mx = fmaxf(mx, fmaxf(s[i], s[i + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      alpha[h] = fast_exp2((m[h] - mx) * sc);    // exp2(-inf) = 0 on the first tile
      m[h] = mx;
      const float ms = mx * sc;
      float rs = 0.f;
#pragma unroll
      for (int i = 2 * h; i < BKV / 2; i += 4) {
        s[i] = fast_exp2(fmaf(s[i], sc, -ms));
        s[i + 1] = fast_exp2(fmaf(s[i + 1], sc, -ms));
        rs += s[i] + s[i + 1];
      }
      l[h] = fmaf(l[h], alpha[h], rs);
    }
  };
  auto pack_p = [&]() {
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) pf[kk][r] = pack_h2(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
  };
  auto release = [&](int j) {                    // the P V that read tile j's stage has retired
    if (lane == 0) mbar_arrive(kv_empty(j % STAGES));
  };

  mbar_wait(q_full, 0);
  // ---- tile 0: Q K^T alone
  mbar_wait(kv_full(0), 0);
  named_bar_sync(bar_mine, 256);
  wgmma_fence();
  issue_qk(0);
  wgmma_commit();
  named_bar_arrive(bar_other, 256);
  wgmma_wait<0>();
  {
    float alpha[2];
    softmax(0, alpha);                           // O = 0: nothing to rescale
    pack_p();
  }
  // ---- steady state: Q K^T of tile j and P V of tile j - 1 in flight together
  for (int j = 1; j < nkt; ++j) {
    mbar_wait(kv_full(j % STAGES), (j / STAGES) & 1);
    named_bar_sync(bar_mine, 256);
    wgmma_fence();
    issue_qk(j);
    wgmma_commit();
    issue_pv(j - 1);
    wgmma_commit();
    named_bar_arrive(bar_other, 256);
    wgmma_wait<1>();                             // S of tile j is complete; P V of tile j - 1 may still run
    float alpha[2];
    softmax(j, alpha);
    // ptxas schedules a wgmma wait at the top of its basic block, which here would put it before the softmax and
    // serialise the softmax behind P V.  Under a branch ptxas cannot evaluate (kv_div >= 1 is checked on the host) the
    // wait gets a block of its own after the softmax (tests/test_attn_sass_cpu.py checks the MUFU.EX2 stay in between).
    if (p.kv_div > 0) wgmma_wait<0>();
    release(j - 1);
#pragma unroll
    for (int i = 0; i < C::OREG; ++i) o[i] *= alpha[(i >> 1) & 1];
    pack_p();
  }
  // ---- P V of the last tile
  named_bar_sync(bar_mine, 256);
  wgmma_fence();
  issue_pv(nkt - 1);
  wgmma_commit();
  if (g == 0) named_bar_arrive(bar_other, 256);
  wgmma_wait<0>();
  release(nkt - 1);

  // ---- epilogue: O / l -> fp16 -> HBM
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
  }
  const float inv[2] = {1.f / l[0], 1.f / l[1]};
  const int r0 = q0 + g * TQ + 16 * wq + (lane >> 2);
  __half* ob = p.o + b * p.o_bs + head * D;
#pragma unroll
  for (int i = 0; i < C::OREG; i += 2) {
    const int h = (i >> 1) & 1, c = 8 * (i >> 2) + 2 * q4, r = r0 + 8 * h;
    if (c < D && r < p.nq)
      *reinterpret_cast<__half2*>(ob + (long long)r * p.ldo + c) = __floats2half2_rn(o[i] * inv[h], o[i + 1] * inv[h]);
  }
}

template <int D>
int launch(cudaStream_t st, const __half* q, int ldq, const __half* k, int ldk, const __half* v, int ldv, __half* o, int ldo,
           int batch, int nq, int nk, int heads, long long q_bs, long long kv_bs, long long o_bs, int kv_div) {
  using C = TCfg<D>;
  static bool configured = false;
  if (!configured) {
    VS_CHECK_CUDA(cudaFuncSetAttribute(attn_tc_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
    configured = true;
  }
  TAttnArgs a;
  memset(&a, 0, sizeof(a));
  const int bkv = (batch + kv_div - 1) / kv_div;
  {
    const uint64_t dims[4] = {(uint64_t)D, (uint64_t)heads, (uint64_t)nq, (uint64_t)batch};
    const uint64_t str[3] = {(uint64_t)D * 2, (uint64_t)ldq * 2, (uint64_t)(q_bs > 0 ? q_bs : (long long)nq * ldq) * 2};
    const uint32_t box[4] = {64, 1, TQ, 1};
    if (make_tmap_f16(&a.tmQ, q, 4, dims, str, box, 1)) return 3;
  }
  {
    const uint64_t dims[4] = {(uint64_t)D, (uint64_t)heads, (uint64_t)nk, (uint64_t)bkv};
    const uint64_t strk[3] = {(uint64_t)D * 2, (uint64_t)ldk * 2, (uint64_t)(kv_bs > 0 ? kv_bs : (long long)nk * ldk) * 2};
    const uint64_t strv[3] = {(uint64_t)D * 2, (uint64_t)ldv * 2, (uint64_t)(kv_bs > 0 ? kv_bs : (long long)nk * ldv) * 2};
    const uint32_t box[4] = {64, 1, (uint32_t)C::BKV, 1};
    if (make_tmap_f16(&a.tmK, k, 4, dims, strk, box, 1)) return 3;
    if (make_tmap_f16(&a.tmV, v, 4, dims, strv, box, 1)) return 3;
  }
  a.o = o; a.ldo = ldo; a.o_bs = o_bs; a.nq = nq; a.nk = nk; a.kv_div = kv_div;
  a.scale_log2 = 1.4426950408889634f / sqrtf((float)D);
  ProfScope prof(st, PC_ATTN, 4.0 * batch * heads * (double)nq * nk * D, 1, nq, nk, D);
  dim3 grid((nq + 2 * TQ - 1) / (2 * TQ), heads, batch);
  return launch_pdl(attn_tc_kernel<D>, grid, dim3(ATT_THREADS), C::SMEM, st, 1, a);
}

}  // namespace

// Returns -1 when the shape is not handled by the wgmma kernel (caller uses the mma.sync kernel).
int attention_tc(cudaStream_t st, const __half* q, int ldq, const __half* k, int ldk, const __half* v, int ldv, __half* o,
                 int ldo, int batch, int nq, int nk, int heads, int d, long long q_bs, long long kv_bs, long long o_bs,
                 int kv_div) {
  if ((ldq % 8) || (ldk % 8) || (ldv % 8) || (ldo % 2)) return -1;
  if ((q_bs % 8) || (kv_bs % 8)) return -1;
  VS_REQUIRE(kv_div >= 1, "attention_tc: kv_div must be >= 1 (got %d)", kv_div);
  if (d == 40) return launch<40>(st, q, ldq, k, ldk, v, ldv, o, ldo, batch, nq, nk, heads, q_bs, kv_bs, o_bs, kv_div);
  if (d == 80) return launch<80>(st, q, ldq, k, ldk, v, ldv, o, ldo, batch, nq, nk, heads, q_bs, kv_bs, o_bs, kv_div);
  return -1;
}

}  // namespace vs
