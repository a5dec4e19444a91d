// wgmma / TMA flash attention for sm_90a (spatial self-attention N x N and cross-attention N x 77; d = 40 / 80).
//
// One CTA = one warpgroup = (batch, head, 64 queries).  Thread 0 streams 64-key K / V tiles into a two-stage ring with
// TMA (4-D descriptors [d, head, token, batch]; head dims are zero-padded to whole 64-column blocks by the TMA
// out-of-bounds fill, which also zero-fills keys beyond nk and queries beyond nq):
//   S = Q K^T   wgmma.m64n64k16, Q and K from 128-byte-swizzled shared memory (both K-major), fp32 in registers
//   softmax     online, per row: max over the warp quad, exp2 of the scaled scores, lazy-free exact rescale of O and l
//   O += P V    wgmma with the fp16 probabilities as the REGISTER A operand (the S accumulator layout of each warp is
//               the A-fragment layout), V from shared memory as an MN-major B operand
// Several CTAs share an SM (40-80 KB of shared memory each), so one CTA's softmax overlaps another one's MMAs and loads.
//
// Replaces diffusers AttnProcessor2_0 / EDLoRA_AttnProcessor.__call__ (reference utils/edlora_util.py:47-65,
// models/animatediff_models/attention.py:229-241).
#include "common.cuh"
#include "kernels.h"

namespace vs {
namespace {

constexpr int TQ = 64;               // queries per CTA (= wgmma M)
constexpr int BKV = 64;              // keys per tile
constexpr int ATT_THREADS = 128;

template <int D>
struct TCfg {
  static constexpr int NCB = (D + 63) / 64;            // 64-wide (128-byte) column blocks of Q/K/V tiles
  static constexpr int DPK = (D + 15) / 16 * 16;       // padded contraction length of Q K^T
  static constexpr int BLOCK_BYTES = 64 * 128;         // one 64-row x 128-byte swizzled block
  static constexpr int Q_BYTES = NCB * BLOCK_BYTES;
  static constexpr int KV_STAGE_BYTES = 2 * NCB * BLOCK_BYTES;     // K then V
  static constexpr int OREG = (D > 64) ? 32 + 8 : 32;               // O accumulator: one n64 block (+ one n16 block)
  static constexpr int SMEM = Q_BYTES + 2 * KV_STAGE_BYTES + 1024 + 64;
  static_assert(D == 40 || D == 80, "head dims of the tensor-core path");
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
__global__ void __launch_bounds__(ATT_THREADS) attn_tc_kernel(const __grid_constant__ TAttnArgs p) {
  using C = TCfg<D>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t q_s = base;                                   // [NCB][64 rows x 128 B]
  const uint32_t kv_s = q_s + C::Q_BYTES;                      // [2 stages][K: NCB blocks | V: NCB blocks]
  const uint32_t bars = kv_s + 2 * C::KV_STAGE_BYTES;
  const uint32_t q_full = bars;
  auto kv_full = [&](int s) { return bars + 8u * (1 + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q4 = lane & 3;
  const int q0 = blockIdx.x * TQ, head = blockIdx.y, b = blockIdx.z, bk = b / p.kv_div;
  const int nkt = (p.nk + BKV - 1) / BKV;

  if (tid == 0) {
    prefetch_tmap(&p.tmQ); prefetch_tmap(&p.tmK); prefetch_tmap(&p.tmV);
    mbar_init(q_full, 1);
    mbar_init(kv_full(0), 1);
    mbar_init(kv_full(1), 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();                                    // set-up above overlaps the previous kernel's tail
  auto load_kv = [&](int j) {
    const uint32_t s = j & 1, k_dst = kv_s + s * C::KV_STAGE_BYTES, v_dst = k_dst + C::NCB * C::BLOCK_BYTES;
    mbar_expect_tx(kv_full(s), C::KV_STAGE_BYTES);
#pragma unroll
    for (int cb = 0; cb < C::NCB; ++cb) {
      tma_load_4d(k_dst + cb * C::BLOCK_BYTES, &p.tmK, kv_full(s), cb * 64, head, j * BKV, bk);
      tma_load_4d(v_dst + cb * C::BLOCK_BYTES, &p.tmV, kv_full(s), cb * 64, head, j * BKV, bk);
    }
  };
  if (tid == 0) {
    mbar_expect_tx(q_full, C::Q_BYTES);
    for (int cb = 0; cb < C::NCB; ++cb) tma_load_4d(q_s + cb * C::BLOCK_BYTES, &p.tmQ, q_full, cb * 64, head, q0, b);
    load_kv(0);
  }

  const float sc = p.scale_log2;
  float o[C::OREG];
#pragma unroll
  for (int i = 0; i < C::OREG; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};      // rows lane / 4 and lane / 4 + 8 of this warp
  mbar_wait(q_full, 0);
  for (int j = 0; j < nkt; ++j) {
    // every warp is past tile j - 1, so its stage may be refilled with tile j + 1 while tile j is computed
    __syncthreads();
    if (tid == 0 && j + 1 < nkt) load_kv(j + 1);
    mbar_wait(kv_full(j & 1), (j >> 1) & 1);
    const uint32_t k_a = kv_s + (j & 1) * C::KV_STAGE_BYTES, v_a = k_a + C::NCB * C::BLOCK_BYTES;
    // ---- S = Q K^T
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < C::DPK / 16; ++k) {
      const uint32_t off = (uint32_t)((k * 16) / 64) * C::BLOCK_BYTES + (uint32_t)((k * 16) % 64) * 2;
      wgmma_m64n64(s, gmma_desc_sw128(q_s + off), gmma_desc_sw128(k_a + off), k != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    const int kbase = j * BKV;
    if (kbase + BKV > p.nk) {                    // keys beyond nk (last tile only)
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (kbase + 8 * (i >> 2) + 2 * q4 + (i & 1) >= p.nk) s[i] = -INFINITY;
    }
    // ---- online softmax (row h = 0: registers with (i >> 1) even, h = 1: odd)
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = m[h];
#pragma unroll
      for (int i = 2 * h; i < 32; i += 4) mx = fmaxf(mx, fmaxf(s[i], s[i + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      alpha[h] = fast_exp2((m[h] - mx) * sc);    // exp2(-inf) = 0 on the first tile
      m[h] = mx;
      const float ms = mx * sc;
      float rs = 0.f;
#pragma unroll
      for (int i = 2 * h; i < 32; i += 4) {
        s[i] = fast_exp2(fmaf(s[i], sc, -ms));
        s[i + 1] = fast_exp2(fmaf(s[i + 1], sc, -ms));
        rs += s[i] + s[i + 1];
      }
      l[h] = fmaf(l[h], alpha[h], rs);
    }
#pragma unroll
    for (int i = 0; i < C::OREG; ++i) o[i] *= alpha[(i >> 1) & 1];
    // ---- O += P V: P (fp16) as the register A operand, 16 keys per instruction.  All of P is packed before the fence,
    // so no register the wgmmas read is written between them.
    uint32_t a[BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) a[kk][r] = pack_h2(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      const uint32_t v_rows = v_a + kk * 16 * 128;
      wgmma_m64n64_rs<1>(o, a[kk], gmma_desc_sw128_mn(v_rows, C::BLOCK_BYTES), 1u);
      if (D > 64) wgmma_m64n16_rs<1>(o + 32, a[kk], gmma_desc_sw128_mn(v_rows + C::BLOCK_BYTES, C::BLOCK_BYTES), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
  }
  // ---- epilogue: O / l -> fp16 -> HBM
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
  }
  const float inv[2] = {1.f / l[0], 1.f / l[1]};
  const int r0 = q0 + 16 * warp + (lane >> 2);
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
    const uint32_t box[4] = {64, 1, (uint32_t)BKV, 1};
    if (make_tmap_f16(&a.tmK, k, 4, dims, strk, box, 1)) return 3;
    if (make_tmap_f16(&a.tmV, v, 4, dims, strv, box, 1)) return 3;
  }
  a.o = o; a.ldo = ldo; a.o_bs = o_bs; a.nq = nq; a.nk = nk; a.kv_div = kv_div;
  a.scale_log2 = 1.4426950408889634f / sqrtf((float)D);
  ProfScope prof(st, PC_ATTN, 4.0 * batch * heads * (double)nq * nk * D, 1, nq, nk, D);
  dim3 grid((nq + TQ - 1) / TQ, heads, batch);
  return launch_pdl(attn_tc_kernel<D>, grid, dim3(ATT_THREADS), C::SMEM, st, 1, a);
}

}  // namespace

// Returns -1 when the shape is not handled by the wgmma kernel (caller uses the mma.sync kernel).
int attention_tc(cudaStream_t st, const __half* q, int ldq, const __half* k, int ldk, const __half* v, int ldv, __half* o,
                 int ldo, int batch, int nq, int nk, int heads, int d, long long q_bs, long long kv_bs, long long o_bs,
                 int kv_div) {
  if ((ldq % 8) || (ldk % 8) || (ldv % 8) || (ldo % 2)) return -1;
  if ((q_bs % 8) || (kv_bs % 8)) return -1;
  if (d == 40) return launch<40>(st, q, ldq, k, ldk, v, ldv, o, ldo, batch, nq, nk, heads, q_bs, kv_bs, o_bs, kv_div);
  if (d == 80) return launch<80>(st, q, ldq, k, ldk, v, ldv, o, ldo, batch, nq, nk, heads, q_bs, kv_bs, o_bs, kv_div);
  return -1;
}

}  // namespace vs
