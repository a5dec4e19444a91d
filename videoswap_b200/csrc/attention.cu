// Attention kernels, v1: flash-attention-2 style streaming softmax on mma.sync.m16n8k16 (fp16 in, fp32 accumulate).
//  * attention():           spatial self-attention (N x N, d = 40/80/160) and cross-attention (N x 77) --
//                           replaces diffusers AttnProcessor2_0 / EDLoRA_AttnProcessor.__call__
//                           (reference utils/edlora_util.py:47-65, models/animatediff_models/attention.py:229-241).
//  * temporal_attention():  attention across the F frames of every pixel (motion_module.py:305-335), one warp per
//                           (batch, pixel, head); probabilities never touch HBM and no '(b f) d c <-> (b d) f c'
//                           transposes are materialised.
// These are the legacy-tensor-path (HMMA) baseline kernels; the wgmma version (attention_tc.cu) replaces the spatial one for d = 40 / 80.
#include "common.cuh"
#include "kernels.h"

namespace vs {
namespace {

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool pred) {
  const int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// One warp: S[16 x 8*NT] = Q[16 x DP] K[8*NT x DP]^T.  q_s / k_s: shared addresses of row 0, row stride LDS bytes.
template <int DP, int NT>
__device__ __forceinline__ void warp_qk(float (*s)[4], uint32_t q_s, uint32_t k_s, int lds_bytes, int lane) {
#pragma unroll
  for (int n = 0; n < NT; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < DP / 16; ++kk) {
    uint32_t a[4];
    ldsm_x4(q_s + (lane & 15) * lds_bytes + (kk * 16 + (lane >> 4) * 8) * 2, a[0], a[1], a[2], a[3]);
#pragma unroll
    for (int n = 0; n < NT; n += 2) {
      uint32_t b0, b1, b2, b3;
      const int key = n * 8 + (lane & 7) + ((lane >> 4) ? 8 : 0);
      const int ch = kk * 16 + (((lane >> 3) & 1) ? 8 : 0);
      ldsm_x4(k_s + key * lds_bytes + ch * 2, b0, b1, b2, b3);
      mma16816(s[n], a, b0, b1);
      mma16816(s[n + 1], a, b2, b3);
    }
  }
}

// One warp: O[16 x 8*ON] += P[16 x 8*NT] V[8*NT x 8*ON]; P comes from the S accumulators (already exponentiated).
template <int NT, int ON>
__device__ __forceinline__ void warp_pv(float (*o)[4], const float (*s)[4], uint32_t v_s, int lds_bytes, int lane) {
#pragma unroll
  for (int kt = 0; kt < NT / 2; ++kt) {
    uint32_t a[4];
    a[0] = pack_h2(s[2 * kt][0], s[2 * kt][1]);
    a[1] = pack_h2(s[2 * kt][2], s[2 * kt][3]);
    a[2] = pack_h2(s[2 * kt + 1][0], s[2 * kt + 1][1]);
    a[3] = pack_h2(s[2 * kt + 1][2], s[2 * kt + 1][3]);
#pragma unroll
    for (int n = 0; n < ON; n += 2) {
      uint32_t b0, b1, b2, b3;
      const int key = kt * 16 + (lane & 7) + (((lane >> 3) & 1) ? 8 : 0);
      const int ch = n * 8 + ((lane >> 4) ? 8 : 0);
      ldsm_x4_t(v_s + key * lds_bytes + ch * 2, b0, b1, b2, b3);
      mma16816(o[n], a, b0, b1);
      mma16816(o[n + 1], a, b2, b3);
    }
  }
}

// ================================================================================================ spatial / cross
struct AttnParams {
  const __half* q; const __half* k; const __half* v; __half* o;
  int ldq, ldk, ldv, ldo;
  long long q_bs, kv_bs, o_bs;
  int nq, nk, kv_div;
  float scale_log2;
};

template <int D>
struct ACfg {
  static constexpr int DP = (D + 15) / 16 * 16;
  static constexpr int LDS = DP + 8;           // halves per smem row (conflict-free ldmatrix)
  static constexpr int BQ = 64, BKV = 64;
  static constexpr int SMEM = (BQ + 4 * BKV) * LDS * 2;
};

template <int D>
__device__ __forceinline__ void load_rows(uint32_t dst, const __half* src, int ld, int row0, int nrows_valid, int tid,
                                          int nthreads) {
  using C = ACfg<D>;
  constexpr int CH = C::DP / 8;  // 16-byte chunks per row
  for (int i = tid; i < 64 * CH; i += nthreads) {
    const int r = i / CH, c = i % CH;
    const bool ok = (row0 + r < nrows_valid) && (c * 8 < D);
    const __half* s = ok ? src + (long long)(row0 + r) * ld + c * 8 : src;
    cp_async16(dst + (r * C::LDS + c * 8) * 2, s, ok);
  }
}

template <int D>
__global__ void __launch_bounds__(128) attn_kernel(const AttnParams p) {
  using C = ACfg<D>;
  pdl_trigger();
  pdl_wait();
  constexpr int DP = C::DP, LDSB = C::LDS * 2, NT = C::BKV / 8, ON = DP / 8;
  extern __shared__ __align__(16) uint8_t smem[];
  const uint32_t q_s = smem_u32(smem);
  const uint32_t k_s0 = q_s + C::BQ * LDSB;
  const uint32_t v_s0 = k_s0 + 2 * C::BKV * LDSB;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const __half* qp = p.q + b * p.q_bs + h * D;
  const __half* kp = p.k + (b / p.kv_div) * p.kv_bs + h * D;
  const __half* vp = p.v + (b / p.kv_div) * p.kv_bs + h * D;
  const int nkt = (p.nk + C::BKV - 1) / C::BKV;

  load_rows<D>(q_s, qp, p.ldq, qt * C::BQ, p.nq, tid, 128);
  load_rows<D>(k_s0, kp, p.ldk, 0, p.nk, tid, 128);
  load_rows<D>(v_s0, vp, p.ldv, 0, p.nk, tid, 128);
  cp_async_commit();

  float o[ON][4];
#pragma unroll
  for (int n = 0; n < ON; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  for (int j = 0; j < nkt; ++j) {
    cp_async_wait<0>();
    __syncthreads();
    if (j + 1 < nkt) {  // prefetch the next K/V tile into the other buffer (free: every warp is past tile j-1)
      const int nb = (j + 1) & 1;
      load_rows<D>(k_s0 + nb * C::BKV * LDSB, kp, p.ldk, (j + 1) * C::BKV, p.nk, tid, 128);
      load_rows<D>(v_s0 + nb * C::BKV * LDSB, vp, p.ldv, (j + 1) * C::BKV, p.nk, tid, 128);
      cp_async_commit();
    }
    const uint32_t k_s = k_s0 + (j & 1) * C::BKV * LDSB;
    const uint32_t v_s = v_s0 + (j & 1) * C::BKV * LDSB;
    float s[NT][4];
    warp_qk<DP, NT>(s, q_s + warp * 16 * LDSB, k_s, LDSB, lane);
    // mask keys beyond nk (last tile only)
    const int kbase = j * C::BKV;
    if (kbase + C::BKV > p.nk) {
#pragma unroll
      for (int n = 0; n < NT; ++n) {
        const int c = kbase + n * 8 + (lane & 3) * 2;
        if (c >= p.nk) s[n][0] = s[n][2] = -INFINITY;
        if (c + 1 >= p.nk) s[n][1] = s[n][3] = -INFINITY;
      }
    }
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      mx0 = fmaxf(mx0, fmaxf(s[n][0], s[n][1]));
      mx1 = fmaxf(mx1, fmaxf(s[n][2], s[n][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float c0 = exp2f((m0 - mx0) * p.scale_log2), c1 = exp2f((m1 - mx1) * p.scale_log2);
    m0 = mx0; m1 = mx1;
    const float ms0 = mx0 * p.scale_log2, ms1 = mx1 * p.scale_log2;
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      s[n][0] = exp2f(s[n][0] * p.scale_log2 - ms0);
      s[n][1] = exp2f(s[n][1] * p.scale_log2 - ms0);
      s[n][2] = exp2f(s[n][2] * p.scale_log2 - ms1);
      s[n][3] = exp2f(s[n][3] * p.scale_log2 - ms1);
      rs0 += s[n][0] + s[n][1];
      rs1 += s[n][2] + s[n][3];
    }
    l0 = l0 * c0 + rs0;
    l1 = l1 * c1 + rs1;
#pragma unroll
    for (int n = 0; n < ON; ++n) {
      o[n][0] *= c0; o[n][1] *= c0; o[n][2] *= c1; o[n][3] *= c1;
    }
    warp_pv<NT, ON>(o, s, v_s, LDSB, lane);
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  const int r0 = qt * C::BQ + warp * 16 + (lane >> 2), r1 = r0 + 8;
  __half* op = p.o + b * p.o_bs + h * D;
#pragma unroll
  for (int n = 0; n < ON; ++n) {
    const int c = n * 8 + (lane & 3) * 2;
    if (c < D) {
      if (r0 < p.nq) *reinterpret_cast<__half2*>(op + (long long)r0 * p.ldo + c) = __floats2half2_rn(o[n][0] * i0, o[n][1] * i0);
      if (r1 < p.nq) *reinterpret_cast<__half2*>(op + (long long)r1 * p.ldo + c) = __floats2half2_rn(o[n][2] * i1, o[n][3] * i1);
    }
  }
}

template <int D>
int launch_attn(cudaStream_t st, const AttnParams& p, int batch, int heads) {
  using C = ACfg<D>;
  static bool configured = false;
  if (!configured) {
    VS_CHECK_CUDA(cudaFuncSetAttribute(attn_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
    configured = true;
  }
  dim3 grid((p.nq + C::BQ - 1) / C::BQ, heads, batch);
  ProfScope prof(st, PC_ATTN, 4.0 * batch * heads * (double)p.nq * p.nk * D);
  return launch_pdl(attn_kernel<D>, grid, dim3(128), C::SMEM, st, 1, p);
}

// ================================================================================================ explicit probabilities
// The prompt-to-prompt controllers of the reference (utils/p2p_utils/attention_register.py:96,140-150) need the softmax
// probabilities of the small-resolution layers (queries < 32^2) as a tensor [b, h, s, t] they can store and edit between
// softmax and P V.  Two kernels: probabilities to HBM (two sweeps over K: row max / sum, then the normalised values), and
// O = P V from (possibly edited) probabilities.  Only the 16x16 / 8x8 levels run here (12 of the 32 attention calls, 0.3 %
// of the step's FLOPs), so these are plain mma.sync kernels.
template <int D>
__global__ void __launch_bounds__(128) attn_probs_kernel(const AttnParams p, __half* __restrict__ probs, int heads) {
  using C = ACfg<D>;
  constexpr int DP = C::DP, LDSB = C::LDS * 2, NT = C::BKV / 8;
  extern __shared__ __align__(16) uint8_t smem[];
  const uint32_t q_s = smem_u32(smem);
  const uint32_t k_s0 = q_s + C::BQ * LDSB;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const __half* qp = p.q + b * p.q_bs + h * D;
  const __half* kp = p.k + (b / p.kv_div) * p.kv_bs + h * D;
  const int nkt = (p.nk + C::BKV - 1) / C::BKV;
  load_rows<D>(q_s, qp, p.ldq, qt * C::BQ, p.nq, tid, 128);
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f, i0 = 0.f, i1 = 0.f;
  const int r0 = qt * C::BQ + warp * 16 + (lane >> 2), r1 = r0 + 8;
  __half* prow0 = probs + (((long long)b * heads + h) * p.nq + r0) * p.nk;
  __half* prow1 = prow0 + 8LL * p.nk;
  for (int pass = 0; pass < 2; ++pass) {
    load_rows<D>(k_s0, kp, p.ldk, 0, p.nk, tid, 128);
    cp_async_commit();
    for (int j = 0; j < nkt; ++j) {
      cp_async_wait<0>();
      __syncthreads();
      if (j + 1 < nkt) {
        load_rows<D>(k_s0 + ((j + 1) & 1) * C::BKV * LDSB, kp, p.ldk, (j + 1) * C::BKV, p.nk, tid, 128);
        cp_async_commit();
      }
      float s[NT][4];
      warp_qk<DP, NT>(s, q_s + warp * 16 * LDSB, k_s0 + (j & 1) * C::BKV * LDSB, LDSB, lane);
      const int kbase = j * C::BKV;
      if (pass == 0) {
        float mx0 = m0, mx1 = m1;
#pragma unroll
        for (int n = 0; n < NT; ++n) {
          const int c = kbase + n * 8 + (lane & 3) * 2;
          if (c >= p.nk) s[n][0] = s[n][2] = -INFINITY;
          if (c + 1 >= p.nk) s[n][1] = s[n][3] = -INFINITY;
          mx0 = fmaxf(mx0, fmaxf(s[n][0], s[n][1]));
          mx1 = fmaxf(mx1, fmaxf(s[n][2], s[n][3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
        for (int n = 0; n < NT; ++n) {
          rs0 += exp2f((s[n][0] - mx0) * p.scale_log2) + exp2f((s[n][1] - mx0) * p.scale_log2);
          rs1 += exp2f((s[n][2] - mx1) * p.scale_log2) + exp2f((s[n][3] - mx1) * p.scale_log2);
        }
        l0 = l0 * exp2f((m0 - mx0) * p.scale_log2) + rs0;
        l1 = l1 * exp2f((m1 - mx1) * p.scale_log2) + rs1;
        m0 = mx0; m1 = mx1;
      } else {
#pragma unroll
        for (int n = 0; n < NT; ++n) {
          const int c = kbase + n * 8 + (lane & 3) * 2;
          if (r0 < p.nq) {
            if (c < p.nk) prow0[c] = __float2half_rn(exp2f((s[n][0] - m0) * p.scale_log2) * i0);
            if (c + 1 < p.nk) prow0[c + 1] = __float2half_rn(exp2f((s[n][1] - m0) * p.scale_log2) * i0);
          }
          if (r1 < p.nq) {
            if (c < p.nk) prow1[c] = __float2half_rn(exp2f((s[n][2] - m1) * p.scale_log2) * i1);
            if (c + 1 < p.nk) prow1[c + 1] = __float2half_rn(exp2f((s[n][3] - m1) * p.scale_log2) * i1);
          }
        }
      }
      __syncthreads();               // every warp is done with this K buffer before the next sweep / prefetch reuses it
    }
    if (pass == 0) {
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
      l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
      i0 = 1.f / l0; i1 = 1.f / l1;
    }
  }
}

// O[b, q, h*D] = sum_k P[b, h, q, k] V[b / kv_div, k, h*D]   (P fp16 [b, h, nq, nk] row-major)
template <int D>
__global__ void __launch_bounds__(128) attn_pv_kernel(const AttnParams p, const __half* __restrict__ probs, int heads) {
  using C = ACfg<D>;
  constexpr int DP = C::DP, LDSB = C::LDS * 2, ON = DP / 8, LDP = C::BKV + 8, LDPB = LDP * 2;
  extern __shared__ __align__(16) uint8_t smem[];
  const uint32_t p_s = smem_u32(smem);                       // [64 queries][64 keys] fp16, padded rows
  const uint32_t v_s = p_s + C::BQ * LDPB;                   // [64 keys][DP]
  __half* p_sm = reinterpret_cast<__half*>(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const __half* vp = p.v + (b / p.kv_div) * p.kv_bs + h * D;
  const __half* pb = probs + (((long long)b * heads + h) * p.nq) * p.nk;
  const int nkt = (p.nk + C::BKV - 1) / C::BKV;
  float o[ON][4];
#pragma unroll
  for (int n = 0; n < ON; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  for (int j = 0; j < nkt; ++j) {
    __syncthreads();                                         // previous tile consumed
    load_rows<D>(v_s, vp, p.ldv, j * C::BKV, p.nk, tid, 128);
    cp_async_commit();
    for (int e = tid; e < C::BQ * C::BKV; e += 128) {        // P tile (nk may be odd: scalar loads), zero beyond the problem
      const int r = e / C::BKV, c = e % C::BKV;
      const int q = qt * C::BQ + r, k = j * C::BKV + c;
      p_sm[r * LDP + c] = (q < p.nq && k < p.nk) ? pb[(long long)q * p.nk + k] : __float2half(0.f);
    }
    cp_async_wait<0>();
    __syncthreads();
#pragma unroll
    for (int kt = 0; kt < C::BKV / 16; ++kt) {
      uint32_t a[4];
      ldsm_x4(p_s + (warp * 16 + (lane & 15)) * LDPB + (kt * 16 + (lane >> 4) * 8) * 2, a[0], a[1], a[2], a[3]);
#pragma unroll
      for (int n = 0; n < ON; n += 2) {
        uint32_t b0, b1, b2, b3;
        const int key = kt * 16 + (lane & 7) + (((lane >> 3) & 1) ? 8 : 0);
        const int ch = n * 8 + ((lane >> 4) ? 8 : 0);
        ldsm_x4_t(v_s + key * LDSB + ch * 2, b0, b1, b2, b3);
        mma16816(o[n], a, b0, b1);
        mma16816(o[n + 1], a, b2, b3);
      }
    }
  }
  const int r0 = qt * C::BQ + warp * 16 + (lane >> 2), r1 = r0 + 8;
  __half* op = p.o + b * p.o_bs + h * D;
#pragma unroll
  for (int n = 0; n < ON; ++n) {
    const int c = n * 8 + (lane & 3) * 2;
    if (c < D) {
      if (r0 < p.nq) *reinterpret_cast<__half2*>(op + (long long)r0 * p.ldo + c) = __floats2half2_rn(o[n][0], o[n][1]);
      if (r1 < p.nq) *reinterpret_cast<__half2*>(op + (long long)r1 * p.ldo + c) = __floats2half2_rn(o[n][2], o[n][3]);
    }
  }
}

template <int D>
int launch_explicit(cudaStream_t st, const AttnParams& p, __half* probs, int batch, int heads, bool apply) {
  using C = ACfg<D>;
  constexpr int SMEM_P = (C::BQ + 2 * C::BKV) * C::LDS * 2;
  constexpr int SMEM_V = C::BQ * (C::BKV + 8) * 2 + C::BKV * C::LDS * 2;
  static bool configured = false;
  if (!configured) {
    VS_CHECK_CUDA(cudaFuncSetAttribute(attn_probs_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_P));
    VS_CHECK_CUDA(cudaFuncSetAttribute(attn_pv_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_V));
    configured = true;
  }
  dim3 grid((p.nq + C::BQ - 1) / C::BQ, heads, batch);
  ProfScope prof(st, PC_ATTN, 2.0 * batch * heads * (double)p.nq * p.nk * D);
  if (apply) attn_pv_kernel<D><<<grid, 128, SMEM_V, st>>>(p, probs, heads);
  else attn_probs_kernel<D><<<grid, 128, SMEM_P, st>>>(p, probs, heads);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ================================================================================================ temporal
struct TAttnParams {
  const __half* qkv; __half* o;
  int B, F, HW, C, heads;
  float scale_log2;
  long long items;
};

template <int D, int FP, bool VST = true>   // FP = frames padded to 16 or 32; VST: outputs staged in shared memory, 16-byte stores
__global__ void __launch_bounds__(128) tattn_kernel(const TAttnParams p) {
  pdl_trigger();
  pdl_wait();
  constexpr int DP = (D + 15) / 16 * 16, LDS = DP + 8, LDSB = LDS * 2, CH = DP / 8;
  constexpr int MT = FP / 16, NT = FP / 8, ON = DP / 8;
  extern __shared__ __align__(16) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long item = (long long)blockIdx.x * 4 + warp;
  if (item >= p.items) return;   // whole warp exits together; no block-level sync below
  const int head = item % p.heads;
  const long long bp = item / p.heads;
  const int pix = bp % p.HW;
  const int b = bp / p.HW;
  const uint32_t base = smem_u32(smem) + warp * (3 * FP * LDSB);
  const uint32_t q_s = base, k_s = base + FP * LDSB, v_s = base + 2 * FP * LDSB;
  const long long row_stride = (long long)p.HW * 3 * p.C;   // between frames
  const __half* src = p.qkv + ((long long)b * p.F * p.HW + pix) * 3 * p.C + head * D;
  for (int i = lane; i < 3 * FP * CH; i += 32) {
    const int sec = i / (FP * CH), rem = i % (FP * CH), f = rem / CH, c = rem % CH;
    const bool ok = (f < p.F) && (c * 8 < D);
    const __half* s = ok ? src + f * row_stride + sec * p.C + c * 8 : src;
    cp_async16(base + sec * FP * LDSB + (f * LDS + c * 8) * 2, s, ok);
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncwarp();
  __half* dst = p.o + ((long long)b * p.F * p.HW + pix) * p.C + head * D;
  const long long orow = (long long)p.HW * p.C;
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
    float s[NT][4];
    warp_qk<DP, NT>(s, q_s + mt * 16 * LDSB, k_s, LDSB, lane);
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      const int c = n * 8 + (lane & 3) * 2;
      if (c >= p.F) s[n][0] = s[n][2] = -INFINITY;
      if (c + 1 >= p.F) s[n][1] = s[n][3] = -INFINITY;
      mx0 = fmaxf(mx0, fmaxf(s[n][0], s[n][1]));
      mx1 = fmaxf(mx1, fmaxf(s[n][2], s[n][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float ms0 = mx0 * p.scale_log2, ms1 = mx1 * p.scale_log2;
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      s[n][0] = exp2f(s[n][0] * p.scale_log2 - ms0);
      s[n][1] = exp2f(s[n][1] * p.scale_log2 - ms0);
      s[n][2] = exp2f(s[n][2] * p.scale_log2 - ms1);
      s[n][3] = exp2f(s[n][3] * p.scale_log2 - ms1);
      l0 += s[n][0] + s[n][1];
      l1 += s[n][2] + s[n][3];
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    float o[ON][4];
#pragma unroll
    for (int n = 0; n < ON; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    warp_pv<NT, ON>(o, s, v_s, LDSB, lane);
    const float i0 = 1.f / l0, i1 = 1.f / l1;
    const int f0 = mt * 16 + (lane >> 2), f1 = f0 + 8;
    if (VST) {
      // the 16 query rows of this m-tile were read (ldmatrix, above) by this warp only and are dead now: stage the outputs
      // there and write each 80 / 160 / 320-byte head row with 16-byte stores instead of 4-byte fragments
      __syncwarp();
      __half* stage = reinterpret_cast<__half*>(smem) + (size_t)warp * (3 * FP * LDS) + (size_t)mt * 16 * LDS;
#pragma unroll
      for (int n = 0; n < ON; ++n) {
        const int c = n * 8 + (lane & 3) * 2;
        *reinterpret_cast<__half2*>(stage + (lane >> 2) * LDS + c) = __floats2half2_rn(o[n][0] * i0, o[n][1] * i0);
        *reinterpret_cast<__half2*>(stage + ((lane >> 2) + 8) * LDS + c) = __floats2half2_rn(o[n][2] * i1, o[n][3] * i1);
      }
      __syncwarp();
      constexpr int VCH = D / 8;                       // 16-byte chunks per head row
      for (int e = lane; e < 16 * VCH; e += 32) {
        const int fr = e / VCH, ch = e % VCH, f = mt * 16 + fr;
        if (f < p.F) *reinterpret_cast<uint4*>(dst + f * orow + ch * 8) = *reinterpret_cast<const uint4*>(stage + fr * LDS + ch * 8);
      }
    } else {
#pragma unroll
      for (int n = 0; n < ON; ++n) {
        const int c = n * 8 + (lane & 3) * 2;
        if (c < D) {
          if (f0 < p.F) *reinterpret_cast<__half2*>(dst + f0 * orow + c) = __floats2half2_rn(o[n][0] * i0, o[n][1] * i0);
          if (f1 < p.F) *reinterpret_cast<__half2*>(dst + f1 * orow + c) = __floats2half2_rn(o[n][2] * i1, o[n][3] * i1);
        }
      }
    }
  }
}

template <int D, int FP>
int launch_tattn(cudaStream_t st, const TAttnParams& p) {
  constexpr int DP = (D + 15) / 16 * 16;
  constexpr int SMEM = 4 * 3 * FP * (DP + 8) * 2;
  static bool configured = false;
  if (!configured) {
    VS_CHECK_CUDA(cudaFuncSetAttribute(tattn_kernel<D, FP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    VS_CHECK_CUDA(cudaFuncSetAttribute(tattn_kernel<D, FP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    configured = true;
  }
  const long long blocks = (p.items + 3) / 4;
  ProfScope prof(st, PC_TATTN, 8.0 * p.B * p.F * (double)p.HW * p.C);   // bytes: read 3C + write C fp16 per token
  if (get_option("tattn_vst") == 0) return launch_pdl(tattn_kernel<D, FP, false>, dim3((unsigned)blocks), dim3(128), SMEM, st, 1, p);
  return launch_pdl(tattn_kernel<D, FP, true>, dim3((unsigned)blocks), dim3(128), SMEM, st, 1, p);
}

}  // namespace

int attention(cudaStream_t st, const __half* q, int ldq, const __half* k, int ldk, const __half* v, int ldv, __half* o,
              int ldo, int batch, int nq, int nk, int heads, int d, long long q_bstride, long long kv_bstride,
              long long o_bstride, int kv_div) {
  VS_REQUIRE(nq > 0 && nk > 0 && batch > 0, "attention: empty problem");
  VS_REQUIRE((ldq % 8 | ldk % 8 | ldv % 8 | ldo % 2) == 0 && d % 8 == 0, "attention: unaligned leading dims");
  if (get_option("attn_tc") && (d == 40 || d == 80)) {
    const int e = attention_tc(st, q, ldq, k, ldk, v, ldv, o, ldo, batch, nq, nk, heads, d, q_bstride, kv_bstride, o_bstride,
                               kv_div > 0 ? kv_div : 1);
    if (e != -1) return e;
  }
  AttnParams p{q, k, v, o, ldq, ldk, ldv, ldo, q_bstride, kv_bstride, o_bstride, nq, nk, kv_div > 0 ? kv_div : 1,
               1.4426950408889634f / sqrtf((float)d)};
  switch (d) {
    case 40: return launch_attn<40>(st, p, batch, heads);
    case 80: return launch_attn<80>(st, p, batch, heads);
    case 160: return launch_attn<160>(st, p, batch, heads);
    default: VS_REQUIRE(false, "attention: unsupported head dim %d (supported: 40, 80, 160)", d);
  }
}

// Explicit-probability path (attention controllers): probs [batch, heads, nq, nk] fp16 in HBM.
int attention_probs(cudaStream_t st, const __half* q, int ldq, const __half* k, int ldk, __half* probs, int batch, int nq, int nk,
                    int heads, int d, long long q_bstride, long long kv_bstride, int kv_div) {
  VS_REQUIRE(nq > 0 && nk > 0 && batch > 0 && probs, "attention_probs: empty problem");
  VS_REQUIRE((ldq % 8 | ldk % 8) == 0 && d % 8 == 0, "attention_probs: unaligned leading dims");
  AttnParams p{q, k, nullptr, nullptr, ldq, ldk, 0, 0, q_bstride, kv_bstride, 0, nq, nk, kv_div > 0 ? kv_div : 1,
               1.4426950408889634f / sqrtf((float)d)};
  switch (d) {
    case 40: return launch_explicit<40>(st, p, probs, batch, heads, false);
    case 80: return launch_explicit<80>(st, p, probs, batch, heads, false);
    case 160: return launch_explicit<160>(st, p, probs, batch, heads, false);
    default: VS_REQUIRE(false, "attention_probs: unsupported head dim %d (supported: 40, 80, 160)", d);
  }
}
int attention_apply_probs(cudaStream_t st, const __half* probs, const __half* v, int ldv, __half* o, int ldo, int batch, int nq,
                          int nk, int heads, int d, long long kv_bstride, long long o_bstride, int kv_div) {
  VS_REQUIRE(nq > 0 && nk > 0 && batch > 0 && probs, "attention_apply_probs: empty problem");
  VS_REQUIRE((ldv % 8 | ldo % 2) == 0 && d % 8 == 0, "attention_apply_probs: unaligned leading dims");
  AttnParams p{nullptr, nullptr, v, o, 0, 0, ldv, ldo, 0, kv_bstride, o_bstride, nq, nk, kv_div > 0 ? kv_div : 1, 0.f};
  switch (d) {
    case 40: return launch_explicit<40>(st, p, const_cast<__half*>(probs), batch, heads, true);
    case 80: return launch_explicit<80>(st, p, const_cast<__half*>(probs), batch, heads, true);
    case 160: return launch_explicit<160>(st, p, const_cast<__half*>(probs), batch, heads, true);
    default: VS_REQUIRE(false, "attention_apply_probs: unsupported head dim %d (supported: 40, 80, 160)", d);
  }
}

int temporal_attention(cudaStream_t st, const __half* qkv, __half* o, int B, int F, int HW, int C, int heads) {
  VS_REQUIRE(F >= 1 && F <= 32, "temporal_attention: F=%d out of range (1..32)", F);
  VS_REQUIRE(C % heads == 0, "temporal_attention: C %% heads != 0");
  const int d = C / heads;
  TAttnParams p{qkv, o, B, F, HW, C, heads, 1.4426950408889634f / sqrtf((float)d), (long long)B * HW * heads};
  const bool big = F > 16;
  switch (d) {
    case 40: return big ? launch_tattn<40, 32>(st, p) : launch_tattn<40, 16>(st, p);
    case 80: return big ? launch_tattn<80, 32>(st, p) : launch_tattn<80, 16>(st, p);
    case 160: return big ? launch_tattn<160, 32>(st, p) : launch_tattn<160, 16>(st, p);
    default: VS_REQUIRE(false, "temporal_attention: unsupported head dim %d", d);
  }
}

}  // namespace vs
