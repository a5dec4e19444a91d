// CLIP text encoder (SD-1.5's CLIPTextModel, transformers modeling_clip.py) on sm_90a: the two kernels it needs beyond the
// GEMM (with its quick-GELU epilogue, gemm.cu) and ln_kernel (norm.cu).
//  * clip_embed_kernel:   x[s, t, :] = fp16(fp32(tok[ids[s, t]]) + fp32(pos[t]))  (CLIPTextEmbeddings.forward), one
//                         rounding like torch's fp16 add, 16-byte vectors.
//  * causal_attn_kernel:  one CTA per (sequence, head) of CLIPAttention with the causal mask, q / k / v read straight
//                         from the fused QKV GEMM output.  L <= 77 keys fit one tile, so the softmax is exact (row
//                         maximum, exp2, sum, normalise) rather than online.  mma.sync.m16n8k16 with fp32 accumulators:
//                         a 77 x 77 x 64 head is far below wgmma's 64-row granularity and the whole encode is bound by
//                         launch latency.
#include "common.cuh"
#include "kernels.h"

namespace vs {
namespace {

// the mma.sync / ldmatrix wrappers of attention.cu (that file keeps its own copies so its code stays as it is)
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

// ------------------------------------------------------------------------------------------------ embedding
// One thread per 8 channels of one token.  An id outside [0, vocab) (the host rejects them before the launch) writes NaN
// instead of reading outside the table.
__global__ void clip_embed_kernel(const int* __restrict__ ids, int L, long long n_vec, int cv, const __half* __restrict__ tok,
                                  int vocab, const __half* __restrict__ pos, __half* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_vec) return;
  const long long row = i / cv;                 // token index s * L + t
  const int c = (int)(i % cv);
  const int t = (int)(row % L);
  const int id = __ldg(ids + row);
  uint4 o;
  __half2* oh = reinterpret_cast<__half2*>(&o);
  if (id < 0 || id >= vocab) {
    const __half2 nan2 = __half2half2(__ushort_as_half(0x7e00));
    for (int j = 0; j < 4; ++j) oh[j] = nan2;
  } else {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(tok + (long long)id * cv * 8) + c);
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(pos + (long long)t * cv * 8) + c);
    const __half2* ah = reinterpret_cast<const __half2*>(&a);
    const __half2* bh = reinterpret_cast<const __half2*>(&b);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 x = __half22float2(ah[j]), y = __half22float2(bh[j]);
      oh[j] = __floats2half2_rn(x.x + y.x, x.y + y.y);
    }
  }
  reinterpret_cast<uint4*>(out)[i] = o;
}

// ------------------------------------------------------------------------------------------------ causal attention
constexpr int CA_D = 64;                        // head dim (CLIP ViT-L/14 text tower: 768 / 12)
constexpr int CA_ROWS = 80;                     // 5 warps x 16 query rows >= 77 tokens; also the padded key count
constexpr int CA_WARPS = CA_ROWS / 16;
constexpr int CA_LDS = CA_D + 8;                // halves per shared row (conflict-free ldmatrix)
constexpr int CA_NT = CA_ROWS / 8;              // n8 key tiles of S
constexpr int CA_ON = CA_D / 8;                 // n8 channel tiles of O

struct CausalParams {
  const __half* qkv; __half* o;
  int ldqkv, ldo, L, C;
  float sc;                                     // log2(e) / sqrt(d), applied in fp32
};

// CTA (blockIdx.x = sequence, blockIdx.y = head): q, k, v of rows 0 .. L - 1 from the fused QKV output [n L, ldqkv]
// (q at column h d, k at C + h d, v at 2 C + h d), rows L .. 79 zero in shared memory.  Warp w computes the 16 query rows
// 16 w .. 16 w + 15: S = Q K^T, keys j > i or j >= L set to -inf BEFORE the row maximum (a masked probability is exactly
// 0), p = exp2(s sc - max sc), l = sum p in fp32, O = fp16(p) V, out = O / l.  Only rows < L are stored.
__global__ void __launch_bounds__(CA_WARPS * 32) causal_attn_kernel(const CausalParams p) {
  __shared__ __align__(16) __half sq[CA_ROWS * CA_LDS];
  __shared__ __align__(16) __half sk[CA_ROWS * CA_LDS];
  __shared__ __align__(16) __half sv[CA_ROWS * CA_LDS];
  pdl_trigger();
  pdl_wait();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int L = p.L;
  const long long row0 = (long long)blockIdx.x * L;
  const int col = blockIdx.y * CA_D;
  constexpr int CH = CA_D / 8;                  // 16-byte chunks per row
  for (int i = tid; i < 3 * CA_ROWS * CH; i += CA_WARPS * 32) {
    const int m = i / (CA_ROWS * CH), r = (i / CH) % CA_ROWS, c = i % CH;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r < L) v = __ldg(reinterpret_cast<const uint4*>(p.qkv + (row0 + r) * p.ldqkv + m * p.C + col) + c);
    __half* dst = (m == 0 ? sq : m == 1 ? sk : sv) + r * CA_LDS + c * 8;
    *reinterpret_cast<uint4*>(dst) = v;
  }
  __syncthreads();
  if (16 * warp >= L) return;                   // no query row of this warp is stored

  constexpr int LDSB = CA_LDS * 2;
  const uint32_t q_s = smem_u32(sq) + warp * 16 * LDSB, k_s = smem_u32(sk), v_s = smem_u32(sv);
  float s[CA_NT][4];
#pragma unroll
  for (int n = 0; n < CA_NT; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < CA_D / 16; ++kk) {
    uint32_t a[4];
    ldsm_x4(q_s + (lane & 15) * LDSB + (kk * 16 + (lane >> 4) * 8) * 2, a[0], a[1], a[2], a[3]);
#pragma unroll
    for (int n = 0; n < CA_NT; n += 2) {
      uint32_t b0, b1, b2, b3;
      const int key = n * 8 + (lane & 7) + ((lane >> 4) ? 8 : 0);
      const int ch = kk * 16 + (((lane >> 3) & 1) ? 8 : 0);
      ldsm_x4(k_s + key * LDSB + ch * 2, b0, b1, b2, b3);
      mma16816(s[n], a, b0, b1);
      mma16816(s[n + 1], a, b2, b3);
    }
  }
  // rows of this thread: r0 (accumulators 0, 1) and r0 + 8 (2, 3); key j is visible to row i iff j <= i and j < L.  Key 0
  // is visible to every row, so the maximum is finite.
  const int r0 = 16 * warp + (lane >> 2), r1 = r0 + 8;
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int n = 0; n < CA_NT; ++n) {
    const int c = n * 8 + (lane & 3) * 2;
    if (c > r0 || c >= L) s[n][0] = -INFINITY;
    if (c + 1 > r0 || c + 1 >= L) s[n][1] = -INFINITY;
    if (c > r1 || c >= L) s[n][2] = -INFINITY;
    if (c + 1 > r1 || c + 1 >= L) s[n][3] = -INFINITY;
    mx0 = fmaxf(mx0, fmaxf(s[n][0], s[n][1]));
    mx1 = fmaxf(mx1, fmaxf(s[n][2], s[n][3]));
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  const float ms0 = mx0 * p.sc, ms1 = mx1 * p.sc;
  float l0 = 0.f, l1 = 0.f;
#pragma unroll
  for (int n = 0; n < CA_NT; ++n) {
    s[n][0] = exp2f(s[n][0] * p.sc - ms0);      // exp2(-inf) = 0: masked keys carry exactly no weight
    s[n][1] = exp2f(s[n][1] * p.sc - ms0);
    s[n][2] = exp2f(s[n][2] * p.sc - ms1);
    s[n][3] = exp2f(s[n][3] * p.sc - ms1);
    l0 += s[n][0] + s[n][1];
    l1 += s[n][2] + s[n][3];
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);

  // O = P V with the fp16 probabilities as the register A operand (the S accumulator layout is the A fragment layout)
  float o[CA_ON][4];
#pragma unroll
  for (int n = 0; n < CA_ON; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
#pragma unroll
  for (int kt = 0; kt < CA_NT / 2; ++kt) {
    uint32_t a[4];
    a[0] = pack_h2(s[2 * kt][0], s[2 * kt][1]);
    a[1] = pack_h2(s[2 * kt][2], s[2 * kt][3]);
    a[2] = pack_h2(s[2 * kt + 1][0], s[2 * kt + 1][1]);
    a[3] = pack_h2(s[2 * kt + 1][2], s[2 * kt + 1][3]);
#pragma unroll
    for (int n = 0; n < CA_ON; n += 2) {
      uint32_t b0, b1, b2, b3;
      const int key = kt * 16 + (lane & 7) + (((lane >> 3) & 1) ? 8 : 0);
      const int ch = n * 8 + ((lane >> 4) ? 8 : 0);
      ldsm_x4_t(v_s + key * LDSB + ch * 2, b0, b1, b2, b3);
      mma16816(o[n], a, b0, b1);
      mma16816(o[n + 1], a, b2, b3);
    }
  }
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  __half* op = p.o + row0 * p.ldo + col;
#pragma unroll
  for (int n = 0; n < CA_ON; ++n) {
    const int c = n * 8 + (lane & 3) * 2;
    if (r0 < L) *reinterpret_cast<__half2*>(op + (long long)r0 * p.ldo + c) = __floats2half2_rn(o[n][0] * i0, o[n][1] * i0);
    if (r1 < L) *reinterpret_cast<__half2*>(op + (long long)r1 * p.ldo + c) = __floats2half2_rn(o[n][2] * i1, o[n][3] * i1);
  }
}

}  // namespace

int clip_embed(cudaStream_t st, const int* ids, int n, int L, const __half* tok, int vocab, const __half* pos, int C,
               __half* out) {
  VS_REQUIRE(ids && tok && pos && out, "clip_embed: null pointer");
  VS_REQUIRE(n >= 1 && L >= 1 && vocab >= 1 && C >= 8 && C % 8 == 0, "clip_embed: bad shape (n %d, L %d, vocab %d, C %d)",
             n, L, vocab, C);
  VS_REQUIRE(((reinterpret_cast<uintptr_t>(tok) | reinterpret_cast<uintptr_t>(pos) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
             "clip_embed: tables and output must be 16-byte aligned");
  const long long n_vec = (long long)n * L * (C / 8);
  ProfScope prof(st, PC_OTHER, 6.0 * (double)n * L * C);   // bytes: token row + position row read, output written
  return launch_pdl(clip_embed_kernel, dim3((unsigned)((n_vec + 255) / 256)), dim3(256), 0, st, 1, ids, L, n_vec, C / 8, tok,
                    vocab, pos, out);
}

int causal_attention(cudaStream_t st, const __half* qkv, int ldqkv, __half* o, int ldo, int nseq, int L, int heads, int d) {
  VS_REQUIRE(qkv && o, "causal_attention: null pointer");
  VS_REQUIRE(d == CA_D, "causal_attention: head dim %d (supported: %d)", d, CA_D);
  VS_REQUIRE(nseq >= 1 && heads >= 1 && L >= 1 && L <= 77, "causal_attention: bad shape (nseq %d, L %d, heads %d; 1 <= L <= 77)",
             nseq, L, heads);
  VS_REQUIRE(ldqkv >= 3 * heads * d && ldqkv % 8 == 0 && ldo >= heads * d && ldo % 2 == 0,
             "causal_attention: leading dims %d / %d do not fit %d heads of %d", ldqkv, ldo, heads, d);
  VS_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(o) & 3) == 0,
             "causal_attention: unaligned pointers");
  const CausalParams p{qkv, o, ldqkv, ldo, L, heads * d, 1.4426950408889634f / sqrtf((float)d)};
  ProfScope prof(st, PC_ATTN, 4.0 * nseq * heads * (double)L * L * d);
  return launch_pdl(causal_attn_kernel, dim3((unsigned)nseq, (unsigned)heads), dim3(CA_WARPS * 32), 0, st, 1, p);
}

}  // namespace vs
