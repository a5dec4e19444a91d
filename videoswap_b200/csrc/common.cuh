// Shared device/host helpers for the sm_90a kernels: error handling, mbarrier / TMA / wgmma PTX wrappers.
// Hand-written inline PTX; no CUTLASS dependency.
#pragma once
#include <cuda.h>          // CUtensorMap (types only; the driver entry point is fetched at run time)
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace vs {

// ------------------------------------------------------------------------------------------------ host side
void set_error(const char* fmt, ...);
const char* last_error();

#define VS_CHECK_CUDA(expr)                                                                         \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) {                                                                        \
      vs::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return 1;                                                                                     \
    }                                                                                               \
  } while (0)

#define VS_REQUIRE(cond, ...)                \
  do {                                       \
    if (!(cond)) {                           \
      vs::set_error(__VA_ARGS__);            \
      return 2;                              \
    }                                        \
  } while (0)

// Encodes a tiled TMA descriptor over fp16 data.  dims/strides innermost first; strides in BYTES for dims 1..rank-1.
int make_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box, int swizzle /* 0 none, 1 = 128B, 2 = 64B, 3 = 32B */);

int num_sms();
int get_option(const char* name);

#ifdef __CUDACC__
// Launches `kernel` with the programmatic-stream-serialization attribute (see pdl_wait() below) and, for cluster_x > 1,
// a cluster dimension.  Only for kernels that call pdl_wait() before their first global-memory access.
template <typename... KArgs, typename... Args>
int launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (get_option("pdl") != 0) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  VS_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...));
  return 0;
}
#endif

// profiling categories (work = algorithmic FLOPs for tensor kernels, algorithmic bytes for HBM-bound kernels)
enum ProfCat { PC_GEMM = 0, PC_CONV = 1, PC_ATTN = 2, PC_TATTN = 3, PC_GROUPNORM = 4, PC_LAYERNORM = 5, PC_OTHER = 6, PC_COUNT = 7 };
struct ProfScope {
  ProfScope(cudaStream_t st, int cat, double work, int nlaunch = 1, long long m = 0, int n = 0, int k = 0);
  ~ProfScope();
  cudaStream_t st_; int idx_;
};
void prof_enable(bool on);
void prof_reset();
int prof_collect(int cat, double* ms, double* work, long long* count);
int prof_dump(const char* path);   // per-(category, shape) aggregate of the recorded launches as CSV
long long launch_count();
void count_launch(int n);

// ------------------------------------------------------------------------------------------------ device side
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug must trap (-> CUDA error at the next sync) instead of hanging the GPU.
// No printf here: a call anywhere in a kernel makes ptxas serialise every wgmma of that kernel (warning C7510).
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  // try_wait suspends the thread in hardware for a bounded time, so this loop iterates every ~100 cycles; the watchdog
  // counts iterations (2^25 of them is seconds) instead of reading the clock on the hot path
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 25)) __trap();
  }
}

__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// Plain (non-tensor) bulk copy of `bytes` contiguous bytes; src, dst and bytes are multiples of 16.
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// One lane of a fully converged warp.  The single-issuer roles (TMA producers) run their loops with
// the WHOLE warp and predicate only the issuing instructions on this, so that addresses / descriptors stay warp-uniform
// (uniform registers) instead of being re-broadcast through ELECT / VOTE / R2UR sequences inside a divergent branch.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- thread-block clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of `addr` (a shared::cta address of this CTA) in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---- programmatic dependent launch.  A kernel launched with launch_pdl() may start while its predecessor in the stream
// is still draining: everything before pdl_wait() (barrier init, descriptor prefetch) overlaps the
// predecessor's tail; pdl_wait() returns once the predecessor grid has completed and its memory is visible, so NO global
// memory may be read or written before it.  pdl_trigger() lets the successor start being scheduled.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- warpgroup register reallocation: a producer warpgroup that only issues TMA hands registers to the MMA warpgroups
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ---- wgmma (sm_90a warpgroup MMA): D[registers] (+)= A[smem desc] * B[smem desc], fp16 in, fp32 accumulate
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Shared-memory matrix descriptor of a K-major operand with 128-byte swizzle: rows are 128 B (64 fp16) apart inside an
// 8-row swizzle atom, atoms are SBO = 1024 B apart.  Advancing K by 16 elements adds 2 (32 bytes) to the address field.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);   // start address, 16-byte units
  d |= (uint64_t)1 << 16;                        // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset between 8-row groups
  d |= (uint64_t)1 << 62;                        // layout type: SWIZZLE_128B
  return d;
}
// MN-major operand with 128-byte swizzle (e.g. V [keys][64 channels] as the B operand of P V): 8-key groups are
// SBO = 1024 B apart, 64-channel column blocks LBO apart.
__device__ __forceinline__ uint64_t gmma_desc_sw128_mn(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

#define VS_R8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
// m64nNk16 with both operands K-major in shared memory: one instruction for the full width of a tile, N / 2 fp32
// accumulators per thread.  Register i holds row 16 w + lane / 4 + 8 ((i >> 1) & 1) of the warpgroup's 64 rows (w = warp
// in the warpgroup) and column 8 (i >> 2) + 2 (lane & 3) + (i & 1).
template <int N>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t da, uint64_t db, uint32_t scale_d);
#define VS_REGS_0_31 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
#define VS_REGS_32_63 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
#define VS_REGS_64_79 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79"
#define VS_REGS_80_127 "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
// N, accumulator operand list, operand numbers of da / db / scale_d (= N / 2 ...), accumulator constraints
#define VS_WGMMA_SS(N, REGS, IA, IB, IS, ...)                                                                     \
  template <>                                                                                                     \
  __device__ __forceinline__ void wgmma_ss<N>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {           \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #IS ", 0;\n\t"                                         \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 {" REGS "}, %" #IA ", %" #IB ", p, 1, 1, 0, 0;\n\t}" \
                 : __VA_ARGS__                                                                                    \
                 : "l"(da), "l"(db), "r"(scale_d));                                                               \
  }
VS_WGMMA_SS(64, VS_REGS_0_31, 32, 33, 34, VS_R8(0), VS_R8(8), VS_R8(16), VS_R8(24))
VS_WGMMA_SS(128, VS_REGS_0_31 "," VS_REGS_32_63, 64, 65, 66, VS_R8(0), VS_R8(8), VS_R8(16), VS_R8(24), VS_R8(32), VS_R8(40),
            VS_R8(48), VS_R8(56))
VS_WGMMA_SS(160, VS_REGS_0_31 "," VS_REGS_32_63 "," VS_REGS_64_79, 80, 81, 82, VS_R8(0), VS_R8(8), VS_R8(16), VS_R8(24),
            VS_R8(32), VS_R8(40), VS_R8(48), VS_R8(56), VS_R8(64), VS_R8(72))
VS_WGMMA_SS(256, VS_REGS_0_31 "," VS_REGS_32_63 "," VS_REGS_64_79 "," VS_REGS_80_127, 128, 129, 130, VS_R8(0), VS_R8(8),
            VS_R8(16), VS_R8(24), VS_R8(32), VS_R8(40), VS_R8(48), VS_R8(56), VS_R8(64), VS_R8(72), VS_R8(80), VS_R8(88),
            VS_R8(96), VS_R8(104), VS_R8(112), VS_R8(120))
#undef VS_WGMMA_SS
#undef VS_REGS_0_31
#undef VS_REGS_32_63
#undef VS_REGS_64_79
#undef VS_REGS_80_127
template <int TB = 0>
__device__ __forceinline__ void wgmma_m64n16(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, %11;\n\t}"
      : VS_R8(0)
      : "l"(da), "l"(db), "r"(scale_d), "n"(TB));
}
// A from registers (four fp16x2 per thread in the m16n8k16 A-fragment layout of each warp's 16 rows), B from smem;
// tnspB (TB) = 1: B is MN-major.
template <int TB = 0>
__device__ __forceinline__ void wgmma_m64n64_rs(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "{%32,%33,%34,%35}, %36, p, 1, 1, %38;\n\t}"
      : VS_R8(0), VS_R8(8), VS_R8(16), VS_R8(24)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB));
}
template <int TB = 0>
__device__ __forceinline__ void wgmma_m64n16_rs(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1, %14;\n\t}"
      : VS_R8(0)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB));
}
#undef VS_R8

__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.f + __expf(-x)); }   // 2 MUFU + 3 FP32
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
// Exact-erf GELU with erf from Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7, far below fp16 resolution):
// erf(z) = 1 - (a1 t + a2 t^2 + ... + a5 t^5) exp(-z^2), t = 1 / (1 + p z), z >= 0.  Two MUFU ops + ~12 FP32 ops.
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.f)));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * z * z));
  const float erf_abs = fmaf(-poly, e, 1.f);           // erf(|x| / sqrt 2)
  const float erf_s = copysignf(erf_abs, x);
  return 0.5f * x * (1.f + erf_s);
}
// erf-GELU in logistic form, x * Phi(x) = x / (1 + 2^(-x q(x^2))): q is a cubic in x^2 fitted (minimax, |x| <= 5, argument
// clamped beyond) to log2(Phi / (1 - Phi)) / x.  |error| <= 1.2e-5 + 2^-20 |x| over all x -- below the fp16 rounding of
// the result for |gelu| > 0.02 -- at 2 MUFU + 9 FP32 instructions (gelu_erf_fast: 2 MUFU + ~16); used by the GEGLU GEMM
// epilogue, whose instruction count bounds the K = 320 feed-forward GEMM.  The numerator is clamped at -5 too: beyond
// it 1 + e is ~1.5e6, so an unclamped x would return x / 1.5e6 (-0.04 at x = -65504) instead of ~0.
__device__ __forceinline__ float gelu_sig(float x) {
  const float xn = fmaxf(x, -5.f);
  const float xc = fminf(xn, 5.f);
  const float u = xc * xc;
  float q = fmaf(u, 2.47135360e-05f, 7.37690930e-04f);      // coefficients negated: t = -x q(x^2)
  q = fmaf(q, u, -1.05988323e-01f);
  q = fmaf(q, u, -2.30164247e+00f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(xc * q));
  return __fdividef(xn, 1.f + e);
}
// CLIP's quick_gelu, v sigmoid(1.702 v) = v / (1 + 2^t) with t = -1.702 log2(e) v clamped at 64: for v < -26 the true
// value is below 2e-18 and v / (1 + 2^64) is below 4e-15, both 0 in fp16; without the clamp 2^t overflows for v < -52.
// Relative error <= 2^-21 + 2^-23 |t| <= 2^-16.9 (ex2.approx, the fp32 rounding of t, the approximate division).
__device__ __forceinline__ float quick_gelu_f(float v) {
  const float t = fminf(-2.4554669595930157f * v, 64.f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
  return __fdividef(v, 1.f + e);
}
#endif  // __CUDACC__

}  // namespace vs
