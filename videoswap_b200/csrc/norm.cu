// HBM-bound normalisation kernels (NHWC fp16 in/out, fp32 statistics):
//  * GroupNorm(32) statistics + apply(+SiLU).  A "statistics set" is `imgs_per_set` consecutive images: the
//    reference's ResnetBlock3D / conv_norm_out GroupNorm runs on the 5-D [B,C,F,H,W] tensor, so its statistics
//    span all F frames of a batch element (resnet.py:166,177; unet.py:474), whereas Transformer3DModel.norm and the
//    motion-module norm are per frame (attention.py:108, motion_module.py:146).  The input may be a *virtual*
//    channel concat of two tensors (skip connections, unet_blocks.py:618,720): the concat is never materialised
//    un-normalised.
//  * LayerNorm over C with an optional temporal sinusoidal positional encoding added after the norm
//    (motion_module.py:224-228,294).
// Every thread owns a fixed 8-channel vector (16-byte loads) and walks pixels, so per-channel parameters stay in
// registers; reductions are warp shuffle -> shared atomics -> one global atomic per (block, group).
#include "common.cuh"
#include "kernels.h"

namespace vs {
namespace {

struct GnParams {
  const __half* x1; const __half* x2; int c1, c2;
  int C, CV;                 // total channels, 8-channel vectors per pixel
  int hw, imgs_per_set, groups, cpg;
  long long pix_per_set;     // imgs_per_set * hw
  float* sums;               // [nstat, groups, 2]
  const float* gamma; const float* beta; float eps; int silu;
  int count_scale;           // the sums cover count_scale x the local elements (frame shards, after the all-reduce)
  __half* out;
  int rows_per_block;        // pixel rows in flight per block (blockDim.x = CV * rows_per_block)
  int pix_per_block;
};

__device__ __forceinline__ uint4 gn_load(const GnParams& p, long long pix, int cv) {
  const int c = cv * 8;
  if (c < p.c1) return *reinterpret_cast<const uint4*>(p.x1 + pix * p.c1 + c);
  return *reinterpret_cast<const uint4*>(p.x2 + pix * p.c2 + (c - p.c1));
}

// V2: eight per-position (sum, sum of squares) accumulators without predicates (3 instructions per element instead of ~10
// for the per-element group select of V1, whose issue slots -- 64 % active -- bounded the pass); the group split is applied
// once per thread at the end.
template <bool V2>
__global__ void gn_stats_kernel(const GnParams p) {
  extern __shared__ float sh[];   // [groups][2]
  for (int i = threadIdx.x; i < p.groups * 2; i += blockDim.x) sh[i] = 0.f;
  __syncthreads();
  pdl_trigger();
  pdl_wait();
  const int set = blockIdx.y;
  const int cv = threadIdx.x % p.CV, r = threadIdx.x / p.CV;
  const int ga = (cv * 8) / p.cpg, gb = (cv * 8 + 7) / p.cpg;
  const int split = (ga == gb) ? 8 : (gb * p.cpg - cv * 8);   // first `split` channels belong to group ga
  float sa = 0.f, qa = 0.f, sb = 0.f, qb = 0.f;
  float ps[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, pq[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const long long p0 = (long long)blockIdx.x * p.pix_per_block;
  const long long p1 = min(p0 + p.pix_per_block, p.pix_per_set);
  const long long base = (long long)set * p.pix_per_set;
  auto accum = [&](const uint4& v) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      if (V2) {
        ps[2 * j] += f.x; pq[2 * j] = fmaf(f.x, f.x, pq[2 * j]);
        ps[2 * j + 1] += f.y; pq[2 * j + 1] = fmaf(f.y, f.y, pq[2 * j + 1]);
      } else {
        if (2 * j < split) { sa += f.x; qa += f.x * f.x; } else { sb += f.x; qb += f.x * f.x; }
        if (2 * j + 1 < split) { sa += f.y; qa += f.y * f.y; } else { sb += f.y; qb += f.y * f.y; }
      }
    }
  };
  long long i = p0 + r;
  const long long step = p.rows_per_block;
  for (; i + 3 * step < p1; i += 4 * step) {       // 4 independent 16-byte loads in flight per thread
    const uint4 v0 = gn_load(p, base + i, cv), v1 = gn_load(p, base + i + step, cv);
    const uint4 v2 = gn_load(p, base + i + 2 * step, cv), v3 = gn_load(p, base + i + 3 * step, cv);
    accum(v0); accum(v1); accum(v2); accum(v3);
  }
  for (; i < p1; i += step) accum(gn_load(p, base + i, cv));
  if (V2) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (j < split) { sa += ps[j]; qa += pq[j]; } else { sb += ps[j]; qb += pq[j]; }
    }
  }
  atomicAdd(&sh[ga * 2], sa);
  atomicAdd(&sh[ga * 2 + 1], qa);
  if (gb != ga) {
    atomicAdd(&sh[gb * 2], sb);
    atomicAdd(&sh[gb * 2 + 1], qb);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < p.groups * 2; i += blockDim.x) atomicAdd(&p.sums[(long long)set * p.groups * 2 + i], sh[i]);
}

__global__ void gn_apply_kernel(const GnParams p) {
  pdl_trigger();
  pdl_wait();
  const int set = blockIdx.y;
  const int cv = threadIdx.x % p.CV, r = threadIdx.x / p.CV;
  float a[8], b[8];
  const float inv_n = 1.f / ((float)p.pix_per_set * p.cpg * (float)p.count_scale);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = cv * 8 + j;
    const int g = c / p.cpg;
    const float s = p.sums[((long long)set * p.groups + g) * 2], q = p.sums[((long long)set * p.groups + g) * 2 + 1];
    const float mean = s * inv_n;
    const float var = fmaxf(q * inv_n - mean * mean, 0.f);
    const float rstd = rsqrtf(var + p.eps);
    a[j] = rstd * p.gamma[c];
    b[j] = p.beta[c] - mean * a[j];
  }
  const long long p0 = (long long)blockIdx.x * p.pix_per_block;
  const long long p1 = min(p0 + p.pix_per_block, p.pix_per_set);
  const long long base = (long long)set * p.pix_per_set;
  auto apply = [&](const uint4& v, long long pix) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      float y0 = f.x * a[2 * j] + b[2 * j], y1 = f.y * a[2 * j + 1] + b[2 * j + 1];
      if (p.silu) { y0 = silu_f(y0); y1 = silu_f(y1); }
      oh[j] = __floats2half2_rn(y0, y1);
    }
    *reinterpret_cast<uint4*>(p.out + pix * p.C + cv * 8) = o;
  };
  long long i = p0 + r;
  const long long step = p.rows_per_block;
  for (; i + 3 * step < p1; i += 4 * step) {
    const uint4 v0 = gn_load(p, base + i, cv), v1 = gn_load(p, base + i + step, cv);
    const uint4 v2 = gn_load(p, base + i + 2 * step, cv), v3 = gn_load(p, base + i + 3 * step, cv);
    apply(v0, base + i); apply(v1, base + i + step); apply(v2, base + i + 2 * step); apply(v3, base + i + 3 * step);
  }
  for (; i < p1; i += step) apply(gn_load(p, base + i, cv), base + i);
}

// ---------------------------------------------------------------------------------------------- per-frame GroupNorm, one pass
// Transformer3DModel.norm / the motion module's norm (attention.py:108, motion_module.py:146) normalise every frame on its
// own: one image is 2.6 MB at the 64x64 level, 1.3 MB / 0.66 MB / 0.16 MB below -- it fits the shared memory of a thread-block
// CLUSTER (16 / 8 / 4 / 1 CTAs x 164 KB).  So each image is read ONCE: the CTAs of a cluster stage their pixel slices in
// shared memory while accumulating (sum, sum of squares) per group, exchange the 64 partial sums through distributed shared
// memory (ld.shared::cluster) between two cluster barriers, and normalise straight from shared memory.  Replaces the
// statistics kernel + apply kernel pair (two reads, two launches, global atomics) for 36 of the 81 GroupNorms; deterministic
// (fixed summation order).
constexpr int kGnFusedThreads = 480;          // CV * rows with CV = C / 8 in {40, 80, 160}: 12 / 6 / 3 pixel rows
__global__ void __launch_bounds__(kGnFusedThreads, 1) gn_frame_fused_kernel(const GnParams p, int ncta, int ppc) {
  extern __shared__ __align__(16) uint8_t gsm[];
  float* part = reinterpret_cast<float*>(gsm);                   // [64]: this CTA's (sum, sumsq) per group
  float* tot = part + 64;                                         // [64]: cluster totals
  uint4* tile = reinterpret_cast<uint4*>(gsm + 512);              // [ppc][CV] 16-byte vectors
  const int rank = (int)cluster_ctarank();
  const int img = blockIdx.x / ncta;
  const int cv = threadIdx.x % p.CV, r = threadIdx.x / p.CV, rows = blockDim.x / p.CV;
  if (threadIdx.x < 64) part[threadIdx.x] = 0.f;
  __syncthreads();
  pdl_trigger();
  pdl_wait();
  const int ga = (cv * 8) / p.cpg, gb = (cv * 8 + 7) / p.cpg;
  const int split = (ga == gb) ? 8 : (gb * p.cpg - cv * 8);
  const uint4* src = reinterpret_cast<const uint4*>(p.x1) + ((long long)img * p.hw + (long long)rank * ppc) * p.CV + cv;
  float ps[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, pq[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  auto accum = [&](const uint4& v) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      ps[2 * j] += f.x; pq[2 * j] = fmaf(f.x, f.x, pq[2 * j]);
      ps[2 * j + 1] += f.y; pq[2 * j + 1] = fmaf(f.y, f.y, pq[2 * j + 1]);
    }
  };
  int i = r;
  for (; i + 3 * rows < ppc; i += 4 * rows) {                     // 4 independent 16-byte loads in flight per thread
    const uint4 v0 = src[(long long)i * p.CV], v1 = src[(long long)(i + rows) * p.CV];
    const uint4 v2 = src[(long long)(i + 2 * rows) * p.CV], v3 = src[(long long)(i + 3 * rows) * p.CV];
    tile[i * p.CV + cv] = v0; tile[(i + rows) * p.CV + cv] = v1; tile[(i + 2 * rows) * p.CV + cv] = v2; tile[(i + 3 * rows) * p.CV + cv] = v3;
    accum(v0); accum(v1); accum(v2); accum(v3);
  }
  for (; i < ppc; i += rows) {
    const uint4 v = src[(long long)i * p.CV];
    tile[i * p.CV + cv] = v;
    accum(v);
  }
  float sa = 0.f, qa = 0.f, sb = 0.f, qb = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (j < split) { sa += ps[j]; qa += pq[j]; } else { sb += ps[j]; qb += pq[j]; }
  }
  atomicAdd(&part[ga * 2], sa);
  atomicAdd(&part[ga * 2 + 1], qa);
  if (gb != ga) {
    atomicAdd(&part[gb * 2], sb);
    atomicAdd(&part[gb * 2 + 1], qb);
  }
  __syncthreads();
  if (ncta > 1) cluster_sync_all();                               // every CTA's partial sums are complete
  if (threadIdx.x < 64) {
    float t = 0.f;
    if (ncta > 1) {
      const uint32_t mine = smem_u32(&part[threadIdx.x]);
      for (int c = 0; c < ncta; ++c) {                             // fixed order: deterministic
        float v;
        asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(mapa_shared(mine, (uint32_t)c)));
        t += v;
      }
    } else {
      t = part[threadIdx.x];
    }
    tot[threadIdx.x] = t;
  }
  __syncthreads();
  float a[8], b[8];
  const float inv_n = 1.f / ((float)p.hw * p.cpg);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = cv * 8 + j;
    const int g = c / p.cpg;
    const float mean = tot[g * 2] * inv_n;
    const float var = fmaxf(tot[g * 2 + 1] * inv_n - mean * mean, 0.f);
    const float rstd = rsqrtf(var + p.eps);
    a[j] = rstd * p.gamma[c];
    b[j] = p.beta[c] - mean * a[j];
  }
  uint4* dst = reinterpret_cast<uint4*>(p.out) + ((long long)img * p.hw + (long long)rank * ppc) * p.CV + cv;
  for (i = r; i < ppc; i += rows) {
    const uint4 v = tile[i * p.CV + cv];
    const __half2* h = reinterpret_cast<const __half2*>(&v);
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      float y0 = f.x * a[2 * j] + b[2 * j], y1 = f.y * a[2 * j + 1] + b[2 * j + 1];
      if (p.silu) { y0 = silu_f(y0); y1 = silu_f(y1); }
      oh[j] = __floats2half2_rn(y0, y1);
    }
    dst[(long long)i * p.CV] = o;
  }
  if (ncta > 1) cluster_sync_all();                               // nobody leaves while a peer may still read its partial sums
}

int gn_fill(GnParams& p, dim3& grid, int& threads, const __half* x1, int c1, const __half* x2, int c2, int nimg, int hw,
            int imgs_per_set, int groups) {
  const int C = c1 + c2;
  VS_REQUIRE(x1 && c1 > 0 && (c2 == 0 || x2), "groupnorm: bad inputs");
  VS_REQUIRE(c1 % 8 == 0 && c2 % 8 == 0, "groupnorm: channel counts must be multiples of 8 (got %d, %d)", c1, c2);
  VS_REQUIRE(C % groups == 0 && (C / groups) >= 8, "groupnorm: needs >= 8 channels per group (C=%d groups=%d)", C, groups);
  VS_REQUIRE(nimg % imgs_per_set == 0, "groupnorm: nimg %% imgs_per_set != 0");
  VS_REQUIRE(C / 8 <= 1024, "groupnorm: too many channels");
  p.x1 = x1; p.x2 = x2; p.c1 = c1; p.c2 = c2; p.C = C; p.CV = C / 8;
  p.hw = hw; p.imgs_per_set = imgs_per_set; p.groups = groups; p.cpg = C / groups;
  p.pix_per_set = (long long)imgs_per_set * hw;
  int rows = 512 / p.CV;
  if (rows < 1) rows = 1;
  p.rows_per_block = rows;
  threads = p.CV * rows;
  const int nstat = nimg / imgs_per_set;
  // enough blocks to cover the machine ~4x, at least 8 pixel rows per thread
  long long want = (4LL * num_sms() + nstat - 1) / nstat;
  long long ppb = (p.pix_per_set + want - 1) / want;
  const long long min_ppb = (long long)rows * 8;
  if (ppb < min_ppb) ppb = min_ppb;
  p.pix_per_block = (int)ppb;
  grid = dim3((unsigned)((p.pix_per_set + ppb - 1) / ppb), nstat, 1);
  return 0;
}

// ------------------------------------------------------------------------------------------------ LayerNorm
template <int VPL>   // uint4 vectors per lane; C = 8 * (number of vectors), vectors strided by 32 over the warp
__global__ void ln_kernel(const __half* __restrict__ x, int rows, int C, const float* __restrict__ gamma,
                          const float* __restrict__ beta, const float* __restrict__ pe, int hw, int F,
                          __half* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const int nvec = C / 8;
  const __half* xr = x + (long long)warp * C;
  uint4 v[VPL];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      v[i] = *reinterpret_cast<const uint4*>(xr + vi * 8);
      const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h[j]); s += f.x + f.y; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        q += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / C + 1e-5f);
  const float* per = pe ? pe + (long long)((warp / hw) % F) * C : nullptr;
  __half* orow = out + (long long)warp * C;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
      uint4 o;
      __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = vi * 8 + 2 * j;
        const float2 f = __half22float2(h[j]);
        float y0 = (f.x - mean) * rstd * gamma[c] + beta[c];
        float y1 = (f.y - mean) * rstd * gamma[c + 1] + beta[c + 1];
        if (per) { y0 += per[c]; y1 += per[c + 1]; }
        oh[j] = __floats2half2_rn(y0, y1);
      }
      *reinterpret_cast<uint4*>(orow + vi * 8) = o;
    }
  }
}

// Fast path for C = 40 * LPR (320 / 640 / 1280): LPR lanes share a row, every lane owns five 16-byte vectors, so a
// warp normalises 32/LPR rows at once with all lanes busy; persistent grid-stride over row groups; gamma/beta live in
// registers as packed fp16 (they are fp16 model weights, so this is exact).
template <int LPR>
__global__ void __launch_bounds__(256) ln5_kernel(const __half* __restrict__ x, long long rows, const float* __restrict__ gamma,
                                                  const float* __restrict__ beta, const float* __restrict__ pe, int hw, int F,
                                                  __half* __restrict__ out) {
  constexpr int C = LPR * 40, RPW = 32 / LPR;
  const int lane = threadIdx.x & 31, sub = lane % LPR, rw = lane / LPR;
  __half2 g2[5][4], b2[5][4];
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    const int c = (sub + i * LPR) * 8;
    const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c)), gb = __ldg(reinterpret_cast<const float4*>(gamma + c + 4));
    const float4 ba = __ldg(reinterpret_cast<const float4*>(beta + c)), bb = __ldg(reinterpret_cast<const float4*>(beta + c + 4));
    g2[i][0] = __floats2half2_rn(ga.x, ga.y); g2[i][1] = __floats2half2_rn(ga.z, ga.w);
    g2[i][2] = __floats2half2_rn(gb.x, gb.y); g2[i][3] = __floats2half2_rn(gb.z, gb.w);
    b2[i][0] = __floats2half2_rn(ba.x, ba.y); b2[i][1] = __floats2half2_rn(ba.z, ba.w);
    b2[i][2] = __floats2half2_rn(bb.x, bb.y); b2[i][3] = __floats2half2_rn(bb.z, bb.w);
  }
  pdl_trigger();
  pdl_wait();          // gamma / beta above are weights (not produced by the previous kernel)
  const long long warp_global = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  // Two row groups per iteration (2 x 5 independent 16-byte loads in flight per thread) hide the HBM latency that the
  // shuffle reductions would otherwise expose.
  for (long long r0 = warp_global * (2 * RPW); r0 < rows; r0 += nwarps * (2 * RPW)) {
    long long row[2];
    bool active[2];
    uint4 v[2][5];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      row[u] = r0 + u * RPW + rw;
      active[u] = row[u] < rows;
      const __half* xr = x + (active[u] ? row[u] : 0) * C;
#pragma unroll
      for (int i = 0; i < 5; ++i) v[u][i] = *reinterpret_cast<const uint4*>(xr + (sub + i * LPR) * 8);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const __half2* h = reinterpret_cast<const __half2*>(&v[u][i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h[j]); s += f.x + f.y; }
      }
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mean = s * (1.f / C);
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const __half2* h = reinterpret_cast<const __half2*>(&v[u][i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h[j]);
          q += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
        }
      }
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const float rstd = rsqrtf(q * (1.f / C) + 1e-5f);
      if (!active[u]) continue;
      const float* per = pe ? pe + (long long)((row[u] / hw) % F) * C : nullptr;
      __half* orow = out + row[u] * C;
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const int c = (sub + i * LPR) * 8;
        const __half2* h = reinterpret_cast<const __half2*>(&v[u][i]);
        float pv[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (per) {
          const float4 pa = __ldg(reinterpret_cast<const float4*>(per + c)), pb = __ldg(reinterpret_cast<const float4*>(per + c + 4));
          pv[0] = pa.x; pv[1] = pa.y; pv[2] = pa.z; pv[3] = pa.w; pv[4] = pb.x; pv[5] = pb.y; pv[6] = pb.z; pv[7] = pb.w;
        }
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h[j]);
          const float2 gg = __half22float2(g2[i][j]), bb = __half22float2(b2[i][j]);
          const float y0 = (f.x - mean) * rstd * gg.x + bb.x + pv[2 * j];
          const float y1 = (f.y - mean) * rstd * gg.y + bb.y + pv[2 * j + 1];
          oh[j] = __floats2half2_rn(y0, y1);
        }
        *reinterpret_cast<uint4*>(orow + c) = o;
      }
    }
  }
}

// Row statistics only, for a LayerNorm that is folded into the following GEMM (gemm.cu, EPI_F_LN): reads the row once,
// writes (rstd, -mean * rstd); the normalised tensor is never materialised.  Same lane layout as ln5_kernel.
template <int LPR>
__global__ void __launch_bounds__(256) ln_stats_kernel(const __half* __restrict__ x, long long rows, float2* __restrict__ stats) {
  constexpr int C = LPR * 40, RPW = 32 / LPR;
  const int lane = threadIdx.x & 31, sub = lane % LPR, rw = lane / LPR;
  pdl_trigger();
  pdl_wait();
  const long long warp_global = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r0 = warp_global * (2 * RPW); r0 < rows; r0 += nwarps * (2 * RPW)) {
    uint4 v[2][5];
    long long row[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      row[u] = r0 + u * RPW + rw;
      const __half* xr = x + (row[u] < rows ? row[u] : 0) * C;
#pragma unroll
      for (int i = 0; i < 5; ++i) v[u][i] = *reinterpret_cast<const uint4*>(xr + (sub + i * LPR) * 8);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const __half2* h = reinterpret_cast<const __half2*>(&v[u][i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h[j]); s += f.x + f.y; }
      }
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mean = s * (1.f / C);
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const __half2* h = reinterpret_cast<const __half2*>(&v[u][i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h[j]);
          q += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
        }
      }
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const float rstd = rsqrtf(q * (1.f / C) + 1e-5f);
      if (sub == 0 && row[u] < rows) stats[row[u]] = make_float2(rstd, -mean * rstd);
    }
  }
}

}  // namespace

bool ln_fold_supported(int C) { return C == 320 || C == 640 || C == 1280; }

int ln_rowstats(cudaStream_t st, const __half* x, long long rows, int C, float* stats) {
  VS_REQUIRE(ln_fold_supported(C), "ln_rowstats: unsupported C=%d", C);
  const int lpr = C / 40, rpw = 32 / lpr;
  long long need = (rows + rpw * 8 * 4 - 1) / (rpw * 8 * 4);
  if (need < 1) need = 1;
  const long long cap = (long long)num_sms() * 8;
  const int grid = (int)(need < cap ? need : cap);
  ProfScope prof(st, PC_LAYERNORM, 2.0 * rows * (double)C, 1, rows, C, 2);
  float2* s2 = reinterpret_cast<float2*>(stats);
  if (lpr == 8) return launch_pdl(ln_stats_kernel<8>, dim3(grid), dim3(256), 0, st, 1, x, rows, s2);
  if (lpr == 16) return launch_pdl(ln_stats_kernel<16>, dim3(grid), dim3(256), 0, st, 1, x, rows, s2);
  return launch_pdl(ln_stats_kernel<32>, dim3(grid), dim3(256), 0, st, 1, x, rows, s2);
}

// Single-pass per-frame GroupNorm (see gn_frame_fused_kernel).  Returns -1 when the shape does not fit (caller falls back to
// the statistics + apply pair): one source tensor, C / 8 dividing 480 threads, an image slice per CTA <= 164 KB with a
// cluster of <= 16 CTAs.
int groupnorm_frame_fused(cudaStream_t st, const __half* x, int C, int nimg, int hw, int groups, float eps, const float* gamma,
                          const float* beta, bool silu, __half* out) {
  if (get_option("gn_fused") == 0) return -1;
  if (C % 8 != 0 || C % groups != 0 || C / groups < 8 || groups > 32) return -1;
  const int CV = C / 8;
  if (kGnFusedThreads % CV != 0) return -1;
  const size_t img_bytes = (size_t)hw * C * 2, cap = 160 * 1024;
  int ncta = 1;
  while ((img_bytes + ncta - 1) / ncta > cap && ncta < 16) ncta *= 2;
  if ((img_bytes + ncta - 1) / ncta > cap || hw % ncta != 0) return -1;
  // Measured on an H100 80GB HBM3 (400 W power limit), 32 images, single pass vs statistics + apply pair: 64x64x320 (16 CTAs)
  // 91.5 vs 103.6 us, 32x32x640 (8) 49.4 vs 58.9 us, 16x16x1280 (4) 28.1 vs 24.6 us, 8x8x1280 (1) 19.5 vs 23.7 us.  The single
  // pass wins at three of the four levels and in sum, so every cluster size takes it ("gn_fused" != 0).
  const int ppc = hw / ncta;
  const size_t smem = 512 + (size_t)ppc * C * 2;
  static bool configured = false;
  if (!configured) {
    VS_CHECK_CUDA(cudaFuncSetAttribute(gn_frame_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 512 + (int)cap));
    VS_CHECK_CUDA(cudaFuncSetAttribute(gn_frame_fused_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    configured = true;
  }
  GnParams p{};
  p.x1 = x; p.c1 = C; p.C = C; p.CV = CV; p.hw = hw; p.imgs_per_set = 1; p.groups = groups; p.cpg = C / groups;
  p.pix_per_set = hw; p.gamma = gamma; p.beta = beta; p.eps = eps; p.silu = silu ? 1 : 0; p.out = out; p.count_scale = 1;
  ProfScope prof(st, PC_GROUPNORM, 4.0 * nimg * (double)hw * C, 1, (long long)nimg * hw, C, 1);   // read once + write once
  return launch_pdl(gn_frame_fused_kernel, dim3((unsigned)(nimg * ncta)), dim3(kGnFusedThreads), smem, st, ncta, p, ncta, ppc);
}

int groupnorm_stats(cudaStream_t st, const __half* x1, int c1, const __half* x2, int c2, int nimg, int hw,
                    int imgs_per_set, int groups, float* sums, bool zero_first) {
  GnParams p{};
  dim3 grid;
  int threads;
  if (int e = gn_fill(p, grid, threads, x1, c1, x2, c2, nimg, hw, imgs_per_set, groups)) return e;
  p.sums = sums;
  if (zero_first) VS_CHECK_CUDA(cudaMemsetAsync(sums, 0, sizeof(float) * 2 * groups * (nimg / imgs_per_set), st));
  ProfScope prof(st, PC_GROUPNORM, 2.0 * nimg * (double)hw * (c1 + c2));   // bytes read
  if (get_option("gn_stats_v2") != 0) return launch_pdl(gn_stats_kernel<true>, grid, dim3(threads), groups * 2 * sizeof(float), st, 1, p);
  return launch_pdl(gn_stats_kernel<false>, grid, dim3(threads), groups * 2 * sizeof(float), st, 1, p);
}

int groupnorm_apply(cudaStream_t st, const __half* x1, int c1, const __half* x2, int c2, int nimg, int hw,
                    int imgs_per_set, int groups, const float* sums, float eps, const float* gamma, const float* beta,
                    bool silu, __half* out, int count_scale) {
  GnParams p{};
  dim3 grid;
  int threads;
  if (int e = gn_fill(p, grid, threads, x1, c1, x2, c2, nimg, hw, imgs_per_set, groups)) return e;
  p.sums = const_cast<float*>(sums);
  p.gamma = gamma; p.beta = beta; p.eps = eps; p.silu = silu ? 1 : 0; p.out = out;
  p.count_scale = count_scale > 0 ? count_scale : 1;
  ProfScope prof(st, PC_GROUPNORM, 4.0 * nimg * (double)hw * (c1 + c2), 1, (long long)nimg * hw, c1 + c2, imgs_per_set);
  return launch_pdl(gn_apply_kernel, grid, dim3(threads), 0, st, 1, p);
}

int layernorm(cudaStream_t st, const __half* x, int rows, int C, const float* gamma, const float* beta, const float* pe,
              int hw, int F, __half* out) {
  VS_REQUIRE(C % 8 == 0 && C <= 8 * 32 * 8, "layernorm: unsupported C=%d", C);
  const int nvec = C / 8, vpl = (nvec + 31) / 32;
  const int threads = 256, wpb = threads / 32;
  const int blocks = (rows + wpb - 1) / wpb;
  if (hw <= 0) hw = 1;
  if (F <= 0) F = 1;
  ProfScope prof(st, PC_LAYERNORM, 4.0 * rows * (double)C, 1, rows, C, pe ? 1 : 0);
  if (C == 320 || C == 640 || C == 1280) {
    const int lpr = C / 40, rpw = 32 / lpr;
    long long need = ((long long)rows + rpw * 8 * 4 - 1) / (rpw * 8 * 4);   // blocks of 8 warps, >= 2 double row groups per warp
    if (need < 1) need = 1;
    const long long cap = (long long)num_sms() * 8;
    const int grid = (int)(need < cap ? need : cap);
    const long long rows_ll = rows;
    if (lpr == 8) return launch_pdl(ln5_kernel<8>, dim3(grid), dim3(256), 0, st, 1, x, rows_ll, gamma, beta, pe, hw, F, out);
    if (lpr == 16) return launch_pdl(ln5_kernel<16>, dim3(grid), dim3(256), 0, st, 1, x, rows_ll, gamma, beta, pe, hw, F, out);
    return launch_pdl(ln5_kernel<32>, dim3(grid), dim3(256), 0, st, 1, x, rows_ll, gamma, beta, pe, hw, F, out);
  }
  switch (vpl) {
    case 1: ln_kernel<1><<<blocks, threads, 0, st>>>(x, rows, C, gamma, beta, pe, hw, F, out); break;
    case 2: ln_kernel<2><<<blocks, threads, 0, st>>>(x, rows, C, gamma, beta, pe, hw, F, out); break;
    case 3: ln_kernel<3><<<blocks, threads, 0, st>>>(x, rows, C, gamma, beta, pe, hw, F, out); break;
    case 4: ln_kernel<4><<<blocks, threads, 0, st>>>(x, rows, C, gamma, beta, pe, hw, F, out); break;
    case 5: ln_kernel<5><<<blocks, threads, 0, st>>>(x, rows, C, gamma, beta, pe, hw, F, out); break;
    default: ln_kernel<8><<<blocks, threads, 0, st>>>(x, rows, C, gamma, beta, pe, hw, F, out); break;
  }
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace vs
