// Small / pointwise kernels of the denoising step: timestep embedding + tiny linears, conv_in (Cin=4), nearest 2x
// up-sampling, stride-2 im2col, layout conversion at the API boundary, the fused classifier-free-guidance + DDIM
// update (reference pipelines/pipeline_videoswap.py:578-587 + diffusers DDIMScheduler.step), the sparse-point
// adapter splat (models/adapter_model.py:25-47,121-130) and weight re-packing.
#include "common.cuh"
#include "kernels.h"

namespace vs {
namespace {

constexpr int TPB = 256;
inline unsigned blocks_for(size_t n, int per = TPB) { return (unsigned)((n + per - 1) / per); }

// ---------------------------------------------------------------------------------------------- tiny linears
__global__ void small_linear_kernel(const float* __restrict__ x, int rows, int K, const __half* __restrict__ W,
                                    const float* __restrict__ bias, int N, int silu_in, int silu_out,
                                    float* __restrict__ out) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (n >= N) return;
  const __half* w = W + (long long)n * K;
  for (int r0 = 0; r0 < rows; r0 += 8) {
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int k = lane * 2; k < K; k += 64) {
      const float2 wv = __half22float2(*reinterpret_cast<const __half2*>(w + k));
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        if (r0 + r < rows) {
          float a = x[(long long)(r0 + r) * K + k], b = x[(long long)(r0 + r) * K + k + 1];
          if (silu_in) { a = silu_f(a); b = silu_f(b); }
          acc[r] += a * wv.x + b * wv.y;
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
      if (lane == 0 && r0 + r < rows) {
        float v = acc[r] + (bias ? bias[n] : 0.f);
        if (silu_out) v = silu_f(v);
        out[(long long)(r0 + r) * N + n] = v;
      }
    }
  }
}

__global__ void timestep_embedding_kernel(const float* __restrict__ t, int B, int dim, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = dim / 2;
  if (i >= B * half) return;
  const int b = i / half, j = i % half;
  const float freq = expf(-9.210340371976184f * (float)j / (float)half);   // ln(1e4)
  const float arg = t[b] * freq;
  out[b * dim + j] = cosf(arg);            // flip_sin_to_cos=True -> cos first
  out[b * dim + half + j] = sinf(arg);
}

// ---------------------------------------------------------------------------------------------- conv_in (tiny Cin)
__global__ void conv_in_kernel(const __half* __restrict__ x, int nimg, int H, int W, int cin, const __half* __restrict__ w,
                               const float* __restrict__ bias, int cout, __half* __restrict__ out) {
  extern __shared__ float ws[];   // [9*cin][cout]
  const int K = 9 * cin;
  for (int i = threadIdx.x; i < K * cout; i += blockDim.x) {
    const int co = i % cout, k = i / cout;           // k = tap*cin + ci
    const int tap = k / cin, ci = k % cin;
    ws[i] = __half2float(w[((long long)co * cin + ci) * 9 + tap]);   // [co][ci][3][3]
  }
  __syncthreads();
  const int cg = cout / 8;
  const long long total = (long long)nimg * H * W * cg;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = i % cg;
    const long long pix = i / cg;
    const int xq = pix % W, yq = (pix / W) % H;
    const long long img = pix / ((long long)W * H);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = bias ? bias[g * 8 + j] : 0.f;
    for (int tap = 0; tap < 9; ++tap) {
      const int yy = yq + tap / 3 - 1, xx = xq + tap % 3 - 1;
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
      const __half* px = x + ((img * H + yy) * W + xx) * cin;
      for (int ci = 0; ci < cin; ++ci) {
        const float v = __half2float(px[ci]);
        const float* wr = ws + (tap * cin + ci) * cout + g * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += v * wr[j];
      }
    }
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) oh[j] = __floats2half2_rn(acc[2 * j], acc[2 * j + 1]);
    *reinterpret_cast<uint4*>(out + pix * cout + g * 8) = o;
  }
}

// conv_in on the tensor cores: the 36-wide patch of every pixel (9 taps x 4 channels, zero padded to one 64-column
// k-block) is written once as an fp16 row, the weight goes to [cout][64] in the same order, and the wgmma GEMM does the
// rest (the direct kernel above reads the 4-channel input once per output channel block and is much slower).
__global__ void conv_in_patch_kernel(const __half* __restrict__ x, int nimg, int H, int W, uint4* __restrict__ out) {
  const long long total = (long long)nimg * H * W * 8;   // eight 16-byte chunks (two taps each) per pixel
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i & 7);
    const long long pix = i >> 3;
    const int xq = (int)(pix % W), yq = (int)((pix / W) % H);
    const long long img = pix / ((long long)W * H);
    uint2 t[2] = {make_uint2(0u, 0u), make_uint2(0u, 0u)};
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int tap = 2 * c + u;
      const int yy = yq + tap / 3 - 1, xx = xq + tap % 3 - 1;
      if (tap < 9 && yy >= 0 && yy < H && xx >= 0 && xx < W)
        t[u] = *reinterpret_cast<const uint2*>(x + ((img * H + yy) * W + xx) * 4);
    }
    out[i] = make_uint4(t[0].x, t[0].y, t[1].x, t[1].y);
  }
}
__global__ void conv_in_pack_kernel(const __half* __restrict__ w, int cout, __half* __restrict__ out) {   // [co][4][3][3] -> [co][64]
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cout * 64) return;
  const int co = i >> 6, k = i & 63, tap = k >> 2, ci = k & 3;
  out[i] = tap < 9 ? w[(co * 4 + ci) * 9 + tap] : __float2half(0.f);
}

// ---------------------------------------------------------------------------------------------- data movement
// nearest up-sampling to OH x OW with OH in {2H - 1, 2H}: torch's source row floor(yo * H / OH) is yo / 2 for both
__global__ void upsample2x_kernel(const uint4* __restrict__ x, int nimg, int H, int W, int CV, int OH, int OW,
                                  uint4* __restrict__ out) {
  const long long total = (long long)nimg * OH * OW * CV;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cv = i % CV;
    const long long pix = i / CV;
    const int xo = pix % OW, yo = (pix / OW) % OH;
    const long long img = pix / ((long long)OW * OH);
    out[i] = x[((img * H + yo / 2) * W + xo / 2) * CV + cv];
  }
}

__global__ void im2col_s2_kernel(const uint4* __restrict__ x, int nimg, int H, int W, int CV, int Ho, int Wo,
                                 uint4* __restrict__ out) {
  const long long total = (long long)nimg * Ho * Wo * 9 * CV;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cv = i % CV;
    const int tap = (i / CV) % 9;
    const long long opix = i / (9LL * CV);
    const int xo = opix % Wo, yo = (opix / Wo) % Ho;
    const long long img = opix / ((long long)Wo * Ho);
    const int yy = 2 * yo + tap / 3 - 1, xx = 2 * xo + tap % 3 - 1;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = x[((img * H + yy) * W + xx) * CV + cv];
    out[i] = v;
  }
}

__global__ void add_kernel(__half* __restrict__ x, const __half* __restrict__ r, size_t n, float scale) {
  const size_t nv = n / 8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
    uint4 a = reinterpret_cast<uint4*>(x)[i];
    const uint4 b = reinterpret_cast<const uint4*>(r)[i];
    __half2* ah = reinterpret_cast<__half2*>(&a);
    const __half2* bh = reinterpret_cast<const __half2*>(&b);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 fa = __half22float2(ah[j]), fb = __half22float2(bh[j]);
      ah[j] = __floats2half2_rn(fa.x + scale * fb.x, fa.y + scale * fb.y);
    }
    reinterpret_cast<uint4*>(x)[i] = a;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0)
    for (size_t i = nv * 8; i < n; ++i) x[i] = __float2half_rn(__half2float(x[i]) + scale * __half2float(r[i]));
}

template <typename T>
__global__ void ncfhw_to_nhwc_kernel(const T* __restrict__ src, int B, int C, int F, int H, int W, __half* __restrict__ dst) {
  const long long total = (long long)B * F * H * W * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = i % C;
    long long r = i / C;
    const int x = r % W; r /= W;
    const int y = r % H; r /= H;
    const int f = r % F;
    const int b = r / F;
    dst[i] = __float2half_rn((float)src[((((long long)b * C + c) * F + f) * H + y) * W + x]);
  }
}
template <typename T>
__global__ void nhwc_to_ncfhw_kernel(const __half* __restrict__ src, int B, int C, int F, int H, int W, T* __restrict__ dst) {
  const long long total = (long long)B * F * H * W * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int x = r % W; r /= W;
    const int y = r % H; r /= H;
    const int f = r % F; r /= F;
    const int c = r % C;
    const int b = r / C;
    dst[i] = (T)__half2float(src[((((long long)b * F + f) * H + y) * W + x) * C + c]);
  }
}

__global__ void nchw_to_nhwc_kernel(const __half* __restrict__ src, int C, int HW, float scale, __half* __restrict__ dst) {
  __shared__ __half tile[32][33];
  const long long img = blockIdx.z;
  const int c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, p = p0 + threadIdx.x;
    if (c < C && p < HW) tile[j][threadIdx.x] = src[(img * C + c) * HW + p];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int p = p0 + j, c = c0 + threadIdx.x;
    if (c < C && p < HW) dst[(img * HW + p) * C + c] = __float2half_rn(__half2float(tile[threadIdx.x][j]) * scale);
  }
}

// ---------------------------------------------------------------------------------------------- CFG + DDIM
template <typename T>
__global__ void cfg_ddim_kernel(const T* __restrict__ eps2, const T* __restrict__ x, size_t n, int cfg, float g,
                                float c_x, float c_e, const float* __restrict__ d_coef, T* __restrict__ out) {
  // x_prev = sqrt(a_p)/sqrt(a_t) * x + (sqrt(1-a_p) - sqrt(a_p) sqrt(1-a_t)/sqrt(a_t)) * eps   (eta = 0)
  if (d_coef) {   // coefficients in device memory: the launch stays valid inside a replayed CUDA graph
    c_x = d_coef[0];
    c_e = d_coef[1];
  }
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float e = (float)eps2[i];
    if (cfg) {
      const float ec = (float)eps2[n + i];
      e = e + g * (ec - e);
    }
    out[i] = (T)(c_x * (float)x[i] + c_e * e);
  }
}

// ---------------------------------------------------------------------------------------------- CFG + rescale + DDIM(eta)
// The same step for S samples of n_s elements each, with diffusers 0.19.3's stochastic DDIM (eta > 0) and the CFG
// rescale of rescale_noise_cfg (pipeline_videoswap.py:582-584):
//   e  = e_u + g (e_c - e_u)                                   (e = e_u without CFG)
//   e <- e (r std(e_c) / std(e) + 1 - r)                       (CFG and r > 0 only; unbiased std over the sample)
//   x' = c_x x + c_e e + c_n z                                 (z: the caller's noise; absent when null)
// One thread-block cluster per sample (ncta CTAs, each a contiguous slice).  With the rescale each CTA first sums its
// slice's shifted (sum, sum of squares) of e_c and e in fp64, the CTAs exchange the four partials through distributed
// shared memory between two cluster barriers and add them in rank order (no atomics: bit-reproducible), and a second
// sweep re-reads the slice (from L2) to apply the update.  The shift is the sample's first value: with fp64 partials a
// mean of 1e3 at spread 1 keeps its variance.
constexpr int kRsThreads = 512;
constexpr int kRsMaxCta = 16;

template <typename T>
__global__ void __launch_bounds__(kRsThreads) cfg_ddim_rescale_kernel(
    const T* __restrict__ eps2, const T* __restrict__ x, const T* __restrict__ z, long long ns, int S, int ncta, int cfg,
    float g, float c_x, float c_e, float c_n, float r, const float* __restrict__ d_coef, T* __restrict__ out) {
  __shared__ double warp_part[kRsThreads / 32][4];
  __shared__ double part[4], tot[4];
  if (d_coef) {   // coefficients in device memory: (c_x, c_e, c_n, r), replayable inside a CUDA graph
    c_x = d_coef[0];
    c_e = d_coef[1];
    c_n = d_coef[2];
    r = d_coef[3];
  }
  const int s = blockIdx.x / ncta, rank = blockIdx.x % ncta;
  const long long chunk = (ns + ncta - 1) / ncta;
  const long long lo = min(ns, (long long)rank * chunk), hi = min(ns, lo + chunk);
  const T* eu = eps2 + (long long)s * ns;
  const T* ec = eps2 + ((long long)S + s) * ns;
  const T* xs = x + (long long)s * ns;
  const T* zs = z ? z + (long long)s * ns : nullptr;
  T* os = out + (long long)s * ns;
  auto cfg_e = [&](long long i) {
    const float u = (float)eu[i];
    return cfg ? u + g * ((float)ec[i] - u) : u;
  };
  float factor = 1.f;
  if (cfg && r > 0.f) {   // uniform over the cluster: every CTA reads the same r
    const double kc = (double)(float)ec[0], ke = (double)cfg_e(0);
    double sc = 0.0, qc = 0.0, se = 0.0, qe = 0.0;
    for (long long i = lo + threadIdx.x; i < hi; i += kRsThreads) {
      const double dc = (double)(float)ec[i] - kc, de = (double)cfg_e(i) - ke;
      sc += dc; qc = fma(dc, dc, qc);
      se += de; qe = fma(de, de, qe);
    }
    double v[4] = {sc, qc, se, qe};
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v[j] += __shfl_xor_sync(0xffffffffu, v[j], o);
      if (lane == 0) warp_part[wid][j] = v[j];
    }
    __syncthreads();
    if (threadIdx.x < 4) {
      double t = 0.0;
      for (int w = 0; w < kRsThreads / 32; ++w) t += warp_part[w][threadIdx.x];   // fixed order
      part[threadIdx.x] = t;
    }
    __syncthreads();
    if (ncta > 1) cluster_sync_all();                                            // every CTA's partials are complete
    if (threadIdx.x < 4) {
      double t = 0.0;
      if (ncta > 1) {
        const uint32_t mine = smem_u32(&part[threadIdx.x]);
        for (int c = 0; c < ncta; ++c) {                                           // rank order: deterministic
          double pv;
          asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(pv) : "r"(mapa_shared(mine, (uint32_t)c)));
          t += pv;
        }
      } else {
        t = part[threadIdx.x];
      }
      tot[threadIdx.x] = t;
    }
    __syncthreads();
    const double n = (double)ns;
    const double var_c = (tot[1] - tot[0] * tot[0] / n) / (n - 1.0);
    const double var_e = (tot[3] - tot[2] * tot[2] / n) / (n - 1.0);
    factor = (float)((double)r * (sqrt(var_c) / sqrt(var_e)) + (1.0 - (double)r));
  }
  for (long long i = lo + threadIdx.x; i < hi; i += kRsThreads) {
    const float e = cfg_e(i) * factor;
    float v = c_x * (float)xs[i] + c_e * e;
    if (zs) v += c_n * (float)zs[i];
    os[i] = (T)v;
  }
  if (cfg && r > 0.f && ncta > 1) cluster_sync_all();   // nobody leaves while a peer may still read its partials
}

// ---------------------------------------------------------------------------------------------- adapter splat
__device__ __forceinline__ float r16(float v, int on) { return on ? __half2float(__float2half_rn(v)) : v; }

__global__ void adapter_splat_kernel(const float* __restrict__ feat, const float* __restrict__ tracks,
                                     const int* __restrict__ mask, int F, int P, int C, int h, int w, float rate,
                                     int c16, float scale, __half* __restrict__ maps) {
  const int CV = C / 8;
  const long long total = (long long)F * h * w * CV;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cv = i % CV;
    const long long cell = i / CV;
    const int x = cell % w, y = (cell / w) % h, f = cell / ((long long)w * h);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int pt = 0; pt < P; ++pt) {
      if (mask && !mask[pt]) continue;
      const float px = r16(tracks[(f * P + pt) * 2], c16), py = r16(tracks[(f * P + pt) * 2 + 1], c16);
      if (px < 0.f || py < 0.f) continue;
      const float fx = r16(px / rate, c16), fy = r16(py / rate, c16);
      int x1 = (int)fx, y1 = (int)fy;
      const float xf = r16(fx - (float)x1, c16), yf = r16(fy - (float)y1, c16);
      int x2 = x1 + 1, y2 = y1 + 1;
      x1 = max(min(x1, w - 1), 0); x2 = max(min(x2, w - 1), 0);
      y1 = max(min(y1, h - 1), 0); y2 = max(min(y2, h - 1), 0);
      const float ox = r16(1.f - xf, c16), oy = r16(1.f - yf, c16);
      float wsum = 0.f;
      if (y == y1 && x == x1) wsum += r16(ox * oy, c16);
      if (y == y1 && x == x2) wsum += r16(xf * oy, c16);
      if (y == y2 && x == x1) wsum += r16(ox * yf, c16);
      if (y == y2 && x == x2) wsum += r16(xf * yf, c16);
      if (wsum != 0.f) {
        const float* fr = feat + (long long)pt * C + cv * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += r16(fr[j], c16) * wsum;
      }
    }
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) oh[j] = __floats2half2_rn(r16(acc[2 * j], c16) * scale, r16(acc[2 * j + 1], c16) * scale);
    *reinterpret_cast<uint4*>(maps + cell * C + cv * 8) = o;
  }
}

// ---------------------------------------------------------------------------------------------- latent blend (p2p)
// SpatialBlender.get_mask + __call__ (utils/p2p_utils/spatial_blend.py:25-63,65-145) on device.  One block per frame:
//   m[p][pix]   = mean over (layers x heads) of sum_w alpha[p][w] * map[layer][p][frame][head][pix][w]
//   pooled      = 3x3 max pool (stride 1, -inf padding) when `pool`
//   mask[p]     = nearest-resized(pooled) / max(nearest-resized(pooled)) > threshold
//   both        : mask[p] |= mask[0]   (the reference's `mask[:1] + mask` on bool tensors)
// maps: n_maps * n_prompts pointers, each [frames, heads, res_h * res_w, words] fp16.
constexpr int kBlendMaxRes = 1024;      // the controllers only see layers with fewer than 32^2 queries
__global__ void __launch_bounds__(256) blend_mask_kernel(const __half* const* __restrict__ maps, int n_maps, int n_prompts, int frames,
                                                         int heads, int rh, int rw, int words, const float* __restrict__ alpha,
                                                         int pool, int h, int w, float threshold, int both, float* __restrict__ mask) {
  __shared__ float m[kBlendMaxRes], pooled[kBlendMaxRes], red[8];
  const int f = blockIdx.x, res = rh * rw, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float inv = 1.f / (float)(n_maps * heads);
  for (int pr = 0; pr < n_prompts; ++pr) {
    // one warp per pixel: lanes stride over the words
    for (int pix = warp; pix < res; pix += 8) {
      float acc = 0.f;
      for (int l = 0; l < n_maps; ++l) {
        const __half* mp = maps[l * n_prompts + pr] + ((long long)f * heads * res + pix) * words;
        for (int hd = 0; hd < heads; ++hd)
          for (int wd = lane; wd < words; wd += 32) {
            const float a = alpha[pr * words + wd];
            if (a != 0.f) acc += a * __half2float(mp[(long long)hd * res * words + wd]);
          }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) m[pix] = acc * inv;
    }
    __syncthreads();
    for (int pix = tid; pix < res; pix += 256) {
      float v = m[pix];
      if (pool) {
        const int y = pix / rw, x = pix % rw;
        for (int dy = -1; dy <= 1; ++dy)
          for (int dx = -1; dx <= 1; ++dx) {
            const int yy = y + dy, xx = x + dx;
            if (yy >= 0 && yy < rh && xx >= 0 && xx < rw) v = fmaxf(v, m[yy * rw + xx]);
          }
      }
      pooled[pix] = v;
    }
    __syncthreads();
    // F.interpolate(size=(h, w)), mode 'nearest': src = floor(dst * in / out)
    float mx = -INFINITY;
    for (int i = tid; i < h * w; i += 256) {
      const int sy = min((int)floorf((float)(i / w) * ((float)rh / (float)h)), rh - 1);
      const int sx = min((int)floorf((float)(i % w) * ((float)rw / (float)w)), rw - 1);
      mx = fmaxf(mx, pooled[sy * rw + sx]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = red[0];
    for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
    float* out = mask + ((long long)pr * frames + f) * h * w;
    const float* first = mask + (long long)f * h * w;        // prompt 0 of this frame (written by this block earlier)
    for (int i = tid; i < h * w; i += 256) {
      const int sy = min((int)floorf((float)(i / w) * ((float)rh / (float)h)), rh - 1);
      const int sx = min((int)floorf((float)(i % w) * ((float)rw / (float)w)), rw - 1);
      float bit = (pooled[sy * rw + sx] / mx > threshold) ? 1.f : 0.f;      // 0/0 = NaN -> false, like the reference
      if (both && pr > 0 && first[i] != 0.f) bit = 1.f;
      out[i] = bit;
    }
    __syncthreads();
  }
}

// x_tgt = x_src + mask * (x_tgt - x_src) per (channel, frame, pixel), in fp32 (spatial_blend.py:141-142); mask [frames, hw].
// A 0 / 1 mask (all blend_mask produces) selects the source or the target bit for bit: the lerp alone would round
// t - s and return a value near, but not equal to, the target wherever |t| << |s|.  This departs from the reference's
// rounded lerp on purpose: at m = 1 the result is the target itself (the lerp can be a few ulps off), and the operand a
// 0 / 1 mask does not pick is never read, so a non-finite value there (m = 0, t = inf: NaN in the lerp) does not leak
// into the blend.  Fractional masks take the lerp unchanged.
__device__ __forceinline__ float blend_lerp(float s, float t, float mk) {
  return mk == 0.f ? s : (mk == 1.f ? t : s + mk * (t - s));
}
__global__ void latent_blend_kernel(const void* __restrict__ x_src, void* __restrict__ x_tgt, const float* __restrict__ mask,
                                    int is_f32, int channels, int frames, int hw) {
  const long long per_c = (long long)frames * hw, total = per_c * channels;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const float mk = mask[i % per_c];
    if (is_f32) {
      const float s = reinterpret_cast<const float*>(x_src)[i];
      float* t = reinterpret_cast<float*>(x_tgt) + i;
      *t = blend_lerp(s, *t, mk);
    } else {
      const float s = __half2float(reinterpret_cast<const __half*>(x_src)[i]);
      __half* t = reinterpret_cast<__half*>(x_tgt) + i;
      *t = __float2half_rn(blend_lerp(s, __half2float(*t), mk));
    }
  }
}

// ---------------------------------------------------------------------------------------------- packing
__global__ void pack_conv3x3_kernel(const __half* __restrict__ w, int cout, int cin, __half* __restrict__ out) {
  const long long total = (long long)cout * 9 * cin;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ci = i % cin, tap = (i / cin) % 9;
    const long long co = i / (9LL * cin);
    out[i] = w[(co * cin + ci) * 9 + tap];
  }
}
__global__ void pack_conv_subpixel_kernel(const __half* __restrict__ w, int cout, int cin, __half* __restrict__ out) {
  const long long per = (long long)cout * 4 * cin, total = 4 * per;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ci = i % cin, tap = (i / cin) % 4;
    const long long co = (i / (4LL * cin)) % cout;
    const int par = i / per, py = par >> 1, px = par & 1, ty = tap >> 1, tx = tap & 1;
    // source-row tap ty of parity py gathers these 3x3 rows: py=0: ty=0 -> {0}, ty=1 -> {1,2};  py=1: ty=0 -> {0,1}, ty=1 -> {2}
    const int r0 = (py == 0) ? (ty == 0 ? 0 : 1) : (ty == 0 ? 0 : 2), r1 = (py == 0) ? (ty == 0 ? 0 : 2) : (ty == 0 ? 1 : 2);
    const int c0 = (px == 0) ? (tx == 0 ? 0 : 1) : (tx == 0 ? 0 : 2), c1 = (px == 0) ? (tx == 0 ? 0 : 2) : (tx == 0 ? 1 : 2);
    float acc = 0.f;
    for (int r = r0; r <= r1; ++r)
      for (int c = c0; c <= c1; ++c) acc += __half2float(w[(co * cin + ci) * 9 + r * 3 + c]);
    out[i] = __float2half_rn(acc);
  }
}
// The 4 panels of odd target sizes (pack_conv_subpixel with odd_panels): along the odd axis parity 0 has the three
// unsummed taps {0}, {1}, {2}; the other axis collapses as above.  Panels: (py, px) = (0, 0), (0, 1) with 3 row taps,
// then (0, 0), (1, 0) with 3 column taps; 6 taps each.
__global__ void pack_conv_subpixel_odd_kernel(const __half* __restrict__ w, int cout, int cin, __half* __restrict__ out) {
  const long long per = (long long)cout * 6 * cin, total = 4 * per;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ci = i % cin, tap = (i / cin) % 6;
    const long long co = (i / (6LL * cin)) % cout;
    const int panel = i / per;
    const bool odd_rows = panel < 2;
    const int py = odd_rows ? 0 : panel - 2, px = odd_rows ? panel : 0;
    const int ty = odd_rows ? tap >> 1 : tap / 3, tx = odd_rows ? tap & 1 : tap % 3;   // slot along y / x
    auto range = [](int par, bool three, int t, int& a, int& b) {
      if (three) { a = b = t; return; }
      a = (par == 0) ? (t == 0 ? 0 : 1) : (t == 0 ? 0 : 2);
      b = (par == 0) ? (t == 0 ? 0 : 2) : (t == 0 ? 1 : 2);
    };
    int r0, r1, c0, c1;
    range(py, odd_rows, ty, r0, r1);
    range(px, !odd_rows, tx, c0, c1);
    float acc = 0.f;
    for (int r = r0; r <= r1; ++r)
      for (int c = c0; c <= c1; ++c) acc += __half2float(w[(co * cin + ci) * 9 + r * 3 + c]);
    out[i] = __float2half_rn(acc);
  }
}
__global__ void pack_geglu_kernel(const __half* __restrict__ w, const __half* __restrict__ b, int hidden, int K,
                                  int gran, __half* __restrict__ wout, float* __restrict__ bout) {
  const long long total = (long long)2 * hidden * K;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k = i % K;
    const long long pr = i / K;                       // packed row
    const long long tile = pr / (2 * gran);
    const int within = pr % (2 * gran);
    const long long srow = within < gran ? tile * gran + within : (long long)hidden + tile * gran + (within - gran);
    if (w) wout[i] = w[srow * K + k];
    if (b && k == 0) bout[pr] = __half2float(b[srow]);
  }
}
__global__ void f16_to_f32_kernel(const __half* __restrict__ x, size_t n, float* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = __half2float(x[i]);
}

// Folds a LayerNorm (gamma, beta, optional additive positional table pe [pe_len, K]) into the linear layer W [N, K] that
// consumes its output (one block per output row n):
//   wf[n,k] = fp16(W[n,k] gamma[k]);  u[n] = sum_k float(wf[n,k]);  c[n] = sum_k beta[k] W[n,k] + bias[n];
//   cpe[f,n] = sum_k pe[f,k] W[n,k].        (u is summed over the ROUNDED wf so that rstd (x wf^T - mean u) is exact.)
constexpr int kMaxPe = 32;
__global__ void __launch_bounds__(128) ln_fold_kernel(const __half* __restrict__ w, int N, int K, const float* __restrict__ gamma,
                                                      const float* __restrict__ beta, const float* __restrict__ bias,
                                                      const float* __restrict__ pe, int pe_len, __half* __restrict__ wf,
                                                      float* __restrict__ u, float* __restrict__ c, float* __restrict__ cpe) {
  const int n = blockIdx.x;
  float su = 0.f, sc = 0.f, sp[kMaxPe];
#pragma unroll
  for (int f = 0; f < kMaxPe; ++f) sp[f] = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float wv = __half2float(w[(size_t)n * K + k]);
    const __half r = __float2half_rn(wv * gamma[k]);
    wf[(size_t)n * K + k] = r;
    su += __half2float(r);
    sc = fmaf(beta[k], wv, sc);
    if (pe) {
#pragma unroll
      for (int f = 0; f < kMaxPe; ++f)
        if (f < pe_len) sp[f] = fmaf(pe[(size_t)f * K + k], wv, sp[f]);
    }
  }
  __shared__ float red[4][kMaxPe + 2];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  auto wsum = [](float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  };
  su = wsum(su); sc = wsum(sc);
#pragma unroll
  for (int f = 0; f < kMaxPe; ++f) sp[f] = wsum(sp[f]);
  if (lane == 0) {
    red[wid][0] = su; red[wid][1] = sc;
#pragma unroll
    for (int f = 0; f < kMaxPe; ++f) red[wid][2 + f] = sp[f];
  }
  __syncthreads();
  if (threadIdx.x < kMaxPe + 2) {
    const float t = red[0][threadIdx.x] + red[1][threadIdx.x] + red[2][threadIdx.x] + red[3][threadIdx.x];
    if (threadIdx.x == 0) u[n] = t;
    else if (threadIdx.x == 1) c[n] = t + (bias ? bias[n] : 0.f);
    else if (pe && (int)threadIdx.x - 2 < pe_len) cpe[(size_t)(threadIdx.x - 2) * N + n] = t;
  }
}

// ---------------------------------------------------------------------------------------------- VAE decoder entry / exit
// post_quant_conv(z / divisor) (diffusers AutoencoderKL._decode): NCHW [n, 4, h, w] fp16 or fp32 latents -> NHWC fp16 [n, h, w, 4].
// wb: fp32 [4][4] weight then [4] bias.  Fixed order, no contraction: out_c = (((b_c + w_c0 x_0) + w_c1 x_1) + w_c2 x_2) + w_c3 x_3.
template <typename T>
__global__ void vae_latent_in_kernel(const T* __restrict__ z, long long npix, int hw, float divisor, const float* __restrict__ wb,
                                     __half* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const long long img = i / hw, p = i % hw;
    float x[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) x[k] = (float)z[(img * 4 + k) * hw + p] / divisor;
    __half o[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float acc = wb[16 + c];
#pragma unroll
      for (int k = 0; k < 4; ++k) acc = __fadd_rn(acc, __fmul_rn(wb[c * 4 + k], x[k]));
      o[c] = __float2half_rn(acc);
    }
    *reinterpret_cast<uint2*>(out + i * 4) = *reinterpret_cast<const uint2*>(o);
  }
}

// VaeImageProcessor.postprocess of channels 0..2 of the decoder's NHWC fp16 output x [n, H, W, cs]:
//   IMG_SAMPLE  x itself as fp16 NCHW [n, 3, H, W] (AutoencoderKL.decode's sample, not denormalised)
//   IMG_PT      y = clamp(x / 2 + 0.5, 0, 1) as fp32 NCHW;  IMG_NP  y as fp32 NHWC [n, H, W, 3]
//   IMG_PIL     uint8 NHWC round_half_even(y * 255) (numpy's round, then astype(uint8))
__global__ void image_postprocess_kernel(const __half* __restrict__ x, long long npix, int hw, int cs, int format, void* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = *reinterpret_cast<const uint4*>(x + i * cs);
    const __half* h = reinterpret_cast<const __half*>(&v);
    const long long img = i / hw, p = i % hw;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const long long nchw = (img * 3 + c) * hw + p;
      if (format == IMG_SAMPLE) {
        reinterpret_cast<__half*>(out)[nchw] = h[c];
        continue;
      }
      const float y = fminf(fmaxf(__fadd_rn(__fmul_rn(__half2float(h[c]), 0.5f), 0.5f), 0.f), 1.f);
      if (format == IMG_PT) reinterpret_cast<float*>(out)[nchw] = y;
      else if (format == IMG_NP) reinterpret_cast<float*>(out)[i * 3 + c] = y;
      else reinterpret_cast<uint8_t*>(out)[i * 3 + c] = (uint8_t)__float2int_rn(__fmul_rn(y, 255.f));
    }
  }
}

// ---------------------------------------------------------------------------------------------- VAE encoder entry / exit
// Encoder input as NHWC fp16 [n, H, W, 4] with channel 3 zero (so the tensor-core conv_in, ci = 4, runs the 3 -> 128 conv).
// uint8 NHWC frames [n, H, W, 3]: what VaeImageProcessor.preprocess and the fp16 cast of prepare_image_latents compute,
// fl16(fl32(2 fl32(u / 255) - 1)) -- numpy's float32 division, 2 y exact, the subtraction rounded on its own (no FMA).
__global__ void vae_image_in_u8_kernel(const uint8_t* __restrict__ x, long long npix, __half* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    __half o[4];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float y = __fdiv_rn((float)x[i * 3 + c], 255.f);
      o[c] = __float2half_rn(__fsub_rn(__fmul_rn(2.f, y), 1.f));
    }
    o[3] = __float2half_rn(0.f);
    *reinterpret_cast<uint2*>(out + i * 4) = *reinterpret_cast<const uint2*>(o);
  }
}

// float NCHW images [n, 3, H, W] (fp16, or fp32 rounded to fp16 once), already in [-1, 1] (AutoencoderKL.encode's input)
template <typename T>
__global__ void vae_image_in_nchw_kernel(const T* __restrict__ x, long long npix, int hw, __half* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const long long img = i / hw, p = i % hw;
    __half o[4];
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = __float2half_rn((float)x[(img * 3 + c) * hw + p]);
    o[3] = __float2half_rn(0.f);
    *reinterpret_cast<uint2*>(out + i * 4) = *reinterpret_cast<const uint2*>(o);
  }
}

// quant_conv (1x1, 8 -> 8) of conv_out's NHWC fp16 output [n, h, w, 8] in fp32, written as diffusers' `parameters`
// (the moments: mean in channels 0..3, logvar in 4..7) fp16 NCHW [n, 8, h, w].  wb: fp32 [8][8] weight then [8] bias.
// Fixed order, no contraction: out_c = ((b_c + w_c0 x_0) + w_c1 x_1) + ... + w_c7 x_7.
__global__ void vae_moments_kernel(const __half* __restrict__ x, long long npix, int hw, const float* __restrict__ wb,
                                   __half* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = *reinterpret_cast<const uint4*>(x + i * 8);
    const __half* h = reinterpret_cast<const __half*>(&v);
    float xs[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) xs[k] = __half2float(h[k]);
    const long long img = i / hw, p = i % hw;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float acc = wb[64 + c];
#pragma unroll
      for (int k = 0; k < 8; ++k) acc = __fadd_rn(acc, __fmul_rn(wb[c * 8 + k], xs[k]));
      out[(img * 8 + c) * hw + p] = __float2half_rn(acc);
    }
  }
}

// DiagonalGaussianDistribution: scale (mean + exp(0.5 clamp(logvar, -30, 20)) noise) in fp32 from the fp16 parameters
// [n, 8, h, w] and fp16 noise [n, 4, h, w]; without noise scale mean (the mode).  Output fp16 [n, 4, h, w] (layout 0) or
// [1, 4, n, h, w] (layout 1, the frames of one video as the inversion loop takes them).
__global__ void vae_posterior_kernel(const __half* __restrict__ prm, const __half* __restrict__ noise, int nimg, int hw,
                                     float scale, int layout, __half* __restrict__ out) {
  const long long total = (long long)nimg * 4 * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long img = i / (4LL * hw), r = i % (4LL * hw);
    const int c = (int)(r / hw);
    const long long p = r % hw;
    float v = __half2float(prm[(img * 8 + c) * hw + p]);
    if (noise != nullptr) {
      const float lv = fminf(fmaxf(__half2float(prm[(img * 8 + 4 + c) * hw + p]), -30.f), 20.f);
      v = __fadd_rn(v, __fmul_rn(expf(__fmul_rn(0.5f, lv)), __half2float(noise[i])));
    }
    const long long o = layout ? ((long long)c * nimg + img) * hw + p : i;
    out[o] = __float2half_rn(__fmul_rn(scale, v));
  }
}

inline unsigned capped(size_t n) {
  size_t b = (n + TPB - 1) / TPB;
  const size_t cap = (size_t)num_sms() * 16;
  return (unsigned)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

int small_linear(cudaStream_t st, const float* x, int rows, int K, const __half* W, const float* bias, int N, bool silu_in,
                 bool silu_out, float* out) {
  VS_REQUIRE(K % 2 == 0, "small_linear: K must be even");
  small_linear_kernel<<<blocks_for((size_t)N * 32), TPB, 0, st>>>(x, rows, K, W, bias, N, silu_in, silu_out, out);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int timestep_embedding(cudaStream_t st, const float* t, int B, int dim, float* out) {
  timestep_embedding_kernel<<<blocks_for((size_t)B * dim / 2), TPB, 0, st>>>(t, B, dim, out);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int conv_in_3x3(cudaStream_t st, const __half* x, int nimg, int H, int W, int cin, const __half* w, const float* bias,
                int cout, __half* out, __half* scratch) {
  VS_REQUIRE(cout % 8 == 0 && cin <= 8, "conv_in_3x3: needs cout %% 8 == 0 and cin <= 8");
  if (scratch != nullptr && cin == 4) {      // tensor-core path: patch rows [M][64] + weight [cout][64] in `scratch`
    const long long M = (long long)nimg * H * W;
    __half* wp = scratch + M * 64;
    conv_in_patch_kernel<<<capped((size_t)M * 8), TPB, 0, st>>>(x, nimg, H, W, reinterpret_cast<uint4*>(scratch));
    conv_in_pack_kernel<<<blocks_for((size_t)cout * 64), TPB, 0, st>>>(w, cout, wp);
    count_launch(2);
    VS_CHECK_CUDA(cudaGetLastError());
    GemmArgs g;
    g.A = scratch; g.K1 = 64; g.lda1 = 64; g.Bw = wp; g.M = (int)M; g.N = cout; g.bias = bias; g.out = out; g.ldc = cout;
    return gemm_tc(st, g);
  }
  const size_t smem = (size_t)9 * cin * cout * sizeof(float);
  VS_REQUIRE(smem <= 48 * 1024, "conv_in_3x3: weights do not fit shared memory");
  conv_in_kernel<<<capped((size_t)nimg * H * W * (cout / 8)), TPB, smem, st>>>(x, nimg, H, W, cin, w, bias, cout, out);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int upsample_nearest2x(cudaStream_t st, const __half* x, int nimg, int H, int W, int C, __half* out, int OH, int OW) {
  VS_REQUIRE(C % 8 == 0, "upsample: C %% 8 != 0");
  if (OH <= 0) OH = 2 * H;
  if (OW <= 0) OW = 2 * W;
  VS_REQUIRE((OH == 2 * H || OH == 2 * H - 1) && (OW == 2 * W || OW == 2 * W - 1),
             "upsample: output %dx%d is not 2x (or 2x - 1) of the %dx%d input", OH, OW, H, W);
  upsample2x_kernel<<<capped((size_t)nimg * OH * OW * (C / 8)), TPB, 0, st>>>(
      reinterpret_cast<const uint4*>(x), nimg, H, W, C / 8, OH, OW, reinterpret_cast<uint4*>(out));
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int im2col_s2(cudaStream_t st, const __half* x, int nimg, int H, int W, int C, __half* out) {
  VS_REQUIRE(C % 8 == 0, "im2col: C %% 8 != 0");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  im2col_s2_kernel<<<capped((size_t)nimg * Ho * Wo * 9 * (C / 8)), TPB, 0, st>>>(
      reinterpret_cast<const uint4*>(x), nimg, H, W, C / 8, Ho, Wo, reinterpret_cast<uint4*>(out));
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int add_inplace(cudaStream_t st, __half* x, const __half* r, size_t n, float scale) {
  add_kernel<<<capped(n / 8 + 1), TPB, 0, st>>>(x, r, n, scale);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int ncfhw_to_nhwc(cudaStream_t st, const void* src, int src_is_f32, int B, int C, int F, int H, int W, __half* dst) {
  const size_t n = (size_t)B * C * F * H * W;
  if (src_is_f32) ncfhw_to_nhwc_kernel<float><<<capped(n), TPB, 0, st>>>((const float*)src, B, C, F, H, W, dst);
  else ncfhw_to_nhwc_kernel<__half><<<capped(n), TPB, 0, st>>>((const __half*)src, B, C, F, H, W, dst);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int nhwc_to_ncfhw(cudaStream_t st, const __half* src, int B, int C, int F, int H, int W, void* dst, int dst_is_f32) {
  const size_t n = (size_t)B * C * F * H * W;
  if (dst_is_f32) nhwc_to_ncfhw_kernel<float><<<capped(n), TPB, 0, st>>>(src, B, C, F, H, W, (float*)dst);
  else nhwc_to_ncfhw_kernel<__half><<<capped(n), TPB, 0, st>>>(src, B, C, F, H, W, (__half*)dst);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int nchw_to_nhwc(cudaStream_t st, const __half* src, int n, int C, int H, int W, float scale, __half* dst) {
  const int HW = H * W;
  dim3 grid((HW + 31) / 32, (C + 31) / 32, n), block(32, 8);
  nchw_to_nhwc_kernel<<<grid, block, 0, st>>>(src, C, HW, scale, dst);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int cfg_ddim_step(cudaStream_t st, const void* eps2, const void* latents, int is_f32, size_t n, int cfg, float guidance,
                  float a_t, float a_prev, void* out) {
  const float c_x = sqrtf(a_prev) / sqrtf(a_t);
  const float c_e = sqrtf(1.f - a_prev) - sqrtf(a_prev) * sqrtf(1.f - a_t) / sqrtf(a_t);
  if (is_f32) cfg_ddim_kernel<float><<<capped(n), TPB, 0, st>>>((const float*)eps2, (const float*)latents, n, cfg, guidance, c_x, c_e, nullptr, (float*)out);
  else cfg_ddim_kernel<__half><<<capped(n), TPB, 0, st>>>((const __half*)eps2, (const __half*)latents, n, cfg, guidance, c_x, c_e, nullptr, (__half*)out);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int cfg_ddim_step_dev(cudaStream_t st, const void* eps2, const void* latents, int is_f32, size_t n, int cfg, float guidance,
                      const float* d_coef, void* out) {
  if (is_f32) cfg_ddim_kernel<float><<<capped(n), TPB, 0, st>>>((const float*)eps2, (const float*)latents, n, cfg, guidance, 0.f, 0.f, d_coef, (float*)out);
  else cfg_ddim_kernel<__half><<<capped(n), TPB, 0, st>>>((const __half*)eps2, (const __half*)latents, n, cfg, guidance, 0.f, 0.f, d_coef, (__half*)out);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
// One launch of cfg_ddim_rescale_kernel: S clusters of ncta CTAs.  The cluster dimension is only needed when the
// kernel may exchange statistics (CFG with a rescale factor that is > 0 or only known on the device).
static int cfg_ddim_rescale_launch(cudaStream_t st, const void* eps2, const void* latents, const void* noise, int is_f32,
                                   int S, size_t n_s, int cfg, float guidance, float c_x, float c_e, float c_n, float r,
                                   const float* d_coef, void* out) {
  const long long ns = (long long)n_s;
  const long long want = (ns + kRsThreads * 8 - 1) / (kRsThreads * 8);      // ~8 elements per thread
  const int ncta = want < 1 ? 1 : (want > kRsMaxCta ? kRsMaxCta : (int)want);
  const bool cluster = cfg && (d_coef != nullptr || r > 0.f) && ncta > 1;
  static bool configured = false;
  if (!configured) {
    VS_CHECK_CUDA(cudaFuncSetAttribute(cfg_ddim_rescale_kernel<float>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    VS_CHECK_CUDA(cudaFuncSetAttribute(cfg_ddim_rescale_kernel<__half>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    configured = true;
  }
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3((unsigned)(S * ncta));
  lc.blockDim = dim3(kRsThreads);
  lc.stream = st;
  cudaLaunchAttribute attr[1];
  if (cluster) {
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = ncta;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    lc.attrs = attr;
    lc.numAttrs = 1;
  }
  const int esz = is_f32 ? 4 : 2;
  // bytes: e_u (+ e_c), x, z read and x' written once; the rescale's second read of e comes from L2
  ProfScope prof(st, PC_OTHER, (double)S * ns * esz * ((cfg ? 2 : 1) + 2 + (noise ? 1 : 0)));
  if (is_f32)
    VS_CHECK_CUDA(cudaLaunchKernelEx(&lc, cfg_ddim_rescale_kernel<float>, (const float*)eps2, (const float*)latents,
                                     (const float*)noise, ns, S, ncta, cfg, guidance, c_x, c_e, c_n, r, d_coef, (float*)out));
  else
    VS_CHECK_CUDA(cudaLaunchKernelEx(&lc, cfg_ddim_rescale_kernel<__half>, (const __half*)eps2, (const __half*)latents,
                                     (const __half*)noise, ns, S, ncta, cfg, guidance, c_x, c_e, c_n, r, d_coef, (__half*)out));
  return 0;
}
int cfg_ddim_rescale_step(cudaStream_t st, const void* eps2, const void* latents, const void* noise, int is_f32, int S,
                          size_t n_s, int cfg, float guidance, float a_t, float a_prev, float eta, float rescale, void* out) {
  // diffusers 0.19.3 DDIMScheduler.step / _get_variance, in fp64 and rounded once (ops.ddim_coefficients is the same
  // expression in Python, so host- and device-coefficient launches agree bit for bit)
  const double at = a_t, ap = a_prev;
  const double cn = eta == 0.f ? 0.0 : (double)eta * sqrt((1.0 - ap) / (1.0 - at) * (1.0 - at / ap));
  const double cx = sqrt(ap) / sqrt(at);
  const double ce = sqrt(1.0 - ap - cn * cn) - sqrt(ap) * sqrt(1.0 - at) / sqrt(at);
  return cfg_ddim_rescale_launch(st, eps2, latents, noise, is_f32, S, n_s, cfg, guidance, (float)cx, (float)ce, (float)cn,
                                 rescale, nullptr, out);
}
int cfg_ddim_rescale_step_dev(cudaStream_t st, const void* eps2, const void* latents, const void* noise, int is_f32, int S,
                              size_t n_s, int cfg, float guidance, const float* d_coef, void* out) {
  return cfg_ddim_rescale_launch(st, eps2, latents, noise, is_f32, S, n_s, cfg, guidance, 0.f, 0.f, 0.f, 0.f, d_coef, out);
}
int adapter_splat(cudaStream_t st, const float* feat, const float* tracks, const int* point_mask, int F, int P, int C,
                  int h, int w, float rate, int coord_fp16, float scale, __half* maps) {
  VS_REQUIRE(C % 8 == 0, "adapter_splat: C %% 8 != 0");
  adapter_splat_kernel<<<capped((size_t)F * h * w * (C / 8)), TPB, 0, st>>>(feat, tracks, point_mask, F, P, C, h, w, rate,
                                                                            coord_fp16, scale, maps);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int blend_mask(cudaStream_t st, const __half* const* maps, const int* map_res, int n_maps, int n_prompts, int frames, int heads,
               int words, const float* alpha, int pool, int h, int w, float threshold, int both, float* mask) {
  VS_REQUIRE(maps && map_res && alpha && mask && n_maps >= 1 && n_prompts >= 1 && n_prompts <= 2, "blend_mask: bad arguments");
  VS_REQUIRE(frames >= 1 && heads >= 1 && words >= 1 && h >= 1 && w >= 1,
             "blend_mask: frames %d, heads %d, words %d and target %dx%d must all be >= 1", frames, heads, words, h, w);
  VS_REQUIRE(map_res[0] >= 1 && map_res[1] >= 1 && (long long)map_res[0] * map_res[1] <= kBlendMaxRes,
             "blend_mask: map resolution %dx%d must be at least 1x1 and at most %d pixels", map_res[0], map_res[1], kBlendMaxRes);
  blend_mask_kernel<<<frames, 256, 0, st>>>(maps, n_maps, n_prompts, frames, heads, map_res[0], map_res[1], words, alpha, pool, h, w,
                                            threshold, both, mask);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int latent_blend(cudaStream_t st, const void* x_src, void* x_tgt, const float* mask, int is_f32, int channels, int frames, int hw) {
  latent_blend_kernel<<<capped((size_t)channels * frames * hw), TPB, 0, st>>>(x_src, x_tgt, mask, is_f32, channels, frames, hw);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int pack_conv3x3(cudaStream_t st, const __half* w, int cout, int cin, __half* out) {
  pack_conv3x3_kernel<<<capped((size_t)cout * 9 * cin), TPB, 0, st>>>(w, cout, cin, out);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int pack_conv_subpixel(cudaStream_t st, const __half* w, int cout, int cin, __half* out, bool odd_panels) {
  pack_conv_subpixel_kernel<<<capped((size_t)cout * 16 * cin), TPB, 0, st>>>(w, cout, cin, out);
  count_launch(1);
  if (odd_panels) {
    pack_conv_subpixel_odd_kernel<<<capped((size_t)cout * 24 * cin), TPB, 0, st>>>(w, cout, cin, out + (size_t)cout * 16 * cin);
    count_launch(1);
  }
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int pack_geglu(cudaStream_t st, const __half* w, const __half* b, int hidden, int K, int granule, __half* wout, float* bout) {
  VS_REQUIRE(hidden % granule == 0, "pack_geglu: hidden %% granule != 0");
  pack_geglu_kernel<<<capped((size_t)2 * hidden * K), TPB, 0, st>>>(w, b, hidden, K, granule, wout, bout);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int ln_fold(cudaStream_t st, const __half* w, int N, int K, const float* gamma, const float* beta, const float* bias,
            const float* pe, int pe_len, __half* wf, float* u, float* c, float* cpe) {
  VS_REQUIRE(pe_len <= kMaxPe, "ln_fold: positional table longer than %d", kMaxPe);
  VS_REQUIRE(!pe || cpe, "ln_fold: positional table without an output");
  ln_fold_kernel<<<N, 128, 0, st>>>(w, N, K, gamma, beta, bias, pe, pe ? pe_len : 0, wf, u, c, cpe);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int vae_latent_in(cudaStream_t st, const void* z, int z_is_f32, int nimg, int h, int w, float divisor, const float* wb, __half* out) {
  VS_REQUIRE(z && wb && out && nimg > 0 && h > 0 && w > 0 && divisor != 0.f, "vae_latent_in: bad arguments");
  const long long npix = (long long)nimg * h * w;
  ProfScope prof(st, PC_OTHER, (double)npix * (4 * (z_is_f32 ? 4 : 2) + 8));   // bytes read + written
  if (z_is_f32) vae_latent_in_kernel<float><<<capped((size_t)npix), TPB, 0, st>>>((const float*)z, npix, h * w, divisor, wb, out);
  else vae_latent_in_kernel<__half><<<capped((size_t)npix), TPB, 0, st>>>((const __half*)z, npix, h * w, divisor, wb, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int image_postprocess(cudaStream_t st, const __half* x, int nimg, int H, int W, int cs, int format, void* out) {
  VS_REQUIRE(x && out && nimg > 0 && H > 0 && W > 0, "image_postprocess: bad arguments");
  VS_REQUIRE(cs >= 8 && cs % 8 == 0, "image_postprocess: the input's channel count must be a multiple of 8 (got %d)", cs);
  VS_REQUIRE(format >= IMG_SAMPLE && format <= IMG_PIL, "image_postprocess: unknown format %d", format);
  const long long npix = (long long)nimg * H * W;
  const int out_bytes = format == IMG_PIL ? 3 : (format == IMG_SAMPLE ? 6 : 12);
  ProfScope prof(st, PC_OTHER, (double)npix * (16 + out_bytes));
  image_postprocess_kernel<<<capped((size_t)npix), TPB, 0, st>>>(x, npix, H * W, cs, format, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int vae_image_in(cudaStream_t st, const void* x, int src, int nimg, int H, int W, __half* out) {
  VS_REQUIRE(x && out && nimg > 0 && H > 0 && W > 0, "vae_image_in: bad arguments");
  VS_REQUIRE(src >= VAE_IN_U8_NHWC && src <= VAE_IN_F32_NCHW, "vae_image_in: unknown source format %d", src);
  const long long npix = (long long)nimg * H * W;
  const int in_bytes = src == VAE_IN_U8_NHWC ? 3 : (src == VAE_IN_F16_NCHW ? 6 : 12);
  ProfScope prof(st, PC_OTHER, (double)npix * (in_bytes + 8));   // bytes read + written
  if (src == VAE_IN_U8_NHWC) vae_image_in_u8_kernel<<<capped((size_t)npix), TPB, 0, st>>>((const uint8_t*)x, npix, out);
  else if (src == VAE_IN_F16_NCHW) vae_image_in_nchw_kernel<__half><<<capped((size_t)npix), TPB, 0, st>>>((const __half*)x, npix, H * W, out);
  else vae_image_in_nchw_kernel<float><<<capped((size_t)npix), TPB, 0, st>>>((const float*)x, npix, H * W, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int vae_moments(cudaStream_t st, const __half* x, int nimg, int h, int w, const float* wb, __half* out) {
  VS_REQUIRE(x && wb && out && nimg > 0 && h > 0 && w > 0, "vae_moments: bad arguments");
  const long long npix = (long long)nimg * h * w;
  ProfScope prof(st, PC_OTHER, (double)npix * 32);   // 16 bytes read + 16 written per pixel
  vae_moments_kernel<<<capped((size_t)npix), TPB, 0, st>>>(x, npix, h * w, wb, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int vae_posterior(cudaStream_t st, const __half* params, const __half* noise, int nimg, int h, int w, float scale, int layout,
                  __half* out) {
  VS_REQUIRE(params && out && nimg > 0 && h > 0 && w > 0 && (layout | 1) == 1, "vae_posterior: bad arguments");
  const long long n = (long long)nimg * 4 * h * w;
  ProfScope prof(st, PC_OTHER, (double)n * (noise ? 8 : 4));   // bytes read + written
  vae_posterior_kernel<<<capped((size_t)n), TPB, 0, st>>>(params, noise, nimg, h * w, scale, layout, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}
int f16_to_f32(cudaStream_t st, const __half* x, size_t n, float* out) {
  f16_to_f32_kernel<<<capped(n), TPB, 0, st>>>(x, n, out);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace vs
