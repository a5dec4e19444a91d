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
__global__ void upsample2x_kernel(const uint4* __restrict__ x, int nimg, int H, int W, int CV, uint4* __restrict__ out) {
  const long long total = (long long)nimg * 4 * H * W * CV;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cv = i % CV;
    const long long pix = i / CV;
    const int xo = pix % (2 * W), yo = (pix / (2 * W)) % (2 * H);
    const long long img = pix / (4LL * W * H);
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

// x_tgt = x_src + mask * (x_tgt - x_src) per (channel, frame, pixel), in fp32 (spatial_blend.py:141-142); mask [frames, hw]
__global__ void latent_blend_kernel(const void* __restrict__ x_src, void* __restrict__ x_tgt, const float* __restrict__ mask,
                                    int is_f32, int channels, int frames, int hw) {
  const long long per_c = (long long)frames * hw, total = per_c * channels;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const float mk = mask[i % per_c];
    if (is_f32) {
      const float s = reinterpret_cast<const float*>(x_src)[i];
      float* t = reinterpret_cast<float*>(x_tgt) + i;
      *t = s + mk * (*t - s);
    } else {
      const float s = __half2float(reinterpret_cast<const __half*>(x_src)[i]);
      __half* t = reinterpret_cast<__half*>(x_tgt) + i;
      *t = __float2half_rn(s + mk * (__half2float(*t) - s));
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
int upsample_nearest2x(cudaStream_t st, const __half* x, int nimg, int H, int W, int C, __half* out) {
  VS_REQUIRE(C % 8 == 0, "upsample: C %% 8 != 0");
  upsample2x_kernel<<<capped((size_t)nimg * 4 * H * W * (C / 8)), TPB, 0, st>>>(
      reinterpret_cast<const uint4*>(x), nimg, H, W, C / 8, reinterpret_cast<uint4*>(out));
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
  VS_REQUIRE(map_res[0] * map_res[1] <= kBlendMaxRes, "blend_mask: map resolution %dx%d too large", map_res[0], map_res[1]);
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
int pack_conv_subpixel(cudaStream_t st, const __half* w, int cout, int cin, __half* out) {
  pack_conv_subpixel_kernel<<<capped((size_t)cout * 16 * cin), TPB, 0, st>>>(w, cout, cin, out);
  count_launch(1);
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
int f16_to_f32(cudaStream_t st, const __half* x, size_t n, float* out) {
  f16_to_f32_kernel<<<capped(n), TPB, 0, st>>>(x, n, out);
  count_launch(1);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace vs
