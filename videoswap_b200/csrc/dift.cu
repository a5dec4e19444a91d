// DIFT semantic-point read-out (the reference's videoswap/utils/dift_util.py and extract_semantic_point.py:125-204) on
// sm_90a: the three small kernels around the UNet featurizer (vs_unet_forward_features).  All are HBM / latency bound.
//  * dift_noise_kernel:        z = sf (mu + sigma eps1) from the VAE moments of each frame, then DDPM add_noise at t:
//                              sqrt(a_t) z + sqrt(1 - a_t) eps2, fp32, one row per (frame, ensemble member).
//  * dift_point_sample_kernel: ensemble mean of the up_ft map read at integer pixels of nn.Upsample(size=(H, W),
//                              mode="bilinear", align_corners=False) without materialising the up-sampled map; source
//                              indices and the interpolation order of torch's CPU upsample_bilinear2d, in fp32.
//  * dift_cosine_kernel / dift_reduce_kernel: CosineSimilarity(dim=1, eps=1e-8) of target vectors against source rows,
//                              and per-point sums / counts / means over accepted (frame, point) pairs in frame order
//                              (one thread per channel walks the frames: no atomics, same order as the reference's +=).
#include "common.cuh"
#include "kernels.h"

namespace vs {
namespace {

constexpr int kTPB = 256;

inline unsigned grid_for(long long n) { return (unsigned)((n + kTPB - 1) / kTPB); }

__global__ void dift_noise_kernel(const __half* __restrict__ moments, const float* __restrict__ eps1,
                                  const float* __restrict__ eps2, int n, int E, int hw, float sf, float sa, float sb,
                                  float* __restrict__ out) {
  const long long total = (long long)n * E * 4 * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / (4LL * hw), r = i % (4LL * hw);   // row = frame * E + ensemble member
    const int c = (int)(r / hw);
    const long long p = r % hw;
    const long long f = row / E;
    const float mu = __half2float(moments[(f * 8 + c) * hw + p]);
    const float lv = fminf(fmaxf(__half2float(moments[(f * 8 + 4 + c) * hw + p]), -30.f), 20.f);
    const float z = __fmul_rn(__fadd_rn(mu, __fmul_rn(expf(__fmul_rn(0.5f, lv)), eps1[i])), sf);
    out[i] = __fadd_rn(__fmul_rn(sa, z), __fmul_rn(sb, eps2[i]));
  }
}

// torch's area_pixel_compute_source_index (align_corners False, linear) and the neighbour / weight of upsample_bilinear2d
__device__ __forceinline__ void src_index(int dst, int in, int out, int& i0, int& i1, float& l1) {
  const float scale = __fdiv_rn((float)in, (float)out);
  const float s = fmaxf(__fsub_rn(__fmul_rn(scale, __fadd_rn((float)dst, 0.5f)), 0.5f), 0.f);
  i0 = min((int)s, in - 1);                      // only a pixel outside the output (rejected by the host) clamps
  i1 = i0 < in - 1 ? i0 + 1 : in - 1;
  l1 = __fsub_rn(s, (float)i0);
}

// one thread per (frame, point, 8 channels); feat NHWC fp16 [n, E, h, w, C]
__global__ void dift_point_sample_kernel(const __half* __restrict__ feat, int n, int E, int h, int w, int C, int H, int W,
                                         const int* __restrict__ xy, int P, float* __restrict__ out) {
  const int cv = C / 8;
  const long long total = (long long)n * P * cv;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % cv);
  const long long fp = i / cv;                    // frame * P + point
  const long long f = fp / P;
  const int x = xy[fp * 2], y = xy[fp * 2 + 1];
  int y0, y1, x0, x1;
  float ly1, lx1;
  src_index(y, h, H, y0, y1, ly1);
  src_index(x, w, W, x0, x1, lx1);
  const float ly0 = __fsub_rn(1.f, ly1), lx0 = __fsub_rn(1.f, lx1);
  const int ys[2] = {y0, y1}, xs[2] = {x0, x1};
  float m[4][8];                                  // ensemble mean at the four neighbours (mean first, as the reference)
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float s[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = 0.f;
    for (int e = 0; e < E; ++e) {
      const __half* px = feat + ((((f * E + e) * h + ys[k >> 1]) * (long long)w + xs[k & 1]) * C) + c8 * 8;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(px));
      const __half2* vh = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 a = __half22float2(vh[j]);
        s[2 * j] = __fadd_rn(s[2 * j], a.x);
        s[2 * j + 1] = __fadd_rn(s[2 * j + 1], a.y);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) m[k][j] = __fdiv_rn(s[j], (float)E);
  }
  float4* o = reinterpret_cast<float4*>(out + fp * C + c8 * 8);
  float r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    // h0l (w0l x00 + w1l x01) + h1l (w0l x10 + w1l x11), each product and sum rounded (no contraction)
    const float t0 = __fadd_rn(__fmul_rn(m[0][j], lx0), __fmul_rn(m[1][j], lx1));
    const float t1 = __fadd_rn(__fmul_rn(m[2][j], lx0), __fmul_rn(m[3][j], lx1));
    r[j] = __fadd_rn(__fmul_rn(t0, ly0), __fmul_rn(t1, ly1));
  }
  o[0] = make_float4(r[0], r[1], r[2], r[3]);
  o[1] = make_float4(r[4], r[5], r[6], r[7]);
}

// NHWC fp16 [n, E, h, w, C] -> fp32 NCHW [n, C, h, w] ensemble mean; one thread per output element
__global__ void dift_mean_kernel(const __half* __restrict__ feat, int n, int E, int hw, int C, float* __restrict__ out) {
  const long long total = (long long)n * C * hw;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long p = i % hw, c = (i / hw) % C, f = i / ((long long)hw * C);
  float s = 0.f;
  for (int e = 0; e < E; ++e) s = __fadd_rn(s, __half2float(feat[((f * E + e) * hw + p) * C + c]));
  out[i] = __fdiv_rn(s, (float)E);
}

// one warp per (frame, point): cos = (x . y) / (max(|x|, eps) max(|y|, eps)), sums in fp64
__global__ void dift_cosine_kernel(const float* __restrict__ vecs, long long rows, int C, const float* __restrict__ src,
                                   const int* __restrict__ src_row, float* __restrict__ conf) {
  const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* a = vecs + r * C;
  const float* b = src + (long long)src_row[r] * C;
  double ab = 0, aa = 0, bb = 0;
  for (int c = lane; c < C; c += 32) {
    const double x = a[c], y = b[c];
    ab += x * y; aa += x * x; bb += y * y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ab += __shfl_xor_sync(0xffffffffu, ab, o);
    aa += __shfl_xor_sync(0xffffffffu, aa, o);
    bb += __shfl_xor_sync(0xffffffffu, bb, o);
  }
  if (lane == 0) conf[r] = (float)(ab / (fmax(sqrt(aa), 1e-8) * fmax(sqrt(bb), 1e-8)));
}

// one thread per (point, channel): frames in order, fp32 += as the reference's init_embedding[p] += feat
__global__ void dift_reduce_kernel(const float* __restrict__ vecs, const uint8_t* __restrict__ accept, int n, int P, int C,
                                   float* __restrict__ sums, float* __restrict__ counts, float* __restrict__ means) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)P * C) return;
  const int p = (int)(i / C), c = (int)(i % C);
  float s = 0.f, k = 0.f;
  for (int f = 0; f < n; ++f) {
    if (!accept[(long long)f * P + p]) continue;
    s = __fadd_rn(s, vecs[((long long)f * P + p) * C + c]);
    k = __fadd_rn(k, 1.f);
  }
  if (sums) sums[i] = s;
  if (counts && c == 0) counts[p] = k;
  if (means) means[i] = k != 0.f ? __fdiv_rn(s, k) : 0.f;
}

}  // namespace

int dift_noise(cudaStream_t st, const __half* moments, const float* eps1, const float* eps2, int n, int E, int h, int w,
               float sf, float sqrt_a, float sqrt_1ma, float* out) {
  VS_REQUIRE(moments && eps1 && eps2 && out && n > 0 && E > 0 && h > 0 && w > 0, "dift_noise: bad arguments");
  const long long total = (long long)n * E * 4 * h * w;
  ProfScope prof(st, PC_OTHER, (double)total * 12);   // two fp32 noise reads + fp32 write
  const long long b = grid_for(total);
  dift_noise_kernel<<<(unsigned)(b < (long long)num_sms() * 16 ? b : (long long)num_sms() * 16), kTPB, 0, st>>>(
      moments, eps1, eps2, n, E, h * w, sf, sqrt_a, sqrt_1ma, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int dift_point_sample(cudaStream_t st, const __half* feat, int n, int E, int h, int w, int C, int H, int W, const int* xy,
                      int P, float* out) {
  VS_REQUIRE(feat && xy && out && n > 0 && E > 0 && h > 0 && w > 0 && H > 0 && W > 0 && P > 0,
             "dift_point_sample: bad arguments");
  VS_REQUIRE(C > 0 && C % 8 == 0, "dift_point_sample: C = %d must be a positive multiple of 8", C);
  const long long total = (long long)n * P * (C / 8);
  ProfScope prof(st, PC_OTHER, (double)n * P * C * (4.0 * E * 2 + 4));
  dift_point_sample_kernel<<<grid_for(total), kTPB, 0, st>>>(feat, n, E, h, w, C, H, W, xy, P, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int dift_ensemble_mean(cudaStream_t st, const __half* feat, int n, int E, int h, int w, int C, float* out) {
  VS_REQUIRE(feat && out && n > 0 && E > 0 && h > 0 && w > 0 && C > 0, "dift_ensemble_mean: bad arguments");
  const long long total = (long long)n * C * h * w;
  ProfScope prof(st, PC_OTHER, (double)total * (2.0 * E + 4));
  dift_mean_kernel<<<grid_for(total), kTPB, 0, st>>>(feat, n, E, h * w, C, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int dift_point_reduce(cudaStream_t st, const float* vecs, int n, int P, int C, const float* src, const int* src_row,
                      float* conf, const uint8_t* accept, float* sums, float* counts, float* means) {
  VS_REQUIRE(vecs && n > 0 && P > 0 && C > 0, "dift_point_reduce: bad arguments");
  VS_REQUIRE((src == nullptr) == (conf == nullptr) && (src == nullptr) == (src_row == nullptr),
             "dift_point_reduce: src, src_row and conf go together");
  VS_REQUIRE(accept != nullptr || (sums == nullptr && counts == nullptr && means == nullptr),
             "dift_point_reduce: sums / counts / means need the accept flags");
  if (src) {
    const long long rows = (long long)n * P;
    ProfScope prof(st, PC_OTHER, (double)rows * C * 8);
    dift_cosine_kernel<<<grid_for(rows * 32), kTPB, 0, st>>>(vecs, rows, C, src, src_row, conf);
    VS_CHECK_CUDA(cudaGetLastError());
  }
  if (accept) {
    ProfScope prof(st, PC_OTHER, (double)n * P * C * 4);
    dift_reduce_kernel<<<grid_for((long long)P * C), kTPB, 0, st>>>(vecs, accept, n, P, C, sums, counts, means);
    VS_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}

}  // namespace vs
