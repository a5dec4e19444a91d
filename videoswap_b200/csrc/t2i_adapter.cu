// The pieces of diffusers 0.19.3's T2IAdapter (FullAdapter) that the GEMM / implicit-GEMM conv kernels do not cover: the
// image entry (/ 255, fp16 cast and PixelUnshuffle(8) in one pass), the AdapterBlock's 2x2 average pool and the
// t2i_guidance_scale multiply of the features (pipeline_videoswap.py:538-546).  conv_in and block1 (3x3, block1 with the
// ReLU epilogue), in_conv and block2 (1x1, block2 with the residual add) are gemm_tc launches.
#include "common.cuh"
#include "kernels.h"

namespace vs {
namespace {

constexpr int TPB = 256;

inline unsigned capped(size_t n) {
  size_t b = (n + TPB - 1) / TPB;
  const size_t cap = (size_t)num_sms() * 16;
  return (unsigned)(b < 1 ? 1 : (b > cap ? cap : b));
}

// One thread per (output pixel, row i of its 8 x 8 patch): reads the 8 c contiguous bytes of input row 8 y + i,
// columns 8 x .. 8 x + 7, and writes channels c' 64 + 8 i .. c' 64 + 8 i + 7 (one 16-byte store per input channel c').
template <int CH>
__global__ void t2i_image_in_kernel(const uint8_t* __restrict__ x, int nimg, int H, int W, __half* __restrict__ out) {
  const int ho = H / 8, wo = W / 8;
  const long long n = (long long)nimg * ho * wo * 8;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(t & 7);
    const long long pix = t >> 3;                       // (img, y, x) of the output
    const int xo = (int)(pix % wo);
    const long long r = pix / wo;
    const int yo = (int)(r % ho);
    const long long img = r / ho;
    const uint8_t* src = x + ((img * H + 8 * yo + i) * W + 8 * xo) * CH;
    uint8_t v[8 * CH];
    if constexpr (CH == 1) {
      *reinterpret_cast<uint2*>(v) = *reinterpret_cast<const uint2*>(src);            // 8-byte aligned (W % 8 == 0)
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) reinterpret_cast<uint2*>(v)[k] = reinterpret_cast<const uint2*>(src)[k];   // 24 bytes
    }
    __half* dst = out + pix * (64 * CH) + 8 * i;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      __align__(16) __half o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = __float2half_rn(__fdiv_rn((float)v[j * CH + c], 255.f));
      *reinterpret_cast<uint4*>(dst + 64 * c) = *reinterpret_cast<const uint4*>(o);
    }
  }
}

// One thread per (output pixel, 8 channels): ((a + b) + (c + d)) * 0.25 in fp32, one rounding to fp16.
__global__ void avgpool2x2_kernel(const __half* __restrict__ x, int nimg, int H, int W, int C, __half* __restrict__ out) {
  const int ho = H / 2, wo = W / 2, cv = C / 8;
  const long long n = (long long)nimg * ho * wo * cv;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(t % cv);
    const long long pix = t / cv;
    const int xo = (int)(pix % wo);
    const long long r = pix / wo;
    const int yo = (int)(r % ho);
    const long long img = r / ho;
    const __half* p00 = x + ((img * H + 2 * yo) * W + 2 * xo) * C + 8 * c8;
    const uint4 q[4] = {*reinterpret_cast<const uint4*>(p00), *reinterpret_cast<const uint4*>(p00 + C),
                        *reinterpret_cast<const uint4*>(p00 + (long long)W * C),
                        *reinterpret_cast<const uint4*>(p00 + (long long)W * C + C)};
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 a = __half22float2(reinterpret_cast<const __half2*>(&q[0])[k]);
      const float2 b = __half22float2(reinterpret_cast<const __half2*>(&q[1])[k]);
      const float2 c = __half22float2(reinterpret_cast<const __half2*>(&q[2])[k]);
      const float2 d = __half22float2(reinterpret_cast<const __half2*>(&q[3])[k]);
      oh[k] = __floats2half2_rn(__fmul_rn(__fadd_rn(__fadd_rn(a.x, b.x), __fadd_rn(c.x, d.x)), 0.25f),
                                __fmul_rn(__fadd_rn(__fadd_rn(a.y, b.y), __fadd_rn(c.y, d.y)), 0.25f));
    }
    reinterpret_cast<uint4*>(out)[t] = o;
  }
}

// fp16(fp32(x) * scale): torch's fp16 tensor times a Python float
__global__ void scale_f16_kernel(const __half* __restrict__ x, size_t nv, float scale, __half* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
    uint4 a = reinterpret_cast<const uint4*>(x)[i];
    __half2* ah = reinterpret_cast<__half2*>(&a);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(ah[j]);
      ah[j] = __floats2half2_rn(__fmul_rn(f.x, scale), __fmul_rn(f.y, scale));
    }
    reinterpret_cast<uint4*>(out)[i] = a;
  }
}

}  // namespace

int t2i_image_in(cudaStream_t st, const uint8_t* x, int nimg, int H, int W, int c, __half* out) {
  VS_REQUIRE(x && out && nimg > 0 && H > 0 && W > 0, "t2i_image_in: bad arguments");
  VS_REQUIRE(c == 1 || c == 3, "t2i_image_in: frames have 1 (L) or 3 (RGB) channels, got %d", c);
  VS_REQUIRE(H % 8 == 0 && W % 8 == 0, "t2i_image_in: H = %d and W = %d must be multiples of 8", H, W);
  const size_t n = (size_t)nimg * (H / 8) * (W / 8) * 8;
  ProfScope prof(st, PC_OTHER, (double)nimg * H * W * c * 3);   // bytes read + written
  if (c == 1) t2i_image_in_kernel<1><<<capped(n), TPB, 0, st>>>(x, nimg, H, W, out);
  else t2i_image_in_kernel<3><<<capped(n), TPB, 0, st>>>(x, nimg, H, W, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int avgpool2x2(cudaStream_t st, const __half* x, int nimg, int H, int W, int C, __half* out) {
  VS_REQUIRE(x && out && nimg > 0 && H > 0 && W > 0 && C > 0, "avgpool2x2: bad arguments");
  VS_REQUIRE(H % 2 == 0 && W % 2 == 0 && C % 8 == 0, "avgpool2x2: needs an even H (%d) and W (%d) and C %% 8 == 0 (C = %d)",
             H, W, C);
  const size_t n = (size_t)nimg * (H / 2) * (W / 2) * (C / 8);
  ProfScope prof(st, PC_OTHER, (double)nimg * H * W * C * 2 * 1.25);   // bytes read + written
  avgpool2x2_kernel<<<capped(n), TPB, 0, st>>>(x, nimg, H, W, C, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int scale_f16(cudaStream_t st, const __half* x, size_t n, float scale, __half* out) {
  VS_REQUIRE(x && out && n % 8 == 0, "scale_f16: bad arguments (n = %zu must be a multiple of 8)", n);
  ProfScope prof(st, PC_OTHER, (double)n * 4);
  scale_f16_kernel<<<capped(n / 8), TPB, 0, st>>>(x, n / 8, scale, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace vs
