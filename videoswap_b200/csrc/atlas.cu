// Layered-atlas point propagation (the reference's propagate_point_displacement.py and the IMLP_Hash "origin" MLP of
// videoswap/atlas/implicit_neural_networks.py) on sm_90a.  Everything is fp32 on the CUDA cores: the propagation takes
// finite differences with steps of 0.1 and 0.05 and rounds the result to whole pixels, so the MLPs keep fp32 products.
//  * imlp_kernel:          a whole IMLP_Hash forward for a tile of rows in one CTA: the positional encoding, every linear
//                          (ReLU before all but the first, the skip concatenations) and the tanh.  Activations stay in
//                          shared memory ([features][rows], so a thread reads four rows with one 16-byte load); weights
//                          are W^T [K, N] read through the read-only path from L2.  A warp computes a 32 x 32 tile of
//                          the layer, a lane 4 rows x 8 columns, and the warps of a CTA split the layer's tiles.
//  * atlas_fg_inputs / atlas_inv_inputs / atlas_finalize: the element-wise stages around the three networks (finite
//                          difference inputs, the 2x2 Jacobians, the drag in uv space, the warp, alpha and the rounding).
#include "../../include/videoswap_b200.h"
#include "common.cuh"

namespace vs {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxSmem = 227 * 1024;
constexpr float kPi = 3.14159265358979323846f;
constexpr float kDx = 0.1f, kDy = 0.05f;    // compute_Wm's deltax / deltay

struct Net {
  const float* params;
  int in, out, hidden, layers, pe, enc, rows_per_cta;
  unsigned skip;
  bool tanh_out;
};

__host__ __device__ inline int layer_k(const Net& n, int i) {
  return i == 0 ? n.enc : ((n.skip >> i) & 1u) ? n.hidden + n.enc : n.hidden;
}
__host__ __device__ inline int layer_n(const Net& n, int i) { return i == n.layers - 1 ? n.out : n.hidden; }

// acc[r][c] += sum_k src[k][row r] wt[k][col c] over one input segment (smem src [K][R], global wt [K][N])
__device__ __forceinline__ void tile_segment(float (&acc)[4][8], const float* src, int K, int R, int r,
                                             const float* __restrict__ wt, int N, int c) {
#pragma unroll 4
  for (int k = 0; k < K; ++k) {
    const float4 a = *reinterpret_cast<const float4*>(src + k * R + r);
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(wt + (size_t)k * N + c));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(wt + (size_t)k * N + c + 4));
    const float av[4] = {a.x, a.y, a.z, a.w};
    const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
  }
}

// One CTA: rows [row0, row0 + R) of x fp32 [rows, in] -> out fp32 [rows, out].
__global__ void __launch_bounds__(kThreads) imlp_kernel(Net net, const float* __restrict__ x, int rows,
                                                        float* __restrict__ out) {
  extern __shared__ __align__(16) float smem[];
  const int R = net.rows_per_cta, H = net.hidden, E = net.enc;
  float* enc = smem;                       // [E][R]
  float* cur = enc + E * R;                // [H][R]
  float* nxt = cur + H * R;                // [H][R]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int row0 = blockIdx.x * R;

  // positionalEncoding_vec: feature j (2 in) + c is sin(x_c b_j) for c < in, cos(x_(c - in) b_j) otherwise
  for (int i = tid; i < E * R; i += kThreads) {
    const int e = i / R, r = i % R, row = row0 + r;
    float v = 0.f;
    if (row < rows) {
      if (net.pe == 0) {
        v = x[(size_t)row * net.in + e];
      } else {
        const int j = e / (2 * net.in), c = e % (2 * net.in);
        const float arg = __fmul_rn(x[(size_t)row * net.in + (c % net.in)], ldexpf(kPi, j));   // fp32(2^j pi)
        v = c < net.in ? sinf(arg) : cosf(arg);
      }
    }
    enc[e * R + r] = v;
  }
  __syncthreads();

  const float* wl = net.params;
  const float* src = enc;
  for (int l = 0; l < net.layers; ++l) {
    const int K = layer_k(net, l), N = layer_n(net, l);
    const int K1 = l == 0 ? E : H;                         // the first segment: the encoding or the hidden state
    const bool skip = l > 0 && ((net.skip >> l) & 1u);
    const float* bias = wl + (size_t)K * N;
    const bool relu = l < net.layers - 1;                  // ReLU of the next layer's input, applied at the store
    if (N % 32 == 0) {
      const int ct = N / 32, tiles = ct * (R / 32);
      for (int t = warp; t < tiles; t += kWarps) {
        const int c = (t % ct) * 32 + (lane & 3) * 8, r = (t / ct) * 32 + (lane >> 2) * 4;
        float acc[4][8];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        tile_segment(acc, src, K1, R, r, wl, N, c);
        if (skip) tile_segment(acc, enc, E, R, r, wl + (size_t)H * N, N, c);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float b = __ldg(bias + c + j);
          float v[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) v[i] = relu ? fmaxf(__fadd_rn(acc[i][j], b), 0.f) : __fadd_rn(acc[i][j], b);
          *reinterpret_cast<float4*>(nxt + (c + j) * R + r) = make_float4(v[0], v[1], v[2], v[3]);
        }
      }
    } else {                                               // a narrow output layer: one thread per (row, column)
      for (int i = tid; i < N * R; i += kThreads) {
        const int n = i / R, r = i % R;
        float acc = 0.f;
        for (int k = 0; k < K1; ++k) acc = fmaf(src[k * R + r], __ldg(wl + (size_t)k * N + n), acc);
        if (skip)
          for (int k = 0; k < E; ++k) acc = fmaf(enc[k * R + r], __ldg(wl + (size_t)(H + k) * N + n), acc);
        const float v = __fadd_rn(acc, __ldg(bias + n));
        nxt[n * R + r] = relu ? fmaxf(v, 0.f) : v;
      }
    }
    __syncthreads();
    wl = bias + N;
    float* t = cur; cur = nxt; nxt = t;
    src = cur;
  }

  for (int i = tid; i < net.out * R; i += kThreads) {
    const int r = i / net.out, n = i % net.out, row = row0 + r;
    if (row < rows) {
      const float v = cur[n * R + r];
      out[(size_t)row * net.out + n] = net.tanh_out ? tanhf(v) : v;
    }
  }
}

size_t smem_bytes(const Net& n) { return (size_t)(n.enc + 2 * n.hidden) * n.rows_per_cta * sizeof(float); }

// Validates a descriptor (no launch) and fills the kernel's view of it.
int make_net(const vs_imlp_desc* d, const char* what, Net* n) {
  VS_REQUIRE(d != nullptr && d->d_params != nullptr, "%s: null descriptor or parameters", what);
  VS_REQUIRE(((uintptr_t)d->d_params & 15) == 0, "%s: parameters must be 16-byte aligned", what);
  VS_REQUIRE(d->hidden_dim >= 32 && d->hidden_dim <= 256 && d->hidden_dim % 32 == 0,
             "%s: hidden_dim %d is not a multiple of 32 in [32, 256]", what, d->hidden_dim);
  VS_REQUIRE(d->mlp_layers >= 1 && d->mlp_layers <= 32, "%s: mlp_layers %d is not in [1, 32]", what, d->mlp_layers);
  VS_REQUIRE(d->input_dim >= 1 && d->input_dim <= 8, "%s: input_dim %d is not in [1, 8]", what, d->input_dim);
  VS_REQUIRE(d->output_dim >= 1 && d->output_dim <= d->hidden_dim, "%s: output_dim %d is not in [1, hidden_dim]", what,
             d->output_dim);
  VS_REQUIRE(d->pe_dim >= 0 && d->pe_dim <= 16, "%s: pe_dim %d is not in [0, 16]", what, d->pe_dim);
  const unsigned valid = d->mlp_layers >= 32 ? 0xfffffffeu : ((1u << d->mlp_layers) - 1u) & ~1u;
  VS_REQUIRE((d->skip_mask & ~valid) == 0, "%s: skip_mask 0x%x names a layer outside [1, mlp_layers)", what,
             d->skip_mask);
  n->params = d->d_params;
  n->in = d->input_dim;
  n->out = d->output_dim;
  n->hidden = d->hidden_dim;
  n->layers = d->mlp_layers;
  n->pe = d->pe_dim;
  n->enc = d->pe_dim ? 2 * d->input_dim * d->pe_dim : d->input_dim;
  n->skip = d->skip_mask;
  n->tanh_out = d->use_tanh != 0;
  const int col_tiles = d->hidden_dim / 32;
  n->rows_per_cta = 32 * ((kWarps + col_tiles - 1) / col_tiles);   // at least one 32 x 32 tile per warp
  VS_REQUIRE(smem_bytes(*n) <= (size_t)kMaxSmem, "%s: %d encoded features do not fit a %d-row tile in shared memory",
             what, n->enc, n->rows_per_cta);
  return 0;
}

int launch_imlp(cudaStream_t st, const Net& n, const float* x, int rows, float* out) {
  static bool attr = false;
  if (!attr) {
    VS_CHECK_CUDA(cudaFuncSetAttribute(imlp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
    attr = true;
  }
  double flops = 0;
  for (int l = 0; l < n.layers; ++l) flops += 2.0 * layer_k(n, l) * layer_n(n, l);
  ProfScope prof(st, PC_OTHER, flops * rows);
  const unsigned grid = (unsigned)((rows + n.rows_per_cta - 1) / n.rows_per_cta);
  imlp_kernel<<<grid, kThreads, smem_bytes(n), st>>>(n, x, rows, out);
  VS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// pts fp32 [P, 4] = (x, y, dx, dy) normalised; rows p, P + p, 2P + p of fg_in [3P, 3]: xyt, (x + 0.1, y, t), (x, y + 0.05, t)
__global__ void atlas_fg_inputs_kernel(const float* __restrict__ pts, float t_key, int P, float* __restrict__ fg_in) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const float x = pts[p * 4], y = pts[p * 4 + 1];
  const float rows[3][3] = {{x, y, t_key}, {__fadd_rn(x, kDx), y, t_key}, {x, __fadd_rn(y, kDy), t_key}};
#pragma unroll
  for (int s = 0; s < 3; ++s)
#pragma unroll
    for (int j = 0; j < 3; ++j) fg_in[((size_t)s * P + p) * 3 + j] = rows[s][j];
}

// One thread per (point p, frame f), row p F + f: the Jacobian of FG at the keyframe point, delta_uv = dx_dy @ J_fg, and
// the inverse network's inputs [uv, t_f], (u + 0.1, v, t_f), (u, v + 0.05, t_f) at rows q, PF + q, 2PF + q.
__global__ void atlas_inv_inputs_kernel(const float* __restrict__ pts, const float* __restrict__ fg_out, int P, int F,
                                        float* __restrict__ j_fg, float* __restrict__ delta_uv,
                                        float* __restrict__ inv_in) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long PF = (long long)P * F;
  if (q >= PF) return;
  const int p = (int)(q / F), f = (int)(q % F);
  const float u = fg_out[p * 2], v = fg_out[p * 2 + 1];
  const float J[4] = {__fdiv_rn(__fsub_rn(fg_out[(P + p) * 2], u), kDx), __fdiv_rn(__fsub_rn(fg_out[(P + p) * 2 + 1], v), kDx),
                      __fdiv_rn(__fsub_rn(fg_out[(2 * P + p) * 2], u), kDy),
                      __fdiv_rn(__fsub_rn(fg_out[(2 * P + p) * 2 + 1], v), kDy)};
  if (f == 0) {
    const float dx = pts[p * 4 + 2], dy = pts[p * 4 + 3];
#pragma unroll
    for (int i = 0; i < 4; ++i) j_fg[p * 4 + i] = J[i];
    delta_uv[p * 2] = __fadd_rn(__fmul_rn(dx, J[0]), __fmul_rn(dy, J[2]));
    delta_uv[p * 2 + 1] = __fadd_rn(__fmul_rn(dx, J[1]), __fmul_rn(dy, J[3]));
  }
  // torch.arange(F) / (F / 2) - 1 in fp32: a correctly rounded divide by fp32(F / 2), then the subtract
  const float t = __fsub_rn(__fdiv_rn((float)f, (float)(F * 0.5)), 1.f);
  const float rows[3][3] = {{u, v, t}, {__fadd_rn(u, kDx), v, t}, {u, __fadd_rn(v, kDy), t}};
#pragma unroll
  for (int s = 0; s < 3; ++s)
#pragma unroll
    for (int j = 0; j < 3; ++j) inv_in[((long long)s * PF + q) * 3 + j] = rows[s][j];
}

// One thread per (point, frame): J_inv[..., :2], warp = xyt_pred[:2] + delta_uv @ J_inv, the alpha test and the
// pixel: rint((w + 1) / 2 larger_dim) where 0.5 (alpha + 1) > 0.5, else -1.
__global__ void atlas_finalize_kernel(const float* __restrict__ inv_out, const float* __restrict__ alpha,
                                      const float* __restrict__ delta_uv, int P, int F, int larger_dim,
                                      float* __restrict__ j_inv, float* __restrict__ warp, float* __restrict__ tracks) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long PF = (long long)P * F;
  if (q >= PF) return;
  const int p = (int)(q / F), f = (int)(q % F);
  const float* b = inv_out + q * 3;
  const float* xu = inv_out + (PF + q) * 3;
  const float* xv = inv_out + (2 * PF + q) * 3;
  const float J[4] = {__fdiv_rn(__fsub_rn(xu[0], b[0]), kDx), __fdiv_rn(__fsub_rn(xu[1], b[1]), kDx),
                      __fdiv_rn(__fsub_rn(xv[0], b[0]), kDy), __fdiv_rn(__fsub_rn(xv[1], b[1]), kDy)};
  const float du = delta_uv[p * 2], dv = delta_uv[p * 2 + 1];
  const bool vis = __fmul_rn(0.5f, __fadd_rn(alpha[q], 1.f)) > 0.5f;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const float w = __fadd_rn(b[j], __fadd_rn(__fmul_rn(du, J[j]), __fmul_rn(dv, J[2 + j])));
    warp[q * 2 + j] = w;
    const float px = rintf(__fmul_rn(__fdiv_rn(__fadd_rn(w, 1.f), 2.f), (float)larger_dim));   // half to even
    tracks[((long long)f * P + p) * 2 + j] = vis ? px : -1.f;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) j_inv[q * 4 + i] = J[i];
}

}  // namespace
}  // namespace vs

using namespace vs;

extern "C" int vs_imlp_forward(void* stream, const vs_imlp_desc* net, const float* d_x, int rows, float* d_out) {
  Net n;
  if (int e = make_net(net, "vs_imlp_forward", &n)) return e;
  VS_REQUIRE(d_x && d_out && rows >= 1, "vs_imlp_forward: null input / output or rows %d < 1", rows);
  return launch_imlp((cudaStream_t)stream, n, d_x, rows, d_out);
}

extern "C" int vs_atlas_propagate(void* stream, const vs_imlp_desc* fg, const vs_imlp_desc* fg_inverse,
                                  const vs_imlp_desc* alpha, const float* d_points, float t_key, int P, int F,
                                  int larger_dim, float* d_ws, float* d_tracks) {
  Net nf, ni, na;
  if (int e = make_net(fg, "vs_atlas_propagate (FG_UV_Mapping)", &nf)) return e;
  if (int e = make_net(fg_inverse, "vs_atlas_propagate (FG_UV_Mapping_Inverse)", &ni)) return e;
  if (int e = make_net(alpha, "vs_atlas_propagate (F_Alpha)", &na)) return e;
  VS_REQUIRE(nf.in == 3 && nf.out == 2, "vs_atlas_propagate: FG_UV_Mapping must map 3 -> 2, not %d -> %d", nf.in, nf.out);
  VS_REQUIRE(ni.in == 3 && ni.out == 3, "vs_atlas_propagate: FG_UV_Mapping_Inverse must map 3 -> 3, not %d -> %d", ni.in,
             ni.out);
  VS_REQUIRE(na.in == 3 && na.out == 1, "vs_atlas_propagate: F_Alpha must map 3 -> 1, not %d -> %d", na.in, na.out);
  VS_REQUIRE(P >= 1 && F >= 1, "vs_atlas_propagate: P = %d and F = %d must both be >= 1", P, F);
  VS_REQUIRE(3LL * P * F <= 0x7fffffffLL, "vs_atlas_propagate: 3 P F = %lld rows is too many", 3LL * P * F);
  VS_REQUIRE(larger_dim >= 1, "vs_atlas_propagate: larger_dim %d < 1", larger_dim);
  VS_REQUIRE(d_points && d_ws && d_tracks, "vs_atlas_propagate: null points, workspace or tracks");
  cudaStream_t st = (cudaStream_t)stream;
  const long long PF = (long long)P * F;
  float* fg_in = d_ws;                // layout: see the header
  float* fg_out = fg_in + 9LL * P;
  float* j_fg = fg_out + 6LL * P;
  float* delta_uv = j_fg + 4LL * P;
  float* inv_in = delta_uv + 2LL * P;
  float* inv_out = inv_in + 9 * PF;
  float* alpha_out = inv_out + 9 * PF;
  float* j_inv = alpha_out + PF;
  float* warp = j_inv + 4 * PF;
  const unsigned eb = (unsigned)((PF + 255) / 256);
  {
    ProfScope prof(st, PC_OTHER, 48.0 * P);
    atlas_fg_inputs_kernel<<<(P + 255) / 256, 256, 0, st>>>(d_points, t_key, P, fg_in);
    VS_CHECK_CUDA(cudaGetLastError());
  }
  if (int e = launch_imlp(st, nf, fg_in, 3 * P, fg_out)) return e;
  {
    ProfScope prof(st, PC_OTHER, 36.0 * PF);
    atlas_inv_inputs_kernel<<<eb, 256, 0, st>>>(d_points, fg_out, P, F, j_fg, delta_uv, inv_in);
    VS_CHECK_CUDA(cudaGetLastError());
  }
  if (int e = launch_imlp(st, ni, inv_in, (int)(3 * PF), inv_out)) return e;
  if (int e = launch_imlp(st, na, inv_out, (int)PF, alpha_out)) return e;   // alpha at the predicted (x, y, t)
  {
    ProfScope prof(st, PC_OTHER, 68.0 * PF);
    atlas_finalize_kernel<<<eb, 256, 0, st>>>(inv_out, alpha_out, delta_uv, P, F, larger_dim, j_inv, warp, d_tracks);
    VS_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}
