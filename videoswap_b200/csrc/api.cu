// extern "C" entry points declared in include/videoswap_b200.h (the model-handle functions live in unet.cu).
#include "../../include/videoswap_b200.h"
#include "common.cuh"
#include "kernels.h"

using namespace vs;

extern "C" const char* vs_last_error(void) { return vs::last_error(); }
extern "C" int vs_version(void) { return 100; }

extern "C" int vs_cfg_ddim_step(void* stream, const void* d_eps2, const void* d_latents, int io_f32, size_t n, int cfg,
                                float guidance, float alpha_t, float alpha_prev, void* d_out) {
  VS_REQUIRE(d_eps2 && d_latents && d_out, "vs_cfg_ddim_step: null pointer");
  VS_REQUIRE(alpha_t > 0.f && alpha_t <= 1.f && alpha_prev > 0.f && alpha_prev <= 1.f, "vs_cfg_ddim_step: alphas must be in (0,1]");
  return cfg_ddim_step((cudaStream_t)stream, d_eps2, d_latents, io_f32, n, cfg, guidance, alpha_t, alpha_prev, d_out);
}

extern "C" int vs_cfg_ddim_step_dev(void* stream, const void* d_eps2, const void* d_latents, int io_f32, size_t n, int cfg,
                                    float guidance, const float* d_coef, void* d_out) {
  VS_REQUIRE(d_eps2 && d_latents && d_out && d_coef, "vs_cfg_ddim_step_dev: null pointer");
  return cfg_ddim_step_dev((cudaStream_t)stream, d_eps2, d_latents, io_f32, n, cfg, guidance, d_coef, d_out);
}

extern "C" int vs_adapter_level(void* stream, const void* d_w0, const void* d_b0, const void* d_w1, const void* d_b1, int E,
                                int mid, int C, const float* d_pe, const float* d_tracks, const int* d_mask, int F, int P,
                                int h, int w, float rate, int coord_fp16, float scale, float* d_ws, void* d_map) {
  cudaStream_t st = (cudaStream_t)stream;
  VS_REQUIRE(d_w0 && d_b0 && d_w1 && d_b1 && d_pe && d_tracks && d_ws && d_map, "vs_adapter_level: null pointer");
  // d_ws: [mid] b0 f32 | [C] b1 f32 | [P, mid] hidden | [P, C] feat
  float* b0 = d_ws;
  float* b1 = b0 + mid;
  float* hid = b1 + C;
  float* feat = hid + (size_t)P * mid;
  if (int e = f16_to_f32(st, (const __half*)d_b0, mid, b0)) return e;
  if (int e = f16_to_f32(st, (const __half*)d_b1, C, b1)) return e;
  if (int e = small_linear(st, d_pe, P, E, (const __half*)d_w0, b0, mid, false, true, hid)) return e;   // Linear + SiLU
  if (int e = small_linear(st, hid, P, mid, (const __half*)d_w1, b1, C, false, false, feat)) return e;
  return adapter_splat(st, feat, d_tracks, d_mask, F, P, C, h, w, rate, coord_fp16, scale, (__half*)d_map);
}

extern "C" int vs_gemm(void* stream, const void* d_A, int K1, const void* d_A2, int K2, const void* d_W, int M, int N,
                       const float* d_bias, const float* d_rowvec, int pix_per_batch, const void* d_residual, void* d_out,
                       int mode, int force_bn) {
  GemmArgs g;
  g.A = (const __half*)d_A; g.K1 = K1; g.lda1 = K1; g.A2 = (const __half*)d_A2; g.K2 = K2; g.lda2 = K2;
  g.Bw = (const __half*)d_W; g.M = M; g.N = N; g.bias = d_bias; g.rowvec = d_rowvec; g.pix_per_batch = pix_per_batch;
  g.residual = (const __half*)d_residual; g.ldr = (mode == EPI_GEGLU) ? N / 2 : N;
  g.out = (__half*)d_out; g.ldc = (mode == EPI_GEGLU) ? N / 2 : N; g.mode = mode; g.force_bn = force_bn;
  return gemm_tc((cudaStream_t)stream, g);
}

extern "C" int vs_conv3x3(void* stream, const void* d_x, int C1, const void* d_x2, int C2, const void* d_w, int nimg, int H,
                          int W, int Cout, const float* d_bias, const float* d_rowvec, int imgs_per_batch,
                          const void* d_residual, void* d_out) {
  GemmArgs g;
  g.A = (const __half*)d_x; g.K1 = C1; g.lda1 = C1; g.A2 = (const __half*)d_x2; g.K2 = C2; g.lda2 = C2;
  g.Bw = (const __half*)d_w; g.taps = 9; g.nimg = nimg; g.H = H; g.W = W; g.M = nimg * H * W; g.N = Cout; g.bias = d_bias;
  g.rowvec = d_rowvec; g.pix_per_batch = imgs_per_batch * H * W; g.residual = (const __half*)d_residual; g.ldr = Cout;
  g.out = (__half*)d_out; g.ldc = Cout;
  return gemm_tc((cudaStream_t)stream, g);
}

extern "C" int vs_pack_conv3x3(void* stream, const void* d_w, int cout, int cin, void* d_out) {
  return pack_conv3x3((cudaStream_t)stream, (const __half*)d_w, cout, cin, (__half*)d_out);
}
extern "C" int vs_pack_geglu(void* stream, const void* d_w, const void* d_b, int hidden, int K, void* d_wout, float* d_bout) {
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = pack_geglu(st, (const __half*)d_w, nullptr, hidden, K, kGegluGranule, (__half*)d_wout, nullptr)) return e;
  return pack_geglu(st, nullptr, (const __half*)d_b, hidden, 1, kGegluGranule, nullptr, d_bout);
}

extern "C" int vs_groupnorm(void* stream, const void* d_x1, int c1, const void* d_x2, int c2, int nimg, int hw,
                            int imgs_per_set, int groups, float eps, const float* d_gamma, const float* d_beta, int silu,
                            float* d_sums, void* d_out) {
  cudaStream_t st = (cudaStream_t)stream;
  if (imgs_per_set == 1 && c2 == 0) {     // per-frame norm of one tensor: the single-pass cluster kernel, as in the UNet forward
    const int e = groupnorm_frame_fused(st, (const __half*)d_x1, c1, nimg, hw, groups, eps, d_gamma, d_beta, silu != 0, (__half*)d_out);
    if (e >= 0) return e;
  }
  if (int e = groupnorm_stats(st, (const __half*)d_x1, c1, (const __half*)d_x2, c2, nimg, hw, imgs_per_set, groups, d_sums)) return e;
  return groupnorm_apply(st, (const __half*)d_x1, c1, (const __half*)d_x2, c2, nimg, hw, imgs_per_set, groups, d_sums, eps,
                         d_gamma, d_beta, silu != 0, (__half*)d_out);
}
extern "C" int vs_layernorm(void* stream, const void* d_x, int rows, int C, const float* d_gamma, const float* d_beta,
                            const float* d_pe, int hw, int F, void* d_out) {
  return layernorm((cudaStream_t)stream, (const __half*)d_x, rows, C, d_gamma, d_beta, d_pe, hw, F, (__half*)d_out);
}
extern "C" int vs_ln_linear(void* stream, const void* d_x, int M, int C, const void* d_w, const float* d_bias, int N,
                            const float* d_gamma, const float* d_beta, const float* d_pe, int pe_len, int hw, int frames,
                            int mode, void* d_wf, float* d_u, float* d_c, float* d_cpe, float* d_stats, void* d_out) {
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = ln_fold(st, (const __half*)d_w, N, C, d_gamma, d_beta, d_bias, d_pe, pe_len, (__half*)d_wf, d_u, d_c, d_cpe)) return e;
  if (int e = ln_rowstats(st, (const __half*)d_x, M, C, d_stats)) return e;
  GemmArgs g;
  g.A = (const __half*)d_x; g.K1 = C; g.lda1 = C; g.Bw = (const __half*)d_wf; g.M = M; g.N = N; g.bias = d_c;
  g.ln_stats = d_stats; g.ln_u = d_u; g.out = (__half*)d_out; g.ldc = mode == EPI_GEGLU ? N / 2 : N; g.mode = mode;
  if (d_pe) { g.rowvec = d_cpe; g.ldrv = N; g.pix_per_batch = hw; g.rv_mod = frames; }
  return gemm_tc(st, g);
}
extern "C" int vs_upsample_conv3x3(void* stream, const void* d_x, int nimg, int H, int W, int C, const void* d_w, int Cout,
                                   const float* d_bias, void* d_wsub, void* d_out) {
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = pack_conv_subpixel(st, (const __half*)d_w, Cout, C, (__half*)d_wsub)) return e;
  for (int par = 0; par < 4; ++par) {
    GemmArgs g;
    g.A = (const __half*)d_x; g.K1 = C; g.lda1 = C; g.Bw = (const __half*)d_wsub + (size_t)par * Cout * 4 * C; g.taps = 4;
    g.sub_py = par >> 1; g.sub_px = par & 1; g.nimg = nimg; g.H = H; g.W = W; g.M = nimg * H * W; g.N = Cout; g.bias = d_bias;
    g.out = (__half*)d_out; g.ldc = Cout;
    if (int e = gemm_tc(st, g)) return e;
  }
  return 0;
}
extern "C" int vs_attention_probs(void* stream, const void* d_q, int ldq, const void* d_k, int ldk, void* d_probs, int batch, int nq,
                                  int nk, int heads, int d, long long q_bstride, long long kv_bstride, int kv_div) {
  return attention_probs((cudaStream_t)stream, (const __half*)d_q, ldq, (const __half*)d_k, ldk, (__half*)d_probs, batch, nq, nk, heads,
                         d, q_bstride, kv_bstride, kv_div);
}
extern "C" int vs_attention_apply_probs(void* stream, const void* d_probs, const void* d_v, int ldv, void* d_o, int ldo, int batch,
                                        int nq, int nk, int heads, int d, long long kv_bstride, long long o_bstride, int kv_div) {
  return attention_apply_probs((cudaStream_t)stream, (const __half*)d_probs, (const __half*)d_v, ldv, (__half*)d_o, ldo, batch, nq, nk,
                               heads, d, kv_bstride, o_bstride, kv_div);
}
extern "C" int vs_blend_mask(void* stream, const void* const* d_maps, int n_maps, int n_prompts, int frames, int heads, int res_h,
                             int res_w, int words, const float* d_alpha, int pool, int h, int w, float threshold, int both,
                             float* d_mask) {
  const int res[2] = {res_h, res_w};
  return blend_mask((cudaStream_t)stream, (const __half* const*)d_maps, res, n_maps, n_prompts, frames, heads, words, d_alpha, pool, h, w,
                    threshold, both, d_mask);
}
extern "C" int vs_latent_blend(void* stream, const void* d_x_src, void* d_x_tgt, const float* d_mask, int io_f32, int channels,
                               int frames, int hw) {
  return latent_blend((cudaStream_t)stream, d_x_src, d_x_tgt, d_mask, io_f32, channels, frames, hw);
}
extern "C" int vs_linear_ln_linear(void* stream, const void* d_x0, int M, int K0, const void* d_w0, const float* d_b0,
                                   const void* d_residual, int C, void* d_x, const void* d_w, const float* d_bias, int N,
                                   const float* d_gamma, const float* d_beta, int mode, void* d_wf, float* d_u, float* d_c,
                                   float* d_parts, int parts_capacity, void* d_out) {
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = ln_fold(st, (const __half*)d_w, N, C, d_gamma, d_beta, d_bias, nullptr, 0, (__half*)d_wf, d_u, d_c, nullptr)) return e;
  GemmArgs g0;                                  // producer: x = x0 W0^T + b0 (+ residual), row statistics from its epilogue
  g0.A = (const __half*)d_x0; g0.K1 = K0; g0.lda1 = K0; g0.Bw = (const __half*)d_w0; g0.M = M; g0.N = C; g0.bias = d_b0;
  g0.residual = (const __half*)d_residual; g0.ldr = C; g0.out = (__half*)d_x; g0.ldc = C; g0.ln_sums_out = d_parts;
  const int parts = gemm_n_tiles(g0);
  VS_REQUIRE(parts >= 1 && parts <= parts_capacity, "vs_linear_ln_linear: %d partial-sum slices do not fit the buffer (%d)", parts, parts_capacity);
  if (int e = gemm_tc(st, g0)) return e;
  GemmArgs g;                                   // consumer: LayerNorm(x) folded into this GEMM, statistics from the slices
  g.A = (const __half*)d_x; g.K1 = C; g.lda1 = C; g.Bw = (const __half*)d_wf; g.M = M; g.N = N; g.bias = d_c;
  g.ln_parts = d_parts; g.ln_nparts = parts; g.ln_u = d_u; g.out = (__half*)d_out; g.ldc = mode == EPI_GEGLU ? N / 2 : N; g.mode = mode;
  return gemm_tc(st, g);
}
extern "C" int vs_attention(void* stream, const void* d_q, int ldq, const void* d_k, int ldk, const void* d_v, int ldv,
                            void* d_o, int ldo, int batch, int nq, int nk, int heads, int d, long long q_bstride,
                            long long kv_bstride, long long o_bstride, int kv_div) {
  return attention((cudaStream_t)stream, (const __half*)d_q, ldq, (const __half*)d_k, ldk, (const __half*)d_v, ldv,
                   (__half*)d_o, ldo, batch, nq, nk, heads, d, q_bstride, kv_bstride, o_bstride, kv_div);
}
extern "C" int vs_temporal_attention(void* stream, const void* d_qkv, void* d_o, int B, int F, int HW, int C, int heads) {
  return temporal_attention((cudaStream_t)stream, (const __half*)d_qkv, (__half*)d_o, B, F, HW, C, heads);
}
extern "C" int vs_conv_in(void* stream, const void* d_x, int nimg, int H, int W, int cin, const void* d_w, const float* d_bias,
                          int cout, void* d_out) {
  return conv_in_3x3((cudaStream_t)stream, (const __half*)d_x, nimg, H, W, cin, (const __half*)d_w, d_bias, cout, (__half*)d_out);
}
extern "C" int vs_upsample2x(void* stream, const void* d_x, int nimg, int H, int W, int C, void* d_out) {
  return upsample_nearest2x((cudaStream_t)stream, (const __half*)d_x, nimg, H, W, C, (__half*)d_out);
}
extern "C" int vs_conv3x3_s2(void* stream, const void* d_x, int nimg, int H, int W, int C, const void* d_w, int Cout,
                             const float* d_bias, void* d_scratch, void* d_out) {
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = im2col_s2(st, (const __half*)d_x, nimg, H, W, C, (__half*)d_scratch)) return e;
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  GemmArgs g;
  g.A = (const __half*)d_scratch; g.K1 = 9 * C; g.lda1 = 9 * C; g.Bw = (const __half*)d_w; g.M = nimg * Ho * Wo; g.N = Cout;
  g.bias = d_bias; g.out = (__half*)d_out; g.ldc = Cout;
  return gemm_tc(st, g);
}

extern "C" int vs_profile_enable(int on) { prof_enable(on != 0); return 0; }
extern "C" int vs_profile_reset(void) { prof_reset(); return 0; }
extern "C" int vs_profile_collect(int category, double* ms, double* work, long long* count) {
  VS_REQUIRE(category >= 0 && category < PC_COUNT && ms && work && count, "vs_profile_collect: bad argument");
  return prof_collect(category, ms, work, count);
}
extern "C" long long vs_launch_count(void) { return launch_count(); }
extern "C" int vs_profile_dump(const char* path) {
  VS_REQUIRE(path != nullptr, "vs_profile_dump: null path");
  return prof_dump(path);
}
extern "C" int vs_set_option(const char* name, int value) {
  VS_REQUIRE(name != nullptr, "vs_set_option: null name");
  return set_option(name, value);
}
