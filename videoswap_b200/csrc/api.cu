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

extern "C" int vs_cfg_ddim_rescale_step(void* stream, const void* d_eps2, const void* d_latents, const void* d_noise,
                                        int io_f32, int S, size_t n_s, int cfg, float guidance, float alpha_t,
                                        float alpha_prev, float eta, float guidance_rescale, void* d_out) {
  VS_REQUIRE(d_eps2 && d_latents && d_out && (d_noise || eta == 0.f), "vs_cfg_ddim_rescale_step: null pointer");
  VS_REQUIRE(S > 0 && n_s > 0, "vs_cfg_ddim_rescale_step: S = %d and n_s = %zu must be > 0", S, n_s);
  VS_REQUIRE(alpha_t > 0.f && alpha_t <= 1.f && alpha_prev > 0.f && alpha_prev <= 1.f,
             "vs_cfg_ddim_rescale_step: alphas must be in (0,1]");
  VS_REQUIRE(eta >= 0.f && (eta == 0.f || alpha_t < 1.f), "vs_cfg_ddim_rescale_step: eta must be >= 0 (and alpha_t < 1 when > 0)");
  VS_REQUIRE(guidance_rescale >= 0.f, "vs_cfg_ddim_rescale_step: guidance_rescale must be >= 0");
  return cfg_ddim_rescale_step((cudaStream_t)stream, d_eps2, d_latents, d_noise, io_f32, S, n_s, cfg, guidance, alpha_t,
                               alpha_prev, eta, guidance_rescale, d_out);
}

extern "C" int vs_cfg_ddim_rescale_step_dev(void* stream, const void* d_eps2, const void* d_latents, const void* d_noise,
                                            int io_f32, int S, size_t n_s, int cfg, float guidance, const float* d_coef,
                                            void* d_out) {
  VS_REQUIRE(d_eps2 && d_latents && d_out && d_coef, "vs_cfg_ddim_rescale_step_dev: null pointer");
  VS_REQUIRE(S > 0 && n_s > 0, "vs_cfg_ddim_rescale_step_dev: S = %d and n_s = %zu must be > 0", S, n_s);
  return cfg_ddim_rescale_step_dev((cudaStream_t)stream, d_eps2, d_latents, d_noise, io_f32, S, n_s, cfg, guidance, d_coef,
                                   d_out);
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

extern "C" int vs_gemm_ex(void* stream, const vs_gemm_desc* d) {
  VS_REQUIRE(d != nullptr, "vs_gemm_ex: null descriptor");
  GemmArgs g;
  g.A = (const __half*)d->A; g.K1 = d->K1; g.lda1 = d->lda1;
  g.A2 = (const __half*)d->A2; g.K2 = d->K2; g.lda2 = d->lda2;
  g.Bw = (const __half*)d->Bw;
  g.M = d->M; g.N = d->N;
  g.taps = d->taps;
  g.sub_py = d->sub_py; g.sub_px = d->sub_px;
  g.nimg = d->nimg; g.H = d->H; g.W = d->W;
  g.bias = d->bias;
  g.rowvec = d->rowvec; g.ldrv = d->ldrv; g.pix_per_batch = d->pix_per_batch; g.rv_mod = d->rv_mod;
  g.ln_stats = d->ln_stats; g.ln_u = d->ln_u;
  g.ln_parts = d->ln_parts; g.ln_nparts = d->ln_nparts;
  g.ln_sums_out = d->ln_sums_out;
  g.residual = (const __half*)d->residual; g.ldr = d->ldr;
  g.out = (__half*)d->out; g.ldc = d->ldc;
  g.mode = d->mode;
  g.force_bn = d->force_bn;
  g.OH = d->OH; g.OW = d->OW;
  g.stride2 = d->stride2;
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
extern "C" int vs_groupnorm_stats(void* stream, const void* d_x1, int c1, const void* d_x2, int c2, int nimg, int hw,
                                  int imgs_per_set, int groups, float* d_sums, int zero_first) {
  VS_REQUIRE(d_sums != nullptr, "vs_groupnorm_stats: null sums");
  return groupnorm_stats((cudaStream_t)stream, (const __half*)d_x1, c1, (const __half*)d_x2, c2, nimg, hw, imgs_per_set, groups,
                         d_sums, zero_first != 0);
}
extern "C" int vs_groupnorm_apply(void* stream, const void* d_x1, int c1, const void* d_x2, int c2, int nimg, int hw,
                                  int imgs_per_set, int groups, const float* d_sums, float eps, const float* d_gamma,
                                  const float* d_beta, int silu, int count_scale, void* d_out) {
  VS_REQUIRE(d_sums && d_out, "vs_groupnorm_apply: null pointer");
  VS_REQUIRE(count_scale >= 1, "vs_groupnorm_apply: count_scale must be >= 1");
  return groupnorm_apply((cudaStream_t)stream, (const __half*)d_x1, c1, (const __half*)d_x2, c2, nimg, hw, imgs_per_set, groups,
                         d_sums, eps, d_gamma, d_beta, silu != 0, (__half*)d_out, count_scale);
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
extern "C" int vs_upsample_conv3x3_sized(void* stream, const void* d_x, int nimg, int H, int W, int C, const void* d_w, int Cout,
                                         const float* d_bias, int OH, int OW, void* d_wpanels, void* d_out) {
  cudaStream_t st = (cudaStream_t)stream;
  VS_REQUIRE(d_x && d_w && d_wpanels && d_out && nimg >= 1 && H >= 1 && W >= 1, "vs_upsample_conv3x3_sized: bad arguments");
  __half* w3x3 = (__half*)d_wpanels;
  __half* wsub = w3x3 + (size_t)Cout * 9 * C;
  if (int e = pack_conv3x3(st, (const __half*)d_w, Cout, C, w3x3)) return e;
  if (int e = pack_conv_subpixel(st, (const __half*)d_w, Cout, C, wsub, true)) return e;
  return upsample_conv3x3(st, (const __half*)d_x, nimg, H, W, C, w3x3, wsub, d_bias, Cout, OH, OW, (__half*)d_out);
}
extern "C" int vs_upsample_nearest(void* stream, const void* d_x, int nimg, int H, int W, int C, int OH, int OW, void* d_out) {
  return upsample_nearest2x((cudaStream_t)stream, (const __half*)d_x, nimg, H, W, C, (__half*)d_out, OH, OW);
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
                                   const float* d_gamma, const float* d_beta, const float* d_pe, int pe_len, int hw,
                                   int frames, int mode, void* d_wf, float* d_u, float* d_c, float* d_cpe, float* d_parts,
                                   int parts_capacity, void* d_out) {
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = ln_fold(st, (const __half*)d_w, N, C, d_gamma, d_beta, d_bias, d_pe, pe_len, (__half*)d_wf, d_u, d_c, d_cpe)) return e;
  GemmArgs g0;                                  // producer: x = x0 W0^T + b0 (+ residual), row statistics from its epilogue
  g0.A = (const __half*)d_x0; g0.K1 = K0; g0.lda1 = K0; g0.Bw = (const __half*)d_w0; g0.M = M; g0.N = C; g0.bias = d_b0;
  g0.residual = (const __half*)d_residual; g0.ldr = C; g0.out = (__half*)d_x; g0.ldc = C; g0.ln_sums_out = d_parts;
  const int parts = gemm_n_tiles(g0);
  VS_REQUIRE(parts >= 1 && parts <= parts_capacity, "vs_linear_ln_linear: %d partial-sum slices do not fit the buffer (%d)", parts, parts_capacity);
  if (int e = gemm_tc(st, g0)) return e;
  GemmArgs g;                                   // consumer: LayerNorm(x) folded into this GEMM, statistics from the slices
  g.A = (const __half*)d_x; g.K1 = C; g.lda1 = C; g.Bw = (const __half*)d_wf; g.M = M; g.N = N; g.bias = d_c;
  g.ln_parts = d_parts; g.ln_nparts = parts; g.ln_u = d_u; g.out = (__half*)d_out; g.ldc = mode == EPI_GEGLU ? N / 2 : N; g.mode = mode;
  if (d_pe) { g.rowvec = d_cpe; g.ldrv = N; g.pix_per_batch = hw; g.rv_mod = frames; }
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
                          int cout, void* d_scratch, void* d_out) {
  return conv_in_3x3((cudaStream_t)stream, (const __half*)d_x, nimg, H, W, cin, (const __half*)d_w, d_bias, cout, (__half*)d_out,
                     (__half*)d_scratch);
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

extern "C" int vs_pack_conv_subpixel(void* stream, const void* d_w, int cout, int cin, void* d_out) {
  VS_REQUIRE(d_w && d_out, "vs_pack_conv_subpixel: null pointer");
  return pack_conv_subpixel((cudaStream_t)stream, (const __half*)d_w, cout, cin, (__half*)d_out);
}
extern "C" int vs_softmax_rows(void* stream, void* d_s, int rows, int n, int ld, float scale) {
  return softmax_rows((cudaStream_t)stream, (__half*)d_s, rows, n, ld, scale);
}
extern "C" int vs_transpose_pad(void* stream, const void* d_src, int rows, int cols, int rows_pad, void* d_dst) {
  return transpose_pad((cudaStream_t)stream, (const __half*)d_src, rows, cols, rows_pad, (__half*)d_dst);
}
extern "C" int vs_vae_latent_in(void* stream, const void* d_z, int z_is_f32, int nimg, int h, int w, float divisor,
                                const float* d_wb, void* d_out) {
  return vae_latent_in((cudaStream_t)stream, d_z, z_is_f32, nimg, h, w, divisor, d_wb, (__half*)d_out);
}
extern "C" int vs_image_postprocess(void* stream, const void* d_x, int nimg, int H, int W, int channels, int format, void* d_out) {
  return image_postprocess((cudaStream_t)stream, (const __half*)d_x, nimg, H, W, channels, format, d_out);
}
extern "C" int vs_downsample_conv3x3(void* stream, const void* d_x, int nimg, int H, int W, int C, const void* d_w_packed,
                                     int Cout, const float* d_bias, void* d_out) {
  VS_REQUIRE(d_x && d_w_packed && d_out, "vs_downsample_conv3x3: null pointer");
  GemmArgs g;
  g.A = (const __half*)d_x; g.K1 = C; g.lda1 = C; g.Bw = (const __half*)d_w_packed; g.taps = 9; g.stride2 = 1;
  g.nimg = nimg; g.H = H; g.W = W; g.M = nimg * (H / 2) * (W / 2); g.N = Cout; g.bias = d_bias; g.out = (__half*)d_out;
  g.ldc = Cout;
  return gemm_tc((cudaStream_t)stream, g);
}
extern "C" int vs_vae_image_in(void* stream, const void* d_x, int src_format, int nimg, int H, int W, void* d_out) {
  return vae_image_in((cudaStream_t)stream, d_x, src_format, nimg, H, W, (__half*)d_out);
}
extern "C" int vs_t2i_image_in(void* stream, const void* d_x, int nimg, int H, int W, int channels, void* d_out) {
  return t2i_image_in((cudaStream_t)stream, (const uint8_t*)d_x, nimg, H, W, channels, (__half*)d_out);
}
extern "C" int vs_avgpool2x2(void* stream, const void* d_x, int nimg, int H, int W, int C, void* d_out) {
  return avgpool2x2((cudaStream_t)stream, (const __half*)d_x, nimg, H, W, C, (__half*)d_out);
}
extern "C" int vs_scale_f16(void* stream, const void* d_x, size_t n, float scale, void* d_out) {
  return scale_f16((cudaStream_t)stream, (const __half*)d_x, n, scale, (__half*)d_out);
}
extern "C" int vs_vae_moments(void* stream, const void* d_x, int nimg, int h, int w, const float* d_wb, void* d_out) {
  return vae_moments((cudaStream_t)stream, (const __half*)d_x, nimg, h, w, d_wb, (__half*)d_out);
}
extern "C" int vs_vae_posterior(void* stream, const void* d_params, const void* d_noise, int nimg, int h, int w, float scale,
                                int layout, void* d_out) {
  return vae_posterior((cudaStream_t)stream, (const __half*)d_params, (const __half*)d_noise, nimg, h, w, scale, layout,
                       (__half*)d_out);
}
extern "C" int vs_clip_embed(void* stream, const int* d_ids_i32, int n, int L, const void* d_tok, int vocab, const void* d_pos, int C,
                             void* d_out) {
  return clip_embed((cudaStream_t)stream, d_ids_i32, n, L, (const __half*)d_tok, vocab, (const __half*)d_pos, C, (__half*)d_out);
}
extern "C" int vs_causal_attention(void* stream, const void* d_qkv, int ldqkv, void* d_o, int ldo, int nseq, int L, int heads,
                                   int d) {
  return causal_attention((cudaStream_t)stream, (const __half*)d_qkv, ldqkv, (__half*)d_o, ldo, nseq, L, heads, d);
}

extern "C" int vs_dift_noise(void* stream, const void* d_moments, const float* d_eps1, const float* d_eps2, int n, int E, int h,
                             int w, float sf, float sqrt_a, float sqrt_1ma, float* d_out) {
  return dift_noise((cudaStream_t)stream, (const __half*)d_moments, d_eps1, d_eps2, n, E, h, w, sf, sqrt_a, sqrt_1ma, d_out);
}
extern "C" int vs_dift_point_sample(void* stream, const void* d_feat, int n, int E, int h, int w, int C, int H, int W,
                                    const int* d_xy, int P, float* d_out) {
  return dift_point_sample((cudaStream_t)stream, (const __half*)d_feat, n, E, h, w, C, H, W, d_xy, P, d_out);
}
extern "C" int vs_dift_ensemble_mean(void* stream, const void* d_feat, int n, int E, int h, int w, int C, float* d_out) {
  return dift_ensemble_mean((cudaStream_t)stream, (const __half*)d_feat, n, E, h, w, C, d_out);
}
extern "C" int vs_dift_point_reduce(void* stream, const float* d_vecs, int n, int P, int C, const float* d_src,
                                    const int* d_src_row, float* d_conf, const void* d_accept, float* d_sums, float* d_counts,
                                    float* d_means) {
  return dift_point_reduce((cudaStream_t)stream, d_vecs, n, P, C, d_src, d_src_row, d_conf, (const uint8_t*)d_accept, d_sums,
                           d_counts, d_means);
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
