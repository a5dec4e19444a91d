// Host-side launchers of the sm_90a kernels (all asynchronous on `st`, no hidden allocation, return 0 on success).
// Activation layout everywhere: NHWC fp16, i.e. tokens [(b f), h*w, C] with C innermost.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vs {

enum EpiMode { EPI_LINEAR = 0, EPI_GEGLU = 1, EPI_QUICK_GELU = 2, EPI_RELU = 3 };

// out[pix, n] = epilogue( sum_k A[pix(+tap shift), k] * Bw[n, k] )
//   * plain GEMM (taps == 1): A is [M, K1] (lda1) optionally followed along K by A2 [M, K2] (channel concat).
//   * 3x3 conv (taps == 9): A is NHWC [nimg, H, W, C1] (+ A2 [.., C2]); Bw is [N, 9*(C1+C2)], tap-major;
//     zero padding comes from TMA out-of-bounds fill.
//   epilogue: + bias[n] + rowvec[pix / pix_per_batch, n] + residual[pix, n]; EPI_GEGLU: value*gelu(gate) on
//   column-interleaved weights (see pack_geglu) -> N/2 output columns; EPI_QUICK_GELU: fp16((acc + bias) sigmoid(1.702
//   (acc + bias))) (CLIP's quick_gelu; plain GEMM with a bias only, BLOCK_N 128 / 256); EPI_RELU: fp16(max(acc + bias, 0))
//   (3x3 conv of one source with a bias only, N % 32 == 0; the T2I-Adapter's resnet block1).
struct GemmArgs {
  const __half* A = nullptr;  int K1 = 0;  int lda1 = 0;
  const __half* A2 = nullptr; int K2 = 0;  int lda2 = 0;
  const __half* Bw = nullptr;                 // [N, taps*(K1+K2)] fp16, K contiguous
  int M = 0, N = 0;
  int taps = 1;                               // 1, 9 (3x3, pad 1) or 4 (sub-pixel phase of nearest up-sampling + 3x3)
  int sub_py = 0, sub_px = 0;                 // taps == 4: output parity; writes pixel (2y+py, 2x+px) of the OH x OW output
  int nimg = 0, H = 0, W = 0;                 // conv geometry (taps == 9 / 4)
  const float* bias = nullptr;                // [N] fp32
  const float* rowvec = nullptr;              // [M / pix_per_batch, ldrv] fp32 (time-embedding add)
  int ldrv = 0;                               // row stride of rowvec (0 = N)
  int pix_per_batch = 1;
  int rv_mod = 0;                             // > 0: row-vector index = (pix / pix_per_batch) % rv_mod (per-frame vectors)
  // LayerNorm folded into this GEMM (A = the LayerNorm's RAW input, Bw = W * gamma, bias = beta W^T + b; see ln_fold):
  const float* ln_stats = nullptr;            // [M, 2] fp32 per-row (rstd, -mean * rstd) from ln_rowstats
  const float* ln_u = nullptr;                // [N] fp32 row sums of Bw
  // ... or, instead of ln_stats, the partial sums the PRODUCER of A wrote from its epilogue (ln_sums_out of that GEMM):
  const float* ln_parts = nullptr;            // [ln_nparts][M][2] fp32 (sum, sum of squares) over column tiles of A's producer
  int ln_nparts = 0;                          // = gemm_n_tiles(producer args)
  // This GEMM's output feeds a LayerNorm: write per-row (sum, sum of squares) of the stored fp16 values, one slice per
  // column tile: [gemm_n_tiles(*this)][M][2] fp32.  Plain linear layers only (+ bias / residual).
  float* ln_sums_out = nullptr;
  const __half* residual = nullptr; int ldr = 0;
  __half* out = nullptr; int ldc = 0;
  int mode = EPI_LINEAR;
  int force_bn = 0;                           // 0 = auto
  // taps == 4: output extent, 2H or 2H - 1 rows and 2W or 2W - 1 columns (0 = 2H / 2W).  Along an odd axis parity 0 has
  // 3 taps, so Bw holds 2x3, 3x2 or 3x3 taps (the panels pack_conv_subpixel / pack_conv3x3 make, see upsample_conv3x3).
  int OH = 0, OW = 0;
  // taps == 9 with stride2 != 0: 3x3 conv with stride 2 of pad(A, (0, 1, 0, 1)) (right / bottom zero padding, diffusers
  // Downsample2D(padding=0)); H, W = the input size (even), M = nimg (H / 2) (W / 2), one dense source, bias only.
  int stride2 = 0;
};
int gemm_tc(cudaStream_t st, const GemmArgs& a);
int gemm_n_tiles(const GemmArgs& a);         // column tiles gemm_tc will use (taps == 1)
constexpr int kGegluGranule = 128;           // value/gate column interleave granule (= BLOCK_N/2 of the GEGLU GEMM)

// ---- normalisation -------------------------------------------------------------------------------------------
// GroupNorm over `nstat` statistics sets; set s covers `imgs_per_set` consecutive images (5-D GroupNorm of the
// reference: imgs_per_set = F; per-frame GroupNorm: imgs_per_set = 1).  Input may be a virtual channel concat.
// sums: [nstat, groups, 2] fp32 (sum, sum of squares); zeroed inside groupnorm_stats.
int groupnorm_stats(cudaStream_t st, const __half* x1, int c1, const __half* x2, int c2, int nimg, int hw,
                    int imgs_per_set, int groups, float* sums, bool zero_first = true);
int groupnorm_apply(cudaStream_t st, const __half* x1, int c1, const __half* x2, int c2, int nimg, int hw,
                    int imgs_per_set, int groups, const float* sums, float eps, const float* gamma,
                    const float* beta, bool silu, __half* out, int count_scale = 1);   // count_scale: `sums` cover that many
                    // times the local elements (frame-sharded 5-D GroupNorm after the all-reduce of the sums)
// Per-frame GroupNorm in ONE pass (image resident in the shared memory of a thread-block cluster); -1 = shape not supported
int groupnorm_frame_fused(cudaStream_t st, const __half* x, int C, int nimg, int hw, int groups, float eps, const float* gamma,
                          const float* beta, bool silu, __half* out);
// LayerNorm over the last dim of [rows, C]; optional temporal positional encoding pe[(row / hw) % F, :] added after.
int layernorm(cudaStream_t st, const __half* x, int rows, int C, const float* gamma, const float* beta,
              const float* pe, int hw, int F, __half* out);

// LayerNorm folded into the GEMM that consumes it (GemmArgs::ln_stats / ln_u): per-row statistics of the raw input and
// the one-time transformation of the weights; C must be 320 / 640 / 1280 (ln_fold_supported).
bool ln_fold_supported(int C);
int ln_rowstats(cudaStream_t st, const __half* x, long long rows, int C, float* stats);   // stats [rows, 2] = (rstd, -mean rstd)
int ln_fold(cudaStream_t st, const __half* w, int N, int K, const float* gamma, const float* beta, const float* bias,
            const float* pe, int pe_len, __half* wf, float* u, float* c, float* cpe);   // see pointwise.cu

// ---- attention -----------------------------------------------------------------------------------------------
// Spatial self/cross attention, all heads: q[b, nq, h, d] (row stride ldq), k/v[b, nk, h, d] (ldk/ldv) -> o (ldo).
int attention(cudaStream_t st, const __half* q, int ldq, const __half* k, int ldk, const __half* v, int ldv,
              __half* o, int ldo, int batch, int nq, int nk, int heads, int d, long long q_bstride,
              long long kv_bstride, long long o_bstride, int kv_div);   // k/v batch index = batch / kv_div
// wgmma/TMA implementation (d = 40, 80); returns -1 if the shape is not supported by it.
int attention_tc(cudaStream_t st, const __half* q, int ldq, const __half* k, int ldk, const __half* v, int ldv,
                 __half* o, int ldo, int batch, int nq, int nk, int heads, int d, long long q_bstride,
                 long long kv_bstride, long long o_bstride, int kv_div);
// Explicit-probability attention for the prompt-to-prompt controllers (small-resolution layers only): softmax
// probabilities [batch, heads, nq, nk] fp16 to HBM, then O = P V from the (possibly edited) probabilities.
int attention_probs(cudaStream_t st, const __half* q, int ldq, const __half* k, int ldk, __half* probs, int batch, int nq, int nk,
                    int heads, int d, long long q_bstride, long long kv_bstride, int kv_div);
int attention_apply_probs(cudaStream_t st, const __half* probs, const __half* v, int ldv, __half* o, int ldo, int batch, int nq,
                          int nk, int heads, int d, long long kv_bstride, long long o_bstride, int kv_div);
// runtime options: "attn_tc" (1 = use the wgmma attention kernel where supported, default 1)
int set_option(const char* name, int value);
int get_option(const char* name);
// Temporal attention across F frames per pixel: qkv [B, F, HW, 3C] -> o [B, F, HW, C].
int temporal_attention(cudaStream_t st, const __half* qkv, __half* o, int B, int F, int HW, int C, int heads);
// Row softmax of s [rows, ld] fp16 in place over the first n columns (fp32 math, logits s * scale); columns n .. ld - 1
// are set to 0.  ld % 8 == 0.
int softmax_rows(cudaStream_t st, __half* s, int rows, int n, int ld, float scale);
// dst [cols, rows_pad] = src [rows, cols]^T with zero columns rows .. rows_pad - 1.
int transpose_pad(cudaStream_t st, const __half* src, int rows, int cols, int rows_pad, __half* dst);

// ---- CLIP text encoder (text.cu) ---------------------------------------------------------------------------------
// out [n L, C] = fp16(tok[ids[s, t]] + pos[t]) (fp32 add, one rounding); ids int32 [n, L], every id in [0, vocab).
int clip_embed(cudaStream_t st, const int* ids, int n, int L, const __half* tok, int vocab, const __half* pos, int C,
               __half* out);
// Causal self-attention of nseq sequences of L <= 77 tokens: q / k / v of head h at columns h d, C + h d, 2 C + h d of
// qkv [nseq L, ldqkv] (C = heads d, d = 64) -> o [nseq L, ldo] at column h d.
int causal_attention(cudaStream_t st, const __half* qkv, int ldqkv, __half* o, int ldo, int nseq, int L, int heads, int d);

// ---- DIFT semantic points (dift.cu) ----------------------------------------------------------------------------------
// out fp32 [n E, 4, h, w] = sqrt_a sf (mu + exp(0.5 clamp(logvar, -30, 20)) eps1) + sqrt_1ma eps2, with mu / logvar of
// frame (row / E) from the VAE moments fp16 [n, 8, h, w]; eps1, eps2 fp32 [n E, 4, h, w].
int dift_noise(cudaStream_t st, const __half* moments, const float* eps1, const float* eps2, int n, int E, int h, int w,
               float sf, float sqrt_a, float sqrt_1ma, float* out);
// out fp32 [n, P, C]: ensemble mean of feat NHWC fp16 [n, E, h, w, C] up-sampled bilinearly (align_corners False) to
// H x W, read at the pixels xy int32 [n, P, 2] = (x, y) in [0, W) x [0, H) (torch's CPU source-index arithmetic).  C % 8 == 0.
int dift_point_sample(cudaStream_t st, const __half* feat, int n, int E, int h, int w, int C, int H, int W, const int* xy,
                      int P, float* out);
// out fp32 NCHW [n, C, h, w] = mean over E of feat NHWC fp16 [n, E, h, w, C]
int dift_ensemble_mean(cudaStream_t st, const __half* feat, int n, int E, int h, int w, int C, float* out);
// vecs fp32 [n, P, C].  With src: conf[f, p] = cosine(vecs[f, p], src[src_row[f P + p]]) (eps 1e-8).  With accept uint8
// [n, P]: sums / means [P, C] and counts [P] over the accepted frames, in frame order (any of the three may be null).
int dift_point_reduce(cudaStream_t st, const float* vecs, int n, int P, int C, const float* src, const int* src_row,
                      float* conf, const uint8_t* accept, float* sums, float* counts, float* means);

// ---- pointwise / small -----------------------------------------------------------------------------------------
int small_linear(cudaStream_t st, const float* x, int rows, int K, const __half* W, const float* bias, int N,
                 bool silu_in, bool silu_out, float* out);     // out[r,n] = act(sum_k f(x[r,k]) W[n,k] + b[n]), fp32
int timestep_embedding(cudaStream_t st, const float* t, int B, int dim, float* out);   // cat(cos, sin)
int conv_in_3x3(cudaStream_t st, const __half* x, int nimg, int H, int W, int cin, const __half* w, const float* bias,
                int cout, __half* out, __half* scratch = nullptr);   // conv_in (tiny Cin): with `scratch` (>= (nimg*H*W +
                // cout) * 64 halves, cin == 4) patch rows + tensor-core GEMM, else a direct CUDA-core kernel
// nearest up-sampling by 2 to an OH x OW output (OH in {2H - 1, 2H}, OW in {2W - 1, 2W}): out[y, x] = in[y / 2, x / 2]
int upsample_nearest2x(cudaStream_t st, const __half* x, int nimg, int H, int W, int C, __half* out, int OH = 0, int OW = 0);
int im2col_s2(cudaStream_t st, const __half* x, int nimg, int H, int W, int C, __half* out);  // [nimg*Ho*Wo, 9*C]
int add_inplace(cudaStream_t st, __half* x, const __half* r, size_t n, float scale);   // x += scale * r
int ncfhw_to_nhwc(cudaStream_t st, const void* src, int src_is_f32, int B, int C, int F, int H, int W, __half* dst);
int nhwc_to_ncfhw(cudaStream_t st, const __half* src, int B, int C, int F, int H, int W, void* dst, int dst_is_f32);
int nchw_to_nhwc(cudaStream_t st, const __half* src, int n, int C, int H, int W, float scale, __half* dst);
// VAE decoder entry: post_quant_conv(z / divisor), z NCHW [nimg, 4, h, w] (fp16, or fp32 with z_is_f32) -> NHWC fp16
// [nimg, h, w, 4]; wb fp32 = weight [4][4] then bias [4].
int vae_latent_in(cudaStream_t st, const void* z, int z_is_f32, int nimg, int h, int w, float divisor, const float* wb, __half* out);
// VAE decoder exit: channels 0..2 of NHWC fp16 x [nimg, H, W, cs] (cs % 8 == 0) in one of the formats below.
enum ImageFormat { IMG_SAMPLE = 0, IMG_PT = 1, IMG_NP = 2, IMG_PIL = 3 };
int image_postprocess(cudaStream_t st, const __half* x, int nimg, int H, int W, int cs, int format, void* out);
// VAE encoder entry: images -> NHWC fp16 [nimg, H, W, 4] with channel 3 zero.  uint8 NHWC frames [nimg, H, W, 3] are
// normalised as VaeImageProcessor.preprocess does (2 (u / 255) - 1); float NCHW [nimg, 3, H, W] are taken as they are.
enum VaeImageSource { VAE_IN_U8_NHWC = 0, VAE_IN_F16_NCHW = 1, VAE_IN_F32_NCHW = 2 };
int vae_image_in(cudaStream_t st, const void* x, int src, int nimg, int H, int W, __half* out);
// VAE encoder exit: quant_conv of conv_out's NHWC fp16 [nimg, h, w, 8] in fp32 -> moments fp16 NCHW [nimg, 8, h, w];
// wb fp32 = weight [8][8] then bias [8].
int vae_moments(cudaStream_t st, const __half* x, int nimg, int h, int w, const float* wb, __half* out);
// scale (mean + exp(0.5 clamp(logvar, -30, 20)) noise) (noise fp16 [nimg, 4, h, w], or null: scale mean) from the moments,
// fp16 [nimg, 4, h, w] (layout 0) or [1, 4, nimg, h, w] (layout 1).
int vae_posterior(cudaStream_t st, const __half* params, const __half* noise, int nimg, int h, int w, float scale, int layout,
                  __half* out);
// eps = u + s (c - u); x_prev = sqrt(a_p) (x - sqrt(1-a_t) eps)/sqrt(a_t) + sqrt(1-a_p) eps.  eps2: [2, n] (uncond
// first) or [1, n] when guidance is disabled (cfg == 0).
int cfg_ddim_step(cudaStream_t st, const void* eps2, const void* latents, int is_f32, size_t n, int cfg,
                  float guidance, float a_t, float a_prev, void* out);
// Same, with the two DDIM coefficients (c_x, c_e) read from device memory (CUDA-graph replayable across timesteps).
int cfg_ddim_step_dev(cudaStream_t st, const void* eps2, const void* latents, int is_f32, size_t n, int cfg,
                      float guidance, const float* d_coef, void* out);
// S samples of n_s elements: CFG, the per-sample rescale toward std(e_c) (rescale > 0, CFG only) and the DDIM step with
// eta: x' = c_x x + c_e e + c_n noise (noise [S, n_s] or null).  eps2: [2 S, n_s] (uncond block first) or [S, n_s].
int cfg_ddim_rescale_step(cudaStream_t st, const void* eps2, const void* latents, const void* noise, int is_f32, int S,
                          size_t n_s, int cfg, float guidance, float a_t, float a_prev, float eta, float rescale, void* out);
// Same, with (c_x, c_e, c_n, rescale) read from device memory.
int cfg_ddim_rescale_step_dev(cudaStream_t st, const void* eps2, const void* latents, const void* noise, int is_f32, int S,
                              size_t n_s, int cfg, float guidance, const float* d_coef, void* out);
// ---- T2I-Adapter (t2i_adapter.cu) --------------------------------------------------------------------------------
// uint8 frames [nimg, H, W, c] (c = 1 or 3, H and W multiples of 8) -> the pixel-unshuffled fp16 NHWC input of conv_in,
// [nimg, H / 8, W / 8, 64 c] with out[.., c' 64 + 8 i + j] = fp16(fp32(in[8 y + i, 8 x + j, c']) / 255).
int t2i_image_in(cudaStream_t st, const uint8_t* x, int nimg, int H, int W, int c, __half* out);
// 2x2 average pool, stride 2, NHWC fp16 [nimg, H, W, C] (H, W even, C % 8 == 0) -> [nimg, H / 2, W / 2, C], fp32 sum.
int avgpool2x2(cudaStream_t st, const __half* x, int nimg, int H, int W, int C, __half* out);
// out[i] = fp16(fp32(x[i]) * scale), n % 8 == 0; out may be x.
int scale_f16(cudaStream_t st, const __half* x, size_t n, float scale, __half* out);
// SparsePointAdapter splat: feat [P, C] fp32, tracks [F, P, 2] fp32 -> maps NHWC [F, h, w, C] fp16 (zeroed inside)
int adapter_splat(cudaStream_t st, const float* feat, const float* tracks, const int* point_mask, int F, int P, int C,
                  int h, int w, float rate, int coord_fp16, float scale, __half* maps);

// ---- multi-GPU exchanges (comm.cu; NCCL bound at run time) -----------------------------------------------------------
}  // namespace vs
struct vs_comm;
namespace vs {
int comm_rank(const vs_comm* c);
int comm_size(const vs_comm* c);
int comm_all_reduce_sum_f32(vs_comm* c, cudaStream_t st, float* buf, size_t n);             // in place
int comm_all_gather(vs_comm* c, cudaStream_t st, const void* send, void* recv, size_t bytes);
// frames <-> pixels re-sharding: src [n_outer][k][chunk] -> dst [k][n_outer][chunk] (gather = 0) or the inverse (gather = 1)
int comm_all_to_all_rows(vs_comm* c, cudaStream_t st, const __half* src, __half* dst, int n_outer, size_t chunk, int gather);

// ---- latent blend of the attention controllers (spatial_blend.py): see pointwise.cu
int blend_mask(cudaStream_t st, const __half* const* maps, const int* map_res, int n_maps, int n_prompts, int frames, int heads,
               int words, const float* alpha, int pool, int h, int w, float threshold, int both, float* mask);
int latent_blend(cudaStream_t st, const void* x_src, void* x_tgt, const float* mask, int is_f32, int channels, int frames, int hw);

// ---- weight packing --------------------------------------------------------------------------------------------
int pack_conv3x3(cudaStream_t st, const __half* w, int cout, int cin, __half* out);   // [co,ci,3,3] -> [co,tap,ci]
// nearest-2x upsampling followed by a 3x3 conv == four 2x2 convs on the LOW-resolution input, one per output parity
// (py, px): rows 2y+py-1..2y+py+1 of the up-sampled image come from source rows {y-1, y, y} (py = 0) or {y, y, y+1}
// (py = 1), so the 3 row taps collapse to 2 with weights {w[-1], w[0]+w[1]} / {w[-1]+w[0], w[1]}; same along x.
// out: [4 parities (py*2+px)][co][2x2 taps][ci] fp16 (weights summed in fp32, rounded once).  2.25x fewer FLOPs and no
// materialised up-sampled tensor.
// With odd_panels, 4 more panels follow for targets of odd size 2n - 1 (F.interpolate(size=...) of the reference's
// forward_upsample_size path): there row 2n - 1 of the up-sampled image is padding, so parity 0 keeps the taps
// {w[-1], w[0], w[1]} apart (the third one reads a shifted view, see gemm.cu): [co][3x2 taps][ci] for (py, px) = (0, 0),
// (0, 1) with an odd height, then [co][2x3 taps][ci] for (0, 0), (1, 0) with an odd width (24 taps; 40 in all).  Parity
// (0, 0) with both axes odd is the plain 3x3 panel (pack_conv3x3).
int pack_conv_subpixel(cudaStream_t st, const __half* w, int cout, int cin, __half* out, bool odd_panels = false);
// Upsample3D: nearest up-sampling of NHWC x [nimg, H, W, C] to OH x OW, then the 3x3 conv, as 4 sub-pixel launches.
// w3x3: pack_conv3x3 panel (needed only for odd OH / OW); wsub: pack_conv_subpixel panels (with odd_panels for odd sizes).
int upsample_conv3x3(cudaStream_t st, const __half* x, int nimg, int H, int W, int C, const __half* w3x3, const __half* wsub,
                     const float* bias, int cout, int OH, int OW, __half* out);
int pack_geglu(cudaStream_t st, const __half* w, const __half* b, int hidden, int K, int granule, __half* wout,
               float* bout);   // rows interleaved value/gate in `granule` blocks; w or b may be null (pack one only)
int f16_to_f32(cudaStream_t st, const __half* x, size_t n, float* out);

}  // namespace vs
