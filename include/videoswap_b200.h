/* videoswap_b200 -- C ABI of the H100-native denoising hot path of showlab/VideoSwap.
 *
 * The reference has no FFI boundary (it is pure Python on PyTorch/diffusers); its seam for this path is the Python
 * call  AnimateDiffUNet3DModel.forward  (videoswap/models/animatediff_models/unet.py:328-481)  plus the CFG combine and
 * scheduler step of the denoising loop  (videoswap/pipelines/pipeline_videoswap.py:568-587).  This header is the
 * C-ABI a Python binding (ctypes, see INTEGRATION.md) calls instead; every entry point cites what it replaces.
 *
 * Conventions: every function returns 0 on success, non-zero on error (message: vs_last_error()).  All pointers
 * named d_* are DEVICE pointers owned by the caller (e.g. torch tensors' data_ptr()); `stream` is a cudaStream_t
 * passed as void*.  Calls are asynchronous on that stream; the library never synchronises the device.  The handle
 * owns the packed weights and the activation workspace; nothing is allocated after the first forward of a given
 * shape (CUDA-graph capturable).  One host thread per handle.
 */
#ifndef VIDEOSWAP_B200_H
#define VIDEOSWAP_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* vs_last_error(void);
int vs_version(void);

/* ---- model handle ---------------------------------------------------------------------------------------------
 * Mirrors the constructor arguments of AnimateDiffUNet3DModel that the SD-1.5 + AnimateDiff configuration uses
 * (unet.py:36-100; options/model_cfg/inference.yml of the reference). */
typedef struct vs_unet_config {
  int in_channels, out_channels;
  int block_out_channels[4];
  int layers_per_block;
  int num_heads;                 /* `attention_head_dim` of the SD-1.5 config == number of heads (unet.py:158) */
  int cross_attention_dim;
  int norm_num_groups;
  float norm_eps;
  int use_motion_module;
  int motion_down[4];            /* motion modules present in down block i / up block i */
  int motion_up[4];
  int motion_mid;
  int motion_num_heads;
  int pe_max_len;                /* temporal_position_encoding_max_len */
} vs_unet_config;

typedef struct vs_unet vs_unet;

int vs_unet_create(const vs_unet_config* cfg, vs_unet** out);
void vs_unet_destroy(vs_unet* h);

/* Replaces  unet.load_state_dict(...)  (pipeline_videoswap.py:303,418; convert_edlora_to_diffusers.py:94-96):
 * takes n tensors by diffusers state_dict key name (fp16 device pointers, shapes implied by the config) and re-packs
 * them into kernel layouts (conv [Co,tap,Ci]; fused QKV; GEGLU-interleaved FF).  May be called repeatedly (LoRA merge
 * / restore between editing prompts).  Unknown names are an error; missing names keep their previous value. */
int vs_unet_load_weights(vs_unet* h, void* stream, int n, const char* const* names, const void* const* d_ptrs,
                         const int64_t* numels);
/* Number of parameter tensors the handle expects and the i-th name (for completeness checks). */
int vs_unet_num_params(const vs_unet* h);
const char* vs_unet_param_name(const vs_unet* h, int i);

/* Replaces  AnimateDiffUNet3DModel.forward  (unet.py:328-481).
 *   d_sample   [B, C_in, F, H, W]  (fp16 if !io_f32 else fp32), NCFHW exactly as the reference passes it
 *   d_timesteps DEVICE array of B floats (the reference broadcasts a scalar timestep to B, unet.py:389); a device
 *              pointer keeps the call CUDA-graph replayable with a new timestep
 *   d_ehs      encoder hidden states fp16: [B, 77, D] (ehs_layers == 0) or ED-LoRA [B, L, 77, D] (ehs_layers == L;
 *              layer i of the 16 cross-attention layers reads slice i, utils/edlora_util.py:40-41,96-98)
 *   d_residuals 4 adapter maps (or NULL): NHWC fp16 [(B F), H_l, W_l, C_l] if residuals_nhwc else NCHW fp16
 *              [(B F), C_l, H_l, W_l] as the reference passes them (down_block_additional_residuals, unet.py:336);
 *              residual_scale multiplies them (t2i_guidance_scale, pipeline_videoswap.py:544-545)
 *   d_out      [B, C_out, F, H, W] same dtype as d_sample
 * Any H, W >= 1 (unet.py:356-364,454-457): level l has H_l = ceil(H_(l-1) / 2) (the stride-2 convs) and every up-sampler
 * targets the size of the skip it feeds; the adapter maps must have those level sizes. */
int vs_unet_forward(vs_unet* h, void* stream, const void* d_sample, int io_f32, int B, int F, int H, int W,
                    const float* d_timesteps, const void* d_ehs, int ehs_tokens, int ehs_layers,
                    const void* const* d_residuals, int residuals_nhwc, float residual_scale, void* d_out);
/* The DIFT featurizer (the reference's dift_util.py MyUNet2DConditionModel): the same forward as a UNet2DConditionModel --
 * time embedding, conv_in, down path, mid block and up blocks 0..up_ft_index, WITHOUT any motion module -- stopping after
 * up block up_ft_index and its up-sampler (the reference's up_ft[up_ft_index]).  Pass F = 1 with every image on B, so the
 * ResNet GroupNorm statistics are per image as in the 2-D UNet.  d_feat: NHWC fp16 [B F, h_k, w_k, C_k], C_k =
 * block_out_channels[3 - k] at level 2 - k for k < 3 (block_out_channels[0] at level 0 for k = 3), on the level sizes of
 * vs_unet_forward.  Fails before any launch for up_ft_index outside 0..3, a frame-sharded handle or a set attention hook. */
int vs_unet_forward_features(vs_unet* h, void* stream, const void* d_sample, int io_f32, int B, int F, int H, int W,
                             const float* d_timesteps, const void* d_ehs, int ehs_tokens, int ehs_layers, int up_ft_index,
                             void* d_feat);
/* The time embedding exactly as vs_unet_forward runs it, with the handle's loaded weights: d_timesteps fp32 [B] ->
 * d_emb fp32 [B, 4 block_out_channels[0]] (time_embedding(Timesteps(t))) and d_proj fp32 [B, tproj_n], every resnet's
 * time_emb_proj(SiLU(emb)) side by side in registration order (down blocks, mid block, up blocks; tproj_n is the sum of
 * their output channels).  Uses neither the workspace nor a captured graph's buffers. */
int vs_unet_time_embedding(vs_unet* h, void* stream, const float* d_timesteps, int B, float* d_emb, float* d_proj);
size_t vs_unet_workspace_bytes(const vs_unet* h);
/* The activation workspace is one arena that only grows: a forward of a smaller shape re-uses it.  A captured CUDA graph
 * holds raw pointers into it, so the owner of a graph pins the arena (pin != 0; unpin with 0 when the graph dies): while
 * pinned, a forward that would need a LARGER arena fails instead of re-allocating.  vs_unet_reserve_workspace sizes the
 * arena for a shape ahead of time (e.g. the CFG batch before the B = 1 inversion graph is captured). */
int vs_unet_pin_workspace(vs_unet* h, int pin);
int vs_unet_reserve_workspace(vs_unet* h, int B, int F, int H, int W);
/* ---- multi-GPU (SURVEY.md 8e; the reference has no inference-time parallelism) --------------------------------------
 * One process per GPU.  A vs_comm wraps one NCCL communicator (bound at run time with dlopen); the caller distributes
 * the 128-byte unique id (e.g. torch.distributed broadcast) and calls vs_comm_create on every rank of the group.
 * Frame sharding: rank `shard` of `nshards` holds frames [shard F/k, (shard+1) F/k) of ONE batch element and passes that
 * LOCAL frame count to vs_unet_forward.  Per forward the library exchanges (i) the (sum, sum of squares) of the 45
 * cross-frame GroupNorms (all-reduce of 64 floats each) and (ii) a frames <-> pixels all-to-all around each of the 20
 * motion modules; everything else is per frame.  The two CFG halves live on two such groups and swap their noise
 * predictions with vs_comm_all_gather before vs_cfg_ddim_step.  All exchanges are asynchronous on `stream` and CUDA-
 * graph capturable. */
typedef struct vs_comm vs_comm;
int vs_comm_unique_id(void* out128);
int vs_comm_create(const void* id128, int rank, int nranks, vs_comm** out);
void vs_comm_destroy(vs_comm* c);
int vs_comm_all_gather(vs_comm* c, void* stream, const void* d_send, void* d_recv, size_t bytes_per_rank);
int vs_comm_all_reduce_sum_f32(vs_comm* c, void* stream, float* d_buf, size_t n);
int vs_unet_set_frame_shard(vs_unet* h, vs_comm* frame_comm, int shard, int nshards);

/* ---- attention controllers (prompt-to-prompt; utils/p2p_utils/attention_register.py:15-97,140-150) ---------------------
 * The reference swaps a control processor into every attn1 / attn2: layers with fewer than 32^2 queries materialise their
 * softmax probabilities [(b f), heads, s, t] and pass them through `controller(attn, is_cross, place_in_unet)` before P V.
 * Here: while a hook is set, vs_unet_forward runs exactly those layers (the 16x16 / 8x8 levels) through the explicit-
 * probability kernels and calls the hook between the softmax and P V with the DEVICE tensor (fp16, contiguous); the hook
 * may read it (store) and overwrite it in place (refine / replace) with work enqueued on `stream`.  `layer` = index of the
 * transformer block in registration order (down -> mid -> up, 0..15), `place` = 0 down / 1 mid / 2 up.  Hook mode runs
 * eagerly (it cannot be captured in a CUDA graph).  max_queries <= 0 selects the reference's 32^2. */
typedef void (*vs_attention_hook)(void* user, int layer, int is_cross, int place, void* d_probs, int batch, int heads, int nq,
                                  int nk, void* stream);
int vs_unet_set_attention_hook(vs_unet* h, vs_attention_hook hook, void* user, int max_queries);
/* The two halves of that path as stand-alone entry points (parity tests): probabilities [batch, heads, nq, nk] fp16, then
 * O = P V.  Same argument conventions as vs_attention. */
int vs_attention_probs(void* stream, const void* d_q, int ldq, const void* d_k, int ldk, void* d_probs, int batch, int nq, int nk,
                       int heads, int d, long long q_bstride, long long kv_bstride, int kv_div);
int vs_attention_apply_probs(void* stream, const void* d_probs, const void* d_v, int ldv, void* d_o, int ldo, int batch, int nq,
                             int nk, int heads, int d, long long kv_bstride, long long o_bstride, int kv_div);
/* Latent blend of the controllers (utils/p2p_utils/spatial_blend.py:25-63,141-142) on device.
 * vs_blend_mask: d_maps = DEVICE array of n_maps * n_prompts pointers (layer-major, prompt 0 = source, 1 = target), each an
 * fp16 cross-attention map [frames, heads, res_h * res_w, words]; d_alpha [n_prompts, words] fp32 word selector;
 * mask[p, f, y, x] = (nearest-resize(maxpool3x3(mean_{layer,head} sum_w alpha map)) / max > threshold), and with `both`
 * mask[p] |= mask[0].  d_mask: [n_prompts, frames, h, w] fp32.
 * vs_latent_blend: x_tgt = x_src + mask * (x_tgt - x_src), x [channels, frames, h*w] (fp16 or fp32), mask [frames, h*w]. */
int vs_blend_mask(void* stream, const void* const* d_maps, int n_maps, int n_prompts, int frames, int heads, int res_h, int res_w,
                  int words, const float* d_alpha, int pool, int h, int w, float threshold, int both, float* d_mask);
int vs_latent_blend(void* stream, const void* d_x_src, void* d_x_tgt, const float* d_mask, int io_f32, int channels, int frames,
                    int hw);

/* Debug taps: after the next forward, copies of named intermediate activations (NHWC fp16) can be fetched. */
int vs_unet_enable_taps(vs_unet* h, int enable);
int vs_unet_num_taps(const vs_unet* h);
int vs_unet_get_tap(const vs_unet* h, int i, const char** name, const void** d_ptr, int* nimg, int* hh, int* ww, int* c);
int vs_unet_copy_tap(const vs_unet* h, void* stream, int i, void* d_dst);   /* NHWC fp16 [nimg, hh, ww, c] */

/* Replaces the CFG combine + DDIMScheduler.step of the loop body (pipeline_videoswap.py:578-587; diffusers
 * DDIMScheduler.step, eta = 0):  eps = eps_u + g (eps_c - eps_u);  x' = sqrt(a_p) (x - sqrt(1-a_t) eps)/sqrt(a_t)
 * + sqrt(1-a_p) eps.   d_eps2: [2, n] (uncond first) when cfg != 0 else [1, n]; d_latents/d_out: [n]. */
int vs_cfg_ddim_step(void* stream, const void* d_eps2, const void* d_latents, int io_f32, size_t n, int cfg,
                     float guidance, float alpha_t, float alpha_prev, void* d_out);

/* Same update with the two coefficients in DEVICE memory: d_coef[0] = sqrt(a_p)/sqrt(a_t),
 * d_coef[1] = sqrt(1-a_p) - sqrt(a_p) sqrt(1-a_t)/sqrt(a_t).  Together with the device-side timestep of vs_unet_forward
 * this makes one whole denoising step capturable in a CUDA graph that is replayed for every timestep. */
int vs_cfg_ddim_step_dev(void* stream, const void* d_eps2, const void* d_latents, int io_f32, size_t n, int cfg,
                         float guidance, const float* d_coef, void* d_out);

/* The loop body's update for S videos of n_s = C F h w elements each, with diffusers 0.19.3's stochastic DDIM (eta) and
 * the CFG rescale (pipeline_videoswap.py:578-587, rescale_noise_cfg):
 *   eps = eps_u + g (eps_c - eps_u);  with cfg and guidance_rescale r > 0: eps *= r std(eps_c) / std(eps) + (1 - r), the
 *   unbiased standard deviations taken per video;  x' = c_x x + c_e eps + c_n z,  c_n = eta sqrt(variance(t, t_prev)),
 *   c_e = sqrt(1 - a_p - c_n^2) - sqrt(a_p) sqrt(1 - a_t) / sqrt(a_t),  c_x = sqrt(a_p) / sqrt(a_t).
 * d_eps2: [2 S, n_s] (the S uncond predictions first) when cfg != 0, else [S, n_s]; d_latents, d_noise (z), d_out:
 * [S, n_s].  d_noise may be NULL only when eta == 0.  One launch, one thread-block cluster per video; deterministic. */
int vs_cfg_ddim_rescale_step(void* stream, const void* d_eps2, const void* d_latents, const void* d_noise, int io_f32, int S,
                             size_t n_s, int cfg, float guidance, float alpha_t, float alpha_prev, float eta,
                             float guidance_rescale, void* d_out);

/* Same update with d_coef[0..3] = (c_x, c_e, c_n, r) in DEVICE memory (CUDA-graph replayable); d_noise NULL: no noise
 * term. */
int vs_cfg_ddim_rescale_step_dev(void* stream, const void* d_eps2, const void* d_latents, const void* d_noise, int io_f32,
                                 int S, size_t n_s, int cfg, float guidance, const float* d_coef, void* d_out);

/* Replaces  SparsePointAdapter.forward  (models/adapter_model.py:97-136): MLP_l(point_embedding) then bilinear splat.
 *   d_w0 [mid, E], d_b0 [mid], d_w1 [C, mid], d_b1 [C] fp16; d_point_embedding [P, E] fp32; d_tracks [F, P, 2] fp32
 *   (x, y; negative = invisible); d_point_mask [P] int32 or NULL (index_list); d_ws: >= P*(mid + C) floats scratch.
 *   d_map: NHWC fp16 [F, h, w, C] with h = img_h / rate, w = img_w / rate; values multiplied by `scale`. */
int vs_adapter_level(void* stream, const void* d_w0, const void* d_b0, const void* d_w1, const void* d_b1, int E, int mid,
                     int C, const float* d_point_embedding, const float* d_tracks, const int* d_point_mask, int F, int P,
                     int h, int w, float rate, int coord_fp16, float scale, float* d_ws, void* d_map);

/* ---- per-kernel entry points (used by the parity tests; same kernels the forward uses) -------------------------- */
/* One launch of the tensor-core GEMM / implicit-GEMM convolution with every argument the UNet forward can pass (field for
 * field the library's internal GEMM arguments; zero-initialise and set what is used).
 *   out[pix, n] = epilogue( sum_k [A | A2][pix (+ tap shift), k] * Bw[n, k] )
 *   taps 1: A [M, K1] (row stride lda1) (+ A2 [M, K2], lda2, channel concat along K); taps 9: NHWC [nimg, H, W, K1] 3x3
 *   convolution, pad 1 (M = nimg H W); taps 4: one output parity (sub_py, sub_px) of nearest-2x + 3x3 into an OH x OW output
 *   (OH = 2H or 2H - 1, OW = 2W or 2W - 1; 0 = 2H / 2W).  Bw [N, taps (K1 + K2)], where taps = 4 except for parity 0 along
 *   an odd output axis, which has 3 taps along it (6 or 9 in all; see vs_upsample_conv3x3_sized for the panels).
 *   Epilogue: + bias[n] + rowvec[((pix / pix_per_batch) % rv_mod if rv_mod > 0), n] (row stride ldrv, 0 = N) + residual[pix, n]
 *   (row stride ldr; may alias `out`); mode 1 = GEGLU on packed weights (N / 2 output columns); mode 2 = quick-GELU,
 *   fp16(v sigmoid(1.702 v)) with v = acc + bias in fp32 (CLIP's MLP fc1: taps 1, bias only, N % 32 == 0, BLOCK_N 128 / 256);
 *   mode 3 = ReLU, fp16(max(acc + bias, 0)) (the T2I-Adapter's block1: taps 9, one source, bias only, N % 32 == 0).  Folded LayerNorm of A:
 *   ln_u [N] with ln_stats [M, 2] (rstd, -mean rstd) or ln_parts [ln_nparts][M][2] (sum, sum of squares).
 *   ln_sums_out [n_tiles][M][2]: (sum, sum of squares) of the stored fp16 outputs per row and column tile of width BN.
 *   force_bn 0 = automatic column-tile width, else 64 / 128 / 160 / 256.
 *   stride2 (with taps 9): 3x3 conv with stride 2 of the input zero-padded by one column on the right and one row at the
 *   bottom only (diffusers Downsample2D(padding=0)); H, W = the input size (both even), M = nimg (H / 2) (W / 2), output
 *   NHWC [nimg, H / 2, W / 2, N]; A dense (lda1 = K1, K1 % 64 == 0), no A2, bias only, N % 32 == 0. */
typedef struct vs_gemm_desc {
  const void* A; int K1; int lda1;
  const void* A2; int K2; int lda2;
  const void* Bw;
  int M, N;
  int taps;
  int sub_py, sub_px;
  int nimg, H, W;
  const float* bias;
  const float* rowvec; int ldrv; int pix_per_batch; int rv_mod;
  const float* ln_stats; const float* ln_u;
  const float* ln_parts; int ln_nparts;
  float* ln_sums_out;
  const void* residual; int ldr;
  void* out; int ldc;
  int mode;
  int force_bn;
  int OH, OW;
  int stride2;
} vs_gemm_desc;
int vs_gemm_ex(void* stream, const vs_gemm_desc* desc);
int vs_pack_conv3x3(void* stream, const void* d_w, int cout, int cin, void* d_out);
int vs_pack_geglu(void* stream, const void* d_w, const void* d_b, int hidden, int K, void* d_wout, float* d_bout);
int vs_groupnorm(void* stream, const void* d_x1, int c1, const void* d_x2, int c2, int nimg, int hw, int imgs_per_set,
                 int groups, float eps, const float* d_gamma, const float* d_beta, int silu, float* d_sums, void* d_out);
/* The two halves of the statistics + apply GroupNorm as the frame-sharded forward runs them: vs_groupnorm_stats ADDS the
 * (sum, sum of squares) of each set of imgs_per_set images to d_sums [nimg / imgs_per_set, groups, 2] (zeroed first only
 * when zero_first != 0); vs_groupnorm_apply normalises with sums that cover count_scale times the local elements (the
 * all-reduced sums of count_scale frame shards). */
int vs_groupnorm_stats(void* stream, const void* d_x1, int c1, const void* d_x2, int c2, int nimg, int hw, int imgs_per_set,
                       int groups, float* d_sums, int zero_first);
int vs_groupnorm_apply(void* stream, const void* d_x1, int c1, const void* d_x2, int c2, int nimg, int hw, int imgs_per_set,
                       int groups, const float* d_sums, float eps, const float* d_gamma, const float* d_beta, int silu,
                       int count_scale, void* d_out);
int vs_layernorm(void* stream, const void* d_x, int rows, int C, const float* d_gamma, const float* d_beta,
                 const float* d_pe, int hw, int F, void* d_out);
/* LayerNorm(x) (+ pe[(row / hw) % frames]) followed by a linear layer (mode 0) or GEGLU projection (mode 1, packed
 * weights), with the norm folded into ONE GEMM on the raw input (motion_module.py:224-228,294 + the q/k/v projection;
 * attention.py:229-256).  C in {320, 640, 1280}.  Scratch: d_wf [N, C] fp16, d_u / d_c [N] fp32, d_cpe [pe_len, N] fp32
 * (only with d_pe), d_stats [M, 2] fp32.  The UNet forward uses the same kernels with the folding done at load time. */
int vs_ln_linear(void* stream, const void* d_x, int M, int C, const void* d_w, const float* d_bias, int N,
                 const float* d_gamma, const float* d_beta, const float* d_pe, int pe_len, int hw, int frames, int mode,
                 void* d_wf, float* d_u, float* d_c, float* d_cpe, float* d_stats, void* d_out);
/* The form the UNet forward uses: the linear layer that PRODUCES the LayerNorm's input (x = x0 W0^T + b0 (+ residual),
 * fp16, written to d_x) also emits the per-row (sum, sum of squares) of what it stores, one slice per column tile of its
 * epilogue (d_parts: [parts_capacity][M][2] fp32), and the consuming GEMM derives mean / rstd from those slices -- no
 * statistics pass over x (attention.py:229-256 / motion_module.py:224-234: proj_in -> norm1 -> to_q/k/v, ...).
 * d_pe / pe_len / hw / frames / d_cpe as in vs_ln_linear: the motion module's temporal positional encoding. */
int vs_linear_ln_linear(void* stream, const void* d_x0, int M, int K0, const void* d_w0, const float* d_b0,
                        const void* d_residual, int C, void* d_x, const void* d_w, const float* d_bias, int N,
                        const float* d_gamma, const float* d_beta, const float* d_pe, int pe_len, int hw, int frames,
                        int mode, void* d_wf, float* d_u, float* d_c, float* d_cpe, float* d_parts, int parts_capacity,
                        void* d_out);
int vs_attention(void* stream, const void* d_q, int ldq, const void* d_k, int ldk, const void* d_v, int ldv, void* d_o,
                 int ldo, int batch, int nq, int nk, int heads, int d, long long q_bstride, long long kv_bstride,
                 long long o_bstride, int kv_div);
int vs_temporal_attention(void* stream, const void* d_qkv, void* d_o, int B, int F, int HW, int C, int heads);
/* conv_in (3x3, pad 1, tiny cin).  With d_scratch (>= (nimg H W + cout) * 64 halves) and cin == 4: patch rows + the
 * tensor-core GEMM with K = 64, as the UNet forward runs it; d_scratch NULL (or cin != 4): a direct CUDA-core kernel. */
int vs_conv_in(void* stream, const void* d_x, int nimg, int H, int W, int cin, const void* d_w, const float* d_bias,
               int cout, void* d_scratch, void* d_out);
int vs_upsample2x(void* stream, const void* d_x, int nimg, int H, int W, int C, void* d_out);
/* Upsample3D (resnet.py:21-69): nearest 2x then conv3x3, computed as four 2x2 sub-pixel convolutions on the low-resolution
 * input (weights pre-summed per output parity; 2.25x fewer FLOPs, no materialised up-sampled tensor).  d_w: [Cout, C, 3, 3]
 * fp16 as in the state_dict; d_wsub: scratch for the 4 panels, 16 * Cout * C halves; d_out: NHWC [nimg, 2H, 2W, Cout]. */
int vs_upsample_conv3x3(void* stream, const void* d_x, int nimg, int H, int W, int C, const void* d_w, int Cout,
                        const float* d_bias, void* d_wsub, void* d_out);
/* The same to an explicit output size, as the UNet's up path runs it (the reference's forward_upsample_size path,
 * unet.py:356-364,454-457): nearest up-sampling of [nimg, H, W, C] to OH x OW (OH = 2H or 2H - 1, OW = 2W or 2W - 1,
 * torch's nearest: source row y / 2) then conv3x3.  Along an odd axis the last up-sampled row/column is padding, so
 * parity 0 keeps its three weight taps apart.  d_wpanels: scratch for the packed panels, 49 * Cout * C halves (the 3x3
 * panel, then the 40 taps of the sub-pixel panels); d_out: NHWC [nimg, OH, OW, Cout]. */
int vs_upsample_conv3x3_sized(void* stream, const void* d_x, int nimg, int H, int W, int C, const void* d_w, int Cout,
                              const float* d_bias, int OH, int OW, void* d_wpanels, void* d_out);
/* Nearest up-sampling of NHWC [nimg, H, W, C] to [nimg, OH, OW, C] (OH in {2H - 1, 2H}, OW in {2W - 1, 2W}). */
int vs_upsample_nearest(void* stream, const void* d_x, int nimg, int H, int W, int C, int OH, int OW, void* d_out);
int vs_conv3x3_s2(void* stream, const void* d_x, int nimg, int H, int W, int C, const void* d_w_packed, int Cout,
                  const float* d_bias, void* d_scratch, void* d_out);

/* ---- VAE decoder (diffusers 0.19.3 AutoencoderKL.decode + VaeImageProcessor.postprocess; the reference's loop ends with
 * them, pipeline_videoswap.py:603-610).  The decoder is a sequence of the GEMM / conv / GroupNorm entry points above and
 * these five. */
/* The four sub-pixel panels of vs_upsample_conv3x3 (d_out: 16 * cout * cin halves), packed once so that the four parity
 * launches (vs_gemm_ex, taps 4, Bw = panel py * 2 + px) can run without re-packing. */
int vs_pack_conv_subpixel(void* stream, const void* d_w, int cout, int cin, void* d_out);
/* Single-head attention with d = 512 (the VAE mid block) as S = Q K^T -> P -> O = P V through vs_gemm_ex:
 * vs_softmax_rows: d_s [rows, ld] fp16 in place, p = softmax(s * scale) over the first n columns with fp32 math; columns
 * n .. ld - 1 are set to 0 and never read (ld % 8 == 0).
 * vs_transpose_pad: d_dst [cols, rows_pad] = d_src [rows, cols]^T (fp16), columns rows .. rows_pad - 1 zero: V^T as the
 * K-major B operand of O = P V with K = rows_pad. */
int vs_softmax_rows(void* stream, void* d_s, int rows, int n, int ld, float scale);
int vs_transpose_pad(void* stream, const void* d_src, int rows, int cols, int rows_pad, void* d_dst);
/* Decoder entry: post_quant_conv(z / divisor) of NCHW latents d_z [nimg, 4, h, w] (fp16, or fp32 with z_is_f32) in fp32,
 * to NHWC fp16 d_out [nimg, h, w, 4].  d_wb: fp32 weight [4][4] then bias [4]. */
int vs_vae_latent_in(void* stream, const void* d_z, int z_is_f32, int nimg, int h, int w, float divisor, const float* d_wb,
                     void* d_out);
/* Decoder exit: channels 0..2 of NHWC fp16 d_x [nimg, H, W, channels] (channels % 8 == 0), y = clamp(x / 2 + 0.5, 0, 1):
 * format 0 the sample x itself, fp16 NCHW [nimg, 3, H, W]; 1 ("pt") y fp32 NCHW; 2 ("np") y fp32 NHWC [nimg, H, W, 3];
 * 3 ("pil") uint8 NHWC round-half-even(y * 255). */
int vs_image_postprocess(void* stream, const void* d_x, int nimg, int H, int W, int channels, int format, void* d_out);

/* ---- VAE encoder (diffusers 0.19.3 AutoencoderKL.encode + DiagonalGaussianDistribution; the reference's
 * prepare_image_latents, pipeline_videoswap.py:204-233).  The encoder is a sequence of the GEMM / conv / conv_in /
 * GroupNorm / attention entry points above and these four. */
/* Downsample2D(padding=0): 3x3 conv with stride 2 of NHWC d_x [nimg, H, W, C] zero-padded by one column on the right and
 * one row at the bottom (H, W even, C % 64 == 0), as an implicit GEMM on the tensor cores (no im2col): vs_gemm_ex with
 * taps 9 and stride2 = 1.  d_w_packed: vs_pack_conv3x3 panel [Cout, 9 C]; d_out NHWC [nimg, H / 2, W / 2, Cout]. */
int vs_downsample_conv3x3(void* stream, const void* d_x, int nimg, int H, int W, int C, const void* d_w_packed, int Cout,
                          const float* d_bias, void* d_out);
/* Encoder entry: NHWC fp16 d_out [nimg, H, W, 4] with channel 3 zero (the input of vs_conv_in with cin = 4).  src_format
 * 0: uint8 NHWC frames [nimg, H, W, 3], normalised as VaeImageProcessor.preprocess + the fp16 cast compute it,
 * fl16(fl32(2 fl32(u / 255) - 1)); 1 / 2: fp16 / fp32 NCHW [nimg, 3, H, W] already in [-1, 1], rounded to fp16. */
int vs_vae_image_in(void* stream, const void* d_x, int src_format, int nimg, int H, int W, void* d_out);
/* Encoder exit: quant_conv (1x1, 8 -> 8) in fp32 of conv_out's NHWC fp16 d_x [nimg, h, w, 8] -> the moments
 * (DiagonalGaussianDistribution.parameters: mean in channels 0..3, logvar in 4..7) fp16 NCHW d_out [nimg, 8, h, w].
 * d_wb: fp32 weight [8][8] then bias [8]. */
int vs_vae_moments(void* stream, const void* d_x, int nimg, int h, int w, const float* d_wb, void* d_out);
/* The posterior: scale (mean + exp(0.5 clamp(logvar, -30, 20)) noise) in fp32 from the moments d_params [nimg, 8, h, w]
 * and fp16 d_noise [nimg, 4, h, w]; d_noise NULL gives scale mean (the mode).  d_out fp16 [nimg, 4, h, w] (layout 0) or
 * [1, 4, nimg, h, w] (layout 1: the frames of one video, as the inversion loop takes them). */
int vs_vae_posterior(void* stream, const void* d_params, const void* d_noise, int nimg, int h, int w, float scale, int layout,
                     void* d_out);

/* ---- T2I-Adapter (diffusers 0.19.3 T2IAdapter with adapter_type "full_adapter": the reference's image-condition branch,
 * pipeline_videoswap.py:538-546).  The adapter is a sequence of vs_gemm_ex (conv_in and block1 as taps 9, block1 with
 * mode 3; in_conv and block2 as taps 1, block2 with the residual) and these three. */
/* Entry: uint8 frames d_x [nimg, H, W, channels] (channels 1 = "L" or 3 = "RGB", H and W multiples of 8, 8-byte aligned) ->
 * the PixelUnshuffle(8) of fp16(fp32(u) / 255) as NHWC fp16 d_out [nimg, H / 8, W / 8, 64 channels], channel
 * c 64 + 8 i + j of output pixel (y, x) = input pixel (8 y + i, 8 x + j), channel c (torch's PixelUnshuffle order). */
int vs_t2i_image_in(void* stream, const void* d_x, int nimg, int H, int W, int channels, void* d_out);
/* AvgPool2d(2, stride 2) of NHWC fp16 d_x [nimg, H, W, C] (H, W even, C % 8 == 0) -> d_out [nimg, H / 2, W / 2, C]:
 * the four values summed in fp32, times 0.25, rounded once. */
int vs_avgpool2x2(void* stream, const void* d_x, int nimg, int H, int W, int C, void* d_out);
/* d_out[i] = fp16(fp32(d_x[i]) * scale) for n fp16 values (n % 8 == 0, 16-byte aligned; d_out may be d_x): the
 * t2i_guidance_scale multiply of the adapter's fp16 features, rounded as torch rounds `v * scale`. */
int vs_scale_f16(void* stream, const void* d_x, size_t n, float scale, void* d_out);

/* ---- CLIP text encoder (transformers CLIPTextModel, SD-1.5's text_encoder; the reference's prompt encoding,
 * pipeline_videoswap.py:273-423 and utils/edlora_util.py:116-196).  The encoder is a sequence of vs_layernorm, vs_gemm_ex
 * (fused QKV with bias; out_proj / fc2 with bias and the in-place residual; fc1 with mode 2) and these two. */
/* CLIPTextEmbeddings: d_out fp16 [n L, C] = fp16(fp32(d_tok[ids[s, t]]) + fp32(d_pos[t])), one rounding as torch's fp16 add.
 * d_ids_i32 int32 [n, L] on the device, every id in [0, vocab) (the caller checks; an id outside writes NaN); d_tok fp16
 * [vocab, C], d_pos fp16 [>= L, C]; C % 8 == 0, all three 16-byte aligned. */
int vs_clip_embed(void* stream, const int* d_ids_i32, int n, int L, const void* d_tok, int vocab, const void* d_pos, int C,
                  void* d_out);
/* Causal self-attention (CLIPAttention with the causal mask, no padding mask) of nseq sequences of 1 <= L <= 77 tokens,
 * every head of d = 64 in one launch: q / k / v of head h at columns h d, C + h d and 2 C + h d (C = heads d) of the fused
 * QKV GEMM output d_qkv [nseq L, ldqkv] (ldqkv >= 3 C); softmax(q k^T / sqrt(d)) v of head h goes to columns h d .. h d + d - 1
 * of d_o [nseq L, ldo].  The 1 / sqrt(d) scale is applied in fp32 inside the kernel. */
int vs_causal_attention(void* stream, const void* d_qkv, int ldqkv, void* d_o, int ldo, int nseq, int L, int heads, int d);

/* ---- DIFT semantic points (the reference's dift_util.py / extract_semantic_point.py:125-204) ----------------------------
 * d_out fp32 [n E, 4, h, w] = sqrt_a sf (mu + exp(0.5 clamp(logvar, -30, 20)) eps1) + sqrt_1ma eps2: the posterior draw of
 * frame r / E (moments fp16 [n, 8, h, w] of vs_vae_moments) then DDPM add_noise; d_eps1, d_eps2 fp32 [n E, 4, h, w]. */
int vs_dift_noise(void* stream, const void* d_moments, const float* d_eps1, const float* d_eps2, int n, int E, int h, int w,
                  float sf, float sqrt_a, float sqrt_1ma, float* d_out);
/* d_out fp32 [n, P, C]: the ensemble mean of d_feat (NHWC fp16 [n, E, h, w, C], C % 8 == 0) up-sampled as
 * nn.Upsample(size=(H, W), mode="bilinear") and read at the pixels d_xy int32 [n, P, 2] = (x, y), 0 <= x < W, 0 <= y < H.
 * Source indices and interpolation order are those of torch's CPU upsample_bilinear2d in fp32; no map is materialised. */
int vs_dift_point_sample(void* stream, const void* d_feat, int n, int E, int h, int w, int C, int H, int W, const int* d_xy,
                         int P, float* d_out);
/* d_out fp32 NCHW [n, C, h, w] = the mean over E of d_feat NHWC fp16 [n, E, h, w, C] (SDFeaturizer.forward's map). */
int vs_dift_ensemble_mean(void* stream, const void* d_feat, int n, int E, int h, int w, int C, float* d_out);
/* d_vecs fp32 [n, P, C].  With d_src (fp32 rows [*, C]), d_src_row int32 [n, P] and d_conf fp32 [n, P]: the cosine
 * similarity (CosineSimilarity(dim=1, eps=1e-8)) of each vector against its source row.  With d_accept uint8 [n, P]: the
 * per-point sums / means fp32 [P, C] and counts fp32 [P] over the accepted frames, accumulated in frame order (each of the
 * three may be NULL; a point never accepted has mean 0). */
int vs_dift_point_reduce(void* stream, const float* d_vecs, int n, int P, int C, const float* d_src, const int* d_src_row,
                         float* d_conf, const void* d_accept, float* d_sums, float* d_counts, float* d_means);

/* ---- layered-atlas point propagation (the reference's propagate_point_displacement.py) ---------------------------------
 * One IMLP_Hash network with mlp_type 'origin' (videoswap/atlas/implicit_neural_networks.py): the positional encoding
 * (pe_dim 0 = pe_type 'none'; pe_dim > 0 = 'encoding', feature j (2 input_dim) + c = sin(x_c b_j) for c < input_dim and
 * cos(x_(c - input_dim) b_j) after, b_j = fp32(2^j pi)), then mlp_layers linears with a ReLU before every one but the first;
 * layer i with bit i of skip_mask set takes torch.cat((x, encoded input), 1); tanh on the output when use_tanh.
 * d_params: fp32, 16-byte aligned, for each layer i in order W_i^T [K_i, N_i] (the transposed nn.Linear weight) then the
 * bias [N_i]; K_0 = E (the encoded width: input_dim, or 2 input_dim pe_dim), K_i = hidden_dim (+ E with the skip bit),
 * N_i = hidden_dim except N_(mlp_layers - 1) = output_dim.  fp32 FMA on the CUDA cores. */
typedef struct vs_imlp_desc {
  const float* d_params;
  int input_dim;      /* 1 .. 8 */
  int output_dim;     /* 1 .. hidden_dim */
  int hidden_dim;     /* 32 .. 256, a multiple of 32 */
  int mlp_layers;     /* 1 .. 32 */
  int pe_dim;         /* 0 .. 16 */
  uint32_t skip_mask; /* bits 1 .. mlp_layers - 1 only */
  int use_tanh;
} vs_imlp_desc;
/* d_out fp32 [rows, output_dim] = the network on d_x fp32 [rows, input_dim], rows >= 1, in one launch.  A descriptor
 * outside the ranges above (or one whose encoded width does not fit the row tile's shared memory) fails before any launch. */
int vs_imlp_forward(void* stream, const vs_imlp_desc* net, const float* d_x, int rows, float* d_out);
/* propagate_point_sequence for P edited points over F frames in six launches, whatever P and F, with no host sync.
 * fg (3 -> 2), fg_inverse (3 -> 3), alpha (3 -> 1): FG_UV_Mapping, FG_UV_Mapping_Inverse and F_Alpha.
 * d_points fp32 [P, 4] = (x, y, dx, dy): the keyframe point and the drag, normalised as x / (larger_dim / 2) - 1 (the drag as
 * the difference of two normalised coordinates); t_key the normalised keyframe time.  The frame axis is
 * fp32(f) / fp32(F / 2) - 1 in fp32.  d_tracks fp32 [F, P, 2] = (x, y) pixels, rint((w + 1) / 2 larger_dim) of the warp w
 * where 0.5 (alpha + 1) > 0.5 (alpha evaluated at the inverse network's predicted (x, y, t)), else -1.
 * d_ws fp32, 21 P + 25 P F floats, left holding the stages (row q = p F + f; rows of fg_in / fg_out are base, x + 0.1,
 * y + 0.05 for every point, those of inv_in / inv_out base, u + 0.1, v + 0.05 for every q):
 *   fg_in [3P, 3] | fg_out [3P, 2] | J_fg [P, 2, 2] | delta_uv [P, 2] | inv_in [3PF, 3] | inv_out [3PF, 3] | alpha [PF] |
 *   J_inv [PF, 2, 2] (x, y columns) | warp [PF, 2]
 * Fails before any launch on a bad descriptor, a network of the wrong shape, P < 1, F < 1 or larger_dim < 1. */
int vs_atlas_propagate(void* stream, const vs_imlp_desc* fg, const vs_imlp_desc* fg_inverse, const vs_imlp_desc* alpha,
                       const float* d_points, float t_key, int P, int F, int larger_dim, float* d_ws, float* d_tracks);

/* ---- measurement hooks (bench.py): per-launch CUDA-event timing on the launching stream, by kernel category
 * 0 gemm, 1 conv3x3, 2 spatial/cross attention (and the VAE's row softmax, the CLIP causal attention), 3 temporal attention, 4 groupnorm, 5 layernorm,
 * 6 other.
 * `work` = algorithmic FLOPs (categories 0-2) or algorithmic bytes (3-5) summed over the recorded launches. */
int vs_profile_enable(int on);
int vs_profile_reset(void);
int vs_profile_collect(int category, double* ms, double* work, long long* count);
long long vs_launch_count(void);   /* kernels launched by this library since load */
int vs_profile_dump(const char* path);   /* CSV: category, shape (m,n,k), work per launch, launches, total ms */
/* Runtime A/B switches (defaults = the shipped configuration; unknown names are an error):
 *   "attn_tc"      1  wgmma/TMA attention kernel for head dims 40/80; 0 forces the mma.sync kernel
 *   "gemm_stages"  0  limit of the shared-memory ring depth of the GEMM (0 = as many as fit)
 *   "gemm_ctas"    0  cap on the persistent grid of the GEMM (0 = one CTA per SM); a smaller grid gives every CTA more
 *                     tiles, so the same problem runs another tile schedule (schedule-invariance tests)
 *   "gemm_epi_slot" 1 the short-K linears and GEGLUs (K <= 640) fetch their epilogue operands into shared-memory slots
 *                     during the main loop; 0 = the epilogue reads them from global memory (bit-identical; tests)
 *   "ln_fold"      1  LayerNorms folded into the consuming GEMM; 0 = stand-alone LayerNorm kernel
 *   "ln_fuse"      1  row statistics of folded LayerNorms written by the producing GEMM's epilogue; 0 = ln_stats pass
 *   "tattn_vst"    1  temporal attention writes its outputs with 16-byte stores from a shared-memory stage; 0 = 4-byte stores
 *   "gn_fused"     1  per-frame GroupNorms (Transformer3DModel.norm, motion-module norm) as ONE pass with the image resident
 *                     in the shared memory of a thread-block cluster (up to 16 CTAs x 160 KB); 0 = statistics + apply kernels
 *   "subpixel"     1  nearest-2x + conv3x3 as four sub-pixel convs; 0 = materialise the up-sampled tensor, then conv3x3
 *   "gn_stats_v2"  0  1 = GroupNorm statistics kernel with per-position accumulators instead of a per-element group select (no gain)
 *   "pdl"          1  programmatic dependent launch between the hot kernels; 0 = plain stream order */
int vs_set_option(const char* name, int value);

#ifdef __cplusplus
}
#endif
#endif
