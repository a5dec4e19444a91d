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
 *   d_out      [B, C_out, F, H, W] same dtype as d_sample */
int vs_unet_forward(vs_unet* h, void* stream, const void* d_sample, int io_f32, int B, int F, int H, int W,
                    const float* d_timesteps, const void* d_ehs, int ehs_tokens, int ehs_layers,
                    const void* const* d_residuals, int residuals_nhwc, float residual_scale, void* d_out);
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

/* Replaces  SparsePointAdapter.forward  (models/adapter_model.py:97-136): MLP_l(point_embedding) then bilinear splat.
 *   d_w0 [mid, E], d_b0 [mid], d_w1 [C, mid], d_b1 [C] fp16; d_point_embedding [P, E] fp32; d_tracks [F, P, 2] fp32
 *   (x, y; negative = invisible); d_point_mask [P] int32 or NULL (index_list); d_ws: >= P*(mid + C) floats scratch.
 *   d_map: NHWC fp16 [F, h, w, C] with h = img_h / rate, w = img_w / rate; values multiplied by `scale`. */
int vs_adapter_level(void* stream, const void* d_w0, const void* d_b0, const void* d_w1, const void* d_b1, int E, int mid,
                     int C, const float* d_point_embedding, const float* d_tracks, const int* d_point_mask, int F, int P,
                     int h, int w, float rate, int coord_fp16, float scale, float* d_ws, void* d_map);

/* ---- per-kernel entry points (used by the parity tests; same kernels the forward uses) -------------------------- */
int vs_gemm(void* stream, const void* d_A, int K1, const void* d_A2, int K2, const void* d_W, int M, int N,
            const float* d_bias, const float* d_rowvec, int pix_per_batch, const void* d_residual, void* d_out, int mode,
            int force_bn);
int vs_conv3x3(void* stream, const void* d_x, int C1, const void* d_x2, int C2, const void* d_w_packed, int nimg, int H,
               int W, int Cout, const float* d_bias, const float* d_rowvec, int imgs_per_batch, const void* d_residual,
               void* d_out);
int vs_pack_conv3x3(void* stream, const void* d_w, int cout, int cin, void* d_out);
int vs_pack_geglu(void* stream, const void* d_w, const void* d_b, int hidden, int K, void* d_wout, float* d_bout);
int vs_groupnorm(void* stream, const void* d_x1, int c1, const void* d_x2, int c2, int nimg, int hw, int imgs_per_set,
                 int groups, float eps, const float* d_gamma, const float* d_beta, int silu, float* d_sums, void* d_out);
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
 * statistics pass over x (attention.py:229-256 / motion_module.py:224-234: proj_in -> norm1 -> to_q/k/v, ...). */
int vs_linear_ln_linear(void* stream, const void* d_x0, int M, int K0, const void* d_w0, const float* d_b0,
                        const void* d_residual, int C, void* d_x, const void* d_w, const float* d_bias, int N,
                        const float* d_gamma, const float* d_beta, int mode, void* d_wf, float* d_u, float* d_c,
                        float* d_parts, int parts_capacity, void* d_out);
int vs_attention(void* stream, const void* d_q, int ldq, const void* d_k, int ldk, const void* d_v, int ldv, void* d_o,
                 int ldo, int batch, int nq, int nk, int heads, int d, long long q_bstride, long long kv_bstride,
                 long long o_bstride, int kv_div);
int vs_temporal_attention(void* stream, const void* d_qkv, void* d_o, int B, int F, int HW, int C, int heads);
int vs_conv_in(void* stream, const void* d_x, int nimg, int H, int W, int cin, const void* d_w, const float* d_bias,
               int cout, void* d_out);
int vs_upsample2x(void* stream, const void* d_x, int nimg, int H, int W, int C, void* d_out);
/* Upsample3D (resnet.py:21-69): nearest 2x then conv3x3, computed as four 2x2 sub-pixel convolutions on the low-resolution
 * input (weights pre-summed per output parity; 2.25x fewer FLOPs, no materialised up-sampled tensor).  d_w: [Cout, C, 3, 3]
 * fp16 as in the state_dict; d_wsub: scratch for the 4 panels, 16 * Cout * C halves; d_out: NHWC [nimg, 2H, 2W, Cout]. */
int vs_upsample_conv3x3(void* stream, const void* d_x, int nimg, int H, int W, int C, const void* d_w, int Cout,
                        const float* d_bias, void* d_wsub, void* d_out);
int vs_conv3x3_s2(void* stream, const void* d_x, int nimg, int H, int W, int C, const void* d_w_packed, int Cout,
                  const float* d_bias, void* d_scratch, void* d_out);

/* ---- measurement hooks (bench.py): per-launch CUDA-event timing on the launching stream, by kernel category
 * 0 gemm, 1 conv3x3, 2 spatial/cross attention, 3 temporal attention, 4 groupnorm, 5 layernorm, 6 other.
 * `work` = algorithmic FLOPs (categories 0-2) or algorithmic bytes (3-5) summed over the recorded launches. */
int vs_profile_enable(int on);
int vs_profile_reset(void);
int vs_profile_collect(int category, double* ms, double* work, long long* count);
long long vs_launch_count(void);   /* kernels launched by this library since load */
int vs_profile_dump(const char* path);   /* CSV: category, shape (m,n,k), work per launch, launches, total ms */
/* Runtime A/B switches (defaults = the shipped configuration; unknown names are an error):
 *   "attn_tc"      1  wgmma/TMA attention kernel for head dims 40/80; 0 forces the mma.sync kernel
 *   "gemm_stages"  0  limit of the shared-memory ring depth of the GEMM (0 = as many as fit)
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
