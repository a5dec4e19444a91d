// Host-side launchers of the sm_90a kernels (all asynchronous on `st`, no hidden allocation, return 0 on success).
// Activation layout everywhere: NHWC fp16, i.e. tokens [(b f), h*w, C] with C innermost.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vs {

enum EpiMode { EPI_LINEAR = 0, EPI_GEGLU = 1 };

// out[pix, n] = epilogue( sum_k A[pix(+tap shift), k] * Bw[n, k] )
//   * plain GEMM (taps == 1): A is [M, K1] (lda1) optionally followed along K by A2 [M, K2] (channel concat).
//   * 3x3 conv (taps == 9): A is NHWC [nimg, H, W, C1] (+ A2 [.., C2]); Bw is [N, 9*(C1+C2)], tap-major;
//     zero padding comes from TMA out-of-bounds fill.
//   epilogue: + bias[n] + rowvec[pix / pix_per_batch, n] + residual[pix, n]; EPI_GEGLU: value*gelu(gate) on
//   column-interleaved weights (see pack_geglu) -> N/2 output columns.
struct GemmArgs {
  const __half* A = nullptr;  int K1 = 0;  int lda1 = 0;
  const __half* A2 = nullptr; int K2 = 0;  int lda2 = 0;
  const __half* Bw = nullptr;                 // [N, taps*(K1+K2)] fp16, K contiguous
  int M = 0, N = 0;
  int taps = 1;                               // 1, 9 (3x3, pad 1) or 4 (2x2 sub-pixel phase of nearest-2x + 3x3)
  int sub_py = 0, sub_px = 0;                 // taps == 4: output parity; writes pixel (2y+py, 2x+px) of the 2H x 2W output
  int nimg = 0, H = 0, W = 0;                 // conv geometry (taps == 9)
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

// ---- pointwise / small -----------------------------------------------------------------------------------------
int small_linear(cudaStream_t st, const float* x, int rows, int K, const __half* W, const float* bias, int N,
                 bool silu_in, bool silu_out, float* out);     // out[r,n] = act(sum_k f(x[r,k]) W[n,k] + b[n]), fp32
int timestep_embedding(cudaStream_t st, const float* t, int B, int dim, float* out);   // cat(cos, sin)
int conv_in_3x3(cudaStream_t st, const __half* x, int nimg, int H, int W, int cin, const __half* w, const float* bias,
                int cout, __half* out, __half* scratch = nullptr);   // conv_in (tiny Cin): with `scratch` (>= (nimg*H*W +
                // cout) * 64 halves, cin == 4) patch rows + tensor-core GEMM, else a direct CUDA-core kernel
int upsample_nearest2x(cudaStream_t st, const __half* x, int nimg, int H, int W, int C, __half* out);
int im2col_s2(cudaStream_t st, const __half* x, int nimg, int H, int W, int C, __half* out);  // [nimg*Ho*Wo, 9*C]
int add_inplace(cudaStream_t st, __half* x, const __half* r, size_t n, float scale);   // x += scale * r
int ncfhw_to_nhwc(cudaStream_t st, const void* src, int src_is_f32, int B, int C, int F, int H, int W, __half* dst);
int nhwc_to_ncfhw(cudaStream_t st, const __half* src, int B, int C, int F, int H, int W, void* dst, int dst_is_f32);
int nchw_to_nhwc(cudaStream_t st, const __half* src, int n, int C, int H, int W, float scale, __half* dst);
// eps = u + s (c - u); x_prev = sqrt(a_p) (x - sqrt(1-a_t) eps)/sqrt(a_t) + sqrt(1-a_p) eps.  eps2: [2, n] (uncond
// first) or [1, n] when guidance is disabled (cfg == 0).
int cfg_ddim_step(cudaStream_t st, const void* eps2, const void* latents, int is_f32, size_t n, int cfg,
                  float guidance, float a_t, float a_prev, void* out);
// Same, with the two DDIM coefficients (c_x, c_e) read from device memory (CUDA-graph replayable across timesteps).
int cfg_ddim_step_dev(cudaStream_t st, const void* eps2, const void* latents, int is_f32, size_t n, int cfg,
                      float guidance, const float* d_coef, void* out);
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
int pack_conv_subpixel(cudaStream_t st, const __half* w, int cout, int cin, __half* out);
int pack_geglu(cudaStream_t st, const __half* w, const __half* b, int hidden, int K, int granule, __half* wout,
               float* bout);   // rows interleaved value/gate in `granule` blocks; w or b may be null (pack one only)
int f16_to_f32(cudaStream_t st, const __half* x, size_t n, float* out);

}  // namespace vs
