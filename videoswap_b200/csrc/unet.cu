// Host-side executor of the reference's AnimateDiffUNet3DModel.forward (videoswap/models/animatediff_models/unet.py:
// 328-481 and unet_blocks.py) on top of the sm_90a kernels.  Owns the packed weights and a static activation
// workspace; activations are NHWC fp16 ([(b f), h*w, C] tokens), so none of the reference's rearrange/permute/concat
// copies exist.  Weight names are the reference's state_dict keys.
#include <math.h>
#include <string.h>

#include <functional>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/videoswap_b200.h"
#include "common.cuh"
#include "kernels.h"

using namespace vs;

namespace {

enum LoadKind { LK_COPY_F16, LK_TO_F32, LK_CONV3, LK_CONV_UP, LK_GEGLU_W, LK_GEGLU_B, LK_IGNORE };

struct Loader {
  LoadKind kind;
  void* dst;
  int64_t numel;
  int a, b;   // conv: co, ci; geglu: hidden, K
};

struct Lin { __half* w = nullptr; float* b = nullptr; int N = 0, K = 0; };
struct Conv3 { __half* w = nullptr; float* b = nullptr; int co = 0, ci = 0; __half* wsub = nullptr; };   // wsub: 4 sub-pixel panels
struct Norm { float* g = nullptr; float* b = nullptr; int C = 0; };
// A linear layer with the LayerNorm in front of it folded in (kernels.h ln_fold): gamma-scaled weights, row sums, offsets
struct LnLin { __half* wf = nullptr; float* u = nullptr; float* c = nullptr; float* cpe = nullptr; };
struct FoldJob { const __half* w; int N, K; const float* gamma; const float* beta; const float* bias; const float* pe; int pe_len; LnLin dst; };
struct Resnet {
  Norm n1, n2; Conv3 c1, c2; Lin sc; bool has_sc = false; int cin = 0, cout = 0; int temb_off = 0;
};
struct Transformer {
  int C = 0, layer = 0;
  Norm norm, ln1, ln2, ln3; Lin proj_in, proj_out, out1, out2, ff2;
  __half* wqkv = nullptr; __half* wq = nullptr; __half* wkv = nullptr; __half* ff1w = nullptr; float* ff1b = nullptr;
  LnLin f_qkv, f_q, f_ff;               // ln1 -> QKV, ln2 -> to_q, ln3 -> GEGLU with the LayerNorm folded in
};
struct Motion {
  int C = 0;
  Norm norm, ln[2], ff_norm; Lin proj_in, proj_out, out[2], ff2;
  __half* wqkv[2] = {nullptr, nullptr}; __half* ff1w = nullptr; float* ff1b = nullptr;
  LnLin f_qkv[2], f_ff;                 // (LN + temporal PE) -> QKV, ff_norm -> GEGLU folded
};
struct Layer { Resnet res; bool has_tr = false; Transformer tr; bool has_mo = false; Motion mo; };
struct Block { std::vector<Layer> layers; bool has_sampler = false; Conv3 sampler; };

struct Act { __half* p; int c; };   // NHWC activation view at the current resolution

}  // namespace

struct vs_unet {
  vs_unet_config cfg;
  std::vector<void*> allocs;
  std::unordered_map<std::string, Loader> loaders;
  std::vector<std::string> names;
  std::vector<FoldJob> folds;           // re-derived lazily (next forward) after weight loads
  bool folds_dirty = true;

  // parameters
  __half* conv_in_w = nullptr; float* conv_in_b = nullptr;
  Lin te1, te2;                         // time_embedding.linear_1/2
  __half* tproj_w = nullptr; float* tproj_b = nullptr; int tproj_n = 0;   // all resnets' time_emb_proj, stacked
  Block down[4], up[4];
  Layer mid0; Resnet mid1;              // mid: resnet0 + transformer, then resnet1
  Norm norm_out; Conv3 conv_out;
  float* pe[4] = {nullptr, nullptr, nullptr, nullptr};   // [pe_max_len, C_l] fp32 per level

  // workspace
  size_t ws_bytes = 0; void* ws = nullptr;   // arena: grows monotonically, never shrinks (captured CUDA graphs hold raw
  int wsB = 0, wsF = 0, wsH = 0, wsW = 0;     // pointers into it); `ws_pinned` > 0 forbids the re-allocation altogether
  int ws_pinned = 0;
  int n_groupnorms = 0;                        // GroupNorm calls of one forward (sizes the statistics slices)
  __half *XIN, *XN, *T, *TN, *QKV, *ATT, *HH, *SC, *P0, *P1, *SCR, *KV, *RES, *OUT;
  std::vector<__half*> skip;            // 12 skip buffers
  float *F_T, *F_TE0, *F_TE1, *F_EMB, *F_TPROJ, *F_SUMS, *F_LNS, *F_LNP;

  // frame sharding (SURVEY 8e): this rank holds F/k frames of ONE batch element; exchanges over `fcomm` (comm.cu)
  vs_comm* fcomm = nullptr;
  int fshard = 0, fnshards = 1;

  // attention controllers (SURVEY 8f-2): when a hook is set, every spatial attention with fewer than hook_max_q queries
  // materialises its probabilities [(b f), heads, s, t] in `probs`, hands them to the hook, then applies them to V
  vs_attention_hook hook = nullptr; void* hook_user = nullptr; int hook_max_q = 0;
  __half* probs = nullptr; size_t probs_elems = 0;

  // debug taps
  bool taps_on = false;
  struct Tap { std::string name; void* p; int n, h, w, c; };
  std::vector<Tap> taps;

  ~vs_unet() {
    for (void* p : allocs) cudaFree(p);
    if (ws) cudaFree(ws);
    if (probs) cudaFree(probs);
    for (auto& t : taps) cudaFree(t.p);
  }

  template <typename T>
  T* alloc(size_t n) {
    void* p = nullptr;
    if (cudaMalloc(&p, n * sizeof(T)) != cudaSuccess) { set_error("cudaMalloc of %zu bytes failed", n * sizeof(T)); return nullptr; }
    cudaMemset(p, 0, n * sizeof(T));
    allocs.push_back(p);
    return reinterpret_cast<T*>(p);
  }
  void reg(const std::string& name, LoadKind k, void* dst, int64_t numel, int a = 0, int b = 0) {
    loaders[name] = Loader{k, dst, numel, a, b};
    names.push_back(name);
  }
  float* f32(const std::string& name, int64_t n) { float* p = alloc<float>(n); reg(name, LK_TO_F32, p, n); return p; }
  __half* f16(const std::string& name, int64_t n) { __half* p = alloc<__half>(n); reg(name, LK_COPY_F16, p, n); return p; }
  Norm norm(const std::string& p, int C) { Norm n; n.C = C; n.g = f32(p + ".weight", C); n.b = f32(p + ".bias", C); return n; }
  Lin lin(const std::string& p, int N, int K, bool bias = true) {
    Lin l; l.N = N; l.K = K; l.w = f16(p + ".weight", (int64_t)N * K); if (bias) l.b = f32(p + ".bias", N); return l;
  }
  // LayerNorm `n` (+ positional table pe [pe_len, K]) folded into the linear layer w [N, K] (+ bias): the folded copy is
  // re-derived from the unfolded weights after every vs_unet_load_weights (LoRA merges replace the weights).
  LnLin fold(const __half* w, int N, int K, const Norm& n, const float* bias, const float* pe, int pe_len) {
    LnLin f;
    if (!ln_fold_supported(K)) return f;
    f.wf = alloc<__half>((size_t)N * K);
    f.u = alloc<float>(N);
    f.c = alloc<float>(N);
    if (pe) f.cpe = alloc<float>((size_t)pe_len * N);
    folds.push_back(FoldJob{w, N, K, n.g, n.b, bias, pe, pe_len, f});
    return f;
  }
  Conv3 conv3(const std::string& p, int co, int ci) {
    Conv3 c; c.co = co; c.ci = ci;
    const int co_pad = co < 64 ? 64 : co;             // tiny-N convs (conv_out) read a zero-padded weight panel
    c.w = alloc<__half>((int64_t)co_pad * 9 * ci);
    reg(p + ".weight", LK_CONV3, c.w, (int64_t)co * ci * 9, co, ci);
    c.b = f32(p + ".bias", co);
    return c;
  }
};

namespace {

void build_resnet(vs_unet* h, Resnet& r, const std::string& p, int cin, int cout, int temb, int& toff) {
  r.cin = cin; r.cout = cout;
  r.n1 = h->norm(p + ".norm1", cin);
  r.c1 = h->conv3(p + ".conv1", cout, cin);
  r.temb_off = toff;
  h->reg(p + ".time_emb_proj.weight", LK_COPY_F16, h->tproj_w + (int64_t)toff * temb, (int64_t)cout * temb);
  h->reg(p + ".time_emb_proj.bias", LK_TO_F32, h->tproj_b + toff, cout);
  toff += cout;
  r.n2 = h->norm(p + ".norm2", cout);
  r.c2 = h->conv3(p + ".conv2", cout, cout);
  r.has_sc = cin != cout;
  if (r.has_sc) r.sc = h->lin(p + ".conv_shortcut", cout, cin);
}

void build_attn_fused(vs_unet* h, const std::string& p, int C, __half*& wqkv, Lin& out) {
  wqkv = h->alloc<__half>((int64_t)3 * C * C);
  h->reg(p + ".to_q.weight", LK_COPY_F16, wqkv, (int64_t)C * C);
  h->reg(p + ".to_k.weight", LK_COPY_F16, wqkv + (int64_t)C * C, (int64_t)C * C);
  h->reg(p + ".to_v.weight", LK_COPY_F16, wqkv + (int64_t)2 * C * C, (int64_t)C * C);
  out = h->lin(p + ".to_out.0", C, C);
}

void build_ff(vs_unet* h, const std::string& p, int C, __half*& w1, float*& b1, Lin& ff2) {
  w1 = h->alloc<__half>((int64_t)8 * C * C);
  b1 = h->alloc<float>(8 * C);
  h->reg(p + ".net.0.proj.weight", LK_GEGLU_W, w1, (int64_t)8 * C * C, 4 * C, C);
  h->reg(p + ".net.0.proj.bias", LK_GEGLU_B, b1, 8 * C, 4 * C, 1);
  ff2 = h->lin(p + ".net.2", C, 4 * C);
}

void build_transformer(vs_unet* h, Transformer& t, const std::string& p, int C, int ctx, int layer) {
  t.C = C; t.layer = layer;
  t.norm = h->norm(p + ".norm", C);
  t.proj_in = h->lin(p + ".proj_in", C, C);
  const std::string q = p + ".transformer_blocks.0";
  build_attn_fused(h, q + ".attn1", C, t.wqkv, t.out1);
  t.ln1 = h->norm(q + ".norm1", C);
  t.wq = h->f16(q + ".attn2.to_q.weight", (int64_t)C * C);
  t.wkv = h->alloc<__half>((int64_t)2 * C * ctx);
  h->reg(q + ".attn2.to_k.weight", LK_COPY_F16, t.wkv, (int64_t)C * ctx);
  h->reg(q + ".attn2.to_v.weight", LK_COPY_F16, t.wkv + (int64_t)C * ctx, (int64_t)C * ctx);
  t.out2 = h->lin(q + ".attn2.to_out.0", C, C);
  t.ln2 = h->norm(q + ".norm2", C);
  build_ff(h, q + ".ff", C, t.ff1w, t.ff1b, t.ff2);
  t.ln3 = h->norm(q + ".norm3", C);
  t.proj_out = h->lin(p + ".proj_out", C, C);
  t.f_qkv = h->fold(t.wqkv, 3 * C, C, t.ln1, nullptr, nullptr, 0);
  t.f_q = h->fold(t.wq, C, C, t.ln2, nullptr, nullptr, 0);
  t.f_ff = h->fold(t.ff1w, 8 * C, C, t.ln3, t.ff1b, nullptr, 0);
}

void build_motion(vs_unet* h, Motion& m, const std::string& p0, int C) {
  const std::string p = p0 + ".temporal_transformer";
  m.C = C;
  m.norm = h->norm(p + ".norm", C);
  m.proj_in = h->lin(p + ".proj_in", C, C);
  const std::string q = p + ".transformer_blocks.0";
  for (int i = 0; i < 2; ++i) {
    const std::string a = q + ".attention_blocks." + std::to_string(i);
    build_attn_fused(h, a, C, m.wqkv[i], m.out[i]);
    h->reg(a + ".processor.pos_encoder.pe", LK_IGNORE, nullptr, 0);   // closed-form table, rebuilt internally
  }
  for (int i = 0; i < 2; ++i) m.ln[i] = h->norm(q + ".norms." + std::to_string(i), C);
  build_ff(h, q + ".ff", C, m.ff1w, m.ff1b, m.ff2);
  m.ff_norm = h->norm(q + ".ff_norm", C);
  m.proj_out = h->lin(p + ".proj_out", C, C);
  const float* pe = nullptr;            // the table depends on C only: any level with this channel count will do
  for (int l = 0; l < 4; ++l) if (h->cfg.block_out_channels[l] == C) pe = h->pe[l];
  if (pe && h->cfg.pe_max_len <= 32) {
    for (int i = 0; i < 2; ++i) m.f_qkv[i] = h->fold(m.wqkv[i], 3 * C, C, m.ln[i], nullptr, pe, h->cfg.pe_max_len);
    m.f_ff = h->fold(m.ff1w, 8 * C, C, m.ff_norm, m.ff1b, nullptr, 0);
  }
}

int up_in_channels(const vs_unet_config& c, int i, int j, int* skip) {
  const int n = 4;
  int rev[4];
  for (int k = 0; k < n; ++k) rev[k] = c.block_out_channels[n - 1 - k];
  const int out_c = rev[i];
  const int prev = rev[i > 0 ? i - 1 : 0];
  const int in_c = rev[i + 1 < n ? i + 1 : n - 1];
  const int nl = c.layers_per_block + 1;
  *skip = (j == nl - 1) ? in_c : out_c;
  return (j == 0) ? prev : out_c;
}

}  // namespace

// =================================================================================================== create
extern "C" int vs_unet_create(const vs_unet_config* cfg, vs_unet** out) {
  VS_REQUIRE(cfg && out, "vs_unet_create: null argument");
  VS_REQUIRE(cfg->layers_per_block >= 1 && cfg->layers_per_block <= 4, "bad layers_per_block");
  for (int i = 0; i < 4; ++i)
    VS_REQUIRE(cfg->block_out_channels[i] % 64 == 0 && (cfg->block_out_channels[i] / cfg->num_heads == 40 ||
               cfg->block_out_channels[i] / cfg->num_heads == 80 || cfg->block_out_channels[i] / cfg->num_heads == 160),
               "block_out_channels[%d]=%d unsupported (need C %% 64 == 0 and head dim in {40,80,160})", i,
               cfg->block_out_channels[i]);
  VS_REQUIRE(cfg->cross_attention_dim % 64 == 0, "cross_attention_dim must be a multiple of 64");
  VS_REQUIRE(cfg->norm_num_groups >= 1 && cfg->norm_num_groups <= 32, "norm_num_groups must be in [1, 32] (statistics slices hold 32 groups)");
  vs_unet* h = new vs_unet();
  h->cfg = *cfg;
  const int* boc = cfg->block_out_channels;
  const int temb = boc[0] * 4, ctx = cfg->cross_attention_dim, lpb = cfg->layers_per_block;
  // temporal positional-encoding tables (closed form of motion_module.py:242-251)
  for (int l = 0; l < 4; ++l) {
    const int C = boc[l], L = cfg->pe_max_len;
    std::vector<float> t((size_t)L * C);
    for (int pos = 0; pos < L; ++pos)
      for (int i2 = 0; i2 < C; i2 += 2) {
        const float div = expf((float)i2 * (-logf(10000.0f) / (float)C));
        t[(size_t)pos * C + i2] = sinf((float)pos * div);
        if (i2 + 1 < C) t[(size_t)pos * C + i2 + 1] = cosf((float)pos * div);
      }
    h->pe[l] = h->alloc<float>((size_t)L * C);
    if (!h->pe[l]) { delete h; return 1; }
    cudaMemcpy(h->pe[l], t.data(), t.size() * sizeof(float), cudaMemcpyHostToDevice);
  }
  h->conv_in_w = h->f16("conv_in.weight", (int64_t)boc[0] * cfg->in_channels * 9);
  h->conv_in_b = h->f32("conv_in.bias", boc[0]);
  h->te1 = h->lin("time_embedding.linear_1", temb, boc[0]);
  h->te2 = h->lin("time_embedding.linear_2", temb, temb);
  // total stacked time_emb_proj rows
  int tn = 0;
  {
    int cout = boc[0];
    for (int i = 0; i < 4; ++i) { cout = boc[i]; tn += lpb * cout; }
    tn += 2 * boc[3];
    for (int i = 0; i < 4; ++i) tn += (lpb + 1) * boc[3 - i];
  }
  h->tproj_n = tn;
  h->tproj_w = h->alloc<__half>((int64_t)tn * temb);
  h->tproj_b = h->alloc<float>(tn);
  int toff = 0, layer = 0;
  int cout = boc[0];
  for (int i = 0; i < 4; ++i) {
    const int cin = cout;
    cout = boc[i];
    const std::string p = "down_blocks." + std::to_string(i);
    Block& b = h->down[i];
    b.layers.resize(lpb);
    for (int j = 0; j < lpb; ++j) {
      Layer& L = b.layers[j];
      build_resnet(h, L.res, p + ".resnets." + std::to_string(j), j == 0 ? cin : cout, cout, temb, toff);
      if (i < 3) { L.has_tr = true; build_transformer(h, L.tr, p + ".attentions." + std::to_string(j), cout, ctx, layer++); }
      if (cfg->use_motion_module && cfg->motion_down[i]) { L.has_mo = true; build_motion(h, L.mo, p + ".motion_modules." + std::to_string(j), cout); }
    }
    if (i < 3) { b.has_sampler = true; b.sampler = h->conv3(p + ".downsamplers.0.conv", cout, cout); }
  }
  build_resnet(h, h->mid0.res, "mid_block.resnets.0", boc[3], boc[3], temb, toff);
  h->mid0.has_tr = true;
  build_transformer(h, h->mid0.tr, "mid_block.attentions.0", boc[3], ctx, layer++);
  if (cfg->use_motion_module && cfg->motion_mid) { h->mid0.has_mo = true; build_motion(h, h->mid0.mo, "mid_block.motion_modules.0", boc[3]); }
  build_resnet(h, h->mid1, "mid_block.resnets.1", boc[3], boc[3], temb, toff);
  for (int i = 0; i < 4; ++i) {
    const std::string p = "up_blocks." + std::to_string(i);
    Block& b = h->up[i];
    const int oc = boc[3 - i];
    b.layers.resize(lpb + 1);
    for (int j = 0; j <= lpb; ++j) {
      Layer& L = b.layers[j];
      int skipc;
      const int run = up_in_channels(*cfg, i, j, &skipc);
      build_resnet(h, L.res, p + ".resnets." + std::to_string(j), run + skipc, oc, temb, toff);
      if (i > 0) { L.has_tr = true; build_transformer(h, L.tr, p + ".attentions." + std::to_string(j), oc, ctx, layer++); }
      if (cfg->use_motion_module && cfg->motion_up[i]) { L.has_mo = true; build_motion(h, L.mo, p + ".motion_modules." + std::to_string(j), oc); }
    }
    if (i < 3) {
      b.has_sampler = true;
      Conv3& c = b.sampler;           // [co, 9, ci] followed by 4 x [co, 4, ci]
      c.co = oc; c.ci = oc;
      c.w = h->alloc<__half>((size_t)oc * 9 * oc + (size_t)16 * oc * oc);
      c.wsub = c.w + (size_t)oc * 9 * oc;
      h->reg(p + ".upsamplers.0.conv.weight", LK_CONV_UP, c.w, (int64_t)oc * oc * 9, oc, oc);
      c.b = h->f32(p + ".upsamplers.0.conv.bias", oc);
    }
  }
  h->norm_out = h->norm("conv_norm_out", boc[0]);
  h->conv_out = h->conv3("conv_out", cfg->out_channels, boc[0]);
  VS_REQUIRE(toff == tn, "internal: time_emb_proj stacking mismatch (%d vs %d)", toff, tn);
  {   // GroupNorm calls per forward: 2 per resnet, 1 per transformer, 1 per motion module, conv_norm_out
    int n = 1 + 2 /*mid1*/;
    auto count = [&](const Layer& L) { n += 2 + (L.has_tr ? 1 : 0) + (L.has_mo ? 1 : 0); };
    for (int i = 0; i < 4; ++i) { for (const Layer& L : h->down[i].layers) count(L); for (const Layer& L : h->up[i].layers) count(L); }
    count(h->mid0);
    h->n_groupnorms = n;
  }
  for (void* p : h->allocs) if (!p) { delete h; return 1; }
  VS_CHECK_CUDA(cudaGetLastError());
  *out = h;
  return 0;
}

extern "C" void vs_unet_destroy(vs_unet* h) { delete h; }
extern "C" int vs_unet_num_params(const vs_unet* h) { return (int)h->names.size(); }
extern "C" const char* vs_unet_param_name(const vs_unet* h, int i) { return h->names[i].c_str(); }
extern "C" size_t vs_unet_workspace_bytes(const vs_unet* h) { return h->ws_bytes; }

extern "C" int vs_unet_load_weights(vs_unet* h, void* stream, int n, const char* const* names, const void* const* ptrs,
                                    const int64_t* numels) {
  cudaStream_t st = (cudaStream_t)stream;
  for (int i = 0; i < n; ++i) {
    auto it = h->loaders.find(names[i]);
    VS_REQUIRE(it != h->loaders.end(), "vs_unet_load_weights: unknown parameter '%s'", names[i]);
    const Loader& L = it->second;
    if (L.kind == LK_IGNORE) continue;
    VS_REQUIRE(numels[i] == L.numel, "vs_unet_load_weights: '%s' has %lld elements, expected %lld", names[i],
               (long long)numels[i], (long long)L.numel);
    const __half* src = (const __half*)ptrs[i];
    int e = 0;
    switch (L.kind) {
      case LK_COPY_F16:
        VS_CHECK_CUDA(cudaMemcpyAsync(L.dst, src, (size_t)L.numel * 2, cudaMemcpyDeviceToDevice, st));
        break;
      case LK_TO_F32: e = f16_to_f32(st, src, (size_t)L.numel, (float*)L.dst); break;
      case LK_CONV3: e = pack_conv3x3(st, src, L.a, L.b, (__half*)L.dst); break;
      case LK_CONV_UP:                  // up-sampler conv: the plain 3x3 panel (A/B path) and the four 2x2 sub-pixel panels
        e = pack_conv3x3(st, src, L.a, L.b, (__half*)L.dst);
        if (!e) e = pack_conv_subpixel(st, src, L.a, L.b, (__half*)L.dst + (size_t)L.a * 9 * L.b);
        break;
      case LK_GEGLU_W: e = pack_geglu(st, src, nullptr, L.a, L.b, kGegluGranule, (__half*)L.dst, nullptr); break;
      case LK_GEGLU_B: e = pack_geglu(st, nullptr, src, L.a, 1, kGegluGranule, nullptr, (float*)L.dst); break;
      default: break;
    }
    if (e) return e;
  }
  h->folds_dirty = true;                // the LayerNorm-folded copies are re-derived once, at the next forward
  return 0;
}

// =================================================================================================== forward
namespace {

struct Ctx {
  vs_unet* h; cudaStream_t st;
  int B, F, NI, H, W;      // W/H are the CURRENT resolution during the walk
  const __half* ehs; int ehs_tokens, ehs_layers;
  int gn_idx = 0;          // GroupNorm call counter: every call owns a slice of F_SUMS, all zeroed by ONE memset per forward
  int place = 0;           // 0 down / 1 mid / 2 up: the `place_in_unet` the attention controllers are told
  int ln_parts = 0;        // > 0: F_LNP holds that many per-row partial-sum slices of the tensor the last `linear` wrote
};

// every GroupNorm call of a forward owns one slice [NI, 32 groups, 2] of F_SUMS (h->n_groupnorms of them, counted at create)
inline float* next_sums(Ctx& c) {
  if (c.gn_idx >= c.h->n_groupnorms) { set_error("internal: more GroupNorm calls (%d) than statistics slices (%d)", c.gn_idx + 1, c.h->n_groupnorms); return nullptr; }
  return c.h->F_SUMS + (size_t)(c.gn_idx++) * ((size_t)c.NI * 64);
}
#define NEXT_SUMS(var) float* var = next_sums(c); if (!var) return 2

#define RUN(expr) do { if (int _e = (expr)) return _e; } while (0)

int tap(Ctx& c, const std::string& name, const __half* p, int C) {
  vs_unet* h = c.h;
  if (!h->taps_on) return 0;
  const size_t bytes = (size_t)c.NI * c.H * c.W * C * 2;
  void* d = nullptr;
  VS_CHECK_CUDA(cudaMalloc(&d, bytes));
  VS_CHECK_CUDA(cudaMemcpyAsync(d, p, bytes, cudaMemcpyDeviceToDevice, c.st));
  h->taps.push_back({name, d, c.NI, c.H, c.W, C});
  return 0;
}

// ln_out: the output feeds a LayerNorm that is folded into the next GEMM -> the epilogue also writes the row statistics
// (per column tile) into F_LNP and c.ln_parts says how many slices (0 when the fused statistics are switched off).
int linear(Ctx& c, const __half* A, int M, const Lin& l, const __half* residual, __half* out, bool ln_out = false) {
  GemmArgs g;
  g.A = A; g.K1 = l.K; g.lda1 = l.K; g.Bw = l.w; g.M = M; g.N = l.N; g.bias = l.b;
  g.residual = residual; g.ldr = l.N; g.out = out; g.ldc = l.N;
  c.ln_parts = 0;
  if (ln_out && get_option("ln_fuse") != 0 && get_option("ln_fold") != 0 && ln_fold_supported(l.N) && l.N % 32 == 0) {
    const int parts = gemm_n_tiles(g);
    if (parts >= 1 && (long long)M * parts <= 4LL * c.NI * c.h->wsH * c.h->wsW) {   // capacity of F_LNP (float2 slots)
      g.ln_sums_out = c.h->F_LNP;
      c.ln_parts = parts;
    }
  }
  return gemm_tc(c.st, g);
}

int conv(Ctx& c, const __half* x, int C1, const Conv3& w, const float* rowvec, const __half* residual, __half* out) {
  GemmArgs g;
  g.A = x; g.K1 = C1; g.lda1 = C1; g.Bw = w.w; g.taps = 9; g.nimg = c.NI; g.H = c.H; g.W = c.W;
  g.M = c.NI * c.H * c.W; g.N = w.co; g.bias = w.b; g.rowvec = rowvec; g.ldrv = c.h->tproj_n; g.pix_per_batch = c.F * c.H * c.W;
  g.residual = residual; g.ldr = w.co; g.out = out; g.ldc = w.co;
  return gemm_tc(c.st, g);
}

int resnet(Ctx& c, const Resnet& r, const __half* in1, int C1, const __half* in2, int C2, __half* out) {
  vs_unet* h = c.h;
  const int hw = c.H * c.W, G = h->cfg.norm_num_groups;
  const float eps = h->cfg.norm_eps;
  VS_REQUIRE(C1 + C2 == r.cin, "internal: resnet input channels %d+%d != %d", C1, C2, r.cin);
  const int k = h->fnshards;          // frame shards: the 5-D GroupNorm statistics span all of them (resnet.py:166,177)
  NEXT_SUMS(sums);
  RUN(groupnorm_stats(c.st, in1, C1, in2, C2, c.NI, hw, c.F, G, sums, false));
  if (k > 1) RUN(comm_all_reduce_sum_f32(h->fcomm, c.st, sums, (size_t)c.B * G * 2));
  RUN(groupnorm_apply(c.st, in1, C1, in2, C2, c.NI, hw, c.F, G, sums, eps, r.n1.g, r.n1.b, true, h->XN, k));
  RUN(conv(c, h->XN, r.cin, r.c1, h->F_TPROJ + r.temb_off, nullptr, h->T));
  sums = next_sums(c);
  if (!sums) return 2;
  RUN(groupnorm_stats(c.st, h->T, r.cout, nullptr, 0, c.NI, hw, c.F, G, sums, false));
  if (k > 1) RUN(comm_all_reduce_sum_f32(h->fcomm, c.st, sums, (size_t)c.B * G * 2));
  RUN(groupnorm_apply(c.st, h->T, r.cout, nullptr, 0, c.NI, hw, c.F, G, sums, eps, r.n2.g, r.n2.b, true, h->XN, k));
  const __half* residual = in1;
  if (r.has_sc) {
    GemmArgs g;
    g.A = in1; g.K1 = C1; g.lda1 = C1; g.A2 = in2; g.K2 = C2; g.lda2 = C2; g.Bw = r.sc.w; g.M = c.NI * hw; g.N = r.cout;
    g.bias = r.sc.b; g.out = h->SC; g.ldc = r.cout;
    RUN(gemm_tc(c.st, g));
    residual = h->SC;
  } else {
    VS_REQUIRE(in2 == nullptr, "internal: concat input without shortcut conv");
  }
  RUN(conv(c, h->XN, r.cout, r.c2, nullptr, residual, out));
  return 0;
}

// LayerNorm + linear with the norm folded into the GEMM: row statistics of the raw input, then ONE GEMM on the raw input
// (no normalised tensor is written or read).  pe_frames > 0: per-frame positional offsets (temporal LayerNorm + PE).
bool use_fold(const LnLin& f) { return f.wf != nullptr && get_option("ln_fold") != 0; }
int ln_linear(Ctx& c, const __half* x, int M, int C, const LnLin& f, int N, int mode, int hw, int pe_frames, __half* out, int ldc) {
  vs_unet* h = c.h;
  GemmArgs g;
  g.A = x; g.K1 = C; g.lda1 = C; g.Bw = f.wf; g.M = M; g.N = N; g.bias = f.c; g.ln_u = f.u;
  if (c.ln_parts > 0) {            // the GEMM that wrote x left its row statistics in F_LNP
    g.ln_parts = h->F_LNP; g.ln_nparts = c.ln_parts;
    c.ln_parts = 0;
  } else {
    RUN(ln_rowstats(c.st, x, M, C, h->F_LNS));
    g.ln_stats = h->F_LNS;
  }
  g.out = out; g.ldc = ldc; g.mode = mode;
  if (pe_frames > 0) { g.rowvec = f.cpe; g.ldrv = N; g.pix_per_batch = hw; g.rv_mod = pe_frames; }
  return gemm_tc(c.st, g);
}

int geglu_ff(Ctx& c, const __half* tn, int M, int C, const __half* w1, const float* b1, const Lin& ff2, __half* t) {
  vs_unet* h = c.h;
  GemmArgs g;
  g.A = tn; g.K1 = C; g.lda1 = C; g.Bw = w1; g.M = M; g.N = 8 * C; g.bias = b1; g.out = h->HH; g.ldc = 4 * C; g.mode = EPI_GEGLU;
  RUN(gemm_tc(c.st, g));
  return linear(c, h->HH, M, ff2, t, t);
}

// Spatial attention with the controller hook: explicit probabilities for the small-resolution layers while a hook is set
// (attention_register.py:96,140-150: xformers / flash path for >= 32^2 queries, controller path below).
int attention_hooked(Ctx& c, const Transformer& t, int is_cross, int place, const __half* q, int ldq, const __half* k, int ldk,
                     const __half* v, int ldv, __half* o, int ldo, int nq, int nk, int heads, int d, long long q_bs, long long kv_bs,
                     long long o_bs, int kv_div) {
  vs_unet* h = c.h;
  if (h->hook == nullptr || nq >= h->hook_max_q)
    return attention(c.st, q, ldq, k, ldk, v, ldv, o, ldo, c.NI, nq, nk, heads, d, q_bs, kv_bs, o_bs, kv_div);
  const size_t need = (size_t)c.NI * heads * nq * nk;
  if (need > h->probs_elems) {          // controller mode runs eagerly (never inside a captured graph)
    if (h->probs) { VS_CHECK_CUDA(cudaStreamSynchronize(c.st)); cudaFree(h->probs); h->probs = nullptr; }
    VS_CHECK_CUDA(cudaMalloc(&h->probs, need * sizeof(__half)));
    h->probs_elems = need;
  }
  RUN(attention_probs(c.st, q, ldq, k, ldk, h->probs, c.NI, nq, nk, heads, d, q_bs, kv_bs, kv_div));
  h->hook(h->hook_user, t.layer, is_cross, place, h->probs, c.NI, heads, nq, nk, (void*)c.st);
  return attention_apply_probs(c.st, h->probs, v, ldv, o, ldo, c.NI, nq, nk, heads, d, kv_bs, o_bs, kv_div);
}

int transformer(Ctx& c, const Transformer& t, __half* x) {
  vs_unet* h = c.h;
  const int hw = c.H * c.W, C = t.C, M = c.NI * hw, heads = h->cfg.num_heads, d = C / heads;
  NEXT_SUMS(sums);
  {
    const int e = groupnorm_frame_fused(c.st, x, C, c.NI, hw, h->cfg.norm_num_groups, 1e-6f, t.norm.g, t.norm.b, false, h->XN);
    if (e > 0) return e;
    if (e < 0) {
      RUN(groupnorm_stats(c.st, x, C, nullptr, 0, c.NI, hw, 1, h->cfg.norm_num_groups, sums, false));
      RUN(groupnorm_apply(c.st, x, C, nullptr, 0, c.NI, hw, 1, h->cfg.norm_num_groups, sums, 1e-6f, t.norm.g, t.norm.b, false, h->XN));
    }
  }
  RUN(linear(c, h->XN, M, t.proj_in, nullptr, h->T, use_fold(t.f_qkv)));
  // self-attention
  if (use_fold(t.f_qkv)) {
    RUN(ln_linear(c, h->T, M, C, t.f_qkv, 3 * C, EPI_LINEAR, hw, 0, h->QKV, 3 * C));
  } else {
    RUN(layernorm(c.st, h->T, M, C, t.ln1.g, t.ln1.b, nullptr, 1, 1, h->TN));
    GemmArgs g; g.A = h->TN; g.K1 = C; g.lda1 = C; g.Bw = t.wqkv; g.M = M; g.N = 3 * C; g.out = h->QKV; g.ldc = 3 * C; RUN(gemm_tc(c.st, g));
  }
  RUN(attention_hooked(c, t, 0, c.place, h->QKV, 3 * C, h->QKV + C, 3 * C, h->QKV + 2 * C, 3 * C, h->ATT, C, hw, hw, heads, d,
                       (long long)hw * 3 * C, (long long)hw * 3 * C, (long long)hw * C, 1));
  RUN(linear(c, h->ATT, M, t.out1, h->T, h->T, use_fold(t.f_q)));
  // cross-attention to the (ED-LoRA layer-selected) text embeddings; K/V were projected once per (batch, layer)
  if (use_fold(t.f_q)) {
    RUN(ln_linear(c, h->T, M, C, t.f_q, C, EPI_LINEAR, hw, 0, h->QKV, C));
  } else {
    RUN(layernorm(c.st, h->T, M, C, t.ln2.g, t.ln2.b, nullptr, 1, 1, h->TN));
    GemmArgs g; g.A = h->TN; g.K1 = C; g.lda1 = C; g.Bw = t.wq; g.M = M; g.N = C; g.out = h->QKV; g.ldc = C; RUN(gemm_tc(c.st, g));
  }
  {
    const int nk = c.ehs_tokens;
    const int ctx = h->cfg.cross_attention_dim;
    const int L = c.ehs_layers > 0 ? c.ehs_layers : 1;
    const int li = c.ehs_layers > 0 ? t.layer : 0;
    VS_REQUIRE(li < L, "ED-LoRA embeddings have %d layers but layer %d was requested", L, li);
    for (int b = 0; b < c.B; ++b) {
      GemmArgs g;
      g.A = c.ehs + ((long long)(b * L + li) * nk) * ctx; g.K1 = ctx; g.lda1 = ctx; g.Bw = t.wkv; g.M = nk; g.N = 2 * C;
      g.out = h->KV + (long long)b * nk * 2 * C; g.ldc = 2 * C;
      RUN(gemm_tc(c.st, g));
    }
    RUN(attention_hooked(c, t, 1, c.place, h->QKV, C, h->KV, 2 * C, h->KV + C, 2 * C, h->ATT, C, hw, nk, heads, d, (long long)hw * C,
                         (long long)nk * 2 * C, (long long)hw * C, c.F));
  }
  RUN(linear(c, h->ATT, M, t.out2, h->T, h->T, use_fold(t.f_ff)));
  // feed-forward
  if (use_fold(t.f_ff)) {
    RUN(ln_linear(c, h->T, M, C, t.f_ff, 8 * C, EPI_GEGLU, hw, 0, h->HH, 4 * C));
    RUN(linear(c, h->HH, M, t.ff2, h->T, h->T));
  } else {
    RUN(layernorm(c.st, h->T, M, C, t.ln3.g, t.ln3.b, nullptr, 1, 1, h->TN));
    RUN(geglu_ff(c, h->TN, M, C, t.ff1w, t.ff1b, t.ff2, h->T));
  }
  RUN(linear(c, h->T, M, t.proj_out, x, x));
  return 0;
}

int motion(Ctx& c, const Motion& m, int level, __half* x) {
  vs_unet* h = c.h;
  const int hw_all = c.H * c.W, C = m.C, M = c.NI * hw_all;
  // Frame shards: the temporal attention couples the F frames of every pixel and everything else inside the module is per
  // pixel, so the module runs on ALL frames x 1/k of the pixels: frames <-> pixels all-to-all of the GroupNorm output on
  // the way in and of proj_out's result on the way back (2 C values per token instead of K and V per attention).
  const int k = h->fnshards;
  const int Ft = c.F * k;                     // frames the attention sees
  const int hw = hw_all / k;                  // pixels per frame this rank owns inside the module
  VS_REQUIRE(Ft <= h->cfg.pe_max_len, "video_length %d exceeds temporal_position_encoding_max_len %d", Ft, h->cfg.pe_max_len);
  if (k > 1) VS_REQUIRE(c.B == 1 && hw_all % k == 0, "frame sharding needs batch 1 per rank and h*w (%d) divisible by the %d shards", hw_all, k);
  NEXT_SUMS(sums);
  {
    const int e = groupnorm_frame_fused(c.st, x, C, c.NI, hw_all, 32, 1e-6f, m.norm.g, m.norm.b, false, h->XN);
    if (e > 0) return e;
    if (e < 0) {
      RUN(groupnorm_stats(c.st, x, C, nullptr, 0, c.NI, hw_all, 1, 32, sums, false));
      RUN(groupnorm_apply(c.st, x, C, nullptr, 0, c.NI, hw_all, 1, 32, sums, 1e-6f, m.norm.g, m.norm.b, false, h->XN));
    }
  }
  const __half* xin = h->XN;
  if (k > 1) {
    RUN(comm_all_to_all_rows(h->fcomm, c.st, h->XN, h->SC, c.F, (size_t)hw * C, 0));    // [F/k, k, hw C] -> [k, F/k, hw C] = [F, hw, C]
    xin = h->SC;
  }
  RUN(linear(c, xin, M, m.proj_in, nullptr, h->T, use_fold(m.f_qkv[0])));
  for (int i = 0; i < 2; ++i) {
    if (use_fold(m.f_qkv[i])) {
      RUN(ln_linear(c, h->T, M, C, m.f_qkv[i], 3 * C, EPI_LINEAR, hw, Ft, h->QKV, 3 * C));
    } else {
      RUN(layernorm(c.st, h->T, M, C, m.ln[i].g, m.ln[i].b, h->pe[level], hw, Ft, h->TN));
      GemmArgs g; g.A = h->TN; g.K1 = C; g.lda1 = C; g.Bw = m.wqkv[i]; g.M = M; g.N = 3 * C; g.out = h->QKV; g.ldc = 3 * C; RUN(gemm_tc(c.st, g));
    }
    RUN(temporal_attention(c.st, h->QKV, h->ATT, c.B, Ft, hw, C, h->cfg.motion_num_heads));
    RUN(linear(c, h->ATT, M, m.out[i], h->T, h->T, i == 0 ? use_fold(m.f_qkv[1]) : use_fold(m.f_ff)));
  }
  if (use_fold(m.f_ff)) {
    RUN(ln_linear(c, h->T, M, C, m.f_ff, 8 * C, EPI_GEGLU, hw, 0, h->HH, 4 * C));
    RUN(linear(c, h->HH, M, m.ff2, h->T, h->T));
  } else {
    RUN(layernorm(c.st, h->T, M, C, m.ff_norm.g, m.ff_norm.b, nullptr, 1, 1, h->TN));
    RUN(geglu_ff(c, h->TN, M, C, m.ff1w, m.ff1b, m.ff2, h->T));
  }
  if (k > 1) {
    RUN(linear(c, h->T, M, m.proj_out, nullptr, h->XN));
    RUN(comm_all_to_all_rows(h->fcomm, c.st, h->XN, h->SC, c.F, (size_t)hw * C, 1));    // back to [F/k, hw_all, C]
    return add_inplace(c.st, x, h->SC, (size_t)M * C, 1.f);     // the module's residual: fp16 add, as in the fused epilogue
  }
  RUN(linear(c, h->T, M, m.proj_out, x, x));
  return 0;
}

size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

// Lays the activation arena out for (B, F, H, W).  The arena only ever GROWS (a smaller shape re-uses it with a new
// layout), and never while it is pinned: a captured CUDA graph holds raw pointers into it, so a re-allocation would leave
// the graph reading and writing freed memory (vs_unet_pin_workspace; GraphedStep pins).
int ensure_workspace(vs_unet* h, int B, int F, int H, int W) {
  if (h->ws && h->wsB == B && h->wsF == F && h->wsH == H && h->wsW == W) return 0;
  const int* boc = h->cfg.block_out_channels;
  const size_t NI = (size_t)B * F;
  // per-level pixel counts
  size_t hw[4]; int hh = H, ww = W;
  for (int l = 0; l < 4; ++l) { hw[l] = (size_t)hh * ww; hh = (hh - 1) / 2 + 1; ww = (ww - 1) / 2 + 1; }
  size_t maxC = 0, maxCat = 0;
  for (int l = 0; l < 4; ++l) {
    maxC = std::max(maxC, NI * hw[l] * boc[l]);
    maxCat = std::max(maxCat, NI * hw[l] * (size_t)(boc[l] + boc[std::min(l + 1, 3)]) );
    maxCat = std::max(maxCat, NI * hw[l] * (size_t)(2 * boc[l]));
  }
  std::vector<std::pair<__half**, size_t>> req;
  auto want = [&](__half** p, size_t elems) { req.push_back({p, elems}); };
  want(&h->XIN, NI * hw[0] * 8);
  want(&h->XN, maxCat);
  want(&h->T, maxC); want(&h->TN, maxC); want(&h->QKV, 3 * maxC); want(&h->ATT, maxC); want(&h->HH, 4 * maxC);
  // P0 / P1 ping-pong the running sample of the mid / up path, including the up-samplers' outputs, which carry the channel
  // count of the COARSER level at the finer resolution (e.g. 640 channels at 64x64: twice the largest block tensor).
  // (Round 1 sized them with maxC: the last up-sampler's output overran its buffer into the neighbouring one -- harmless
  // only while that neighbour happened to be dead; caught by the 64x64 reference fixture once the sub-pixel conv read it.)
  size_t maxP = maxC;
  for (int l = 0; l < 3; ++l) maxP = std::max(maxP, NI * hw[l] * (size_t)boc[l + 1]);
  want(&h->SC, maxC); want(&h->P0, maxP); want(&h->P1, maxP);
  want(&h->SCR, std::max(std::max(NI * hw[1] * 9 * boc[0], 4 * maxC), (NI * hw[0] + boc[0]) * 64));   // im2col (stride-2) /
                // nearest-upsample scratch / conv_in patch rows
  want(&h->KV, (size_t)B * 128 * 2 * boc[3]);
  want(&h->RES, maxC);
  want(&h->OUT, NI * hw[0] * 8);
  // skips: conv_in, then per down block lpb layers (+ down-sampler output)
  h->skip.assign(0, nullptr);
  std::vector<size_t> skip_elems;
  skip_elems.push_back(NI * hw[0] * boc[0]);
  for (int i = 0; i < 4; ++i) {
    for (int j = 0; j < h->cfg.layers_per_block; ++j) skip_elems.push_back(NI * hw[i] * boc[i]);
    if (i < 3) skip_elems.push_back(NI * hw[i + 1] * boc[i]);
  }
  h->skip.resize(skip_elems.size());
  for (size_t i = 0; i < skip_elems.size(); ++i) want(&h->skip[i], skip_elems[i]);
  size_t total = 0;
  for (auto& r : req) total += align_up(r.second * 2);
  const int temb = boc[0] * 4;
  const size_t fl = align_up(4 * 64) + align_up((size_t)B * boc[0] * 4) + 2 * align_up((size_t)B * temb * 4) +
                    align_up((size_t)B * h->tproj_n * 4) + align_up((size_t)h->n_groupnorms * NI * 64 * 4) +
                    align_up(NI * hw[0] * 2 * 4) + align_up(NI * hw[0] * 4 * 2 * 4);
  total += fl;
  if (total > h->ws_bytes) {
    VS_REQUIRE(h->ws_pinned == 0, "vs_unet_forward: shape [%d,%d,%d,%d] needs a %zu-byte workspace but the current one "
               "(%zu bytes) is pinned by a captured CUDA graph; run the largest shape first or call "
               "vs_unet_reserve_workspace before capturing", B, F, H, W, total, h->ws_bytes);
    if (h->ws) { VS_CHECK_CUDA(cudaDeviceSynchronize()); cudaFree(h->ws); h->ws = nullptr; h->ws_bytes = 0; }
    VS_CHECK_CUDA(cudaMalloc(&h->ws, total));
    h->ws_bytes = total;
  }
  char* p = (char*)h->ws;
  for (auto& r : req) { *r.first = (__half*)p; p += align_up(r.second * 2); }
  h->F_T = (float*)p; p += align_up(4 * 64);
  h->F_TE0 = (float*)p; p += align_up((size_t)B * boc[0] * 4);
  h->F_TE1 = (float*)p; p += align_up((size_t)B * temb * 4);
  h->F_EMB = (float*)p; p += align_up((size_t)B * temb * 4);
  h->F_TPROJ = (float*)p; p += align_up((size_t)B * h->tproj_n * 4);
  h->F_SUMS = (float*)p; p += align_up((size_t)h->n_groupnorms * NI * 64 * 4);
  h->F_LNS = (float*)p; p += align_up(NI * hw[0] * 2 * 4);
  h->F_LNP = (float*)p;            // LayerNorm partial sums: up to 4 column-tile slices of [NI * hw0] float2
  h->wsB = B; h->wsF = F; h->wsH = H; h->wsW = W;
  return 0;
}

}  // namespace

extern "C" int vs_unet_set_frame_shard(vs_unet* h, vs_comm* comm, int shard, int nshards) {
  VS_REQUIRE(h != nullptr && nshards >= 1 && shard >= 0 && shard < nshards, "vs_unet_set_frame_shard: bad arguments");
  VS_REQUIRE(nshards == 1 || (comm != nullptr && comm_size(comm) == nshards && comm_rank(comm) == shard),
             "vs_unet_set_frame_shard: the communicator must have exactly one rank per shard, ranked by shard");
  h->fcomm = nshards > 1 ? comm : nullptr;
  h->fshard = shard; h->fnshards = nshards;
  return 0;
}

extern "C" int vs_unet_set_attention_hook(vs_unet* h, vs_attention_hook hook, void* user, int max_queries) {
  VS_REQUIRE(h != nullptr, "vs_unet_set_attention_hook: null handle");
  VS_REQUIRE(hook == nullptr || h->ws_pinned == 0, "attention hooks run eagerly: release the captured CUDA graph first");
  h->hook = hook; h->hook_user = user; h->hook_max_q = max_queries > 0 ? max_queries : 32 * 32;
  return 0;
}

extern "C" int vs_unet_pin_workspace(vs_unet* h, int pin) {
  VS_REQUIRE(h != nullptr, "vs_unet_pin_workspace: null handle");
  h->ws_pinned += pin ? 1 : -1;
  if (h->ws_pinned < 0) h->ws_pinned = 0;
  return 0;
}
extern "C" int vs_unet_reserve_workspace(vs_unet* h, int B, int F, int H, int W) {
  VS_REQUIRE(h && B >= 1 && F >= 1 && H >= 1 && W >= 1, "vs_unet_reserve_workspace: bad arguments");
  return ensure_workspace(h, B, F, H, W);
}

extern "C" int vs_unet_enable_taps(vs_unet* h, int enable) {
  for (auto& t : h->taps) cudaFree(t.p);
  h->taps.clear();
  h->taps_on = enable != 0;
  return 0;
}
extern "C" int vs_unet_num_taps(const vs_unet* h) { return (int)h->taps.size(); }
extern "C" int vs_unet_get_tap(const vs_unet* h, int i, const char** name, const void** p, int* n, int* hh, int* ww, int* c) {
  VS_REQUIRE(i >= 0 && i < (int)h->taps.size(), "tap index out of range");
  const auto& t = h->taps[i];
  *name = t.name.c_str(); *p = t.p; *n = t.n; *hh = t.h; *ww = t.w; *c = t.c;
  return 0;
}

extern "C" int vs_unet_copy_tap(const vs_unet* h, void* stream, int i, void* d_dst) {
  VS_REQUIRE(i >= 0 && i < (int)h->taps.size(), "tap index out of range");
  const auto& t = h->taps[i];
  VS_CHECK_CUDA(cudaMemcpyAsync(d_dst, t.p, (size_t)t.n * t.h * t.w * t.c * 2, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

extern "C" int vs_unet_forward(vs_unet* h, void* stream, const void* d_sample, int io_f32, int B, int F, int H, int W,
                               const float* d_timesteps, const void* d_ehs, int ehs_tokens, int ehs_layers,
                               const void* const* d_residuals, int residuals_nhwc, float residual_scale, void* d_out) {
  VS_REQUIRE(h && d_sample && d_timesteps && d_ehs && d_out, "vs_unet_forward: null argument");
  VS_REQUIRE(B >= 1 && F >= 1 && H >= 1 && W >= 1, "vs_unet_forward: bad shape");
  VS_REQUIRE(ehs_tokens >= 1 && ehs_tokens <= 128, "vs_unet_forward: ehs_tokens out of range");
  VS_REQUIRE(h->cfg.in_channels <= 8 && h->cfg.out_channels <= 8, "in/out channels > 8 unsupported");
  VS_REQUIRE(h->fnshards == 1 || B == 1, "frame-sharded forward: one batch element per rank (got B = %d)", B);
  cudaStream_t st = (cudaStream_t)stream;
  RUN(ensure_workspace(h, B, F, H, W));
  if (h->folds_dirty) {
    for (const FoldJob& f : h->folds)
      RUN(ln_fold(st, f.w, f.N, f.K, f.gamma, f.beta, f.bias, f.pe, f.pe_len, f.dst.wf, f.dst.u, f.dst.c, f.dst.cpe));
    h->folds_dirty = false;
  }
  if (h->taps_on) { for (auto& t : h->taps) cudaFree(t.p); h->taps.clear(); }
  const vs_unet_config& cf = h->cfg;
  const int* boc = cf.block_out_channels;
  const int temb = boc[0] * 4, lpb = cf.layers_per_block;
  Ctx c{h, st, B, F, B * F, H, W, (const __half*)d_ehs, ehs_tokens, ehs_layers};

  VS_CHECK_CUDA(cudaMemsetAsync(h->F_SUMS, 0, (size_t)h->n_groupnorms * c.NI * 64 * sizeof(float), st));
  // ---- time embedding (unet.py:376-397): Timesteps -> Linear -> SiLU -> Linear; then every resnet's projection of
  //      SiLU(emb) in one stacked tiny-M linear (resnet.py:171-172)
  RUN(timestep_embedding(st, d_timesteps, B, boc[0], h->F_TE0));
  RUN(small_linear(st, h->F_TE0, B, boc[0], h->te1.w, h->te1.b, temb, false, true, h->F_TE1));
  RUN(small_linear(st, h->F_TE1, B, temb, h->te2.w, h->te2.b, temb, false, false, h->F_EMB));
  RUN(small_linear(st, h->F_EMB, B, temb, h->tproj_w, h->tproj_b, h->tproj_n, true, false, h->F_TPROJ));

  // ---- conv_in
  RUN(ncfhw_to_nhwc(st, d_sample, io_f32, B, cf.in_channels, F, H, W, h->XIN));
  int si = 0;
  RUN(conv_in_3x3(st, h->XIN, c.NI, H, W, cf.in_channels, h->conv_in_w, h->conv_in_b, boc[0], h->skip[si], h->SCR));
  RUN(tap(c, "conv_in", h->skip[si], boc[0]));
  const __half* cur = h->skip[si];
  int curC = boc[0];
  std::vector<std::pair<const __half*, int>> skips;
  skips.push_back({cur, curC});
  ++si;

  // ---- down path
  for (int i = 0; i < 4; ++i) {
    const Block& blk = h->down[i];
    const __half* res_l = nullptr;
    if (d_residuals && d_residuals[i]) {
      if (residuals_nhwc) res_l = (const __half*)d_residuals[i];
      else {
        // all four levels share RES sequentially: convert right before use
        res_l = h->RES;
      }
    }
    for (int j = 0; j < lpb; ++j) {
      const Layer& L = blk.layers[j];
      __half* out = h->skip[si];
      RUN(resnet(c, L.res, cur, curC, nullptr, 0, out));
      curC = L.res.cout;
      if (L.has_tr) RUN(transformer(c, L.tr, out));
      if (L.has_mo) RUN(motion(c, L.mo, i, out));
      if (i < 3 && j == lpb - 1 && res_l) {
        const size_t n = (size_t)c.NI * c.H * c.W * curC;
        if (!residuals_nhwc) RUN(nchw_to_nhwc(st, (const __half*)d_residuals[i], c.NI, curC, c.H, c.W, residual_scale, h->RES));
        RUN(add_inplace(st, out, res_l, n, residuals_nhwc ? residual_scale : 1.f));
      }
      RUN(tap(c, "down_blocks." + std::to_string(i) + "." + std::to_string(j), out, curC));
      cur = out;
      skips.push_back({cur, curC});
      ++si;
    }
    if (blk.has_sampler) {
      // Downsample3D: 3x3 stride-2 pad-1 conv (resnet.py:72-95) = stride-2 im2col + GEMM
      const int Ho = (c.H - 1) / 2 + 1, Wo = (c.W - 1) / 2 + 1;
      RUN(im2col_s2(st, cur, c.NI, c.H, c.W, curC, h->SCR));
      GemmArgs g;
      g.A = h->SCR; g.K1 = 9 * curC; g.lda1 = 9 * curC; g.Bw = blk.sampler.w; g.M = c.NI * Ho * Wo; g.N = blk.sampler.co;
      g.bias = blk.sampler.b; g.out = h->skip[si]; g.ldc = blk.sampler.co;
      RUN(gemm_tc(st, g));
      c.H = Ho; c.W = Wo;
      cur = h->skip[si];
      skips.push_back({cur, curC});
      ++si;
    }
    if (i == 3 && res_l) {
      // DownBlock3D: residual added to the running sample only, the skip stays untouched (unet.py:432-438)
      const size_t n = (size_t)c.NI * c.H * c.W * curC;
      if (!residuals_nhwc) RUN(nchw_to_nhwc(st, (const __half*)d_residuals[i], c.NI, curC, c.H, c.W, residual_scale, h->RES));
      VS_CHECK_CUDA(cudaMemcpyAsync(h->P0, cur, n * 2, cudaMemcpyDeviceToDevice, st));
      RUN(add_inplace(st, h->P0, res_l, n, residuals_nhwc ? residual_scale : 1.f));
      cur = h->P0;
    }
  }
  // ---- mid
  c.place = 1;
  {
    __half* o = (cur == h->P0) ? h->P1 : h->P0;
    RUN(resnet(c, h->mid0.res, cur, curC, nullptr, 0, o));
    RUN(transformer(c, h->mid0.tr, o));
    if (h->mid0.has_mo) RUN(motion(c, h->mid0.mo, 3, o));
    __half* o2 = (o == h->P0) ? h->P1 : h->P0;
    RUN(resnet(c, h->mid1, o, curC, nullptr, 0, o2));
    RUN(tap(c, "mid_block", o2, curC));
    cur = o2;
  }
  // ---- up path
  c.place = 2;
  for (int i = 0; i < 4; ++i) {
    const Block& blk = h->up[i];
    for (int j = 0; j <= lpb; ++j) {
      const Layer& L = blk.layers[j];
      const auto sk = skips.back();
      skips.pop_back();
      __half* o = (cur == h->P0) ? h->P1 : h->P0;
      RUN(resnet(c, L.res, cur, curC, sk.first, sk.second, o));
      curC = L.res.cout;
      if (L.has_tr) RUN(transformer(c, L.tr, o));
      if (L.has_mo) RUN(motion(c, L.mo, 3 - i, o));
      RUN(tap(c, "up_blocks." + std::to_string(i) + "." + std::to_string(j), o, curC));
      cur = o;
    }
    if (blk.has_sampler) {
      // Upsample3D: nearest [1,2,2] then 3x3 conv (resnet.py:54,67) = four 2x2 sub-pixel convs on the low-resolution input
      // (2.25x fewer FLOPs, the up-sampled tensor is never written); "subpixel" = 0 keeps the materialising path (A/B)
      __half* o = (cur == h->P0) ? h->P1 : h->P0;
      if (get_option("subpixel") != 0) {
        for (int par = 0; par < 4; ++par) {
          GemmArgs g;
          g.A = cur; g.K1 = curC; g.lda1 = curC; g.Bw = blk.sampler.wsub + (size_t)par * blk.sampler.co * 4 * curC; g.taps = 4;
          g.sub_py = par >> 1; g.sub_px = par & 1; g.nimg = c.NI; g.H = c.H; g.W = c.W; g.M = c.NI * c.H * c.W; g.N = blk.sampler.co;
          g.bias = blk.sampler.b; g.out = o; g.ldc = blk.sampler.co;
          RUN(gemm_tc(st, g));
        }
        c.H *= 2; c.W *= 2;
      } else {
        RUN(upsample_nearest2x(st, cur, c.NI, c.H, c.W, curC, h->SCR));
        c.H *= 2; c.W *= 2;
        RUN(conv(c, h->SCR, curC, blk.sampler, nullptr, nullptr, o));
      }
      cur = o;
    }
  }
  VS_REQUIRE(c.H == H && c.W == W, "input H/W (%d,%d) must be multiples of 8 (the reference's forward_upsample_size path is not implemented)", H, W);
  // ---- out: GroupNorm(5-D) + SiLU + conv_out
  NEXT_SUMS(osums);
  RUN(groupnorm_stats(st, cur, curC, nullptr, 0, c.NI, H * W, F, cf.norm_num_groups, osums, false));
  if (h->fnshards > 1) RUN(comm_all_reduce_sum_f32(h->fcomm, st, osums, (size_t)B * cf.norm_num_groups * 2));
  RUN(groupnorm_apply(st, cur, curC, nullptr, 0, c.NI, H * W, F, cf.norm_num_groups, osums, cf.norm_eps, h->norm_out.g, h->norm_out.b, true, h->XN,
                      h->fnshards));
  {
    GemmArgs g;
    g.A = h->XN; g.K1 = curC; g.lda1 = curC; g.Bw = h->conv_out.w; g.taps = 9; g.nimg = c.NI; g.H = H; g.W = W;
    g.M = c.NI * H * W; g.N = cf.out_channels; g.bias = h->conv_out.b; g.out = h->OUT; g.ldc = cf.out_channels;
    RUN(gemm_tc(st, g));
  }
  RUN(tap(c, "conv_out", h->OUT, cf.out_channels));
  RUN(nhwc_to_ncfhw(st, h->OUT, B, cf.out_channels, F, H, W, d_out, io_f32));
  return 0;
}
