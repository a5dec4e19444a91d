"""TEST INFRASTRUCTURE ONLY (never imported by videoswap_b200/): CPU fp32 restatement of the reference's
per-timestep denoising path, written functionally over a flat diffusers-style state_dict.

Follows (reference file:line, relative to the reference repository):
  * AnimateDiffUNet3DModel.forward            videoswap/models/animatediff_models/unet.py:328-481
  * block containers                          .../unet_blocks.py:258-265, 366-412, 480-508, 605-651, 715-740
  * ResnetBlock3D / Up/Downsample3D           .../resnet.py:163-193, 21-95   (5-D GroupNorm couples frames)
  * Transformer3DModel / BasicTransformerBlock .../attention.py:95-145, 221-256
  * VanillaTemporalModule + processor + PE    .../motion_module.py:138-162, 222-255, 278-340
  * EDLoRA cross-attention layer selection    videoswap/utils/edlora_util.py:18-82, 85-99
  * SparsePointAdapter + bilinear splat       videoswap/models/adapter_model.py:25-47, 97-136
  * CFG + DDIM loop body                      videoswap/pipelines/pipeline_videoswap.py:552-601
  * diffusers==0.19.3 (requirements.txt:2; NOT vendored): Attention, FeedForward/GEGLU (erf GELU),
    Timesteps/TimestepEmbedding, DDIMScheduler.step / set_timesteps, DDIMInverseScheduler.step
    -- restated from the published algorithm.

Pinning: the reference ships no tests/golden vectors (SURVEY.md section 4), so this oracle is pinned against the
reference's OWN model files executed from a checkout of the reference through oracle/diffusers_stub (see
oracle/make_golden.py -> tests/golden/*.pt).  The diffusers pieces themselves remain "parity unpinned"
(no diffusers install is available offline); DESIGN.md states this.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F


@dataclass
class OracleConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Sequence[int] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    heads: int = 8                      # `attention_head_dim` of SD-1.5 config == number of heads (unet.py:158)
    cross_attention_dim: int = 768
    norm_groups: int = 32
    norm_eps: float = 1e-5              # ResNet / conv_norm_out GroupNorm (unet.py:154,254)
    motion_heads: int = 8
    motion_resolutions: Sequence[int] = (1, 2, 4, 8)
    motion_mid_block: bool = False
    motion_decoder_only: bool = False
    use_motion_module: bool = True


Tensor = torch.Tensor
SD = Dict[str, Tensor]

# Attention controller hook (utils/p2p_utils/attention_register.py:15-97,140-150): when set, every spatial attention with
# fewer than 32^2 queries passes its probabilities [b, h, s, t] through ATTN_HOOK(probs, is_cross, place_in_unet) between
# the softmax and P V, exactly where the reference's control processors call `self.controller(...)`.
ATTN_HOOK = None
_PLACE = "down"

# False: softmax(q k^T) v spelled out (the arithmetic the oracle is pinned with).  True: F.scaled_dot_product_attention,
# used only when bench.py runs this same graph in fp16 on the GPU as the "library baseline" (cuDNN / cuBLASLt / SDPA).
USE_SDPA = False


# ----------------------------------------------------------------------------------------------------------------
# small ops
# ----------------------------------------------------------------------------------------------------------------
def _lin(sd: SD, p: str, x: Tensor) -> Tensor:
    return F.linear(x, sd[p + ".weight"], sd.get(p + ".bias"))


def _conv_per_frame(sd: SD, p: str, x: Tensor, stride: int = 1) -> Tensor:
    """InflatedConv3d: a 2-D conv applied to every frame independently (resnet.py:9-18)."""
    b, c, f, h, w = x.shape
    wgt = sd[p + ".weight"]
    y = F.conv2d(x.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w), wgt, sd.get(p + ".bias"), stride=stride,
                 padding=wgt.shape[-1] // 2)
    return y.reshape(b, f, y.shape[1], y.shape[2], y.shape[3]).permute(0, 2, 1, 3, 4)


def _gn5d(sd: SD, p: str, x: Tensor, groups: int, eps: float) -> Tensor:
    """GroupNorm on the 5-D tensor: statistics over (C/groups, F, H, W) -- frames are coupled (resnet.py:166,177)."""
    return F.group_norm(x, groups, sd[p + ".weight"], sd[p + ".bias"], eps)


def _gn_frame(sd: SD, p: str, x_bf: Tensor, groups: int, eps: float) -> Tensor:
    """GroupNorm on (b f) c h w: per-frame statistics (attention.py:108, motion_module.py:146)."""
    return F.group_norm(x_bf, groups, sd[p + ".weight"], sd[p + ".bias"], eps)


def _ln(sd: SD, p: str, x: Tensor) -> Tensor:
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], 1e-5)


def _mha(q: Tensor, k: Tensor, v: Tensor, heads: int) -> Tensor:
    """softmax(q k^T / sqrt(d)) v with heads split from the channel dim (diffusers Attention, P2)."""
    b, nq, c = q.shape
    d = c // heads
    qh = q.reshape(b, nq, heads, d).transpose(1, 2)
    kh = k.reshape(b, k.shape[1], heads, d).transpose(1, 2)
    vh = v.reshape(b, v.shape[1], heads, d).transpose(1, 2)
    if USE_SDPA:
        return F.scaled_dot_product_attention(qh, kh, vh).transpose(1, 2).reshape(b, nq, c)
    if b * heads * nq * kh.shape[2] > (1 << 30):      # bound the score matrix (N = 4096, 16+ frames): batch chunks
        o = torch.cat([torch.matmul((torch.matmul(qh[i:i + 2], kh[i:i + 2].transpose(-1, -2)) * (d ** -0.5)).softmax(dim=-1),
                                    vh[i:i + 2]) for i in range(0, b, 2)])
        return o.transpose(1, 2).reshape(b, nq, c)
    s = torch.matmul(qh, kh.transpose(-1, -2)) * (d ** -0.5)
    o = torch.matmul(s.softmax(dim=-1), vh)
    return o.transpose(1, 2).reshape(b, nq, c)


def _attn(sd: SD, p: str, x: Tensor, ctx: Tensor, heads: int, is_cross: Optional[bool] = None) -> Tensor:
    q = _lin(sd, p + ".to_q", x)
    k = _lin(sd, p + ".to_k", ctx)
    v = _lin(sd, p + ".to_v", ctx)
    if ATTN_HOOK is not None and is_cross is not None and q.shape[1] < 32 ** 2:
        b, nq, c = q.shape
        d = c // heads
        qh = q.reshape(b, nq, heads, d).transpose(1, 2)
        kh = k.reshape(b, k.shape[1], heads, d).transpose(1, 2)
        vh = v.reshape(b, v.shape[1], heads, d).transpose(1, 2)
        probs = (torch.matmul(qh, kh.transpose(-1, -2)) * (d ** -0.5)).softmax(dim=-1)       # get_attention_scores
        probs = ATTN_HOOK(probs, is_cross, _PLACE)
        o = torch.matmul(probs, vh).transpose(1, 2).reshape(b, nq, c)
        return _lin(sd, p + ".to_out.0", o)
    return _lin(sd, p + ".to_out.0", _mha(q, k, v, heads))


def _geglu_ff(sd: SD, p: str, x: Tensor) -> Tensor:
    """FeedForward = Linear(C, 8C) -> value * gelu_erf(gate) -> Linear(4C, C); first half value, second gate (P3)."""
    h, g = _lin(sd, p + ".net.0.proj", x).chunk(2, dim=-1)
    return _lin(sd, p + ".net.2", h * F.gelu(g))


def timestep_embedding(t: Tensor, dim: int) -> Tensor:
    """Timesteps(dim, flip_sin_to_cos=True, freq_shift=0): cat(cos, sin) of t * exp(-ln(1e4) i / half) (P1)."""
    half = dim // 2
    freq = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    arg = t.float()[:, None] * freq[None, :]
    return torch.cat([torch.cos(arg), torch.sin(arg)], dim=-1)


def temporal_pe(length: int, dim: int) -> Tensor:
    """PositionalEncoding table (motion_module.py:242-251); closed form, so any length is well defined."""
    pos = torch.arange(length, dtype=torch.float32)[:, None]
    div = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * (-math.log(10000.0) / dim))
    pe = torch.zeros(length, dim)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


# ----------------------------------------------------------------------------------------------------------------
# modules
# ----------------------------------------------------------------------------------------------------------------
def resnet_block(sd: SD, p: str, x: Tensor, temb: Tensor, cfg: OracleConfig) -> Tensor:
    h = F.silu(_gn5d(sd, p + ".norm1", x, cfg.norm_groups, cfg.norm_eps))
    h = _conv_per_frame(sd, p + ".conv1", h)
    h = h + _lin(sd, p + ".time_emb_proj", F.silu(temb))[:, :, None, None, None]
    h = F.silu(_gn5d(sd, p + ".norm2", h, cfg.norm_groups, cfg.norm_eps))
    h = _conv_per_frame(sd, p + ".conv2", h)
    if (p + ".conv_shortcut.weight") in sd:
        x = _conv_per_frame(sd, p + ".conv_shortcut", x)
    return x + h


def transformer3d(sd: SD, p: str, x: Tensor, ehs: Tensor, layer_idx: int, cfg: OracleConfig) -> Tensor:
    """Spatial transformer on every frame; `ehs` is [B,77,D] or ED-LoRA [B,L,77,D] (layer picked by layer_idx)."""
    b, c, f, h, w = x.shape
    xb = x.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
    ctx = ehs[:, layer_idx] if ehs.dim() == 4 else ehs
    ctx = ctx[:, None].expand(b, f, *ctx.shape[1:]).reshape(b * f, ctx.shape[1], ctx.shape[2])
    t = _gn_frame(sd, p + ".norm", xb, cfg.norm_groups, 1e-6)
    t = F.conv2d(t, sd[p + ".proj_in.weight"], sd[p + ".proj_in.bias"])
    t = t.permute(0, 2, 3, 1).reshape(b * f, h * w, c)
    q = p + ".transformer_blocks.0"
    n1 = _ln(sd, q + ".norm1", t)
    t = t + _attn(sd, q + ".attn1", n1, n1, cfg.heads, is_cross=False)
    t = t + _attn(sd, q + ".attn2", _ln(sd, q + ".norm2", t), ctx, cfg.heads, is_cross=True)
    t = t + _geglu_ff(sd, q + ".ff", _ln(sd, q + ".norm3", t))
    t = t.reshape(b * f, h, w, c).permute(0, 3, 1, 2)
    t = F.conv2d(t, sd[p + ".proj_out.weight"], sd[p + ".proj_out.bias"])
    out = t + xb
    return out.reshape(b, f, c, h, w).permute(0, 2, 1, 3, 4)


def motion_module(sd: SD, p: str, x: Tensor, cfg: OracleConfig) -> Tensor:
    """AnimateDiff VanillaTemporalModule: attention across the F frames of every pixel (motion_module.py)."""
    p = p + ".temporal_transformer"
    b, c, f, h, w = x.shape
    xb = x.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
    t = _gn_frame(sd, p + ".norm", xb, 32, 1e-6)     # norm_num_groups is fixed at 32 (motion_module.py:97)
    t = t.permute(0, 2, 3, 1).reshape(b * f, h * w, c)
    t = _lin(sd, p + ".proj_in", t)
    q = p + ".transformer_blocks.0"
    pe = temporal_pe(f, c).to(x)
    for i in (0, 1):
        n = _ln(sd, f"{q}.norms.{i}", t)
        # '(b f) d c -> (b d) f c', add PE after the LayerNorm, to the tensor that feeds q, k and v (P5)
        n = n.reshape(b, f, h * w, c).permute(0, 2, 1, 3).reshape(b * h * w, f, c) + pe[None]
        a = _attn(sd, f"{q}.attention_blocks.{i}", n, n, cfg.motion_heads)
        a = a.reshape(b, h * w, f, c).permute(0, 2, 1, 3).reshape(b * f, h * w, c)
        t = t + a
    t = t + _geglu_ff(sd, q + ".ff", _ln(sd, q + ".ff_norm", t))
    t = _lin(sd, p + ".proj_out", t)
    t = t.reshape(b * f, h, w, c).permute(0, 3, 1, 2)
    out = t + xb
    return out.reshape(b, f, c, h, w).permute(0, 2, 1, 3, 4)


def _has_motion(sd: SD, p: str) -> bool:
    return (p + ".temporal_transformer.proj_in.weight") in sd


def _add_residual(x: Tensor, r: Tensor) -> Tensor:
    """'(b f) c h w -> b c f h w' then add (unet_blocks.py:399-402, unet.py:434-438)."""
    b = x.shape[0]
    return x + r.reshape(b, -1, *r.shape[1:]).permute(0, 2, 1, 3, 4)


def unet_forward(sd: SD, cfg: OracleConfig, sample: Tensor, timestep, ehs: Tensor,
                 residuals: Optional[List[Tensor]] = None, taps: Optional[Dict[str, Tensor]] = None) -> Tensor:
    """sample [B,C,F,H,W] fp32, timestep scalar/[B], ehs [B,77,D] or [B,L,77,D]; residuals: 4 x [(B F),C_l,H_l,W_l].
    `taps` (optional dict) receives intermediate activations keyed by module prefix."""
    def tap(name, t):
        if taps is not None:
            taps[name] = t.detach().clone()

    B = sample.shape[0]
    t = torch.as_tensor(timestep).reshape(-1).expand(B)
    boc = list(cfg.block_out_channels)
    temb = timestep_embedding(t, boc[0]).to(sample)          # fp32 sinusoid, cast to the model dtype (unet.py:396)
    temb = _lin(sd, "time_embedding.linear_2", F.silu(_lin(sd, "time_embedding.linear_1", temb)))
    tap("temb", temb)
    residuals = list(residuals) if residuals is not None else None

    x = _conv_per_frame(sd, "conv_in", sample)
    tap("conv_in", x)
    skips = [x]
    attn_idx = 0
    nlev = len(boc)
    global _PLACE
    _PLACE = "down"
    # down path
    for i in range(nlev):
        cross = i < nlev - 1            # CrossAttn x3 then DownBlock3D (unet.py:47-52)
        res = residuals.pop(0) if residuals else None
        for j in range(cfg.layers_per_block):
            p = f"down_blocks.{i}"
            x = resnet_block(sd, f"{p}.resnets.{j}", x, temb, cfg)
            if cross:
                x = transformer3d(sd, f"{p}.attentions.{j}", x, ehs, attn_idx, cfg)
                attn_idx += 1
            if _has_motion(sd, f"{p}.motion_modules.{j}"):
                x = motion_module(sd, f"{p}.motion_modules.{j}", x, cfg)
            if cross and j == cfg.layers_per_block - 1 and res is not None:
                x = _add_residual(x, res)          # before skip append and before the down-sampler (P6)
            tap(f"{p}.{j}", x)
            skips.append(x)
        if i < nlev - 1:
            x = _conv_per_frame(sd, f"down_blocks.{i}.downsamplers.0.conv", x, stride=2)
            skips.append(x)
        if not cross and res is not None:
            x = _add_residual(x, res)              # after the block; skips unaffected (P6)
    # mid
    _PLACE = "mid"
    x = resnet_block(sd, "mid_block.resnets.0", x, temb, cfg)
    x = transformer3d(sd, "mid_block.attentions.0", x, ehs, attn_idx, cfg)
    attn_idx += 1
    if _has_motion(sd, "mid_block.motion_modules.0"):
        x = motion_module(sd, "mid_block.motion_modules.0", x, cfg)
    x = resnet_block(sd, "mid_block.resnets.1", x, temb, cfg)
    tap("mid_block", x)
    # up path
    _PLACE = "up"
    for i in range(nlev):
        cross = i > 0                   # UpBlock3D then CrossAttnUp x3
        p = f"up_blocks.{i}"
        for j in range(cfg.layers_per_block + 1):
            x = torch.cat([x, skips.pop()], dim=1)
            x = resnet_block(sd, f"{p}.resnets.{j}", x, temb, cfg)
            if cross:
                x = transformer3d(sd, f"{p}.attentions.{j}", x, ehs, attn_idx, cfg)
                attn_idx += 1
            if _has_motion(sd, f"{p}.motion_modules.{j}"):
                x = motion_module(sd, f"{p}.motion_modules.{j}", x, cfg)
            tap(f"{p}.{j}", x)
        if i < nlev - 1:
            x = F.interpolate(x, scale_factor=(1.0, 2.0, 2.0), mode="nearest")
            x = _conv_per_frame(sd, f"{p}.upsamplers.0.conv", x)
    x = F.silu(_gn5d(sd, "conv_norm_out", x, cfg.norm_groups, cfg.norm_eps))
    x = _conv_per_frame(sd, "conv_out", x)
    tap("conv_out", x)
    return x


# ----------------------------------------------------------------------------------------------------------------
# adapter (adapter_model.py) -- coordinates are cast to the latents dtype by the pipeline (P7)
# ----------------------------------------------------------------------------------------------------------------
def adapter_forward(sd: SD, pred_tracks: Tensor, size, point_embedding: Tensor, channels=(320, 640, 1280, 1280),
                    downsample_rate=(8, 16, 32, 64), index_list=None) -> List[Tensor]:
    """pred_tracks [F,P,2] (x,y; <0 = invisible), size=(w,h), point_embedding [P,E] -> 4 x [F,C_l,h_l,w_l].
    Arithmetic is done in pred_tracks.dtype for the coordinates and point_embedding.dtype for the maps."""
    w, h = size
    nf, npts = pred_tracks.shape[:2]
    pts = [i for i in range(npts) if index_list is None or i in index_list]
    out = []
    for lv, (ch, rate) in enumerate(zip(channels, downsample_rate)):
        feat = _lin(sd, f"model_list.{lv}.mlp.2", F.silu(_lin(sd, f"model_list.{lv}.mlp.0", point_embedding)))
        lw, lh = w // rate, h // rate
        m = torch.zeros(nf, ch, lh, lw, dtype=feat.dtype)
        for pi in pts:
            for fi in range(nf):
                px, py = pred_tracks[fi, pi]
                if px < 0 or py < 0:
                    continue
                x, y = px / rate, py / rate
                x1, y1 = int(x), int(y)
                fx, fy = x - x1, y - y1
                x2, y2 = x1 + 1, y1 + 1
                x1, x2 = max(min(x1, lw - 1), 0), max(min(x2, lw - 1), 0)
                y1, y2 = max(min(y1, lh - 1), 0), max(min(y2, lh - 1), 0)
                m[fi, :, y1, x1] += feat[pi] * ((1 - fx) * (1 - fy))
                m[fi, :, y1, x2] += feat[pi] * (fx * (1 - fy))
                m[fi, :, y2, x1] += feat[pi] * ((1 - fx) * fy)
                m[fi, :, y2, x2] += feat[pi] * (fx * fy)
        out.append(m)
    return out


# ----------------------------------------------------------------------------------------------------------------
# DDIM scheduler (diffusers 0.19.3 DDIMScheduler / DDIMInverseScheduler, eta = 0) and the loop body
# ----------------------------------------------------------------------------------------------------------------
@dataclass
class DDIM:
    num_train_timesteps: int = 1000
    beta_start: float = 0.00085
    beta_end: float = 0.012
    steps_offset: int = 1
    alphas_cumprod: Tensor = field(init=False)

    def __post_init__(self):
        betas = torch.linspace(self.beta_start ** 0.5, self.beta_end ** 0.5, self.num_train_timesteps,
                               dtype=torch.float32) ** 2          # "scaled_linear"
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = self.alphas_cumprod[0]         # set_alpha_to_one=False

    def timesteps(self, n: int) -> List[int]:
        """'leading' spacing: (arange(n) * (T // n))[::-1] + steps_offset  (P10)."""
        ratio = self.num_train_timesteps // n
        return [int(i * ratio + self.steps_offset) for i in range(n)][::-1]

    def step(self, eps: Tensor, t: int, x: Tensor, n: int) -> Tensor:
        prev = t - self.num_train_timesteps // n
        a_t = self.alphas_cumprod[t]
        a_p = self.alphas_cumprod[prev] if prev >= 0 else self.final_alpha_cumprod
        x0 = (x - (1 - a_t) ** 0.5 * eps) / a_t ** 0.5
        return a_p ** 0.5 * x0 + (1 - a_p) ** 0.5 * eps

    def inverse_timesteps(self, n: int) -> List[int]:
        """DDIMInverseScheduler.set_timesteps: arange(n) * ratio + steps_offset, ascending (both conventions)."""
        return self.timesteps(n)[::-1]

    def inverse_step(self, eps: Tensor, t: int, x: Tensor, n: int, convention: str = "0.19.3") -> Tensor:
        """DDIMInverseScheduler.step, x_t -> x_{t+ratio} (unpinned: no diffusers offline, see header).
        "0.19.3" (the release the reference pins): prev_timestep = t + ratio; x0 from alpha[t]; target alpha[t + ratio],
        beyond the table alphas_cumprod[-1] (set_alpha_to_zero False via the SD config's set_alpha_to_one False).
        "0.21": the sample sits at t - ratio and moves to t."""
        ratio = self.num_train_timesteps // n
        if convention == "0.19.3":
            a_cur = self.alphas_cumprod[t]
            a_nxt = self.alphas_cumprod[t + ratio] if t + ratio < self.num_train_timesteps else self.alphas_cumprod[-1]
        else:
            prev = t - ratio
            a_nxt = self.alphas_cumprod[t]
            a_cur = self.alphas_cumprod[prev] if prev >= 0 else self.final_alpha_cumprod
        x0 = (x - (1 - a_cur) ** 0.5 * eps) / a_cur ** 0.5
        return a_nxt ** 0.5 * x0 + (1 - a_nxt) ** 0.5 * eps


def cfg_combine(eps2: Tensor, guidance: float) -> Tensor:
    """noise_pred_uncond + s (noise_pred_text - noise_pred_uncond); uncond is the FIRST half (pipeline:578-580)."""
    u, c = eps2.chunk(2)
    return u + guidance * (c - u)


def denoise_step(sd: SD, cfg: OracleConfig, sched: DDIM, latents: Tensor, t: int, n_steps: int, ehs2: Tensor,
                 guidance: float, residuals: Optional[List[Tensor]] = None) -> Tensor:
    """One iteration of pipeline_videoswap.py:555-587 with CFG: latents [1,4,F,H,W] -> latents."""
    x2 = torch.cat([latents] * 2)
    res2 = [torch.cat([r] * 2, dim=0) for r in residuals] if residuals is not None else None
    eps2 = unet_forward(sd, cfg, x2, t, ehs2, res2)
    return sched.step(cfg_combine(eps2, guidance), t, latents, n_steps)


def denoise_loop(sd: SD, cfg: OracleConfig, latents: Tensor, pos: Tensor, neg: Tensor, n_steps: int, guidance: float,
                 adapter_state: Optional[List[Tensor]] = None, t2i_start: float = 0.0, t2i_end: float = 1.0,
                 max_iters: Optional[int] = None) -> Tensor:
    """pipeline_videoswap.py:552-610: the loop with the adapter window (`i <= len * t2i_end and i >= len * t2i_start`,
    :561) and the final 'b c f h w -> (b f) c h w' (:603).  adapter_state: 4 x [(F),C,h,w] already scaled by
    t2i_guidance_scale (:544-545); `max_iters` truncates the loop (tests run a few iterations of the 50-step schedule)."""
    sched = DDIM()
    ts = sched.timesteps(n_steps)
    ehs2 = torch.cat([neg, pos]) if guidance > 1.0 else pos
    for i, t in enumerate(ts):
        if max_iters is not None and i >= max_iters:
            break
        res = adapter_state if (adapter_state is not None and len(ts) * t2i_start <= i <= len(ts) * t2i_end) else None
        if guidance > 1.0:
            latents = denoise_step(sd, cfg, sched, latents, t, n_steps, ehs2, guidance, res)
        else:
            latents = sched.step(unet_forward(sd, cfg, latents, t, ehs2, res), t, latents, n_steps)
    b, c, f, h, w = latents.shape
    return latents.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)


def invert_loop(sd: SD, cfg: OracleConfig, latents: Tensor, ehs: Tensor, n_steps: int, convention: str = "0.19.3",
                max_iters: Optional[int] = None) -> Tensor:
    """pipeline_videoswap.py:677-703 with guidance_scale = 1: UNet at the scheduler's timestep, inverse DDIM step."""
    sched = DDIM()
    for i, t in enumerate(sched.inverse_timesteps(n_steps)):
        if max_iters is not None and i >= max_iters:
            break
        latents = sched.inverse_step(unet_forward(sd, cfg, latents, t, ehs), t, latents, n_steps, convention)
    return latents
