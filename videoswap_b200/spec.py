"""Architecture spec of the reference's AnimateDiffUNet3DModel (SD-1.5 UNet + AnimateDiff motion modules):
parameter names/shapes exactly as the reference's `state_dict()` produces them
(videoswap/models/animatediff_models/unet.py:32-255 and unet_blocks.py of the reference), so that
`load_state_dict` / ED-LoRA weight merging (utils/convert_edlora_to_diffusers.py:36-79) keep working.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass, field, asdict
from typing import Dict, List, Sequence, Tuple


@dataclass
class UNetConfig:
    sample_size: int = 64
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    attention_head_dim: int = 8            # == number of heads (reference quirk, unet.py:158)
    cross_attention_dim: int = 768
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    # AnimateDiff additions (options/model_cfg/inference.yml of the reference)
    use_motion_module: bool = True
    motion_module_resolutions: Tuple[int, ...] = (1, 2, 4, 8)
    motion_module_mid_block: bool = False
    motion_module_decoder_only: bool = False
    motion_num_attention_heads: int = 8
    temporal_position_encoding_max_len: int = 24

    def to_dict(self):
        return asdict(self)

    @property
    def time_embed_dim(self) -> int:
        return self.block_out_channels[0] * 4

    def down_has_motion(self, i: int) -> bool:
        return self.use_motion_module and (2 ** i in self.motion_module_resolutions) and not self.motion_module_decoder_only

    def up_has_motion(self, i: int) -> bool:
        return self.use_motion_module and (2 ** (3 - i) in self.motion_module_resolutions)

    def up_resnet_in_channels(self, i: int, j: int) -> Tuple[int, int]:
        """(channels of the running tensor, channels of the popped skip) for up_blocks.i.resnets.j
        (unet_blocks.py:551-556 of the reference)."""
        boc = list(self.block_out_channels)
        rev = boc[::-1]
        n = len(boc)
        out_c = rev[i]
        prev = rev[max(i - 1, 0)] if i > 0 else rev[0]
        in_c = rev[min(i + 1, n - 1)]
        nl = self.layers_per_block + 1
        skip = in_c if j == nl - 1 else out_c
        run = prev if j == 0 else out_c
        return run, skip


def _resnet(sh, p, cin, cout, temb):
    sh[p + ".norm1.weight"] = (cin,)
    sh[p + ".norm1.bias"] = (cin,)
    sh[p + ".conv1.weight"] = (cout, cin, 3, 3)
    sh[p + ".conv1.bias"] = (cout,)
    sh[p + ".time_emb_proj.weight"] = (cout, temb)
    sh[p + ".time_emb_proj.bias"] = (cout,)
    sh[p + ".norm2.weight"] = (cout,)
    sh[p + ".norm2.bias"] = (cout,)
    sh[p + ".conv2.weight"] = (cout, cout, 3, 3)
    sh[p + ".conv2.bias"] = (cout,)
    if cin != cout:
        sh[p + ".conv_shortcut.weight"] = (cout, cin, 1, 1)
        sh[p + ".conv_shortcut.bias"] = (cout,)


def _attn(sh, p, c, ctx):
    sh[p + ".to_q.weight"] = (c, c)
    sh[p + ".to_k.weight"] = (c, ctx)
    sh[p + ".to_v.weight"] = (c, ctx)
    sh[p + ".to_out.0.weight"] = (c, c)
    sh[p + ".to_out.0.bias"] = (c,)


def _ff(sh, p, c):
    sh[p + ".net.0.proj.weight"] = (8 * c, c)
    sh[p + ".net.0.proj.bias"] = (8 * c,)
    sh[p + ".net.2.weight"] = (c, 4 * c)
    sh[p + ".net.2.bias"] = (c,)


def _norm(sh, p, c):
    sh[p + ".weight"] = (c,)
    sh[p + ".bias"] = (c,)


def _transformer(sh, p, c, ctx):
    _norm(sh, p + ".norm", c)
    sh[p + ".proj_in.weight"] = (c, c, 1, 1)
    sh[p + ".proj_in.bias"] = (c,)
    q = p + ".transformer_blocks.0"
    _attn(sh, q + ".attn1", c, c)
    _norm(sh, q + ".norm1", c)
    _attn(sh, q + ".attn2", c, ctx)
    _norm(sh, q + ".norm2", c)
    _ff(sh, q + ".ff", c)
    _norm(sh, q + ".norm3", c)
    sh[p + ".proj_out.weight"] = (c, c, 1, 1)
    sh[p + ".proj_out.bias"] = (c,)


def _motion(sh, p, c, pe_len):
    p = p + ".temporal_transformer"
    _norm(sh, p + ".norm", c)
    sh[p + ".proj_in.weight"] = (c, c)
    sh[p + ".proj_in.bias"] = (c,)
    q = p + ".transformer_blocks.0"
    for i in (0, 1):
        a = f"{q}.attention_blocks.{i}"
        _attn(sh, a, c, c)
        sh[a + ".processor.pos_encoder.pe"] = (1, pe_len, c)     # buffer (test.py:63 key remap targets this name)
    for i in (0, 1):
        _norm(sh, f"{q}.norms.{i}", c)
    _ff(sh, q + ".ff", c)
    _norm(sh, q + ".ff_norm", c)
    sh[p + ".proj_out.weight"] = (c, c)
    sh[p + ".proj_out.bias"] = (c,)


def unet_param_shapes(cfg: UNetConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    sh: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    boc = list(cfg.block_out_channels)
    n = len(boc)
    temb = cfg.time_embed_dim
    ctx = cfg.cross_attention_dim
    pe = cfg.temporal_position_encoding_max_len
    sh["conv_in.weight"] = (boc[0], cfg.in_channels, 3, 3)
    sh["conv_in.bias"] = (boc[0],)
    sh["time_embedding.linear_1.weight"] = (temb, boc[0])
    sh["time_embedding.linear_1.bias"] = (temb,)
    sh["time_embedding.linear_2.weight"] = (temb, temb)
    sh["time_embedding.linear_2.bias"] = (temb,)
    cout = boc[0]
    for i in range(n):
        cin, cout = cout, boc[i]
        p = f"down_blocks.{i}"
        cross = i < n - 1
        for j in range(cfg.layers_per_block):
            if cross:
                _transformer(sh, f"{p}.attentions.{j}", cout, ctx)
        for j in range(cfg.layers_per_block):
            _resnet(sh, f"{p}.resnets.{j}", cin if j == 0 else cout, cout, temb)
        for j in range(cfg.layers_per_block):
            if cfg.down_has_motion(i):
                _motion(sh, f"{p}.motion_modules.{j}", cout, pe)
        if i < n - 1:
            sh[f"{p}.downsamplers.0.conv.weight"] = (cout, cout, 3, 3)
            sh[f"{p}.downsamplers.0.conv.bias"] = (cout,)
    c = boc[-1]
    _transformer(sh, "mid_block.attentions.0", c, ctx)
    _resnet(sh, "mid_block.resnets.0", c, c, temb)
    _resnet(sh, "mid_block.resnets.1", c, c, temb)
    if cfg.use_motion_module and cfg.motion_module_mid_block:
        _motion(sh, "mid_block.motion_modules.0", c, pe)
    rev = boc[::-1]
    for i in range(n):
        p = f"up_blocks.{i}"
        cross = i > 0
        out_c = rev[i]
        for j in range(cfg.layers_per_block + 1):
            if cross:
                _transformer(sh, f"{p}.attentions.{j}", out_c, ctx)
        for j in range(cfg.layers_per_block + 1):
            run, skip = cfg.up_resnet_in_channels(i, j)
            _resnet(sh, f"{p}.resnets.{j}", run + skip, out_c, temb)
        for j in range(cfg.layers_per_block + 1):
            if cfg.up_has_motion(i):
                _motion(sh, f"{p}.motion_modules.{j}", out_c, pe)
        if i < n - 1:
            sh[f"{p}.upsamplers.0.conv.weight"] = (out_c, out_c, 3, 3)
            sh[f"{p}.upsamplers.0.conv.bias"] = (out_c,)
    _norm(sh, "conv_norm_out", boc[0])
    sh["conv_out.weight"] = (cfg.out_channels, boc[0], 3, 3)
    sh["conv_out.bias"] = (cfg.out_channels,)
    return sh


@dataclass
class VAEConfig:
    """The decoder side of diffusers 0.19.3 AutoencoderKL as SD-1.5 configures it (vae/config.json)."""
    in_channels: int = 3
    out_channels: int = 3
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    latent_channels: int = 4
    norm_num_groups: int = 32
    scaling_factor: float = 0.18215
    sample_size: int = 512

    def to_dict(self):
        return asdict(self)


def _vae_resnet(sh, p, cin, cout):
    """ResnetBlock2D with temb_channels=None (no time_emb_proj)."""
    for n, c in (("norm1", cin), ("norm2", cout)):
        _norm(sh, f"{p}.{n}", c)
    sh[p + ".conv1.weight"] = (cout, cin, 3, 3)
    sh[p + ".conv1.bias"] = (cout,)
    sh[p + ".conv2.weight"] = (cout, cout, 3, 3)
    sh[p + ".conv2.bias"] = (cout,)
    if cin != cout:
        sh[p + ".conv_shortcut.weight"] = (cout, cin, 1, 1)
        sh[p + ".conv_shortcut.bias"] = (cout,)


def vae_param_shapes(cfg: VAEConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    """Decoder-side AutoencoderKL state_dict (diffusers 0.19.3 names: the mid-block attention as to_q / to_k / to_v /
    to_out.0).  The encoder and quant_conv are not part of it."""
    sh: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    lc, boc = cfg.latent_channels, list(cfg.block_out_channels)
    sh["post_quant_conv.weight"] = (lc, lc, 1, 1)
    sh["post_quant_conv.bias"] = (lc,)
    c = boc[-1]
    sh["decoder.conv_in.weight"] = (c, lc, 3, 3)
    sh["decoder.conv_in.bias"] = (c,)
    _vae_resnet(sh, "decoder.mid_block.resnets.0", c, c)
    a = "decoder.mid_block.attentions.0"
    _norm(sh, a + ".group_norm", c)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        sh[f"{a}.{n}.weight"] = (c, c)
        sh[f"{a}.{n}.bias"] = (c,)
    _vae_resnet(sh, "decoder.mid_block.resnets.1", c, c)
    rev = boc[::-1]
    prev = rev[0]
    for i, out in enumerate(rev):
        for j in range(cfg.layers_per_block + 1):
            _vae_resnet(sh, f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else out, out)
        if i < len(rev) - 1:
            sh[f"decoder.up_blocks.{i}.upsamplers.0.conv.weight"] = (out, out, 3, 3)
            sh[f"decoder.up_blocks.{i}.upsamplers.0.conv.bias"] = (out,)
        prev = out
    _norm(sh, "decoder.conv_norm_out", boc[0])
    sh["decoder.conv_out.weight"] = (cfg.out_channels, boc[0], 3, 3)
    sh["decoder.conv_out.bias"] = (cfg.out_channels,)
    return sh


def vae_encoder_param_shapes(cfg: VAEConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    """Encoder-side AutoencoderKL state_dict (diffusers 0.19.3 names): Encoder (conv_in, DownEncoderBlock2D x 4 of
    layers_per_block resnets with a stride-2 Downsample2D on all but the last, UNetMidBlock2D, conv_norm_out, conv_out to
    2 x latent_channels with double_z) and quant_conv."""
    sh: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    lc, boc = cfg.latent_channels, list(cfg.block_out_channels)
    sh["encoder.conv_in.weight"] = (boc[0], cfg.in_channels, 3, 3)
    sh["encoder.conv_in.bias"] = (boc[0],)
    prev = boc[0]
    for i, out in enumerate(boc):
        for j in range(cfg.layers_per_block):
            _vae_resnet(sh, f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else out, out)
        if i < len(boc) - 1:
            sh[f"encoder.down_blocks.{i}.downsamplers.0.conv.weight"] = (out, out, 3, 3)
            sh[f"encoder.down_blocks.{i}.downsamplers.0.conv.bias"] = (out,)
        prev = out
    c = boc[-1]
    _vae_resnet(sh, "encoder.mid_block.resnets.0", c, c)
    a = "encoder.mid_block.attentions.0"
    _norm(sh, a + ".group_norm", c)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        sh[f"{a}.{n}.weight"] = (c, c)
        sh[f"{a}.{n}.bias"] = (c,)
    _vae_resnet(sh, "encoder.mid_block.resnets.1", c, c)
    _norm(sh, "encoder.conv_norm_out", c)
    sh["encoder.conv_out.weight"] = (2 * lc, c, 3, 3)
    sh["encoder.conv_out.bias"] = (2 * lc,)
    sh["quant_conv.weight"] = (2 * lc, 2 * lc, 1, 1)
    sh["quant_conv.bias"] = (2 * lc,)
    return sh


def adapter_param_shapes(embedding_channels=1280, channels=(320, 640, 1280, 1280), mid_dim=128):
    """SparsePointAdapter state_dict (videoswap/models/adapter_model.py:50-70 of the reference)."""
    sh = OrderedDict()
    for l, ch in enumerate(channels):
        sh[f"model_list.{l}.mlp.0.weight"] = (mid_dim, embedding_channels)
        sh[f"model_list.{l}.mlp.0.bias"] = (mid_dim,)
        sh[f"model_list.{l}.mlp.2.weight"] = (ch, mid_dim)
        sh[f"model_list.{l}.mlp.2.bias"] = (ch,)
    return sh


@dataclass
class CLIPTextConfig:
    """The fields of SD-1.5's text_encoder/config.json (transformers CLIPTextConfig) that shape the model."""
    vocab_size: int = 49408
    hidden_size: int = 768
    intermediate_size: int = 3072
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    max_position_embeddings: int = 77
    hidden_act: str = "quick_gelu"
    layer_norm_eps: float = 1e-5

    def to_dict(self):
        return asdict(self)


def clip_text_param_shapes(cfg: CLIPTextConfig = CLIPTextConfig()) -> "OrderedDict[str, Tuple[int, ...]]":
    """CLIPTextModel.state_dict() keys and shapes (transformers modeling_clip.py) without the `position_ids` buffer that
    older checkpoints carry: 196 tensors and 123,060,480 parameters for SD-1.5."""
    C, F = cfg.hidden_size, cfg.intermediate_size
    sh: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    sh["text_model.embeddings.token_embedding.weight"] = (cfg.vocab_size, C)
    sh["text_model.embeddings.position_embedding.weight"] = (cfg.max_position_embeddings, C)
    for i in range(cfg.num_hidden_layers):
        p = f"text_model.encoder.layers.{i}"
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            sh[f"{p}.self_attn.{n}.weight"] = (C, C)
            sh[f"{p}.self_attn.{n}.bias"] = (C,)
        sh[f"{p}.layer_norm1.weight"] = (C,)
        sh[f"{p}.layer_norm1.bias"] = (C,)
        sh[f"{p}.mlp.fc1.weight"] = (F, C)
        sh[f"{p}.mlp.fc1.bias"] = (F,)
        sh[f"{p}.mlp.fc2.weight"] = (C, F)
        sh[f"{p}.mlp.fc2.bias"] = (C,)
        sh[f"{p}.layer_norm2.weight"] = (C,)
        sh[f"{p}.layer_norm2.bias"] = (C,)
    sh["text_model.final_layer_norm.weight"] = (C,)
    sh["text_model.final_layer_norm.bias"] = (C,)
    return sh
