"""Functional restatement of diffusers 0.19.3 `AutoencoderKL._decode` and `VaeImageProcessor.postprocess` for the SD-1.5 VAE
(the checker of videoswap_b200/vae.py).  Unpinned: the reference checkout has no VAE code of its own (it imports
diffusers' AutoencoderKL, pipeline_videoswap.py:95) and diffusers is not a dependency here, so each function says which
diffusers 0.19.3 code it restates instead of being compared with it.

Device- and dtype-agnostic torch: the tests run it on the CPU in fp32; tools/gpu_vae_decode.py runs the same functions on
CUDA in fp16 (cuDNN convolutions, scaled_dot_product_attention) as the stock-PyTorch baseline."""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

EPS = 1e-6        # resnet_eps = 1e-6 in Decoder / UNetMidBlock2D / UpDecoderBlock2D (models/vae.py, unet_2d_blocks.py)
GROUPS = 32       # norm_num_groups


def param_shapes(block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=4, out_channels=3):
    """The decoder-side state_dict keys in module registration order: AutoencoderKL.__init__ (post_quant_conv = Conv2d(4, 4, 1)),
    Decoder.__init__ (conv_in, mid_block, up_blocks with layers_per_block + 1 resnets and an Upsample2D(use_conv=True) on
    all but the last, conv_norm_out, conv_out), ResnetBlock2D(temb_channels=None) and the mid-block
    Attention(heads=1, bias=True, norm_num_groups=32) under its 0.19.3 names."""
    sh = OrderedDict()

    def resnet(p, cin, cout):
        sh[p + ".norm1.weight"], sh[p + ".norm1.bias"] = (cin,), (cin,)
        sh[p + ".conv1.weight"], sh[p + ".conv1.bias"] = (cout, cin, 3, 3), (cout,)
        sh[p + ".norm2.weight"], sh[p + ".norm2.bias"] = (cout,), (cout,)
        sh[p + ".conv2.weight"], sh[p + ".conv2.bias"] = (cout, cout, 3, 3), (cout,)
        if cin != cout:
            sh[p + ".conv_shortcut.weight"], sh[p + ".conv_shortcut.bias"] = (cout, cin, 1, 1), (cout,)

    lc = latent_channels
    sh["post_quant_conv.weight"], sh["post_quant_conv.bias"] = (lc, lc, 1, 1), (lc,)
    top = block_out_channels[-1]
    sh["decoder.conv_in.weight"], sh["decoder.conv_in.bias"] = (top, lc, 3, 3), (top,)
    resnet("decoder.mid_block.resnets.0", top, top)
    resnet("decoder.mid_block.resnets.1", top, top)
    a = "decoder.mid_block.attentions.0"
    sh[a + ".group_norm.weight"], sh[a + ".group_norm.bias"] = (top,), (top,)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        sh[f"{a}.{n}.weight"], sh[f"{a}.{n}.bias"] = (top, top), (top,)
    rev = list(reversed(block_out_channels))
    prev = rev[0]
    for i, out in enumerate(rev):
        for j in range(layers_per_block + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else out, out)
        if i != len(rev) - 1:
            sh[f"decoder.up_blocks.{i}.upsamplers.0.conv.weight"] = (out, out, 3, 3)
            sh[f"decoder.up_blocks.{i}.upsamplers.0.conv.bias"] = (out,)
        prev = out
    c0 = block_out_channels[0]
    sh["decoder.conv_norm_out.weight"], sh["decoder.conv_norm_out.bias"] = (c0,), (c0,)
    sh["decoder.conv_out.weight"], sh["decoder.conv_out.bias"] = (out_channels, c0, 3, 3), (out_channels,)
    return sh


def _conv(x, sd, p, pad=1):
    return F.conv2d(x, sd[p + ".weight"], sd[p + ".bias"], padding=pad)


def _gn(x, sd, p):
    return F.group_norm(x, GROUPS, sd[p + ".weight"], sd[p + ".bias"], EPS)


def resnet_block(x, sd, p):
    """ResnetBlock2D.forward with temb=None, output_scale_factor=1, dropout inactive (models/resnet.py)."""
    h = _conv(F.silu(_gn(x, sd, p + ".norm1")), sd, p + ".conv1")
    h = _conv(F.silu(_gn(h, sd, p + ".norm2")), sd, p + ".conv2")
    if p + ".conv_shortcut.weight" in sd:
        x = _conv(x, sd, p + ".conv_shortcut", pad=0)
    return x + h


def attention(x, sd, p):
    """Attention(query_dim=C, heads=1, dim_head=C, residual_connection=True, bias=True) run by AttnProcessor2_0
    (models/attention_processor.py): group_norm, to_q / to_k / to_v, SDPA with scale 1 / sqrt(C), to_out[0], + residual,
    / rescale_output_factor (1)."""
    n, C, H, W = x.shape
    h = _gn(x, sd, p + ".group_norm").view(n, C, H * W).transpose(1, 2)
    q, k, v = (F.linear(h, sd[f"{p}.{t}.weight"], sd[f"{p}.{t}.bias"]) for t in ("to_q", "to_k", "to_v"))
    o = F.scaled_dot_product_attention(q[:, None], k[:, None], v[:, None], scale=1.0 / math.sqrt(C))[:, 0]
    o = F.linear(o, sd[p + ".to_out.0.weight"], sd[p + ".to_out.0.bias"])
    return o.transpose(1, 2).reshape(n, C, H, W) + x


def upsample(x, sd, p):
    """Upsample2D(use_conv=True).forward: F.interpolate(scale_factor=2.0, mode="nearest"), then conv (3x3, pad 1)."""
    return _conv(F.interpolate(x, scale_factor=2.0, mode="nearest"), sd, p + ".conv")


def decode(z, sd, layers_per_block=2, taps=None):
    """AutoencoderKL._decode: post_quant_conv, then Decoder.forward (conv_in, UNetMidBlock2D: resnet, attention, resnet;
    UpDecoderBlock2D x 4; conv_norm_out, SiLU, conv_out).  z [n, 4, h, w] -> sample [n, 3, 8h, 8w].  taps: dict that
    receives each block's output (NCHW)."""
    def tap(name, t):
        if taps is not None:
            taps[name] = t

    x = _conv(z, sd, "post_quant_conv", pad=0)
    x = _conv(x, sd, "decoder.conv_in")
    tap("conv_in", x)
    x = resnet_block(x, sd, "decoder.mid_block.resnets.0")
    x = attention(x, sd, "decoder.mid_block.attentions.0")
    tap("mid_block.attentions.0", x)
    x = resnet_block(x, sd, "decoder.mid_block.resnets.1")
    tap("mid_block", x)
    i = 0
    while f"decoder.up_blocks.{i}.resnets.0.conv1.weight" in sd:
        for j in range(layers_per_block + 1):
            x = resnet_block(x, sd, f"decoder.up_blocks.{i}.resnets.{j}")
        if f"decoder.up_blocks.{i}.upsamplers.0.conv.weight" in sd:
            x = upsample(x, sd, f"decoder.up_blocks.{i}.upsamplers.0")
        tap(f"up_blocks.{i}", x)
        i += 1
    x = _conv(F.silu(_gn(x, sd, "decoder.conv_norm_out")), sd, "decoder.conv_out")
    tap("conv_out", x)
    return x


def postprocess(image, output_type="pil"):
    """VaeImageProcessor.postprocess (image_processor.py) with do_normalize=True: denormalize = (x / 2 + 0.5).clamp(0, 1);
    "pt" returns that tensor, "np" pt_to_numpy (NHWC float32), "pil" numpy_to_pil's (images * 255).round().astype("uint8")
    (as a uint8 array; PIL.Image.fromarray of it is the image)."""
    y = (image / 2 + 0.5).clamp(0, 1)
    if output_type == "pt":
        return y
    y = y.cpu().permute(0, 2, 3, 1).float().numpy()
    if output_type == "np":
        return y
    return (y * 255).round().astype("uint8")
