"""Functional restatement of the encode side of diffusers 0.19.3 `AutoencoderKL` for the SD-1.5 VAE (the checker of
`AutoencoderKL.encode` in videoswap_b200/vae.py): `Encoder`, `DownEncoderBlock2D`, `Downsample2D(padding=0)`,
`quant_conv`, `DiagonalGaussianDistribution` and the PIL path of `VaeImageProcessor.preprocess`.  Unpinned for the same
reason as tests/vae_oracle.py (whose resnet, attention, conv and GroupNorm functions it reuses): the reference checkout has
no VAE code of its own (it imports diffusers' AutoencoderKL, pipeline_videoswap.py:95) and diffusers is not a dependency
here, so each function says which diffusers 0.19.3 code it restates.

Device- and dtype-agnostic torch: the tests run it on the CPU in fp32; tools/gpu_vae_encode.py runs the same functions on
CUDA in fp16 (cuDNN convolutions, scaled_dot_product_attention) as the stock-PyTorch baseline."""
from __future__ import annotations

from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from tests.vae_oracle import _conv, _gn, attention, resnet_block


def param_shapes(block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=4, in_channels=3):
    """The encode-side state_dict keys: Encoder.__init__ (models/vae.py: conv_in = Conv2d(3, 128, 3, padding=1);
    DownEncoderBlock2D(num_layers=layers_per_block, add_downsample=not is_final_block, downsample_padding=0) per level;
    UNetMidBlock2D with one Attention(heads=1) under its 0.19.3 names; conv_norm_out; conv_out = Conv2d(512,
    2 * latent_channels, 3, padding=1) for double_z=True) and AutoencoderKL.__init__'s quant_conv = Conv2d(8, 8, 1)."""
    sh = OrderedDict()

    def resnet(p, cin, cout):
        sh[p + ".norm1.weight"], sh[p + ".norm1.bias"] = (cin,), (cin,)
        sh[p + ".conv1.weight"], sh[p + ".conv1.bias"] = (cout, cin, 3, 3), (cout,)
        sh[p + ".norm2.weight"], sh[p + ".norm2.bias"] = (cout,), (cout,)
        sh[p + ".conv2.weight"], sh[p + ".conv2.bias"] = (cout, cout, 3, 3), (cout,)
        if cin != cout:
            sh[p + ".conv_shortcut.weight"], sh[p + ".conv_shortcut.bias"] = (cout, cin, 1, 1), (cout,)

    c0, top = block_out_channels[0], block_out_channels[-1]
    sh["encoder.conv_in.weight"], sh["encoder.conv_in.bias"] = (c0, in_channels, 3, 3), (c0,)
    prev = c0
    for i, out in enumerate(block_out_channels):
        for j in range(layers_per_block):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else out, out)
        if i != len(block_out_channels) - 1:
            sh[f"encoder.down_blocks.{i}.downsamplers.0.conv.weight"] = (out, out, 3, 3)
            sh[f"encoder.down_blocks.{i}.downsamplers.0.conv.bias"] = (out,)
        prev = out
    a = "encoder.mid_block.attentions.0"
    sh[a + ".group_norm.weight"], sh[a + ".group_norm.bias"] = (top,), (top,)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        sh[f"{a}.{n}.weight"], sh[f"{a}.{n}.bias"] = (top, top), (top,)
    resnet("encoder.mid_block.resnets.0", top, top)
    resnet("encoder.mid_block.resnets.1", top, top)
    sh["encoder.conv_norm_out.weight"], sh["encoder.conv_norm_out.bias"] = (top,), (top,)
    z = 2 * latent_channels
    sh["encoder.conv_out.weight"], sh["encoder.conv_out.bias"] = (z, top, 3, 3), (z,)
    sh["quant_conv.weight"], sh["quant_conv.bias"] = (z, z, 1, 1), (z,)
    return sh


def downsample(x, sd, p):
    """Downsample2D(use_conv=True, padding=0).forward (models/resnet.py): `if self.use_conv and self.padding == 0:
    pad = (0, 1, 0, 1); hidden_states = F.pad(hidden_states, pad, mode="constant", value=0)`, then the 3x3 conv with
    stride 2 and padding 0."""
    x = F.pad(x, (0, 1, 0, 1), mode="constant", value=0)
    return F.conv2d(x, sd[p + ".conv.weight"], sd[p + ".conv.bias"], stride=2)


def encode(x, sd, layers_per_block=2, taps=None):
    """AutoencoderKL.encode without tiling: Encoder.forward (conv_in; DownEncoderBlock2D x 4: resnets, then the
    down-sampler; UNetMidBlock2D: resnet, attention, resnet; conv_norm_out, SiLU, conv_out), then quant_conv.
    x [n, 3, H, W] -> the moments [n, 8, H / 8, W / 8].  taps: dict that receives each block's output (NCHW)."""
    def tap(name, t):
        if taps is not None:
            taps[name] = t

    x = _conv(x, sd, "encoder.conv_in")
    tap("conv_in", x)
    i = 0
    while f"encoder.down_blocks.{i}.resnets.0.conv1.weight" in sd:
        for j in range(layers_per_block):
            x = resnet_block(x, sd, f"encoder.down_blocks.{i}.resnets.{j}")
        if f"encoder.down_blocks.{i}.downsamplers.0.conv.weight" in sd:
            x = downsample(x, sd, f"encoder.down_blocks.{i}.downsamplers.0")
        tap(f"down_blocks.{i}", x)
        i += 1
    x = resnet_block(x, sd, "encoder.mid_block.resnets.0")
    x = attention(x, sd, "encoder.mid_block.attentions.0")
    tap("mid_block.attentions.0", x)
    x = resnet_block(x, sd, "encoder.mid_block.resnets.1")
    tap("mid_block", x)
    x = _conv(F.silu(_gn(x, sd, "encoder.conv_norm_out")), sd, "encoder.conv_out")
    tap("conv_out", x)
    return _conv(x, sd, "quant_conv", pad=0)


def posterior(moments, noise=None):
    """DiagonalGaussianDistribution (models/vae.py): mean, logvar = chunk(parameters, 2, dim=1); logvar =
    clamp(logvar, -30, 20); std = exp(0.5 logvar); sample = mean + std * noise (noise = randn_tensor(mean.shape, ...));
    mode() = mean.  Returns (sample or mode, mean, logvar, std)."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    std = torch.exp(0.5 * logvar)
    return (mean if noise is None else mean + std * noise), mean, logvar, std


def preprocess(frames):
    """VaeImageProcessor.preprocess of a list of PIL images (image_processor.py, vae_scale_factor 8, resample "lanczos",
    do_normalize): resize to (w - w % 8, h - h % 8), pil_to_numpy (np.array(image).astype(np.float32) / 255.0, stacked),
    numpy_to_pt (NHWC -> NCHW), normalize (2.0 * images - 1.0).  Returns fp32 [F, 3, H, W]."""
    from PIL import Image
    arrs = []
    for im in frames:
        w, h = (x - x % 8 for x in im.size)
        im = im.resize((w, h), resample=Image.LANCZOS)
        arrs.append(np.array(im).astype(np.float32) / 255.0)
    images = torch.from_numpy(np.stack(arrs, axis=0).transpose(0, 3, 1, 2))
    return 2.0 * images - 1.0
