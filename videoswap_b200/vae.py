"""diffusers 0.19.3 `AutoencoderKL` (SD-1.5's VAE) on the native kernels, with diffusers' config and state_dict names.
Decoder: the reference's loop ends with `vae.decode(latents / scaling_factor)` and `VaeImageProcessor.postprocess`
(videoswap/pipelines/pipeline_videoswap.py:603-610); `decode_postprocess` replaces the two calls, `decode` the first.
Encoder: `prepare_image_latents` starts the edit with `vae.encode(image).latent_dist.sample(generator) * scaling_factor`
(pipeline_videoswap.py:204-233); `encode` returns the same `AutoencoderKLOutput(latent_dist=DiagonalGaussianDistribution)`.

Executor: a short sequence over `ops`, activations NHWC fp16, every frame of a call in one pass (the GroupNorms are per
image, so frames stay independent).  The mid block's single-head attention (d = 512) runs per frame as GEMMs around a row
softmax: S = Q K^T into one [hw, hw_pad] buffer, P = softmax(S / sqrt(512)) in place, O = P V with V transposed.  The
encoder's stride-2 down-samplers run as implicit GEMMs on parity views of their input (ops.downsample_conv3x3)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch

from . import ops
from .noise import randn_tensor
from .spec import VAEConfig, vae_encoder_param_shapes, vae_param_shapes
from .weights import config_kwargs, missing_keys_text, read_pretrained_dir, seeded_state_dict

EPS = 1e-6                     # resnet_eps of the SD-1.5 decoder (GroupNorms of resnets, attention and conv_norm_out)
CONV_OUT_PAD = 8               # conv_out's 3 output channels padded to 8 so the conv kernel's stores stay 16-byte aligned

# Pre-0.14 diffusers names of the mid-block attention, still shipped in SD-1.5 VAE files ([C, C] or 1x1-conv [C, C, 1, 1])
_OLD_ATTN = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}
_ENCODER_PREFIXES = ("encoder.", "quant_conv.")   # the encode half's keys; every other key belongs to the decode half
_DECODER_ATTN = "decoder.mid_block.attentions.0"
_ENCODER_ATTN = "encoder.mid_block.attentions.0"


@dataclass
class DecoderOutput:
    sample: torch.Tensor


def _convert_half(sd: Dict[str, torch.Tensor], shapes, attn: str):
    """The keys of one VAE half in sd, renamed and reshaped to that half's `shapes` -> (dict, missing keys).  attn is the
    half's mid-block attention: under "encoder." the half is the encoder / quant_conv keys, otherwise every other key;
    keys of the other half are skipped.  Old attention names under attn are renamed; a key of the half that `shapes`
    does not know, a key given twice or a wrong shape raises."""
    encoder = attn.startswith("encoder.")
    out = {}
    for k, v in sd.items():
        if k.startswith(_ENCODER_PREFIXES) != encoder:
            continue
        name = k
        head, _, leaf = k.rpartition(".")
        parent, _, old = head.rpartition(".")
        if parent == attn and old in _OLD_ATTN:
            name = f"{attn}.{_OLD_ATTN[old]}.{leaf}"
        if name not in shapes:
            raise KeyError(f"unexpected key in the VAE state_dict: {k}")
        if name in out:
            raise KeyError(f"{k}: {name} is given twice (old and new attention names)")
        want = shapes[name]
        if tuple(v.shape) != want:
            # the attention's linear weights, the only 2-D entries, may come as 1x1-conv weights
            if name.startswith(attn + ".") and len(want) == 2 and tuple(v.shape) == want + (1, 1):
                v = v.reshape(want)
            else:
                raise ValueError(f"{k}: shape {tuple(v.shape)}, expected {want}")
        out[name] = v
    return out, [k for k in shapes if k not in out]


def convert_state_dict(sd: Dict[str, torch.Tensor], cfg: VAEConfig) -> Dict[str, torch.Tensor]:
    """A full or decoder-only AutoencoderKL state_dict -> the decoder keys of vae_param_shapes(cfg), in their shapes.
    Old attention names are renamed, encoder / quant_conv keys dropped; any other unknown key, a wrong shape or a missing
    decoder key raises."""
    out, missing = _convert_half(sd, vae_param_shapes(cfg), _DECODER_ATTN)
    if missing:
        raise KeyError(f"missing decoder keys in the VAE state_dict: {missing_keys_text(missing)}")
    return out


def convert_encoder_state_dict(sd: Dict[str, torch.Tensor], cfg: VAEConfig) -> Dict[str, torch.Tensor]:
    """A full AutoencoderKL state_dict -> the encoder / quant_conv keys of vae_encoder_param_shapes(cfg), in their shapes.
    The same old attention names as convert_state_dict are renamed (encoder.mid_block.attentions.0); decoder keys are
    skipped; an unknown encoder key, a wrong shape or a missing encoder key raises."""
    out, missing = _convert_half(sd, vae_encoder_param_shapes(cfg), _ENCODER_ATTN)
    if missing:
        raise KeyError(f"missing encoder keys in the VAE state_dict: {missing_keys_text(missing)}")
    return out


@dataclass
class AutoencoderKLOutput:
    latent_dist: "DiagonalGaussianDistribution"


class DiagonalGaussianDistribution:
    """diffusers' posterior over the moments `parameters` [n, 8, h, w] fp16 (mean in channels 0..3, logvar in 4..7).
    `sample` and `mode` run the vae_posterior kernel; mean / logvar / std / var are views and small tensors for callers."""

    def __init__(self, parameters: torch.Tensor):
        self.parameters = parameters

    @property
    def mean(self) -> torch.Tensor:
        return self.parameters[:, :4]

    @property
    def logvar(self) -> torch.Tensor:
        return self.parameters[:, 4:].clamp(-30.0, 20.0)

    @property
    def std(self) -> torch.Tensor:
        return torch.exp(0.5 * self.logvar)

    @property
    def var(self) -> torch.Tensor:
        return torch.exp(self.logvar)

    def noise(self, generator=None) -> torch.Tensor:
        """The standard normal draw of diffusers 0.19.3 `randn_tensor(mean.shape, generator, device, dtype=fp16)`
        (noise.randn_tensor): one draw per frame for a list of generators."""
        shape = (self.parameters.shape[0], 4) + tuple(self.parameters.shape[2:])
        return randn_tensor(shape, generator, self.parameters.device, torch.float16)

    def sample(self, generator=None, scale: float = 1.0, video: bool = False) -> torch.Tensor:
        """scale (mean + std noise) with the noise of `noise(generator)`, fp16 [n, 4, h, w] (video=True: [1, 4, n, h, w])."""
        return ops.vae_posterior(self.parameters, self.noise(generator), scale, video)

    def mode(self, scale: float = 1.0, video: bool = False) -> torch.Tensor:
        return ops.vae_posterior(self.parameters, None, scale, video)


def padded_keys(nk: int) -> int:
    """Row stride of S / P: O = P V runs with K = this, which the GEMM needs to be a multiple of 8."""
    return -(-nk // 8) * 8


def attend(q, k, v, s, vt, out):
    """One frame of single-head attention, out = softmax(q k^T / sqrt(d)) v: q, k, v [hw, d] fp16; scratch s
    [hw, padded_keys(hw)] (S, then P in place) and vt [d, padded_keys(hw)] (V^T with zero padding columns)."""
    hw, d = q.shape
    ops.scores(q, k, s)
    ops.softmax_rows(s, hw, 1.0 / math.sqrt(d))
    ops.transpose_pad(v, s.shape[1], out=vt)
    return ops.gemm(s, vt, out=out)


def _tap(taps, name, t):
    """Records a block's NHWC output in the executors' debugging dict, when one is given."""
    if taps is not None:
        taps[name] = t


class AutoencoderKL:
    """diffusers' AutoencoderKL (decode and encode) on CUDA.  init="seeded" draws test weights for both halves
    (weights.seeded_state_dict), "empty" waits for load_state_dict."""

    def __init__(self, init: str = "seeded", device="cuda", **config):
        self.config = VAEConfig(**config)
        cfg = self.config
        if cfg.latent_channels != 4 or cfg.out_channels != 3:
            raise ValueError("the native decoder takes 4 latent channels and makes 3 image channels")
        self.device = torch.device(device)
        self._w = None
        self._we = None                     # encoder weights (None: the last state_dict had no complete encoder half)
        self._enc_missing = list(vae_encoder_param_shapes(cfg))
        if init == "seeded":
            self.load_state_dict(seeded_state_dict({**vae_param_shapes(cfg), **vae_encoder_param_shapes(cfg)}, seed=7))
        elif init != "empty":
            raise ValueError(f"init must be 'seeded' or 'empty', got {init!r}")

    # ------------------------------------------------------------------------------------------------ construction
    @classmethod
    def from_config(cls, config, **kw):
        """diffusers-style: keys of VAEConfig are used, the rest of a config.json (class name, block types, ...) ignored."""
        if not isinstance(config, dict):
            config = config.to_dict()
        if config.get("act_fn", "silu") != "silu":
            raise ValueError(f"unsupported act_fn {config['act_fn']!r}")
        return cls(**kw, **config_kwargs(config, VAEConfig))

    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = "vae", device="cuda"):
        """A local diffusers directory: config.json + diffusion_pytorch_model.safetensors (or .bin)."""
        config, sd = read_pretrained_dir(path, subfolder, "diffusion_pytorch_model.safetensors",
                                         "diffusion_pytorch_model.bin")
        return cls.from_config(config, init="empty", device=device).load_state_dict(sd)

    # ------------------------------------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        """Converts (convert_state_dict) and packs every decoder weight once: conv3x3 panels, sub-pixel panels of the
        up-samplers, the attention's q / k / v as one [3C, C] weight, conv_out padded to 8 output channels.  The encoder
        half (convert_encoder_state_dict) is packed too when sd holds all of it; otherwise `encode` raises, naming the
        missing keys."""
        if self.device.type != "cuda":
            raise RuntimeError("AutoencoderKL (videoswap_b200) runs on CUDA only")
        enc, self._enc_missing = _convert_half(sd, vae_encoder_param_shapes(self.config), _ENCODER_ATTN)
        sd = convert_state_dict(sd, self.config)
        self._w = self._pack_decoder(sd)
        self._we = self._pack_encoder(enc) if not self._enc_missing else None
        return self

    def _loaders(self, sd):
        """(fp16, fp32) loaders of sd's tensors onto the device."""
        dev = self.device
        return (lambda k: sd[k].detach().to(dev, torch.float16).contiguous(),
                lambda k: sd[k].detach().to(dev, torch.float32).contiguous())

    def _pack_resnet(self, sd, p):
        h16, f32 = self._loaders(sd)

        def norm(q):
            return f32(q + ".weight"), f32(q + ".bias")
        r = {"norm1": norm(p + ".norm1"), "norm2": norm(p + ".norm2"),
             "conv1": (ops.pack_conv3x3(h16(p + ".conv1.weight")), f32(p + ".conv1.bias")),
             "conv2": (ops.pack_conv3x3(h16(p + ".conv2.weight")), f32(p + ".conv2.bias"))}
        if p + ".conv_shortcut.weight" in sd:
            w = h16(p + ".conv_shortcut.weight")
            r["shortcut"] = (w.reshape(w.shape[0], w.shape[1]).contiguous(), f32(p + ".conv_shortcut.bias"))
        return r

    def _pack_attention(self, sd, a):
        h16, f32 = self._loaders(sd)
        return {"norm": (f32(a + ".group_norm.weight"), f32(a + ".group_norm.bias")),
                "qkv": (torch.cat([h16(f"{a}.{n}.weight") for n in ("to_q", "to_k", "to_v")]).contiguous(),
                        torch.cat([f32(f"{a}.{n}.bias") for n in ("to_q", "to_k", "to_v")]).contiguous()),
                "out": (h16(a + ".to_out.0.weight"), f32(a + ".to_out.0.bias"))}

    def _pack_encoder(self, sd):
        """conv_in's [128, 3, 3, 3] weight zero-padded to 4 input channels (the tensor-core conv_in), conv3x3 panels of the
        resnets, down-samplers and conv_out (8 output channels, no padding needed), quant_conv as fp32 weight + bias."""
        h16, f32 = self._loaders(sd)
        cfg = self.config
        wi = h16("encoder.conv_in.weight")
        wi4 = torch.zeros((wi.shape[0], 4, 3, 3), dtype=torch.float16, device=self.device)
        wi4[:, :3] = wi
        n = len(cfg.block_out_channels)
        return {
            "conv_in": (wi4, f32("encoder.conv_in.bias")),
            "down": [{"resnets": [self._pack_resnet(sd, f"encoder.down_blocks.{i}.resnets.{j}") for j in range(cfg.layers_per_block)],
                      "downsampler": (ops.pack_conv3x3(h16(f"encoder.down_blocks.{i}.downsamplers.0.conv.weight")),
                                      f32(f"encoder.down_blocks.{i}.downsamplers.0.conv.bias")) if i < n - 1 else None}
                     for i in range(n)],
            "mid": [self._pack_resnet(sd, f"encoder.mid_block.resnets.{j}") for j in (0, 1)],
            "attn": self._pack_attention(sd, "encoder.mid_block.attentions.0"),
            "norm_out": (f32("encoder.conv_norm_out.weight"), f32("encoder.conv_norm_out.bias")),
            "conv_out": (ops.pack_conv3x3(h16("encoder.conv_out.weight")), f32("encoder.conv_out.bias")),
            "moments": torch.cat([f32("quant_conv.weight").flatten(), f32("quant_conv.bias")]).contiguous(),
        }

    def _pack_decoder(self, sd):
        dev = self.device
        h16, f32 = self._loaders(sd)
        cfg = self.config
        n_up = len(cfg.block_out_channels)
        w = {
            "latent_in": torch.cat([f32("post_quant_conv.weight").flatten(), f32("post_quant_conv.bias")]).contiguous(),
            "conv_in": (h16("decoder.conv_in.weight"), f32("decoder.conv_in.bias")),
            "mid": [self._pack_resnet(sd, f"decoder.mid_block.resnets.{j}") for j in (0, 1)],
            "attn": self._pack_attention(sd, "decoder.mid_block.attentions.0"),
            "up": [{"resnets": [self._pack_resnet(sd, f"decoder.up_blocks.{i}.resnets.{j}") for j in range(cfg.layers_per_block + 1)],
                    "upsampler": (ops.pack_conv_subpixel(h16(f"decoder.up_blocks.{i}.upsamplers.0.conv.weight")),
                                  f32(f"decoder.up_blocks.{i}.upsamplers.0.conv.bias")) if i < n_up - 1 else None}
                   for i in range(n_up)],
            "norm_out": (f32("decoder.conv_norm_out.weight"), f32("decoder.conv_norm_out.bias")),
        }
        wo = torch.zeros((CONV_OUT_PAD,) + tuple(sd["decoder.conv_out.weight"].shape[1:]), dtype=torch.float16, device=dev)
        wo[:cfg.out_channels] = h16("decoder.conv_out.weight")
        bo = torch.zeros(CONV_OUT_PAD, dtype=torch.float32, device=dev)
        bo[:cfg.out_channels] = f32("decoder.conv_out.bias")
        w["conv_out"] = (ops.pack_conv3x3(wo), bo)
        return w

    # ------------------------------------------------------------------------------------------------ executor
    def _groups(self):
        return self.config.norm_num_groups

    def _resnet(self, x, r):
        """ResnetBlock2D with temb=None: conv2(silu(gn2(conv1(silu(gn1(x)))))) + shortcut(x), output_scale_factor 1."""
        n, H, W, ci = x.shape
        h = ops.groupnorm(x, *r["norm1"], self._groups(), EPS, silu=True)
        h = ops.conv3x3(h, *r["conv1"])
        h = ops.groupnorm(h, *r["norm2"], self._groups(), EPS, silu=True)
        sc = x
        if "shortcut" in r:
            ws, bs = r["shortcut"]
            sc = ops.gemm(x.view(n * H * W, ci), ws, bias=bs).view(n, H, W, ws.shape[0])
        return ops.conv3x3(h, *r["conv2"], residual=sc)

    def _attention(self, x, a):
        """Attention(heads=1, residual_connection=True) under AttnProcessor2_0: to_out(softmax(q k^T / sqrt(C)) v) + x."""
        n, H, W, C = x.shape
        hw = H * W
        ld = padded_keys(hw)
        h = ops.groupnorm(x, *a["norm"], self._groups(), EPS).view(n * hw, C)
        wqkv, bqkv = a["qkv"]
        # q, k, v from row blocks of the packed weight, each its own contiguous tensor: K is the B operand of S = Q K^T,
        # which the GEMM reads with unit-stride rows
        q, k, v = (ops.gemm(h, wqkv[i * C:(i + 1) * C], bias=bqkv[i * C:(i + 1) * C]) for i in range(3))
        s = torch.empty((hw, ld), dtype=torch.float16, device=x.device)
        vt = torch.empty((C, ld), dtype=torch.float16, device=x.device)
        o = torch.empty((n * hw, C), dtype=torch.float16, device=x.device)
        for f in range(n):
            rows = slice(f * hw, (f + 1) * hw)
            attend(q[rows], k[rows], v[rows], s, vt, o[rows])
        wo, bo = a["out"]
        return ops.gemm(o, wo, bias=bo, residual=x.view(n * hw, C)).view(n, H, W, C)

    def _mid_block(self, x, w, taps):
        """UNetMidBlock2D of either half: resnet, attention, resnet."""
        x = self._resnet(x, w["mid"][0])
        x = self._attention(x, w["attn"])
        _tap(taps, "mid_block.attentions.0", x)
        x = self._resnet(x, w["mid"][1])
        _tap(taps, "mid_block", x)
        return x

    def _out(self, x, w, taps):
        """The tail of either half: conv_out(silu(conv_norm_out(x)))."""
        x = ops.groupnorm(x, *w["norm_out"], self._groups(), EPS, silu=True)
        x = ops.conv3x3(x, *w["conv_out"])
        _tap(taps, "conv_out", x)
        return x

    def _run(self, z, divisor, fmt, taps=None):
        """post_quant_conv(z / divisor) -> Decoder -> image_postprocess(fmt).  taps: dict that receives each block's NHWC
        output (debugging)."""
        if self._w is None:
            raise RuntimeError("AutoencoderKL has no weights: load_state_dict first")
        if not z.is_cuda:
            raise RuntimeError("AutoencoderKL (videoswap_b200) runs on CUDA only")
        if z.dim() != 4 or z.shape[1] != self.config.latent_channels:
            raise ValueError(f"expected latents [n, {self.config.latent_channels}, h, w], got {tuple(z.shape)}")
        w = self._w
        z = z.contiguous() if z.dtype in (torch.float16, torch.float32) else z.float().contiguous()
        x = ops.vae_latent_in(z, divisor, w["latent_in"])
        x = ops.conv_in(x, *w["conv_in"])
        _tap(taps, "conv_in", x)
        x = self._mid_block(x, w, taps)
        for i, blk in enumerate(w["up"]):
            for r in blk["resnets"]:
                x = self._resnet(x, r)
            if blk["upsampler"] is not None:
                x = ops.upsample_conv3x3_packed(x, *blk["upsampler"])
            _tap(taps, f"up_blocks.{i}", x)
        return ops.image_postprocess(self._out(x, w, taps), fmt)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True):
        """AutoencoderKL.decode: CUDA latents [n, 4, h, w] (fp16 / fp32) -> sample fp16 [n, 3, 8h, 8w] (not clamped)."""
        sample = self._run(z, 1.0, ops.IMG_SAMPLE)
        return DecoderOutput(sample=sample) if return_dict else (sample,)

    @torch.no_grad()
    def decode_postprocess(self, latents: torch.Tensor, output_type: str = "pil"):
        """VaeImageProcessor.postprocess(decode(latents / scaling_factor)) in one pass (pipeline_videoswap.py:603-610):
        "pt" fp32 [n, 3, H, W] in [0, 1], "np" fp32 numpy [n, H, W, 3], "pil" a list of RGB PIL images."""
        fmt = {"pt": ops.IMG_PT, "np": ops.IMG_NP, "pil": ops.IMG_PIL}.get(output_type)
        if fmt is None:
            raise ValueError(f"output_type must be 'pt', 'np' or 'pil', got {output_type!r}")
        img = self._run(latents, self.config.scaling_factor, fmt)
        if output_type == "pt":
            return img
        img = img.cpu().numpy()
        if output_type == "np":
            return img
        from PIL import Image
        return [Image.fromarray(a) for a in img]

    # ------------------------------------------------------------------------------------------------ encoder
    def _encode_run(self, x, taps=None):
        """vae_image_in -> Encoder -> quant_conv: x uint8 frames [n, H, W, 3] or float images [n, 3, H, W] in [-1, 1]
        (CUDA) -> the moments fp16 [n, 8, H / 8, W / 8].  taps: dict that receives each block's NHWC output (debugging)."""
        if self._we is None:
            raise RuntimeError("AutoencoderKL has no encoder weights: the last state_dict lacked "
                               + missing_keys_text(self._enc_missing))
        if not x.is_cuda:
            raise RuntimeError("AutoencoderKL (videoswap_b200) runs on CUDA only")
        if x.dim() != 4:
            raise ValueError(f"expected 4-D images, got {tuple(x.shape)}")
        H, W = (x.shape[1], x.shape[2]) if x.dtype == torch.uint8 else (x.shape[2], x.shape[3])
        if H % 8 or W % 8:
            raise ValueError(f"the encoder takes images whose height and width are multiples of 8, got {tuple(x.shape)}")
        w = self._we
        x = ops.vae_image_in(x.contiguous())
        x = ops.conv_in(x, *w["conv_in"])
        _tap(taps, "conv_in", x)
        for i, blk in enumerate(w["down"]):
            for r in blk["resnets"]:
                x = self._resnet(x, r)
            if blk["downsampler"] is not None:
                x = ops.downsample_conv3x3(x, *blk["downsampler"])
            _tap(taps, f"down_blocks.{i}", x)
        x = self._mid_block(x, w, taps)
        return ops.vae_moments(self._out(x, w, taps), w["moments"])

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """AutoencoderKL.encode: CUDA images [n, 3, H, W] (fp16 / fp32, in [-1, 1]; H, W multiples of 8) ->
        AutoencoderKLOutput(latent_dist=DiagonalGaussianDistribution) over the moments [n, 8, H / 8, W / 8]."""
        if x.dim() != 4 or x.shape[1] != self.config.in_channels or x.dtype not in (torch.float16, torch.float32):
            raise ValueError(f"expected fp16 / fp32 images [n, {self.config.in_channels}, H, W], got {tuple(x.shape)} {x.dtype}")
        dist = DiagonalGaussianDistribution(self._encode_run(x))
        return AutoencoderKLOutput(latent_dist=dist) if return_dict else (dist,)

    @torch.no_grad()
    def encode_frames(self, frames: torch.Tensor) -> DiagonalGaussianDistribution:
        """The posterior of uint8 RGB frames [n, H, W, 3] (CUDA), normalised as VaeImageProcessor.preprocess does."""
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
            raise ValueError(f"expected uint8 frames [n, H, W, 3], got {tuple(frames.shape)} {frames.dtype}")
        return DiagonalGaussianDistribution(self._encode_run(frames))
