"""diffusers 0.19.3 `T2IAdapter` with adapter_type "full_adapter" (FullAdapter) on the native kernels, with diffusers'
config and state_dict names: the adapter of the reference's image-condition branch (videoswap/pipelines/
pipeline_videoswap.py:538-546), where `conditions` is a list of per-frame images (depth, sketch, pose, ... maps) and
`adapter(_preprocess_adapter_image(conditions, height, width))` gives the four UNet down-block residuals.

Executor, activations NHWC fp16, every frame in one pass:
  t2i_image_in (u8 / 255, fp16, PixelUnshuffle(8)) -> conv_in (3x3) -> 4 AdapterBlocks, block i:
    [i > 0: avgpool2x2] -> [in_conv 1x1 when the width changes] -> num_res_blocks x (x + block2(relu(block1(x))))
  with block1 a 3x3 conv whose epilogue applies the bias and the ReLU, and block2 a 1x1 GEMM whose epilogue adds the
  bias and then the residual x in fp16 (torch's rounding order of `conv(h) + x`).
The features after each block are the residuals, at strides 8 / 16 / 32 / 64 of the frames."""
from __future__ import annotations

from dataclasses import asdict, dataclass
from typing import Dict, List, Optional, Tuple

import torch

from . import ops
from .weights import config_kwargs, missing_keys_text, read_pretrained_dir, seeded_state_dict

SIZE_MULTIPLE = 64             # frame sides the adapter takes: where floor and ceil pooling agree at every level


@dataclass
class T2IAdapterConfig:
    """diffusers 0.19.3 T2IAdapter's config (config.json)."""
    in_channels: int = 3
    channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    num_res_blocks: int = 2
    downscale_factor: int = 8
    adapter_type: str = "full_adapter"

    def to_dict(self):
        return asdict(self)


def t2i_adapter_param_shapes(cfg: T2IAdapterConfig) -> Dict[str, Tuple[int, ...]]:
    """The FullAdapter's state_dict keys and shapes: adapter.conv_in, adapter.body.{i}.in_conv (blocks whose width
    changes), adapter.body.{i}.resnets.{j}.block1 (3x3) / block2 (1x1)."""
    ch = cfg.channels
    cin = cfg.in_channels * cfg.downscale_factor ** 2
    sh = {"adapter.conv_in.weight": (ch[0], cin, 3, 3), "adapter.conv_in.bias": (ch[0],)}
    for i, c in enumerate(ch):
        prev = ch[max(i - 1, 0)]
        p = f"adapter.body.{i}"
        if prev != c:
            sh[f"{p}.in_conv.weight"] = (c, prev, 1, 1)
            sh[f"{p}.in_conv.bias"] = (c,)
        for j in range(cfg.num_res_blocks):
            q = f"{p}.resnets.{j}"
            sh[f"{q}.block1.weight"] = (c, c, 3, 3)
            sh[f"{q}.block1.bias"] = (c,)
            sh[f"{q}.block2.weight"] = (c, c, 1, 1)
            sh[f"{q}.block2.bias"] = (c,)
    return sh


def check_config(cfg: T2IAdapterConfig):
    """Raises for what the native adapter does not implement (NotImplementedError) or what diffusers rejects too."""
    if cfg.adapter_type == "light_adapter":
        raise NotImplementedError("T2IAdapter: adapter_type 'light_adapter' (LightAdapter) is not implemented; "
                                  "only 'full_adapter' is")
    if cfg.adapter_type != "full_adapter":
        raise ValueError(f"T2IAdapter: unknown adapter_type {cfg.adapter_type!r}")
    if cfg.downscale_factor != 8:
        raise NotImplementedError(f"T2IAdapter: downscale_factor {cfg.downscale_factor} is not implemented; only 8 is "
                                  "(the pixel-unshuffle kernel)")
    if cfg.in_channels not in (1, 3):
        raise NotImplementedError(f"T2IAdapter: in_channels {cfg.in_channels} is not implemented; 1 (L) and 3 (RGB) are")
    if not cfg.channels or cfg.num_res_blocks < 1:
        raise ValueError("T2IAdapter: needs at least one block and one resnet per block")
    if any(c <= 0 or c % 64 for c in cfg.channels):
        raise NotImplementedError(f"T2IAdapter: channel counts {tuple(cfg.channels)} must be multiples of 64 "
                                  "(the implicit-GEMM conv's K blocks)")


def convert_state_dict(sd: Dict[str, torch.Tensor], cfg: T2IAdapterConfig) -> Dict[str, torch.Tensor]:
    """A diffusers T2IAdapter state_dict -> the same keys, checked strictly against t2i_adapter_param_shapes(cfg): an
    unknown key, a wrong shape or a missing key raises."""
    shapes = t2i_adapter_param_shapes(cfg)
    out = {}
    for k, v in sd.items():
        if k not in shapes:
            raise KeyError(f"unexpected key in the T2IAdapter state_dict: {k}")
        if tuple(v.shape) != shapes[k]:
            raise ValueError(f"{k}: shape {tuple(v.shape)}, expected {shapes[k]}")
        out[k] = v
    missing = [k for k in shapes if k not in out]
    if missing:
        raise KeyError(f"missing keys in the T2IAdapter state_dict: {missing_keys_text(missing)}")
    return out


def preprocess_frames(frames, in_channels: int) -> torch.Tensor:
    """The PIL half of diffusers 0.19.3 `_preprocess_adapter_image(frames, height, width)` with (width, height) of frame 0,
    as pipeline_videoswap.py:539-541 calls it: every frame of another size is resized to it with LANCZOS; "L" frames give
    one channel and "RGB" frames three.  Returns uint8 [F, H, W, c] (CPU) for one upload; the division by 255 runs on the
    device (t2i_image_in).  Raises ValueError, before anything reaches the GPU, for anything but a non-empty list of
    "L" / "RGB" PIL images of one mode with c == in_channels, and for sides that are not multiples of 64 px."""
    import numpy as np
    from PIL import Image
    if isinstance(frames, Image.Image):
        frames = [frames]
    if not isinstance(frames, (list, tuple)) or not frames or not all(isinstance(f, Image.Image) for f in frames):
        raise ValueError("T2IAdapter conditions must be a list of PIL images (one per frame)")
    modes = {f.mode for f in frames}
    if not modes <= {"L", "RGB"}:
        raise ValueError(f"T2IAdapter conditions must be 'L' or 'RGB' PIL images, got modes {sorted(modes)}")
    if len(modes) != 1:
        raise ValueError(f"T2IAdapter conditions mix image modes {sorted(modes)}")
    c = 1 if frames[0].mode == "L" else 3
    if c != in_channels:
        raise ValueError(f"T2IAdapter has in_channels={in_channels}, the conditions are {frames[0].mode!r} images "
                         f"with {c} channel(s)")
    width, height = frames[0].size
    if width % SIZE_MULTIPLE or height % SIZE_MULTIPLE:
        raise ValueError(f"T2IAdapter conditions must have sides that are multiples of {SIZE_MULTIPLE} px, got "
                         f"{width}x{height}")
    arrs = []
    for f in frames:
        if f.size != (width, height):
            f = f.resize((width, height), resample=Image.LANCZOS)
        a = np.asarray(f, dtype=np.uint8)
        arrs.append(a[..., None] if a.ndim == 2 else a)
    return torch.from_numpy(np.stack(arrs))


class T2IAdapter:
    """diffusers' T2IAdapter (full_adapter) on CUDA.  init="seeded" draws test weights (weights.seeded_state_dict),
    "empty" waits for load_state_dict.  The weights are converted (strictly) at load_state_dict and uploaded and packed
    at the first call."""

    def __init__(self, in_channels: int = 3, channels: Tuple[int, ...] = (320, 640, 1280, 1280), num_res_blocks: int = 2,
                 downscale_factor: int = 8, adapter_type: str = "full_adapter", init: str = "seeded", device="cuda"):
        self.config = T2IAdapterConfig(in_channels, tuple(channels), num_res_blocks, downscale_factor, adapter_type)
        check_config(self.config)
        self.device = torch.device(device)
        self._sd: Optional[Dict[str, torch.Tensor]] = None
        self._w = None
        if init == "seeded":
            self.load_state_dict(seeded_state_dict(t2i_adapter_param_shapes(self.config), seed=11))
        elif init != "empty":
            raise ValueError(f"init must be 'seeded' or 'empty', got {init!r}")

    @property
    def total_downscale_factor(self) -> int:
        return self.config.downscale_factor * 2 ** (len(self.config.channels) - 1)

    # ------------------------------------------------------------------------------------------------ construction
    @classmethod
    def from_config(cls, config, **kw):
        """diffusers-style: keys of T2IAdapterConfig are used, the rest of a config.json ignored.  A MultiAdapter config
        raises NotImplementedError."""
        if not isinstance(config, dict):
            config = config.to_dict()
        if config.get("_class_name", "T2IAdapter") == "MultiAdapter":
            raise NotImplementedError("MultiAdapter (several adapters summed) is not implemented; load one T2IAdapter")
        return cls(**kw, **config_kwargs(config, T2IAdapterConfig))

    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = None, device="cuda"):
        """A local diffusers directory: config.json + diffusion_pytorch_model.safetensors (or .bin)."""
        config, sd = read_pretrained_dir(path, subfolder, "diffusion_pytorch_model.safetensors",
                                         "diffusion_pytorch_model.bin")
        return cls.from_config(config, init="empty", device=device).load_state_dict(sd)

    # ------------------------------------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        """Checks sd strictly (convert_state_dict) and keeps it; the device copies are made at the next call."""
        self._sd = convert_state_dict(sd, self.config)
        self._w = None
        return self

    def state_dict(self) -> Dict[str, torch.Tensor]:
        if self._sd is None:
            raise RuntimeError("T2IAdapter has no weights: load_state_dict first")
        return dict(self._sd)

    def _pack(self):
        """fp16 conv3x3 panels (conv_in, block1), fp16 [Co, Ci] 1x1 weights (in_conv, block2), fp32 biases."""
        if self.device.type != "cuda":
            raise RuntimeError("T2IAdapter (videoswap_b200) runs on CUDA only")
        dev, sd = self.device, self._sd

        def h16(k):
            return sd[k].detach().to(dev, torch.float16).contiguous()

        def f32(k):
            return sd[k].detach().to(dev, torch.float32).contiguous()

        def conv1x1(p):
            w = h16(p + ".weight")
            return w.reshape(w.shape[0], w.shape[1]).contiguous(), f32(p + ".bias")
        body = []
        for i in range(len(self.config.channels)):
            p = f"adapter.body.{i}"
            body.append({
                "in_conv": conv1x1(p + ".in_conv") if p + ".in_conv.weight" in sd else None,
                "resnets": [{"block1": (ops.pack_conv3x3(h16(f"{p}.resnets.{j}.block1.weight")), f32(f"{p}.resnets.{j}.block1.bias")),
                             "block2": conv1x1(f"{p}.resnets.{j}.block2")} for j in range(self.config.num_res_blocks)]})
        return {"conv_in": (ops.pack_conv3x3(h16("adapter.conv_in.weight")), f32("adapter.conv_in.bias")), "body": body}

    # ------------------------------------------------------------------------------------------------ executor
    def preprocess(self, frames) -> torch.Tensor:
        """preprocess_frames with this adapter's in_channels: uint8 [F, H, W, c] on the CPU (no launch)."""
        return preprocess_frames(frames, self.config.in_channels)

    @torch.no_grad()
    def forward(self, frames, scale: float = 1.0, as_nchw: bool = False) -> List[torch.Tensor]:
        """frames: a list of F PIL images (see preprocess_frames), or the uint8 [F, H, W, c] tensor preprocess returns.
        Returns the four features as NHWC fp16 [F, H / s, W / s, C_l] (s = 8, 16, 32, 64), each times `scale` -- the
        reference's `v * t2i_guidance_scale` on the fp16 features (pipeline_videoswap.py:544-545).  Like the reference,
        the native code rounds twice: each feature is rounded to fp16, then the product fp32(v) * fp32(scale) is rounded
        to fp16 again, so the result equals torch's fp16 `v * scale` bit for bit.  With scale == 1 no multiply runs.
        as_nchw=True returns the reference's [F, C_l, h, w] layout instead.  The adapter always computes in fp16."""
        if self._sd is None:
            raise RuntimeError("T2IAdapter has no weights: load_state_dict first")
        u8 = frames if isinstance(frames, torch.Tensor) else self.preprocess(frames)
        if u8.dtype != torch.uint8 or u8.dim() != 4 or u8.shape[3] != self.config.in_channels:
            raise ValueError(f"expected uint8 frames [F, H, W, {self.config.in_channels}], got {tuple(u8.shape)} {u8.dtype}")
        if u8.shape[1] % SIZE_MULTIPLE or u8.shape[2] % SIZE_MULTIPLE:
            raise ValueError(f"T2IAdapter frames must have sides that are multiples of {SIZE_MULTIPLE} px, got "
                             f"{u8.shape[2]}x{u8.shape[1]}")
        if self.device.type != "cuda":
            raise RuntimeError("T2IAdapter (videoswap_b200) runs on CUDA only")
        if self._w is None:
            self._w = self._pack()
        w = self._w
        x = ops.t2i_image_in(u8.to(self.device).contiguous())
        x = ops.conv3x3(x, *w["conv_in"])
        feats = []
        for i, blk in enumerate(w["body"]):
            if i > 0:
                x = ops.avgpool2x2(x)
            n, h, wd, c = x.shape
            if blk["in_conv"] is not None:
                wi, bi = blk["in_conv"]
                x = ops.gemm(x.view(n * h * wd, c), wi, bias=bi).view(n, h, wd, wi.shape[0])
                c = wi.shape[0]
            for r in blk["resnets"]:
                t = ops.conv3x3_relu(x, *r["block1"])
                w2, b2 = r["block2"]
                x = ops.gemm(t.view(n * h * wd, c), w2, bias=b2, residual=x.view(n * h * wd, c)).view(n, h, wd, c)
            feats.append(x)
        if scale != 1.0:
            feats = [ops.scale_f16(f, scale, out=f) for f in feats]
        if as_nchw:
            feats = [f.permute(0, 3, 1, 2).contiguous() for f in feats]
        return feats

    __call__ = forward
