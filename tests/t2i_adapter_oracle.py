"""CPU fp32 restatement of diffusers 0.19.3's `FullAdapter` (T2IAdapter with adapter_type "full_adapter") and of
`_preprocess_adapter_image` (pipelines/t2i_adapter/pipeline_stable_diffusion_adapter.py), the checker of the native
T2IAdapter.  It is written from the published architecture with F.pixel_unshuffle / conv2d / relu / avg_pool2d; it is
NOT pinned to diffusers' own code (the reference repository ships no adapter code and diffusers is not installed here),
so it checks the native kernels against the architecture as restated, at sizes where its one uncertain detail -- the
pooling's rounding -- does not matter (frame sides that are multiples of 64 px)."""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch
import torch.nn.functional as F


def preprocess_adapter_image(images, height: int, width: int) -> torch.Tensor:
    """_preprocess_adapter_image for a list of PIL images: each resized to (width, height) with LANCZOS (PIL returns a
    copy when the size already matches), [h, w] / [h, w, c] expanded to [1, h, w, c], concatenated, / 255 in fp32 and
    transposed to NCHW."""
    from PIL import Image
    if isinstance(images, Image.Image):
        images = [images]
    arrs = [np.array(i.resize((width, height), resample=Image.LANCZOS)) for i in images]
    arrs = [a[None, ..., None] if a.ndim == 2 else a[None, ...] for a in arrs]
    x = np.concatenate(arrs, axis=0).astype(np.float32) / 255.0
    return torch.from_numpy(x.transpose(0, 3, 1, 2).copy())


def full_adapter(sd: Dict[str, torch.Tensor], x: torch.Tensor, channels=(320, 640, 1280, 1280), num_res_blocks: int = 2,
                 downscale_factor: int = 8, dtype=torch.float32) -> List[torch.Tensor]:
    """FullAdapter.forward in `dtype` (fp32 for the checker; fp16 on the GPU is torch eager's run of the module):
    unshuffle -> conv_in -> blocks (avg pool 2x2 for i > 0, in_conv where the width changes, resnets
    x + block2(relu(block1(x)))); returns the features after each block (NCHW)."""
    w = {k: v.to(dtype) for k, v in sd.items()}
    x = F.pixel_unshuffle(x.to(dtype), downscale_factor)
    x = F.conv2d(x, w["adapter.conv_in.weight"], w["adapter.conv_in.bias"], padding=1)
    feats = []
    for i in range(len(channels)):
        p = f"adapter.body.{i}"
        if i > 0:
            x = F.avg_pool2d(x, kernel_size=2, stride=2, ceil_mode=True)
        if p + ".in_conv.weight" in w:
            x = F.conv2d(x, w[p + ".in_conv.weight"], w[p + ".in_conv.bias"])
        for j in range(num_res_blocks):
            q = f"{p}.resnets.{j}"
            h = F.relu(F.conv2d(x, w[q + ".block1.weight"], w[q + ".block1.bias"], padding=1))
            x = F.conv2d(h, w[q + ".block2.weight"], w[q + ".block2.bias"]) + x
        feats.append(x)
    return feats
