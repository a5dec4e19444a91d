"""Gaussian draws with the semantics of diffusers 0.19.3 `randn_tensor` (utils/torch_utils.py), which the reference
calls for the initial latents (pipeline_videoswap.py:178-202), the VAE posterior sample and the stochastic DDIM step:
the draw happens on the generator's device when that is the CPU and is then moved, a list of generators draws one batch
row each, and a CUDA generator cannot fill a tensor for another device type."""
from __future__ import annotations

import torch


def randn_tensor(shape, generator=None, device=None, dtype=None) -> torch.Tensor:
    """A contiguous standard normal tensor of `shape` on `device`, drawn exactly as randn_tensor draws it for `generator`
    (None, a torch.Generator, or a list of shape[0] of them)."""
    shape = tuple(shape)
    device = torch.device(device) if device is not None else torch.device("cpu")

    def draw(g, shp):
        rdev = device
        if g is not None and g.device.type != device.type:
            if g.device.type != "cpu":
                raise ValueError(f"cannot draw a {device} tensor from a generator on {g.device}")
            rdev = torch.device("cpu")
        return torch.randn(shp, generator=g, device=rdev, dtype=dtype).to(device)

    if isinstance(generator, (list, tuple)):
        if len(generator) != shape[0]:
            raise ValueError(f"{len(generator)} generators for a batch of {shape[0]}")
        return torch.cat([draw(g, (1,) + shape[1:]) for g in generator]).contiguous()
    return draw(generator, shape).contiguous()
