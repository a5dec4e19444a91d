"""DDIM scheduler state for the denoising loop (host side only: tables and index arithmetic; the update itself is the
fused CFG+DDIM CUDA kernel).  Semantics of diffusers 0.19.3 `DDIMScheduler` as configured by SD-1.5's
scheduler_config.json, which is what the reference instantiates (test.py:77, pipeline_videoswap.py:503,587):
scaled_linear betas 0.00085 -> 0.012 over 1000 train steps, 'leading' spacing, steps_offset 1, set_alpha_to_one False,
no clipping.  eta is the caller's (0 unless given): its noise scale eta sqrt(variance(t)) enters the fused step."""
from __future__ import annotations

from typing import List

import torch


class DDIMScheduler:
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 beta_schedule: str = "scaled_linear", steps_offset: int = 1, set_alpha_to_one: bool = False):
        if beta_schedule == "scaled_linear":
            betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        elif beta_schedule == "linear":
            betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        else:
            raise ValueError(beta_schedule)
        self.num_train_timesteps = num_train_timesteps
        self.steps_offset = steps_offset
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.num_inference_steps = None
        self.timesteps: List[int] = []

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.num_train_timesteps // num_inference_steps
        self.timesteps = [int(i * ratio + self.steps_offset) for i in range(num_inference_steps)][::-1]

    def scale_model_input(self, sample, timestep=None):
        return sample

    def variance(self, timestep: int) -> float:
        """diffusers 0.19.3 `_get_variance(t, prev_t)`: (1 - a_prev) / (1 - a_t) (1 - a_t / a_prev), with
        final_alpha_cumprod as a_prev at the last step; eta sqrt(variance) is the stochastic step's noise scale."""
        a_t, a_p = self.alphas(timestep)
        return (1.0 - a_p) / (1.0 - a_t) * (1.0 - a_t / a_p)

    def alphas(self, timestep: int):
        """(alpha_cumprod[t], alpha_cumprod[prev_t]) for the step taken at `timestep`."""
        prev = int(timestep) - self.num_train_timesteps // self.num_inference_steps
        a_t = float(self.alphas_cumprod[int(timestep)])
        a_p = float(self.alphas_cumprod[prev]) if prev >= 0 else float(self.final_alpha_cumprod)
        return a_t, a_p


class DDIMInverseScheduler(DDIMScheduler):
    """x_t -> x_{t+ratio} (DDIM inversion, pipeline_videoswap.py:163,667,696: built with
    `DDIMInverseScheduler.from_config(scheduler.config)`).

    diffusers changed this scheduler's index convention after the release the reference pins (requirements.txt:2,
    diffusers==0.19.3), so it is a constructor switch:
      * "0.19.3" (default = the pinned release): timesteps ascend 1, 21, ..., 981; the step taken at `t` evaluates the UNet
        at t (the level the sample is AT), uses alpha[t] for x0 and moves to alpha[t + ratio]; past the table the final
        alpha is alphas_cumprod[-1] because `set_alpha_to_one=False` of the SD config maps onto `set_alpha_to_zero=False`.
      * "0.21": the later convention -- the UNet is evaluated at the TARGET timestep t, the sample sits at t - ratio.
    No diffusers install exists offline, so both are restated from the published sources ('parity unpinned', DESIGN.md)."""

    def __init__(self, *a, convention: str = "0.19.3", **k):
        super().__init__(*a, **k)
        if convention not in ("0.19.3", "0.21"):
            raise ValueError("convention must be '0.19.3' or '0.21'")
        self.convention = convention
        self.last_alpha_cumprod = self.alphas_cumprod[-1]

    def set_timesteps(self, num_inference_steps: int, device=None):
        super().set_timesteps(num_inference_steps, device)
        self.timesteps = self.timesteps[::-1]

    def alphas(self, timestep: int):
        """(alpha of the level the sample is at, alpha of the level it moves to) for the step taken at `timestep`."""
        ratio = self.num_train_timesteps // self.num_inference_steps
        if self.convention == "0.19.3":
            nxt = int(timestep) + ratio
            a_next = float(self.alphas_cumprod[nxt]) if nxt < self.num_train_timesteps else float(self.last_alpha_cumprod)
            return float(self.alphas_cumprod[int(timestep)]), a_next
        prev = int(timestep) - ratio
        a_cur = float(self.alphas_cumprod[prev]) if prev >= 0 else float(self.final_alpha_cumprod)
        return a_cur, float(self.alphas_cumprod[int(timestep)])
