"""References for sampling from noise: restatements of the diffusers 0.19.3 pieces the reference pipeline calls
(`DDIMScheduler.step` with eta and a generator, `_get_variance`, `rescale_noise_cfg`, `randn_tensor`, and the
pipeline's `prepare_latents`), an independent closed-form fp64 statement of the same step, and the per-element check of
the fused CFG + rescale + stochastic-DDIM kernel (`cfg_ddim_rescale_kernel`, through `ops.cfg_ddim_rescale_step`).

No diffusers install exists offline, so the restatements follow the published 0.19.3 sources line by line; the closed
form below is derived by hand and the CPU tests check the two against each other at all 50 timesteps.

Closed form (a_t = alphas_cumprod[t], a_p = alphas_cumprod[t - 20] or final_alpha_cumprod at the last step):
    variance = (1 - a_p) / (1 - a_t) (1 - a_t / a_p),   c_n = eta sqrt(variance),
    c_x = sqrt(a_p / a_t),   c_e = sqrt(1 - a_p - c_n^2) - sqrt(a_p (1 - a_t) / a_t),
    x' = c_x x + c_e e + c_n z.
Rescale (CFG only): e <- e (r std(e_c) / std(e) + 1 - r), unbiased standard deviations per sample.

Kernel bound (u = 2^-24).  The reference is fp64 on the kernel's own inputs with the exact coefficients.  The kernel
rounds each fp64 coefficient to fp32 (u |c| each); forms e = e_u + g (e_c - e_u) in fp32 (|dE| <= 3 u g |e_c - e_u|
+ 2 u |E|); takes the factor f from fp64 sums of its own fp32 e, whose standard deviation differs from the exact one by
at most rms(dE) (|df| <= r (s_c / s_e) rms(dE) / s_e + 2 u f); rounds e f once; and adds the three terms with at most
three roundings.  B = u (|c_x x| + |c_e E f| + |c_n z|) + |c_e| (f dE + |E| df + u |E f|) + 4 u (|c_x x| + |c_e|
|E f| + |c_n z|), times (1 + 16 u).  fp16 latents are checked by the distance from the reference to the reals that round
to the output (ddim_probes.beyond_rounding).  As in tests/ddim_probes.py the comparator allows twice the bound."""
from __future__ import annotations

import math

import torch

from tests import ddim_probes as D

U = 2.0 ** -24
TOL = 2.0


# ------------------------------------------------------------------------------------------------ diffusers 0.19.3
def randn_tensor(shape, generator=None, device=None, dtype=None, layout=None):
    """diffusers.utils.torch_utils.randn_tensor (0.19.3)."""
    rand_device = device
    batch_size = shape[0]
    layout = layout or torch.strided
    device = device or torch.device("cpu")
    if generator is not None:
        gen_device_type = generator.device.type if not isinstance(generator, list) else generator[0].device.type
        if gen_device_type != device.type and gen_device_type == "cpu":
            rand_device = "cpu"
        elif gen_device_type != device.type and gen_device_type == "cuda":
            raise ValueError(f"Cannot generate a {device} tensor from a generator of type {gen_device_type}.")
    if isinstance(generator, list):
        shape = (1,) + tuple(shape[1:])
        latents = [torch.randn(shape, generator=generator[i], device=rand_device, dtype=dtype, layout=layout)
                   for i in range(batch_size)]
        latents = torch.cat(latents, dim=0).to(device)
    else:
        latents = torch.randn(shape, generator=generator, device=rand_device, dtype=dtype, layout=layout).to(device)
    return latents


def prepare_latents(batch_size, num_channels_latents, video_length, height, width, dtype, device, generator,
                    latents=None, vae_scale_factor=8, init_noise_sigma=1.0):
    """pipeline_videoswap.py:178-202."""
    shape = (batch_size, num_channels_latents, video_length, height // vae_scale_factor, width // vae_scale_factor)
    if isinstance(generator, list) and len(generator) != batch_size:
        raise ValueError("generator list length does not match the batch size")
    if latents is None:
        latents = randn_tensor(shape, generator=generator, device=device, dtype=dtype)
    else:
        latents = latents.to(device)
    return latents * init_noise_sigma


def rescale_noise_cfg(noise_cfg, noise_pred_text, guidance_rescale=0.0):
    """diffusers' rescale_noise_cfg (Lin et al. 2023, 3.4)."""
    std_text = noise_pred_text.std(dim=list(range(1, noise_pred_text.ndim)), keepdim=True)
    std_cfg = noise_cfg.std(dim=list(range(1, noise_cfg.ndim)), keepdim=True)
    noise_pred_rescaled = noise_cfg * (std_text / std_cfg)
    return guidance_rescale * noise_pred_rescaled + (1 - guidance_rescale) * noise_cfg


class DDIMScheduler:
    """The parts of diffusers 0.19.3 DDIMScheduler the pipeline uses, with SD-1.5's scheduler config."""

    def __init__(self, dtype=torch.float32):
        betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0).to(dtype)
        self.final_alpha_cumprod = self.alphas_cumprod[0]
        self.num_train_timesteps = 1000
        self.init_noise_sigma = 1.0

    def set_timesteps(self, n):
        self.num_inference_steps = n
        ratio = self.num_train_timesteps // n
        self.timesteps = [i * ratio + 1 for i in range(n)][::-1]

    def _get_variance(self, timestep, prev_timestep):
        alpha_prod_t = self.alphas_cumprod[timestep]
        alpha_prod_t_prev = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
        beta_prod_t = 1 - alpha_prod_t
        beta_prod_t_prev = 1 - alpha_prod_t_prev
        return (beta_prod_t_prev / beta_prod_t) * (1 - alpha_prod_t / alpha_prod_t_prev)

    def step(self, model_output, timestep, sample, eta=0.0, generator=None, variance_noise=None):
        prev_timestep = timestep - self.num_train_timesteps // self.num_inference_steps
        alpha_prod_t = self.alphas_cumprod[timestep]
        alpha_prod_t_prev = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
        beta_prod_t = 1 - alpha_prod_t
        pred_original_sample = (sample - beta_prod_t ** 0.5 * model_output) / alpha_prod_t ** 0.5
        pred_epsilon = model_output
        variance = self._get_variance(timestep, prev_timestep)
        std_dev_t = eta * variance ** 0.5
        pred_sample_direction = (1 - alpha_prod_t_prev - std_dev_t ** 2) ** 0.5 * pred_epsilon
        prev_sample = alpha_prod_t_prev ** 0.5 * pred_original_sample + pred_sample_direction
        if eta > 0:
            if variance_noise is None:
                variance_noise = randn_tensor(model_output.shape, generator=generator, device=model_output.device,
                                              dtype=model_output.dtype)
            prev_sample = prev_sample + std_dev_t * variance_noise
        return prev_sample


# ------------------------------------------------------------------------------------------------ closed form (fp64)
def closed_form_coefficients(a_t: float, a_p: float, eta: float):
    """(c_x, c_e, c_n, variance) in Python floats (fp64)."""
    var = (1.0 - a_p) / (1.0 - a_t) * (1.0 - a_t / a_p)
    c_n = eta * math.sqrt(var)
    return math.sqrt(a_p / a_t), math.sqrt(1.0 - a_p - c_n * c_n) - math.sqrt(a_p * (1.0 - a_t) / a_t), c_n, var


def step_pairs():
    """[(t, a_t, a_p)] of the 50-step forward loop (ddim_probes.pairs("forward"))."""
    return D.pairs("forward")


# ------------------------------------------------------------------------------------------------ kernel reference + bound
def ref_bound(eps, x, z, g, cfg, a_t, a_p, eta, r):
    """(ref, B) in fp64 on x's device for S = x.shape[0] samples; eps [2 S, ...] (uncond block first) or [S, ...]."""
    S = x.shape[0]
    xd = x.reshape(S, -1).double()
    n = xd.shape[1]
    e2 = eps.reshape(-1, n).double()
    eu = e2[:S]
    c_x, c_e, c_n, _ = closed_form_coefficients(float(a_t), float(a_p), eta)
    if cfg:
        ec = e2[S:2 * S]
        d = ec - eu
        E = eu + g * d
        dE = 3 * U * g * d.abs() + 2 * U * E.abs()
    else:
        E, dE = eu, torch.zeros_like(eu)
    f = torch.ones(S, 1, dtype=torch.float64, device=xd.device)
    df = torch.zeros_like(f)
    if cfg and r > 0:
        s_c = ec.std(dim=1, keepdim=True)
        s_e = E.std(dim=1, keepdim=True)
        f = r * s_c / s_e + (1 - r)
        rms = dE.pow(2).mean(dim=1, keepdim=True).sqrt()
        df = r * (s_c / s_e) * (rms / s_e) * 1.01 + 2 * U * f.abs()
    Ef = E * f
    zd = z.reshape(S, -1).double() if z is not None else torch.zeros_like(xd)
    ref = c_x * xd + c_e * Ef + c_n * zd
    tx, te, tz = (c_x * xd).abs(), abs(c_e) * Ef.abs(), (c_n * zd).abs()
    bound = U * (tx + te + tz) + abs(c_e) * (f.abs() * dE + E.abs() * df + U * Ef.abs()) + 4 * U * (tx + te + tz)
    return ref.reshape(x.shape), (bound * (1 + 16 * U)).reshape(x.shape)


def worst_ratio(out, ref, bound) -> float:
    """Worst error / bound over all elements (fp16 outputs: the distance to the reals that round to the output)."""
    o = out.reshape(-1)
    rf = ref.reshape(-1)
    if o.dtype == torch.float16:
        lo = torch.nextafter(o, torch.full_like(o, -math.inf)).double()
        hi = torch.nextafter(o, torch.full_like(o, math.inf)).double()
        od = o.double()
        err = torch.clamp(torch.maximum((od + lo) / 2 - rf, rf - (od + hi) / 2), min=0.0)
    else:
        err = (o.double() - rf).abs()
    if not bool(torch.isfinite(err).all()):
        return math.inf
    return (err / bound.reshape(-1).clamp_min(1e-300)).max().item()


def inputs(S, shape, dtype, cfg, seed, device="cpu"):
    """(eps, x, z) for S samples of `shape` (C, F, h, w).  Sample s has its own scale (1, 0.5, ...) so the samples'
    statistics differ; the conditional prediction differs from the unconditional one by ~0.3 N(0, 1)."""
    gen = torch.Generator().manual_seed(seed)
    full = (S,) + tuple(shape)
    scale = torch.tensor([0.5 ** s for s in range(S)]).view(S, *([1] * len(shape)))
    x = 2 * torch.randn(full, generator=gen)
    eu = torch.randn(full, generator=gen) * scale
    ec = eu + 0.3 * torch.randn(full, generator=gen) * scale
    z = torch.randn(full, generator=gen)
    eps = torch.cat([eu, ec]) if cfg else eu
    return eps.to(dtype).to(device), x.to(dtype).to(device), z.to(dtype).to(device)


def check_schedule(step, S, shape, dtype, cfg, eta, r, g=7.5, seed=0, device="cpu", noise=True):
    """step(eps, x, z, g, cfg, a_t, a_p, eta, r) -> out at every step of the 50-step loop against ref_bound.
    Returns {"err": worst ratio, "ok", "what"}."""
    eps, x, z = inputs(S, shape, dtype, cfg, seed, device)
    if not noise:
        z = None
    worst, where = 0.0, None
    for t, a_t, a_p in step_pairs():
        out = step(eps, x, z, g, cfg, a_t, a_p, eta, r)
        ref, bound = ref_bound(eps, x, z, g, cfg, a_t, a_p, eta, r)
        q = worst_ratio(out, ref, bound)
        if not q <= worst:
            worst, where = q, t
    what = (f"S {S} {tuple(shape)} {str(dtype)[6:]} cfg {int(cfg)} eta {eta} r {r}: worst err / bound {worst:.3g} "
            f"at t = {where}")
    return {"err": worst, "ok": worst <= TOL, "what": what}
