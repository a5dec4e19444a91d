"""Per-element checks of the fused classifier-free-guidance + DDIM update (`cfg_ddim_kernel` in pointwise.cu, through
`vs_cfg_ddim_step` / `vs_cfg_ddim_step_dev`) at every (a_t, a_p) the denoising and inversion loops use.  Kernel-agnostic:
the step is a callable step(eps, x, g, cfg, a_t, a_p) -> out and the alphas come from a provider alphas(schedule, t), so
the same checks run the CUDA kernel with the project's schedulers (tests/test_ddim_probes_gpu.py) and a torch emulation
of the kernel's arithmetic with planted bugs (tests/test_ddim_probes_cpu.py).

Schedules (`pairs`).  The SD-1.5 table alphas_cumprod (scaled_linear betas 0.00085 -> 0.012 over 1000 steps, fp32, as
diffusers computes it) is restated here, and with it the index arithmetic of the three loops, so a wrong table entry
or end-of-table alpha in the project's schedulers shows:
  * "forward": DDIMScheduler, 50 steps at t = 981, 961, ..., 1, a_t = ac[t], a_p = ac[t - 20]; the last step (t = 1) goes
    to final_alpha_cumprod = ac[0] (set_alpha_to_one False);
  * "inverse_0.19.3": t = 1, 21, ..., 981, a_t = ac[t], a_p = ac[t + 20]; the last step runs past the table to ac[999];
  * "inverse_0.21": t = 1, ..., 981, a_t = ac[t - 20], a_p = ac[t]; the first step starts before the table, at ac[0].

Reference.  fp64 on the kernel's own inputs, with a_t and a_p rounded to fp32 as the C ABI passes them:
    c_x = sqrt(a_p) / sqrt(a_t),  c_e = T1 - T2,  T1 = sqrt(1 - a_p),  T2 = sqrt(a_p) sqrt(1 - a_t) / sqrt(a_t),
    E = eu + g (ec - eu) (E = eu without CFG),  ref = c_x x + c_e E.

Bound (u = 2^-24; every fp32 operation rounds once, |delta| <= u).  The library evaluates the coefficients in fp32
(pointwise.cu cfg_ddim_step):
  * c_x: two square roots and a division:  |dc_x| <= 3 u c_x.
  * c_e: T1 takes the rounding of 1 - a_p (halved by the root) and the root's own: 1.5 u T1; T2 takes three roots, the
    rounding of 1 - a_t (halved), a product and a division: 5.5 u T2; the subtraction adds u |c_e|.  The error is bounded
    by the magnitudes of the two TERMS, not by |c_e|: at the last forward step they cancel to 1 part in ~30.
    |dc_e| <= (1.5 T1 + 5.5 T2 + |c_e|) u.  Coefficients computed in fp64 and rounded to fp32 (`ops.ddim_coefficients`,
    the graphed step) are within u |c| of the exact ones, inside the same bound.
  * the guidance lerp e = eu + g (ec - eu): the difference, the product (or an FMA) and the sum:
    |dE| <= (2 u + u^2) g |ec - eu| (1 + u) + u |E|.
  * the two-term update c_x x + c_e e (with or without an FMA): (2 u + u^2) (|c_x x| + |c_e e|) with the kernel's c_e, e.
Summing, B32 = |dc_x| |x| + |dc_e| (|E| + |dE|) + |c_e| |dE| + (2 u + u^2) (1 + 4 u) (|c_x x| + (|c_e| + |dc_e|) (|E| + |dE|)),
with each constant rounded up by 0.5 u to absorb the second-order terms.  fp32 latents: |out - ref| <= B32.  fp16
latents: the fp32 value v (|v - ref| <= B32) is rounded to nearest, so out must be the rounding of some v in
[ref - B32, ref + B32]; the reported error is the distance from ref to the set of reals that round to out
(`beyond_rounding`).  Every check reports the worst error / B32; as in tests/step_probes.py the comparator allows twice
the bound (ratio <= 2), and the emulation of the kernel's arithmetic stays within the bound itself (ratio <= 1, half the
comparator's allowance).  The bound is tight to a factor of ~1.5: at t = 701 the library's fp32 c_x is 1.7 u c_x off,
and with the product and sum roundings the emulation reaches 0.58 of B32 there (0.65 at worst over the schedules)."""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
TRAIN_STEPS, STEPS = 1000, 50
RATIO = TRAIN_STEPS // STEPS
SCHEDULES = ("forward", "inverse_0.19.3", "inverse_0.21")
TOL = 2.0            # the comparator: worst error / B32 <= 2


def alphas_cumprod() -> torch.Tensor:
    """SD-1.5's table: scaled_linear betas in fp32 and their cumulative product, as diffusers computes it."""
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, TRAIN_STEPS, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def pairs(schedule: str):
    """[(t, a_t, a_p)] of the 50 steps of one loop, in loop order (see the module docstring)."""
    ac = alphas_cumprod().tolist()
    leading = [i * RATIO + 1 for i in range(STEPS)]
    if schedule == "forward":
        return [(t, ac[t], ac[t - RATIO] if t - RATIO >= 0 else ac[0]) for t in leading[::-1]]
    if schedule == "inverse_0.19.3":
        return [(t, ac[t], ac[t + RATIO] if t + RATIO < TRAIN_STEPS else ac[-1]) for t in leading]
    if schedule == "inverse_0.21":
        return [(t, ac[t - RATIO] if t - RATIO >= 0 else ac[0], ac[t]) for t in leading]
    raise ValueError(schedule)


def library_coefficients(a_t: float, a_p: float):
    """(c_x, c_e) as the library evaluates them from the fp32 alphas (pointwise.cu cfg_ddim_step), as fp32 scalars."""
    at, ap, one = np.float32(a_t), np.float32(a_p), np.float32(1.0)
    c_x = np.sqrt(ap) / np.sqrt(at)
    c_e = np.sqrt(one - ap) - np.sqrt(ap) * np.sqrt(one - at) / np.sqrt(at)
    return np.float32(c_x), np.float32(c_e)


# ------------------------------------------------------------------------------------------------ reference and bound
def ddim_ref_bound(eps, x, g, cfg, a_t, a_p):
    """(ref, B32) in fp64 on eps's device; eps is [2 n] (uncond | cond) with CFG, else [n]."""
    at, ap = float(np.float32(a_t)), float(np.float32(a_p))
    sa, sp = math.sqrt(at), math.sqrt(ap)
    c_x = sp / sa
    t1, t2 = math.sqrt(1.0 - ap), sp * math.sqrt(1.0 - at) / sa
    c_e = t1 - t2
    n = x.numel()
    xd = x.reshape(-1).double()
    eu = eps.reshape(-1)[:n].double()
    if cfg:
        d = eps.reshape(-1)[n:2 * n].double() - eu
        E = eu + g * d
        dE = (2 * U + U * U) * (1 + U) * (1 + U) * g * d.abs() + 1.5 * U * E.abs()
    else:
        E, dE = eu, torch.zeros_like(eu)
    dcx = 3.5 * U * c_x
    dce = (2.0 * t1 + 6.0 * t2 + 1.5 * abs(c_e)) * U
    ref = c_x * xd + c_e * E
    ea = E.abs() + dE
    bound = dcx * xd.abs() + dce * ea + abs(c_e) * dE + (2 * U + U * U) * (1 + 4 * U) * (c_x * xd.abs() + (abs(c_e) + dce) * ea)
    return ref, bound * (1 + 8 * U)


def beyond_rounding(out: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    """fp16 out: the distance (fp64) from ref to the interval of reals that round to out (0 if ref rounds to out).
    fp32 out: |out - ref|.  Computed on the CPU."""
    out, ref = out.cpu(), ref.cpu()
    if out.dtype != torch.float16:
        return (out.double() - ref).abs()
    o = out.reshape(ref.shape)
    lo = torch.nextafter(o, torch.full_like(o, -math.inf)).double()
    hi = torch.nextafter(o, torch.full_like(o, math.inf)).double()
    od = o.double()
    return torch.clamp(torch.maximum((od + lo) / 2 - ref, ref - (od + hi) / 2), min=0.0)


def _ratio(err, bound):
    if not bool(torch.isfinite(err).all()):
        return math.inf
    return (err / bound.cpu().clamp_min(1e-300)).max().item()


# ------------------------------------------------------------------------------------------------ inputs
def inputs(n, dtype, cfg, seed, device="cpu"):
    """(eps, x): x ~ 2 N(0, 1) (latents in mid-loop), eps ~ N(0, 1); the conditional half differs from the unconditional
    one by ~0.3 N(0, 1), as a guided prediction does.  Without CFG eps is the first n elements of a [2 n] buffer whose
    second half is distinct, so a launch that reads eps[n + i] reads in-bounds values that differ."""
    gen = torch.Generator().manual_seed(seed)
    x = (2 * torch.randn(n, generator=gen)).to(dtype)
    eu = torch.randn(n, generator=gen)
    ec = eu + 0.3 * torch.randn(n, generator=gen)
    buf = torch.cat([eu, ec]).to(dtype).to(device)
    return (buf if cfg else buf[:n]), x.to(device)


def check_schedule(step, alphas, schedule, dtype, cfg, n, g=7.5, seed=0, device="cpu"):
    """Runs step(eps, x, g, cfg, a_t, a_p) at every step of `schedule` with the alphas the provider gives, against the
    reference at the restated alphas.  Returns {"err": worst error / B32, "ok", "what"}."""
    eps, x = inputs(n, dtype, cfg, seed, device)
    worst, where = 0.0, None
    for t, a_t, a_p in pairs(schedule):
        got_t, got_p = alphas(schedule, t)
        out = step(eps, x, g, cfg, got_t, got_p)
        ref, bound = ddim_ref_bound(eps, x, g, cfg, a_t, a_p)
        r = _ratio(beyond_rounding(out.reshape(-1), ref), bound)
        if not r <= worst:
            worst, where = r, t
    what = f"{schedule} {str(dtype)[6:]} cfg {int(cfg)} n {n}: worst err / bound {worst:.3g} at t = {where}"
    return {"err": worst, "ok": worst <= TOL, "what": what}


def check_coefficients(step_coef, schedule, dtype, cfg, n, coefficients, g=7.5, seed=0, device="cpu"):
    """step_coef(eps, x, g, cfg, c_x, c_e) with coefficients(a_t, a_p) -> (c_x, c_e): the device-coefficient launch
    at every step of `schedule`, against the reference and its bound."""
    eps, x = inputs(n, dtype, cfg, seed, device)
    worst, where = 0.0, None
    for t, a_t, a_p in pairs(schedule):
        c_x, c_e = coefficients(a_t, a_p)
        out = step_coef(eps, x, g, cfg, c_x, c_e)
        ref, bound = ddim_ref_bound(eps, x, g, cfg, a_t, a_p)
        r = _ratio(beyond_rounding(out.reshape(-1), ref), bound)
        if not r <= worst:
            worst, where = r, t
    what = f"{schedule} {str(dtype)[6:]} cfg {int(cfg)} n {n} (device coefficients): worst err / bound {worst:.3g} at t = {where}"
    return {"err": worst, "ok": worst <= TOL, "what": what}
