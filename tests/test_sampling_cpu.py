"""Sampling from noise without a GPU: the diffusers 0.19.3 restatements of tests/sampling_ref.py against the
independent fp64 closed form at all 50 timesteps, the project's coefficients, variance and noise helper against them,
the argument checks of VideoSwapPipeline.__call__ and of the C ABI, and a torch emulation of the fused kernel's
arithmetic -- with planted bugs -- through the same per-element check the GPU tests use."""
import ctypes as C
import math

import pytest
import torch

from tests import sampling_ref as R
from videoswap_b200 import _lib, ops
from videoswap_b200.noise import randn_tensor
from videoswap_b200.pipeline import VideoSwapPipeline
from videoswap_b200.scheduler import DDIMScheduler
from videoswap_b200.unet import AnimateDiffUNet3DModel

ETAS = (0.0, 0.5, 1.0)


@pytest.mark.parametrize("eta", ETAS)
def test_diffusers_step_matches_closed_form_every_timestep(eta):
    """DDIMScheduler.step(eta, variance_noise) and _get_variance in fp64 == the closed form, including the last step
    (prev_t < 0 -> final_alpha_cumprod)."""
    sch = R.DDIMScheduler(dtype=torch.float64)
    sch.set_timesteps(50)
    gen = torch.Generator().manual_seed(1)
    x, e, z = (torch.randn(2, 4, 3, 5, 7, generator=gen, dtype=torch.float64) for _ in range(3))
    seen_last = False
    for t in sch.timesteps:
        prev = t - 20
        a_t = float(sch.alphas_cumprod[t])
        a_p = float(sch.alphas_cumprod[prev]) if prev >= 0 else float(sch.final_alpha_cumprod)
        seen_last |= prev < 0
        c_x, c_e, c_n, var = R.closed_form_coefficients(a_t, a_p, eta)
        assert math.isclose(float(sch._get_variance(t, prev)), var, rel_tol=1e-12)
        got = sch.step(e, t, x, eta=eta, variance_noise=z)
        want = c_x * x + c_e * e + c_n * z
        assert torch.allclose(got, want, rtol=1e-11, atol=1e-12), (t, (got - want).abs().max().item())
    assert seen_last


def test_diffusers_step_draws_its_noise_from_the_generator():
    """step(eta, generator) == step(eta, variance_noise = randn_tensor(shape, generator)) for the same seed."""
    sch = R.DDIMScheduler()
    sch.set_timesteps(50)
    x, e = torch.randn(1, 4, 2, 6, 6), torch.randn(1, 4, 2, 6, 6)
    a = sch.step(e, 981, x, eta=1.0, generator=torch.Generator().manual_seed(7))
    b = sch.step(e, 981, x, eta=1.0, variance_noise=torch.randn(x.shape, generator=torch.Generator().manual_seed(7)))
    assert torch.equal(a, b)


@pytest.mark.parametrize("r", (0.0, 0.7, 1.0))
def test_rescale_noise_cfg_matches_closed_form(r):
    gen = torch.Generator().manual_seed(2)
    text = torch.randn(2, 4, 3, 5, 7, generator=gen, dtype=torch.float64) * torch.tensor([1.0, 1e-3]).view(2, 1, 1, 1, 1)
    cfg = text * 3.0 + torch.randn(2, 4, 3, 5, 7, generator=gen, dtype=torch.float64)
    got = R.rescale_noise_cfg(cfg, text, r)
    for s in range(2):   # independent: numpy-free per-sample Bessel std
        n = text[s].numel()
        sd = lambda v: math.sqrt(float(((v - v.mean()) ** 2).sum()) / (n - 1))   # noqa: E731
        f = r * sd(text[s]) / sd(cfg[s]) + (1 - r)
        assert torch.allclose(got[s], cfg[s] * f, rtol=1e-12, atol=0)


def test_scheduler_variance_and_coefficients_match_the_restatement():
    """scheduler.DDIMScheduler.variance == _get_variance on the same fp32 table evaluated in fp64 (diffusers' own fp32
    evaluation loses ~1e-5 to cancellation at the last step); ops.ddim_coefficients(eta) == the closed form at every
    step; at eta = 0 its first two values are bit-equal to the two-value call (today's)."""
    ours, ref, ref32 = DDIMScheduler(), R.DDIMScheduler(dtype=torch.float64), R.DDIMScheduler()
    ours.set_timesteps(50)
    ref.set_timesteps(50)
    assert ours.timesteps == ref.timesteps
    for t in ours.timesteps:
        prev = t - 20
        assert math.isclose(ours.variance(t), float(ref._get_variance(t, prev)), rel_tol=1e-12)
        assert math.isclose(ours.variance(t), float(ref32._get_variance(t, prev)), rel_tol=1e-4)
        a_t, a_p = ours.alphas(t)
        two = ops.ddim_coefficients(a_t, a_p)
        zero = ops.ddim_coefficients(a_t, a_p, 0.0)
        assert len(two) == 2 and zero[:2] == two and zero[2] == 0.0
        old_x = math.sqrt(a_p) / math.sqrt(a_t)
        old_e = math.sqrt(1.0 - a_p) - math.sqrt(a_p) * math.sqrt(1.0 - a_t) / math.sqrt(a_t)
        assert two == (old_x, old_e)
        for eta in (0.5, 1.0):
            c = ops.ddim_coefficients(a_t, a_p, eta)
            want = R.closed_form_coefficients(a_t, a_p, eta)[:3]
            for got_c, want_c in zip(c, want):
                assert math.isclose(got_c, want_c, rel_tol=1e-12, abs_tol=1e-15)
            assert math.isclose(c[2], eta * math.sqrt(ours.variance(t)), rel_tol=1e-12)
    with pytest.raises(ValueError):
        ops.ddim_coefficients(0.5, 0.6, -0.1)


def test_noise_helper_draws_torch_randn():
    shape = (3, 4, 2, 5, 6)
    for dtype in (torch.float32, torch.float16):
        got = randn_tensor(shape, torch.Generator().manual_seed(11), "cpu", dtype)
        assert torch.equal(got, torch.randn(shape, generator=torch.Generator().manual_seed(11), dtype=dtype))
        gens = [torch.Generator().manual_seed(s) for s in (3, 4, 5)]
        got = randn_tensor(shape, gens, "cpu", dtype)
        want = torch.cat([torch.randn((1,) + shape[1:], generator=torch.Generator().manual_seed(s), dtype=dtype)
                          for s in (3, 4, 5)])
        assert torch.equal(got, want)
        ref = R.randn_tensor(shape, [torch.Generator().manual_seed(s) for s in (3, 4, 5)], torch.device("cpu"), dtype)
        assert torch.equal(got, ref)
    with pytest.raises(ValueError):
        randn_tensor(shape, [torch.Generator()] * 2, "cpu", torch.float32)


def _pipe():
    return VideoSwapPipeline(AnimateDiffUNet3DModel(init="empty"))


def test_prepare_latents_matches_the_reference():
    pipe = _pipe()
    for gen in (lambda: torch.Generator().manual_seed(5), lambda: [torch.Generator().manual_seed(s) for s in (5, 6)]):
        got = pipe.prepare_latents(2, 3, 96, 128, torch.float16, "cpu", gen())
        want = R.prepare_latents(2, 4, 3, 96, 128, torch.float16, torch.device("cpu"), gen())
        assert got.shape == (2, 4, 3, 12, 16) and torch.equal(got, want)
    sz = pipe.unet.config.sample_size
    assert pipe.prepare_latents(1, 2, device="cpu", dtype=torch.float32).shape == (1, 4, 2, sz, sz)


def test_call_argument_errors():
    pipe = _pipe()
    emb = torch.zeros(1, 77, 768)
    with pytest.raises(ValueError, match="video_length"):
        pipe(emb, None, negative_prompt_embeds=emb)
    with pytest.raises(ValueError, match="generators"):
        pipe(emb, None, negative_prompt_embeds=emb, video_length=2, generator=[torch.Generator()] * 2)
    emb2 = torch.zeros(2, 77, 768)
    with pytest.raises(ValueError, match="one video"):
        pipe(emb2, None, negative_prompt_embeds=emb2, video_length=2, conditions={})
    with pytest.raises(ValueError, match="one video"):
        pipe(emb2, None, negative_prompt_embeds=emb2, video_length=2, controller=object())
    with pytest.raises(ValueError, match="eta"):
        pipe(emb, None, negative_prompt_embeds=emb, video_length=2, eta=-1.0)
    with pytest.raises(ValueError, match="videos"):
        pipe(emb2, torch.zeros(1, 4, 1, 8, 8), negative_prompt_embeds=emb2)
    with pytest.raises(ValueError, match="generators"):
        pipe.prepare_latents(2, 2, generator=[torch.Generator()], device="cpu")


def test_c_abi_rejects_bad_arguments_before_launching():
    """Null pointers, S = 0, eta < 0 and alphas outside (0, 1] return an error without touching the (dummy) pointers."""
    lib = _lib.lib()
    p = C.c_void_p(16)
    f = lib.vs_cfg_ddim_rescale_step
    ok = dict(eps=p, lat=p, noise=p, S=1, n=8, a_t=0.5, a_p=0.6, eta=0.5, r=0.7)

    def call(**k):
        a = {**ok, **k}
        return f(None, a["eps"], a["lat"], a["noise"], 0, a["S"], a["n"], 1, 7.5, a["a_t"], a["a_p"], a["eta"], a["r"], p)

    for bad in (dict(eps=None), dict(lat=None), dict(noise=None), dict(S=0), dict(n=0), dict(eta=-0.5),
                dict(a_t=0.0), dict(a_t=1.5), dict(a_p=-0.1), dict(a_p=1.01), dict(r=-1.0)):
        assert call(**bad) != 0, bad
    assert b"vs_cfg_ddim_rescale_step" in lib.vs_last_error()
    g = lib.vs_cfg_ddim_rescale_step_dev
    assert g(None, p, p, None, 0, 1, 8, 1, 7.5, None, p) != 0                    # no coefficient vector
    assert g(None, p, p, None, 0, 0, 8, 1, 7.5, p, p) != 0                       # S = 0
    assert g(None, None, p, None, 0, 1, 8, 1, 7.5, p, p) != 0


# ------------------------------------------------------------------------------------------------ emulated kernel
def _emulate(bug=None):
    """The kernel's arithmetic in torch: fp32 guidance lerp, fp64 per-sample statistics of its own fp32 e (shifted),
    fp32 factor and update, coefficients from ops.ddim_coefficients rounded to fp32.  `bug` plants one mistake."""
    def step(eps, x, z, g, cfg, a_t, a_p, eta, r):
        S = x.shape[0]
        n = x[0].numel()
        e2 = eps.reshape(-1, n).float()
        eu = e2[:S]
        e = eu + g * (e2[S:] - eu) if cfg else eu
        c_x, c_e, c_n = (torch.tensor(v, dtype=torch.float32) for v in ops.ddim_coefficients(a_t, a_p, eta))
        if bug == "cn_variance":
            c_n = torch.tensor(eta * ((1 - a_p) / (1 - a_t) * (1 - a_t / a_p)), dtype=torch.float32)
        f = torch.ones(S, 1, dtype=torch.float32)
        if cfg and r > 0:
            ec = e2[S:]
            if bug == "naive_fp32":
                def sd(v):
                    s, q = v.sum(1, keepdim=True), (v * v).sum(1, keepdim=True)
                    return ((q - s * s / n) / (n - 1)).clamp_min(0).sqrt().double()
            else:
                def sd(v):
                    d = v.double() - v[:, :1].double()
                    return ((d.pow(2).sum(1, keepdim=True) - d.sum(1, keepdim=True) ** 2 / n) / (n - 1)).sqrt()
            if bug == "pooled":
                sc, se = sd(ec.reshape(1, -1)).expand(S, 1), sd(e.reshape(1, -1)).expand(S, 1)
            else:
                sc, se = sd(ec), sd(e)
            f = (r * (sc / se) + (1 - r)).float()
        out = c_x * x.reshape(S, n).float() + c_e * (e * f)
        if z is not None:
            zz = z.reshape(S, n).float()
            if bug == "noise_shift":
                zz = torch.roll(zz, 1, dims=1)
            out = out + c_n * zz
        return out.to(x.dtype).reshape(x.shape)
    return step


@pytest.mark.parametrize("dtype", (torch.float16, torch.float32))
@pytest.mark.parametrize("cfg", (True, False))
@pytest.mark.parametrize("eta,r", ((0.5, 0.0), (1.0, 0.7), (0.5, 1.0)))
def test_emulated_kernel_within_bound(dtype, cfg, eta, r):
    res = R.check_schedule(_emulate(), 2, (4, 2, 9, 11), dtype, cfg, eta, r, seed=3)
    assert res["err"] <= 1.0, res["what"]


def _probe_pooled(step):
    """Two samples with spreads 1 and 1e-3: statistics pooled across samples give the second one the wrong factor."""
    gen = torch.Generator().manual_seed(9)
    shape = (2, 4, 2, 9, 11)
    sc = torch.tensor([1.0, 1e-3]).view(2, 1, 1, 1, 1)
    eu = torch.randn(shape, generator=gen) * sc
    ec = eu + 0.3 * torch.randn(shape, generator=gen) * sc
    x = torch.randn(shape, generator=gen) * sc
    eps = torch.cat([eu, ec])
    return _ratio_at(step, eps, x, None, 0.0, 1.0)


def _probe_mean(step):
    """Mean 1e3 with spread 1 (fp32): naive fp32 sums lose the variance to cancellation."""
    gen = torch.Generator().manual_seed(10)
    shape = (1, 4, 8, 32, 32)
    eu = 1e3 + torch.randn(shape, generator=gen)
    ec = 1e3 + 1.2 * torch.randn(shape, generator=gen)
    x = torch.randn(shape, generator=gen)
    return _ratio_at(step, torch.cat([eu, ec]), x, None, 0.0, 0.7)


def _probe_onehot(step, dtype=torch.float32):
    """One-hot noise in sample 1: a wrong c_n or a wrong noise index moves the output by ~c_n at that element."""
    gen = torch.Generator().manual_seed(12)
    shape = (2, 4, 2, 9, 11)
    x = torch.randn(shape, generator=gen).to(dtype)
    eu = torch.randn(shape, generator=gen)
    eps = torch.cat([eu, eu + 0.3 * torch.randn(shape, generator=gen)]).to(dtype)
    z = torch.zeros(shape, dtype=dtype)
    z[1, 2, 1, 4, 7] = 1.0
    return _ratio_at(step, eps, x, z, 1.0, 0.0)


def _ratio_at(step, eps, x, z, eta, r, g=7.5):
    worst = 0.0
    for t, a_t, a_p in R.step_pairs()[::7]:
        out = step(eps.to(x.device), x, z, g, True, a_t, a_p, eta, r)
        ref, bound = R.ref_bound(eps.to(x.device), x, z, g, True, a_t, a_p, eta, r)
        worst = max(worst, R.worst_ratio(out, ref, bound))
    return worst


PROBES = {"pooled": _probe_pooled, "naive_fp32": _probe_mean, "cn_variance": _probe_onehot, "noise_shift": _probe_onehot}


@pytest.mark.parametrize("bug", sorted(PROBES))
def test_probes_fail_a_wrong_kernel(bug):
    probe = PROBES[bug]
    assert probe(_emulate()) <= 1.0
    assert probe(_emulate(bug)) > 10 * R.TOL, bug
