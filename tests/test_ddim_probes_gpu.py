"""Per-element tests of the fused CFG + DDIM update (pytest -m gpu), with the schedules, reference and bound of
tests/ddim_probes.py: every step of the forward loop and of both inversion conventions, fp16 and fp32, with and
without CFG, at an odd n and at an n past the capped grid; the device-coefficient launch with the graphed step's fp64
coefficients (within the bound) and with the library's own fp32 expression (bit-identical to the host-alpha launch);
then one captured GraphedStep per direction replayed at all 50 timesteps against the eager loop."""
import numpy as np
import pytest
import torch

from tests import ddim_probes as D
from tests import unet_checks as UC
from videoswap_b200 import ops
from videoswap_b200.scheduler import DDIMInverseScheduler, DDIMScheduler

pytestmark = pytest.mark.gpu

# 1 300 001 elements: odd, and 2.40 times the capped grid (132 SMs x 16 blocks x 256 threads = 540 672), so every
# thread goes round the grid-stride loop at least twice and some three times
SIZES = (12_345, 1_300_001)


def _alphas():
    fwd = DDIMScheduler()
    fwd.set_timesteps(D.STEPS)
    inv = {c: DDIMInverseScheduler(convention=c) for c in ("0.19.3", "0.21")}
    for s in inv.values():
        s.set_timesteps(D.STEPS)
    return lambda schedule, t: fwd.alphas(t) if schedule == "forward" else inv[schedule.split("_")[1]].alphas(t)


def _step(eps, x, g, cfg, a_t, a_p):
    return ops.cfg_ddim_step(eps, x, g, a_t, a_p, cfg=cfg)


def _step_coef(eps, x, g, cfg, c_x, c_e):
    coef = torch.tensor([float(c_x), float(c_e)], dtype=torch.float32, device="cuda")
    return ops.cfg_ddim_step(eps, x, g, cfg=cfg, coef=coef)


@pytest.mark.parametrize("schedule", D.SCHEDULES)
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("cfg", [True, False])
@pytest.mark.parametrize("n", SIZES)
def test_cfg_ddim_every_timestep_within_bound(schedule, dtype, cfg, n):
    r = D.check_schedule(_step, _alphas(), schedule, dtype, cfg, n, seed=n % 97, device="cuda")
    print(r["what"])
    assert r["ok"], r["what"]


@pytest.mark.parametrize("schedule", D.SCHEDULES)
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("cfg", [True, False])
def test_device_coefficients_within_bound(schedule, dtype, cfg):
    """The graphed step's coefficients: ops.ddim_coefficients in fp64, rounded to fp32 on upload."""
    r = D.check_coefficients(_step_coef, schedule, dtype, cfg, SIZES[1], ops.ddim_coefficients, seed=3, device="cuda")
    print(r["what"])
    assert r["ok"], r["what"]


@pytest.mark.parametrize("schedule", D.SCHEDULES)
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_device_coefficients_bit_identical_to_host_alphas(schedule, dtype):
    """With (c_x, c_e) from the library's own fp32 expression, vs_cfg_ddim_step_dev equals vs_cfg_ddim_step bit for bit
    at every step, with and without CFG."""
    view = torch.int16 if dtype == torch.float16 else torch.int32
    for cfg in (True, False):
        eps, x = D.inputs(SIZES[0], dtype, cfg, 5, device="cuda")
        for t, a_t, a_p in D.pairs(schedule):
            host = _step(eps, x, 7.5, cfg, a_t, a_p)
            dev = _step_coef(eps, x, 7.5, cfg, *D.library_coefficients(a_t, a_p))
            assert torch.equal(host.view(view), dev.view(view)), (schedule, t, cfg)


# ------------------------------------------------------------------------------------------------ GraphedStep
def _eager_inverse(pipe, lat, t, emb):
    """The body of VideoSwapPipeline.invert at timestep t."""
    eps = pipe.unet(lat, t, encoder_hidden_states=emb, return_dict=False)[0]
    a_cur, a_next = pipe.inverse_scheduler.alphas(t)
    return ops.cfg_ddim_step(eps, lat, 1.0, a_cur, a_next, cfg=False)


@pytest.mark.parametrize("inverse", [False, True])
def test_graphed_step_every_timestep(inverse):
    """One captured graph replayed at all 50 timesteps of its loop, each replay fed the eager loop's latents for that
    step: >= 60 dB against the eager step (the GroupNorm statistics' float-atomic order is the only difference)."""
    from videoswap_b200 import VideoSwapPipeline
    from videoswap_b200.pipeline import GraphedStep
    m, _ = UC.get_model()
    pipe = VideoSwapPipeline(m, DDIMScheduler(), inverse_scheduler=DDIMInverseScheduler())
    pipe.scheduler.set_timesteps(D.STEPS)
    pipe.inverse_scheduler.set_timesteps(D.STEPS)
    lat = UC.randn((1, 4, 2, 8, 8), 41).half().cuda()
    emb = UC.randn((2, 16, 77, 768), 42).half().cuda()
    if inverse:
        emb = emb[1:2].contiguous()
        g = GraphedStep(pipe, lat, emb, 1.0, inverse=True)
        timesteps = pipe.inverse_scheduler.timesteps
    else:
        g = GraphedStep(pipe, lat, emb, 7.5)
        timesteps = pipe.scheduler.timesteps
    assert len(timesteps) == D.STEPS
    worst = float("inf")
    for t in timesteps:
        ref = _eager_inverse(pipe, lat, t, emb) if inverse else pipe.step(lat, t, emb, 7.5)
        out = g(lat, t).clone()
        torch.cuda.synchronize()
        assert torch.isfinite(out).all(), t
        p = UC.psnr(out, ref)
        worst = min(worst, p)
        assert p >= 60.0, (t, p)
        lat = ref.contiguous()
    print(f"\n{'inverse' if inverse else 'forward'} graph: worst {worst:.1f} dB over {len(timesteps)} replays, "
          f"final |latents| max {float(lat.abs().max()):.3g}")
    assert np.isfinite(worst)
