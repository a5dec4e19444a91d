"""Sampling from noise on the H100 (pytest -m gpu): the fused CFG + rescale + stochastic-DDIM kernel
(ops.cfg_ddim_rescale_step) element by element against fp64 at every timestep (tests/sampling_ref.py), the probes that
a wrong kernel fails, bit-reproducibility (repeat launches, device against host coefficients, graph replay), and
VideoSwapPipeline.__call__ from noise against the CPU oracle loop with the same draws."""
import pytest
import torch

from oracle import unet3d_oracle as O
from tests import sampling_ref as R
from tests import unet_checks as UC
from tests.test_sampling_cpu import PROBES, _emulate
from videoswap_b200 import ops
from videoswap_b200.noise import randn_tensor
from videoswap_b200.pipeline import GraphedStep, VideoSwapPipeline
from videoswap_b200.scheduler import DDIMScheduler

pytestmark = pytest.mark.gpu

SHAPES = ((4, 16, 64, 64), (4, 16, 56, 96), (4, 3, 45, 60))


def _host_step(eps, x, z, g, cfg, a_t, a_p, eta, r):
    return ops.cfg_ddim_rescale_step(eps, x, g, a_t, a_p, eta=eta, guidance_rescale=r, noise=z, cfg=cfg)


def _dev_step(eps, x, z, g, cfg, a_t, a_p, eta, r):
    c_x, c_e, c_n = ops.ddim_coefficients(a_t, a_p, eta)
    coef = torch.tensor([c_x, c_e, c_n, r], dtype=torch.float32, device=x.device)
    return ops.cfg_ddim_rescale_step(eps, x, g, noise=z, cfg=cfg, coef=coef)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("S", (1, 2))
@pytest.mark.parametrize("cfg", (True, False))
@pytest.mark.parametrize("dtype", (torch.float16, torch.float32))
@pytest.mark.parametrize("r", (0.0, 0.7, 1.0))
@pytest.mark.parametrize("eta", (0.5, 1.0))
def test_kernel_every_timestep_within_bound(eta, r, dtype, cfg, S, shape):
    res = R.check_schedule(_host_step, S, shape, dtype, cfg, eta, r, seed=S + 7, device="cuda")
    print("\n" + res["what"])
    assert res["ok"], res["what"]


def _on_gpu(step):
    def run(eps, x, z, *a):
        return step(eps.cuda(), x.cuda(), None if z is None else z.cuda(), *a).cpu()
    return run


@pytest.mark.parametrize("probe", sorted(set(PROBES.values()), key=lambda p: p.__name__), ids=lambda p: p.__name__)
def test_probes_pass_the_kernel(probe):
    """Pooled statistics (spreads 1 and 1e-3), cancellation (mean 1e3, spread 1) and a one-hot noise tensor: the kernel
    stays within the bound, and the emulation of a kernel with the matching bug does not (tests/test_sampling_cpu.py)."""
    assert probe(_on_gpu(_host_step)) <= R.TOL
    assert probe(_on_gpu(_dev_step)) <= R.TOL
    for bug, p in PROBES.items():
        if p is probe:
            assert probe(_emulate(bug)) > 10 * R.TOL, bug


@pytest.mark.parametrize("dtype", (torch.float16, torch.float32))
def test_bit_reproducible_and_device_coefficients_equal_host(dtype):
    eps, x, z = R.inputs(2, SHAPES[0], dtype, True, seed=21, device="cuda")
    for t, a_t, a_p in R.step_pairs():
        a = _host_step(eps, x, z, 7.5, True, a_t, a_p, 1.0, 0.7)
        b = _host_step(eps, x, z, 7.5, True, a_t, a_p, 1.0, 0.7)
        c = _dev_step(eps, x, z, 7.5, True, a_t, a_p, 1.0, 0.7)
        assert torch.equal(a, b), t
        assert torch.equal(a, c), t


def test_kernel_graph_replay_equals_eager_loop():
    """The device-coefficient launch captured once and replayed over 10 steps, with the noise buffer filled eagerly from
    a generator before each replay, equals the eager loop with host coefficients bit for bit."""
    shape = (2,) + SHAPES[1]
    eps, x0, _ = R.inputs(2, SHAPES[1], torch.float16, True, seed=22, device="cuda")
    coef = torch.zeros(4, dtype=torch.float32, device="cuda")
    noise = torch.zeros(shape, dtype=torch.float16, device="cuda")
    lat = x0.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.cfg_ddim_rescale_step(eps, lat, 7.5, noise=noise, coef=coef)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.cfg_ddim_rescale_step(eps, lat, 7.5, noise=noise, coef=coef)
    g_eager, g_graph = torch.Generator().manual_seed(5), torch.Generator().manual_seed(5)
    ref = x0.clone()
    for t, a_t, a_p in R.step_pairs()[:10]:
        ref = _host_step(eps, ref, randn_tensor(shape, g_eager, "cuda", torch.float16), 7.5, True, a_t, a_p, 1.0, 0.7)
        c_x, c_e, c_n = ops.ddim_coefficients(a_t, a_p, 1.0)
        coef.copy_(torch.tensor([c_x, c_e, c_n, 0.7]))
        noise.copy_(randn_tensor(shape, g_graph, "cuda", torch.float16))
        graph.replay()
        lat.copy_(out)
        assert torch.equal(lat, ref), t


def test_graphed_step_with_eta_and_rescale():
    """GraphedStep(eta, guidance_rescale) replayed at 8 timesteps, fed the eager loop's latents: its noise buffer holds
    the eager draw bit for bit and the step is >= 60 dB from pipe.step (the UNet's GroupNorm atomics differ)."""
    m, _ = UC.get_model()
    pipe = VideoSwapPipeline(m, DDIMScheduler())
    pipe.scheduler.set_timesteps(50)
    lat = UC.randn((1, 4, 2, 8, 8), 41).half().cuda()
    emb = UC.randn((2, 16, 77, 768), 42).half().cuda()
    gs = GraphedStep(pipe, lat, emb, 7.5, eta=1.0, guidance_rescale=0.7)
    g_eager, g_graph, g_check = (torch.Generator().manual_seed(3) for _ in range(3))
    for t in pipe.scheduler.timesteps[:8]:
        ref = pipe.step(lat, t, emb, 7.5, eta=1.0, guidance_rescale=0.7, generator=g_eager)
        out = gs(lat, t, generator=g_graph).clone()
        torch.cuda.synchronize()
        assert torch.equal(gs.noise, randn_tensor(lat.shape, g_check, "cuda", torch.float16)), t
        assert torch.isfinite(out).all()
        assert UC.psnr(out, ref) >= 60.0, (t, UC.psnr(out, ref))
        lat = ref.contiguous()


def _oracle_loop(sd, lat0, pos, neg, steps, guidance, eta, r, gen):
    """The reference's loop in fp32 on the CPU: oracle UNet, CFG, rescale_noise_cfg, DDIMScheduler.step(eta) with the
    draw randn_tensor(shape, gen, dtype=fp16) that the fp16 pipeline makes."""
    sch = R.DDIMScheduler()
    sch.set_timesteps(50)
    x = lat0.float()
    ehs2 = torch.cat([neg, pos]).float()
    for t in sch.timesteps[:steps]:
        eps2 = O.unet_forward(sd, O.OracleConfig(), torch.cat([x] * 2), t, ehs2)
        eu, ec = eps2.chunk(2)
        e = eu + guidance * (ec - eu)
        if r > 0:
            e = R.rescale_noise_cfg(e, ec, r)
        z = R.randn_tensor(x.shape, gen, torch.device("cpu"), torch.float16).float()
        x = sch.step(e, t, x, eta=eta, variance_noise=z)
    return x


@pytest.mark.parametrize("eta,r", ((1.0, 0.7), (0.5, 0.0), (0.0, 1.0)))
def test_call_from_noise_matches_oracle(eta, r):
    m, sd = UC.get_model()
    pipe = VideoSwapPipeline(m, DDIMScheduler())
    pos, neg = UC.randn((1, 16, 77, 768), 22).half(), UC.randn((1, 16, 77, 768), 23).half()
    steps = 3
    out = pipe(pos.cuda(), None, negative_prompt_embeds=neg.cuda(), video_length=2, height=64, width=64,
               generator=torch.Generator().manual_seed(31), eta=eta, guidance_rescale=r, max_iters=steps).videos
    torch.cuda.synchronize()
    gen = torch.Generator().manual_seed(31)
    lat0 = R.prepare_latents(1, 4, 2, 64, 64, torch.float16, torch.device("cpu"), gen)
    with torch.no_grad():
        ref = _oracle_loop(sd, lat0, pos.float(), neg.float(), steps, 7.5, eta, r, gen)
    ref = ref.permute(0, 2, 1, 3, 4).reshape(out.shape)
    p = UC.psnr(out, ref)
    print(f"\n__call__ from noise, eta {eta} guidance_rescale {r}: {p:.1f} dB against the oracle")
    assert p >= 40.0, p


class _StubUNet:
    """A deterministic stand-in for the UNet: eps = 0.8 sin(1.3 x + t / 1000) + (first embedding value of the row), so
    pipeline-level checks can compare bits."""

    class config:
        sample_size = 8
        in_channels = 4

    device = torch.device("cuda")

    def __call__(self, x, t, encoder_hidden_states=None, down_block_additional_residuals=None, return_dict=False):
        B = x.shape[0]
        h = encoder_hidden_states.reshape(B, -1)[:, :1].to(x.dtype).view(B, 1, 1, 1, 1)
        return ((torch.sin(x * 1.3 + float(t) / 1000) * 0.8 + h).contiguous(),)


def _stub_embeds(b, seed):
    return UC.randn((b, 77, 768), seed).half().cuda()


def test_same_seed_same_latents_and_prompt_list_equals_single_calls():
    pipe = VideoSwapPipeline(_StubUNet(), DDIMScheduler())
    pos, neg = _stub_embeds(2, 1), _stub_embeds(2, 2)
    kw = dict(video_length=3, height=48, width=40, eta=1.0, guidance_rescale=0.7, max_iters=6)
    a = pipe(pos[:1], None, negative_prompt_embeds=neg[:1], generator=torch.Generator().manual_seed(4), **kw).videos
    b = pipe(pos[:1], None, negative_prompt_embeds=neg[:1], generator=torch.Generator().manual_seed(4), **kw).videos
    assert torch.equal(a, b)
    both = pipe(pos, None, negative_prompt_embeds=neg,
                generator=[torch.Generator().manual_seed(4), torch.Generator().manual_seed(9)], **kw).videos
    c = pipe(pos[1:], None, negative_prompt_embeds=neg[1:], generator=torch.Generator().manual_seed(9), **kw).videos
    assert both.shape == (6, 4, 6, 5)
    assert torch.equal(both[:3], a) and torch.equal(both[3:], c)
    assert not torch.equal(a, c)
    gpu_gen = torch.Generator(device="cuda").manual_seed(4)
    d = pipe(pos[:1], None, negative_prompt_embeds=neg[:1], generator=gpu_gen, **kw).videos
    assert d.shape == a.shape and torch.isfinite(d).all()


def test_cuda_generator_with_cpu_target_raises():
    with pytest.raises(ValueError, match="generator"):
        randn_tensor((1, 4, 2, 8, 8), torch.Generator(device="cuda"), "cpu", torch.float32)


def test_given_latents_without_eta_or_rescale_take_the_deterministic_kernel():
    """With given latents and eta = guidance_rescale = 0 the loop is ops.cfg_ddim_step's, bit for bit."""
    pipe = VideoSwapPipeline(_StubUNet(), DDIMScheduler())
    pos, neg = _stub_embeds(1, 3), _stub_embeds(1, 4)
    lat = UC.randn((1, 4, 2, 8, 8), 5).half().cuda()
    out = pipe(pos, lat, negative_prompt_embeds=neg, max_iters=5).videos
    sch = DDIMScheduler()
    sch.set_timesteps(50)
    x = lat
    emb = torch.cat([neg, pos])
    for t in sch.timesteps[:5]:
        eps = _StubUNet()(torch.cat([x] * 2), t, emb)[0]
        x = ops.cfg_ddim_step(eps, x, 7.5, *sch.alphas(t))
    assert torch.equal(out, x.permute(0, 2, 1, 3, 4).reshape(out.shape))
