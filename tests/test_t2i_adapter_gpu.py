"""The native T2IAdapter on the H100 (pytest -m gpu): the three kernels it adds (pixel-unshuffled image entry, 2x2
average pool, ReLU epilogue of the 3x3 conv) element by element, the whole adapter against the fp32 restatement of
diffusers' FullAdapter (tests/t2i_adapter_oracle.py), and VideoSwapPipeline.__call__ with image conditions against the
CPU oracle loop fed with the restatement's residuals, plus a GraphedStep replay with those residuals."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

from oracle import unet3d_oracle as O
from tests import t2i_adapter_oracle as TO
from tests import unet_checks as UC
from videoswap_b200 import DDIMScheduler, T2IAdapter, VideoSwapPipeline, _lib, ops, t2i_adapter_param_shapes
from videoswap_b200.pipeline import GraphedStep
from videoswap_b200.weights import seeded_state_dict

pytestmark = pytest.mark.gpu


def _u8(shape, seed):
    x = torch.randint(0, 256, shape, generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)
    x.view(-1)[:2] = torch.tensor([0, 255], dtype=torch.uint8)        # both ends of the range
    return x


def _frames(n, size, mode, seed):
    rng = np.random.default_rng(seed)
    w, h = size
    shape = (h, w) if mode == "L" else (h, w, 3)
    return [Image.fromarray(rng.integers(0, 256, shape, dtype=np.uint8), mode) for _ in range(n)]


# ------------------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("c", (1, 3))
@pytest.mark.parametrize("size", ((64, 128), (448, 768), (8, 16)), ids=lambda s: f"{s[0]}x{s[1]}")
def test_image_in_bit_exact(c, size):
    u8 = _u8((3, size[0], size[1], c), seed=c)
    out = ops.t2i_image_in(u8.cuda()).cpu()
    ref = F.pixel_unshuffle((u8.permute(0, 3, 1, 2).float() / 255).half(), 8).permute(0, 2, 3, 1)
    assert out.shape == ref.shape and torch.equal(out, ref)


@pytest.mark.parametrize("shape", ((2, 14, 24, 320), (16, 56, 96, 320), (3, 2, 2, 1280), (1, 8, 6, 8)),
                         ids=lambda s: "x".join(map(str, s)))
def test_avgpool_within_one_ulp(shape):
    x = (torch.randn(shape, generator=torch.Generator().manual_seed(1)) * 4).half()
    x[0, 0, 0, 0] = x[0, 0, 1, 0] = x[0, 1, 0, 0] = 65504.0       # fp16 max: the window's sum leaves fp16's range
    x[0, 0, 0, 1:3] = torch.tensor([-3e-7, 6e-8]).half()            # subnormals
    out = ops.avgpool2x2(x.cuda()).cpu().float()
    ref = F.avg_pool2d(x.float().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    ulp = torch.clamp(ref.abs(), min=2.0 ** -14) * 2.0 ** -10          # >= one fp16 ulp at |ref| (subnormal spacing 2^-24)
    assert ((out - ref).abs() <= ulp).all(), (out - ref).abs().max()


def _conv_ref(x, wp, b):
    """fp32 relu(conv3x3(x) + b) and the per-element magnitude sum_k |x_k w_k| + |b| of the terms."""
    co, ci = wp.shape[0], x.shape[3]
    w = wp.float().view(co, 3, 3, ci).permute(0, 3, 1, 2)
    xn = x.float().permute(0, 3, 1, 2)
    pre = F.conv2d(xn, w, b, padding=1)
    mag = F.conv2d(xn.abs(), w.abs(), b.abs(), padding=1)
    return F.relu(pre).permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1), pre.permute(0, 2, 3, 1)


@pytest.mark.parametrize("co", (64, 320, 640, 1280))
def test_relu_conv_sign_probes(co):
    """(1) Bias-only: x = 0, bias negative in even channels and positive in odd ones -> exactly relu(b); a missing ReLU
    or a ReLU applied before the bias leaves the negative channels negative.  (2) One-hot taps: a single 1 in the input,
    tap t of channel n weighted s_n (t + 1) / 8 and bias -s_n / 2, so acc + b changes sign across the taps (dyadic values,
    exact).  (3) Random operands within the per-element bound of fp32 accumulation plus one fp16 rounding."""
    dev = "cuda"
    ci, n, H, W = 64, 2, 6, 10
    sgn = torch.tensor([(-1.0) ** (k + 1) for k in range(co)])
    b = sgn * (0.25 + torch.arange(co) % 7 / 8)
    wp = torch.zeros(co, 9 * ci).half()
    out = ops.conv3x3_relu(torch.zeros(n, H, W, ci, dtype=torch.float16, device=dev), wp.to(dev), b.to(dev)).cpu()
    assert torch.equal(out, F.relu(b).half().expand(n, H, W, co)), "bias-only probe"

    x = torch.zeros(n, H, W, ci).half()
    x[1, 3, 4, 5] = 1.0
    w = torch.zeros(co, 9, ci)
    w[:, :, 5] = sgn[:, None] * (torch.arange(9)[None, :] + 1) / 8
    wp = w.reshape(co, 9 * ci).half()
    bb = -sgn / 2
    out = ops.conv3x3_relu(x.to(dev), wp.to(dev), bb.to(dev)).cpu()
    ref, _, pre = _conv_ref(x, wp, bb)
    assert (pre > 0).any() and (pre < 0).any()
    assert torch.equal(out, ref.half()), "one-hot tap probe"

    g = torch.Generator().manual_seed(co)
    x = torch.randn(n, H, W, ci, generator=g).half()
    wp = (torch.randn(co, 9 * ci, generator=g) / 24).half()
    bb = torch.randn(co, generator=g)
    out = ops.conv3x3_relu(x.to(dev), wp.to(dev), bb.to(dev)).cpu().float()
    ref, mag, pre = _conv_ref(x, wp, bb)
    # the kernel's and the CPU reference's fp32 sums each within (K + 2) u sum |terms|, then one fp16 rounding
    bound = 2 * mag * (9 * ci + 2) * 2.0 ** -24 + ref.abs() * 2.0 ** -11 + 2.0 ** -25
    assert ((out - ref).abs() <= bound).all(), (out - ref).abs().max()
    assert (out[pre < -bound] == 0).all()


def test_relu_conv_refuses_other_epilogues():
    x = torch.zeros(1, 4, 4, 64, dtype=torch.float16, device="cuda")
    wp = torch.zeros(64, 9 * 64, dtype=torch.float16, device="cuda")
    out = torch.empty_like(x)
    with pytest.raises(_lib.VSError, match="ReLU epilogue"):
        ops._gemm_ex(A=x.data_ptr(), K1=64, lda1=64, Bw=wp.data_ptr(), M=16, N=64, taps=9, nimg=1, H=4, W=4,
                     residual=x.data_ptr(), ldr=64, out=out.data_ptr(), ldc=64, mode=ops.EPI_RELU)
    with pytest.raises(_lib.VSError, match="ReLU epilogue"):
        ops._gemm_ex(A=x.data_ptr(), K1=64, lda1=64, Bw=wp[:, :64].contiguous().data_ptr(), M=16, N=64,
                     out=out.data_ptr(), ldc=64, mode=ops.EPI_RELU)


def test_scale_is_torch_fp16_multiply():
    x = (torch.randn(4, 7, 12, 320, generator=torch.Generator().manual_seed(2)) * 3).half().cuda()
    for s in (0.5, 0.7, 1.3, 4.0):
        assert torch.equal(ops.scale_f16(x, s), x * s), s
    y = x.clone()
    ops.scale_f16(y, 0.7, out=y)
    assert torch.equal(y, x * 0.7)


# ------------------------------------------------------------------------------------------------------- whole adapter
# Thresholds from fp16 rounding.  Each level's feature passes through ~2 + 4 num_res_blocks fp16 roundings (conv_in,
# in_conv, block1, block2, the residual add) of relative size <= 2^-11, and the seeded convs (weights U(+-1/sqrt(fan_in)))
# carry errors with a gain below 1, so the relative RMS error stays near sqrt(12) 2^-11 ~ 2e-3 of the features' RMS:
# about 55 dB against a range of ~6 RMS.  PSNR >= 45 dB leaves a factor ~3 in RMS error; a wrong tap, channel order or
# ReLU costs far more (tens of dB).  Per element: |out - ref| <= 2^-6 max|ref| of the level, ~ 8x the largest error the
# same rounding count gives at 4 RMS.  Measured on an H100 80GB HBM3 (700 W): 83-88 dB, max errors below 2^-9 max|ref|.
PSNR_MIN, ELEM_FRAC = 45.0, 2.0 ** -6


def _adapter(in_channels, channels=(320, 640, 1280, 1280), seed=11):
    ad = T2IAdapter(in_channels=in_channels, channels=channels, init="empty")
    sd = seeded_state_dict(t2i_adapter_param_shapes(ad.config), seed=seed)
    ad.load_state_dict(sd)
    return ad, {k: v.half().float() for k, v in sd.items()}          # the oracle sees the fp16-rounded weights


@pytest.mark.parametrize("in_channels", (3, 1))
@pytest.mark.parametrize("n,size", ((16, (768, 448)), (2, (128, 64))), ids=("16x448x768", "2x64x128"))
def test_adapter_matches_restatement(in_channels, n, size):
    ad, sd = _adapter(in_channels)
    frames = _frames(n, size, "L" if in_channels == 1 else "RGB", seed=n + in_channels)
    feats = ad(frames)
    torch.cuda.synchronize()
    x = TO.preprocess_adapter_image(frames, size[1], size[0]).half().float()
    with torch.no_grad():
        ref = TO.full_adapter(sd, x)
    for lv, (f, r) in enumerate(zip(feats, ref)):
        s = 8 * 2 ** lv
        assert tuple(f.shape) == (n, size[1] // s, size[0] // s, r.shape[1])
        o = f.float().cpu().permute(0, 3, 1, 2)
        p = UC.psnr(o, r)
        err = (o - r).abs().max().item()
        print(f"level {lv}: psnr {p:.1f} dB, max err {err:.3g} of max |ref| {r.abs().max().item():.3g}")
        assert torch.isfinite(o).all()
        assert p >= PSNR_MIN, (lv, p)
        assert err <= ELEM_FRAC * r.abs().max().item(), (lv, err)
    nchw = ad(frames, scale=0.7, as_nchw=True)
    for f, g in zip(feats, nchw):
        assert torch.equal(g, (f * 0.7).permute(0, 3, 1, 2).contiguous())


# ---------------------------------------------------------------------------------------------------------- pipeline
def test_pipeline_with_image_conditions_matches_oracle():
    """pipe(..., conditions=frames, t2i_guidance_scale=0.5, t2i_end=0.5) over a 4-step schedule (the window holds
    iterations 0-2, not 3) against the oracle loop fed with 0.5 x the restatement's features; then a GraphedStep built
    with the same residuals replays pipe.step within the UNet's run-to-run envelope (GroupNorm float atomics)."""
    m, sd = UC.get_model()
    ad, asd = _adapter(3)
    pipe = VideoSwapPipeline(m, DDIMScheduler(), adapter=ad)
    Fr, hw = 2, 8
    frames = _frames(Fr, (hw * 8, hw * 8), "RGB", seed=4)
    lat = UC.randn((1, 4, Fr, hw, hw), 21).half()
    pos, neg = UC.randn((1, 16, 77, 768), 22).half(), UC.randn((1, 16, 77, 768), 23).half()
    out = pipe(pos.cuda(), lat.cuda(), negative_prompt_embeds=neg.cuda(), conditions=frames, num_inference_steps=4,
               guidance_scale=7.5, t2i_guidance_scale=0.5, t2i_end=0.5).videos
    torch.cuda.synchronize()
    x = TO.preprocess_adapter_image(frames, hw * 8, hw * 8).half().float()
    with torch.no_grad():
        state = [0.5 * f for f in TO.full_adapter(asd, x)]
        ref = O.denoise_loop(sd, O.OracleConfig(), lat.float(), pos.float(), neg.float(), 4, 7.5, state, 0.0, 0.5)
        never = O.denoise_loop(sd, O.OracleConfig(), lat.float(), pos.float(), neg.float(), 4, 7.5, None, 0.0, 0.5)
    p, p_never = UC.psnr(out, ref), UC.psnr(out, never)
    print(f"pipeline: psnr {p:.1f} dB; against the loop without the adapter {p_never:.1f} dB")
    assert tuple(out.shape) == tuple(ref.shape) == (Fr, 4, hw, hw)
    assert p >= 40.0 and p_never < p - 3.0, (p, p_never)

    embeds = torch.cat([neg, pos]).cuda()
    res = pipe._residuals_for_cfg(ad(frames, scale=0.5), True)
    pipe.scheduler.set_timesteps(50)
    latc = lat.cuda().contiguous()
    gs = GraphedStep(pipe, latc, embeds, 7.5, residuals=res)
    for t in pipe.scheduler.timesteps[:3]:
        want = pipe.step(latc, t, embeds, 7.5, list(res))
        got = gs(latc, t).clone()
        torch.cuda.synchronize()
        assert torch.isfinite(got).all()
        assert UC.psnr(got, want) >= 60.0, (t, UC.psnr(got, want))
        latc = want.contiguous()
