"""VAE encoder tests on the GPU (pytest -m gpu): the stride-2 down-sampler conv per element against fp64 with the bound of
tests/downsample_checks.py (impulse probes and random inputs) and bit-identical to the im2col GEMM, its tile-schedule
invariance, the image-in / moments / posterior kernels, the whole encoder against tests/vae_encoder_oracle.py, per-frame
independence, seeded sampling, and DDIM inversion from video frames through the pipeline.

The encoder oracle runs in fp32 on the same GPU with TF32 off (cuDNN / cuBLAS fp32), on the same fp16-rounded weights and
input; at 512 x 512 the CPU would need minutes per frame."""
import contextlib
import math

import numpy as np
import pytest
import torch

import videoswap_b200 as V
from oracle import unet3d_oracle as O
from tests import downsample_checks as D
from tests import unet_checks as U
from tests import vae_encoder_oracle as EO
from videoswap_b200 import _lib, ops
from videoswap_b200 import vae as VAE

pytestmark = pytest.mark.gpu
UR = 2.0 ** -24


@contextlib.contextmanager
def _fp32_exact():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


# ---------------------------------------------------------------------------------------------------- stride-2 conv
DS_CASES = [(C, n, H, W) for C, sizes in (
    (128, ((5, 8, 8), (3, 64, 64), (2, 90, 120), (1, 256, 256))),
    (256, ((3, 8, 8), (2, 64, 64), (1, 90, 120), (1, 256, 256))),
    (512, ((4, 8, 8), (1, 64, 64), (2, 90, 120))),
) for n, H, W in sizes]


@pytest.mark.parametrize("case", DS_CASES, ids=lambda c: "C{}_n{}_{}x{}".format(*c))
def test_downsample_conv_per_element(case):
    """Impulses at the last row / column of every image, around the conv-tile edges and on every image of a tile, then
    random inputs: every element within the bound (twice the kernel's worst case), and bit-identical to ops.gemm on the
    tap-major im2col with the same packed weight (the same K order)."""
    C, n, H, W = case
    w, b = D.weights(C, C, seed=C + H)
    wp, wd, bd = D.pack(w).cuda(), w.cuda(), b.float().cuda()
    worst = 0.0
    for kind, x in (("impulse", D.probe_input(n, H, W, C, seed=H + n)),
                    ("random", torch.randn(n, H, W, C, generator=torch.Generator().manual_seed(W)).half())):
        x = x.cuda()
        out = ops.downsample_conv3x3(x, wp, bd)
        gem = ops.gemm(D.im2col(x).contiguous(), wp, bias=bd).view(out.shape)
        torch.cuda.synchronize()
        err, where = D.compare(out, x, wd, bd)
        worst = max(worst, err)
        print(f"\n{case} {kind}: worst err / bound {err:.3g} at flat index {where}")
        assert torch.isfinite(out).all()
        assert err <= 1.0, (kind, err, where)
        assert torch.equal(out, gem), f"{kind}: differs from the im2col GEMM"
    print(f"worst err / bound {worst:.3g}")


def _ds_problem(C, n, H, W, seed):
    w, b = D.weights(C, C, seed)
    wp, bd = D.pack(w).cuda(), b.float().cuda()
    x = torch.randn(n, H, W, C, generator=torch.Generator().manual_seed(seed)).half().cuda()
    return lambda: ops.downsample_conv3x3(x, wp, bd)


@pytest.mark.parametrize("case", [(128, 2, 64, 64), (256, 5, 8, 8), (512, 1, 90, 120)], ids=lambda c: "C{}_n{}_{}x{}".format(*c))
def test_downsample_schedule_invariance(case):
    run = _ds_problem(*case, seed=sum(case))
    try:
        ops.set_option("gemm_ctas", 0)
        ops.set_option("gemm_stages", 0)
        base = run()
        for stages in (0, 3):
            ops.set_option("gemm_stages", stages)
            for ctas in (1, 2, 3, 5, 8):
                ops.set_option("gemm_ctas", ctas)
                out = run()
                torch.cuda.synchronize()
                assert torch.equal(base, out), f"{case}: differs at gemm_ctas={ctas} gemm_stages={stages}"
    finally:
        ops.set_option("gemm_ctas", 0)
        ops.set_option("gemm_stages", 0)


def test_downsample_rejects_odd_sizes():
    x = torch.zeros(1, 10, 9, 128, dtype=torch.float16, device="cuda")
    wp = torch.zeros(128, 9 * 128, dtype=torch.float16, device="cuda")
    with pytest.raises(_lib.VSError, match="even"):
        ops.downsample_conv3x3(x, wp)


# ---------------------------------------------------------------------------------------------------- entry / exit kernels
def test_image_in_uint8_bit_exact():
    u = np.concatenate([np.arange(256, dtype=np.uint8).reshape(1, 16, 16, 1).repeat(3, 3),
                        np.random.default_rng(3).integers(0, 256, (1, 16, 16, 3), dtype=np.uint8)])
    frames = np.concatenate([u, np.random.default_rng(4).integers(0, 256, (2, 16, 16, 3), dtype=np.uint8)])
    y = frames.astype(np.float32) / 255.0                          # pil_to_numpy
    assert y.dtype == np.float32
    ref = (2.0 * torch.from_numpy(y) - 1.0).half()                 # normalize, then the fp16 cast
    out = ops.vae_image_in(torch.from_numpy(frames).cuda()).cpu()
    assert torch.equal(out[..., :3], ref) and bool((out[..., 3] == 0).all())
    big = np.random.default_rng(5).integers(0, 256, (3, 40, 56, 3), dtype=np.uint8)
    ref = (2.0 * torch.from_numpy(big.astype(np.float32) / 255.0) - 1.0).half()
    assert torch.equal(ops.vae_image_in(torch.from_numpy(big).cuda()).cpu()[..., :3], ref)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_image_in_float_bit_exact(dtype):
    x = (torch.rand(3, 3, 24, 40, generator=torch.Generator().manual_seed(6)) * 2 - 1).to(dtype).cuda()
    out = ops.vae_image_in(x)
    assert torch.equal(out[..., :3], x.half().permute(0, 2, 3, 1)) and bool((out[..., 3] == 0).all())


def test_moments_kernel():
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(3, 45, 60, 8, generator=g) * 4).half().cuda()
    wb = (torch.randn(72, generator=g) * 0.5).cuda()
    out = ops.vae_moments(x, wb)
    xf = x.float()
    ref = []
    for c in range(8):                               # the kernel's fixed order: ((b + w0 x0) + w1 x1) + ...
        acc = wb[64 + c].expand_as(xf[..., 0])
        for k in range(8):
            acc = acc + wb[c * 8 + k] * xf[..., k]
        ref.append(acc)
    ref = torch.stack(ref, 1).half()
    assert tuple(out.shape) == (3, 8, 45, 60) and torch.equal(out, ref)
    xd, wd = x.double(), wb.double()
    r64 = torch.einsum("nhwk,ck->nchw", xd, wd[:64].view(8, 8)) + wd[64:, None, None]
    mag = torch.einsum("nhwk,ck->nchw", xd.abs(), wd[:64].view(8, 8).abs()) + wd[64:, None, None].abs()
    err = ((out.double() - r64).abs() / (2 * (2.0 ** -11 * r64.abs() + 2.0 ** -25 + 10 * UR * mag))).max().item()
    print(f"\nmoments: worst err / bound {err:.3g}")
    assert err <= 1.0


@pytest.mark.parametrize("with_noise", [True, False])
def test_posterior_kernel(with_noise):
    g = torch.Generator().manual_seed(10)
    n, h, w = 3, 20, 24
    prm = torch.randn(n, 8, h, w, generator=g) * 3
    prm[:, 4:] = torch.linspace(-45.0, 25.0, 4 * h * w).view(4, h, w)[None].expand(n, 4, h, w)   # both clamp ends
    prm = prm.half().cuda()
    noise = torch.randn(n, 4, h, w, generator=g).clamp(-2.5, 2.5).half().cuda() if with_noise else None
    sf = 0.18215
    out = ops.vae_posterior(prm, noise, sf)
    vid = ops.vae_posterior(prm, noise, sf, video=True)
    assert tuple(vid.shape) == (1, 4, n, h, w) and torch.equal(vid[0].permute(1, 0, 2, 3), out)
    mean, lv = prm[:, :4].double(), prm[:, 4:].double().clamp(-30, 20)
    assert bool((prm[:, 4:] < -30).any()) and bool((prm[:, 4:] > 20).any())
    if with_noise:
        t = torch.exp(0.5 * lv) * noise.double()
        ref = sf * (mean + t)
        slack = 8 * UR * (mean.abs() + t.abs()) * sf
    else:
        ref, slack = sf * mean, 2 * UR * sf * mean.abs()
    err = ((out.double() - ref).abs() / (2 * (2.0 ** -11 * ref.abs() + 2.0 ** -25 + slack))).max().item()
    print(f"\nposterior ({'sample' if with_noise else 'mode'}): worst err / bound {err:.3g}")
    assert torch.isfinite(out).all() and err <= 1.0


# ---------------------------------------------------------------------------------------------------- whole encoder
_VAE = {}


def _model():
    """Native VAE + the oracle's fp32 encoder state dict with the same fp16-rounded conv / linear weights (quant_conv,
    biases and norms are fp32 on both sides), on the GPU."""
    if "m" not in _VAE:
        m = V.AutoencoderKL()
        cfg = m.config
        sd = VAE.convert_encoder_state_dict(V.seeded_state_dict(V.vae_encoder_param_shapes(cfg), 7), cfg)
        sd = {k: (v.half().float() if v.dim() >= 2 and not k.startswith("quant_conv") else v).cuda() for k, v in sd.items()}
        _VAE["m"] = (m, sd)
    return _VAE["m"]


def _images(shape, seed):
    """Smooth images in [-1, 1] with some fine detail (a sum of random sinusoids plus noise), fp16."""
    n, _, H, W = shape
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    img = torch.zeros(shape)
    for _ in range(6):
        f = torch.rand(n, 3, 1, 1, generator=g) * 12
        ph = torch.rand(n, 3, 1, 1, generator=g) * 6.3
        img += torch.sin(f * (xx + 0.7 * yy) * 6.3 + ph)
    img = img / 6 + 0.15 * torch.randn(shape, generator=g)
    return img.clamp(-1, 1).half()


@pytest.mark.parametrize("shape", [(2, 3, 64, 64), (1, 3, 512, 512), (1, 3, 360, 480)])
def test_encoder_vs_oracle(shape):
    m, sd = _model()
    x = _images(shape, 31).cuda()
    dist = m.encode(x).latent_dist
    with torch.no_grad(), _fp32_exact():
        ref = EO.encode(x.float(), sd)
    _, rmean, rlogvar, _ = EO.posterior(ref)
    assert tuple(dist.parameters.shape) == (shape[0], 8, shape[2] // 8, shape[3] // 8)
    db_m, db_l = U.psnr(dist.mean, rmean), U.psnr(dist.logvar, rlogvar)
    print(f"\nencoder {shape}: mean {db_m:.1f} dB, logvar {db_l:.1f} dB")
    assert torch.isfinite(dist.parameters).all() and db_m >= 40.0 and db_l >= 40.0


def test_encoder_taps_vs_oracle():
    m, sd = _model()
    x = _images((1, 3, 128, 128), 32).cuda()
    taps, ref_taps = {}, {}
    m._encode_run(x, taps=taps)
    with torch.no_grad(), _fp32_exact():
        EO.encode(x.float(), sd, taps=ref_taps)
    assert taps.keys() == ref_taps.keys()
    worst = math.inf
    for name, t in taps.items():
        r = ref_taps[name]
        db = U.psnr(t[..., :r.shape[1]].permute(0, 3, 1, 2), r)
        print(f"\n  tap {name}: {db:.1f} dB")
        worst = min(worst, db)
        assert db >= 40.0, name
    print(f"\nworst tap {worst:.1f} dB")


def test_encoding_is_per_frame():
    m, _ = _model()
    x = _images((4, 3, 64, 96), 33).cuda()
    together = m.encode(x).latent_dist.parameters
    alone = torch.cat([m.encode(x[i:i + 1]).latent_dist.parameters for i in range(4)])
    db = U.psnr(together, alone)
    print(f"\n4 frames together vs one at a time: {db:.1f} dB")
    assert db >= 70.0


def test_encode_rejects_bad_sizes_and_missing_weights():
    m, _ = _model()
    with pytest.raises(ValueError, match="multiples of 8"):
        m.encode(torch.zeros(1, 3, 60, 64, dtype=torch.float16, device="cuda"))
    dec_only = V.AutoencoderKL(init="empty").load_state_dict(V.seeded_state_dict(V.vae_param_shapes(V.VAEConfig()), 7))
    with pytest.raises(RuntimeError, match="encoder.conv_in.weight"):
        dec_only.encode(torch.zeros(1, 3, 64, 64, dtype=torch.float16, device="cuda"))


def test_sampling_is_seeded():
    m, _ = _model()
    dist = m.encode(_images((2, 3, 64, 64), 34).cuda()).latent_dist
    g = torch.Generator("cuda")
    a = dist.sample(g.manual_seed(5))
    b = dist.sample(g.manual_seed(5))
    assert torch.equal(a, b) and not torch.equal(a, dist.sample(g.manual_seed(6)))
    noise = torch.randn(dist.mean.shape, generator=g.manual_seed(5), device="cuda", dtype=torch.float16)
    mean, std = dist.mean.double(), torch.exp(0.5 * dist.parameters[:, 4:].double().clamp(-30, 20))
    ref = mean + std * noise.double()
    slack = 8 * UR * (mean.abs() + (std * noise.double()).abs())
    err = ((a.double() - ref).abs() / (2 * (2.0 ** -11 * ref.abs() + 2.0 ** -25 + slack))).max().item()
    print(f"\nsample vs mean + std noise: worst err / bound {err:.3g}")
    assert err <= 1.0
    cpu = dist.sample(torch.Generator().manual_seed(5))         # a CPU generator draws on the CPU, as randn_tensor does
    noise_cpu = torch.randn(dist.mean.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float16)
    assert torch.equal(cpu, ops.vae_posterior(dist.parameters, noise_cpu.cuda()))
    assert torch.equal(dist.mode(), ops.vae_posterior(dist.parameters, None))


# ---------------------------------------------------------------------------------------------------- pipeline
def _frames(n, H, W, seed):
    from PIL import Image
    x = ((_images((n, 3, H, W), seed).float() + 1) * 127.5).round().clamp(0, 255).to(torch.uint8)
    return [Image.fromarray(f.permute(1, 2, 0).numpy(), "RGB") for f in x]


def _pipe():
    unet, sd = U.get_model()
    m, _ = _model()
    return V.VideoSwapPipeline(unet, V.DDIMScheduler(), vae=m), sd


def test_invert_from_video_vs_oracle():
    pipe, usd = _pipe()
    m, sd = _model()
    frames = _frames(2, 64, 64, 35)
    emb = U.randn((1, 77, 768), 36).half()
    out = pipe.invert(emb.cuda(), video=frames, generator=torch.Generator("cuda").manual_seed(0), max_iters=3).latents
    assert out.dtype == torch.float16 and tuple(out.shape) == (1, 4, 2, 8, 8)
    x = EO.preprocess(frames)
    with torch.no_grad(), _fp32_exact():
        moments = EO.encode(x.half().float().cuda(), sd)
    noise = torch.randn((2, 4, 8, 8), generator=torch.Generator("cuda").manual_seed(0), device="cuda", dtype=torch.float16)
    lat, _, _, _ = EO.posterior(moments, noise.float())
    lat = (m.config.scaling_factor * lat).permute(1, 0, 2, 3).unsqueeze(0).cpu()
    assert U.psnr(pipe.prepare_image_latents(frames, torch.Generator("cuda").manual_seed(0)), lat) >= 40.0
    with torch.no_grad():
        ref = O.invert_loop(usd, O.OracleConfig(), lat.float(), emb.float(), 50, max_iters=3)
    db = U.psnr(out, ref)
    print(f"\ninvert(video=2 PIL frames 64x64) vs oracle encode + invert_loop: {db:.1f} dB")
    assert db >= 40.0


def test_invert_video_and_latents_agree():
    pipe, _ = _pipe()
    frames = _frames(2, 64, 64, 37)
    emb = U.randn((1, 77, 768), 38).half().cuda()
    a = pipe.invert(emb, video=frames, generator=torch.Generator("cuda").manual_seed(1), max_iters=2).latents
    lat = pipe.prepare_image_latents(frames, torch.Generator("cuda").manual_seed(1))
    # GroupNorm statistics are summed with atomics, so two runs agree to the last bits only
    assert U.psnr(pipe.prepare_image_latents(frames, torch.Generator("cuda").manual_seed(1)), lat) >= 70.0
    b = pipe.invert(emb, lat, max_iters=2).latents
    db = U.psnr(a, b)
    print(f"\ninvert(video=...) vs invert(prepare_image_latents(...)): {db:.1f} dB")
    assert db >= 60.0
    t = EO.preprocess(frames).cuda()                                # the tensor form of the same frames
    assert U.psnr(pipe.prepare_image_latents(t, torch.Generator("cuda").manual_seed(1)), lat) >= 70.0
    z = torch.randn(2, 4, 8, 8, device="cuda")                      # latents pass through, unscaled
    assert torch.equal(pipe.prepare_image_latents(z), z.half().permute(1, 0, 2, 3).unsqueeze(0))
    with pytest.raises(ValueError, match="exactly one"):
        pipe.invert(emb, lat, video=frames)
    with pytest.raises(ValueError, match="exactly one"):
        pipe.invert(emb)
    from PIL import Image
    odd = [f.resize((70, 66)) for f in frames]                      # resized down to 64 x 64 with LANCZOS
    assert tuple(pipe.prepare_image_latents(odd).shape) == (1, 4, 2, 8, 8)
    with pytest.raises(ValueError, match="RGB"):
        pipe.prepare_image_latents([f.convert("L") for f in frames])
    assert isinstance(odd[0], Image.Image)
    with pytest.raises(ValueError, match="vae"):
        V.VideoSwapPipeline(pipe.unet).invert(emb, video=frames)
