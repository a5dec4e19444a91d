"""VAE decoder tests on the GPU (pytest -m gpu): GroupNorm at 4 channels per group with the per-element bound of
tests/norm_probes.py, the row softmax and the single-head d = 512 attention against fp64 with bounds from the kernels'
arithmetic, the entry / exit / transpose kernels bit-exact against torch, the whole decoder against the CPU oracle
(tests/vae_oracle.py), per-frame independence, and the pipeline's decoded outputs."""
import math

import numpy as np
import pytest
import torch

import videoswap_b200 as V
from tests import norm_probes as P
from tests import unet_checks as U
from tests import vae_oracle as VO
from videoswap_b200 import ops
from videoswap_b200 import vae as VAE

pytestmark = pytest.mark.gpu
UR = 2.0 ** -24


# ---------------------------------------------------------------------------------------------------- GroupNorm, cpg = 4
def _gn(x1, x2, gamma, beta, eps, imgs_per_set, silu):
    return ops.groupnorm(x1, gamma, beta, P.GROUPS, eps, imgs_per_set=imgs_per_set, silu=silu, x2=x2)


GN_CASES = {f"{B}x{H}x{W}x128_{'silu' if s else 'plain'}": (B, H, W, s)
            for B, H, W in ((1, 64, 64), (1, 512, 512), (4, 64, 64)) for s in (True, False)}


@pytest.mark.parametrize("name", sorted(GN_CASES))
def test_groupnorm_4_channels_per_group(name):
    """C = 128 in 32 groups: every 8-channel vector holds two groups (split 4).  Group-distinct statistics make a vector's
    second group normalised with the first one's wrong by O(1); impulses sit at the first and last channel of both groups
    of a vector (split_channels) on the schedules' edge pixels."""
    B, H, W, silu = GN_CASES[name]
    assert P.split_channels(128)[:2] == [3, 0]
    r = P.check_groupnorm(_gn, B, 1, H, W, 128, silu=silu, eps=1e-6, launches=2, seed=100 + H + B)
    torch.cuda.synchronize()
    print(f"\n{name}: worst err / bound {r['err']:.4g}; {r.get('report', '')}")
    assert r["ok"], f"{name}: {r.get('what', '')}: worst err / bound {r['err']:.4g}"


# ---------------------------------------------------------------------------------------------------- row softmax
def softmax_bound(s16, n, p):
    """Per-element bound of softmax_rows_kernel on fp16 logits s16 [rows, >= n] against the fp64 softmax p.
    t_j = fl((s_j - m) c) with c = fl(log2(e) / sqrt(512)) (s_j - m exact): argument error <= 4 u |t_j|, so exp2f (2 ulp)
    gives e_j within (4 u + ln2 4 u |t_j|) e_j; l sums <= D = 8 ceil(ld / 2048) + 12 positive terms deep (a thread's run,
    5 shuffles, 7 warp partials), so within (D u + max_j(4 u + ln2 4 u |t_j|)) l; the division rounds once (u) and the
    fp16 store 2^-11 relative or 2^-25 absolute.  The comparator allows twice that."""
    ld = s16.shape[1]
    s = s16[:, :n].double()
    c = 1.4426950408889634 / math.sqrt(512)
    t = ((s - s.amax(1, keepdim=True)) * c).abs()
    D = 8 * math.ceil(ld / 2048) + 12
    rel = 2.0 ** -11 + UR * (1 + 4 + 4 + D) + math.log(2) * 4 * UR * (t + t.amax(1, keepdim=True))
    return 2 * (rel * p + 2.0 ** -25)


def _logits(rows, n, seed):
    """fp16 S [rows, n]: row 0 one dominant logit, row 1 logits spread over +-40, the rest N(0, sigma^2) logits with sigma
    from 0.3 to 12 (logit = s / sqrt(512))."""
    g = torch.Generator().manual_seed(seed)
    r = math.sqrt(512)
    sig = torch.exp(torch.linspace(math.log(0.3), math.log(12.0), rows))[:, None]
    s = torch.randn(rows, n, generator=g) * sig * r
    s[0] = torch.randn(n, generator=g) * r
    s[0, n // 3] = 30 * r
    s[1] = torch.linspace(-40, 40, n)[torch.randperm(n, generator=g)] * r
    return s.clamp(-65000, 65000).half()


@pytest.mark.parametrize("n", [64, 77, 2700, 4096])
def test_softmax_rows(n):
    rows, ld = 96, VAE.padded_keys(n) + (8 if n % 8 == 0 else 0)     # also a padded stride when n is aligned
    s16 = _logits(rows, n, n).cuda()
    buf = torch.full((rows, ld), float("nan"), dtype=torch.float16, device="cuda")
    buf[:, :n] = s16
    ops.softmax_rows(buf, n, 1.0 / math.sqrt(512))
    p = torch.softmax(s16.double() / math.sqrt(512), 1)
    err = ((buf[:, :n].double() - p).abs() / softmax_bound(s16, n, p)).max().item()
    print(f"\nsoftmax n {n}: worst err / bound {err:.4g}")
    assert torch.isfinite(buf[:, :n]).all()
    assert bool((buf[:, n:] == 0).all()) and not bool(torch.signbit(buf[:, n:]).any()), "padding columns are not +0"
    assert err <= 1.0


# ---------------------------------------------------------------------------------------------------- attention
def _qkv(hw, seed, sigma=2.0):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(hw, 512, generator=g) * math.sqrt(sigma)
    k = torch.randn(hw, 512, generator=g) * math.sqrt(sigma)
    v = torch.randn(hw, 512, generator=g)
    return q.half().cuda(), k.half().cuda(), v.half().cuda()


def _attend(q, k, v):
    hw = q.shape[0]
    ld = VAE.padded_keys(hw)
    s = torch.empty((hw, ld), dtype=torch.float16, device="cuda")
    vt = torch.empty((512, ld), dtype=torch.float16, device="cuda")
    return VAE.attend(q, k, v, s, vt, torch.empty((hw, 512), dtype=torch.float16, device="cuda"))


@pytest.mark.parametrize("hw", [64, 2700, 4096])
def test_attention_one_hot_probe(hw):
    """V[sel(c), c] = 1: out[:, c] = P[:, sel(c)], one probability per element (sel covers the first, last and padding-
    adjacent keys).  Bound: the softmax bound plus the fp16 rounding of S = q.k (2^-11 |S| + 2^-15 sum|q||k| for the fp32
    accumulation over d = 512) as a logit error dt, which moves p_j by at most (dt_j + max dt) p_j (x 1.1)."""
    q, k, _ = _qkv(hw, hw)
    sel = (torch.arange(512) * 7 + 3) % hw
    sel[:4] = torch.tensor([0, hw - 1, hw - 2, min(64, hw - 1)])
    v = torch.zeros(hw, 512, dtype=torch.float16)
    v[sel, torch.arange(512)] = 1.0
    out = _attend(q, k, v.cuda())
    qd, kd = q.double(), k.double()
    S = qd @ kd.t()
    p = torch.softmax(S / math.sqrt(512), 1)
    dt = (2.0 ** -11 * S.abs() + 2.0 ** -15 * (qd.abs() @ kd.abs().t())) / math.sqrt(512)
    dt = dt + dt.amax(1, keepdim=True)
    s16 = (qd @ kd.t()).half()
    sc = sel.cuda()
    bound = softmax_bound(s16, hw, p)[:, sc] + 2 * 1.1 * dt[:, sc] * p[:, sc]
    err = ((out.double() - p[:, sc]).abs() / bound).max().item()
    print(f"\nattention one-hot hw {hw}: worst err / bound {err:.4g}")
    assert torch.isfinite(out).all() and err <= 1.0


@pytest.mark.parametrize("hw", [64, 2700, 4096])
def test_mid_block_attention_random(hw):
    """The whole block (GroupNorm, q / k / v, attention, to_out + residual) on seeded weights against an fp64 restatement
    on the same fp16 input and weights; the attention's contribution out - x must agree to >= 45 dB."""
    vae = V.AutoencoderKL()
    H, W = {64: (8, 8), 2700: (45, 60), 4096: (64, 64)}[hw]
    x = (U.randn((2, H, W, 512), hw) * 2).half().cuda()
    out = vae._attention(x, vae._w["attn"])
    sd = {k: v.double().cuda() for k, v in VAE.convert_state_dict(V.seeded_state_dict(V.vae_param_shapes(vae.config), 7),
                                                                   vae.config).items() if "attentions" in k}
    sd = {k: (v.half().double() if v.dim() == 2 else v) for k, v in sd.items()}
    ref = VO.attention(x.double().permute(0, 3, 1, 2), sd, "decoder.mid_block.attentions.0").permute(0, 2, 3, 1)
    db = U.psnr((out.double() - x.double()).cpu(), (ref - x.double()).cpu())
    print(f"\nmid-block attention hw {hw}: {db:.1f} dB")
    assert db >= 45.0


# ---------------------------------------------------------------------------------------------------- bit-exact kernels
def test_transpose_pad_bit_exact():
    x = U.randn((2700, 512), 5).half().cuda()
    out = torch.full((512, 2704), float("nan"), dtype=torch.float16, device="cuda")
    ops.transpose_pad(x, 2704, out=out)
    ref = torch.cat([x.t(), torch.zeros(512, 4, dtype=torch.float16, device="cuda")], 1)
    assert torch.equal(out, ref)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_latent_in_bit_exact(dtype):
    z = (U.randn((3, 4, 45, 60), 6) * 0.9).to(dtype).cuda()
    wb = U.randn((20,), 7).cuda()
    sf = 0.18215
    out = ops.vae_latent_in(z, sf, wb)
    x = z.float() / torch.full_like(z, sf, dtype=torch.float32)          # true division (a scalar divisor is a reciprocal)
    ref = []
    for c in range(4):
        acc = wb[16 + c].expand_as(x[:, 0])
        for k in range(4):
            acc = acc + wb[c * 4 + k] * x[:, k]
        ref.append(acc)
    ref = torch.stack(ref, -1).half()
    assert torch.equal(out, ref)
    one = ops.vae_latent_in(z, 1.0, wb)                                    # decode(): no scaling
    assert not torch.equal(one, out)


def test_image_postprocess_bit_exact():
    from tests.test_vae_cpu import _crafted
    vals, _ = _crafted()
    g = torch.Generator().manual_seed(8)
    n, H, W = 2, 37, 53
    x = torch.randn(n, H, W, 8, generator=g).half()
    flat = x.view(-1)
    flat[:vals.numel()] = vals
    x = x.cuda()
    xs = x[..., :3].permute(0, 3, 1, 2).float().cpu()
    assert torch.equal(ops.image_postprocess(x, ops.IMG_SAMPLE).cpu(), x[..., :3].permute(0, 3, 1, 2).cpu())
    assert torch.equal(ops.image_postprocess(x, ops.IMG_PT).cpu(), VO.postprocess(xs, "pt"))
    assert np.array_equal(ops.image_postprocess(x, ops.IMG_NP).cpu().numpy(), VO.postprocess(xs, "np"))
    assert np.array_equal(ops.image_postprocess(x, ops.IMG_PIL).cpu().numpy(), VO.postprocess(xs, "pil"))


# ---------------------------------------------------------------------------------------------------- whole decoder
_VAE = {}


def _model():
    """Native decoder + the oracle's fp32 state dict with the same fp16-rounded conv / linear weights (post_quant_conv,
    biases and norms are fp32 on both sides)."""
    if "m" not in _VAE:
        m = V.AutoencoderKL()
        sd = VAE.convert_state_dict(V.seeded_state_dict(V.vae_param_shapes(m.config), 7), m.config)
        sd = {k: (v.half().float() if v.dim() >= 2 and not k.startswith("post_quant_conv") else v) for k, v in sd.items()}
        _VAE["m"] = (m, sd)
    return _VAE["m"]


@pytest.mark.parametrize("shape", [(2, 4, 8, 8), (1, 4, 64, 64), (1, 4, 45, 60)])
def test_decoder_vs_oracle(shape):
    m, sd = _model()
    z = U.randn(shape, 11)
    out = m.decode(z.cuda()).sample
    assert out.dtype == torch.float16 and tuple(out.shape) == (shape[0], 3, 8 * shape[2], 8 * shape[3])
    with torch.no_grad():
        ref = VO.decode(z, sd)
    db = U.psnr(out.cpu(), ref)
    print(f"\ndecoder {shape}: {db:.1f} dB (sample range {ref.min().item():.3g} .. {ref.max().item():.3g})")
    assert torch.isfinite(out).all() and db >= 40.0


def test_decoder_taps_vs_oracle():
    m, sd = _model()
    z = U.randn((1, 4, 16, 16), 12)
    taps, ref_taps = {}, {}
    m._run(z.cuda(), 1.0, ops.IMG_SAMPLE, taps=taps)
    with torch.no_grad():
        VO.decode(z, sd, taps=ref_taps)
    assert taps.keys() == ref_taps.keys()
    worst = math.inf
    for name, t in taps.items():
        r = ref_taps[name]
        db = U.psnr(t[..., :r.shape[1]].permute(0, 3, 1, 2).cpu(), r)
        print(f"\n  tap {name}: {db:.1f} dB")
        worst = min(worst, db)
        assert db >= 40.0, name
    print(f"\nworst tap {worst:.1f} dB")


def test_decoding_is_per_frame():
    m, _ = _model()
    z = U.randn((4, 4, 32, 32), 13).half().cuda()
    together = m.decode(z).sample
    alone = torch.cat([m.decode(z[i:i + 1]).sample for i in range(4)])
    db = U.psnr(together, alone)
    print(f"\n4 frames together vs one at a time: {db:.1f} dB")
    assert db >= 70.0


# ---------------------------------------------------------------------------------------------------- pipeline
def _pipe():
    unet, _ = U.get_model()
    m, _ = _model()
    return V.VideoSwapPipeline(unet, V.DDIMScheduler(), vae=m)


def test_pipeline_decodes_frames():
    pipe = _pipe()
    lat = U.randn((1, 4, 2, 8, 8), 21).half().cuda()
    pos, neg = U.randn((1, 16, 77, 768), 22).half().cuda(), U.randn((1, 16, 77, 768), 23).half().cuda()
    kw = dict(negative_prompt_embeds=neg, num_inference_steps=50, guidance_scale=7.5, max_iters=1)
    latents = pipe(pos, lat, output_type="latent", **kw).videos
    pt = pipe(pos, lat, output_type="pt", **kw).videos
    ref = pipe.decode_latents(latents, "pt")
    assert pt.dtype == torch.float32 and tuple(pt.shape) == (2, 3, 64, 64)
    assert float(pt.min()) >= 0.0 and float(pt.max()) <= 1.0
    db = U.psnr(pt, ref)
    print(f"\npipeline 'pt' vs decode_latents of the 'latent' run: {db:.1f} dB")
    assert db >= 60.0
    arr = pipe(pos, lat, output_type="np", **kw).videos
    assert isinstance(arr, np.ndarray) and arr.dtype == np.float32 and arr.shape == (2, 64, 64, 3)
    ims = pipe(pos, lat, output_type="pil", **kw).videos
    assert isinstance(ims, list) and len(ims) == 2
    assert all(im.mode == "RGB" and im.size == (64, 64) for im in ims)
    five = pipe.decode_latents(latents.reshape(1, 2, 4, 8, 8).permute(0, 2, 1, 3, 4), "pt")     # [b, c, f, h, w] form
    assert U.psnr(five, ref) >= 60.0


def test_second_load_reproduces_the_decode():
    m = V.AutoencoderKL()
    z = U.randn((1, 4, 16, 16), 14).cuda()
    first = m.decode(z).sample.clone()
    m.load_state_dict(V.seeded_state_dict(V.vae_param_shapes(m.config), 9))
    other = m.decode(z).sample
    m.load_state_dict(V.seeded_state_dict(V.vae_param_shapes(m.config), 7))
    again = m.decode(z).sample
    assert U.psnr(other, first) < 40.0
    assert U.psnr(again, first) >= 70.0
