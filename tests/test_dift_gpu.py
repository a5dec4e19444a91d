"""DIFT semantic points on the GPU: the read-out kernels per element against fp64, the read-out against the reference
fixture (tests/golden/dift.pt), vs_unet_forward_features against the full forward and across motion modules and batches,
and the featurizer against the fp32 oracle (tests/dift_oracle.py)."""
import ctypes as C
import math
import os

import pytest
import torch

from oracle import unet3d_oracle as O
from oracle.make_golden_dift import IMG, colours
from tests import dift_oracle as D
from videoswap_b200 import (AnimateDiffUNet3DModel, AutoencoderKL, SDFeaturizer, UNetConfig, _lib, dift,
                            extract_point_embedding, ops, seeded_state_dict, unet_param_shapes)

pytestmark = pytest.mark.gpu

GOLD = torch.load(os.path.join(os.path.dirname(__file__), "golden", "dift.pt"), weights_only=False)
EPS32 = 2.0 ** -24


def _g(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------------------------- kernels
def _fp64_read(feat, size, xy):
    """fp64 bilinear read of the ensemble mean, with the source indices computed in fp32 as torch does."""
    f = feat.double().cpu()
    n, E, h, w, Cc = f.shape
    m = f.mean(1)
    H, W = size
    y0, y1, ly1 = D._src_index(xy[..., 1].cpu().long(), h, H)
    x0, x1, lx1 = D._src_index(xy[..., 0].cpu().long(), w, W)
    ly1, lx1 = ly1.double()[..., None], lx1.double()[..., None]
    b = torch.arange(n)[:, None]
    c00, c01, c10, c11 = m[b, y0, x0], m[b, y0, x1], m[b, y1, x0], m[b, y1, x1]
    ref = (1 - ly1) * ((1 - lx1) * c00 + lx1 * c01) + ly1 * ((1 - lx1) * c10 + lx1 * c11)
    scale = torch.stack([c00.abs(), c01.abs(), c10.abs(), c11.abs()]).amax(0)
    return ref, scale


@pytest.mark.parametrize("C_", [320, 640, 1280])
def test_point_sample_per_element(C_):
    """Every (frame, point, channel) against fp64: borders, corners and interior points at non-integer ratios (37/5,
    50/7); bound: the fp32 mean (E adds, a divide) and the six rounded products / sums of the interpolation."""
    n, E, h, w, H, W = 2, 3, 5, 7, 37, 50
    feat = torch.randn((n, E, h, w, C_), generator=_g(C_)).half()
    pts = [(0, 0), (W - 1, H - 1), (0, H - 1), (W - 1, 0), (W // 2, 0), (0, H // 2)]
    rnd = torch.stack([torch.randint(0, W, (20,), generator=_g(1)), torch.randint(0, H, (20,), generator=_g(2))], -1)
    xy = torch.cat([torch.tensor(pts), rnd]).int()[None].repeat(n, 1, 1).contiguous()
    got = ops.dift_point_sample(feat.cuda(), (H, W), xy.cuda()).double().cpu()
    ref, scale = _fp64_read(feat, (H, W), xy)
    bound = (E + 8) * EPS32 * scale + 1e-30
    ratio = ((got - ref).abs() / bound).max().item()
    print(f"dift_point_sample C={C_}: worst error {ratio:.3f} of the bound")
    assert ratio <= 1.0


def test_ensemble_mean_and_noise():
    n, E, h, w, C_ = 2, 4, 3, 5, 64
    feat = torch.randn((n, E, h, w, C_), generator=_g(5)).half()
    got = ops.dift_ensemble_mean(feat.cuda()).cpu()
    ref = feat.double().mean(1).permute(0, 3, 1, 2)
    assert (got.double() - ref).abs().max().item() <= (E + 2) * EPS32 * feat.float().abs().max().item()
    mom = torch.randn((n, 8, h, w), generator=_g(6)).half()
    e1, e2 = torch.randn((n * E, 4, h, w), generator=_g(7)), torch.randn((n * E, 4, h, w), generator=_g(8))
    x = ops.dift_noise(mom.cuda(), e1.cuda(), e2.cuda(), 0.18215, 0.75, 0.66).cpu()
    r = D.noisy_latents(mom.double(), e1.double(), e2.double(), 0.18215, 0.75, 0.66)
    assert x.shape == (n * E, 4, 1, h, w)
    assert (x.double() - r).abs().max().item() <= 1e-5 * r.abs().max().item()


def test_reduce_kernel_against_fp64():
    n, P, C_ = 5, 7, 1280
    v = torch.randn((n, P, C_), generator=_g(9))
    acc = torch.rand((n, P), generator=_g(10)) > 0.4
    acc[:, 3] = False
    s, c, m = ops.dift_point_reduce(v.cuda(), acc.cuda())
    ref = (v.double() * acc[..., None]).sum(0)
    cnt = acc.sum(0).double()
    assert torch.equal(c.cpu().double(), cnt)
    assert (s.cpu().double() - ref).abs().max().item() <= n * EPS32 * 2 * v.abs().max().item()
    assert torch.equal(m[3].cpu(), torch.zeros(C_))
    src = torch.randn((2 * P, C_), generator=_g(11))
    row = torch.randint(0, 2 * P, (n, P), generator=_g(12)).int()
    conf = ops.dift_point_cosine(v.cuda(), src.cuda(), row.cuda()).cpu()
    a, b = v.double(), src.double()[row.long()]
    cref = (a * b).sum(-1) / (a.norm(dim=-1) * b.norm(dim=-1))
    assert (conf.double() - cref).abs().max().item() <= 4 * EPS32


# ---------------------------------------------------------------------------------------------------------------- fixture
def _stored_featurizer(maps):
    calls = []
    dev_maps = maps.cuda()

    def featurize(idx):
        out = dev_maps[len(calls):len(calls) + len(idx)]
        calls.extend(idx)
        return out.permute(0, 2, 3, 1)[:, None].contiguous()
    return featurize, calls


@pytest.mark.parametrize("branch", ["human", "object"])
def test_read_out_matches_reference(branch):
    """Every accept / reject decision and filtered track exactly; embeddings within 4 fp32 ulps of their magnitude per
    element (the bilinear products may round differently from the reference's CPU kernel)."""
    rec = GOLD[branch]
    featurize, calls = _stored_featurizer(rec["maps"])
    emb, tracks, conf = dift.read_out(rec["tracks_in"], featurize, IMG, branch == "human", rec.get("keyframe"),
                                      frames_per_batch=3)
    assert calls == rec["calls"]
    assert torch.equal(tracks, rec["tracks_out"])
    err = (emb - rec["embedding"]).abs().max().item() / rec["embedding"].abs().max().item()
    print(f"{branch}: embedding error {err:.3g} of the largest element")
    assert err <= 4 * 2.0 ** -23
    if conf is not None:
        m = ~rec["confidence"].isnan()
        assert torch.equal(conf.isnan(), ~m)
        assert torch.equal(dift.accepts(conf[m]), dift.accepts(rec["confidence"][m]))
        print(f"object: confidence error {(conf[m] - rec['confidence'][m]).abs().max().item():.3g}")
        assert (conf[m] - rec["confidence"][m]).abs().max().item() <= 1e-5


class _StoredFeaturizer:
    """extract_point_embedding's view of a featurizer: vae.device and features(), here from stored maps."""

    class vae:
        device = torch.device("cuda")

    def __init__(self, maps):
        self.featurize, self.calls = _stored_featurizer(maps)
        self.prompts = []

    def features(self, images, prompt, generator=None):
        assert images.dtype == torch.uint8 and tuple(images.shape[1:]) == IMG + (3,)
        self.prompts.append(prompt)
        return self.featurize([None] * images.shape[0])


@pytest.mark.parametrize("branch", ["human", "object"])
def test_extract_point_embedding_matches_reference(branch):
    from PIL import Image
    rec = GOLD[branch]
    n = rec["tracks_in"].shape[0]
    frames = [Image.new("RGB", (IMG[1], IMG[0]), c) for c in colours(n)]
    tap = {"pred_tracks": rec["tracks_in"].clone(), "point_name2id": {}}
    fz = _StoredFeaturizer(rec["maps"])
    out = extract_point_embedding(tap, frames, fz, "dog", branch == "human", rec.get("keyframe"), frames_per_batch=2)
    assert torch.equal(tap["pred_tracks"], rec["tracks_in"])          # the input dict is left alone
    assert set(fz.prompts) == {rec["prompt"]}
    assert torch.equal(out["pred_tracks"], rec["tracks_out"])
    assert out["point_embedding"].dtype == torch.float32 and out["point_embedding"].device.type == "cpu"
    assert (out["point_embedding"] - rec["embedding"]).abs().max().item() <= 4 * 2.0 ** -23 * rec["embedding"].abs().max().item()


def test_argument_checks():
    from PIL import Image
    rec = GOLD["human"]
    fz = _StoredFeaturizer(rec["maps"])
    tap = {"pred_tracks": rec["tracks_in"]}
    for size in [(IMG[1] + 4, IMG[0]), (IMG[1], IMG[0] - 2)]:
        with pytest.raises(ValueError, match="multiple of 8"):
            extract_point_embedding(tap, [Image.new("RGB", size)] * 3, fz, "dog", True)
    with pytest.raises(ValueError, match="differ in size"):
        extract_point_embedding(tap, [Image.new("RGB", (40, 32))] * 2 + [Image.new("RGB", (48, 32))], fz, "dog", True)
    with pytest.raises(ValueError, match="frames"):
        extract_point_embedding(tap, [Image.new("RGB", (40, 32))] * 2, fz, "dog", True)
    m, _ = _models()
    m._sync_weights(torch.device("cuda"))
    x = torch.randn((2, 4, 1, 8, 8), device="cuda")
    e = torch.randn((2, 77, CTX), device="cuda")
    with pytest.raises(ValueError, match="up_ft_index"):
        m.forward_features(x, 261, e, 4)
    out = torch.empty(1, dtype=torch.float16, device="cuda")
    t = torch.full((2,), 261.0, device="cuda")
    eh = e.half()
    for bad in (-1, 4):
        with pytest.raises(_lib.VSError, match="up_ft_index"):
            _lib.call("vs_unet_forward_features", m._handle, torch.cuda.current_stream().cuda_stream, x.data_ptr(), 1, 2, 1,
                      8, 8, t.data_ptr(), eh.data_ptr(), 77, 0, bad, out.data_ptr())
    hook = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                       C.c_void_p)(lambda *a: None)
    _lib.call("vs_unet_set_attention_hook", m._handle, hook, None, 0)
    try:
        n0 = _lib.lib().vs_launch_count()
        with pytest.raises(_lib.VSError, match="attention"):
            m.forward_features(x, 261, e, 1)
        assert _lib.lib().vs_launch_count() == n0              # rejected before any launch
    finally:
        _lib.call("vs_unet_set_attention_hook", m._handle, None, None, 0)
    # (frame sharding needs a communicator of >= 2 ranks to be set; vs_unet_forward_features rejects it the same way)


# ---------------------------------------------------------------------------------------------------------------- UNet
_MODELS = {}
CTX = 768


def _models():
    """(motion-free SD-1.5 UNet, the same 2-D weights inside a UNet with motion modules), seeded, fp16 on CUDA, and the
    2-D state dict as the fp16 values in fp32."""
    if not _MODELS:
        sd2 = seeded_state_dict(unet_param_shapes(UNetConfig(use_motion_module=False)), seed=0)
        m2 = AnimateDiffUNet3DModel(init="empty", use_motion_module=False)
        m2.load_state_dict(sd2)
        m3 = AnimateDiffUNet3DModel(init="empty")
        sd3 = seeded_state_dict(unet_param_shapes(m3.cfg), seed=3)
        sd3.update(sd2)
        m3.load_state_dict(sd3)
        _MODELS["m"] = (m2.half().cuda(), m3.half().cuda())
        _MODELS["sd"] = {k: v.half().float() for k, v in sd2.items()}
    return _MODELS["m"]


@pytest.mark.parametrize("hw", [(8, 12), (9, 13)])
def test_features_index3_equal_full_forward_tap(hw):
    m2, _ = _models()
    x = torch.randn((3, 4, 1) + hw, generator=_g(20)).cuda()
    e = torch.randn((3, 77, CTX), generator=_g(21)).cuda()
    taps = {}
    m2(x, 261, e, _taps=taps)
    f = m2.forward_features(x, 261, e, 3)
    assert f.shape == taps["up_blocks.3.2"].shape
    _same_forward(f, taps["up_blocks.3.2"], f"up_ft[3] vs full-forward tap up_blocks.3.2 at {hw}")


@pytest.mark.parametrize("k", [0, 1, 2, 3])
def test_motion_modules_are_skipped(k):
    """The 3-D UNet gives the motion-free UNet's features; and up_ft[k] matches the fp32 oracle, odd latent."""
    m2, m3 = _models()
    x = torch.randn((2, 4, 1, 9, 13), generator=_g(22)).cuda()
    e = torch.randn((2, 77, CTX), generator=_g(23)).cuda()
    f2 = m2.forward_features(x, 261, e, k)
    f3 = m3.forward_features(x, 261, e, k)
    _same_forward(f3, f2, f"up_ft[{k}]: UNet with motion modules vs motion-free")
    ref = D.up_ft(_MODELS["sd"], O.OracleConfig(use_motion_module=False), x.cpu().half().float(), 261,
                  e.cpu().half().float(), k)
    got = f2.float().cpu().permute(0, 3, 1, 2)
    assert got.shape == ref.shape
    p = _psnr(got, ref)
    print(f"up_ft[{k}] SD-1.5 UNet vs fp32 oracle: {p:.1f} dB")
    assert p >= 40.0


def test_batch_invariance():
    """A frame featurized alone and inside a batch of frames gives the same features, given the same noise."""
    m2, _ = _models()
    E = 4
    x = torch.randn((3 * E, 4, 1, 9, 13), generator=_g(24)).cuda()
    e = torch.randn((1, 77, CTX), generator=_g(25)).cuda().expand(3 * E, -1, -1)
    whole = m2.forward_features(x, 261, e, 1)
    alone = m2.forward_features(x[E:2 * E].contiguous(), 261, e[:E], 1)
    _same_forward(alone, whole[E:2 * E], "a frame alone vs inside a batch of 3")


def _same_forward(a, b, what):
    """Two forwards over the same inputs.  The UNet's GroupNorm statistics are summed with float atomics, so two runs of
    the same forward differ by fp16 rounding noise; 'the same' is >= 60 dB here (unrelated inputs are near 0 dB)."""
    p = _psnr(a.float().cpu(), b.float().cpu())
    print(f"{what}: {p:.1f} dB")
    assert p >= 60.0, (what, p)


def _psnr(a, b):
    mse = ((a.double() - b.double()) ** 2).mean().item()
    rng = (b.max() - b.min()).item()
    return float("inf") if mse == 0 else 10 * math.log10(rng * rng / mse)


# ---------------------------------------------------------------------------------------------------------------- full SD
def test_full_architecture_against_oracle():
    """SD-1.5 architecture, seeded weights, injected moments and noise: the ensemble-mean map of up_ft[1] against the fp32
    oracle (>= 40 dB), and every point embedding of the human read-out at cosine >= 0.999."""
    m, _ = _models()
    sd16 = _MODELS["sd"]
    n, E, h, w = 2, 2, 16, 24
    mom = torch.randn((n, 8, h, w), generator=_g(30)).half()
    mom[:, 4:] = -2.0
    e1, e2 = torch.randn((n * E, 4, h, w), generator=_g(31)), torch.randn((n * E, 4, h, w), generator=_g(32))
    ehs = torch.randn((1, 77, 768), generator=_g(33)).half()
    a = float(torch.tensor(0.8) ** 0.5)
    b = float(torch.tensor(0.2) ** 0.5)
    x = ops.dift_noise(mom.cuda(), e1.cuda(), e2.cuda(), 0.18215, a, b)
    feat = m.forward_features(x, 261, ehs.cuda().expand(n * E, -1, -1), 1)
    feat = feat.view(n, E, *feat.shape[1:])
    got = ops.dift_ensemble_mean(feat).cpu()
    with torch.no_grad():
        ref = D.featurize(sd16, O.OracleConfig(use_motion_module=False), mom.float(), e1, e2, 0.18215, a, b, 261,
                          ehs.float(), 1)
    p = _psnr(got, ref)
    H, W = 8 * h, 8 * w
    tracks = torch.rand((n, 6, 2), generator=_g(34)) * torch.tensor([W - 1.0, H - 1.0])
    tracks[0, 0] = torch.tensor([W - 1.0, H - 1.0])
    tracks[1, 1] = torch.tensor([0.0, 0.0])
    emb, _, _ = dift.read_out(tracks, lambda idx: feat[idx], (H, W), True)
    emb_ref, _, _ = dift.read_out(tracks, lambda idx: ref[idx].permute(0, 2, 3, 1)[:, None], (H, W), True,
                                  kernels=D.EmulatedReadOut)
    cos = torch.nn.functional.cosine_similarity(emb.double(), emb_ref.double(), dim=1)
    print(f"full SD featurizer vs fp32 oracle: map {p:.1f} dB, point embeddings cosine >= {cos.min().item():.6f}")
    assert p >= 40.0 and cos.min().item() >= 0.999


def test_sd_featurizer_runs_the_pieces():
    """SDFeaturizer.forward on seeded VAE and UNet equals dift_noise -> forward_features -> mean with the
    same generator state, and features() of two images equals the images featurized one by one (SD-1.5 UNet, seeded VAE)."""
    m2, _ = _models()
    vae = AutoencoderKL()
    fz = SDFeaturizer(m2, vae, None, None)
    fz.encode_prompt = lambda prompt: torch.randn((1, 77, CTX), generator=_g(40)).half().cuda()
    img = torch.rand((2, 3, 64, 96), generator=_g(41)) * 2 - 1
    got = fz.forward(img[:1], "photo of a dog", ensemble_size=3, generator=_g(42))
    mom = vae.encode(img[:1].cuda()).latent_dist.parameters
    e1, e2 = dift._draw_noise(1, 3, 8, 12, _g(42), "cuda")
    sa, sb = fz._alphas(261)
    x = ops.dift_noise(mom, e1, e2, vae.config.scaling_factor, sa, sb)
    f = m2.forward_features(x, 261, fz.encode_prompt("").expand(3, -1, -1), 1)
    _same_forward(got, ops.dift_ensemble_mean(f.view(1, 3, *f.shape[1:])), "SDFeaturizer.forward vs its pieces")
    both = fz.features(img, "p", ensemble_size=2, generator=_g(43))
    g = _g(43)
    one = torch.cat([fz.features(img[i:i + 1], "p", ensemble_size=2, generator=g) for i in range(2)])
    _same_forward(one, both, "features() of two images vs one by one")
