"""DIFT semantic points on the CPU: the fp32 oracle (tests/dift_oracle.py) against the reference fixture
(oracle/make_golden_dift.py -> tests/golden/dift.pt), and the read-out's host logic (videoswap_b200.dift.read_out) with a
torch emulation of the kernels' arithmetic, which must reproduce the reference's decisions, and which planted bugs break."""
import os

import pytest
import torch

from oracle import unet3d_oracle as O
from oracle.make_golden_dift import UNET, human_case, object_case, unet_config, unet_inputs
from tests import dift_oracle as D
from videoswap_b200 import dift
from videoswap_b200.spec import unet_param_shapes
from videoswap_b200.weights import seeded_state_dict

GOLD = torch.load(os.path.join(os.path.dirname(__file__), "golden", "dift.pt"), weights_only=False)


def _psnr(a, b):
    mse = ((a - b) ** 2).mean().item()
    rng = (b.max() - b.min()).item()
    return float("inf") if mse == 0 else 10 * torch.log10(torch.tensor(rng * rng / mse)).item()


@pytest.fixture(scope="module")
def tiny_sd():
    return seeded_state_dict(unet_param_shapes(unet_config()), seed=0)


@pytest.mark.parametrize("size", UNET["sizes"])
def test_oracle_up_ft_matches_reference(tiny_sd, size):
    """up_ft[k], k = 0..3, of the oracle without motion modules equals the reference's 2-D UNet (hooks on up_blocks[k]),
    at an even and an odd latent size."""
    cfg = O.OracleConfig(block_out_channels=UNET["boc"], cross_attention_dim=UNET["ctx"], norm_groups=UNET["groups"],
                         use_motion_module=False)
    x, ehs = unet_inputs(*size)
    for k in range(4):
        with torch.no_grad():
            got = D.up_ft(tiny_sd, cfg, x, UNET["t"], ehs, k)
        ref = GOLD["unet"]["feats"][tuple(size)][k]
        assert got.shape == ref.shape, (k, got.shape, ref.shape)
        p = _psnr(got, ref)
        assert p >= 100.0, (size, k, p)


def _featurize_stored(maps):
    """A featurizer over stored maps [m, C, h, w] in call order, as NHWC fp16 [n, 1, h, w, C]."""
    calls = []

    def featurize(idx):
        out = maps[len(calls):len(calls) + len(idx)]
        calls.extend(idx)
        return out.permute(0, 2, 3, 1)[:, None].contiguous()
    return featurize, calls


def _run(branch, kernels=D.EmulatedReadOut):
    rec = GOLD[branch]
    featurize, calls = _featurize_stored(rec["maps"])
    kf = rec.get("keyframe")
    emb, tracks, conf = dift.read_out(rec["tracks_in"], featurize, GOLD["image_size"], branch == "human", kf,
                                      frames_per_batch=2, kernels=kernels)
    return rec, emb, tracks, conf, calls


def _matches(branch, kernels=D.EmulatedReadOut):
    rec, emb, tracks, conf, calls = _run(branch, kernels)
    ok = torch.equal(tracks, rec["tracks_out"]) and calls == rec["calls"]
    ok = ok and (emb - rec["embedding"]).abs().max().item() <= 1e-6 * max(1.0, rec["embedding"].abs().max().item())
    if conf is not None:
        ok = ok and torch.equal(conf.isnan(), rec["confidence"].isnan())
        c, r = conf[~conf.isnan()], rec["confidence"][~conf.isnan()]
        ok = ok and (c - r).abs().max().item() <= 1e-5
    return ok


@pytest.mark.parametrize("branch", ["human", "object"])
def test_emulated_read_out_reproduces_reference(branch):
    """Embeddings, confidences, filtered tracks and the featurizer call order (keyframe first) of both branches."""
    rec, emb, tracks, conf, calls = _run(branch)
    assert calls == rec["calls"]
    assert torch.equal(tracks, rec["tracks_out"])
    err = (emb - rec["embedding"]).abs().max().item()
    assert err <= 1e-6 * rec["embedding"].abs().max().item(), err
    assert torch.equal(emb.norm(dim=1) == 0, rec["embedding"].norm(dim=1) == 0)
    if branch == "object":
        assert torch.equal(conf.isnan(), rec["confidence"].isnan())
        m = ~conf.isnan()
        assert (conf[m] - rec["confidence"][m]).abs().max().item() <= 1e-5
        assert torch.equal(dift.accepts(conf[m]), dift.accepts(rec["confidence"][m]))


def test_fixture_covers_the_edge_cases():
    h, o = GOLD["human"], GOLD["object"]
    ht, ot = h["tracks_in"], o["tracks_in"]
    assert ((ht - ht.floor()) == 0.5).any() and (ht == -0.4).any() and (ht == -1).any()
    assert (ot == -1).any() and ((ot[..., 0] >= GOLD["image_size"][1]) | (ot[..., 1] >= GOLD["image_size"][0])).any()
    c = o["confidence"][~o["confidence"].isnan()]
    assert (c >= 0.35).any() and (c < 0.35).any() and (c - 0.35).abs().min() > 1e-3
    assert (h["embedding"].norm(dim=1) == 0).any()           # a point never visible keeps a zero embedding
    assert h["prompt"] == "photo of a dog" and o["calls"][0] == o["keyframe"]


def test_query_matches_reference():
    """DIFT_Demo.query at a negative target point: the two reads and the cosine of the emulation."""
    q = GOLD["query"]
    maps = GOLD["object"]["maps"]
    H, W = GOLD["image_size"]
    src_xy = torch.tensor([[[int(q["query_point"][1]), int(q["query_point"][0])]]])
    tgt = (int(q["target_point"][1]) % W, int(q["target_point"][0]) % H)
    nhwc = maps.permute(0, 2, 3, 1)[:, None]
    s = D.EmulatedReadOut.sample(nhwc[q["source"]:q["source"] + 1], (H, W), src_xy)[0]
    t = D.EmulatedReadOut.sample(nhwc[q["target"]:q["target"] + 1], (H, W), torch.tensor([[tgt]]))
    assert (t[0, 0] - q["feat"]).abs().max().item() <= 1e-6 * q["feat"].abs().max().item()
    c = D.EmulatedReadOut.cosine(t, s, torch.zeros((1, 1), dtype=torch.int32))
    assert abs(c.item() - q["confidence"]) <= 1e-5


def test_bilinear_emulation_matches_torch_upsample():
    """The emulated source indices and weights against nn.Upsample at every pixel, non-integer ratios."""
    g = torch.Generator().manual_seed(3)
    m = torch.randn((1, 16, 5, 6), generator=g)
    H, W = 32, 40
    xy = torch.stack(torch.meshgrid(torch.arange(W), torch.arange(H), indexing="xy"), -1).reshape(1, -1, 2)
    got = D.EmulatedReadOut.sample(m.permute(0, 2, 3, 1)[:, None], (H, W), xy)[0]
    ref = torch.nn.Upsample(size=(H, W), mode="bilinear")(m)[0].permute(1, 2, 0).reshape(-1, 16)
    assert (got - ref).abs().max().item() <= 1e-6


class _AlignCorners(D.EmulatedReadOut):
    align_corners = True


class _CountRejected(D.EmulatedReadOut):
    count_rejected = True


@pytest.mark.parametrize("bug", ["round_half_up", "align_corners", "no_negative_wrap", "greater_than", "count_rejected"])
def test_planted_bugs_are_caught(monkeypatch, bug):
    kernels = D.EmulatedReadOut
    if bug == "round_half_up":
        monkeypatch.setattr(dift, "round_half_even", lambda t: torch.floor(t + 0.5).to(torch.int64))
    elif bug == "align_corners":
        kernels = _AlignCorners
    elif bug == "no_negative_wrap":
        monkeypatch.setattr(dift, "wrap_index", lambda i, size: i.clamp_min(0))
    elif bug == "greater_than":
        # `>` and `>=` differ only at a confidence equal to the threshold: move the threshold onto one
        monkeypatch.setattr(dift, "CONFIDENCE_THRESHOLD", float(_run("object")[3][0, 0]))
        monkeypatch.setattr(dift, "accepts", lambda c: c > dift.CONFIDENCE_THRESHOLD)
        rec, emb, tracks, conf, _ = _run("object", kernels)
        monkeypatch.setattr(dift, "accepts", lambda c: c >= dift.CONFIDENCE_THRESHOLD)
        rec2, emb2, tracks2, conf2, _ = _run("object", kernels)
        assert not torch.equal(tracks, tracks2)
        return
    elif bug == "count_rejected":
        kernels = _CountRejected
    assert not (_matches("human", kernels) and _matches("object", kernels)), bug


def test_noise_draws_follow_the_reference():
    """_draw_noise with a CPU generator gives, frame by frame, the reference's `latent_dist.sample()` draw of
    randn_tensor(shape, dtype=fp32) and then `torch.randn_like(latents)` from the same generator state."""
    n, E, h, w = 3, 4, 5, 6
    e1, e2 = dift._draw_noise(n, E, h, w, torch.Generator().manual_seed(9), "cpu")
    torch.manual_seed(9)                        # the reference draws from the default generator
    r1, r2 = [], []
    for _ in range(n):
        lat = torch.randn((E, 4, h, w), generator=None, device="cpu", dtype=torch.float32)   # randn_tensor
        r1.append(lat)
        r2.append(torch.randn_like(lat))
    assert torch.equal(e1, torch.cat(r1)) and torch.equal(e2, torch.cat(r2))


@pytest.mark.parametrize("bad", [("human", (0, 0), (40.0, 3.0)), ("human", (1, 2), (3.0, 31.5)),
                                 ("object", (2, 1), (-41.0, 3.0))])
def test_out_of_image_points_raise(bad):
    branch, (f, p), xy = bad
    rec = GOLD[branch]
    tracks = rec["tracks_in"].clone()
    tracks[f, p] = torch.tensor(xy)
    featurize, _ = _featurize_stored(rec["maps"])
    with pytest.raises(ValueError, match=f"frame {f}, point {p}"):
        dift.read_out(tracks, featurize, GOLD["image_size"], branch == "human", rec.get("keyframe"),
                      kernels=D.EmulatedReadOut)


def test_fixture_is_small():
    assert os.path.getsize(os.path.join(os.path.dirname(__file__), "golden", "dift.pt")) < 1 << 20


@pytest.mark.parametrize("case", ["human", "object"])
def test_case_builders_match_fixture(case):
    """The tests' inputs are the generator's (seeded) inputs."""
    maps, tracks = (human_case() if case == "human" else object_case()[:2])
    assert torch.equal(maps.half(), GOLD[case]["maps"]) and torch.equal(tracks, GOLD[case]["tracks_in"])
