"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/dift.pt from the REFERENCE's own code on the CPU:

  * unet: up_ft[k], k = 0..3, of the reference's AnimateDiffUNet3DModel built with use_motion_module=False (the 2-D SD
    UNet; DESIGN.md 6) at F = 1, seeded weights, read with a forward hook on up_blocks[k] (the block's output after its
    up-sampler, what dift_util.py's MyUNet2DConditionModel collects), at an even and an odd latent size.
  * human / object: extract_semantic_point.extract_point_embedding (both branches) and dift_util.DIFT_Demo.query, with
    SDFeaturizer replaced by a stub that returns stored feature maps (fp16-representable fp32, so a native read-out sees
    identical inputs) in call order.  Frames are solid colours written as JPEG so the reference's keyframe path
    round-trips; the frame directory is walked in sorted order (the reference walks Path.iterdir() unsorted).
    Imports go through throw-away sys.modules stubs for controlnet_aux, cotracker.predictor, matplotlib.pyplot, imageio
    and the diffusers names dift_util imports.

Run where the reference tree is checked out:  VIDEOSWAP_REFERENCE=<checkout> python -m oracle.make_golden_dift
"""
import os
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden import OUT, randn  # noqa: E402
from oracle.ref_loader import ADDITIONAL_KWARGS, REFERENCE_ROOT, SD15_UNET_CONFIG, load_reference  # noqa: E402
from videoswap_b200.spec import UNetConfig, unet_param_shapes  # noqa: E402
from videoswap_b200.weights import seeded_state_dict  # noqa: E402

# tiny UNet (the tiny cases of oracle/make_golden.py) without motion modules; 8x12 and 9x13 latents (odd sides take the
# reference's forward_upsample_size path)
UNET = dict(boc=(32, 64, 128, 128), ctx=64, groups=8, batch=2, t=261, sizes=[(8, 12), (9, 13)])
IMG = (32, 40)          # frame height, width: multiples of 8
MAP = (5, 6)            # feature map: non-integer up-sampling ratios 6.4 and 6.67
C = 1280                # the reference's init_embedding width


def unet_inputs(h, w):
    """Shared with the tests: sample [B, 4, 1, h, w], embeddings [B, 77, ctx]."""
    return randn((UNET["batch"], 4, 1, h, w), 22), randn((UNET["batch"], 77, UNET["ctx"]), 23)


def unet_config():
    return UNetConfig(block_out_channels=UNET["boc"], cross_attention_dim=UNET["ctx"], norm_num_groups=UNET["groups"],
                      use_motion_module=False)


def run_unet():
    ns = load_reference()
    cfg = dict(SD15_UNET_CONFIG, block_out_channels=UNET["boc"], cross_attention_dim=UNET["ctx"],
               norm_num_groups=UNET["groups"])
    model = ns.AnimateDiffUNet3DModel.from_config(cfg, **dict(ADDITIONAL_KWARGS, use_motion_module=False))
    ns.revise_edlora_unet_attention_forward(model)
    model.eval()
    sd = seeded_state_dict(unet_param_shapes(unet_config()), seed=0)
    model.load_state_dict(sd, strict=True)
    got = {}
    for k, blk in enumerate(model.up_blocks):
        blk.register_forward_hook(lambda m, a, o, k=k: got.__setitem__(k, o.detach().clone()))
    out = {}
    for h, w in UNET["sizes"]:
        x, ehs = unet_inputs(h, w)
        got.clear()
        with torch.no_grad():
            model(x, UNET["t"], ehs, return_dict=False)
        # [B, C, 1, h_k, w_k] -> [B, C, h_k, w_k]
        out[(h, w)] = {k: v[:, :, 0].contiguous() for k, v in got.items()}
        print("unet", (h, w), {k: tuple(v.shape) for k, v in out[(h, w)].items()})
    return out


# ---------------------------------------------------------------------------------------------------------------- read-out
def _stub_modules():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        return m

    class _Any:
        def __init__(self, *a, **k):
            pass

        @classmethod
        def from_pretrained(cls, *a, **k):
            return cls()

    stubs = {
        "controlnet_aux": mod("controlnet_aux", OpenposeDetector=_Any),
        "controlnet_aux.util": mod("controlnet_aux.util", HWC3=lambda x: x, resize_image=lambda x, resolution: x),
        "cotracker": mod("cotracker"),
        "cotracker.predictor": mod("cotracker.predictor", CoTrackerPredictor=_Any),
        "matplotlib": mod("matplotlib"),
        "matplotlib.pyplot": mod("matplotlib.pyplot", get_cmap=lambda name: None),
        "imageio": mod("imageio"),
        "diffusers": mod("diffusers", DDIMScheduler=_Any, StableDiffusionPipeline=_Any),
        "diffusers.models": mod("diffusers.models"),
        "diffusers.models.unet_2d_condition": mod("diffusers.models.unet_2d_condition", UNet2DConditionModel=_Any),
    }
    return stubs


def import_reference_readout():
    """(extract_semantic_point, dift_util) of the reference, imported under the stubs, which are removed again."""
    saved = {k: sys.modules.get(k) for k in list(_stub_modules()) + ["videoswap", "videoswap.utils",
                                                                      "videoswap.utils.dift_util",
                                                                      "videoswap.utils.vis_util", "extract_semantic_point"]}
    sys.modules.update(_stub_modules())
    sys.path.insert(0, REFERENCE_ROOT)
    try:
        import importlib
        esp = importlib.import_module("extract_semantic_point")
        du = importlib.import_module("videoswap.utils.dift_util")
    finally:
        sys.path.remove(REFERENCE_ROOT)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return esp, du


def colours(n):
    return [(30 + 50 * i, 220 - 45 * i, 90 + 20 * (i % 2)) for i in range(n)]


def human_case():
    """Shared with the tests: 3 frames, 7 points; maps [3, C, h, w] (fp16 values)."""
    g = torch.Generator().manual_seed(31)
    maps = torch.randn((3, C) + MAP, generator=g).half().float()
    H, W = IMG
    t = torch.tensor([
        [[2.5, 3.5], [-0.4, 7.0], [-1.0, 5.0], [W - 1.0, H - 1.0], [-1.0, -1.0], [10.49, 0.5], [17.5, 30.6]],
        [[3.5, 2.5], [5.0, -0.4], [4.0, -1.0], [W - 1.4, 0.0], [-1.0, -1.0], [-0.5, 12.5], [18.0, 29.0]],
        [[0.0, 0.0], [-0.4, -0.4], [20.2, 11.8], [0.5, H - 0.6], [-1.0, -1.0], [33.5, 1.5], [-3.0, 30.0]],
    ], dtype=torch.float32)
    return maps, t


def object_case():
    """Shared with the tests: 4 frames, keyframe 1, 8 points.  Call-order maps [5, C, h, w]: the keyframe's own
    featurization first, then frames 0..3.  The keyframe map S is a common vector plus noise; frame maps mix it with
    fresh noise by a weight falling from 1 at column 0 to 0 at the last column, so confidences span both sides of 0.35."""
    g = torch.Generator().manual_seed(41)
    h, w = MAP
    v0 = torch.randn((C, 1, 1), generator=g)
    S = v0 + 0.5 * torch.randn((C, h, w), generator=g)
    mix = torch.linspace(1.0, 0.0, w).view(1, 1, w)
    frames = [mix * (v0 + 0.5 * torch.randn((C, h, w), generator=g)) + (1 - mix) * 1.5 * torch.randn((C, h, w), generator=g)
              for _ in range(4)]
    maps = torch.stack([S] + frames).half().float()
    H, W = IMG
    t = torch.tensor([
        # frame 0
        [[2.5, 3.5], [30.0, 5.0], [-1.0, -1.0], [W + 2.0, 3.0], [5.5, 20.5], [-1.0, 10.0], [W + 5.0, H + 1.0], [1.0, 1.0]],
        # frame 1 = keyframe (point 6 out of bounds: skipped, later frames read their source at (-1, -1); point 5 at a
        # low-confidence column: rejected, same)
        [[3.0, 4.0], [20.0, 6.0], [8.0, 8.0], [4.0, 4.0], [6.0, 21.0], [36.0, 10.0], [W + 3.0, 5.0], [2.0, 2.0]],
        # frame 2
        [[1.5, 2.5], [38.6, 31.4], [-1.0, 3.0], [12.0, H + 0.2], [0.0, 31.0], [2.0, 2.0], [3.0, 3.0], [W - 0.4, -1.0]],
        # frame 3
        [[6.0, 6.0], [24.5, 16.5], [-0.4, -0.6], [2.0, 2.0], [35.0, 3.0], [4.0, 28.0], [1.0, 30.0], [-2.0, -3.0]],
    ], dtype=torch.float32)
    return maps, t, 1


class _StubFeaturizer:
    """Stands in for dift_util.SDFeaturizer: the stored maps in call order; records each call's frame (by colour)."""
    maps = None
    calls = []
    cols = None

    def __init__(self, sd_id=None):
        self.n = 0

    def forward(self, img_tensor, prompt, t=261, up_ft_index=1, ensemble_size=8):
        rgb = ((img_tensor.float().mean((1, 2)) / 2 + 0.5) * 255).tolist()
        f = int(np.argmin([sum((a - b) ** 2 for a, b in zip(rgb, c)) for c in self.cols]))
        _StubFeaturizer.calls.append((f, prompt))
        m = self.maps[len(_StubFeaturizer.calls) - 1]
        return m[None].clone()


class _SortedPath(type(Path())):
    def iterdir(self):
        return iter(sorted(super().iterdir()))


def run_branch(esp, du, is_human):
    from PIL import Image
    if is_human:
        maps, tracks = human_case()
        kf = None
    else:
        maps, tracks, kf = object_case()
    n = tracks.shape[0]
    cols = colours(n)
    confs = torch.full(tracks.shape[:2], float("nan"))
    H, W = IMG
    with tempfile.TemporaryDirectory() as d:
        for i, c in enumerate(cols):
            Image.new("RGB", (W, H), c).save(os.path.join(d, f"{i:05d}.jpg"), quality=100)
        _StubFeaturizer.maps, _StubFeaturizer.calls, _StubFeaturizer.cols = maps, [], cols
        esp.SDFeaturizer = _StubFeaturizer
        esp.Path = _SortedPath
        query = du.DIFT_Demo.query
        state = {}

        def query_rec(self, target_img, target_dift, target_img_size, query_point, target_point, visualize=False):
            r = query(self, target_img, target_dift, target_img_size, query_point, target_point, visualize)
            f = _StubFeaturizer.calls[-1][0]
            p = state.setdefault(f, 0)
            while not torch.equal(torch.round(tracks[f, p]), torch.tensor([float(target_point[1]), float(target_point[0])])):
                p += 1
            state[f] = p + 1
            confs[f, p] = float(r[1])
            return r
        esp.DIFT_Demo.query = query_rec
        try:
            tap = {"pred_tracks": tracks.clone(), "point_name2id": {f"p{i}": i for i in range(tracks.shape[1])}}
            ann = os.path.join(d, f"{kf:05d}.json") if kf is not None else None
            out = esp.extract_point_embedding(tap, d, ann, "unused", "dog", is_human=is_human)
        finally:
            esp.DIFT_Demo.query = query
    rec = {"maps": maps.half(), "tracks_in": tracks, "embedding": out["point_embedding"].clone(),
           "tracks_out": out["pred_tracks"].clone(), "calls": [c[0] for c in _StubFeaturizer.calls],
           "prompt": _StubFeaturizer.calls[0][1]}
    if not is_human:
        rec["keyframe"] = kf
        rec["confidence"] = confs
        c = confs[~confs.isnan()]
        print("object confidences:", [round(float(v), 4) for v in c])
        assert (c - 0.35).abs().min() > 1e-3, "a confidence is too close to the threshold"
    print("human" if is_human else "object", "embedding norms", out["point_embedding"].norm(dim=1).tolist())
    return rec


def run_query(du):
    """One direct DIFT_Demo.query with a negative target point (Python wrap)."""
    maps, _, _ = object_case()
    H, W = IMG
    demo = du.DIFT_Demo(None, maps[0][None].clone(), [H, W])
    feat, conf, _ = demo.query(None, maps[2][None].clone(), [H, W], query_point=[4.0, 3.0], target_point=[-1.0, -3.0])
    return {"source": 0, "target": 2, "query_point": (4.0, 3.0), "target_point": (-1.0, -3.0), "feat": feat.clone(),
            "confidence": float(conf)}


if __name__ == "__main__":
    esp, du = import_reference_readout()
    res = {"unet": {"config": UNET, "feats": run_unet()}, "image_size": IMG,
           "human": run_branch(esp, du, True), "object": run_branch(esp, du, False), "query": run_query(du)}
    path = os.path.join(OUT, "dift.pt")
    torch.save(res, path)
    print(path, os.path.getsize(path), "bytes")
