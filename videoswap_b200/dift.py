"""Semantic points on the native path: the DIFT half of the reference's extract_semantic_point.py (lines 114-204) and
videoswap/utils/dift_util.py, which turns tracked points into the `point_embedding [P, 1280]` of a TAP dict
(formats.load_tap).  Point tracking itself (Co-Tracker, OpenPose) is not part of this package.

The featurizer (SDFeaturizer) runs, per frame: the VAE encoder once (the reference encodes the frame E times,
`img_tensor.repeat(E)`; encoding is per image, so the E posterior draws have the same distribution), the posterior draw and
DDPM add_noise at t (the dift_noise kernel), and the 2-D SD UNet as far as up_blocks[up_ft_index] with its up-sampler
(vs_unet_forward_features; the motion modules of a 3-D UNet are skipped, so one set of weights serves both).  Several
frames go into one UNet call with the E members of each frame on the batch axis.

The read-out (extract_point_embedding, DIFT_Demo.query) never builds the up-sampled 1280 x H x W map: dift_point_sample
reads nn.Upsample(size=(H, W), mode="bilinear") at the tracked pixels only, and dift_point_reduce gives the cosine
confidences and the per-point means.  The reference's semantics, quirks included, are kept exactly:

  * Coordinates are rounded with np.round, half to even (2.5 -> 2, -0.5 -> 0).  Frame i's points are pred_tracks[i],
    as (x, y).
  * Human branch (is_human=True): a point counts in a frame iff both ROUNDED coordinates are >= 0, so x = -0.4 counts
    as visible at column 0.  A visible point whose rounded x >= width or y >= height is an IndexError in the reference;
    here it raises ValueError naming the frame and the point.  The tracks are returned unchanged.
  * Object branch (is_human=False): the keyframe is featurized first, with its own noise, and its rounded points are
    the source points.  For each frame and point, a target whose rounded x >= width or y >= height is set to (-1, -1)
    and skipped.  Negative target (and source) coordinates are NOT rejected: they index from the end as Python does,
    so -1 reads the last row or column; below -size the reference raises IndexError, here ValueError.  A target is
    accepted iff its cosine confidence against the source vector is >= 0.35 (CONFIDENCE_THRESHOLD); a rejected
    target is set to (-1, -1) in pred_tracks.
  * The reference's source points are a VIEW of pred_tracks[keyframe]: once the keyframe's own frame has been
    processed, a point it rejected or skipped is (-1, -1) and every later frame reads its source vector at the last
    row and column.  Frames here are walked in frame-index order, so frames before the keyframe (and the keyframe
    itself) use the original source points and later frames the updated ones.  (The reference walks
    Path.iterdir(), unsorted, so there the split depends on the file system.)
  * Embeddings are sums over accepted frames in frame order divided by the count, in fp32; a point never accepted
    keeps a zero embedding.
  * Noise: for each featurized frame, in order, the posterior noise [E, 4, h, w] and then the add_noise noise
    [E, 4, h, w] (the reference's `latent_dist.sample()` and `randn_like`), fp32, from `generator` (a torch.Generator
    on the CPU or the device) or, with None, from the device's default generator.  In the object branch the keyframe
    draws first, then the frames in index order.
"""
from __future__ import annotations

import os
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from . import ops
from .scheduler import DDIMScheduler

CONFIDENCE_THRESHOLD = 0.35


def round_half_even(t: torch.Tensor) -> torch.Tensor:
    """np.round of the coordinates (half to even), as int64."""
    return torch.round(t).to(torch.int64)


def accepts(conf: torch.Tensor) -> torch.Tensor:
    """The object branch's test `confidence >= confidence_threshold`."""
    return conf >= CONFIDENCE_THRESHOLD


def wrap_index(i: torch.Tensor, size: int) -> torch.Tensor:
    """Python indexing of one axis: i < 0 counts from the end (the caller has rejected i >= size and i < -size)."""
    return torch.where(i < 0, i + size, i)


class _NativeReadOut:
    """The read-out kernels (ops); tests substitute a CPU emulation of the same arithmetic."""
    sample = staticmethod(ops.dift_point_sample)
    cosine = staticmethod(ops.dift_point_cosine)
    reduce = staticmethod(ops.dift_point_reduce)


def _draw_noise(n: int, E: int, h: int, w: int, generator, device):
    """(eps1, eps2) fp32 [n E, 4, h, w] on `device`: per frame the posterior draw [E, 4, h, w], then the add_noise draw."""
    if generator is not None and generator.device.type == "cpu":
        dev = torch.device("cpu")
    else:
        dev = torch.device(device)
    e1, e2 = [], []
    for _ in range(n):
        e1.append(torch.randn((E, 4, h, w), generator=generator, device=dev, dtype=torch.float32))
        e2.append(torch.randn((E, 4, h, w), generator=generator, device=dev, dtype=torch.float32))
    return torch.cat(e1).to(device).contiguous(), torch.cat(e2).to(device).contiguous()


class SDFeaturizer:
    """DIFT's SDFeaturizer (dift_util.py:185-227) on the native UNet, VAE encoder and text encoder.

    unet: AnimateDiffUNet3DModel (motion modules, if any, are skipped); vae: AutoencoderKL with its encoder half;
    text_encoder: text.CLIPTextModel; tokenizer: transformers' CLIPTokenizer (or anything with its call interface)."""

    def __init__(self, unet, vae, text_encoder, tokenizer, scheduler: Optional[DDIMScheduler] = None):
        from .pipeline import VideoSwapPipeline
        self.unet, self.vae = unet, vae
        self.scheduler = scheduler or DDIMScheduler()
        # prompts go through the pipeline's own encoder call (plain, no classifier-free guidance)
        self._pipe = VideoSwapPipeline(unet, self.scheduler, vae=vae, text_encoder=text_encoder, tokenizer=tokenizer)
        self._prompts = {}

    @classmethod
    def from_pretrained(cls, path: str, device="cuda"):
        """A local SD-1.5-style diffusers directory (unet/, vae/, text_encoder/, tokenizer/); the UNet is built without
        motion modules."""
        from transformers import CLIPTokenizer

        from .text import CLIPTextModel
        from .unet import AnimateDiffUNet3DModel
        from .vae import AutoencoderKL
        unet = AnimateDiffUNet3DModel.from_pretrained_2d(path, subfolder="unet",
                                                         unet_additional_kwargs={"use_motion_module": False})
        unet = unet.half().to(device)
        vae = AutoencoderKL.from_pretrained(path, subfolder="vae", device=device)
        text = CLIPTextModel.from_pretrained(path, subfolder="text_encoder", device=device)
        tok = CLIPTokenizer.from_pretrained(os.path.join(path, "tokenizer"))
        return cls(unet, vae, text, tok)

    def encode_prompt(self, prompt: str) -> torch.Tensor:
        """[1, 77, 768] fp16: `_encode_prompt(prompt, do_classifier_free_guidance=False)` (cached per prompt)."""
        if prompt not in self._prompts:
            self._prompts[prompt] = self._pipe.encode_prompt(prompt, do_classifier_free_guidance=False, plain=True)
        return self._prompts[prompt]

    def _alphas(self, t: int):
        a = self.scheduler.alphas_cumprod[int(t)]
        return float(a ** 0.5), float((1 - a) ** 0.5)

    @torch.no_grad()
    def features(self, images: torch.Tensor, prompt: str, t: int = 261, up_ft_index: int = 1, ensemble_size: int = 8,
                 generator=None) -> torch.Tensor:
        """up_ft[up_ft_index] of every ensemble member of n images: NHWC fp16 [n, E, h_k, w_k, C_k].  images: uint8 RGB
        frames [n, H, W, 3] or float images [n, 3, H, W] in [-1, 1] (H, W multiples of 8)."""
        if not 0 <= int(up_ft_index) <= 3:
            raise ValueError(f"up_ft_index must be in 0..3, got {up_ft_index}")
        if not 0 <= int(t) < len(self.scheduler.alphas_cumprod):
            raise ValueError(f"t must be in [0, {len(self.scheduler.alphas_cumprod)}), got {t}")
        dev = self.vae.device
        images = images.to(dev)
        if images.dtype == torch.uint8:
            moments = self.vae.encode_frames(images).parameters
        else:
            moments = self.vae.encode(images.contiguous()).latent_dist.parameters
        n, _, h, w = moments.shape
        E = int(ensemble_size)
        eps1, eps2 = _draw_noise(n, E, h, w, generator, dev)
        sa, sb = self._alphas(t)
        x = ops.dift_noise(moments, eps1, eps2, self.vae.config.scaling_factor, sa, sb)
        emb = self.encode_prompt(prompt)
        ehs = emb.expand(n * E, *emb.shape[1:])
        feat = self.unet.forward_features(x, int(t), ehs, up_ft_index)
        return feat.view(n, E, *feat.shape[1:])

    @torch.no_grad()
    def forward(self, img_tensor: torch.Tensor, prompt: str, t: int = 261, up_ft_index: int = 1, ensemble_size: int = 8,
                generator=None) -> torch.Tensor:
        """The reference's forward: img_tensor [1, 3, H, W] or [3, H, W] in [-1, 1] -> the ensemble mean of
        up_ft[up_ft_index], fp32 [1, C, h, w]."""
        if img_tensor.dim() == 3:
            img_tensor = img_tensor[None]
        if img_tensor.dim() != 4 or img_tensor.shape[0] != 1 or img_tensor.shape[1] != 3:
            raise ValueError(f"expected one image [1, 3, H, W] or [3, H, W], got {tuple(img_tensor.shape)}")
        return ops.dift_ensemble_mean(self.features(img_tensor.float(), prompt, t, up_ft_index, ensemble_size, generator))

    __call__ = forward


def _nhwc(dift: torch.Tensor) -> torch.Tensor:
    """An NCHW [1, C, h, w] map as the NHWC fp16 [1, 1, h, w, C] the read-out kernels take."""
    return dift.permute(0, 2, 3, 1).to(torch.float16).contiguous()[:, None]


def _checked_pixel(v, size: int, what: str) -> int:
    i = int(round_half_even(torch.as_tensor(v, dtype=torch.float32)))
    if not -size <= i < size:
        raise ValueError(f"{what} {i} is outside an image axis of {size} pixels")
    return i + size if i < 0 else i


class DIFT_Demo:
    """dift_util.py:230-267 without the full cosine map: `query` reads the up-sampled source and target maps at the two
    points only.  The maps are read as fp16 (the precision of the native featurizer's output)."""

    def __init__(self, source_img, source_dift: torch.Tensor, source_img_size):
        self.source_img = source_img
        self.source_dift = source_dift
        self.source_img_size = tuple(int(s) for s in source_img_size)

    @torch.no_grad()
    def query(self, target_img, target_dift, target_img_size, query_point, target_point, visualize=False):
        """query_point / target_point = (y, x).  Returns (dift_feat fp32 [C], confidence, None)."""
        if visualize:
            raise NotImplementedError("the DIFT heat-map visualisation is not part of videoswap_b200")
        Hs, Ws = self.source_img_size
        Ht, Wt = (int(s) for s in target_img_size)
        dev = target_dift.device
        sxy = torch.tensor([[[_checked_pixel(query_point[1], Ws, "source x"),
                              _checked_pixel(query_point[0], Hs, "source y")]]], dtype=torch.int32, device=dev)
        txy = torch.tensor([[[_checked_pixel(target_point[1], Wt, "target x"),
                              _checked_pixel(target_point[0], Ht, "target y")]]], dtype=torch.int32, device=dev)
        src = ops.dift_point_sample(_nhwc(self.source_dift.to(dev)), (Hs, Ws), sxy)[0]
        tgt = ops.dift_point_sample(_nhwc(target_dift), (Ht, Wt), txy)
        conf = ops.dift_point_cosine(tgt, src, torch.zeros((1, 1), dtype=torch.int32, device=dev))
        return tgt[0, 0], float(conf[0, 0]), None


def read_out(pred_tracks: torch.Tensor, featurize: Callable[[List[int]], torch.Tensor], size, is_human: bool,
             keyframe_index: Optional[int] = None, frames_per_batch: int = 8, kernels=_NativeReadOut):
    """The point read-out of extract_point_embedding over any featurizer: featurize(frame indices) -> NHWC fp16
    [n, E, h, w, C] on the device.  Returns (point_embedding fp32 [P, C] on the CPU, the (filtered) tracks, the cosine
    confidences fp32 [frames, P] of the object branch with NaN where a target was skipped, or None)."""
    H, W = (int(s) for s in size)
    tracks = pred_tracks.detach().to("cpu", torch.float32).clone()
    if tracks.dim() != 3 or tracks.shape[2] != 2:
        raise ValueError(f"pred_tracks must be [frames, points, 2], got {tuple(tracks.shape)}")
    n, P = tracks.shape[:2]
    r = round_half_even(tracks)
    rx, ry = r[..., 0], r[..., 1]
    kf_feat = conf = None
    if is_human:
        valid = (rx >= 0) & (ry >= 0)
        bad = valid & ((rx >= W) | (ry >= H))
        if bad.any():
            f, p = (int(v) for v in bad.nonzero()[0])
            raise ValueError(f"frame {f}, point {p}: rounded (x, y) = ({int(rx[f, p])}, {int(ry[f, p])}) is outside the "
                             f"{W}x{H} image")
        xy = torch.where(valid[..., None], r, 0)
    else:
        if keyframe_index is None or not 0 <= int(keyframe_index) < n:
            raise ValueError(f"the object branch needs a keyframe_index in [0, {n}), got {keyframe_index}")
        kf = int(keyframe_index)
        kf_feat = featurize([kf])
        valid = (rx < W) & (ry < H)                        # rounded x >= width or y >= height: (-1, -1) and skipped
        under = valid & ((rx < -W) | (ry < -H))
        if under.any():
            f, p = (int(v) for v in under.nonzero()[0])
            raise ValueError(f"frame {f}, point {p}: rounded (x, y) = ({int(rx[f, p])}, {int(ry[f, p])}) indexes before "
                             f"the start of the {W}x{H} image")
        xy = torch.where(valid[..., None], torch.stack([wrap_index(rx, W), wrap_index(ry, H)], -1), 0)
    vecs = []
    dev = None
    for i0 in range(0, n, frames_per_batch):
        idx = list(range(i0, min(n, i0 + frames_per_batch)))
        feat = featurize(idx)
        dev = feat.device
        vecs.append(kernels.sample(feat, (H, W), xy[idx].to(device=dev, dtype=torch.int32).contiguous()))
    vecs = torch.cat(vecs)
    if not is_human:
        def sources(row, frames):
            """Source vectors at the rounded keyframe points `row` [P, 2], for points some frame in `frames` reads."""
            sr = round_half_even(row)
            needed = valid[frames].any(0)
            bad = needed & ((sr[:, 0] >= W) | (sr[:, 1] >= H) | (sr[:, 0] < -W) | (sr[:, 1] < -H))
            if bad.any():
                p = int(bad.nonzero()[0])
                raise ValueError(f"keyframe {kf}, point {p}: rounded source (x, y) = ({int(sr[p, 0])}, {int(sr[p, 1])}) "
                                 f"is outside the {W}x{H} image")
            sxy = torch.where(needed[:, None], torch.stack([wrap_index(sr[:, 0], W), wrap_index(sr[:, 1], H)], -1), 0)
            return kernels.sample(kf_feat, (H, W), sxy[None].to(device=dev, dtype=torch.int32).contiguous())[0]

        src_a = sources(tracks[kf], slice(0, kf + 1))
        row = torch.arange(P, dtype=torch.int32, device=dev)[None]
        conf_kf = kernels.cosine(vecs[kf:kf + 1].contiguous(), src_a, row.contiguous()).cpu()[0]
        kept = valid[kf] & accepts(conf_kf)
        row_b = torch.where(kept[:, None], tracks[kf], torch.tensor(-1.0))   # the keyframe row after its own frame
        src_b = sources(row_b, slice(kf + 1, n)) if kf + 1 < n else src_a
        src_row = (torch.arange(P)[None] + P * (torch.arange(n)[:, None] > kf)).to(device=dev, dtype=torch.int32)
        conf = kernels.cosine(vecs, torch.cat([src_a, src_b]).contiguous(), src_row.contiguous()).cpu()
        conf = torch.where(valid, conf, torch.tensor(float("nan")))
        valid = valid & accepts(conf)
        tracks[~valid] = -1.0
    _, _, means = kernels.reduce(vecs, valid.to(device=dev))
    return means.cpu(), tracks, conf


@torch.no_grad()
def extract_point_embedding(tap_dict: dict, frames: Sequence, featurizer: SDFeaturizer, subject_category: str,
                            is_human: bool, keyframe_index: Optional[int] = None, frames_per_batch: int = 8,
                            generator=None) -> dict:
    """extract_semantic_point.py:125-204: frames (a list of RGB PIL images of one size, both sides multiples of 8;
    frame i is pred_tracks[i]) and a TAP dict {'pred_tracks': [frames, P, 2], 'point_name2id': ...} -> a new TAP dict
    with 'point_embedding' fp32 [P, C] (C = 1280) on the CPU and, in the object branch, the filtered 'pred_tracks'.  The
    prompt is f"photo of a {subject_category}"; frames_per_batch frames share one UNet call.  The input dict is not
    modified.  See the module docstring for the semantics."""
    from PIL import Image
    frames = list(frames)
    if not frames or not all(isinstance(f, Image.Image) and f.mode == "RGB" for f in frames):
        raise ValueError("frames must be a non-empty list of RGB PIL images")
    sizes = {f.size for f in frames}
    if len(sizes) != 1:
        raise ValueError(f"frames differ in size: {sorted(sizes)}")
    W, H = frames[0].size
    if W % 8 or H % 8:
        raise ValueError(f"frame size {W}x{H} is not a multiple of 8")
    tracks = tap_dict["pred_tracks"]
    if tracks.shape[0] != len(frames):
        raise ValueError(f"pred_tracks has {tracks.shape[0]} frames, {len(frames)} frames were given")
    if frames_per_batch < 1:
        raise ValueError("frames_per_batch must be >= 1")
    prompt = f"photo of a {subject_category}"
    dev = featurizer.vae.device
    u8 = torch.from_numpy(np.stack([np.asarray(f, dtype=np.uint8) for f in frames]))

    def featurize(idx):
        return featurizer.features(u8[idx].to(dev), prompt, generator=generator)

    emb, filtered, _ = read_out(tracks, featurize, (H, W), is_human, keyframe_index, frames_per_batch)
    out = dict(tap_dict)
    out["point_embedding"] = emb
    if not is_human:
        out["pred_tracks"] = filtered.to(tracks.dtype)
    return out
