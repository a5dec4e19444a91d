"""Host-side mirror of the reference's `SparsePointAdapter` (videoswap/models/adapter_model.py:50-136) and of the
denoising part of `VideoSwapPipeline` (videoswap/pipelines/pipeline_videoswap.py:427-619 `__call__`, :622-721 `invert`).

Scope (SURVEY.md 8): the loop body -- CFG batch duplication, UNet forward, CFG combine (with diffusers'
guidance_rescale), scheduler step (with DDIM eta), adapter residual window -- runs on the native kernels.  The pipeline
takes `prompt_embeds` (one or more videos) and either `latents` or a generator to draw them from, and returns latents.  Given a `text_encoder` (videoswap_b200.text.CLIPTextModel) and the caller's `tokenizer` it also takes prompts
(`encode_prompt`, plain or ED-LoRA); given a `vae` (videoswap_b200.vae.AutoencoderKL) it encodes the source frames for the
DDIM inversion (`prepare_image_latents`, `invert(video=...)`) and decodes the result into frames.
"""
from __future__ import annotations

import copy
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch
from torch import nn

from . import formats, ops, p2p
from .noise import randn_tensor
from .formats import bind_concept_prompt
from .scheduler import DDIMInverseScheduler, DDIMScheduler
from .spec import adapter_param_shapes
from .t2i_adapter import T2IAdapter
from .unet import AnimateDiffUNet3DModel, _Holder
from .vae import AutoencoderKL
from .weights import seeded_state_dict


@dataclass
class TuneAVideoPipelineOutput:
    videos: torch.Tensor


@dataclass
class TuneAVideoInversionPipelineOutput:
    latents: torch.Tensor


class _MLP(nn.Module):
    def __init__(self, in_dim, out_dim, mid_dim):
        super().__init__()
        self.mlp = nn.ModuleList([_Holder((mid_dim, in_dim)), nn.SiLU(), _Holder((out_dim, mid_dim))])


class SparsePointAdapter(nn.Module):
    """Same constructor/state_dict as the reference; `forward` returns NHWC fp16 maps (one per level) produced by the
    native MLP + splat kernels.  `as_nchw=True` returns the reference's [(F), C, h, w] layout instead."""

    def __init__(self, embedding_channels=1280, channels=(320, 640, 1280, 1280), downsample_rate=(8, 16, 32, 64),
                 mid_dim=128, init: str = "seeded"):
        super().__init__()
        self.model_list = nn.ModuleList([_MLP(embedding_channels, ch, mid_dim) for ch in channels])
        self.downsample_rate = list(downsample_rate)
        self.channels = list(channels)
        self.radius = 2
        if init == "seeded":
            self.load_state_dict(seeded_state_dict(adapter_param_shapes(embedding_channels, channels, mid_dim), seed=5))
        self.eval()

    @torch.no_grad()
    def forward(self, point_tracker, size, point_embedding, index_list=None, drop_rate=0.0, loss_type="global",
                scale: float = 1.0, coord_fp16: bool = True, as_nchw: bool = False) -> List[torch.Tensor]:
        if self.training:
            raise NotImplementedError("adapter training (loss mask / point dropout, adapter_model.py:72-95,107-109) is a "
                                      "'next' row (SURVEY 8f-3)")
        dev = point_embedding.device
        if dev.type != "cuda":
            raise RuntimeError("SparsePointAdapter (videoswap_b200) runs on CUDA only")
        tracks = point_tracker.squeeze(0) if point_tracker.dim() == 4 else point_tracker
        emb = point_embedding.squeeze(0) if point_embedding.dim() == 3 else point_embedding
        w, h = size
        nf, npts = tracks.shape[:2]
        mask = None
        if index_list is not None:
            mask = torch.zeros(npts, dtype=torch.int32, device=dev)
            mask[list(index_list)] = 1
        # the reference casts coordinates to the latents dtype (fp16 at inference, pipeline_videoswap.py:533)
        tr = tracks.to(device=dev, dtype=torch.float32).contiguous()
        if coord_fp16:
            tr = tracks.to(device=dev, dtype=torch.float16).float().contiguous()
        emb32 = emb.to(device=dev, dtype=torch.float32).contiguous()
        out = []
        for lv, mlp in enumerate(self.model_list):
            rate = self.downsample_rate[lv]
            p = [t.detach().to(device=dev, dtype=torch.float16).contiguous()
                 for t in (mlp.mlp[0].weight, mlp.mlp[0].bias, mlp.mlp[2].weight, mlp.mlp[2].bias)]
            m = ops.adapter_level(p[0], p[1], p[2], p[3], emb32, tr, h // rate, w // rate, rate, mask, coord_fp16, scale)
            out.append(m.permute(0, 3, 1, 2).contiguous() if as_nchw else m)
        return out


def edit_prompts(source_prompt: str, swap_cfg: Dict) -> Tuple[str, str, str]:
    """The target prompt of one `editing_prompts` entry (pipeline_videoswap.py:337-346) -> (source subject, target subject,
    target prompt).  `replace: "src -> tgt"` replaces every occurrence of src in the source prompt; `replace_other` is then
    applied to the target prompt and must occur there."""
    source_subject, target_subject = (s.strip() for s in swap_cfg["replace"].split("->"))
    if source_subject not in source_prompt:
        raise ValueError(f"replace: the source subject {source_subject!r} is not in the source prompt {source_prompt!r}")
    target_prompt = source_prompt.replace(source_subject, target_subject)
    if swap_cfg.get("replace_other"):
        source_other, target_other = (s.strip() for s in swap_cfg["replace_other"].split("->"))
        if source_other not in target_prompt:
            raise ValueError(f"replace_other: {source_other!r} is not in the target prompt {target_prompt!r}")
        target_prompt = target_prompt.replace(source_other, target_other)
    return source_subject, target_subject, target_prompt


def parse_lora_path(lora_path: str) -> Tuple[str, float, bool]:
    """`lora_path: <file>---<alpha>` -> (file, alpha, enable_edlora); a file whose path contains 'edlora' is an ED-LoRA
    (16 concept tokens per concept, prompts bound per cross-attention layer)."""
    parts = lora_path.split("---")
    if len(parts) != 2:
        raise ValueError(f"lora_path must be '<file>---<alpha>', got {lora_path!r}")
    return parts[0], float(parts[1]), "edlora" in parts[0]


def select_index_list(conditions: Dict, select_point) -> Optional[List[int]]:
    """`select_point` names -> the point columns the adapter keeps (`index_list`); None (or empty): every point."""
    if not select_point:
        return None
    return [conditions["point_name2id"][name] for name in select_point]


def draw_points(frames, conditions: Dict):
    """The `_vispoint` frames (pipeline_videoswap.py:44-83): a green disc of radius 5 at every visible (x, y >= 0) selected
    point, drawn IN PLACE on the given PIL frames; frames past the last tracked frame are left out of the returned list."""
    from PIL import ImageDraw
    tracks = conditions["pred_tracks"]
    index_list = conditions.get("index_list")
    out = []
    for idx, image in enumerate(frames):
        if idx >= len(tracks):
            continue
        draw = ImageDraw.Draw(image)
        for p in range(tracks.shape[1]):
            if index_list is not None and p not in index_list:
                continue
            x, y = (float(v) for v in tracks[idx][p])
            if x >= 0 and y >= 0:
                draw.ellipse((x - 5, y - 5, x + 5, y + 5), fill=(0, 255, 0))
        out.append(image)
    return out


def _frames_to_uint8(frames) -> torch.Tensor:
    """The PIL half of VaeImageProcessor.preprocess (diffusers 0.19.3 image_processor.py, vae_scale_factor 8, resample
    "lanczos"): each frame resized to the next lower multiple of 8 when its size is not one, then stacked as uint8
    [F, H, W, 3] for one upload.  The division by 255 and the normalisation run on the device (vae_image_in)."""
    import numpy as np
    from PIL import Image
    if isinstance(frames, Image.Image):
        frames = [frames]
    if not isinstance(frames, (list, tuple)) or not frames or not all(isinstance(f, Image.Image) for f in frames):
        raise ValueError("video must be a list of PIL images, a [F, 3, H, W] tensor or [F, 4, h, w] latents")
    arrs = []
    for f in frames:
        if f.mode != "RGB":
            raise ValueError(f"video frames must be RGB PIL images, got mode {f.mode!r}")
        w, h = (x - x % 8 for x in f.size)
        if (w, h) != f.size:
            f = f.resize((w, h), resample=Image.LANCZOS)
        arrs.append(np.asarray(f, dtype=np.uint8))
    if len({a.shape for a in arrs}) != 1:
        raise ValueError(f"video frames differ in size: {sorted({a.shape[:2] for a in arrs})}")
    return torch.from_numpy(np.stack(arrs))


class VideoSwapPipeline:
    """The denoising loop of the reference pipeline on the native path.  BASELINE.json's `TuneAVideoPipeline` alias."""

    def __init__(self, unet: AnimateDiffUNet3DModel, scheduler: Optional[DDIMScheduler] = None,
                 adapter: Optional[Union[SparsePointAdapter, T2IAdapter]] = None,
                 inverse_scheduler: Optional[DDIMInverseScheduler] = None, vae: Optional[AutoencoderKL] = None,
                 text_encoder=None, tokenizer=None):
        """adapter: a SparsePointAdapter (conditions: a TAP dict) or a T2IAdapter (conditions: a list of per-frame PIL
        images); several adapters (diffusers' MultiAdapter) are not supported.
        vae: encodes the source video for the inversion (invert(video=...)) and turns the final latents into frames
        (output_type "pt" / "np" / "pil"); without it the pipeline takes and returns latents only.
        text_encoder (text.CLIPTextModel) + tokenizer (transformers' CLIPTokenizer, or anything with its call interface):
        `prompt=` instead of `prompt_embeds` (encode_prompt)."""
        if isinstance(adapter, (list, tuple)):
            raise NotImplementedError("MultiAdapter (several adapters summed) is not implemented; give one adapter")
        self.unet = unet
        self.scheduler = scheduler or DDIMScheduler()
        self.inverse_scheduler = inverse_scheduler or DDIMInverseScheduler()
        self.adapter = adapter
        self.vae = vae
        self.text_encoder = text_encoder
        self.tokenizer = tokenizer
        self.new_concept_cfg = None

    def set_new_concept_cfg(self, new_concept_cfg=None):
        """ED-LoRA concepts (formats.load_new_concept) that encode_prompt binds into 16 per-layer prompts; None: plain
        prompts (pipeline_videoswap.py:174-176)."""
        self.new_concept_cfg = new_concept_cfg

    def _encode(self, texts: List[str]) -> torch.Tensor:
        """One batch through the text encoder: tokenizer(padding="max_length", max_length=model_max_length, truncation)
        -> last_hidden_state [len(texts), 77, 768]."""
        if self.text_encoder is None or self.tokenizer is None:
            raise ValueError("prompts need a VideoSwapPipeline(..., text_encoder=CLIPTextModel, tokenizer=CLIPTokenizer)")
        ids = self.tokenizer(texts, padding="max_length", max_length=self.tokenizer.model_max_length, truncation=True,
                             return_tensors="pt").input_ids
        return self.text_encoder(ids)[0]

    @torch.no_grad()
    def encode_prompt(self, prompt, negative_prompt=None, do_classifier_free_guidance: bool = True,
                      plain: bool = False) -> torch.Tensor:
        """Prompt embeddings, every sequence of the call in one encoder batch, uncond first under CFG:
          * no concept config (or plain=True): diffusers 0.19.3 `_encode_prompt` -> [2 b, 77, 768] (cat(neg, pos); the
            negative defaults to "");
          * with set_new_concept_cfg: `encode_edlora_prompt` (edlora_util.py:116-196) -> [2 b, 16, 77, 768]: each prompt
            bound into 16 per-layer prompts (formats.bind_concept_prompt), each negative encoded once and repeated 16 times.
        Without CFG the uncond half is left out."""
        prompts = [prompt] if isinstance(prompt, str) else list(prompt)
        b = len(prompts)
        uncond: List[str] = []
        if do_classifier_free_guidance:
            if negative_prompt is None:
                uncond = [""] * b
            elif type(prompt) is not type(negative_prompt):
                raise TypeError(f"negative_prompt should be the same type as prompt, got {type(negative_prompt)} != {type(prompt)}")
            elif isinstance(negative_prompt, str):
                uncond = [negative_prompt]
            elif len(negative_prompt) != b:
                raise ValueError(f"negative_prompt has batch size {len(negative_prompt)}, prompt has {b}")
            else:
                uncond = list(negative_prompt)
        if plain or self.new_concept_cfg is None:
            return self._encode(uncond + prompts)
        emb = self._encode(bind_concept_prompt(prompts, self.new_concept_cfg) + uncond)
        L, C = emb.shape[1:]
        pos = emb[:16 * b].view(b, 16, L, C)
        if not do_classifier_free_guidance:
            return pos
        neg = emb[16 * b:].view(b, 1, L, C).repeat(1, 16, 1, 1)
        return torch.cat([neg, pos])

    @property
    def device(self):
        return self.unet.device

    def _residuals_for_cfg(self, adapter_state, cfg: bool):
        """NHWC maps [(F),h,w,C] -> the NCHW [(B F),C,h,w] list the UNet surface takes (B = 2 under CFG)."""
        res = []
        for m in adapter_state:
            r = m.permute(0, 3, 1, 2)
            res.append(torch.cat([r, r], dim=0).contiguous() if cfg else r.contiguous())
        return res

    @torch.no_grad()
    def step_sharded(self, latents: torch.Tensor, t, embeds: torch.Tensor, guidance_scale: float, plan,
                     residuals: Optional[List[torch.Tensor]] = None, coef: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The loop body on ONE video split over ranks (dist_util.ShardPlan; SURVEY 8e).  `latents` [1,4,F/k,h,w] and
        `residuals` 4 x [(F/k),C,h,w] hold THIS rank's frames; `embeds` is the full [2,...] (uncond first).  The rank runs the
        UNet on its CFG half (batch 1; GroupNorm statistics and the motion modules exchange inside the library), the two
        halves swap their noise predictions, and both compute the same DDIM update for their frames.  It takes no eta and
        no guidance_rescale: the rescale's per-video statistics would span the frame shards."""
        from . import dist_util
        cfg = guidance_scale > 1.0
        if cfg and plan.cfg_ranks != 2:
            raise ValueError("frame sharding under CFG needs the CFG split (one batch element per rank)")
        e = embeds[plan.cfg_index:plan.cfg_index + 1] if cfg else embeds
        res = [r for r in residuals] if residuals is not None else None
        eps = self.unet(latents, t, encoder_hidden_states=e, down_block_additional_residuals=res, return_dict=False)[0]
        if cfg:
            eps = dist_util.all_gather_cfg(plan, eps)
        if coef is not None:
            return ops.cfg_ddim_step(eps, latents, guidance_scale, cfg=cfg, coef=coef)
        a_t, a_p = self.scheduler.alphas(t)
        return ops.cfg_ddim_step(eps, latents, guidance_scale, a_t, a_p, cfg=cfg)

    @torch.no_grad()
    def step(self, latents: torch.Tensor, t: int, embeds: torch.Tensor, guidance_scale: float = 7.5,
             residuals: Optional[List[torch.Tensor]] = None, *, eta: float = 0.0, guidance_rescale: float = 0.0,
             generator=None) -> torch.Tensor:
        """One loop body (pipeline_videoswap.py:556-587): CFG batch duplication -> UNet -> CFG combine -> DDIM step.
        `latents` is [b, 4, F, h, w]; `embeds` is [2 b,...] (the b uncond first) when guidance_scale > 1 else [b,...];
        `scheduler.set_timesteps` must have been called.  eta > 0 adds eta sqrt(variance) times the draw
        randn_tensor(latents.shape, generator, latents' device and dtype), as DDIMScheduler.step does; guidance_rescale > 0
        (CFG only) rescales the guided prediction toward the conditional one's standard deviation (rescale_noise_cfg).
        Both run in one fused kernel; without them the step is the eta = 0 kernel.  Returns the new latents."""
        cfg = guidance_scale > 1.0
        a_t, a_p = self.scheduler.alphas(t)
        x_in = torch.cat([latents] * 2) if cfg else latents
        x_in = self.scheduler.scale_model_input(x_in, t)
        eps = self.unet(x_in, t, encoder_hidden_states=embeds, down_block_additional_residuals=residuals, return_dict=False)[0]
        if eta == 0 and not (cfg and guidance_rescale > 0):
            return ops.cfg_ddim_step(eps, latents, guidance_scale, a_t, a_p, cfg=cfg)
        noise = randn_tensor(latents.shape, generator, latents.device, latents.dtype) if eta > 0 else None
        return ops.cfg_ddim_rescale_step(eps, latents, guidance_scale, a_t, a_p, eta=eta,
                                         guidance_rescale=guidance_rescale if cfg else 0.0, noise=noise, cfg=cfg)

    @torch.no_grad()
    def __call__(self, prompt_embeds: Optional[torch.Tensor] = None, latents: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None,
                 conditions: Optional[Dict] = None, num_inference_steps: int = 50, guidance_scale: float = 7.5,
                 t2i_guidance_scale: float = 1.0, t2i_start: float = 0.0, t2i_end: float = 1.0, controller=None,
                 output_type: str = "latent", return_dict: bool = True, callback=None, callback_steps: int = 1,
                 max_iters: Optional[int] = None, *, prompt=None, negative_prompt=None, source_prompt=None, generator=None,
                 video_length: Optional[int] = None, num_images_per_prompt: int = 1, height: Optional[int] = None,
                 width: Optional[int] = None, eta: float = 0.0, guidance_rescale: float = 0.0):
        """prompt_embeds: [b,77,D] / ED-LoRA [b,16,77,D] (conditional); negative_prompt_embeds same shape (uncond).
        Or `prompt` (+ `negative_prompt`): a string, or a list of b prompts, encoded with encode_prompt (exactly one of
        prompt and prompt_embeds).  b videos are denoised in one UNet batch; with `conditions` or a `controller` b must be 1.
        latents [b,4,F,h,w] (e.g. DDIM-inverted), or None: prepare_latents (pipeline_videoswap.py:178-202) draws them with
        randn_tensor(generator) at [b, 4, video_length, height / 8, width / 8] in the prompt embeddings' dtype (height and
        width default to unet.config.sample_size * 8) and scales them by scheduler.init_noise_sigma.  `generator`: one
        torch.Generator or a list of b.  eta > 0: DDIMScheduler.step's noise, drawn from `generator` at every step;
        guidance_rescale > 0: rescale_noise_cfg under CFG.  Mirrors pipeline_videoswap.py:552-610: output_type "latent"
        returns the latents [(b f), 4, h, w]; "pt" / "np" / "pil" decode them with the pipeline's vae (decode_latents).
        `source_prompt` is accepted and unused; `num_images_per_prompt` must be 1.
        conditions: with a SparsePointAdapter the TAP dict (pred_tracks, img_size, point_embedding, index_list); with a
        T2IAdapter one PIL image per frame (pipeline_videoswap.py:538-542, see t2i_adapter.preprocess_frames), whose
        features are computed once per call.  Either way the residuals are scaled by t2i_guidance_scale, duplicated under
        CFG and added at iterations i with len(timesteps) t2i_start <= i <= len(timesteps) t2i_end."""
        if num_images_per_prompt != 1:
            raise NotImplementedError("num_images_per_prompt must be 1 (one edited video per prompt)")
        if (prompt is None) == (prompt_embeds is None):
            raise ValueError("give exactly one of `prompt` and `prompt_embeds`")
        if prompt is not None and negative_prompt_embeds is not None:
            raise ValueError("`prompt` takes `negative_prompt`, not `negative_prompt_embeds`")
        if eta < 0:
            raise ValueError(f"eta must be >= 0, got {eta}")
        if guidance_rescale < 0:
            raise ValueError(f"guidance_rescale must be >= 0, got {guidance_rescale}")
        if prompt is not None:
            batch = 1 if isinstance(prompt, str) else len(prompt)
        else:
            batch = prompt_embeds.shape[0]
        if batch > 1 and (conditions is not None or controller is not None):
            raise ValueError("conditions and attention controllers take one video: give one prompt")
        if isinstance(generator, (list, tuple)) and len(generator) != batch:
            raise ValueError(f"{len(generator)} generators for a batch of {batch} videos")
        if latents is None and video_length is None:
            raise ValueError("drawing the latents from noise needs `video_length`")
        cond_frames = None
        if conditions is not None:
            if self.adapter is None:
                raise ValueError("conditions given but the pipeline has no adapter")
            if isinstance(self.adapter, T2IAdapter):
                if isinstance(conditions, dict):
                    raise ValueError("a T2IAdapter takes a list of per-frame PIL images as conditions, not a TAP dict")
                cond_frames = self.adapter.preprocess(conditions)           # checks only, no launch
                frames = latents.shape[2] if latents is not None else video_length
                if cond_frames.shape[0] != frames:
                    raise ValueError(f"{cond_frames.shape[0]} condition images for {frames} frames")
            elif not isinstance(conditions, dict):
                raise ValueError("a SparsePointAdapter takes a TAP dict as conditions (pred_tracks, img_size, "
                                 "point_embedding, index_list), not a list of images")
        if latents is not None and latents.shape[0] != batch:
            raise ValueError(f"latents hold {latents.shape[0]} videos, the prompts {batch}")
        if output_type != "latent":
            if self.vae is None:
                raise NotImplementedError("decoding needs a VideoSwapPipeline(..., vae=AutoencoderKL); use output_type='latent'")
            if output_type not in ("pt", "np", "pil"):
                raise ValueError(f"output_type must be 'latent', 'pt', 'np' or 'pil', got {output_type!r}")
        cfg = guidance_scale > 1.0
        dev = latents.device if latents is not None else self.device
        if prompt is not None:
            embeds = self.encode_prompt(prompt, negative_prompt, cfg)           # uncond first under CFG
        elif cfg:
            if negative_prompt_embeds is None:
                raise ValueError("classifier-free guidance needs negative_prompt_embeds")
            embeds = torch.cat([negative_prompt_embeds, prompt_embeds], dim=0)     # uncond FIRST (edlora_util.py:190-195)
        else:
            embeds = prompt_embeds
        self.scheduler.set_timesteps(num_inference_steps)
        timesteps = self.scheduler.timesteps
        if latents is None:
            latents = self.prepare_latents(batch, video_length, height, width, embeds.dtype, dev, generator)
        adapter_state = None
        if cond_frames is not None:
            adapter_state = self._residuals_for_cfg(self.adapter(cond_frames, scale=t2i_guidance_scale), cfg)
        elif conditions is not None:
            # the reference casts tracks AND the point embedding to the latents dtype first (pipeline_videoswap.py:528-533)
            emb = conditions["point_embedding"].to(dev)
            if latents.dtype == torch.float16:
                emb = emb.half()
            adapter_state = self.adapter(conditions["pred_tracks"].to(dev), conditions["img_size"], emb,
                                         index_list=conditions["index_list"], scale=t2i_guidance_scale,
                                         coord_fp16=latents.dtype == torch.float16)
            adapter_state = self._residuals_for_cfg(adapter_state, cfg)
        latents = latents.contiguous()
        for i, t in enumerate(timesteps):
            if max_iters is not None and i >= max_iters:      # truncated schedules (tests / benchmarks)
                break
            res = None
            if adapter_state is not None and len(timesteps) * t2i_start <= i <= len(timesteps) * t2i_end:
                res = list(adapter_state)        # the UNet pops from this list (no clone needed: it never writes to them)
            latents = self.step(latents, t, embeds, guidance_scale, res, eta=eta, guidance_rescale=guidance_rescale,
                                generator=generator)
            if controller is not None:           # edit the latents using the attention maps (pipeline_videoswap.py:589-593)
                latents = controller.step_callback(latents).to(latents.dtype)
            if callback is not None and i % callback_steps == 0:
                callback(i, t, latents)
        # the reference always rearranges 'b c f h w -> (b f) c h w' before returning (pipeline_videoswap.py:603-610)
        b, c, f, h, w = latents.shape
        video = latents.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
        if output_type != "latent":
            video = self.decode_latents(video, output_type)
        if not return_dict:
            return video
        return TuneAVideoPipelineOutput(videos=video)

    def prepare_latents(self, batch_size: int, video_length: int, height: Optional[int] = None, width: Optional[int] = None,
                        dtype=torch.float16, device=None, generator=None) -> torch.Tensor:
        """The initial latents of a call without given ones (pipeline_videoswap.py:178-202): randn_tensor([batch_size,
        in_channels, video_length, height // 8, width // 8], generator) * scheduler.init_noise_sigma; height and width
        default to unet.config.sample_size * 8."""
        height = height or self.unet.config.sample_size * 8
        width = width or self.unet.config.sample_size * 8
        shape = (batch_size, self.unet.config.in_channels, video_length, height // 8, width // 8)
        if isinstance(generator, (list, tuple)) and len(generator) != batch_size:
            raise ValueError(f"{len(generator)} generators for a batch of {batch_size} videos")
        latents = randn_tensor(shape, generator, device if device is not None else self.device, dtype)
        return latents * self.scheduler.init_noise_sigma

    @torch.no_grad()
    def decode_latents(self, latents: torch.Tensor, output_type: str = "pil"):
        """Frames of latents [(b f), 4, h, w] (or [b, 4, f, h, w]): image_processor.postprocess(vae.decode(latents /
        scaling_factor)) as pipeline_videoswap.py:603-610 computes it.  "pt": fp32 [(b f), 3, 8h, 8w] in [0, 1]; "np": fp32
        numpy [(b f), 8h, 8w, 3]; "pil": a list of RGB PIL images."""
        if self.vae is None:
            raise NotImplementedError("decoding needs a VideoSwapPipeline(..., vae=AutoencoderKL)")
        if latents.dim() == 5:
            b, c, f, h, w = latents.shape
            latents = latents.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
        return self.vae.decode_postprocess(latents, output_type)

    @torch.no_grad()
    def prepare_image_latents(self, video, generator=None) -> torch.Tensor:
        """VaeImageProcessor.preprocess + prepare_image_latents (pipeline_videoswap.py:204-233, 660-664): the source video
        -> fp16 latents [1, 4, F, h, w] = scaling_factor * vae.encode(frames).latent_dist.sample(generator).  video:
          * a list of RGB PIL frames (all of one size); a size that is not a multiple of 8 is resized down to one with
            LANCZOS, as preprocess does; the frames go to the device as one uint8 [F, H, W, 3] upload;
          * a [F, 3, H, W] tensor in [-1, 1] (H, W multiples of 8);
          * latents [F, 4, h, w], passed through unscaled as the reference passes them.
        generator: a torch.Generator (CPU or CUDA) or one per frame; the noise is the reference's draw for that seed."""
        if self.vae is None:
            raise ValueError("encoding a video needs a VideoSwapPipeline(..., vae=AutoencoderKL)")
        dev = self.vae.device
        if isinstance(video, torch.Tensor):
            if video.dim() != 4 or video.shape[1] not in (3, 4):
                raise ValueError(f"expected a video tensor [F, 3, H, W] or latents [F, 4, h, w], got {tuple(video.shape)}")
            if video.shape[1] == 4:
                lat = video.to(device=dev, dtype=torch.float16)
                return lat.permute(1, 0, 2, 3).unsqueeze(0).contiguous()
            dist = self.vae.encode(video.to(dev).contiguous()).latent_dist
        else:
            frames = _frames_to_uint8(video)
            dist = self.vae.encode_frames(frames.to(dev))
        return dist.sample(generator, scale=self.vae.config.scaling_factor, video=True)

    @torch.no_grad()
    def invert(self, prompt_embeds: Optional[torch.Tensor] = None, latents: Optional[torch.Tensor] = None,
               num_inference_steps: int = 50, return_dict: bool = True, controller=None, max_iters: Optional[int] = None, *,
               video=None, generator=None, prompt=None):
        """DDIM inversion loop (pipeline_videoswap.py:677-703), guidance_scale = 1 (no CFG).  The UNet is evaluated at
        the inverse scheduler's timestep; which noise levels the step connects is the scheduler's `convention`.
        Exactly one of `latents` ([1, 4, F, h, w]) and `video` (see prepare_image_latents, with `generator`) is given, and
        exactly one of `prompt_embeds` and `prompt`; a prompt is encoded plainly even with a concept config, as the
        reference's invert does (pipeline_videoswap.py:658)."""
        if (prompt is None) == (prompt_embeds is None):
            raise ValueError("give exactly one of `prompt` and `prompt_embeds`")
        if (latents is None) == (video is None):
            raise ValueError("invert takes exactly one of `latents` and `video`")
        if prompt is not None:
            prompt_embeds = self.encode_prompt(prompt, do_classifier_free_guidance=False, plain=True)
        if video is not None:
            latents = self.prepare_image_latents(video, generator)
        self.inverse_scheduler.set_timesteps(num_inference_steps)
        latents = latents.contiguous()
        for i, t in enumerate(self.inverse_scheduler.timesteps):
            if max_iters is not None and i >= max_iters:
                break
            eps = self.unet(latents, t, encoder_hidden_states=prompt_embeds, return_dict=False)[0]
            a_cur, a_next = self.inverse_scheduler.alphas(t)
            latents = ops.cfg_ddim_step(eps, latents, 1.0, a_cur, a_next, cfg=False)
            if controller is not None:           # store the maps / latents of this inversion step (pipeline_videoswap.py:698-702)
                latents = controller.step_callback(latents).to(latents.dtype)
        if not return_dict:
            return latents
        return TuneAVideoInversionPipelineOutput(latents=latents.detach().clone())

    @torch.no_grad()
    def validation(self, source_video, source_conditions, source_prompt: str, editing_config: Dict,
                   dtype=torch.float16, train_dataset=None, save_dir=None) -> Dict:
        """The reference's `validation` (pipeline_videoswap.py:272-423), which its test.py runs on an `editing_config`:
        invert the source video once, then run every entry of `editing_prompts` and return {key: list of PIL frames} (plus
        `key + '_vispoint'` with `visualize_point`).

          * Inversion: `invert(prompt=source_prompt, video=source_video)` over `num_inference_steps`; with `use_blend` a
            p2p.AttentionStore (LOW_RESOURCE: no CFG) records the maps and latents and is removed afterwards.  The VAE
            sample uses torch's default generator, as the reference's does.
          * Per edit: `lora_path: <file>---<alpha>` is merged into the UNet and the text encoder (ED-LoRA files -- 'edlora'
            in the path -- also add their concept tokens and bind the prompts) and restored bit-exactly after the edit; the
            concept tokens stay in the tokenizer and the token embedding.  Conditions come from
            `train_dataset.get_conditions(tap_path)` or a copy of `source_conditions`, with `select_point` -> index_list.
            The target prompt is built by edit_prompts.  With `use_blend` the edit runs under p2p.make_controller's
            AttentionRefine (latent and self-attention blending on the subject words, blend_cfg's steps and blend_th).
            guidance_scale, t2i_guidance_scale and negative_prompt are taken from the entry first, then from the config.

        Needs the pipeline's vae, text_encoder and tokenizer.  `save_dir` is only used by `visualize_attention`, which is
        not supported (it renders with the reference's show_cross_attention)."""
        missing = [n for n in ("vae", "text_encoder", "tokenizer") if getattr(self, n) is None]
        if missing:
            raise ValueError(f"validation needs a VideoSwapPipeline with {', '.join(missing)}")
        if editing_config.get("visualize_attention", False):
            raise NotImplementedError("visualize_attention renders maps with the reference's show_cross_attention, "
                                      "which is not part of this package")
        if not editing_config["use_invertion_latents"]:
            raise ValueError("validation edits the DDIM inversion of the source video: use_invertion_latents must be true")
        steps = editing_config["num_inference_steps"]
        use_blend = editing_config.get("use_blend", False)

        store = None
        if use_blend:
            store = p2p.AttentionStore()
            store.LOW_RESOURCE = True
            p2p.register_attention_control(self, store)
        try:
            inverted = self.invert(prompt=source_prompt, video=source_video, num_inference_steps=steps,
                                   controller=store).latents.to(dtype)
        finally:
            if use_blend:
                p2p.register_attention_control(self, None)

        results: Dict = {}
        for key, swap_cfg in editing_config["editing_prompts"].items():
            unet_backup = te_backup = None
            controller = None
            try:
                if swap_cfg.get("lora_path") is not None:
                    path, alpha, enable_edlora = parse_lora_path(swap_cfg["lora_path"])
                    lora = formats.load_edlora(path)
                    concept_cfg = None
                    if enable_edlora and lora["new_concept_embedding"]:
                        concept_cfg = formats.load_new_concept(self.tokenizer, self.text_encoder,
                                                               lora["new_concept_embedding"], enable_edlora=True)
                    unet_backup = formats.merge_edlora_into_unet(self.unet, lora["unet"], alpha)
                    te_backup = formats.merge_edlora_into_text_encoder(self.text_encoder, lora["text_encoder"], alpha)
                    if enable_edlora:
                        self.set_new_concept_cfg(concept_cfg)

                if source_conditions is not None and swap_cfg.get("tap_path"):
                    if train_dataset is None:
                        raise ValueError(f"{key}: tap_path needs a train_dataset with get_conditions(tap_path)")
                    conditions = train_dataset.get_conditions(swap_cfg["tap_path"])
                else:
                    conditions = copy.deepcopy(source_conditions)
                if conditions is not None:
                    conditions["index_list"] = select_index_list(conditions, swap_cfg.get("select_point"))

                source_subject, target_subject, target_prompt = edit_prompts(source_prompt, swap_cfg)
                if use_blend:
                    width, height = source_video[0].size
                    blend_cfg = swap_cfg.get("blend_cfg") or {}
                    th = blend_cfg.get("blend_th", 0.3)
                    controller = p2p.make_controller(
                        self.tokenizer, [source_prompt, target_prompt], is_replace_controller=False,
                        cross_replace_steps=blend_cfg.get("cross_replace_steps", 0.0),
                        self_replace_steps=blend_cfg.get("self_replace_steps", 0.0),
                        blend_words=[source_subject.split(" "), target_subject.split(" ")], additional_attention_store=store,
                        blend_th=(th, th), NUM_DDIM_STEPS=steps, blend_latents=True, blend_self_attention=True,
                        image_height=height, image_width=width, new_concept_cfg=self.new_concept_cfg,
                        device=inverted.device)
                    p2p.register_attention_control(self, controller)

                def pick(name, default):
                    return swap_cfg[name] if name in swap_cfg else editing_config.get(name, default)

                frames = self(prompt=target_prompt, negative_prompt=pick("negative_prompt", None), conditions=conditions,
                              latents=inverted, num_inference_steps=steps, guidance_scale=pick("guidance_scale", 7.5),
                              t2i_guidance_scale=pick("t2i_guidance_scale", 1.0),
                              t2i_start=editing_config.get("t2i_start", 0.0), t2i_end=editing_config.get("t2i_end", 1.0),
                              controller=controller, output_type="pil").videos
                results[key] = copy.deepcopy(frames)
                if conditions is not None and editing_config.get("visualize_point", False):
                    results[key + "_vispoint"] = draw_points(frames, conditions)
            finally:
                if controller is not None:
                    p2p.register_attention_control(self, None)
                if unet_backup is not None:
                    formats.restore_unet(self.unet, unet_backup)
                if te_backup is not None:
                    formats.restore_text_encoder(self.text_encoder, te_backup)
                if swap_cfg.get("lora_path") is not None:
                    self.set_new_concept_cfg(None)
        return results


class GraphedStep:
    """One loop body (CFG duplication -> UNet -> CFG combine -> DDIM update) captured once in a CUDA graph and replayed
    for every timestep: the timestep and the two DDIM coefficients live in device memory (3 floats uploaded from a
    pinned host buffer before each replay), everything else (weights, embeddings, adapter residuals, workspace) is
    static.  Removes ~750 kernel-launch gaps per step.

    With eta > 0 or guidance_rescale > 0 (CFG) the update is the fused rescale / stochastic-DDIM kernel and the device
    vector also holds c_n and the rescale factor (5 floats); with eta > 0 a static noise buffer is filled eagerly from
    the call's generator before each replay, so the graph never draws and the draws are randn_tensor's."""

    def __init__(self, pipe: VideoSwapPipeline, latents: torch.Tensor, embeds: torch.Tensor, guidance_scale: float = 7.5,
                 residuals: Optional[List[torch.Tensor]] = None, inverse: bool = False, plan=None, *, eta: float = 0.0,
                 guidance_rescale: float = 0.0):
        """inverse=True: the DDIM-inversion loop body (pipeline_videoswap.py:677-696, no CFG) -- `__call__` then takes the
        inverse scheduler's timesteps and coefficients.  eta / guidance_rescale: as VideoSwapPipeline.step (not with
        inverse=True or a frame-sharding plan)."""
        self.pipe, self.guidance, self.residuals, self.inverse = pipe, guidance_scale, residuals, inverse
        self.plan = plan if (plan is not None and plan.world > 1) else None    # sharded: latents / residuals are this rank's frames
        if eta < 0 or guidance_rescale < 0:
            raise ValueError("eta and guidance_rescale must be >= 0")
        self.eta = float(eta)
        self.rescale = float(guidance_rescale) if guidance_scale > 1.0 else 0.0     # no rescale without CFG
        self.stochastic = self.eta > 0 or self.rescale > 0
        if self.stochastic and (inverse or self.plan is not None):
            raise ValueError("eta and guidance_rescale apply to the single-process denoising loop only")
        if inverse:
            assert guidance_scale <= 1.0 and residuals is None, "the inversion loop runs without CFG and without adapter residuals"
            if pipe.inverse_scheduler.num_inference_steps is None:
                pipe.inverse_scheduler.set_timesteps(pipe.scheduler.num_inference_steps or 50)
        dev = latents.device
        self.lat = latents.clone().contiguous()
        self.embeds = embeds.contiguous()
        self.noise = torch.zeros_like(self.lat) if self.eta > 0 else None
        nd = 5 if self.stochastic else 3                                  # timestep, c_x, c_e (, c_n, rescale)
        self._h = torch.zeros(nd, dtype=torch.float32).pin_memory()
        self._d = torch.zeros(nd, dtype=torch.float32, device=dev)
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            self._d.copy_(torch.tensor([1.0, 1.0, 0.0, 0.0, 0.0][:nd]))
            for _ in range(2):                                          # warm-up: workspace + weights in place
                self._body()
        cur.wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = self._body()
        # the graph holds raw pointers into the UNet's workspace arena: forbid its re-allocation while this object lives
        from . import _lib
        self._pinned = pipe.unet._handle
        _lib.call("vs_unet_pin_workspace", self._pinned, 1)

    def __del__(self):
        try:
            if getattr(self, "_pinned", None) is not None:
                from . import _lib
                _lib.lib().vs_unet_pin_workspace(self._pinned, 0)
        except Exception:  # noqa: BLE001
            pass

    def _body(self):
        if self.plan is not None:      # the NCCL exchanges are captured with the kernels
            return self.pipe.step_sharded(self.lat, self._d[0:1], self.embeds, self.guidance, self.plan, self.residuals,
                                          coef=self._d[1:3])
        cfg = self.guidance > 1.0
        x_in = torch.cat([self.lat] * 2) if cfg else self.lat
        res = list(self.residuals) if self.residuals is not None else None
        eps = self.pipe.unet(x_in, self._d[0:1], encoder_hidden_states=self.embeds, down_block_additional_residuals=res,
                             return_dict=False)[0]
        if self.stochastic:
            return ops.cfg_ddim_rescale_step(eps, self.lat, self.guidance, noise=self.noise, cfg=cfg, coef=self._d[1:5])
        return ops.cfg_ddim_step(eps, self.lat, self.guidance, cfg=cfg, coef=self._d[1:3])

    def __call__(self, latents: torch.Tensor, t: int, generator=None) -> torch.Tensor:
        """Runs the step at timestep t.  The returned tensor is overwritten by the next call.  With eta > 0 the step's
        noise is drawn from `generator` (a torch.Generator, a list of one per video, or None) before the replay."""
        a_t, a_p = (self.pipe.inverse_scheduler if self.inverse else self.pipe.scheduler).alphas(t)
        if self.stochastic:
            c_x, c_e, c_n = ops.ddim_coefficients(a_t, a_p, self.eta)
            vals = [float(t), c_x, c_e, c_n, self.rescale]
            if self.noise is not None:
                self.noise.copy_(randn_tensor(self.lat.shape, generator, self.lat.device, self.lat.dtype), non_blocking=True)
        else:
            c_x, c_e = ops.ddim_coefficients(a_t, a_p)      # the same update serves both directions: x' = c_x x + c_e eps
            vals = [float(t), c_x, c_e]
        # a fresh pinned staging tensor per call: torch's caching host allocator keeps it alive until the async copy ran
        h = torch.tensor(vals, dtype=torch.float32).pin_memory()
        self._d.copy_(h, non_blocking=True)
        if latents.data_ptr() != self.lat.data_ptr():
            self.lat.copy_(latents, non_blocking=True)
        self.graph.replay()
        return self.out


TuneAVideoPipeline = VideoSwapPipeline
