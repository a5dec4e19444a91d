"""On-disk formats either side of the denoising path (SURVEY.md §8f-4, the data-format half): what the reference's
`test.py` / `validation()` read from disk before the loop starts, turned into the tensors the native path takes.

  TAP.pth            {pred_tracks [T,P,2], point_name2id {name: column}, point_embedding [P,1280]}
                     (videoswap/data/frame_point_dataset.py:62-70)                    -> `conditions` of VideoSwapPipeline.__call__
  adapter.pth        SparsePointAdapter state dict (test.py:69)                       -> `load_adapter`
  motion module ckpt AnimateDiff `mm_sd_v15*.ckpt`, keys `...pos_encoder.pe` -> `...processor.pos_encoder.pe` (test.py:62-64)
  ED-LoRA .pth       {params: {new_concept_embedding, unet, text_encoder}} (utils/convert_edlora_to_diffusers.py:84-103):
                     new concept tokens and their embedding rows (`load_new_concept`), then
                     W <- W + alpha * up @ down for every UNet / text-encoder weight that has a `lora_down` / `lora_up` pair

Host-side, once per edit -- torch is the plumbing here (file I/O, a rank-4 matmul per weight); no kernel of the library is
involved and none of this runs inside the timed step.  The text side works on the native `CLIPTextModel` (text.py) and
the caller's tokenizer (transformers' CLIPTokenizer).  Nothing here imports `oracle/`.
"""
from __future__ import annotations

import copy
import os
from collections import OrderedDict
from typing import Dict, Iterable, List, Mapping, Optional, Sequence, Tuple, Union

import torch

PathOrDict = Union[str, os.PathLike, Mapping]


def _load(obj: PathOrDict):
    if isinstance(obj, (str, os.PathLike)):
        return torch.load(os.fspath(obj), map_location="cpu", weights_only=False)
    return obj


# ------------------------------------------------------------------------------------------------------- TAP.pth
def select_frame_idx(begin_frame_idx: int, end_frame_idx: int, n: int) -> List[int]:
    """Frames a clip is sub-sampled to (frame_point_dataset.py:13-22): a fixed INTEGER stride `total // (n - 1)` from `begin`
    (so the last selected frame is generally not the last frame of the clip)."""
    if n < 2:
        raise ValueError("select_frame_idx needs n >= 2 (the reference divides by n - 1)")
    step = (end_frame_idx - begin_frame_idx) // (n - 1)
    return [int(begin_frame_idx + i * step) for i in range(n)]


def load_tap(tap: PathOrDict, select_id: Optional[Sequence[int]] = None, img_size: Optional[Tuple[int, int]] = None,
             select_point: Optional[Iterable[str]] = None) -> Dict:
    """`SingleVideoPointDataset.get_conditions(tap_path)` (frame_point_dataset.py:62-70) + the `select_point` handling of
    `validation()` (pipeline_videoswap.py:327-334).  Returns the `conditions` dict `VideoSwapPipeline.__call__` consumes:
    pred_tracks [F,P,2] (pixel coordinates, negative = invisible), point_embedding [P,1280], point_name2id, img_size
    (WIDTH, HEIGHT -- the reference passes `(size_x, size_y)`), index_list (columns of the selected points, or None)."""
    d = _load(tap)
    for k in ("pred_tracks", "point_name2id", "point_embedding"):
        if k not in d:
            raise KeyError(f"TAP file has no '{k}' (expected pred_tracks, point_name2id, point_embedding)")
    tracks, emb, name2id = d["pred_tracks"], d["point_embedding"], d["point_name2id"]
    tracks = torch.as_tensor(tracks)
    emb = torch.as_tensor(emb)
    if tracks.dim() != 3 or tracks.shape[-1] != 2:
        raise ValueError(f"pred_tracks must be [T, P, 2], got {tuple(tracks.shape)}")
    if tracks.shape[1] != emb.shape[0]:
        raise ValueError(f"pred_tracks has {tracks.shape[1]} points but point_embedding has {emb.shape[0]} rows")
    if select_id is not None:
        tracks = tracks[list(select_id)]
    cond = {"pred_tracks": tracks, "point_embedding": emb, "point_name2id": dict(name2id),
            "img_size": tuple(img_size) if img_size is not None else d.get("img_size"), "index_list": None}
    if select_point:
        cond["index_list"] = [cond["point_name2id"][n] for n in select_point]     # KeyError on an unknown name, like the reference
    return cond


def select_points(conditions: Mapping, select_point: Optional[Iterable[str]]) -> Dict:
    """Per-edit copy of the source conditions with `index_list` set (pipeline_videoswap.py:325-334)."""
    c = copy.deepcopy(dict(conditions))
    c["index_list"] = [c["point_name2id"][n] for n in select_point] if select_point else None
    return c


# ------------------------------------------------------------------------------------------- motion module / adapter
def remap_motion_module_keys(state_dict: Mapping[str, torch.Tensor]) -> "OrderedDict[str, torch.Tensor]":
    """AnimateDiff checkpoints keep the sinusoid table under `attention_blocks.N.pos_encoder.pe`; the reference's module tree
    (and this one) has it under `.processor.pos_encoder.pe` (test.py:63)."""
    return OrderedDict((k.replace(".pos_encoder", ".processor.pos_encoder"), v) for k, v in state_dict.items())


def load_motion_module(unet, ckpt: PathOrDict):
    """test.py:60-64: load the motion-module weights into a UNet built by `from_pretrained_2d`.  Returns the
    (missing, unexpected) pair of `load_state_dict(strict=False)`; every key of the checkpoint must be consumed."""
    sd = remap_motion_module_keys(_load(ckpt))
    r = unet.load_state_dict(sd, strict=False)
    unexpected = list(r.unexpected_keys if hasattr(r, "unexpected_keys") else r[1])
    if unexpected:
        raise KeyError(f"motion-module checkpoint has {len(unexpected)} keys this UNet does not have, e.g. {unexpected[:3]}")
    return r


def load_adapter(adapter, ckpt: PathOrDict, dtype: Optional[torch.dtype] = None):
    """test.py:67-70: `t2i_adapter.load_state_dict(torch.load(path))` (strict) then `.to(dtype)`."""
    adapter.load_state_dict(_load(ckpt))
    return adapter.to(dtype=dtype) if dtype is not None else adapter


# ------------------------------------------------------------------------------------------------------- ED-LoRA
_UNET_LORA_SITES = ("to_q.weight", "to_k.weight", "to_v.weight", "to_out.0.weight", "ff.net.0.proj.weight", "ff.net.2.weight",
                    "proj_out.weight", "proj_in.weight")
_TEXT_LORA_SITES = ("q_proj.weight", "k_proj.weight", "v_proj.weight", "out_proj.weight", "fc1.weight", "fc2.weight")


def _replace_sites(weight_name: str, sites) -> str:
    k = weight_name
    for site in sites:
        k = k.replace(site, site[:-len("weight")] + "lora_down.weight")
    return k


def lora_down_name(weight_name: str) -> str:
    """Name of the `lora_down` tensor that would modify UNet weight `weight_name` (convert_edlora_to_diffusers.py:45-53): the
    reference applies the eight `.replace` calls IN ORDER to the whole key, so this does too."""
    return _replace_sites(weight_name, _UNET_LORA_SITES)


def text_lora_down_name(weight_name: str) -> str:
    """The same for a text-encoder weight: the six `.replace` calls of convert_edlora_to_diffusers.py:38-44, in order."""
    return _replace_sites(weight_name, _TEXT_LORA_SITES)


def load_edlora(ckpt: PathOrDict) -> Dict:
    """ED-LoRA file -> {'new_concept_embedding': {...}, 'unet': {...}, 'text_encoder': {...}} (absent parts = empty dicts)."""
    d = _load(ckpt)
    d = d["params"] if "params" in d else d
    return {k: d.get(k, {}) for k in ("new_concept_embedding", "unet", "text_encoder")}


def new_concept_token_names(new_concept_embedding: Mapping[str, torch.Tensor], enable_edlora: bool = True) -> Dict[str, List[str]]:
    """Token names `load_new_concept` adds per concept (convert_edlora_to_diffusers.py:4-33): 16 per concept for ED-LoRA (one
    per cross-attention layer), 1 otherwise.  Token ids are the tokenizer's business and are not produced here."""
    n = 16 if enable_edlora else 1
    return {name: [f"<{name}_{i}>" for i in range(n)] for name in new_concept_embedding}


def bind_concept_prompt(prompts: Union[str, Sequence[str]], new_concept_cfg: Mapping) -> List[str]:
    """edlora_util.py:100-111: every prompt becomes 16 prompts, the i-th with each concept name replaced by its i-th token --
    the text encoder then yields the `[b, 16, 77, 768]` embeddings whose layer axis `EDLoRA_AttnProcessor` indexes.
    `new_concept_cfg` is the reference's `{concept: {'concept_token_names': [...], ...}}` (or `{concept: [names]}`, the
    output of `new_concept_token_names`).  Like the reference's `zip`, a concept with fewer than 16 names truncates the list."""
    if isinstance(prompts, str):
        prompts = [prompts]
    out: List[str] = []
    for prompt in prompts:
        layered = [prompt] * 16
        for concept, cfg in new_concept_cfg.items():
            names = cfg["concept_token_names"] if isinstance(cfg, Mapping) else cfg
            layered = [p.replace(concept, n) for p, n in zip(layered, names)]
        out.extend(layered)
    return out


@torch.no_grad()
def merge_edlora_into_unet(unet, lora_unet: Mapping[str, torch.Tensor], alpha: float,
                           strict: bool = False) -> "OrderedDict[str, torch.Tensor]":
    """Step 2 of `convert_edlora` (convert_edlora_to_diffusers.py:36-81, 92-96) IN PLACE on the UNet's own parameters:

        W <- round_to_W_dtype( float32(W) + alpha * (up @ down) )        (1x1-conv weights: squeeze, matmul, unsqueeze)

    -- the same single rounding the reference's `original + alpha * lora` (fp32 promotion) followed by `load_state_dict` into
    fp16 parameters performs.  Unlike the reference no copy of the 2.5 GB state dict is made: only the touched weights are
    saved, and the returned backup restores them bit-exactly (`restore_unet`), which is what `validation()` does with its
    deep-copied state dict after every edit (pipeline_videoswap.py:303, 418).  LoRA tensors that match no weight are ignored
    like the reference ignores them (it only prints the number of merged pairs); `strict=True` raises instead."""
    return _merge_lora(unet, lora_unet, alpha, strict, lora_down_name, "UNet")


def _merge_lora(model, lora: Mapping[str, torch.Tensor], alpha: float, strict: bool, down_name,
                what: str) -> "OrderedDict[str, torch.Tensor]":
    params = dict(model.named_parameters())
    backup: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    used = set()
    for name, w in params.items():
        dn = down_name(name)
        up = dn.replace("lora_down", "lora_up")
        if dn == name or up not in lora:
            continue
        if dn not in lora:
            raise KeyError(f"ED-LoRA has '{up}' but not '{dn}'")
        down_t = lora[dn].to(device=w.device, dtype=torch.float32)
        up_t = lora[up].to(device=w.device, dtype=torch.float32)
        if w.dim() == 4:
            delta = (up_t.squeeze() @ down_t.squeeze()).unsqueeze(-1).unsqueeze(-1)
        else:
            delta = up_t @ down_t
        if delta.shape != w.shape:
            raise ValueError(f"ED-LoRA delta for '{name}' is {tuple(delta.shape)}, weight is {tuple(w.shape)}")
        backup[name] = w.detach().clone()
        w.copy_((w.to(torch.float32) + float(alpha) * delta).to(w.dtype))
        used.update((dn, up))
    stray = [k for k in lora if k not in used and ("lora_down" in k or "lora_up" in k)]
    if stray and strict:
        raise KeyError(f"{len(stray)} ED-LoRA tensors match no {what} weight, e.g. {stray[:3]}")
    _mark_dirty(model)
    return backup


@torch.no_grad()
def restore_unet(unet, backup: Mapping[str, torch.Tensor]) -> None:
    """Undo `merge_edlora_into_unet` (pipeline_videoswap.py:418: `self.unet.load_state_dict(pretrained_unet_state_dict)`)."""
    params = dict(unet.named_parameters())
    for name, saved in backup.items():
        params[name].copy_(saved)
    _mark_dirty(unet)


def _mark_dirty(model):
    mark = getattr(model, "mark_weights_dirty", None)     # native models: re-pack into kernel layouts at the next call
    if mark is not None:
        mark()


@torch.no_grad()
def merge_edlora_into_text_encoder(text_encoder, lora_te: Mapping[str, torch.Tensor], alpha: float,
                                   strict: bool = False) -> "OrderedDict[str, torch.Tensor]":
    """Step 3 of `convert_edlora` (convert_edlora_to_diffusers.py:98-103) in place on the text encoder's weights
    (q / k / v / out_proj, fc1, fc2): the same single fp32 -> fp16 rounding and backup as merge_edlora_into_unet; the native
    CLIPTextModel re-packs at its next call.  Returns the backup for restore_text_encoder."""
    return _merge_lora(text_encoder, lora_te, alpha, strict, text_lora_down_name, "text-encoder")


@torch.no_grad()
def restore_text_encoder(text_encoder, backup: Mapping[str, torch.Tensor]) -> None:
    """Undo merge_edlora_into_text_encoder bit-exactly (pipeline_videoswap.py:419 loads the pre-edit state dict without the
    token embedding): only the merged weights are written, so concept rows of the token embedding stay."""
    restore_unet(text_encoder, backup)


@torch.no_grad()
def load_new_concept(tokenizer, text_encoder, new_concept_embedding: Mapping[str, torch.Tensor],
                     enable_edlora: bool = True) -> Dict[str, Dict[str, List]]:
    """convert_edlora_to_diffusers.py:4-33: per concept, add its tokens `<name_i>` (16 with ED-LoRA, else 1) to the
    tokenizer, grow the token embedding to len(tokenizer) and write the concept's rows.  Returns the reference's
    new_concept_cfg {concept: {'concept_token_ids': [...], 'concept_token_names': [...]}}."""
    cfg: Dict[str, Dict[str, List]] = {}
    for concept, emb in new_concept_embedding.items():
        names = new_concept_token_names({concept: emb}, enable_edlora)[concept]
        added = tokenizer.add_tokens(names)
        if added != 0 and added != len(names):
            raise ValueError(f"some token of {concept!r} is already in the tokenizer")
        ids = [tokenizer.convert_tokens_to_ids(n) for n in names]
        text_encoder.resize_token_embeddings(len(tokenizer))
        table = text_encoder.get_input_embeddings().weight.data
        table[ids] = emb.clone().to(table.device, dtype=table.dtype)
        cfg[concept] = {"concept_token_ids": ids, "concept_token_names": names}
    return cfg
