"""transformers `CLIPTextModel` (SD-1.5's text_encoder) on the native kernels, with transformers' config and state_dict
names.  The reference encodes every prompt with `pipe.text_encoder(ids)[0]` (pipeline_videoswap.py:273-423 through
diffusers' `_encode_prompt`, and utils/edlora_util.py:116-196 for ED-LoRA); `__call__` returns the same
`last_hidden_state`, after `final_layer_norm`.

Executor: a short sequence over `ops`, tokens as rows [n L, 768] fp16, every sequence of a call in one pass (86 launches
for 12 layers): clip_embed, then per pre-LN block  LN1 -> one QKV GEMM on a packed [2304, 768] weight -> causal attention
-> out_proj + bias + residual (in place) -> LN2 -> fc1 + bias + quick-GELU -> fc2 + bias + residual (in place); then the
final LayerNorm.  The tokenizer is the caller's (transformers' CLIPTokenizer from the checkpoint's tokenizer/ folder)."""
from __future__ import annotations

from collections import OrderedDict, namedtuple
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

from . import ops
from .spec import CLIPTextConfig, clip_text_param_shapes
from .weights import config_kwargs, missing_keys_text, read_pretrained_dir, seeded_state_dict

TOKEN_EMBEDDING = "text_model.embeddings.token_embedding.weight"
POSITION_EMBEDDING = "text_model.embeddings.position_embedding.weight"
POSITION_IDS = "text_model.embeddings.position_ids"    # a buffer older checkpoints carry; accepted and ignored
SEED = 9                                               # seeded test weights (init="seeded")

IncompatibleKeys = namedtuple("IncompatibleKeys", ["missing_keys", "unexpected_keys"])


@dataclass
class CLIPTextModelOutput:
    """last_hidden_state [n, L, 768] fp16; hidden_states (output_hidden_states=True): the 13 states before the final
    LayerNorm, the embeddings' output first, as transformers returns them.  output[0] is last_hidden_state; the pooled
    output is not computed (SD does not use it)."""
    last_hidden_state: torch.Tensor
    hidden_states: Optional[Tuple[torch.Tensor, ...]] = None

    def __getitem__(self, i):
        if i == 0 or i == "last_hidden_state":
            return self.last_hidden_state
        if i == "hidden_states":
            return self.hidden_states
        raise IndexError(f"CLIPTextModelOutput[{i!r}]: only [0] (last_hidden_state) exists; the pooled output is not computed")


class _Embedding:
    """What `get_input_embeddings()` returns: `.weight` is the device fp16 table the embedding kernel reads, so in-place
    row writes (load_new_concept) take effect at the next call."""

    def __init__(self, weight: torch.Tensor):
        self.weight = weight


def check_config(cfg: CLIPTextConfig) -> CLIPTextConfig:
    """The kernels implement SD-1.5's text tower only: quick_gelu, width 768, 12 heads of 64, 77 positions."""
    want = {"hidden_act": "quick_gelu", "hidden_size": 768, "num_attention_heads": 12, "max_position_embeddings": 77}
    for k, v in want.items():
        if getattr(cfg, k) != v:
            raise ValueError(f"CLIPTextModel (videoswap_b200) supports SD-1.5's text encoder only: {k} = {getattr(cfg, k)!r}, "
                             f"expected {v!r}")
    if cfg.num_hidden_layers < 1 or cfg.intermediate_size % 32:
        raise ValueError(f"unsupported num_hidden_layers {cfg.num_hidden_layers} / intermediate_size {cfg.intermediate_size}")
    return cfg


class CLIPTextModel:
    """transformers' CLIPTextModel (last_hidden_state) on CUDA.  init="seeded" draws test weights
    (weights.seeded_state_dict), "empty" waits for load_state_dict.  The fp16 weights on the device are the masters:
    state_dict() / named_parameters() return them, and the kernel layouts (the packed QKV weight, fp32 biases and norm
    parameters) are re-made from them at the first call after load_state_dict or mark_weights_dirty()."""

    dtype = torch.float16

    def __init__(self, init: str = "seeded", device="cuda", **config):
        self.config = check_config(CLIPTextConfig(**config))
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("CLIPTextModel (videoswap_b200) runs on CUDA only")
        self._params: "OrderedDict[str, torch.Tensor]" = OrderedDict()
        self._packed = None
        if init == "seeded":
            self.load_state_dict(seeded_state_dict(clip_text_param_shapes(self.config), seed=SEED))
        elif init != "empty":
            raise ValueError(f"init must be 'seeded' or 'empty', got {init!r}")

    # ------------------------------------------------------------------------------------------------ construction
    @classmethod
    def from_config(cls, config, **kw):
        """transformers-style: the keys of CLIPTextConfig are used, the rest of a config.json ignored; a config other than
        SD-1.5's raises (check_config)."""
        return cls(**kw, **config_kwargs(config, CLIPTextConfig))

    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = "text_encoder", device="cuda"):
        """A local diffusers / transformers directory: config.json + model.safetensors (or pytorch_model.bin)."""
        config, sd = read_pretrained_dir(path, subfolder, "model.safetensors", "pytorch_model.bin")
        m = cls.from_config(config, init="empty", device=device)
        m.load_state_dict(sd)
        return m

    # ------------------------------------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """transformers keys -> the fp16 masters.  strict=True needs every key; strict=False updates only the keys given
        (the reference restores the encoder without its token embedding that way, pipeline_videoswap.py:304-305, 419).
        An unknown key or a wrong shape raises in both modes; `position_ids` is ignored.  The token embedding may have
        any number of rows (49408 + 16 per loaded concept)."""
        shapes = clip_text_param_shapes(self.config)
        C = self.config.hidden_size
        staged = {}
        for k, v in sd.items():
            if k == POSITION_IDS:
                continue
            if k not in shapes:
                raise KeyError(f"unexpected key in the CLIP text encoder state_dict: {k}")
            want = shapes[k]
            if k == TOKEN_EMBEDDING and v.dim() == 2 and v.shape[1] == C and v.shape[0] >= 1:
                want = tuple(v.shape)
            if tuple(v.shape) != want:
                raise ValueError(f"{k}: shape {tuple(v.shape)}, expected {want}")
            staged[k] = v
        missing = [k for k in shapes if k not in staged]
        if strict and missing:
            raise KeyError(f"missing keys in the CLIP text encoder state_dict: {missing_keys_text(missing)}")
        for k, v in staged.items():
            cur = self._params.get(k)
            if cur is not None and cur.shape == v.shape:
                cur.copy_(v.detach())
            else:
                self._params[k] = v.detach().to(self.device, torch.float16).contiguous()
        if TOKEN_EMBEDDING in self._params:
            self.config.vocab_size = self._params[TOKEN_EMBEDDING].shape[0]
        self._packed = None
        return IncompatibleKeys(missing, [])

    def state_dict(self) -> "OrderedDict[str, torch.Tensor]":
        """The fp16 masters (device tensors, not copies) under the transformers keys."""
        return OrderedDict(self._params)

    def named_parameters(self):
        return iter(self._params.items())

    def mark_weights_dirty(self):
        """The masters were written in place (e.g. an ED-LoRA merge): re-pack the kernel layouts at the next call."""
        self._packed = None

    def resize_token_embeddings(self, n: int) -> _Embedding:
        """transformers' resize_token_embeddings: the first min(n, rows) rows are kept; new rows start at ZERO (transformers
        draws them at random; load_new_concept overwrites every one of them at once, convert_edlora_to_diffusers.py:21-23)."""
        old = self._params[TOKEN_EMBEDDING]
        new = torch.zeros((int(n), old.shape[1]), dtype=torch.float16, device=self.device)
        k = min(int(n), old.shape[0])
        new[:k] = old[:k]
        self._params[TOKEN_EMBEDDING] = new
        self.config.vocab_size = int(n)
        return _Embedding(new)

    def get_input_embeddings(self) -> _Embedding:
        return _Embedding(self._params[TOKEN_EMBEDDING])

    def _pack(self):
        missing = [k for k in clip_text_param_shapes(self.config) if k != TOKEN_EMBEDDING and k not in self._params]
        if missing or TOKEN_EMBEDDING not in self._params:
            raise RuntimeError(f"CLIPTextModel has no complete weights (missing {missing[:3]}): load_state_dict first")
        P = self._params

        def f32(k):
            return P[k].float().contiguous()

        def norm(k):
            return f32(k + ".weight"), f32(k + ".bias")
        layers = []
        for i in range(self.config.num_hidden_layers):
            p = f"text_model.encoder.layers.{i}"
            a = p + ".self_attn"
            layers.append({
                "ln1": norm(p + ".layer_norm1"),
                "qkv": (torch.cat([P[f"{a}.{n}_proj.weight"] for n in "qkv"]).contiguous(),
                        torch.cat([f32(f"{a}.{n}_proj.bias") for n in "qkv"]).contiguous()),
                "out": (P[a + ".out_proj.weight"], f32(a + ".out_proj.bias")),
                "ln2": norm(p + ".layer_norm2"),
                "fc1": (P[p + ".mlp.fc1.weight"], f32(p + ".mlp.fc1.bias")),
                "fc2": (P[p + ".mlp.fc2.weight"], f32(p + ".mlp.fc2.bias")),
            })
        self._packed = {"layers": layers, "final": norm("text_model.final_layer_norm")}

    # ------------------------------------------------------------------------------------------------ executor
    @torch.no_grad()
    def __call__(self, input_ids: torch.Tensor, output_hidden_states: bool = False) -> CLIPTextModelOutput:
        """input_ids [n, L] integers (CPU or CUDA), 1 <= L <= 77, every id a row of the token embedding (checked on the
        host before anything launches; an id outside raises ValueError)."""
        ids = torch.as_tensor(input_ids)
        if ids.dim() != 2 or ids.dtype.is_floating_point or ids.dtype == torch.bool:
            raise ValueError(f"input_ids must be an integer tensor [n, L], got {tuple(ids.shape)} {ids.dtype}")
        n, L = ids.shape
        if n < 1 or not 1 <= L <= self.config.max_position_embeddings:
            raise ValueError(f"input_ids [n, L] needs n >= 1 and 1 <= L <= {self.config.max_position_embeddings}, got {tuple(ids.shape)}")
        tok = self._params.get(TOKEN_EMBEDDING)
        if tok is None:
            raise RuntimeError("CLIPTextModel has no weights: load_state_dict first")
        ids_host = ids.cpu()
        lo, hi = int(ids_host.min()), int(ids_host.max())
        if lo < 0 or hi >= tok.shape[0]:
            raise ValueError(f"token id {lo if lo < 0 else hi} is outside the token embedding's {tok.shape[0]} rows")
        if self._packed is None:
            self._pack()
        w = self._packed
        heads = self.config.num_attention_heads
        x = ops.clip_embed(ids_host.to(torch.int32).to(self.device), tok, self._params[POSITION_EMBEDDING])
        hidden = [x.clone()] if output_hidden_states else None
        for lw in w["layers"]:
            h = ops.layernorm(x, *lw["ln1"])
            qkv = ops.gemm(h, *lw["qkv"])
            o = ops.causal_attention(qkv, n, L, heads)
            ops.gemm(o, lw["out"][0], bias=lw["out"][1], residual=x, out=x)          # x += out_proj(o), fp16 add
            h = ops.layernorm(x, *lw["ln2"])
            f = ops.gemm(h, lw["fc1"][0], bias=lw["fc1"][1], mode=ops.EPI_QUICK_GELU)
            ops.gemm(f, lw["fc2"][0], bias=lw["fc2"][1], residual=x, out=x)          # x += fc2(quick_gelu(fc1(h)))
            if hidden is not None:
                hidden.append(x.clone())
        y = ops.layernorm(x, *w["final"])
        C = self.config.hidden_size
        hs = tuple(t.view(n, L, C) for t in hidden) if hidden is not None else None
        return CLIPTextModelOutput(last_hidden_state=y.view(n, L, C), hidden_states=hs)
