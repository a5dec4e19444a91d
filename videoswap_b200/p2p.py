"""Attention controllers + latent blend on the native path (SURVEY.md 8f-2).

Mirrors the reference's prompt-to-prompt utilities -- utils/p2p_utils/attention_register.py (`register_attention_control`),
attention_store.py (`AttentionControl`, `AttentionStore`), attention_util.py (`AttentionControlEdit`, `AttentionRefine`,
`AttentionReplace`), spatial_blend.py (`SpatialBlender`) -- with the same call protocol
(`controller(attn, is_cross, place_in_unet)` between softmax and P V for every attention with fewer than 32^2 queries,
`controller.step_callback(latents)` after every scheduler step), but everything stays ON THE DEVICE:

  * the probabilities come from the explicit-probability kernels of libvideoswap_b200 through `vs_unet_set_attention_hook`
    (a zero-copy torch view of the library's buffer is handed to the controller);
  * the store keeps device tensors (the reference does `attn.cpu()` + `copy.deepcopy` per layer per step,
    attention_store.py:95-99);
  * the blend mask and the latent blend are CUDA kernels (`vs_blend_mask`, `vs_latent_blend`).

The edit controllers take their tokenizer-dependent inputs as tensors (`mapper`, `alphas`, `cross_replace_alpha`,
`alpha_layers`).  `make_controller` builds them from the prompts on the host (the word lookup of ptp_utils.py, the per-word
time alphas, the refinement and replacement mappers of seq_aligner.py, restated) and moves them to the device once;
`from_reference()` copies them out of a controller built by the reference's own `make_controller` instead.  The reference's
controller objects can also be registered unchanged (they receive device tensors and do their own `.cpu()`).  The small map
edits (gather / lerp / einsum on [F, 8, 256, 77]) use torch ops on the device tensors."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Mapping, Optional, Sequence, Tuple, Union

import torch

from . import _lib

MAX_QUERIES = 32 ** 2          # attention_register.py:70 / attention_store.py:96: only layers below this are controlled
_PLACES = ("down", "mid", "up")
HOOK_TYPE = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p)


class _DevicePtr:
    """Minimal __cuda_array_interface__ holder: a zero-copy torch view of a buffer owned by the library."""

    def __init__(self, ptr: int, shape: Tuple[int, ...], typestr: str = "<f2"):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 2}


def tensor_view(ptr: int, shape: Tuple[int, ...], device) -> torch.Tensor:
    return torch.as_tensor(_DevicePtr(ptr, shape), device=device)


# ------------------------------------------------------------------------------------------------ processors / registration
class AttnControlProcessor:
    """Marker processor (attention_register.py:100-173): the kernels do the arithmetic, this object carries the controller."""

    def __init__(self, place_in_unet: str, controller):
        self.place_in_unet, self.controller = place_in_unet, controller


class EDLoRA_AttnControlProcessor(AttnControlProcessor):
    def __init__(self, cross_attention_idx: int, place_in_unet: str, controller):
        super().__init__(place_in_unet, controller)
        self.cross_attention_idx = cross_attention_idx


class EmptyControl:
    def step_callback(self, x_t):
        return x_t

    def between_steps(self):
        return

    def __call__(self, attn, is_cross: bool, place_in_unet: str):
        return attn


def register_attention_control(model, controller):
    """attention_register.py:176-211.  `model` is a pipeline (has .unet) or the UNet.  controller None / EmptyControl removes
    the control processors (the UNet then runs the fused flash-attention kernels everywhere, graph-capturable again)."""
    unet = getattr(model, "unet", model)
    remove = controller is None or isinstance(controller, EmptyControl)

    def walk(mod, count_self, count_cross, place):
        for name, layer in mod.named_children():
            if layer.__class__.__name__ == "Attention" and ("attn1" in name or "attn2" in name):
                if remove:
                    from .unet import AttnProcessor
                    layer.set_processor(AttnProcessor())
                elif "attn2" in name:
                    layer.set_processor(EDLoRA_AttnControlProcessor(count_cross, place, controller))
                else:
                    layer.set_processor(AttnControlProcessor(place, controller))
                if "attn1" in name:
                    count_self += 1
                else:
                    count_cross += 1
            else:
                count_self, count_cross = walk(layer, count_self, count_cross, place)
        return count_self, count_cross

    cs, cc = walk(unet.down_blocks, 0, 0, "down")
    cs, cc = walk(unet.mid_block, cs, cc, "mid")
    cs, cc = walk(unet.up_blocks, cs, cc, "up")
    if not remove:
        controller.num_att_layers = cs + cc
    return cs + cc


# ------------------------------------------------------------------------------------------------ stores
class AttentionControl:
    """attention_store.py:21-67."""

    def __init__(self):
        self.LOW_RESOURCE = False     # False: the batch is [uncond | cond] (CFG) and only the conditional half is controlled
        self.cur_step = 0
        self.num_att_layers = -1
        self.cur_att_layer = 0

    def step_callback(self, x_t):
        self.cur_att_layer = 0
        self.cur_step += 1
        self.between_steps()
        return x_t

    def between_steps(self):
        return

    def forward(self, attn, is_cross: bool, place_in_unet: str):
        raise NotImplementedError

    def __call__(self, attn, is_cross: bool, place_in_unet: str):
        if self.LOW_RESOURCE:
            attn = self.forward(attn, is_cross, place_in_unet)
        else:
            h = attn.shape[0]
            attn[h // 2:] = self.forward(attn[h // 2:], is_cross, place_in_unet)
        self.cur_att_layer += 1
        return attn

    def reset(self):
        self.cur_step = 0
        self.cur_att_layer = 0


def _empty_store() -> Dict[str, List[torch.Tensor]]:
    return {"down_cross": [], "mid_cross": [], "up_cross": [], "down_self": [], "mid_self": [], "up_self": []}


class AttentionStore(AttentionControl):
    """attention_store.py:70-133 with device-resident tensors (no .cpu(), no deepcopy)."""

    def __init__(self, keep_all_steps: bool = True):
        super().__init__()
        self.keep_all_steps = keep_all_steps
        self.step_store = _empty_store()
        self.attention_store: Dict[str, List[torch.Tensor]] = {}
        self.latents_store: List[torch.Tensor] = []
        self.attention_store_all_step: List[Dict[str, List[torch.Tensor]]] = []

    def step_callback(self, x_t):
        x_t = super().step_callback(x_t)
        self.latents_store.append(x_t.detach().clone())
        return x_t

    def forward(self, attn, is_cross: bool, place_in_unet: str):
        if attn.shape[-2] < MAX_QUERIES:
            # the library re-uses its probability buffer for the next layer: keep a device copy (the reference copies to the host)
            self.step_store[f"{place_in_unet}_{'cross' if is_cross else 'self'}"].append(attn.detach().clone())
        return attn

    def between_steps(self):
        if len(self.attention_store) == 0:
            # running sum over the steps in fp32 (the reference adds in the maps' own dtype: fp16 at inference)
            self.attention_store = {k: [t.to(torch.float32, copy=True) for t in v] for k, v in self.step_store.items()}
        else:
            for key in self.attention_store:
                for i in range(len(self.attention_store[key])):
                    self.attention_store[key][i] += self.step_store[key][i]
        if self.keep_all_steps:
            self.attention_store_all_step.append(self.step_store)      # the per-step tensors are never written again
        self.step_store = _empty_store()

    def get_average_attention(self):
        return {key: [item / self.cur_step for item in self.attention_store[key]] for key in self.attention_store}

    def reset(self):
        super().reset()
        self.step_store = _empty_store()
        self.attention_store_all_step = []
        self.attention_store = {}
        self.latents_store = []


# ------------------------------------------------------------------------------------------------ blend
class SpatialBlender:
    """spatial_blend.py: mask from the cross-attention maps of the edited words, and the latent blend
    x_t = x_src + mask (x_t - x_src) for start_blend < call count < end_blend.  `alpha_layers`: [n_prompts, 77] (or the
    reference's [n_prompts,1,1,1,1,77]) word selector, 1 = blended word."""

    def __init__(self, alpha_layers: torch.Tensor, start_blend: float = 0.2, end_blend: float = 0.8, th: Sequence[float] = (0.3, 0.3),
                 NUM_DDIM_STEPS: int = 50, prompt_choose: str = "source"):
        assert prompt_choose in ("source", "both")
        self.alpha_layers = alpha_layers.reshape(alpha_layers.shape[0], -1).float()
        self.prompt_choose = prompt_choose
        self.start_blend = int(start_blend * NUM_DDIM_STEPS)
        self.end_blend = int(end_blend * NUM_DDIM_STEPS)
        self.counter = 0
        self.th = tuple(th)
        self.mask_list: List[torch.Tensor] = []

    def _mask(self, maps: List[torch.Tensor], target_h: int, target_w: int) -> torch.Tensor:
        """maps: list of [p, F, heads, r, words] (or [F, heads, r, words]) fp16 device tensors -> mask [p, F, h, w] fp32."""
        items = [m[None] if m.dim() == 4 else m for m in maps]
        p, frames, heads, r, words = items[0].shape
        dev = items[0].device
        ratio = target_h / target_w
        res_h = int((r * ratio) ** 0.5)
        res_w = int(r / res_h)
        assert res_h * res_w == r and all(tuple(i.shape) == tuple(items[0].shape) for i in items), "maps of one resolution expected"
        n_prompts = 1 if self.prompt_choose == "source" else p
        flat = [it[q].to(torch.float16).contiguous() for it in items for q in range(n_prompts)]       # layer-major, prompt-minor
        ptrs = torch.tensor([t.data_ptr() for t in flat], dtype=torch.int64, device=dev)
        alpha = self.alpha_layers[:n_prompts].to(dev).contiguous()
        mask = torch.empty((n_prompts, frames, target_h, target_w), dtype=torch.float32, device=dev)
        _lib.call("vs_blend_mask", torch.cuda.current_stream().cuda_stream, C.c_void_p(ptrs.data_ptr()), len(items), n_prompts, frames,
                  heads, res_h, res_w, words, C.c_void_p(alpha.data_ptr()), 1, target_h, target_w, float(self.th[0]),
                  int(self.prompt_choose == "both"), C.c_void_p(mask.data_ptr()))
        self._keep = (flat, ptrs, alpha)          # alive until the kernel ran
        return mask

    def __call__(self, attention_store, step_in_store: Optional[int] = None, target_h=None, target_w=None, x_t=None):
        if target_h is None and target_w is None and x_t is not None:
            target_h, target_w = x_t.shape[-2:]
        self.counter += 1
        maps = attention_store["down_cross"][2:4] + attention_store["up_cross"][:3]      # spatial_blend.py:88
        mask = self._mask(maps, target_h, target_w)
        self.mask_list.append(mask[0][:, None])
        if x_t is None:
            return mask
        if self.start_blend < self.counter < self.end_blend:
            # x_t: [2, C, F, h, w] = [source (inverted) | target]; only the target row changes (row 0 blends with itself)
            src, tgt = x_t[0].contiguous(), x_t[1].contiguous()
            ch, frames, hh, ww = tgt.shape
            _lib.call("vs_latent_blend", torch.cuda.current_stream().cuda_stream, C.c_void_p(src.data_ptr()), C.c_void_p(tgt.data_ptr()),
                      C.c_void_p(mask[-1].contiguous().data_ptr()), int(tgt.dtype == torch.float32), ch, frames, hh * ww)
            x_t = torch.stack([src, tgt])
        return x_t


# ------------------------------------------------------------------------------------------------ edit controllers
def time_words_alpha(num_steps: int, cross_replace_steps: Union[float, Tuple[float, float]], n_prompts: int = 2, words: int = 77):
    """ptp_utils.get_time_words_attention_alpha for the tokenizer-free case (one 'default_' window for every word)."""
    bounds = (0.0, cross_replace_steps) if isinstance(cross_replace_steps, float) else tuple(cross_replace_steps)
    a = torch.zeros(num_steps + 1, n_prompts - 1, words)
    start, end = int(bounds[0] * a.shape[0]), int(bounds[1] * a.shape[0])
    a[start:end] = 1
    return a.reshape(num_steps + 1, n_prompts - 1, 1, 1, words)


class AttentionControlEdit(AttentionStore):
    """attention_util.py:20-193 (single video, source maps from an inversion-time AttentionStore)."""

    def __init__(self, num_steps: int, cross_replace_alpha: torch.Tensor, self_replace_steps: Union[float, Tuple[float, float]],
                 latent_blend: Optional[SpatialBlender], additional_attention_store: AttentionStore,
                 attention_blend: Optional[SpatialBlender] = None, image_height: int = 512, image_width: int = 512):
        super().__init__(keep_all_steps=False)
        self.additional_attention_store = additional_attention_store
        self.batch_size = 1
        self.cross_replace_alpha = cross_replace_alpha
        if isinstance(self_replace_steps, float):
            self_replace_steps = 0, self_replace_steps
        self.num_self_replace = int(num_steps * self_replace_steps[0]), int(num_steps * self_replace_steps[1])
        self.attention_blend, self.latent_blend = attention_blend, latent_blend
        self.attention_position_counter_dict = {k: 0 for k in _empty_store()}
        self.image_height, self.image_width = image_height, image_width

    def step_callback(self, x_t):
        x_t = super().step_callback(x_t)
        if self.latent_blend is None:
            return x_t
        add = self.additional_attention_store
        step_in_store = len(add.latents_store) - self.cur_step
        inverted = add.latents_store[step_in_store].to(device=x_t.device, dtype=x_t.dtype)
        src_step = add.attention_store_all_step[step_in_store]
        blend_dict = {key: [torch.stack([a, self.attention_store[key][i]]) for i, a in enumerate(src_step[key])]
                      for key in ("down_cross", "mid_cross", "up_cross")}
        out = self.latent_blend(x_t=torch.cat([inverted, x_t], dim=0), attention_store=blend_dict)
        return out[1:]

    def replace_self_attention(self, attn_base, att_replace, reshaped_mask=None):
        if att_replace.shape[-2] >= MAX_QUERIES:
            return att_replace
        attn_base = attn_base.to(att_replace.dtype).unsqueeze(0).expand(att_replace.shape[0], *attn_base.shape)
        if reshaped_mask is not None:
            return reshaped_mask * att_replace + (1 - reshaped_mask) * attn_base
        return attn_base

    def replace_cross_attention(self, attn_base, att_replace):
        raise NotImplementedError

    def forward(self, attn, is_cross: bool, place_in_unet: str):
        super().forward(attn, is_cross, place_in_unet)
        if attn.shape[-2] >= MAX_QUERIES:
            return attn
        key = f"{place_in_unet}_{'cross' if is_cross else 'self'}"
        current_pos = self.attention_position_counter_dict[key]
        self.attention_position_counter_dict[key] += 1
        add = self.additional_attention_store
        step_in_store = len(add.attention_store_all_step) - self.cur_step - 1
        step_dict = add.attention_store_all_step[step_in_store]
        attn_base = step_dict[key][current_pos]
        if is_cross or (self.num_self_replace[0] <= self.cur_step < self.num_self_replace[1]):
            video_length = attn.shape[0] // self.batch_size
            attn = attn.reshape(self.batch_size, video_length, *attn.shape[1:])
            if is_cross:
                alpha_words = self.cross_replace_alpha[self.cur_step].to(device=attn.device, dtype=attn.dtype)
                attn = self.replace_cross_attention(attn_base, attn) * alpha_words + (1 - alpha_words) * attn
            else:
                reshaped_mask = None
                if self.attention_blend is not None:
                    rate = int(((self.image_height * self.image_width) / attn.shape[-2]) ** 0.5)
                    h, w = self.image_height // rate, self.image_width // rate
                    mask = self.attention_blend(target_h=h, target_w=w, attention_store=step_dict, step_in_store=step_in_store)
                    reshaped_mask = mask.permute(1, 0, 2, 3).reshape(mask.shape[1], mask.shape[0], h * w)[..., None].to(attn.dtype)
                attn = self.replace_self_attention(attn_base, attn, reshaped_mask)
            attn = attn.reshape(self.batch_size * video_length, *attn.shape[2:])
        return attn

    def between_steps(self):
        super().between_steps()
        self.step_store = _empty_store()
        self.attention_position_counter_dict = {k: 0 for k in _empty_store()}


class AttentionReplace(AttentionControlEdit):
    def __init__(self, mapper: torch.Tensor, *a, **k):
        super().__init__(*a, **k)
        self.mapper = mapper                     # [n_prompts - 1, 77, 77]

    def replace_cross_attention(self, attn_base, att_replace):
        m = self.mapper.to(device=att_replace.device, dtype=att_replace.dtype)
        return torch.einsum("thpw,bwn->bthpn", attn_base.to(att_replace.dtype), m)


class AttentionRefine(AttentionControlEdit):
    def __init__(self, mapper: torch.Tensor, alphas: torch.Tensor, *a, **k):
        super().__init__(*a, **k)
        self.mapper = mapper                     # [n_prompts - 1, 77] long (-1 = new word)
        self.alphas = alphas.reshape(alphas.shape[0], 1, 1, alphas.shape[-1])

    def replace_cross_attention(self, attn_base, att_replace):
        mp = self.mapper.to(att_replace.device)
        base = attn_base.to(att_replace.dtype)[:, :, :, mp].permute(3, 0, 1, 2, 4)
        al = self.alphas.to(device=att_replace.device, dtype=att_replace.dtype)
        return base * al + att_replace * (1 - al)


def from_reference(ref_controller, additional_attention_store: AttentionStore, num_steps: int):
    """Builds the device-native twin of a controller made by the reference's `make_controller` (tokenizer-dependent tensors are
    copied, not re-derived)."""
    def blender(b):
        if b is None:
            return None
        nb = SpatialBlender(b.alpha_layers, th=b.th, NUM_DDIM_STEPS=b.NUM_DDIM_STEPS or num_steps, prompt_choose=b.prompt_choose)
        nb.start_blend, nb.end_blend = b.start_blend, b.end_blend
        return nb
    common = dict(num_steps=num_steps, cross_replace_alpha=ref_controller.cross_replace_alpha, self_replace_steps=0.0,
                  latent_blend=blender(ref_controller.latent_blend), additional_attention_store=additional_attention_store,
                  attention_blend=blender(ref_controller.attention_blend), image_height=ref_controller.image_height,
                  image_width=ref_controller.image_width)
    if hasattr(ref_controller, "alphas"):
        c = AttentionRefine(ref_controller.mapper, ref_controller.alphas, **common)
    else:
        c = AttentionReplace(ref_controller.mapper, **common)
    c.num_self_replace = tuple(ref_controller.num_self_replace)
    return c


# ------------------------------------------------------------------------------------------------ controllers from prompts
MAX_NUM_WORDS = 77


def get_word_inds(text: str, word_place, tokenizer) -> List[int]:
    """Token positions (1 = the first token after BOS) of a whitespace word of `text` (seq_aligner / ptp_utils
    `get_word_inds`).  `word_place`: a word (every occurrence counts) or a word index.  Tokens are attributed to words by the
    length of their decoded text, so a word the tokenizer splits yields several positions."""
    split_text = text.split(" ")
    if isinstance(word_place, str):
        places = [i for i, w in enumerate(split_text) if w == word_place]
    elif isinstance(word_place, int):
        places = [word_place]
    else:
        places = list(word_place)
    out: List[int] = []
    if places:
        pieces = [tokenizer.decode([t]).strip("#") for t in tokenizer.encode(text)][1:-1]
        cur_len, ptr = 0, 0
        for i, piece in enumerate(pieces):
            cur_len += len(piece)
            if ptr in places:
                out.append(i + 1)
            if cur_len >= len(split_text[ptr]):
                ptr, cur_len = ptr + 1, 0
    return out


def _concept_word_inds(text: str, word: str, tokenizer, new_concept_cfg) -> List[int]:
    """ptp_utils.get_word_inds: with ED-LoRA concepts the text and the word are first bound to the layer-0 concept tokens."""
    if new_concept_cfg is not None:
        from .formats import bind_concept_prompt
        text, word = bind_concept_prompt(text, new_concept_cfg)[0], bind_concept_prompt(word, new_concept_cfg)[0]
    return get_word_inds(text, word, tokenizer)


def _window(bounds) -> Tuple[float, float]:
    return (0.0, float(bounds)) if isinstance(bounds, (int, float)) else (bounds[0], bounds[1])


def get_time_words_attention_alpha(prompts: Sequence[str], num_steps: int, cross_replace_steps, tokenizer,
                                   max_num_words: int = MAX_NUM_WORDS, new_concept_cfg=None) -> torch.Tensor:
    """ptp_utils.get_time_words_attention_alpha -> [num_steps + 1, n_prompts - 1, 1, 1, max_num_words].  Row s, word w is 1
    while the cross-attention of w is replaced at step s.  `cross_replace_steps`: a fraction f (window [0, f)), a pair, or a
    dict {word: fraction or pair} whose 'default_' entry (else (0, 1)) covers every word and whose other entries overwrite
    the window of that word's tokens in each target prompt."""
    steps = dict(cross_replace_steps) if isinstance(cross_replace_steps, Mapping) else {"default_": cross_replace_steps}
    steps.setdefault("default_", (0.0, 1.0))
    alpha = torch.zeros(num_steps + 1, len(prompts) - 1, max_num_words)

    def update(bounds, prompt_ind, word_inds):
        lo, hi = _window(bounds)
        start, end = int(lo * alpha.shape[0]), int(hi * alpha.shape[0])
        alpha[:start, prompt_ind, word_inds] = 0
        alpha[start:end, prompt_ind, word_inds] = 1
        alpha[end:, prompt_ind, word_inds] = 0

    for i in range(len(prompts) - 1):
        update(steps["default_"], i, torch.arange(max_num_words))
    for key, item in steps.items():
        if key == "default_":
            continue
        for i in range(1, len(prompts)):
            inds = _concept_word_inds(prompts[i], key, tokenizer, new_concept_cfg)
            if inds:
                update(item, i - 1, torch.tensor(inds))
    return alpha.reshape(num_steps + 1, len(prompts) - 1, 1, 1, max_num_words)


def _global_align(x: Sequence[int], y: Sequence[int]) -> List[Tuple[int, int]]:
    """Needleman-Wunsch alignment of two token sequences (match +1, mismatch -1, gap 0; ties prefer a gap in x, then a gap
    in y, then the diagonal), traced back from the end.  Returns, for every token j of y in order, (j, i): the token of x it
    is aligned with, or -1 for a token y inserts."""
    nx, ny = len(x), len(y)
    score = [[0] * (ny + 1) for _ in range(nx + 1)]
    trace = [[0] * (ny + 1) for _ in range(nx + 1)]
    for j in range(1, ny + 1):
        trace[0][j] = 1
    for i in range(1, nx + 1):
        trace[i][0] = 2
    trace[0][0] = 4
    for i in range(1, nx + 1):
        for j in range(1, ny + 1):
            left, up = score[i][j - 1], score[i - 1][j]
            diag = score[i - 1][j - 1] + (1 if x[i - 1] == y[j - 1] else -1)
            best = max(left, up, diag)
            score[i][j] = best
            trace[i][j] = 1 if best == left else (2 if best == up else 3)
    pairs: List[Tuple[int, int]] = []
    i, j = nx, ny
    while i > 0 or j > 0:
        t = trace[i][j]
        if t == 3:
            i, j = i - 1, j - 1
            pairs.append((j, i))
        elif t == 1:
            j -= 1
            pairs.append((j, -1))
        elif t == 2:
            i -= 1
        else:
            break
    pairs.reverse()
    return pairs


def get_refinement_mapper(prompts: Sequence[str], tokenizer, max_len: int = MAX_NUM_WORDS) -> Tuple[torch.Tensor, torch.Tensor]:
    """seq_aligner.get_refinement_mapper -> (mapper [n - 1, max_len] int64, alphas [n - 1, max_len] float32).  Token j of
    each target prompt reads the source token mapper[j] (-1 and alpha 0 for an inserted token); positions past the target's
    tokens read the positions after them."""
    x = tokenizer.encode(prompts[0])
    mappers, alphas = [], []
    for p in prompts[1:]:
        y = tokenizer.encode(p)
        base = torch.tensor(_global_align(x, y), dtype=torch.int64).reshape(-1, 2)
        n = base.shape[0]
        a = torch.ones(max_len)
        a[:n] = base[:, 1].ne(-1).float()
        m = torch.zeros(max_len, dtype=torch.int64)
        m[:n] = base[:, 1]
        m[n:] = len(y) + torch.arange(max_len - len(y))
        mappers.append(m)
        alphas.append(a)
    return torch.stack(mappers), torch.stack(alphas)


def get_replacement_mapper(prompts: Sequence[str], tokenizer, max_len: int = MAX_NUM_WORDS) -> torch.Tensor:
    """seq_aligner.get_replacement_mapper -> [n - 1, max_len, max_len] float32.  The prompts must have the same number of
    words (ValueError otherwise); each word that differs maps its source tokens onto its target tokens (1 where the counts
    agree, else 1 / number of target tokens), every other position maps to itself."""
    x = prompts[0]
    words_x = x.split(" ")
    mappers = []
    for y in prompts[1:]:
        words_y = y.split(" ")
        if len(words_x) != len(words_y):
            raise ValueError(f"attention replacement edit can only be applied on prompts with the same length but prompt A "
                             f"has {len(words_x)} words and prompt B has {len(words_y)} words.")
        changed = [i for i in range(len(words_y)) if words_y[i] != words_x[i]]
        src = [get_word_inds(x, i, tokenizer) for i in changed]
        tgt = [get_word_inds(y, i, tokenizer) for i in changed]
        m = torch.zeros(max_len, max_len, dtype=torch.float64)
        i = j = cur = 0
        while i < max_len and j < max_len:
            if cur < len(src) and src[cur][0] == i:
                s, t = src[cur], tgt[cur]
                if len(s) == len(t):
                    m[s, t] = 1
                else:
                    for tt in t:
                        m[s, tt] = 1 / len(t)
                cur += 1
                i += len(s)
                j += len(t)
            elif cur < len(src):
                m[i, j] = 1
                i, j = i + 1, j + 1
            else:
                m[j, j] = 1          # the reference writes the diagonal at the target position here
                i, j = i + 1, j + 1
        mappers.append(m.float())
    return torch.stack(mappers)


def word_selector(prompts: Sequence[str], words, tokenizer, new_concept_cfg=None) -> torch.Tensor:
    """SpatialBlender's `alpha_layers` ([n_prompts, 77], 1 = a token of one of the prompt's blend words)."""
    alpha = torch.zeros(len(prompts), MAX_NUM_WORDS)
    for i, (prompt, words_) in enumerate(zip(prompts, words)):
        for word in ([words_] if isinstance(words_, str) else words_):
            ind = _concept_word_inds(prompt, word, tokenizer, new_concept_cfg)
            if ind:
                alpha[i, ind] = 1
    return alpha


def make_controller(tokenizer, prompts: List[str], is_replace_controller: bool, cross_replace_steps,
                    self_replace_steps=0.0, blend_words=None, additional_attention_store: Optional[AttentionStore] = None,
                    blend_th=(0.3, 0.3), NUM_DDIM_STEPS: Optional[int] = None, blend_latents: bool = False,
                    blend_self_attention: bool = False, image_height: int = 512, image_width: int = 512, *,
                    new_concept_cfg=None, device=None) -> AttentionControlEdit:
    """attention_util.make_controller with the reference's signature: an AttentionReplace (equal word counts) or an
    AttentionRefine for [source, target] prompts, with a latent SpatialBlender (prompt_choose 'both', blend window 0.2-0.8
    of the steps) when `blend_latents` and a self-attention one ('source', 0-2) when `blend_self_attention`, both selecting
    the tokens of `blend_words` ([source words, target words]; None or 'None': no blending).

    All text work runs on the host; the tensors go to `device` once (default: CUDA when available, as the reference).
    `new_concept_cfg` (default: the tokenizer's `new_concept_cfg` attribute, where the reference keeps it): ED-LoRA
    concepts whose layer-0 tokens the blend words and the per-word cross_replace_steps are looked up as.  The mappers are
    computed on the prompts as written, like the reference's.  The native controllers read the source maps and latents of
    an inversion, so `additional_attention_store` and `NUM_DDIM_STEPS` are required."""
    if NUM_DDIM_STEPS is None:
        raise ValueError("make_controller needs NUM_DDIM_STEPS (the number of denoising steps)")
    if additional_attention_store is None:
        raise ValueError("make_controller needs additional_attention_store: the AttentionStore of the source's inversion")
    if len(prompts) != 2:
        raise ValueError(f"one video is edited with [source_prompt, target_prompt]; got {len(prompts)} prompts")
    if new_concept_cfg is None:
        new_concept_cfg = getattr(tokenizer, "new_concept_cfg", None)
    dev = torch.device(device if device is not None else ("cuda" if torch.cuda.is_available() else "cpu"))
    latent_blend = attention_blend = None
    if blend_words is not None and not (isinstance(blend_words, str) and blend_words == "None"):
        sel = word_selector(prompts, blend_words, tokenizer, new_concept_cfg).to(dev)
        if blend_latents:
            latent_blend = SpatialBlender(sel, start_blend=0.2, end_blend=0.8, th=blend_th, NUM_DDIM_STEPS=NUM_DDIM_STEPS,
                                          prompt_choose="both")
        if blend_self_attention:
            attention_blend = SpatialBlender(sel, start_blend=0.0, end_blend=2, th=blend_th, NUM_DDIM_STEPS=NUM_DDIM_STEPS,
                                             prompt_choose="source")
    alpha = get_time_words_attention_alpha(prompts, NUM_DDIM_STEPS, cross_replace_steps, tokenizer,
                                           new_concept_cfg=new_concept_cfg)
    common = dict(num_steps=NUM_DDIM_STEPS, cross_replace_alpha=alpha.to(dev), self_replace_steps=self_replace_steps,
                  latent_blend=latent_blend, additional_attention_store=additional_attention_store,
                  attention_blend=attention_blend, image_height=image_height, image_width=image_width)
    if is_replace_controller:
        return AttentionReplace(get_replacement_mapper(prompts, tokenizer).to(dev), **common)
    mapper, alphas = get_refinement_mapper(prompts, tokenizer)
    return AttentionRefine(mapper.to(dev), alphas.to(dev), **common)
