"""Host-side mirror of the reference's `AnimateDiffUNet3DModel`
(videoswap/models/animatediff_models/unet.py:32-523 of the reference) backed by libvideoswap_b200.so.

What is mirrored (SURVEY.md 8b.1): constructor arguments / `.config`, the module tree and state_dict key names
(`down_blocks.N.attentions.M.transformer_blocks.0.attn2...`), `Attention` objects with `set_processor` / `heads` /
`to_q`..., `load_state_dict` (weights are re-packed into kernel layouts on the next forward), the `forward` signature,
in-place `pop(0)` consumption of `down_block_additional_residuals`, `UNet3DConditionOutput`.

The torch modules below are parameter HOLDERS only: all arithmetic happens in the sm_90a kernels.  There is no
PyTorch/CPU fallback; a missing shared library or a CPU tensor raises.
"""
from __future__ import annotations

import ctypes as C
import json
import os
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Tuple, Union

import torch
from torch import nn

from . import _lib
from .spec import UNetConfig, unet_param_shapes
from .weights import seeded_state_dict, temporal_pe_table


@dataclass
class UNet3DConditionOutput:
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


class _Config(dict):
    """dict with attribute access, like diffusers' FrozenDict (`unet.config.in_channels`)."""
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


class _Holder(nn.Module):
    """weight (+bias) parameter holder with the given shapes (uninitialised; filled by load_state_dict)."""
    def __init__(self, wshape, bias=True):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(wshape), requires_grad=False)
        if bias:
            self.bias = nn.Parameter(torch.empty((wshape[0],)), requires_grad=False)

    def forward(self, *a, **k):
        raise RuntimeError("parameter holder: computation runs in libvideoswap_b200.so via AnimateDiffUNet3DModel.forward")


class AttnProcessor:
    """Default processor marker (the kernels implement diffusers' AttnProcessor2_0 semantics)."""


class _PosEncoder(nn.Module):
    def __init__(self, dim, max_len):
        super().__init__()
        self.register_buffer("pe", temporal_pe_table(max_len, dim))


class VanillaAttentionProcessor(nn.Module):
    """Holder for the motion module's processor sub-module: owns the `pos_encoder.pe` buffer so that the key
    `...attention_blocks.N.processor.pos_encoder.pe` exists (reference test.py:63 remaps checkpoints onto it)."""
    def __init__(self, dim, max_len):
        super().__init__()
        self.pos_encoder = _PosEncoder(dim, max_len)
        self.is_cross_attention = False


class Attention(nn.Module):
    """Mirror of diffusers' `Attention` object surface walked by the reference
    (utils/edlora_util.py:85-99, utils/p2p_utils/attention_register.py:176-211).  Class name must be 'Attention'."""
    def __init__(self, query_dim, cross_attention_dim=None, heads=8, dim_head=64, processor=None):
        super().__init__()
        inner = heads * dim_head
        ctx = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.sliceable_head_dim = heads
        self.group_norm = None
        self.spatial_norm = None
        self.norm_cross = None
        self.added_kv_proj_dim = None
        self.residual_connection = False
        self.rescale_output_factor = 1.0
        self.upcast_attention = False
        self.upcast_softmax = False
        self.to_q = _Holder((inner, query_dim), bias=False)
        self.to_k = _Holder((inner, ctx), bias=False)
        self.to_v = _Holder((inner, ctx), bias=False)
        self.to_out = nn.ModuleList([_Holder((query_dim, inner)), nn.Dropout(0.0)])
        self.set_processor(processor if processor is not None else AttnProcessor())

    def set_processor(self, processor):
        if hasattr(self, "processor") and isinstance(self.processor, nn.Module) and not isinstance(processor, nn.Module):
            self._modules.pop("processor")
        self.processor = processor

    def head_to_batch_dim(self, t):
        b, s, c = t.shape
        return t.reshape(b, s, self.heads, c // self.heads).permute(0, 2, 1, 3).reshape(b * self.heads, s, c // self.heads)

    def batch_to_head_dim(self, t):
        bh, s, d = t.shape
        return t.reshape(bh // self.heads, self.heads, s, d).permute(0, 2, 1, 3).reshape(bh // self.heads, s, d * self.heads)

    def prepare_attention_mask(self, attention_mask, target_length, batch_size=None, out_dim=3):
        return attention_mask

    def forward(self, *a, **k):
        raise RuntimeError("Attention modules are executed inside the fused UNet forward, not individually")


class _GEGLU(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.proj = _Holder((8 * dim, dim))


class FeedForward(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.net = nn.ModuleList([_GEGLU(dim), nn.Dropout(0.0), _Holder((dim, 4 * dim))])


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, heads, ctx):
        super().__init__()
        self.attn1 = Attention(dim, None, heads, dim // heads)
        self.norm1 = _Holder((dim,))
        self.attn2 = Attention(dim, ctx, heads, dim // heads)
        self.norm2 = _Holder((dim,))
        self.ff = FeedForward(dim)
        self.norm3 = _Holder((dim,))


class Transformer3DModel(nn.Module):
    def __init__(self, dim, heads, ctx):
        super().__init__()
        self.norm = _Holder((dim,))
        self.proj_in = _Holder((dim, dim, 1, 1))
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(dim, heads, ctx)])
        self.proj_out = _Holder((dim, dim, 1, 1))


class TemporalTransformerBlock(nn.Module):
    def __init__(self, dim, heads, pe_len):
        super().__init__()
        self.attention_blocks = nn.ModuleList(
            [Attention(dim, None, heads, dim // heads, processor=VanillaAttentionProcessor(dim, pe_len)) for _ in range(2)])
        self.norms = nn.ModuleList([_Holder((dim,)) for _ in range(2)])
        self.ff = FeedForward(dim)
        self.ff_norm = _Holder((dim,))


class TemporalTransformer3DModel(nn.Module):
    def __init__(self, dim, heads, pe_len):
        super().__init__()
        self.norm = _Holder((dim,))
        self.proj_in = _Holder((dim, dim))
        self.transformer_blocks = nn.ModuleList([TemporalTransformerBlock(dim, heads, pe_len)])
        self.proj_out = _Holder((dim, dim))


class VanillaTemporalModule(nn.Module):
    def __init__(self, dim, heads, pe_len):
        super().__init__()
        self.temporal_transformer = TemporalTransformer3DModel(dim, heads, pe_len)


class ResnetBlock3D(nn.Module):
    def __init__(self, cin, cout, temb):
        super().__init__()
        self.norm1 = _Holder((cin,))
        self.conv1 = _Holder((cout, cin, 3, 3))
        self.time_emb_proj = _Holder((cout, temb))
        self.norm2 = _Holder((cout,))
        self.conv2 = _Holder((cout, cout, 3, 3))
        if cin != cout:
            self.conv_shortcut = _Holder((cout, cin, 1, 1))


class _Sampler(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = _Holder((c, c, 3, 3))


class _Block(nn.Module):
    has_cross_attention = False

    def __init__(self, resnets, attentions=None, motion=None, down=None, up=None):
        super().__init__()
        if attentions is not None:
            self.attentions = nn.ModuleList(attentions)
            self.has_cross_attention = True
        self.resnets = nn.ModuleList(resnets)
        self.motion_modules = nn.ModuleList(motion if motion is not None else [])
        if down is not None:
            self.downsamplers = nn.ModuleList([down])
        if up is not None:
            self.upsamplers = nn.ModuleList([up])
        self.gradient_checkpointing = False


class CrossAttnDownBlock3D(_Block):
    pass


class DownBlock3D(_Block):
    pass


class UNetMidBlock3DCrossAttn(_Block):
    pass


class UpBlock3D(_Block):
    pass


class CrossAttnUpBlock3D(_Block):
    pass


class _TimeEmb(nn.Module):
    def __init__(self, cin, dim):
        super().__init__()
        self.linear_1 = _Holder((dim, cin))
        self.linear_2 = _Holder((dim, dim))


class AnimateDiffUNet3DModel(nn.Module):
    """Drop-in for the reference class of the same name (registered under that name in videoswap_b200.MODEL_REGISTRY).
    BASELINE.json calls it `UNet3DConditionModel`; that alias is exported too."""
    _supports_gradient_checkpointing = True

    def __init__(self, sample_size: Optional[int] = 64, in_channels: int = 4, out_channels: int = 4,
                 block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280), layers_per_block: int = 2,
                 attention_head_dim: int = 8, cross_attention_dim: int = 768, norm_num_groups: int = 32,
                 norm_eps: float = 1e-5, use_motion_module: bool = True,
                 motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block: bool = False,
                 motion_module_decoder_only: bool = False, motion_module_type: Optional[str] = "Vanilla",
                 motion_module_kwargs: Optional[Dict[str, Any]] = None,
                 unet_use_cross_frame_attention: Optional[bool] = False,
                 unet_use_temporal_attention: Optional[bool] = False, init: str = "seeded", **ignored):
        super().__init__()
        if unet_use_cross_frame_attention or unet_use_temporal_attention:
            raise NotImplementedError("unet_use_cross_frame_attention / unet_use_temporal_attention are false in every "
                                      "shipped config (options/model_cfg/inference.yml:2-3) and are not implemented")
        if use_motion_module and motion_module_type not in (None, "Vanilla"):
            raise ValueError(f"unknown motion_module_type {motion_module_type}")
        mk = dict(motion_module_kwargs or {})
        self.cfg = UNetConfig(
            sample_size=sample_size or 64, in_channels=in_channels, out_channels=out_channels,
            block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
            attention_head_dim=attention_head_dim, cross_attention_dim=cross_attention_dim,
            norm_num_groups=norm_num_groups, norm_eps=norm_eps, use_motion_module=use_motion_module,
            motion_module_resolutions=tuple(motion_module_resolutions), motion_module_mid_block=motion_module_mid_block,
            motion_module_decoder_only=motion_module_decoder_only,
            motion_num_attention_heads=mk.get("num_attention_heads", 8),
            temporal_position_encoding_max_len=mk.get("temporal_position_encoding_max_len", 24))
        self.config = _Config(self.cfg.to_dict(), motion_module_kwargs=mk, motion_module_type=motion_module_type,
                              center_input_sample=False, _class_name="AnimateDiffUNet3DModel")
        self.sample_size = sample_size
        cfg = self.cfg
        boc, temb, ctx, heads = list(cfg.block_out_channels), cfg.time_embed_dim, cfg.cross_attention_dim, cfg.attention_head_dim
        mh, pe = cfg.motion_num_attention_heads, cfg.temporal_position_encoding_max_len
        n, lpb = len(boc), cfg.layers_per_block
        self.conv_in = _Holder((boc[0], in_channels, 3, 3))
        self.time_embedding = _TimeEmb(boc[0], temb)
        downs, cout = [], boc[0]
        for i in range(n):
            cin, cout = cout, boc[i]
            res = [ResnetBlock3D(cin if j == 0 else cout, cout, temb) for j in range(lpb)]
            mot = [VanillaTemporalModule(cout, mh, pe) for _ in range(lpb)] if cfg.down_has_motion(i) else None
            if i < n - 1:
                downs.append(CrossAttnDownBlock3D(res, [Transformer3DModel(cout, heads, ctx) for _ in range(lpb)], mot,
                                                  down=_Sampler(cout)))
            else:
                downs.append(DownBlock3D(res, None, mot))
        self.down_blocks = nn.ModuleList(downs)
        c = boc[-1]
        self.mid_block = UNetMidBlock3DCrossAttn(
            [ResnetBlock3D(c, c, temb), ResnetBlock3D(c, c, temb)], [Transformer3DModel(c, heads, ctx)],
            [VanillaTemporalModule(c, mh, pe)] if (use_motion_module and motion_module_mid_block) else None)
        ups, rev = [], boc[::-1]
        for i in range(n):
            oc = rev[i]
            res = []
            for j in range(lpb + 1):
                run, skip = cfg.up_resnet_in_channels(i, j)
                res.append(ResnetBlock3D(run + skip, oc, temb))
            mot = [VanillaTemporalModule(oc, mh, pe) for _ in range(lpb + 1)] if cfg.up_has_motion(i) else None
            upsampler = _Sampler(oc) if i < n - 1 else None
            if i == 0:
                ups.append(UpBlock3D(res, None, mot, up=upsampler))
            else:
                ups.append(CrossAttnUpBlock3D(res, [Transformer3DModel(oc, heads, ctx) for _ in range(lpb + 1)], mot,
                                              up=upsampler))
        self.up_blocks = nn.ModuleList(ups)
        self.num_upsamplers = n - 1
        self.conv_norm_out = _Holder((boc[0],))
        self.conv_out = _Holder((out_channels, boc[0], 3, 3))

        self._handle = None
        self._dirty = True
        self._t_buf = None
        expected = unet_param_shapes(cfg)
        mine = {k: tuple(v.shape) for k, v in super().state_dict().items()}
        assert mine == dict(expected), "internal: module tree does not match the architecture spec"
        if init in ("seeded", "reference"):
            sd0 = seeded_state_dict(expected, seed=0)
            if init == "reference":
                # the reference zero-initialises every temporal_transformer.proj_out (motion_module.py:76-77), so a motion
                # module is an exact identity until a motion checkpoint is loaded; keys a checkpoint does not cover must
                # keep THAT behaviour (from_pretrained_2d loads with strict=False; test.py makes the motion ckpt optional)
                for k in sd0:
                    if ".temporal_transformer.proj_out." in k:
                        sd0[k] = torch.zeros_like(sd0[k])
            self.load_state_dict(sd0)
        elif init != "empty":
            raise ValueError("init must be 'seeded' (tests: non-zero motion proj_out), 'reference' or 'empty'")
        self.eval()

    # ------------------------------------------------------------------------------------------ reference surface
    @classmethod
    def from_config(cls, config, **kwargs):
        import inspect
        sig = inspect.signature(cls.__init__).parameters
        init = {k: v for k, v in dict(config).items() if k in sig}
        init.update({k: v for k, v in kwargs.items() if k in sig})
        init.setdefault("init", "reference")      # zero motion proj_out like the reference's constructor
        return cls(**init)

    @classmethod
    def from_pretrained_2d(cls, pretrained_model_path, subfolder=None, unet_additional_kwargs=None):
        """Same contract as the reference (unet.py:483-523): reads `config.json` + `diffusion_pytorch_model.bin` of a 2-D
        SD UNet and loads it with strict=False (motion-module weights stay at their initial values)."""
        if subfolder is not None:
            pretrained_model_path = os.path.join(pretrained_model_path, subfolder)
        config_file = os.path.join(pretrained_model_path, "config.json")
        if not os.path.isfile(config_file):
            raise RuntimeError(f"{config_file} does not exist")
        with open(config_file) as f:
            config = json.load(f)
        model = cls.from_config(config, **(unet_additional_kwargs or {}))
        model_file = os.path.join(pretrained_model_path, "diffusion_pytorch_model.bin")
        if not os.path.isfile(model_file):
            raise RuntimeError(f"{model_file} does not exist")
        m, u = model.load_state_dict(torch.load(model_file, map_location="cpu"), strict=False)
        print(f"### missing keys: {len(m)}; \n### unexpected keys: {len(u)};")
        return model

    @property
    def dtype(self):
        return self.conv_in.weight.dtype

    @property
    def device(self):
        return self.conv_in.weight.device

    def enable_gradient_checkpointing(self):
        for b in list(self.down_blocks) + list(self.up_blocks):
            b.gradient_checkpointing = True

    def set_attention_slice(self, slice_size):
        pass  # attention never materialises probabilities; slicing is meaningless here

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        r = super().load_state_dict(state_dict, strict=strict, **kw)
        self._dirty = True
        return r

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._dirty = True
        return r

    def mark_weights_dirty(self):
        """Call after mutating parameters in place (outside load_state_dict / .to()) so they are re-packed."""
        self._dirty = True

    # ------------------------------------------------------------------------------------------ native handle
    def _ensure_handle(self):
        if self._handle is not None:
            return
        cfg = self.cfg
        s = _lib.UNetConfigStruct()
        s.in_channels, s.out_channels = cfg.in_channels, cfg.out_channels
        for i, c in enumerate(cfg.block_out_channels):
            s.block_out_channels[i] = c
        s.layers_per_block = cfg.layers_per_block
        s.num_heads = cfg.attention_head_dim
        s.cross_attention_dim = cfg.cross_attention_dim
        s.norm_num_groups = cfg.norm_num_groups
        s.norm_eps = cfg.norm_eps
        s.use_motion_module = int(cfg.use_motion_module)
        for i in range(4):
            s.motion_down[i] = int(cfg.down_has_motion(i))
            s.motion_up[i] = int(cfg.up_has_motion(i))
        s.motion_mid = int(cfg.use_motion_module and cfg.motion_module_mid_block)
        s.motion_num_heads = cfg.motion_num_attention_heads
        s.pe_max_len = cfg.temporal_position_encoding_max_len
        h = C.c_void_p()
        _lib.call("vs_unet_create", C.byref(s), C.byref(h))
        self._handle = h

    def _sync_weights(self, device):
        self._ensure_handle()
        if not self._dirty:
            return
        sd = super().state_dict()
        names = [k for k in sd if not k.endswith(".pe")]
        stream = torch.cuda.current_stream().cuda_stream
        CH = 64                                     # bounded staging memory: convert + upload in chunks
        for i in range(0, len(names), CH):
            chunk = names[i:i + CH]
            tensors = [sd[k].detach().to(device=device, dtype=torch.float16).contiguous() for k in chunk]
            arr_n = (C.c_char_p * len(chunk))(*[k.encode() for k in chunk])
            arr_p = (C.c_void_p * len(chunk))(*[t.data_ptr() for t in tensors])
            arr_c = (C.c_int64 * len(chunk))(*[t.numel() for t in tensors])
            _lib.call("vs_unet_load_weights", self._handle, stream, len(chunk), arr_n, arr_p, arr_c)
            torch.cuda.current_stream().synchronize()   # staging tensors die at the end of the iteration
        self._dirty = False

    def _prepare_inputs(self, dev, timestep, n, encoder_hidden_states=None, sample_dtype=None):
        """What every CUDA entry point does before its launch.  It refuses a device other than CUDA and a sample dtype
        other than fp16 / fp32 (sample_dtype None: there is no sample) before any weight upload, then syncs the weights.
        Returns (t, ehs): the timestep (a number, or a tensor of 1 or n values) as a contiguous fp32 [n] tensor on dev,
        and encoder_hidden_states as a contiguous fp16 tensor on dev (None when not given)."""
        if dev.type != "cuda":
            raise RuntimeError("AnimateDiffUNet3DModel (videoswap_b200) runs on CUDA only: there is no CPU path")
        if sample_dtype is not None and sample_dtype not in (torch.float16, torch.float32):
            raise TypeError("sample must be fp16 or fp32")
        with torch.cuda.device(dev):
            self._sync_weights(dev)
            if torch.is_tensor(timestep):
                t = timestep.to(device=dev, dtype=torch.float32).reshape(-1)
            else:
                t = torch.tensor([float(timestep)], dtype=torch.float32, device=dev)
            t = t.expand(n).contiguous()
            ehs = None
            if encoder_hidden_states is not None:
                ehs = encoder_hidden_states.to(device=dev, dtype=torch.float16).contiguous()
        return t, ehs

    def _check_processors(self):
        """Validates the processors the reference's helpers may have swapped in and returns the attention controller the
        control processors carry (utils/p2p_utils/attention_register.py), or None."""
        idx = 0
        controller = None
        for blocks in (self.down_blocks, [self.mid_block], self.up_blocks):
            for blk in blocks:
                for tr in getattr(blk, "attentions", []):
                    p = tr.transformer_blocks[0].attn2.processor
                    ci = getattr(p, "cross_attention_idx", None)
                    if ci is not None and ci != idx:
                        raise NotImplementedError("ED-LoRA cross_attention_idx differs from registration order")
                    for a in (tr.transformer_blocks[0].attn1, tr.transformer_blocks[0].attn2):
                        ctl = getattr(a.processor, "controller", None)
                        if ctl is not None:
                            if controller is not None and ctl is not controller:
                                raise NotImplementedError("all attention layers must share ONE controller (as "
                                                          "register_attention_control sets them, attention_register.py:176-211)")
                            controller = ctl
                    idx += 1
        return controller

    def level_sizes(self, H: int, W: int):
        """(H_l, W_l) of the four levels: the stride-2 convs of the down path give H_{l+1} = ceil(H_l / 2)."""
        sizes = [(H, W)]
        for _ in range(3):
            h, w = sizes[-1]
            sizes.append(((h + 1) // 2, (w + 1) // 2))
        return sizes

    def _check_residuals(self, residuals, n, H, W):
        """The library reads residual l as [(B F), C_l, H_l, W_l]: anything else is refused before any launch."""
        if len(residuals) > 4:
            raise ValueError(f"down_block_additional_residuals: at most 4 tensors, got {len(residuals)}")
        for l, (r, (h, w)) in enumerate(zip(residuals, self.level_sizes(H, W))):
            want = (n, self.cfg.block_out_channels[l], h, w)
            if tuple(r.shape) != want:
                raise ValueError(f"down_block_additional_residuals[{l}] has shape {tuple(r.shape)}; the UNet reads "
                                 f"{list(want)} ([(B F), C_l, H_l, W_l] with H_l = ceil(H_(l-1) / 2)) at latent {H}x{W}")

    def __del__(self):
        try:
            if self._handle is not None:
                _lib.lib().vs_unet_destroy(self._handle)
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, sample: torch.Tensor, timestep: Union[torch.Tensor, float, int], encoder_hidden_states: torch.Tensor,
                class_labels=None, attention_mask=None, cross_attention_kwargs=None,
                down_block_additional_residuals: Optional[List[torch.Tensor]] = None, return_dict: bool = True,
                _taps: Optional[dict] = None):
        if class_labels is not None or attention_mask is not None:
            raise NotImplementedError("class_labels / attention_mask are unused on the reference's path and unsupported")
        if sample.dim() != 5:
            raise ValueError(f"Expected sample of shape [B,C,F,H,W], got {tuple(sample.shape)}")
        B, Cin, F, H, W = sample.shape
        if Cin != self.cfg.in_channels:
            raise ValueError(f"sample has {Cin} channels, expected {self.cfg.in_channels}")
        dev = sample.device
        controller = self._check_processors()
        if controller is not None and (H % 8 or W % 8):
            raise NotImplementedError("attention controllers need latent H and W to be multiples of 8 (their latent blend "
                                      "rebuilds each map's height and width from its token count and the aspect ratio)")
        if down_block_additional_residuals is not None:
            self._check_residuals(down_block_additional_residuals, B * F, H, W)
        t, ehs = self._prepare_inputs(dev, timestep, B, encoder_hidden_states, sample.dtype)
        with torch.cuda.device(dev):
            io_f32 = sample.dtype == torch.float32
            x = sample.contiguous()
            if ehs.dim() == 4:
                layers, tokens = ehs.shape[1], ehs.shape[2]
            elif ehs.dim() == 3:
                layers, tokens = 0, ehs.shape[1]
            else:
                raise ValueError("encoder_hidden_states must be [B,N,D] or [B,L,N,D]")
            if ehs.shape[0] != B or ehs.shape[-1] != self.cfg.cross_attention_dim:
                raise ValueError("encoder_hidden_states batch / feature size mismatch")
            res_ptrs = None
            keep = []
            if down_block_additional_residuals is not None and len(down_block_additional_residuals) > 0:
                res_ptrs = (C.c_void_p * 4)()
                for i in range(4):
                    if len(down_block_additional_residuals) == 0:
                        break
                    r = down_block_additional_residuals.pop(0)           # consumed in place, like unet.py:422,435
                    r = r.to(device=dev, dtype=torch.float16).contiguous()
                    keep.append(r)
                    res_ptrs[i] = r.data_ptr()
            out = torch.empty_like(x)
            if _taps is not None:
                _lib.call("vs_unet_enable_taps", self._handle, 1)
            hook_err = []
            if controller is not None:
                # attention controllers (SURVEY 8f-2): the library hands every small-resolution layer's probabilities
                # [(b f), heads, s, t] to the controller between softmax and P V, as a zero-copy view of its device buffer
                from . import p2p

                def _hook(user, layer, is_cross, place, ptr, batch, heads, nq, nk, stream):
                    if hook_err:
                        return
                    try:
                        view = p2p.tensor_view(ptr, (batch, heads, nq, nk), dev)
                        res = controller(view, bool(is_cross), p2p._PLACES[place])
                        if res is not None and res.data_ptr() != view.data_ptr():
                            view.copy_(res.to(device=dev, dtype=torch.float16).reshape(view.shape))
                    except BaseException as e:  # noqa: BLE001  (ctypes would swallow it: re-raised after the forward)
                        hook_err.append(e)
                cb = p2p.HOOK_TYPE(_hook)
                _lib.call("vs_unet_set_attention_hook", self._handle, cb, None, p2p.MAX_QUERIES)
            try:
                _lib.call("vs_unet_forward", self._handle, torch.cuda.current_stream().cuda_stream, x.data_ptr(), int(io_f32),
                          B, F, H, W, t.data_ptr(), ehs.data_ptr(), tokens, layers, res_ptrs, 0, 1.0, out.data_ptr())
            finally:
                if controller is not None:
                    _lib.call("vs_unet_set_attention_hook", self._handle, None, None, 0)
            if hook_err:
                raise hook_err[0]
            if _taps is not None:
                n = _lib.lib().vs_unet_num_taps(self._handle)
                for i in range(n):
                    name, ptr = C.c_char_p(), C.c_void_p()
                    ni, hh, ww, cc = C.c_int(), C.c_int(), C.c_int(), C.c_int()
                    _lib.call("vs_unet_get_tap", self._handle, i, C.byref(name), C.byref(ptr), C.byref(ni), C.byref(hh),
                              C.byref(ww), C.byref(cc))
                    buf = torch.empty((ni.value, hh.value, ww.value, cc.value), dtype=torch.float16, device=dev)
                    _lib.call("vs_unet_copy_tap", self._handle, torch.cuda.current_stream().cuda_stream, i, buf.data_ptr())
                    _taps[name.value.decode()] = buf
                _lib.call("vs_unet_enable_taps", self._handle, 0)
            self._keepalive = (x, t, ehs, keep)      # inputs must outlive the asynchronous kernels
        if not return_dict:
            return (out,)
        return UNet3DConditionOutput(sample=out)


    @torch.no_grad()
    def forward_features(self, sample: torch.Tensor, timestep: Union[torch.Tensor, float, int],
                         encoder_hidden_states: torch.Tensor, up_ft_index: int = 1) -> torch.Tensor:
        """The DIFT featurizer's partial forward (dift_util.py MyUNet2DConditionModel): the 2-D UNet -- every motion
        module skipped -- up to and including up block `up_ft_index` with its up-sampler.  sample [N, C, 1, H, W] (fp16 /
        fp32; every image on the batch axis, so each one gets its own GroupNorm statistics), encoder_hidden_states
        [N, 77, D] -> up_ft[up_ft_index] as NHWC fp16 [N, h_k, w_k, C_k]."""
        if sample.dim() != 5 or sample.shape[2] != 1 or sample.shape[1] != self.cfg.in_channels:
            raise ValueError(f"expected sample [N, {self.cfg.in_channels}, 1, H, W], got {tuple(sample.shape)}")
        if not 0 <= int(up_ft_index) <= 3:
            raise ValueError(f"up_ft_index must be in 0..3, got {up_ft_index}")
        N, _, _, H, W = sample.shape
        if encoder_hidden_states.dim() != 3 or encoder_hidden_states.shape[0] != N or \
                encoder_hidden_states.shape[-1] != self.cfg.cross_attention_dim:
            raise ValueError(f"encoder_hidden_states must be [{N}, tokens, {self.cfg.cross_attention_dim}], got "
                             f"{tuple(encoder_hidden_states.shape)}")
        dev = sample.device
        k = int(up_ft_index)
        lh, lw = self.level_sizes(H, W)[2 - k] if k < 3 else (H, W)
        ck = self.cfg.block_out_channels[3 - k]
        t, ehs = self._prepare_inputs(dev, timestep, N, encoder_hidden_states, sample.dtype)
        with torch.cuda.device(dev):
            x = sample.contiguous()
            out = torch.empty((N, lh, lw, ck), dtype=torch.float16, device=dev)
            _lib.call("vs_unet_forward_features", self._handle, torch.cuda.current_stream().cuda_stream, x.data_ptr(),
                      int(x.dtype == torch.float32), N, 1, H, W, t.data_ptr(), ehs.data_ptr(), ehs.shape[1], 0, k,
                      out.data_ptr())
            self._keepalive = (x, t, ehs)
        return out

    @torch.no_grad()
    def time_embedding_rows(self, timesteps: torch.Tensor):
        """The forward's time embedding for timesteps [B] -> (emb fp32 [B, time_embed_dim], proj fp32 [B, tproj_n]): proj
        holds every resnet's time_emb_proj(SiLU(emb)) side by side, in the order the library registers the resnets."""
        dev = self.conv_in.weight.device
        B = timesteps.numel()
        t, _ = self._prepare_inputs(dev, timesteps, B)
        tproj_n = sum(m.time_emb_proj.weight.shape[0] for m in self.modules() if isinstance(getattr(m, "time_emb_proj", None), _Holder))
        with torch.cuda.device(dev):
            emb = torch.empty((B, self.cfg.time_embed_dim), dtype=torch.float32, device=dev)
            proj = torch.empty((B, tproj_n), dtype=torch.float32, device=dev)
            _lib.call("vs_unet_time_embedding", self._handle, torch.cuda.current_stream().cuda_stream, t.data_ptr(), B,
                      emb.data_ptr(), proj.data_ptr())
            self._keepalive = (t,)
        return emb, proj


UNet3DConditionModel = AnimateDiffUNet3DModel
