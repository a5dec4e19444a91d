"""CPU tests of the VAE decoder's host side: the decoder-side state_dict surface against the oracle's restatement of
diffusers 0.19.3, the old / new attention names, loud failures on unknown and missing keys, the latents-only pipeline,
and the postprocess arithmetic of the image_postprocess kernel against VaeImageProcessor.postprocess."""
import numpy as np
import pytest
import torch

import videoswap_b200 as V
from tests import vae_oracle as VO
from videoswap_b200 import vae as VAE


def _sd(seed=7):
    return V.seeded_state_dict(V.vae_param_shapes(V.VAEConfig()), seed=seed)


def test_decoder_keys_and_shapes_match_the_oracle():
    cfg = V.VAEConfig()
    assert (cfg.block_out_channels, cfg.layers_per_block, cfg.latent_channels, cfg.norm_num_groups, cfg.scaling_factor) == \
        ((128, 256, 512, 512), 2, 4, 32, 0.18215)
    shapes = V.vae_param_shapes(cfg)
    assert dict(shapes) == dict(VO.param_shapes())
    assert sum(int(np.prod(s)) for s in shapes.values()) == 49_490_199
    assert sum(1 for k in shapes if k.endswith("conv_shortcut.weight")) == 2          # up blocks 2 and 3, first resnet
    assert sum(1 for k in shapes if ".upsamplers.0.conv.weight" in k) == 3


def test_old_and_new_attention_names_give_the_same_weights():
    new = _sd()
    a = "decoder.mid_block.attentions.0"
    old = {}
    for k, v in new.items():
        for o, n in VAE._OLD_ATTN.items():
            if k.startswith(f"{a}.{n}."):
                leaf = k.rsplit(".", 1)[1]
                k = f"{a}.{o}.{leaf}"
                if leaf == "weight":
                    v = v[..., None, None]                      # the 1x1-conv form of older checkpoints
                break
        old[k] = v
    assert f"{a}.query.weight" in old and old[f"{a}.proj_attn.weight"].shape == (512, 512, 1, 1)
    full = dict(old)
    full["encoder.conv_in.weight"] = torch.zeros(128, 3, 3, 3)        # the encode half is accepted and ignored
    full["quant_conv.weight"] = torch.zeros(8, 8, 1, 1)
    cfg = V.VAEConfig()
    a_, b_ = VAE.convert_state_dict(new, cfg), VAE.convert_state_dict(full, cfg)
    assert a_.keys() == b_.keys()
    assert all(torch.equal(a_[k], b_[k]) for k in a_)


def test_unknown_and_missing_keys_raise():
    cfg = V.VAEConfig()
    sd = _sd()
    with pytest.raises(KeyError, match="unexpected"):
        VAE.convert_state_dict({**sd, "decoder.mid_block.attentions.0.to_x.weight": torch.zeros(512, 512)}, cfg)
    with pytest.raises(KeyError, match="unexpected"):
        VAE.convert_state_dict({**sd, "decoder.conv_out.lora.weight": torch.zeros(3)}, cfg)
    sd2 = dict(sd)
    del sd2["decoder.up_blocks.3.resnets.0.conv_shortcut.bias"]
    with pytest.raises(KeyError, match="missing"):
        VAE.convert_state_dict(sd2, cfg)
    with pytest.raises(ValueError, match="shape"):
        VAE.convert_state_dict({**sd, "decoder.conv_out.weight": torch.zeros(4, 128, 3, 3)}, cfg)
    dup = {**sd, "decoder.mid_block.attentions.0.query.weight": torch.zeros(512, 512)}
    with pytest.raises(KeyError, match="twice"):
        VAE.convert_state_dict(dup, cfg)


def test_cpu_device_is_rejected_loudly():
    with pytest.raises(RuntimeError, match="CUDA only"):
        V.AutoencoderKL(device="cpu")


def test_pipeline_without_vae_still_returns_latents_only():
    pipe = V.VideoSwapPipeline(V.AnimateDiffUNet3DModel(init="empty"))
    assert pipe.vae is None
    for ot in ("pil", "pt", "np"):
        with pytest.raises(NotImplementedError):
            pipe(torch.zeros(1, 77, 768), torch.zeros(1, 4, 1, 8, 8), output_type=ot)
    with pytest.raises(NotImplementedError):
        pipe.decode_latents(torch.zeros(1, 4, 8, 8))


def _crafted():
    """fp16 decoder outputs: 0, +-1, +-1.0001, values far outside [-1, 1], and every fp16 x in [-1, 1] whose
    fl32(fl32(x / 2 + 0.5) * 255) lands exactly on a half."""
    every = torch.arange(-0x3c00, 0x3c01, dtype=torch.int32)
    h = torch.where(every < 0, (-every) | 0x8000, every).to(torch.int16).view(torch.float16)
    y = (h.float() * 0.5 + 0.5) * 255
    halves = h[(y - y.floor()) == 0.5]
    base = torch.tensor([0.0, 1.0, -1.0, 1.0001, -1.0001, 3.0, -7.5, 65504.0, -65504.0]).half()
    return torch.cat([base, halves]), halves.numel()


def test_postprocess_arithmetic_matches_the_oracle():
    """image_postprocess computes y = min(max(fl(fl(x * 0.5) + 0.5), 0), 1) in fp32 and uint8 = round-half-even(fl(y * 255))
    (__float2int_rn); VaeImageProcessor.postprocess computes (x / 2 + 0.5).clamp(0, 1) and numpy's (y * 255).round()."""
    x, n_half = _crafted()
    assert n_half >= 2                          # x = 0 (127.5) and one more
    img = x.float().reshape(1, 1, 1, -1).expand(1, 3, 1, -1).contiguous()
    xs = x.float().numpy()
    y = np.minimum(np.maximum(np.float32(xs * np.float32(0.5)) + np.float32(0.5), np.float32(0)), np.float32(1))
    u8 = np.rint(y * np.float32(255)).astype(np.uint8)
    assert np.array_equal(VO.postprocess(img, "pt")[0, 0, 0].numpy(), y)
    assert np.array_equal(VO.postprocess(img, "np")[0, 0, :, 0], y)
    assert np.array_equal(VO.postprocess(img, "pil")[0, 0, :, 0], u8)
    assert u8[0] == 128 and u8[1] == 255 and u8[2] == 0 and u8[3] == 255 and u8[4] == 0
