"""A complete pretrained directory and test-config inputs on disk, from the seeded weights the other GPU tests use, for
`videoswap_b200.run` (tests/test_run_gpu.py, tools/gpu_run_config.py):

  <root>/sd/unet/           config.json (SD-1.5's 2-D UNet config) + diffusion_pytorch_model.bin (2-D weights, fp16)
  <root>/sd/vae/            config.json + diffusion_pytorch_model.safetensors (decoder and encoder)
  <root>/sd/text_encoder/   config.json + model.safetensors
  <root>/sd/tokenizer/      a byte-level CLIP BPE vocabulary of 49408 entries (vocab.json, merges.txt, tokenizer_config.json)
  <root>/sd/scheduler/      SD-1.5's scheduler_config.json
  <root>/motion_module.ckpt AnimateDiff-format motion-module weights (`...pos_encoder.pe` keys)
  <root>/adapter.pth        SparsePointAdapter state dict
  <root>/edlora_<c>.pth     ED-LoRA file with two concepts; <root>/TAP_*.pth track files; <root>/frames/ PNG frames

The UNet weights are seeded_state_dict(unet_param_shapes, seed=0) (tests/unet_checks.get_model), the VAE's seed 7, the text
encoder's text.SEED and the adapter's seed 5 -- the init="seeded" weights of each class."""
from __future__ import annotations

import json
import os
import shutil
from dataclasses import asdict

import torch

from videoswap_b200 import formats, spec, text
from videoswap_b200.weights import seeded_state_dict

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
UNET_2D_CONFIG = {
    "_class_name": "UNet2DConditionModel", "_diffusers_version": "0.6.0", "act_fn": "silu", "attention_head_dim": 8,
    "block_out_channels": [320, 640, 1280, 1280], "center_input_sample": False, "cross_attention_dim": 768,
    "down_block_types": ["CrossAttnDownBlock2D"] * 3 + ["DownBlock2D"], "downsample_padding": 1, "flip_sin_to_cos": True,
    "freq_shift": 0, "in_channels": 4, "layers_per_block": 2, "mid_block_scale_factor": 1, "norm_eps": 1e-05,
    "norm_num_groups": 32, "out_channels": 4, "sample_size": 64, "up_block_types": ["UpBlock2D"] + ["CrossAttnUpBlock2D"] * 3}
# SD-1.5's scheduler/scheduler_config.json: a PNDM config, which the reference loads as a DDIMScheduler
SCHEDULER_CONFIG = {"_class_name": "PNDMScheduler", "_diffusers_version": "0.6.0", "beta_end": 0.012,
                    "beta_schedule": "scaled_linear", "beta_start": 0.00085, "num_train_timesteps": 1000,
                    "set_alpha_to_one": False, "skip_prk_steps": True, "steps_offset": 1, "trained_betas": None,
                    "clip_sample": False}


def _bytes_to_unicode():
    """GPT-2 / CLIP's reversible byte -> printable character table."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return [chr(c) for c in cs]


def write_tokenizer(d, words=()):
    """A CLIPTokenizer directory that loads offline: the 512 byte-level symbols, one merge chain per word of `words` (so
    those words are single tokens, as common words are in CLIP's vocabulary), padding entries up to 49406, then
    <|startoftext|> 49406 and <|endoftext|> 49407."""
    os.makedirs(d, exist_ok=True)
    base = _bytes_to_unicode()
    vocab = base + [c + "</w>" for c in base]
    merges = []
    for w in sorted({w.lower() for w in words if w.isalpha() and len(w) > 1}):
        cur = w[0]
        for i, c in enumerate(w[1:], 1):
            nxt = c + "</w>" if i == len(w) - 1 else c
            merges.append(f"{cur} {nxt}")
            cur += nxt
            if cur not in vocab:
                vocab.append(cur)
    merges = list(dict.fromkeys(merges))
    if not merges:                      # the tokenizer wants at least one merge
        merges, vocab = ["a b"], vocab + ["ab"]
    vocab += [f"<unused{i}>" for i in range(49406 - len(vocab))]
    vocab += ["<|startoftext|>", "<|endoftext|>"]
    with open(os.path.join(d, "vocab.json"), "w") as f:
        json.dump({t: i for i, t in enumerate(vocab)}, f)
    with open(os.path.join(d, "merges.txt"), "w") as f:
        f.write("#version: 0.2\n" + "\n".join(merges))
    with open(os.path.join(d, "tokenizer_config.json"), "w") as f:
        json.dump({"model_max_length": 77, "do_lower_case": True, "bos_token": "<|startoftext|>",
                   "eos_token": "<|endoftext|>", "unk_token": "<|endoftext|>", "pad_token": "<|endoftext|>"}, f)


def _half(sd):
    return {k: (v if k.endswith(".pe") else v.half()) for k, v in sd.items()}


def write_pretrained(root, words=()) -> dict:
    """The pretrained directory, the motion module, the adapter and the model configs; returns their paths."""
    from safetensors.torch import save_file
    sd_dir = os.path.join(root, "sd")
    unet_sd = seeded_state_dict(spec.unet_param_shapes(spec.UNetConfig()), seed=0)
    os.makedirs(os.path.join(sd_dir, "unet"), exist_ok=True)
    with open(os.path.join(sd_dir, "unet", "config.json"), "w") as f:
        json.dump(UNET_2D_CONFIG, f)
    torch.save(_half({k: v for k, v in unet_sd.items() if "motion_modules" not in k}),
               os.path.join(sd_dir, "unet", "diffusion_pytorch_model.bin"))
    motion = os.path.join(root, "motion_module.ckpt")
    torch.save(_half({k.replace(".processor.pos_encoder", ".pos_encoder"): v for k, v in unet_sd.items()
                      if "motion_modules" in k}), motion)
    del unet_sd

    vcfg = spec.VAEConfig()
    os.makedirs(os.path.join(sd_dir, "vae"), exist_ok=True)
    with open(os.path.join(sd_dir, "vae", "config.json"), "w") as f:
        json.dump({"_class_name": "AutoencoderKL", "act_fn": "silu", **asdict(vcfg)}, f)
    save_file(seeded_state_dict({**spec.vae_param_shapes(vcfg), **spec.vae_encoder_param_shapes(vcfg)}, seed=7),
              os.path.join(sd_dir, "vae", "diffusion_pytorch_model.safetensors"))

    tcfg = spec.CLIPTextConfig()
    os.makedirs(os.path.join(sd_dir, "text_encoder"), exist_ok=True)
    with open(os.path.join(sd_dir, "text_encoder", "config.json"), "w") as f:
        json.dump({"architectures": ["CLIPTextModel"], **asdict(tcfg)}, f)
    save_file(seeded_state_dict(spec.clip_text_param_shapes(tcfg), seed=text.SEED),
              os.path.join(sd_dir, "text_encoder", "model.safetensors"))

    write_tokenizer(os.path.join(sd_dir, "tokenizer"), words)
    os.makedirs(os.path.join(sd_dir, "scheduler"), exist_ok=True)
    with open(os.path.join(sd_dir, "scheduler", "scheduler_config.json"), "w") as f:
        json.dump(SCHEDULER_CONFIG, f)

    adapter = os.path.join(root, "adapter.pth")
    torch.save(seeded_state_dict(spec.adapter_param_shapes(), seed=5), adapter)
    cfg_dir = os.path.join(root, "model_cfg")
    os.makedirs(cfg_dir, exist_ok=True)
    for name in ("inference.yml", "point_adapter.yml"):
        shutil.copy(os.path.join(GOLD, "model_cfg", name), cfg_dir)
    return {"pretrained_model_path": sd_dir, "motion_module_path": motion, "pretrained_adapter_path": adapter,
            "inference_config_path": os.path.join(cfg_dir, "inference.yml"),
            "model_config_path": os.path.join(cfg_dir, "point_adapter.yml")}


def write_edlora(path, concepts, seed=401):
    """An ED-LoRA file: rank-4 LoRA pairs on the down_blocks.1 / up_blocks.2.attentions.0 projections of the UNet and on
    three text-encoder layers, and a 16 x 768 embedding per concept."""
    g = torch.Generator().manual_seed(seed)
    lora_unet = {}
    for k, shape in spec.unet_param_shapes(spec.UNetConfig()).items():
        dn = formats.lora_down_name(k)
        if dn == k or "motion_modules" in k or not any(s in k for s in ("down_blocks.1.", "up_blocks.2.attentions.0.")):
            continue
        down, up = 0.05 * torch.randn((4, shape[1]), generator=g), 0.05 * torch.randn((shape[0], 4), generator=g)
        if len(shape) == 4:
            down, up = down[:, :, None, None], up[:, :, None, None]
        lora_unet[dn], lora_unet[dn.replace("lora_down", "lora_up")] = down, up
    lora_te = {}
    for i in (0, 6, 11):
        for site, (o, n) in (("self_attn.q_proj", (768, 768)), ("mlp.fc1", (3072, 768))):
            lora_te[f"text_model.encoder.layers.{i}.{site}.lora_down.weight"] = 0.05 * torch.randn(4, n, generator=g)
            lora_te[f"text_model.encoder.layers.{i}.{site}.lora_up.weight"] = 0.05 * torch.randn(o, 4, generator=g)
    emb = {c: 0.02 * torch.randn(16, 768, generator=g) for c in concepts}
    torch.save({"params": {"new_concept_embedding": emb, "unet": lora_unet, "text_encoder": lora_te}}, path)
    return path


def write_tap(path, frames, width, height, names, seed):
    """A TAP file of `frames` frames: tracks inside the frame (point 1 invisible in frame 0), one embedding per point."""
    g = torch.Generator().manual_seed(seed)
    tracks = torch.rand((frames, len(names), 2), generator=g) * torch.tensor([width - 20.0, height - 20.0]) + 10
    tracks[0, 1] = -1.0
    torch.save({"pred_tracks": tracks, "point_embedding": torch.randn((len(names), 1280), generator=g),
                "point_name2id": {n: i for i, n in enumerate(names)}}, path)
    return path


def write_frames(d, n, width, height, seed=7):
    """n PNG frames of a smooth pattern drifting one cell per frame (image-like input for the VAE, not noise)."""
    import numpy as np
    from PIL import Image
    os.makedirs(d, exist_ok=True)
    g = torch.Generator().manual_seed(seed)
    base = torch.rand((max(height // 16, 1), max(width // 16, 1), 3), generator=g)
    for f in range(n):
        img = torch.roll(base, shifts=f, dims=1).permute(2, 0, 1)[None]
        img = torch.nn.functional.interpolate(img, size=(height, width), mode="bilinear", align_corners=False)[0]
        Image.fromarray((img.permute(1, 2, 0) * 255).round().byte().numpy().astype(np.uint8), "RGB").save(
            os.path.join(d, f"{f:05d}.png"))
    return d
