"""Deterministic, construction-order-independent synthetic weights.  No pretrained checkpoints exist offline
(SURVEY.md 0.5), so parity and benchmarks use the real architecture with weights drawn per key from a generator
seeded by (seed, crc32(key)).  Motion-module `proj_out` is given NON-zero weights on purpose: the reference
zero-initialises it (motion_module.py:76-77), which would make every motion module an identity and leave the
temporal path untested.  Also the helpers the host model classes share to read a local pretrained directory and to
report a state_dict's missing keys."""
from __future__ import annotations

import json
import math
import os
import zlib
from collections import OrderedDict
from dataclasses import fields
from typing import Dict, List, Optional, Tuple

import torch


def temporal_pe_table(length: int, dim: int) -> torch.Tensor:
    """Closed-form sinusoid of the reference's PositionalEncoding (motion_module.py:242-251)."""
    pos = torch.arange(length, dtype=torch.float32)[:, None]
    div = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * (-math.log(10000.0) / dim))
    pe = torch.zeros(1, length, dim)
    pe[0, :, 0::2] = torch.sin(pos * div)
    pe[0, :, 1::2] = torch.cos(pos * div)
    return pe


def seeded_state_dict(shapes: Dict[str, Tuple[int, ...]], seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    sd = OrderedDict()
    for name, shape in shapes.items():
        if name.endswith(".pe"):
            sd[name] = temporal_pe_table(shape[1], shape[2])
            continue
        g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(name.encode())) % (2 ** 63 - 1))
        if len(shape) >= 2:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            bound = 1.0 / math.sqrt(fan_in)
            t = (torch.rand(shape, generator=g) * 2 - 1) * bound
        elif name.endswith(".weight"):          # 1-D weights are norm scales
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            t = 0.02 * torch.randn(shape, generator=g)
        sd[name] = t
    return sd


def missing_keys_text(missing: List[str]) -> str:
    """The first five of a state_dict's missing keys and their count, for error messages."""
    return f"{missing[:5]}{' ...' if len(missing) > 5 else ''} ({len(missing)} keys)"


def config_kwargs(config, config_cls) -> dict:
    """The entries of a config.json dict (or of an object with to_dict()) that are fields of the dataclass config_cls,
    JSON lists as tuples; the rest (class name, block types, ...) is dropped."""
    if not isinstance(config, dict):
        config = config.to_dict()
    known = {f.name for f in fields(config_cls)}
    return {k: (tuple(v) if isinstance(v, list) else v) for k, v in config.items() if k in known}


def read_pretrained_dir(path: str, subfolder: Optional[str], safetensors_name: str,
                        bin_name: str) -> Tuple[dict, Dict[str, torch.Tensor]]:
    """A local diffusers / transformers model directory (path/subfolder, or path itself without a subfolder) -> (its
    parsed config.json, its state_dict on the CPU).  The weights come from safetensors_name when it exists, else from
    bin_name (loaded with weights_only=True)."""
    d = os.path.join(path, subfolder) if subfolder else path
    cfg_path = os.path.join(d, "config.json")
    if not os.path.exists(cfg_path):
        raise RuntimeError(f"{cfg_path} not found")
    with open(cfg_path) as f:
        config = json.load(f)
    st, bn = os.path.join(d, safetensors_name), os.path.join(d, bin_name)
    if os.path.exists(st):
        from safetensors.torch import load_file
        sd = load_file(st)
    elif os.path.exists(bn):
        sd = torch.load(bn, map_location="cpu", weights_only=True)
    else:
        raise RuntimeError(f"no {safetensors_name} / {bin_name} in {d}")
    return config, sd
