"""CPU tests of the pretrained-directory reader and the config filter that AutoencoderKL.from_pretrained and
CLIPTextModel.from_pretrained share: config.json plus a .bin, safetensors preferred over .bin, the errors for a missing
config.json or weight file, and a config.json filtered to a config dataclass's fields."""
import json

import pytest
import torch

from videoswap_b200.spec import CLIPTextConfig, VAEConfig
from videoswap_b200.weights import config_kwargs, read_pretrained_dir

ST, BIN = "diffusion_pytorch_model.safetensors", "diffusion_pytorch_model.bin"
CONFIG = {"_class_name": "AutoencoderKL", "block_out_channels": [64, 128], "act_fn": "silu", "sample_size": 256}


def _weights(seed):
    g = torch.Generator().manual_seed(seed)
    return {"decoder.conv_in.weight": torch.randn(8, 4, 3, 3, generator=g), "decoder.conv_in.bias": torch.randn(8, generator=g)}


def _dir(tmp_path, subfolder="vae"):
    d = tmp_path / subfolder
    d.mkdir(parents=True)
    (d / "config.json").write_text(json.dumps(CONFIG))
    return d


def _equal(a, b):
    return a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def test_bin_directory(tmp_path):
    d = _dir(tmp_path)
    torch.save(_weights(1), d / BIN)
    config, sd = read_pretrained_dir(str(tmp_path), "vae", ST, BIN)
    assert config == CONFIG
    assert _equal(sd, _weights(1))
    config, sd = read_pretrained_dir(str(d), None, ST, BIN)            # no subfolder: the directory itself
    assert config == CONFIG and _equal(sd, _weights(1))


def test_safetensors_wins_over_bin(tmp_path):
    safetensors_torch = pytest.importorskip("safetensors.torch")
    d = _dir(tmp_path)
    torch.save(_weights(1), d / BIN)
    safetensors_torch.save_file(_weights(2), str(d / ST))
    _, sd = read_pretrained_dir(str(tmp_path), "vae", ST, BIN)
    assert _equal(sd, _weights(2)) and not _equal(sd, _weights(1))


def test_missing_config_json(tmp_path):
    d = tmp_path / "text_encoder"
    d.mkdir()
    torch.save(_weights(1), d / "pytorch_model.bin")
    with pytest.raises(RuntimeError, match="config.json not found"):
        read_pretrained_dir(str(tmp_path), "text_encoder", "model.safetensors", "pytorch_model.bin")


def test_missing_weight_file(tmp_path):
    d = _dir(tmp_path, "text_encoder")
    torch.save(_weights(1), d / "other.bin")
    with pytest.raises(RuntimeError, match="no model.safetensors / pytorch_model.bin in .*text_encoder"):
        read_pretrained_dir(str(tmp_path), "text_encoder", "model.safetensors", "pytorch_model.bin")


def test_bin_is_loaded_weights_only(tmp_path):
    d = _dir(tmp_path)
    torch.save({"decoder.conv_in.bias": torch.zeros(8), "extra": object()}, d / BIN)
    with pytest.raises(Exception, match="[Ww]eights.only"):
        read_pretrained_dir(str(tmp_path), "vae", ST, BIN)


def test_config_filter_drops_unknown_keys_and_makes_lists_tuples():
    kw = config_kwargs(CONFIG, VAEConfig)
    assert kw == {"block_out_channels": (64, 128), "sample_size": 256}
    assert VAEConfig(**kw).block_out_channels == (64, 128)
    clip = {"architectures": ["CLIPTextModel"], "hidden_size": 768, "num_hidden_layers": 2, "projection_dim": 768}
    assert config_kwargs(clip, CLIPTextConfig) == {"hidden_size": 768, "num_hidden_layers": 2}
    assert config_kwargs(VAEConfig(layers_per_block=3), VAEConfig) == VAEConfig(layers_per_block=3).to_dict()
