"""CPU tests of the native T2IAdapter's host side: the config and state_dict checks (diffusers 0.19.3 FullAdapter key
names), from_pretrained on local .bin and safetensors directories, the frame preprocessing against the restated
_preprocess_adapter_image (tests/t2i_adapter_oracle.py), and every refusal, raised before anything reaches the GPU."""
import json

import numpy as np
import pytest
import torch
from PIL import Image

from tests import t2i_adapter_oracle as TO
from videoswap_b200 import SparsePointAdapter, T2IAdapter, T2IAdapterConfig, VideoSwapPipeline, t2i_adapter_param_shapes
from videoswap_b200.t2i_adapter import convert_state_dict, preprocess_frames
from videoswap_b200.weights import seeded_state_dict

SMALL = {"in_channels": 1, "channels": (64, 128), "num_res_blocks": 1}


def _frames(n, size, mode, seed=0):
    rng = np.random.default_rng(seed)
    w, h = size
    shape = (h, w) if mode == "L" else (h, w, 3)
    return [Image.fromarray(rng.integers(0, 256, shape, dtype=np.uint8), mode) for _ in range(n)]


def test_default_keys_follow_diffusers():
    sh = t2i_adapter_param_shapes(T2IAdapterConfig())
    assert sh["adapter.conv_in.weight"] == (320, 192, 3, 3)
    assert sh["adapter.body.1.in_conv.weight"] == (640, 320, 1, 1)
    assert sh["adapter.body.2.in_conv.weight"] == (1280, 640, 1, 1)
    assert "adapter.body.0.in_conv.weight" not in sh and "adapter.body.3.in_conv.weight" not in sh
    assert sh["adapter.body.3.resnets.1.block1.weight"] == (1280, 1280, 3, 3)
    assert sh["adapter.body.0.resnets.0.block2.weight"] == (320, 320, 1, 1)
    assert len(sh) == 2 + 4 * 2 * 4 + 2 * 2        # conv_in, 4 blocks x 2 resnets x (block1, block2), two in_convs
    assert t2i_adapter_param_shapes(T2IAdapterConfig(in_channels=1))["adapter.conv_in.weight"] == (320, 64, 3, 3)


def test_strict_state_dict():
    cfg = T2IAdapterConfig(**SMALL)
    sd = seeded_state_dict(t2i_adapter_param_shapes(cfg), seed=3)
    assert convert_state_dict(sd, cfg).keys() == sd.keys()
    with pytest.raises(KeyError, match="unexpected key.*adapter.body.0.in_conv.weight"):
        convert_state_dict({**sd, "adapter.body.0.in_conv.weight": torch.zeros(64, 64, 1, 1)}, cfg)
    bad = dict(sd)
    bad["adapter.body.1.resnets.0.block2.weight"] = torch.zeros(128, 128)
    with pytest.raises(ValueError, match="block2.weight: shape"):
        convert_state_dict(bad, cfg)
    part = dict(sd)
    del part["adapter.conv_in.bias"]
    with pytest.raises(KeyError, match="missing keys.*conv_in.bias"):
        convert_state_dict(part, cfg)
    with pytest.raises(KeyError):
        T2IAdapter(**SMALL, init="empty", device="cpu").load_state_dict(part)


def test_unsupported_configs_raise():
    with pytest.raises(NotImplementedError, match="light_adapter"):
        T2IAdapter(adapter_type="light_adapter", device="cpu")
    with pytest.raises(NotImplementedError, match="downscale_factor 16"):
        T2IAdapter(downscale_factor=16, device="cpu")
    with pytest.raises(ValueError, match="adapter_type"):
        T2IAdapter(adapter_type="other", device="cpu")
    with pytest.raises(NotImplementedError, match="MultiAdapter"):
        T2IAdapter.from_config({"_class_name": "MultiAdapter", "adapters": []}, device="cpu")
    with pytest.raises(NotImplementedError, match="MultiAdapter"):
        VideoSwapPipeline(None, adapter=[T2IAdapter(**SMALL, device="cpu"), T2IAdapter(**SMALL, device="cpu")])
    with pytest.raises(NotImplementedError, match="multiples of 64"):
        T2IAdapter(channels=(320, 100), device="cpu")


@pytest.mark.parametrize("fmt", ("bin", "safetensors"))
@pytest.mark.parametrize("subfolder", (None, "adapter"))
def test_from_pretrained(tmp_path, fmt, subfolder):
    cfg = T2IAdapterConfig(**SMALL)
    sd = seeded_state_dict(t2i_adapter_param_shapes(cfg), seed=9)
    d = tmp_path / subfolder if subfolder else tmp_path
    d.mkdir(parents=True, exist_ok=True)
    conf = {"_class_name": "T2IAdapter", "_diffusers_version": "0.19.3", "adapter_type": "full_adapter",
            "channels": [64, 128], "downscale_factor": 8, "in_channels": 1, "num_res_blocks": 1}
    (d / "config.json").write_text(json.dumps(conf))
    if fmt == "bin":
        torch.save(sd, d / "diffusion_pytorch_model.bin")
    else:
        pytest.importorskip("safetensors.torch").save_file(dict(sd), str(d / "diffusion_pytorch_model.safetensors"))
    ad = T2IAdapter.from_pretrained(str(tmp_path), subfolder=subfolder, device="cpu")
    assert ad.config == cfg and ad.total_downscale_factor == 16
    got = ad.state_dict()
    assert got.keys() == sd.keys() and all(torch.equal(got[k], sd[k]) for k in sd)


@pytest.mark.parametrize("mode", ("L", "RGB"))
def test_preprocessing_matches_restatement(mode):
    """Frame 0 sets the size; a frame of another size is resized with LANCZOS; u8 / 255 in fp32 is the restatement's
    input exactly."""
    frames = _frames(3, (128, 64), mode)
    frames[1] = _frames(1, (100, 77), mode, seed=5)[0]
    u8 = preprocess_frames(frames, 1 if mode == "L" else 3)
    assert u8.dtype == torch.uint8 and tuple(u8.shape) == (3, 64, 128, 1 if mode == "L" else 3)
    ref = TO.preprocess_adapter_image(frames, 64, 128)
    assert torch.equal(u8.permute(0, 3, 1, 2).float() / 255.0, ref)
    assert torch.equal(u8[1].permute(2, 0, 1).float() / 255.0,
                       TO.preprocess_adapter_image([frames[1].resize((128, 64), Image.LANCZOS)], 64, 128)[0])


def test_bad_frames_raise_before_any_launch():
    """Every refusal is a ValueError from the CPU checks: the adapter here lives on the CPU, so a check that let a bad
    input through would end in the RuntimeError of the missing device instead."""
    ad = T2IAdapter(device="cpu")
    ad1 = T2IAdapter(in_channels=1, device="cpu")
    cases = [
        (ad, [], "list of PIL images"),
        (ad, [torch.zeros(3, 64, 64)], "list of PIL images"),
        (ad, _frames(2, (64, 64), "RGB") + _frames(1, (64, 64), "L"), "mix image modes"),
        (ad, [Image.new("RGBA", (64, 64))], "'L' or 'RGB'"),
        (ad, [Image.new("P", (64, 64))], "'L' or 'RGB'"),
        (ad, _frames(2, (64, 64), "L"), "in_channels=3"),
        (ad1, _frames(2, (64, 64), "RGB"), "in_channels=1"),
        (ad, _frames(2, (96, 64), "RGB"), "multiples of 64"),
        (ad, _frames(2, (448, 760), "RGB"), "multiples of 64"),
        (ad, torch.zeros(2, 64, 64, 1, dtype=torch.uint8), r"uint8 frames \[F, H, W, 3\]"),
        (ad, torch.zeros(2, 64, 72, 3, dtype=torch.uint8), "multiples of 64"),
    ]
    for a, frames, msg in cases:
        with pytest.raises(ValueError, match=msg):
            a(frames)
    with pytest.raises(RuntimeError, match="CUDA only"):
        ad(_frames(1, (64, 64), "RGB"))


def test_pipeline_refuses_mismatched_conditions_before_any_launch():
    pos = torch.zeros(1, 77, 768, dtype=torch.float16)
    lat = torch.zeros(1, 4, 3, 8, 8, dtype=torch.float16)
    pipe = VideoSwapPipeline(None, adapter=T2IAdapter(device="cpu"))
    with pytest.raises(ValueError, match="2 condition images for 3 frames"):
        pipe(pos, lat, guidance_scale=1.0, conditions=_frames(2, (64, 64), "RGB"))
    with pytest.raises(ValueError, match="2 condition images for 3 frames"):
        pipe(pos, None, guidance_scale=1.0, video_length=3, conditions=_frames(2, (64, 64), "RGB"))
    with pytest.raises(ValueError, match="not a TAP dict"):
        pipe(pos, lat, guidance_scale=1.0, conditions={"pred_tracks": torch.zeros(1, 3, 1, 2)})
    with pytest.raises(ValueError, match="multiples of 64"):
        pipe(pos, lat, guidance_scale=1.0, conditions=_frames(3, (64, 72), "RGB"))
    with pytest.raises(ValueError, match="one video"):
        pipe(torch.zeros(2, 77, 768), torch.zeros(2, 4, 3, 8, 8), guidance_scale=1.0, conditions=_frames(3, (64, 64), "RGB"))
    point = VideoSwapPipeline(None, adapter=SparsePointAdapter())
    with pytest.raises(ValueError, match="TAP dict"):
        point(pos, lat, guidance_scale=1.0, conditions=_frames(3, (64, 64), "RGB"))
    with pytest.raises(ValueError, match="no adapter"):
        VideoSwapPipeline(None)(pos, lat, guidance_scale=1.0, conditions=_frames(3, (64, 64), "RGB"))
