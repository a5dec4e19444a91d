"""`videoswap_b200.run.run_config` end to end on a complete pretrained directory written from the seeded test weights
(tests/run_fixtures.py): the full-size UNet with a motion-module checkpoint, the VAE, the text encoder, a CLIPTokenizer
loaded from its vocabulary files, SD-1.5's scheduler config, the point adapter, an ED-LoRA file and two TAP files.

The config: 16 frames of 320x240 on disk, 4 selected (total_frames 12), Resize 256 + CenterCrop 256, 4 DDIM steps,
`use_blend`, `visualize_point`, two edits -- one with `lora_path`, `tap_path` and `select_point`, one plain -- saved as
`frame_gif`.

GroupNorm sums its statistics with float atomics, so two runs of one flow agree to the last bits only (see
tests/test_validation_gpu.py).  The bar for the edited frames is therefore the run-to-run envelope of two direct
`pipe.validation` calls on the runner's own objects after the same seeding: run_config's frames must agree with both at
least as closely as they agree with each other, minus 3 dB (the envelope capped at 50 dB).  What involves no GPU work
-- the source frames and their files -- must be identical byte for byte between runs."""
import copy
import math
import os

import numpy as np
import pytest
import torch

from tests import run_fixtures as F
from videoswap_b200 import run

pytestmark = pytest.mark.gpu

STEPS, FRAMES, SIZE = 4, 4, 256
SOURCE = "a kitten playing with a ball of yarn"
NAMES = ["head", "tail", "paw", "ear", "nose", "back"]
SEED = 74831


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    root = tmp_path_factory.mktemp("run")
    words = SOURCE.split() + ["small", "puppy", "low", "quality", "blurry"]
    paths = F.write_pretrained(str(root), words=words)
    lora = F.write_edlora(str(root / "edlora_catA.pth"), ["<catA1>", "<catA2>"])
    frames = F.write_frames(str(root / "frames"), 16, 320, 240)
    tap_src = F.write_tap(str(root / "TAP.pth"), 16, SIZE, SIZE, NAMES, seed=402)
    tap_edit = F.write_tap(str(root / "TAP_catA.pth"), 16, SIZE, SIZE, NAMES, seed=403)
    opt = {
        "name": "run_gpu_test", "manual_seed": SEED, "mixed_precision": "fp16",
        "datasets": {"type": "SingleVideoPointDataset", "path": frames, "tap_path": tap_src, "prompt": SOURCE,
                     "num_frames": FRAMES, "total_frames": 12,
                     "video_transform": [{"type": "Resize", "size": SIZE}, {"type": "CenterCrop", "size": SIZE},
                                         {"type": "ToTensor"}, {"type": "Normalize", "mean": [0.5], "std": [0.5]}]},
        "models": {"unet": {"type": "AnimateDiffUNet3DModel", "inference_config_path": paths["inference_config_path"],
                            "motion_module_path": paths["motion_module_path"]},
                   "adapter": {"type": "SparsePointAdapter", "model_config_path": paths["model_config_path"]}},
        "path": {"pretrained_model_path": paths["pretrained_model_path"],
                 "pretrained_adapter_path": paths["pretrained_adapter_path"]},
        "val": {"val_pipeline": "VideoSwapPipeline", "save_type": "frame_gif", "fps": 8, "editing_config": {
            "use_invertion_latents": True, "use_blend": True, "guidance_scale": 7.5, "visualize_point": True,
            "num_inference_steps": STEPS, "negative_prompt": "low quality", "t2i_guidance_scale": 0.5, "t2i_start": 0.0,
            "t2i_end": 0.5,
            "editing_prompts": {
                "kitten_to_catA": {"replace": "kitten -> <catA1> <catA2>", "lora_path": f"{lora}---0.7",
                                   "tap_path": tap_edit, "select_point": ["tail", "head"],
                                   "blend_cfg": {"cross_replace_steps": 0.0, "self_replace_steps": 0.0, "blend_th": 0.3}},
                "kitten_to_puppy": {"replace": "kitten -> small puppy", "lora_path": None, "tap_path": None,
                                    "select_point": None, "guidance_scale": 5.0, "negative_prompt": "blurry"}}}},
    }
    return {"root": root, "opt": opt}


def _with_vis(opt, d):
    opt = copy.deepcopy(opt)
    opt["path"]["visualization"] = str(d)
    return opt


def _recording(monkeypatch, real=run.save_video_to_dir):
    """save_video_to_dir that also keeps a copy of every video it saves, by suffix."""
    saved = {}

    def rec(video, save_dir, save_suffix, save_type="frame", fps=8):
        saved[save_suffix] = [np.asarray(f).copy() for f in video]
        return real(video, save_dir, save_suffix, save_type=save_type, fps=fps)
    monkeypatch.setattr(run, "save_video_to_dir", rec)
    return saved


def _files(d):
    out = {}
    for dirpath, _, names in os.walk(d):
        for n in names:
            with open(os.path.join(dirpath, n), "rb") as f:
                out[os.path.relpath(os.path.join(dirpath, n), d)] = f.read()
    return out


def _psnr(a, b):
    a, b = np.stack(a).astype(np.float64), np.stack(b).astype(np.float64)
    mse = float(((a - b) ** 2).mean())
    return math.inf if mse == 0 else 10 * math.log10(255.0 ** 2 / mse)


def test_run_config_writes_test_py_files_and_equals_validation(setup, monkeypatch):
    s = setup
    keys = ["kitten_to_catA", "kitten_to_catA_vispoint", "kitten_to_puppy", "kitten_to_puppy_vispoint"]
    runs = []
    for i in range(2):
        saved = _recording(monkeypatch)
        vis = s["root"] / f"vis{i}"
        last = run.run_config(_with_vis(s["opt"], vis))
        torch.cuda.synchronize()
        runs.append((saved, _files(vis)))
        # the files test.py writes for save_type frame_gif, and nothing else
        want = {os.path.join("source", "source.gif")} | {os.path.join("source", "frames", f"{f:05d}_source.jpg")
                                                         for f in range(FRAMES)}
        for k in keys:
            want |= {os.path.join(k, f"{k}.gif")} | {os.path.join(k, "frames", f"{f:05d}_{k}.jpg") for f in range(FRAMES)}
        assert set(runs[-1][1]) == want
        assert last == str(vis / keys[-1])
        assert sorted(saved) == sorted(["source"] + keys)
        assert all(len(saved[k]) == FRAMES and saved[k][0].shape == (SIZE, SIZE, 3) for k in saved)

    # no GPU work in the source video: the same bytes every run
    for name, blob in runs[0][1].items():
        if name.startswith("source"):
            assert runs[1][1][name] == blob, name

    # the same flow on the runner's own objects: prepare() seeds, then validation, as run_config does
    opt, pipe, ds = run.prepare(_with_vis(s["opt"], s["root"] / "unused"))
    direct = []
    for _ in range(2):
        run.set_seed(opt["manual_seed"])
        frames = ds.get_frames()
        assert all(np.array_equal(np.asarray(f), g) for f, g in zip(frames, runs[0][0]["source"]))
        res = pipe.validation(frames, ds.get_conditions(), SOURCE, opt["val"]["editing_config"], train_dataset=ds)
        torch.cuda.synchronize()
        direct.append({k: [np.asarray(f) for f in v] for k, v in res.items()})
    assert sorted(direct[0]) == keys
    for k in keys:
        env = min(_psnr(direct[0][k], direct[1][k]), 50.0)
        got = min(_psnr(runs[0][0][k], direct[0][k]), _psnr(runs[0][0][k], direct[1][k]),
                  _psnr(runs[1][0][k], direct[0][k]), _psnr(runs[1][0][k], direct[1][k]))
        again = _psnr(runs[0][0][k], runs[1][0][k])
        print(f"\n{k}: run_config vs validation {got:.1f} dB, run_config twice {again:.1f} dB, validation twice "
              f"{_psnr(direct[0][k], direct[1][k]):.1f} dB; JPEG bytes equal between runs: "
              f"{all(runs[0][1][n] == runs[1][1][n] for n in runs[0][1] if n.startswith(k + os.sep))}")
        assert got >= env - 3.0, k
        assert again >= env - 3.0, k
    # the edits reach the output: the two differ from each other and from the source
    assert _psnr(runs[0][0]["kitten_to_catA"], runs[0][0]["kitten_to_puppy"]) < 30.0
    assert _psnr(runs[0][0]["kitten_to_puppy"], runs[0][0]["source"]) < 30.0
