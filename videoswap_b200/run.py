"""Run a test config of the reference (options/test_videoswap/**.yml) on the native path, as its `test.py` does:

    python -m videoswap_b200.run -opt options/test_videoswap/animal/2001_catheadturn_T05_Iter100/2001_catheadturn_T05_Iter100.yml

reads the config, seeds, loads the models of `path.pretrained_model_path` (the UNet with its motion module, the point
adapter, the VAE, the text encoder, the tokenizer and the DDIM scheduler), reads the frames and the tracks, runs
`VideoSwapPipeline.validation` on `val.editing_config`, and saves the source and every edited video under
`path.visualization` (default `results/<name>/visualization` in the working directory).  Relative paths in the config are
taken from the working directory, as the reference takes them from its checkout.

Differences from test.py: no `accelerate` (one process, one GPU), fp16 only, no log file and no copy of the config in
the results directory, and `save_type: video` needs `imageio` (with its ffmpeg plugin) to write mp4."""
from __future__ import annotations

import argparse
import copy
import json
import os
import random
import warnings
from typing import Dict, List, Mapping, Optional, Tuple

import torch

from . import formats
from .data import SingleVideoPointDataset, build_transforms

# diffusers 0.19.3 DDIMScheduler arguments: the ones the native scheduler takes, the ones it implements at one value only,
# and the ones that only act together with clip_sample or thresholding (which are off)
_SCHEDULER_ARGS = ("num_train_timesteps", "beta_start", "beta_end", "beta_schedule", "steps_offset", "set_alpha_to_one")
_SCHEDULER_FIXED = {"trained_betas": None, "clip_sample": False, "prediction_type": "epsilon", "thresholding": False,
                    "timestep_spacing": "leading", "rescale_betas_zero_snr": False}
_SCHEDULER_UNUSED = ("clip_sample_range", "dynamic_thresholding_ratio", "sample_max_value")
# diffusers' defaults for the arguments the native scheduler takes, where a config leaves them out
_SCHEDULER_DEFAULTS = {"num_train_timesteps": 1000, "beta_start": 0.0001, "beta_end": 0.02, "beta_schedule": "linear",
                       "steps_offset": 0, "set_alpha_to_one": True}


def load_config(path: str) -> Dict:
    """The YAML file as a plain dict (yaml.safe_load: `!!float 5e-4` is a float, `~` is None)."""
    import yaml
    with open(path) as f:
        return yaml.safe_load(f)


def parse_options(opt: Dict, root_path: Optional[str] = None) -> Dict:
    """Fills in what the reference's set_path_logger adds for a test run: `path.results_root` = <root>/results/<name> and
    `path.visualization` = <results_root>/visualization, unless the config gives them.  root_path defaults to the working
    directory.  Changes opt in place and returns it."""
    root = os.path.abspath(root_path or os.getcwd())
    paths = opt.setdefault("path", {})
    if paths.get("results_root") is None:
        paths["results_root"] = os.path.join(root, "results", opt["name"])
    if paths.get("visualization") is None:
        paths["visualization"] = os.path.join(paths["results_root"], "visualization")
    return opt


def check_options(opt: Mapping) -> None:
    """Everything of a config the native path cannot run, refused before any file is read or model built: a
    mixed_precision other than fp16, a unet type other than AnimateDiffUNet3DModel, an adapter type other than
    SparsePointAdapter, a pipeline other than VideoSwapPipeline, and a video transform other than Resize, CenterCrop,
    ToTensor and Normalize."""
    if opt.get("mixed_precision") != "fp16":
        raise ValueError(f"mixed_precision {opt.get('mixed_precision')!r} is not supported: the native path runs in fp16 "
                         "only (mixed_precision: fp16)")
    unet_type = opt["models"]["unet"].get("type")
    if unet_type != "AnimateDiffUNet3DModel":
        raise NotImplementedError(f"unet type {unet_type!r} is not supported (AnimateDiffUNet3DModel is)")
    adapter_type = opt["models"]["adapter"].get("type")
    if adapter_type != "SparsePointAdapter":
        raise NotImplementedError(f"adapter type {adapter_type!r} is not supported (SparsePointAdapter is)")
    pipeline = opt["val"].get("val_pipeline", "VideoSwapPipeline")
    if pipeline not in ("VideoSwapPipeline", "TuneAVideoPipeline"):
        raise NotImplementedError(f"val_pipeline {pipeline!r} is not supported (VideoSwapPipeline is)")
    if opt["datasets"].get("type", "SingleVideoPointDataset") != "SingleVideoPointDataset":
        raise NotImplementedError(f"dataset type {opt['datasets']['type']!r} is not supported (SingleVideoPointDataset is)")
    build_transforms(opt["datasets"]["video_transform"])


def scheduler_kwargs(config: Mapping) -> Dict:
    """A scheduler_config.json -> the keyword arguments of the native DDIMScheduler, with the overrides of the
    reference's VideoSwapPipeline.__init__ (pipeline_videoswap.py:104-136): steps_offset becomes 1 and clip_sample False.
    An argument of diffusers' DDIMScheduler that the native scheduler does not implement at the config's value raises
    ValueError naming it.  Arguments the config leaves out take diffusers' defaults.  Keys DDIMScheduler does not take
    (another scheduler's, such as PNDM's skip_prk_steps) are ignored with a warning, as diffusers ignores them."""
    config = {**_SCHEDULER_DEFAULTS, **config}
    if config["steps_offset"] != 1:
        warnings.warn(f"scheduler steps_offset {config['steps_offset']} is outdated; using 1, as the reference does")
        config["steps_offset"] = 1
    if config.get("clip_sample", True) is True:
        config["clip_sample"] = False
    kwargs, ignored = {}, []
    for key, value in config.items():
        if key in _SCHEDULER_ARGS:
            kwargs[key] = value
        elif key in _SCHEDULER_FIXED:
            if value != _SCHEDULER_FIXED[key]:
                raise ValueError(f"scheduler config: {key}={value!r} is not implemented by the native DDIM scheduler "
                                 f"(it implements {key}={_SCHEDULER_FIXED[key]!r})")
        elif key not in _SCHEDULER_UNUSED and not key.startswith("_"):
            ignored.append(key)
    if kwargs["beta_schedule"] not in ("linear", "scaled_linear"):
        raise ValueError(f"scheduler config: beta_schedule={kwargs['beta_schedule']!r} is not implemented by the native "
                         "DDIM scheduler (linear and scaled_linear are)")
    if kwargs["set_alpha_to_one"] is not False:
        # diffusers' DDIMInverseScheduler maps it onto set_alpha_to_zero, which ends the inversion at alpha 0
        raise ValueError("scheduler config: set_alpha_to_one=True is not implemented by the native DDIM inverse scheduler "
                         "(it implements set_alpha_to_one=False)")
    if ignored:
        warnings.warn(f"scheduler config keys {ignored} are not DDIMScheduler arguments and are ignored, as diffusers "
                      "ignores them")
    return kwargs


def read_scheduler_config(pretrained_model_path: str) -> Dict:
    """scheduler_kwargs of <pretrained_model_path>/scheduler/scheduler_config.json."""
    with open(os.path.join(pretrained_model_path, "scheduler", "scheduler_config.json")) as f:
        return scheduler_kwargs(json.load(f))


def set_seed(seed: int) -> None:
    """accelerate's set_seed without the CUDA-side call: random, numpy and torch's default generator (which also seeds
    the CUDA generators)."""
    import numpy as np
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)


def load_pipeline(opt: Mapping, sched_kwargs: Mapping, tokenizer=None):
    """test.py:52-89 on the native classes: the models of opt's paths in fp16 on the GPU, in a VideoSwapPipeline with
    the concept config of `new_concept_cfg.json` when the pretrained directory has one.  tokenizer: used instead of
    CLIPTokenizer.from_pretrained(<pretrained_model_path>/tokenizer) when given."""
    import yaml

    from .pipeline import SparsePointAdapter, VideoSwapPipeline
    from .scheduler import DDIMInverseScheduler, DDIMScheduler
    from .text import CLIPTextModel
    from .unet import AnimateDiffUNet3DModel
    from .vae import AutoencoderKL
    path = opt["path"]["pretrained_model_path"]
    unet_opt, adapter_opt = opt["models"]["unet"], opt["models"]["adapter"]

    with open(unet_opt["inference_config_path"]) as f:
        unet_kwargs = yaml.safe_load(f)["unet_additional_kwargs"]
    unet = AnimateDiffUNet3DModel.from_pretrained_2d(path, subfolder="unet", unet_additional_kwargs=unet_kwargs)
    if unet_opt.get("motion_module_path"):
        formats.load_motion_module(unet, unet_opt["motion_module_path"])
    unet = unet.half().cuda()

    with open(adapter_opt["model_config_path"]) as f:
        adapter = SparsePointAdapter(**yaml.safe_load(f))
    adapter = formats.load_adapter(adapter, opt["path"]["pretrained_adapter_path"], dtype=torch.float16).cuda()

    if tokenizer is None:
        from transformers import CLIPTokenizer
        tokenizer = CLIPTokenizer.from_pretrained(path, subfolder="tokenizer")
    pipe = VideoSwapPipeline(unet, DDIMScheduler(**sched_kwargs), adapter=adapter,
                             inverse_scheduler=DDIMInverseScheduler(**sched_kwargs),
                             vae=AutoencoderKL.from_pretrained(path, subfolder="vae"),
                             text_encoder=CLIPTextModel.from_pretrained(path, subfolder="text_encoder"), tokenizer=tokenizer)
    concept_path = os.path.join(path, "new_concept_cfg.json")
    if os.path.exists(concept_path):
        with open(concept_path) as f:
            pipe.set_new_concept_cfg(json.load(f))
    return pipe


def prepare(opt: Mapping, tokenizer=None) -> Tuple[Dict, object, SingleVideoPointDataset]:
    """test.py:24-95: a copy of opt with its paths and seed filled in, the pipeline, and the dataset.  Every refusal
    (check_options, the scheduler config) comes before any model is built."""
    opt = parse_options(copy.deepcopy(dict(opt)))
    check_options(opt)
    sched = read_scheduler_config(opt["path"]["pretrained_model_path"])
    if "video" in opt["val"].get("save_type", "frame_gif").split("_"):
        _imageio()                                  # fail before the models load, not after the edits ran
    if opt.get("manual_seed") is None:
        opt["manual_seed"] = random.randint(1, 10000)
        print(f"manual_seed: {opt['manual_seed']}")
    set_seed(opt["manual_seed"])
    pipe = load_pipeline(opt, sched, tokenizer)
    dataset = SingleVideoPointDataset(opt["datasets"])
    return opt, pipe, dataset


def save_results(opt: Mapping, source_frames: List, results: Mapping) -> str:
    """test.py:112-126: the source video under <visualization>/source, every result under <visualization>/<key> (or
    <visualization> itself when save_type has no 'frame'), suffixed `<key>_<name>` with `use_suffix`.  Returns the
    directory of the last result, as test.py does."""
    vis, val = opt["path"]["visualization"], opt["val"]
    save_type, fps = val.get("save_type", "frame_gif"), val.get("fps", 8)
    save_dir = os.path.join(vis, "source")
    save_video_to_dir(source_frames, save_dir=save_dir, save_suffix="source", save_type=save_type, fps=fps)
    for key, video in results.items():
        save_dir = os.path.join(vis, key) if "frame" in save_type else vis
        suffix = f"{key}_{opt['name']}" if val.get("use_suffix", False) else f"{key}"
        save_video_to_dir(video, save_dir=save_dir, save_suffix=suffix, save_type=save_type, fps=fps)
    return save_dir


def run_config(opt: Mapping, tokenizer=None) -> str:
    """test.py's `test` on the native path: prepare, validation on val.editing_config, save.  opt is not changed.
    Returns the directory of the last saved video."""
    opt, pipe, dataset = prepare(opt, tokenizer)
    source_frames = dataset.get_frames()
    results = pipe.validation(source_frames, dataset.get_conditions(), opt["datasets"]["prompt"],
                              opt["val"]["editing_config"], train_dataset=dataset, save_dir=opt["path"]["visualization"])
    return save_results(opt, source_frames, results)


# --------------------------------------------------------------------------------------------------------- saving
def save_images_as_gif(images: List, save_path: str, fps=5) -> None:
    """vis_util.py:52-64: PIL's GIF writer, every frame int(1000 / fps) ms, looping."""
    images[0].save(save_path, save_all=True, append_images=images[1:], loop=0, duration=int(1000 / fps))


def _imageio():
    try:
        import imageio
    except ImportError as e:
        raise ImportError("save_type 'video' writes mp4 through the imageio package (with imageio-ffmpeg), which is not "
                          "installed; install it or use save_type 'frame', 'gif' or 'frame_gif'") from e
    return imageio


def export_to_video(video_frames: List, output_video_path: str, fps=8) -> str:
    """vis_util.py:91-101: the frames as an mp4 through imageio."""
    import numpy as np
    imageio = _imageio()
    os.makedirs(os.path.dirname(output_video_path), exist_ok=True)
    writer = imageio.get_writer(output_video_path, fps=fps)
    for img in video_frames:
        writer.append_data(np.array(img))
    writer.close()
    return output_video_path


def save_video_to_dir(edit_video: List, save_dir: str, save_suffix: str, save_type: str = "frame", fps=8) -> None:
    """vis_util.py:67-88: save_type is '_'-joined parts: 'frame' writes frames/{idx:05d}_{suffix}.jpg, 'gif'
    {suffix}.gif, 'video' {suffix}.mp4 (needs imageio)."""
    parts = save_type.split("_")
    if "video" in parts:
        _imageio()
    os.makedirs(save_dir, exist_ok=True)
    if "frame" in parts:
        frame_dir = os.path.join(save_dir, "frames")
        os.makedirs(frame_dir, exist_ok=True)
        for idx, img in enumerate(edit_video):
            img.save(os.path.join(frame_dir, f"{idx:05d}_{save_suffix}.jpg"))
    if "gif" in parts:
        save_images_as_gif(edit_video, os.path.join(save_dir, f"{save_suffix}.gif"), fps=fps)
    if "video" in parts:
        export_to_video(edit_video, os.path.join(save_dir, f"{save_suffix}.mp4"), fps=fps)


def main(argv=None) -> str:
    parser = argparse.ArgumentParser(description="Run a VideoSwap test config (options/test_videoswap/**.yml) natively")
    parser.add_argument("-opt", type=str, required=True, help="path to the YAML config")
    args = parser.parse_args(argv)
    save_dir = run_config(load_config(args.opt))
    print(f"saved to {save_dir}")
    return save_dir


if __name__ == "__main__":
    main()
