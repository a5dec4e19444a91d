"""Times `python -m videoswap_b200.run` at the shipped size: a pretrained directory written from the seeded test weights
(tests/run_fixtures.py) in a temporary directory, 64 PNG frames of 1280x720 of which 16 are selected and resized to
448x768, 50 DDIM steps, `use_blend`, `visualize_point`, two edits (one with an ED-LoRA file, a TAP file and select_point,
one plain), saved as `frame_gif`.

Runs run_config's steps one after another in one process, the host clock around synchronised work: loading (config,
scheduler, models from disk, frames, tracks: `run.prepare`), the inversion with the attention store, the edits (the rest
of `validation`: controllers, ED-LoRA merge and restore, the CFG loops, the decodes) and saving (`run.save_results`).
Run 1 is what a user's fresh process pays (first launches, weight packing); later runs load the models again from the
same files.  Prints one JSON line (also written to --out).

    python tools/gpu_run_config.py [--steps 50] [--runs 2] [--out f.json]"""
import argparse
import gc
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SOURCE = "a silver jeep driving down a curvy road in the countryside"
NAMES = [f"p{i}" for i in range(12)]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"gpu": f"unknown ({e})"}


def make_config(tmp, steps):
    from tests import run_fixtures as F
    words = SOURCE.split() + ["yellow", "porsche", "car", "lowres", "worst", "quality"]
    paths = F.write_pretrained(tmp, words=words)
    lora = F.write_edlora(os.path.join(tmp, "edlora_car.pth"), ["<carA1>", "<carA2>"])
    frames = F.write_frames(os.path.join(tmp, "frames"), 64, 1280, 720)
    tap_src = F.write_tap(os.path.join(tmp, "TAP.pth"), 64, 768, 448, NAMES, seed=402)
    tap_edit = F.write_tap(os.path.join(tmp, "TAP_car.pth"), 64, 768, 448, NAMES, seed=403)
    return {
        "name": "gpu_run_config", "manual_seed": 74831, "mixed_precision": "fp16",
        "datasets": {"type": "SingleVideoPointDataset", "path": frames, "tap_path": tap_src, "prompt": SOURCE,
                     "num_frames": 16, "total_frames": 64,
                     "video_transform": [{"type": "Resize", "size": [448, 768]}, {"type": "ToTensor"},
                                         {"type": "Normalize", "mean": [0.5], "std": [0.5]}]},
        "models": {"unet": {"type": "AnimateDiffUNet3DModel", "inference_config_path": paths["inference_config_path"],
                            "motion_module_path": paths["motion_module_path"]},
                   "adapter": {"type": "SparsePointAdapter", "model_config_path": paths["model_config_path"]}},
        "path": {"pretrained_model_path": paths["pretrained_model_path"],
                 "pretrained_adapter_path": paths["pretrained_adapter_path"]},
        "val": {"val_pipeline": "VideoSwapPipeline", "save_type": "frame_gif", "fps": 8, "editing_config": {
            "use_invertion_latents": True, "use_blend": True, "guidance_scale": 7.5, "visualize_point": True,
            "num_inference_steps": steps, "negative_prompt": "lowres, worst quality", "t2i_guidance_scale": 0.5,
            "t2i_start": 0.0, "t2i_end": 0.5,
            "editing_prompts": {
                "jeep_to_carA": {"replace": "silver jeep -> <carA1> <carA2>", "lora_path": f"{lora}---0.7",
                                 "tap_path": tap_edit, "select_point": ["p1", "p3", "p5"],
                                 "blend_cfg": {"cross_replace_steps": 0.0, "self_replace_steps": 0.0, "blend_th": 0.3}},
                "jeep_to_porsche": {"replace": "silver jeep -> yellow porsche car", "tap_path": None,
                                    "select_point": None}}}},
    }


def one_run(opt, vis):
    import torch

    from videoswap_b200 import run
    opt = dict(opt, path=dict(opt["path"], visualization=vis))
    spans = {}

    def sync_time():
        torch.cuda.synchronize()
        return time.perf_counter()

    t0 = sync_time()
    opt, pipe, ds = run.prepare(opt)
    frames = ds.get_frames()
    cond = ds.get_conditions()
    t1 = sync_time()
    invert = pipe.invert

    def timed_invert(*a, **k):
        s = sync_time()
        r = invert(*a, **k)
        spans["invert"] = sync_time() - s
        return r
    pipe.invert = timed_invert
    res = pipe.validation(frames, cond, opt["datasets"]["prompt"], opt["val"]["editing_config"], train_dataset=ds,
                          save_dir=vis)
    t2 = sync_time()
    run.save_results(opt, frames, res)
    t3 = sync_time()
    del pipe
    gc.collect()
    torch.cuda.empty_cache()
    return {"total_s": round(t3 - t0, 3), "load_s": round(t1 - t0, 3), "invert_s": round(spans["invert"], 3),
            "edits_s": round(t2 - t1 - spans["invert"], 3), "save_s": round(t3 - t2, 3), "outputs": sorted(res)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        opt = make_config(tmp, args.steps)
        write_s = time.perf_counter() - t0
        runs = [one_run(opt, os.path.join(tmp, f"vis{i}")) for i in range(args.runs)]
    out = {"what": "videoswap_b200.run: run_config's steps, seeded weights from disk", "frames": 16, "size": [448, 768],
           "steps": args.steps, "edits": 2, "fixture_write_s": round(write_s, 1), "runs": runs,
           "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), **gpu_info()}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
