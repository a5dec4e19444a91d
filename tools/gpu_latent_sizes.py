"""Step time at latent sizes that are not multiples of 8 against the next multiple-of-8 size (bench.py's residuals are
floor-sized, so it only runs multiples of 8).  The CUDA-graph CFG step of the benchmark (16 frames, ED-LoRA embeddings,
adapter residuals, here on the ceil chain of level sizes) is timed at 45x60 against 48x64 and at 90x160 against 96x160,
the two shapes of a pair alternating `--reps` times; plus one eager pass per shape with the per-category kernel profile.

    python tools/gpu_latent_sizes.py --steps 10 --warmup 3 --out latent_sizes.json
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import CATS, ClockSampler, gpu_weights  # noqa: E402
from videoswap_b200 import AnimateDiffUNet3DModel, DDIMScheduler, VideoSwapPipeline, _lib  # noqa: E402
from videoswap_b200.pipeline import GraphedStep  # noqa: E402

PAIRS = [((45, 60), (48, 64)), ((90, 160), (96, 160))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    Fr, K, W = args.frames, args.steps, max(args.warmup, 1)
    model = AnimateDiffUNet3DModel(init="empty")
    model.load_state_dict(gpu_weights(model.cfg, dev), assign=True)
    pipe = VideoSwapPipeline(model, DDIMScheduler())
    pipe.scheduler.set_timesteps(50)
    ts = pipe.scheduler.timesteps
    shapes = [s for pair in PAIRS for s in pair]
    model(torch.zeros(1, 4, 1, 8, 8, dtype=torch.float16, device=dev), 1, torch.zeros(1, 77, 768, dtype=torch.float16, device=dev))
    # one arena for every shape: the graphs pin it, so it is sized for the largest shape before the first capture
    big = max(shapes, key=lambda s: s[0] * s[1])
    _lib.call("vs_unet_reserve_workspace", model._handle, 2, Fr, big[0], big[1])
    g = torch.Generator(device=dev).manual_seed(100)
    embeds = torch.randn((2, 16, 77, 768), device=dev, generator=g).half()
    lib = _lib.lib()
    result = {"gpu": torch.cuda.get_device_name(dev), "frames": Fr, "steps": K, "warmup": W, "reps": args.reps, "shapes": {}}
    graphs, inputs = {}, {}
    for (h, w) in shapes:
        lat0 = torch.randn((1, 4, Fr, h, w), device=dev, generator=g).half()
        res = [(0.1 * torch.randn((2 * Fr, c, lh, lw), device=dev, generator=g)).half()
               for c, (lh, lw) in zip(model.cfg.block_out_channels, model.level_sizes(h, w))]
        inputs[(h, w)] = (lat0, res)
        # eager pass with the per-launch profile (per category: ms / step, launches / step)
        lat = lat0
        for i in range(W):
            lat = pipe.step(lat, ts[i % len(ts)], embeds, 7.5, list(res))
        torch.cuda.synchronize()
        lib.vs_profile_reset()
        lib.vs_profile_enable(1)
        for i in range(K):
            lat = pipe.step(lat, ts[(W + i) % len(ts)], embeds, 7.5, list(res))
        torch.cuda.synchronize()
        lib.vs_profile_enable(0)
        prof = {}
        for ci, name in enumerate(CATS):
            a, b, c = C.c_double(), C.c_double(), C.c_longlong()
            _lib.call("vs_profile_collect", ci, C.byref(a), C.byref(b), C.byref(c))
            prof[name] = {"ms_per_step": a.value / K, "launches_per_step": c.value / K}
        lib.vs_profile_reset()
        result["shapes"][f"{h}x{w}"] = {"profile": prof, "graph_ms": [], "finite": bool(torch.isfinite(lat).all().item())}
        graphs[(h, w)] = GraphedStep(pipe, lat0, embeds, 7.5, res)
    sampler = ClockSampler(0)
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.reps):
        for pair in PAIRS:
            for s in pair:
                gs, lat = graphs[s], inputs[s][0]
                for i in range(W):
                    lat = gs(lat, ts[i % len(ts)])
                torch.cuda.synchronize()
                e0.record()
                for i in range(K):
                    lat = gs(lat, ts[(W + i) % len(ts)])
                e1.record()
                torch.cuda.synchronize()
                r = result["shapes"][f"{s[0]}x{s[1]}"]
                r["graph_ms"].append(e0.elapsed_time(e1) / K)
                r["finite"] = r["finite"] and bool(torch.isfinite(lat).all().item())
    result["clock"] = sampler.stop()
    for r in result["shapes"].values():
        ms = sorted(r["graph_ms"])
        r["median_ms_per_step"] = ms[len(ms) // 2]
    result["odd_not_slower"] = {f"{a[0]}x{a[1]} <= {b[0]}x{b[1]}":
                                result["shapes"][f"{a[0]}x{a[1]}"]["median_ms_per_step"] <= result["shapes"][f"{b[0]}x{b[1]}"]["median_ms_per_step"]
                                for a, b in PAIRS}
    del graphs
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
