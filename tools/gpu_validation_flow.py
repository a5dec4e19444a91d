"""Times one `VideoSwapPipeline.validation` with `use_blend` at the shipped size: 16 frames of 448x768, seeded full-size
UNet, VAE, text encoder and adapter, the chunk tokenizer of oracle/, DDIM inversion with the attention store, then each edit
(controller built from the prompts, refine + self-attention and latent blending, CFG) with its decode.  The phases are
timed with the host clock around synchronised work (torch.cuda.synchronize before and after each), by wrapping the
pipeline's `invert`, `__call__` and `decode_latents`.  Prints one JSON line (also written to --out).

    python tools/gpu_validation_flow.py [--steps 50] [--edits 2] [--out f.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, FRAMES = 448, 768, 16
SOURCE = "a silver jeep driving down a curvy road in the countryside"
EDITS = {"jeep_to_porsche": {"replace": "silver jeep -> yellow Porsche car",
                             "blend_cfg": {"cross_replace_steps": 0.5, "self_replace_steps": 0.5, "blend_th": 0.3}},
         "jeep_to_truck": {"replace": "silver jeep -> red pickup truck", "replace_other": "countryside -> desert",
                           "blend_cfg": {"cross_replace_steps": 0.2, "self_replace_steps": 0.3, "blend_th": 0.2}}}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"gpu": f"unknown ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--edits", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from PIL import Image

    import videoswap_b200 as V
    from oracle.chunk_tokenizer import ChunkTokenizer
    from tests import unet_checks as U

    phases = []

    def timed(name, fn, *a, **k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn(*a, **k)
        torch.cuda.synchronize()
        phases.append((name, time.perf_counter() - t0))
        return r

    class TimedPipeline(V.VideoSwapPipeline):
        def invert(self, *a, **k):
            return timed("invert", super().invert, *a, **k)

        def __call__(self, *a, **k):
            return timed("edit", super().__call__, *a, **k)

        def decode_latents(self, *a, **k):
            return timed("decode", super().decode_latents, *a, **k)

    unet, _ = U.get_model()
    te = V.CLIPTextModel()
    pipe = TimedPipeline(unet, V.DDIMScheduler(), adapter=V.SparsePointAdapter().half().cuda(),
                         inverse_scheduler=V.DDIMInverseScheduler(), vae=V.AutoencoderKL(), text_encoder=te,
                         tokenizer=ChunkTokenizer(base_vocab=te.get_input_embeddings().weight.shape[0]))
    g = torch.Generator().manual_seed(7)
    base = torch.rand((H // 16, W // 16, 3), generator=g)
    frames = []
    for f in range(FRAMES):             # a smooth, slowly moving pattern (the VAE sees image-like input, not noise)
        img = torch.roll(base, shifts=f, dims=1).permute(2, 0, 1)[None]
        img = torch.nn.functional.interpolate(img, size=(H, W), mode="bilinear", align_corners=False)[0]
        frames.append(Image.fromarray((img.permute(1, 2, 0) * 255).round().byte().numpy(), "RGB"))
    P = 12
    cond = {"pred_tracks": torch.rand((FRAMES, P, 2), generator=g) * torch.tensor([W, H]),
            "point_embedding": torch.randn((P, 1280), generator=g), "point_name2id": {f"p{i}": i for i in range(P)},
            "img_size": (W, H), "index_list": None}
    config = {"use_invertion_latents": True, "use_blend": True, "guidance_scale": 7.5, "num_inference_steps": args.steps,
              "negative_prompt": "lowres, worst quality", "t2i_guidance_scale": 0.5, "t2i_start": 0.0, "t2i_end": 0.3,
              "editing_prompts": dict(list(EDITS.items())[:args.edits])}

    # warm-up at 2 steps (weight packing, workspace, first launches), then the timed run
    pipe.validation(frames, cond, SOURCE, dict(config, num_inference_steps=2, editing_prompts=dict(list(EDITS.items())[:1])))
    phases.clear()
    torch.manual_seed(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = pipe.validation(frames, cond, SOURCE, config)
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    edits = [s for n, s in phases if n == "edit"]
    decodes = [s for n, s in phases if n == "decode"]
    out = {"what": "VideoSwapPipeline.validation, use_blend, seeded weights", "frames": FRAMES, "size": [H, W],
           "steps": args.steps, "edits": len(edits), "total_s": round(total, 3),
           "invert_s": round(sum(s for n, s in phases if n == "invert"), 3),
           "edit_s": [round(s, 3) for s in edits], "decode_s_within_edit": [round(s, 3) for s in decodes],
           "edit_ms_per_step_excluding_decode": [round(1000 * (e - d) / args.steps, 1) for e, d in zip(edits, decodes)],
           "outputs": sorted(res), "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), **gpu_info()}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
