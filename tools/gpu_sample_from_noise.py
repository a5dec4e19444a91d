"""Times sampling from noise: the fused CFG + rescale + stochastic-DDIM step and one 50-step call from noise.

usage: gpu_sample_from_noise.py [--launches N] [--steps K] [--json PATH]

  * The step kernel (ops.cfg_ddim_rescale_step, fp16, CFG 7.5, eta 1, guidance_rescale 0.7) with CUDA events over
    --launches back-to-back launches, against the same formula in eager PyTorch (guidance lerp, per-sample std,
    rescale, DDIM update with noise), at [S, 4, 16, 64, 64] for S = 1, 2 and at [1, 4, 16, 56, 96].  GB/s counts the
    bytes the step must move once (uncond + cond predictions, latents, noise read; latents written) over kernel time,
    and is set against the 3.35 TB/s of the H100 SXM data sheet.
  * VideoSwapPipeline.__call__ from noise (16 frames of 512 x 512, CFG, eta 1, guidance_rescale 0.7, seeded weights of
    the real architecture) over --steps steps, eager, and the same loop under GraphedStep(eta=, guidance_rescale=).
The GPU name and its power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("--launches", type=int, default=500)
ap.add_argument("--steps", type=int, default=50)
ap.add_argument("--json", default=None)
args = ap.parse_args()
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from videoswap_b200 import ops  # noqa: E402
from videoswap_b200.scheduler import DDIMScheduler  # noqa: E402

if not torch.cuda.is_available():
    sys.exit("gpu_sample_from_noise.py needs a GPU")
HBM = 3.35e12


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = (s.strip() for s in q.split(","))
        return {"gpu": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})"}


def timed(fn, n):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / n   # us


def eager_step(eps, x, z, g, c_x, c_e, c_n, r):
    eu, ec = eps.chunk(2)
    e = eu + g * (ec - eu)
    dims = list(range(1, e.ndim))
    e = r * (e * (ec.std(dim=dims, keepdim=True) / e.std(dim=dims, keepdim=True))) + (1 - r) * e
    return c_x * x + c_e * e + c_n * z


def kernel_rows():
    sch = DDIMScheduler()
    sch.set_timesteps(50)
    a_t, a_p = sch.alphas(501)
    c_x, c_e, c_n = ops.ddim_coefficients(a_t, a_p, 1.0)
    rows = []
    for shape in ((1, 4, 16, 64, 64), (2, 4, 16, 64, 64), (1, 4, 16, 56, 96)):
        x = torch.randn(shape, device="cuda").half()
        z = torch.randn(shape, device="cuda").half()
        eps = torch.randn((2 * shape[0],) + shape[1:], device="cuda").half()
        out = torch.empty_like(x)
        us = timed(lambda: ops.cfg_ddim_rescale_step(eps, x, 7.5, a_t, a_p, eta=1.0, guidance_rescale=0.7, noise=z,
                                                     out=out), args.launches)
        us_eager = timed(lambda: eager_step(eps, x, z, 7.5, c_x, c_e, c_n, 0.7), max(20, args.launches // 5))
        ref = eager_step(eps.double(), x.double(), z.double(), 7.5, c_x, c_e, c_n, 0.7)
        nbytes = 5 * x.numel() * 2
        rows.append({"shape": list(shape), "kernel_us": round(us, 2), "eager_torch_us": round(us_eager, 2),
                     "kernel_GBps": round(nbytes / us * 1e-3, 1), "share_of_3.35TBps": round(nbytes / us * 1e6 / HBM, 3),
                     "max_abs_err_vs_fp64": float((out.double() - ref).abs().max())})
        print(json.dumps(rows[-1]), flush=True)
    return rows


def call_rows():
    from videoswap_b200 import AnimateDiffUNet3DModel, VideoSwapPipeline, seeded_state_dict, unet_param_shapes
    from videoswap_b200.pipeline import GraphedStep
    model = AnimateDiffUNet3DModel(init="empty")
    model.load_state_dict(seeded_state_dict(unet_param_shapes(model.cfg), seed=0))
    model = model.half().cuda()
    pipe = VideoSwapPipeline(model, DDIMScheduler())
    g = torch.Generator().manual_seed(0)
    pos, neg = (torch.randn((1, 16, 77, 768), generator=g).half().cuda() for _ in range(2))
    kw = dict(video_length=16, height=512, width=512, eta=1.0, guidance_rescale=0.7, max_iters=args.steps)
    pipe(pos, None, negative_prompt_embeds=neg, generator=torch.Generator().manual_seed(1), **dict(kw, max_iters=2))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eager = pipe(pos, None, negative_prompt_embeds=neg, generator=torch.Generator().manual_seed(1), **kw).videos
    torch.cuda.synchronize()
    t_eager = time.perf_counter() - t0

    pipe.scheduler.set_timesteps(50)
    gen = torch.Generator().manual_seed(1)
    lat = pipe.prepare_latents(1, 16, 512, 512, torch.float16, "cuda", gen)
    emb = torch.cat([neg, pos])
    gs = GraphedStep(pipe, lat, emb, 7.5, eta=1.0, guidance_rescale=0.7)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    x = lat
    for t in pipe.scheduler.timesteps[:args.steps]:
        x = gs(x, t, generator=gen)
    torch.cuda.synchronize()
    t_graph = time.perf_counter() - t0
    graphed = x.permute(0, 2, 1, 3, 4).reshape(eager.shape)
    mse = float(((graphed.float() - eager.float()) ** 2).mean())
    rng = float(eager.float().max() - eager.float().min())
    import math
    row = {"call": "16 frames 512x512, CFG 7.5, eta 1, guidance_rescale 0.7", "steps": args.steps,
           "eager_s": round(t_eager, 3), "graphed_s": round(t_graph, 3),
           "graphed_vs_eager_psnr_db": (float("inf") if mse == 0 else round(10 * math.log10(rng * rng / mse), 1))}
    print(json.dumps(row), flush=True)
    return [row]


info = gpu_info()
print(json.dumps(info), flush=True)
report = {"info": info, "kernel": kernel_rows(), "call": call_rows(), "info_after": gpu_info()}
if args.json:
    os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
    with open(args.json, "w") as f:
        json.dump(report, f, indent=1)
