"""Times the T2IAdapter call: the native adapter against the same FullAdapter in stock PyTorch eager fp16 (the
functions of tests/t2i_adapter_oracle.py on CUDA, cuDNN convs), 16 frames of 448x768, seeded weights.

usage: gpu_t2i_adapter.py [--iters N] [--rounds R] [--out f.json]

  * native_device: T2IAdapter.forward from the uint8 frames already on the GPU (t2i_image_in, convs, pools);
  * native_call: T2IAdapter.forward from the list of PIL images (host preprocessing, upload, device work);
  * eager_fp16: the restatement in fp16 from the fp16 NCHW frames already on the GPU.
Arms alternate over --rounds rounds of --iters calls each, each round ending in a device synchronise (host clock);
the median round is reported in ms per call.  PSNR of the native features against the eager ones, per level.
The GPU name and its power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--out", default=None)
args = ap.parse_args()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

from tests import t2i_adapter_oracle as TO  # noqa: E402
from tests.unet_checks import psnr  # noqa: E402
from videoswap_b200 import T2IAdapter, t2i_adapter_param_shapes  # noqa: E402
from videoswap_b200.weights import seeded_state_dict  # noqa: E402

if not torch.cuda.is_available():
    sys.exit("gpu_t2i_adapter.py needs a GPU")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = (s.strip() for s in q.split(","))
        return {"gpu": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})"}


def main():
    F_, W, H = 16, 768, 448
    ad = T2IAdapter(init="empty")
    sd = seeded_state_dict(t2i_adapter_param_shapes(ad.config), seed=11)
    ad.load_state_dict(sd)
    sd16 = {k: v.half().cuda() for k, v in sd.items()}
    rng = np.random.default_rng(0)
    frames = [Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8), "RGB") for _ in range(F_)]
    u8 = ad.preprocess(frames).cuda()
    x16 = (u8.permute(0, 3, 1, 2).float() / 255).half().contiguous()

    arms = {"native_device": lambda: ad(u8), "native_call": lambda: ad(frames),
            "eager_fp16": lambda: TO.full_adapter(sd16, x16, dtype=torch.float16)}
    with torch.no_grad():
        for fn in arms.values():
            for _ in range(2):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                t0 = time.perf_counter()
                for _ in range(args.iters):
                    fn()
                torch.cuda.synchronize()
                times[k].append((time.perf_counter() - t0) * 1e3 / args.iters)
        nat, ref = ad(u8), TO.full_adapter(sd16, x16, dtype=torch.float16)
        torch.cuda.synchronize()
    rep = {"frames": F_, "size": f"{H}x{W}", **gpu_info(),
           "ms": {k: statistics.median(v) for k, v in times.items()}, "ms_rounds": times,
           "psnr_native_vs_eager_per_level": [psnr(n.permute(0, 3, 1, 2), r) for n, r in zip(nat, ref)],
           "peak_mem_gb": torch.cuda.max_memory_allocated() / 1e9}
    print(json.dumps(rep, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
