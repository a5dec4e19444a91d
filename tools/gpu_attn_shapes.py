"""Times the spatial attention launches of one UNet step (16 frames 512x512, CFG: 32 images, 8 heads) with CUDA events.

usage: gpu_attn_shapes.py [seconds per shape, default 1.0]

Each shape is warmed up, then timed as three windows of back-to-back launches (about a third of the time budget each);
the median window gives ms per launch and algorithmic TFLOP/s (4 B h Nq Nk d).  The GPU name, its power limit and the SM
clock sampled right after the timed windows are printed with the numbers, since the rate depends on them.
"""
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from videoswap_b200 import ops  # noqa: E402

HEADS, IMGS, FRAMES = 8, 32, 16
# (name, d, Nq, Nk, kv_div): level 0 (64x64 latent, C = 320) and level 1 (32x32, C = 640); cross-attention keys are the 77
# text tokens, shared by the 16 frames of each CFG half
SHAPES = [
    ("self_d40_n4096", 40, 4096, 4096, 1),
    ("self_d80_n1024", 80, 1024, 1024, 1),
    ("cross_d40_n4096_nk77", 40, 4096, 77, FRAMES),
    ("cross_d80_n1024_nk77", 80, 1024, 77, FRAMES),
]


def _smi(fields):
    dev = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
    try:
        r = subprocess.run(["nvidia-smi", "-i", dev, f"--query-gpu={fields}", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True)
    except OSError:
        return []
    return [f.strip() for f in r.stdout.strip().split(",")] if r.returncode == 0 else []


def _inputs(d, nq, nk, kv_div, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = HEADS * d
    if kv_div == 1:
        qkv = torch.randn(IMGS, nq, 3 * C, device="cuda", generator=g).half()
        return qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    q = torch.randn(IMGS, nq, C, device="cuda", generator=g).half()
    kv = torch.randn(IMGS // kv_div, nk, 2 * C, device="cuda", generator=g).half()
    return q, kv[..., :C], kv[..., C:]


def _time(fn, seconds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        fn()
    e1.record()
    e1.synchronize()
    reps = max(10, math.ceil(seconds / 3 * 1e3 / (e0.elapsed_time(e1) / 3)))
    windows = []
    for _ in range(3):
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        e1.synchronize()
        windows.append(e0.elapsed_time(e1) / reps)
    return sorted(windows)[1], windows, reps


def main():
    assert torch.cuda.is_available(), "gpu_attn_shapes.py needs a GPU"
    seconds = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    card = _smi("name,power.limit")
    print(f"gpu: {card[0] if card else torch.cuda.get_device_name()}, power limit: {card[1] + ' W' if len(card) > 1 else 'unknown'}")
    rows = []
    for i, (name, d, nq, nk, kv_div) in enumerate(SHAPES):
        q, k, v = _inputs(d, nq, nk, kv_div, 1000 + i)
        ms, windows, reps = _time(lambda: ops.attention(q, k, v, HEADS, kv_div=kv_div), seconds)
        clk = _smi("clocks.sm")
        tflops = 4.0 * IMGS * HEADS * nq * nk * d / (ms * 1e-3) / 1e12
        rows.append(dict(shape=name, d=d, nq=nq, nk=nk, kv_div=kv_div, ms=ms, tflops=tflops, windows_ms=windows,
                         launches_per_window=reps, sm_clock_mhz=clk[0] if clk else None))
        print(f"{name:24s} {ms:8.3f} ms  {tflops:7.1f} TFLOP/s  (windows {', '.join(f'{w:.3f}' for w in windows)} ms; "
              f"{reps} launches each; SM clock after: {clk[0] if clk else '?'} MHz)")
    if os.environ.get("REPORT_JSON"):
        with open(os.environ["REPORT_JSON"], "w") as f:
            json.dump(dict(gpu=card[0] if card else None, power_limit_w=card[1] if len(card) > 1 else None, shapes=rows), f,
                      indent=1)


if __name__ == "__main__":
    main()
