"""VAE encode timing: the native AutoencoderKL encoder against the same encode in stock PyTorch eager fp16 on the same GPU.

  python tools/gpu_vae_encode.py [--iters 3] [--rounds 3] [--out FILE]

Workloads: 16 frames at 512x512 and 16 frames at 448x768 (the size most of the reference's shipped configs use); seeded
weights of the SD-1.5 encoder.  Both arms compute the moments (Encoder + quant_conv) of the same fp16 images.  Baseline:
the functions of tests/vae_encoder_oracle.py on CUDA in fp16 (cuDNN convolutions, scaled_dot_product_attention, aten
GroupNorm), i.e. diffusers' encode without diffusers.  Each round times `iters` encodes of each arm with CUDA events
after a warm-up of both, arms alternating; the median round is reported.  Also printed: PSNR between the two arms' moments,
the algorithmic TFLOP/s of the native 3x3-conv launches including the stride-2 down-samplers (FLOPs counted from the
layer shapes here, time from the library's per-category profile in a separate run), GPU name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import ctypes as C  # noqa: E402

import torch  # noqa: E402

import videoswap_b200 as V  # noqa: E402
from tests import vae_encoder_oracle as EO  # noqa: E402
from tests.unet_checks import psnr  # noqa: E402
from videoswap_b200 import _lib  # noqa: E402
from videoswap_b200 import vae as VAE  # noqa: E402

WORKLOADS = [(16, 512, 512), (16, 448, 768)]
PC_CONV = 1


def conv3x3_flops(cfg, n, H, W):
    """Algorithmic FLOPs of the encoder's 3x3 convolutions that run as conv launches: resnet conv1 / conv2, the stride-2
    down-samplers (9 taps per output pixel), conv_out (512 -> 8).  conv_in runs as a K = 64 GEMM and is not counted."""
    boc = list(cfg.block_out_channels)
    conv = lambda co, ci, hh, ww: 2.0 * n * hh * ww * co * ci * 9
    f, prev, h, w = 0.0, boc[0], H, W
    for i, out in enumerate(boc):
        for j in range(cfg.layers_per_block):
            f += conv(out, prev if j == 0 else out, h, w) + conv(out, out, h, w)
        if i < len(boc) - 1:
            h, w = h // 2, w // 2
            f += conv(out, out, h, w)
        prev = out
    c = boc[-1]
    f += 2 * (conv(c, c, h, w) + conv(c, c, h, w))                       # mid-block resnets
    return f + conv(2 * cfg.latent_channels, c, h, w)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    info = gpu_info()
    m = V.AutoencoderKL()
    sd16 = {k: v.to(dev, torch.float16) for k, v in
            VAE.convert_encoder_state_dict(V.seeded_state_dict(V.vae_encoder_param_shapes(m.config), 7), m.config).items()}
    lib = _lib.lib()
    results = []
    for n, H, W in WORKLOADS:
        x = (torch.rand((n, 3, H, W), generator=torch.Generator().manual_seed(1)) * 2 - 1).half().to(dev)
        native = lambda: m.encode(x).latent_dist.parameters
        with torch.no_grad():
            base = lambda: EO.encode(x, sd16)
            native(), base()
            torch.cuda.synchronize()
            rounds = []
            for _ in range(args.rounds):                         # alternating arms
                tn, on = timed(native, args.iters)
                tb, ob = timed(base, args.iters)
                rounds.append((tn, tb))
        tn = sorted(r[0] for r in rounds)[len(rounds) // 2]
        tb = sorted(r[1] for r in rounds)[len(rounds) // 2]
        db = psnr(on, ob)
        lib.vs_profile_reset()
        lib.vs_profile_enable(1)
        m.encode(x)
        torch.cuda.synchronize()
        ms, work, cnt = C.c_double(), C.c_double(), C.c_longlong()
        _lib.check(lib.vs_profile_collect(PC_CONV, C.byref(ms), C.byref(work), C.byref(cnt)))
        lib.vs_profile_enable(0)
        fl = conv3x3_flops(m.config, n, H, W)
        r = {"workload": f"{n} frames, {H}x{W} -> latent {H // 8}x{W // 8}", "native_ms": round(tn, 2),
             "pytorch_eager_fp16_ms": round(tb, 2), "speedup": round(tb / tn, 3),
             "rounds_ms": [[round(a, 2), round(b, 2)] for a, b in rounds], "moments_psnr_db": round(db, 1),
             "conv3x3_tflop": round(fl / 1e12, 2), "conv3x3_launches": cnt.value, "conv3x3_ms": round(ms.value, 2),
             "conv3x3_tflops_per_s": round(fl / (ms.value * 1e-3) / 1e12, 1) if ms.value > 0 else None, "gpu": info}
        print(json.dumps(r), flush=True)
        results.append(r)
        del x, on, ob
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
