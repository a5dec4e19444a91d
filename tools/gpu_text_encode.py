"""CLIP text-encoder timing: the native CLIPTextModel against the same encode in stock PyTorch eager fp16 on the same GPU.

  python tools/gpu_text_encode.py [--iters 20] [--rounds 5] [--out FILE]

Workloads: n = 1 and 2 sequences of 77 tokens (one prompt; a prompt and its negative under CFG), 17 (one ED-LoRA prompt,
16 per-layer sequences, plus its negative) and 34; seeded weights of SD-1.5's text encoder.  Baseline: the functions of
tests/clip_oracle.py on CUDA in fp16 with scaled_dot_product_attention(is_causal=True) (cuBLAS GEMMs, aten LayerNorm),
i.e. transformers' CLIPTextModel without transformers; when transformers is importable its own CLIPTextModel in fp16 runs
as a third arm.  Each round times `iters` encodes of each arm with CUDA events after a warm-up of all arms, arms
alternating; the median round is reported, with the PSNR between the native and eager outputs, the native launch count
per encode, and the GPU name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import videoswap_b200 as V  # noqa: E402
from tests import clip_oracle as CO  # noqa: E402
from tests.unet_checks import psnr  # noqa: E402
from videoswap_b200 import _lib  # noqa: E402

WORKLOADS = [1, 2, 17, 34]


def eager_attention(x, sd, name, heads):
    """CLIPAttention with SDPA's causal path (what transformers' sdpa attention runs)."""
    n, L, C = x.shape
    d = C // heads
    q, k, v = (CO.linear(x, sd, f"{name}.{t}_proj").view(n, L, heads, d).transpose(1, 2) for t in "qkv")
    o = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(n, L, C)
    return CO.linear(o, sd, f"{name}.out_proj")


def eager_encode(sd, ids, layers=12, heads=12):
    x = CO.embeddings(sd, ids)
    for i in range(layers):
        p = f"text_model.encoder.layers.{i}"
        x = x + eager_attention(CO.layer_norm(x, sd, f"{p}.layer_norm1"), sd, f"{p}.self_attn", heads)
        h = CO.layer_norm(x, sd, f"{p}.layer_norm2")
        x = x + CO.linear(CO.quick_gelu(CO.linear(h, sd, f"{p}.mlp.fc1")), sd, f"{p}.mlp.fc2")
    return CO.layer_norm(x, sd, "text_model.final_layer_norm")


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def time_arm(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.environ.get("REPORT_JSON"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_text_encode.py needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    model = V.CLIPTextModel()
    sd = model.state_dict()                                     # fp16 device masters
    hf = None
    try:
        import transformers
        cfg = transformers.CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                                          num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu",
                                          attn_implementation="sdpa")
        hf = transformers.CLIPTextModel(cfg).eval()
        hf.load_state_dict({k: v.float().cpu() for k, v in sd.items()})
        hf = hf.half().cuda()
    except ImportError:
        pass
    rows = []
    g = torch.Generator().manual_seed(0)
    for n in WORKLOADS:
        ids = torch.randint(0, 49406, (n, 77), generator=g)
        ids[:, 0], ids[:, -1] = 49406, 49407
        ids_d = ids.cuda()
        arms = {"native": lambda: model(ids_d), "eager": lambda: eager_encode(sd, ids_d)}
        if hf is not None:
            arms["transformers"] = lambda: hf(ids_d)
        with torch.no_grad():
            for f in arms.values():                             # warm-up (module loads, cuBLAS heuristics)
                f(); f()
            torch.cuda.synchronize()
            n0 = _lib.lib().vs_launch_count()
            out = model(ids_d).last_hidden_state
            launches = _lib.lib().vs_launch_count() - n0
            ref = eager_encode(sd, ids_d)
            times = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, f in arms.items():
                    times[k].append(time_arm(f, args.iters))
        r = {"n": n, "launches": launches, "psnr_native_vs_eager": psnr(out, ref)}
        r.update({f"{k}_ms": statistics.median(v) for k, v in times.items()})
        r["eager_over_native"] = r["eager_ms"] / r["native_ms"]
        rows.append(r)
        print(json.dumps(r))
    report = {"gpu": gpu_info(), "iters": args.iters, "rounds": args.rounds, "rows": rows}
    print(f"GPU: {report['gpu']}")
    print(f"{'n':>4} {'native ms':>10} {'eager ms':>9} {'hf ms':>7} {'eager/native':>13} {'PSNR dB':>8} {'launches':>9}")
    for r in rows:
        print(f"{r['n']:>4} {r['native_ms']:>10.3f} {r['eager_ms']:>9.3f} {r.get('transformers_ms', float('nan')):>7.3f} "
              f"{r['eager_over_native']:>13.2f} {r['psnr_native_vs_eager']:>8.1f} {r['launches']:>9}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
