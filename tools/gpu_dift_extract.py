"""DIFT semantic-point timing: the native featurizer and read-out against the same computation in stock PyTorch eager fp16
on the same GPU.

  python tools/gpu_dift_extract.py [--iters 2] [--rounds 3] [--frames 16] [--out FILE]

Workloads: frames of 448x768 (the size most of the reference's shipped configs use) and 512x512; seeded weights of the
SD-1.5 VAE encoder and UNet (no motion modules), t = 261, up_ft_index 1, ensemble E = 8.
  * featurize: one frame -> the ensemble-mean up_ft[1] map.  Native: SDFeaturizer.features + dift_ensemble_mean (VAE
    encode once, dift_noise, vs_unet_forward_features on B = 8).  Eager: tests/vae_encoder_oracle.encode, the noising in
    torch and tests/dift_oracle.up_ft (oracle/unet3d_oracle.py, stopped after up_blocks[1]) on CUDA in fp16 with B = 8,
    then the mean -- the reference's per-frame work without diffusers (the reference also encodes the frame 8 times).
  * clip: extract_point_embedding (human branch, 12 points) over `frames` frames, 8 frames per UNet call.  Eager: the
    per-frame featurize above, then nn.Upsample of the map to the frame size and the reads, as the reference does.
Arms alternate; each round times `iters` runs of each after a warm-up of both; the median round is reported, with the
GPU name and power limit read in the same run.  The prompt embedding is computed once outside the timed region."""
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
from oracle import unet3d_oracle as O  # noqa: E402
from tests import dift_oracle as D  # noqa: E402
from tests import vae_encoder_oracle as EO  # noqa: E402
from videoswap_b200 import vae as VAE  # noqa: E402

SIZES = [(448, 768), (512, 512)]
E = 8


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
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from PIL import Image
    dev = torch.device("cuda:0")
    info = gpu_info()
    unet = V.AnimateDiffUNet3DModel(init="empty", use_motion_module=False)
    sd = V.seeded_state_dict(V.unet_param_shapes(unet.cfg), seed=0)
    unet.load_state_dict(sd)
    unet = unet.half().cuda()
    usd16 = {k: v.to(dev, torch.float16) for k, v in sd.items()}
    vae = V.AutoencoderKL()
    esd16 = {k: v.to(dev, torch.float16) for k, v in
             VAE.convert_encoder_state_dict(V.seeded_state_dict(V.vae_encoder_param_shapes(vae.config), 7), vae.config).items()}
    fz = V.SDFeaturizer(unet, vae, None, None)
    ehs = torch.randn((1, 77, 768), generator=torch.Generator().manual_seed(3)).half().cuda()
    fz.encode_prompt = lambda prompt: ehs
    a = fz.scheduler.alphas_cumprod[261]
    sa, sb = float(a ** 0.5), float((1 - a) ** 0.5)
    sf = vae.config.scaling_factor
    ocfg = O.OracleConfig(use_motion_module=False)
    results = []
    for H, W in SIZES:
        g = torch.Generator().manual_seed(1)
        u8 = (torch.rand((args.frames, H, W, 3), generator=g) * 255).to(torch.uint8)
        frames = [Image.fromarray(f.numpy()) for f in u8]
        tracks = torch.rand((args.frames, 12, 2), generator=g) * torch.tensor([W - 1.0, H - 1.0])
        x1 = u8[:1].to(dev)

        def native_frame():
            return V.ops.dift_ensemble_mean(fz.features(x1, "p", ensemble_size=E))

        def eager_frame(img_u8):
            with torch.no_grad():
                x = (img_u8.permute(0, 3, 1, 2).half() / 255 - 0.5) * 2
                mom = EO.encode(x, esd16)
                e1 = torch.randn((E, 4) + mom.shape[2:], device=dev, dtype=torch.float16)
                e2 = torch.randn_like(e1)
                lat = D.noisy_latents(mom, e1, e2, sf, sa, sb).half()
                f = D.up_ft(usd16, ocfg, lat, 261, ehs.expand(E, -1, -1), 1)
                return f.float().mean(0, keepdim=True)

        def native_clip():
            return V.extract_point_embedding({"pred_tracks": tracks}, frames, fz, "dog", True, frames_per_batch=8)

        def eager_clip():
            emb = torch.zeros((12, 1280), device=dev)
            for i in range(args.frames):
                m = F.interpolate(eager_frame(u8[i:i + 1].to(dev)), size=(H, W), mode="bilinear")
                p = torch.round(tracks[i]).long()
                emb += m[0, :, p[:, 1].to(dev), p[:, 0].to(dev)].T
            return emb / args.frames

        row = {"H": H, "W": W, "E": E, "frames": args.frames}
        for name, nat, eag in (("featurize_ms", native_frame, lambda: eager_frame(x1)), ("clip_ms", native_clip, eager_clip)):
            nat(), eag()
            torch.cuda.synchronize()
            rounds = []
            for _ in range(args.rounds):
                tn, _ = timed(nat, args.iters)
                te, _ = timed(eag, args.iters)
                rounds.append((tn, te))
            tn = statistics.median(r[0] for r in rounds)
            te = statistics.median(r[1] for r in rounds)
            row[name] = {"native": round(tn, 2), "eager_fp16": round(te, 2), "speedup": round(te / tn, 2)}
        row["per_frame_clip_ms_native"] = round(row["clip_ms"]["native"] / args.frames, 2)
        results.append(row)
        print(json.dumps(row), flush=True)
    out = {"gpu": info, "results": results}
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
