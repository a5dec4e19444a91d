"""Point-drag propagation timing: the native vs_atlas_propagate against tests/atlas_oracle.py run eagerly in stock
PyTorch fp32 on the same GPU.

  python tools/gpu_atlas_propagate.py [--iters 20] [--rounds 5] [--out FILE]

Workload: the shipped size -- F = 72 frames, larger_dim = 768, 10 of 20 TAP points dragged -- with the reference's atlas
network configs (FG_UV_Mapping / FG_UV_Mapping_Inverse 6 x 256, F_Alpha 8 x 256 with pe_dim 5) and seeded weights.  Both
arms run from already-loaded points and end with the tracks on the CPU (one device-to-host copy).  The eager arm batches
the points as the restatement does (it is not the reference's per-point loop with one host sync per frame).  Arms
alternate; each round times `iters` calls of each after a warm-up; the median round is reported, with the GPU name and
power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import make_golden_atlas as M  # noqa: E402
from tests import atlas_oracle as A  # noqa: E402
from videoswap_b200 import atlas  # noqa: E402

F, LARGER_DIM, POINTS, MOVED = 72, 768, 20, 10


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    cfgs = (M.FG, M.FG_INV, M.ALPHA)
    sds = M.nets_for(65)
    nets = tuple(atlas.IMLP_Hash(**c, device="cuda") for c in cfgs)
    for n, sd in zip(nets, sds):
        n.load_state_dict(sd)
    dev_sds = tuple({k: v.cuda() for k, v in sd.items()} for sd in sds)
    g = torch.Generator().manual_seed(3)
    src = {f"p{i}": [float(v) for v in torch.rand(2, generator=g) * 600 + 80] for i in range(POINTS)}
    tgt = {k: [v[0] + 30.0, v[1] - 20.0] for k, v in list(src.items())[:MOVED]}
    name2id = {k: i for i, k in enumerate(src)}
    cols, pts, t_key = A.normalised_points(src, tgt, name2id, 17, LARGER_DIM, F)

    def native():
        res, _ = atlas.propagate_points(nets, pts, float(t_key), F, LARGER_DIM)
        return res.cpu()

    def eager():
        return A.propagate(dev_sds, cfgs, pts.cuda(), t_key, F, LARGER_DIM)["tracks"].cpu()

    with torch.no_grad():
        r_nat, r_eag = native(), eager()
        differ = int((r_nat != r_eag).any(-1).sum())
        for _ in range(3):
            native(), eager()
        torch.cuda.synchronize()
        times = {"native": [], "eager": []}
        for _ in range(a.rounds):
            for name, fn in (("native", native), ("eager", eager)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.iters):
                    fn()
                torch.cuda.synchronize()
                times[name].append((time.perf_counter() - t0) * 1e3 / a.iters)
    rep = {"gpu": gpu_info(), "frames": F, "larger_dim": LARGER_DIM, "points": POINTS, "moved": MOVED,
           "native_ms": statistics.median(times["native"]), "eager_ms": statistics.median(times["eager"]),
           "rounds": times, "track_entries_differing": differ}
    rep["speedup"] = rep["eager_ms"] / rep["native_ms"]
    print(f"GPU: {rep['gpu']}")
    print(f"propagation F={F} larger_dim={LARGER_DIM} {MOVED}/{POINTS} points moved: native {rep['native_ms']:.3f} ms, "
          f"eager torch {rep['eager_ms']:.3f} ms (x{rep['speedup']:.1f}); frames x points whose track differs: {differ}")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
