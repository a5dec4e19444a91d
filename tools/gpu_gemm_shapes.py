"""Times the short-K linears of one UNet step (16 frames 512x512, CFG: 32 images) with CUDA events.

usage: gpu_gemm_shapes.py [--seconds S] [--stages 0,3,4] [--root TREE] [--json PATH]

Every transformer / motion-module linear with K <= 640 runs here at its step shape with the epilogue it has in the UNet:
the out-projections add the residual in place and write the next LayerNorm's row statistics (LNOUT + RES), proj_in writes
them only (LNOUT), the QKV / to_q GEMMs fold a LayerNorm whose statistics come from the producer's slices (LN), the
motion module's QKV adds its positional rows too (LN + RV).  Each shape is warmed up, then timed as three windows of
back-to-back launches; the median window gives us per launch, TFLOP/s and the bytes the launch must move (A, weights,
output, residual, statistics) over its time.  --stages sweeps the `gemm_stages` ring-depth limit (0 = the default).
--root times the library of another build tree (e.g. a checkout of the parent commit) with this same script.  The GPU
name, its power limit and the median SM clock sampled after the windows are printed with the numbers.
"""
import argparse
import json
import math
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--seconds", type=float, default=0.6, help="time budget per shape and ring depth")
ap.add_argument("--stages", default="0", help="comma-separated gemm_stages values (0 = as many as fit)")
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))), help="build tree to time")
ap.add_argument("--json", default=os.environ.get("REPORT_JSON"), help="write the rows here as JSON")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))
import torch  # noqa: E402

from videoswap_b200 import ops  # noqa: E402

FRAMES = 16
# (name, M, N, K, epilogue, LayerNorm slices of the producer): level 0 (64x64 latent, C = 320, 131072 rows) and level 1
# (32x32, C = 640, 32768 rows); the slices are the producer's 160-column tiles
SHAPES = [
    ("l0_proj_in_lnout", 131072, 320, 320, "LNOUT", 0),
    ("l0_to_out_lnout_res", 131072, 320, 320, "LNOUT+RES", 0),
    ("l0_proj_out_res", 131072, 320, 320, "RES", 0),
    ("l0_to_q_ln", 131072, 320, 320, "LN", 2),
    ("l0_qkv_ln", 131072, 960, 320, "LN", 2),
    ("l0_qkv_ln_rv", 131072, 960, 320, "LN+RV", 2),
    ("l1_proj_in_lnout", 32768, 640, 640, "LNOUT", 0),
    ("l1_to_out_lnout_res", 32768, 640, 640, "LNOUT+RES", 0),
    ("l1_proj_out_res", 32768, 640, 640, "RES", 0),
    ("l1_to_q_ln", 32768, 640, 640, "LN", 4),
    ("l1_qkv_ln", 32768, 1920, 640, "LN", 4),
    ("l1_qkv_ln_rv", 32768, 1920, 640, "LN+RV", 4),
]


def _smi(fields):
    dev = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
    try:
        r = subprocess.run(["nvidia-smi", "-i", dev, f"--query-gpu={fields}", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True)
    except OSError:
        return []
    return [f.strip() for f in r.stdout.strip().split(",")] if r.returncode == 0 else []


def _case(M, N, K, epi, parts, seed):
    """The launch as a closure over seeded operands, and the bytes it has to move."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).half()
    W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).half()
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    out = (torch.randn(M, N, device="cuda", generator=g)).half()     # also the in-place residual
    f = dict(A=A.data_ptr(), K1=K, lda1=K, Bw=W.data_ptr(), M=M, N=N, bias=bias.data_ptr(), out=out.data_ptr(), ldc=N)
    keep = [A, W, bias, out]
    nbytes = 2 * (M * K + N * K + M * N)
    if "RES" in epi:
        f.update(residual=out.data_ptr(), ldr=N)
        nbytes += 2 * M * N
    if "LNOUT" in epi:
        sums = torch.empty((ops.max_column_tiles(N), M, 2), device="cuda")
        keep.append(sums)
        f.update(ln_sums_out=sums.data_ptr())
        nbytes += 8 * M * -(-N // 160)
    if epi.startswith("LN+") or epi == "LN":
        lp = torch.rand((parts, M, 2), device="cuda", generator=g) * torch.tensor([0.0, float(K) / parts], device="cuda")
        u = torch.randn(N, device="cuda", generator=g)
        keep += [lp, u]
        f.update(ln_parts=lp.data_ptr(), ln_nparts=parts, ln_u=u.data_ptr())
        nbytes += 8 * M * parts
    if "RV" in epi:
        hw = M // (2 * FRAMES)                                      # pixels of one frame
        rv = torch.randn(FRAMES, N, device="cuda", generator=g)
        keep.append(rv)
        f.update(rowvec=rv.data_ptr(), ldrv=N, pix_per_batch=hw, rv_mod=FRAMES)
    return (lambda: ops._gemm_ex(**f)), nbytes, keep


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
    windows, clocks = [], []
    for _ in range(3):
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        e1.synchronize()
        windows.append(e0.elapsed_time(e1) / reps)
        c = _smi("clocks.sm")
        if c:
            clocks.append(float(c[0]))
    return sorted(windows)[1], windows, reps, (sorted(clocks)[len(clocks) // 2] if clocks else None)


def main():
    assert torch.cuda.is_available(), "gpu_gemm_shapes.py needs a GPU"
    card = _smi("name,power.limit")
    print(f"tree: {os.path.abspath(args.root)}")
    print(f"gpu: {card[0] if card else torch.cuda.get_device_name()}, power limit: {card[1] + ' W' if len(card) > 1 else 'unknown'}")
    rows = []
    for stages in [int(s) for s in args.stages.split(",")]:
        ops.set_option("gemm_stages", stages)
        for i, (name, M, N, K, epi, parts) in enumerate(SHAPES):
            fn, nbytes, keep = _case(M, N, K, epi, parts, 1000 + i)
            ms, windows, reps, clk = _time(fn, args.seconds)
            us = ms * 1e3
            tflops = 2.0 * M * N * K / (ms * 1e-3) / 1e12
            gbs = nbytes / (ms * 1e-3) / 1e9
            rows.append(dict(shape=name, M=M, N=N, K=K, epi=epi, stages=stages, us=us, tflops=tflops, gb_s=gbs,
                             windows_ms=windows, launches_per_window=reps, sm_clock_mhz=clk))
            print(f"stages {stages}  {name:22s} {M:6d}x{N:4d}x{K:3d} {epi:9s} {us:8.1f} us  {tflops:6.1f} TFLOP/s  "
                  f"{gbs:6.0f} GB/s  (windows {', '.join(f'{w * 1e3:.1f}' for w in windows)} us; {reps} each; "
                  f"SM clock {clk if clk is not None else '?'} MHz)")
            del keep
    ops.set_option("gemm_stages", 0)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(tree=os.path.abspath(args.root), gpu=card[0] if card else None,
                           power_limit_w=card[1] if len(card) > 1 else None, shapes=rows), f, indent=1)


if __name__ == "__main__":
    main()
