"""Tile-schedule invariance of the persistent GEMM / implicit-GEMM conv kernel (pytest -m gpu).

A tile's outputs come from the same instruction sequence whichever CTA and whichever of the two ping-pong consumers
computes it, and wherever its k-blocks land in the shared-memory ring.  So for a fixed column-tile width the output (and
the LayerNorm row-statistics slices) must be BIT-identical when the grid is capped to a few CTAs ("gemm_ctas": each CTA
then walks many 128-row units, its consumers skip each other's k-blocks across ring wraps, and single-half units follow
one another) and when the ring is shallower ("gemm_stages").  Any difference is a schedule bug.  One run at the shipped
configuration is also checked against a PyTorch fp32 restatement.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import kernel_checks as KC
from videoswap_b200 import ops

pytestmark = pytest.mark.gpu

GRID_CAPS = (1, 2, 3, 5, 8)
RING_DEPTHS = (0, 3)


def _w(n, k, seed):
    return KC._rand((n, k), seed, 1 / math.sqrt(k)).half()


def linear(M, N, K, bn=0, residual=False, seed=0):
    A = KC._rand((M, K), seed).half()
    W = _w(N, K, seed + 1)
    b = KC._rand((N,), seed + 2).float()
    R = KC._rand((M, N), seed + 3).half() if residual else None

    def run():
        return [ops.gemm(A, W, bias=b, residual=R, force_bn=bn)]

    def check(outs):
        ref = A.float() @ W.float().t() + b
        return KC._res(outs[0], ref + R.float() if residual else ref)
    return run, check


def geglu(M=1000, C=320, seed=300):
    A = KC._rand((M, C), seed).half()
    W = _w(8 * C, C, seed + 1)
    bh = KC._rand((8 * C,), seed + 2, 0.1).half()
    wp, bp = ops.pack_geglu(W, bh)

    def run():
        return [ops.gemm(A, wp, bias=bp, mode=ops.EPI_GEGLU)]

    def check(outs):
        v, g = (A.float() @ W.float().t() + bh.float()).chunk(2, -1)
        return KC._res(outs[0], v * F.gelu(g))
    return run, check


def inplace_ln_sums(M=128 * 9 + 9, N=640, K=320, seed=310):
    """residual is out, + row statistics (the transformer's out1 / out2 call)."""
    A = KC._rand((M, K), seed).half()
    W = _w(N, K, seed + 1)
    b = KC._rand((N,), seed + 2).float()
    R = KC._rand((M, N), seed + 3).half()

    def run():
        out = R.clone()
        sums = torch.zeros((ops.max_column_tiles(N), M, 2), dtype=torch.float32, device=KC.DEV)
        ops.gemm(A, W, bias=b, residual=out, out=out, ln_sums=sums)
        return [out, sums]

    def check(outs):
        ref = ((A.float() @ W.float().t() + b).half().float() + R.float()).half()
        return KC._all(KC._res(outs[0], ref), KC.ln_sums_res(outs[0], outs[1].sum(0, keepdim=True), N))
    return run, check


def ln_parts_pe(B=1, Ft=16, hw=20, C=320, seed=320):
    """Producer row statistics -> LayerNorm fold with the temporal PE row vector (the motion module's to_qkv)."""
    M = B * Ft * hw
    x0 = KC._rand((M, C), seed).half()
    W0 = _w(C, C, seed + 1)
    b0 = (KC._rand((C,), seed + 2) + 1.0).float()
    R = KC._rand((M, C), seed + 3).half()
    gamma = (1 + 0.1 * KC._rand((C,), seed + 4)).float()
    beta = (0.1 * KC._rand((C,), seed + 5)).float()
    table = KC._rand((24, C), seed + 6).float()
    W = _w(3 * C, C, seed + 7)

    def run():
        return list(ops.linear_ln_linear(x0, W0, b0, W, gamma, beta, residual=R, pe=table, hw=hw, frames=Ft))

    def check(outs):
        x, out = outs
        y = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5) + table[(torch.arange(M, device=KC.DEV) // hw) % Ft]
        xr = (x0.float() @ W0.float().t() + b0).half().float() + R.float()
        return KC._all(KC._res(out, y @ W.float().t()), KC._res(x, xr))
    return run, check


def conv(n=4, H=16, W=16, c1=320, c2=0, co=320, rowvec=True, residual=True, seed=330):
    x1 = KC._rand((n, H, W, c1), seed).half()
    x2 = KC._rand((n, H, W, c2), seed + 1).half() if c2 else None
    w = KC._rand((co, c1 + c2, 3, 3), seed + 2, 1 / math.sqrt(9 * (c1 + c2))).half()
    wp = ops.pack_conv3x3(w)
    b = KC._rand((co,), seed + 3).float()
    table = KC._rand((n // 2, 4 * co), seed + 4).float() if rowvec else None
    rv = table[:, co:2 * co] if rowvec else None
    R = KC._rand((n, H, W, co), seed + 5).half() if residual else None

    def run():
        return [ops.conv3x3(x1, wp, bias=b, x2=x2, rowvec=rv, imgs_per_batch=2, residual=R)]

    def check(outs):
        x = x1 if x2 is None else torch.cat([x1, x2], -1)
        ref = KC._conv_ref(x, w, b)
        if rowvec:
            ref = ref + rv.repeat_interleave(2, 0)[:, None, None, :]
        if residual:
            ref = ref + R.float()
        return KC._res(outs[0], ref)
    return run, check


# Ring depths at the shipped configuration: 12 / 9 / 7 / 5 stages for BN 64 / 128 / 160 / 256 (3 with gemm_stages = 3).
PROBLEMS = {
    "bn64_k64_odd_m": lambda: linear(128 * 7 + 64, 320, 64, bn=64, seed=340),              # num_kb 1 < depth; m_tiles 15
    "bn128_k_eq_depth": lambda: linear(128 * 6 + 9, 640, 64 * 9, bn=128, residual=True, seed=341),   # num_kb 9 = depth
    "bn160_k5120": lambda: linear(128 * 2 + 64, 320, 5120, bn=160, seed=342),              # num_kb 80 > 2 x depth; 5 tiles
    "bn256_odd_m": lambda: linear(128 * 5 + 9, 768, 320, bn=256, residual=True, seed=343),  # m_tiles 11, n_tiles 3
    "auto_bn_odd_m": lambda: linear(64 * 13, 1280, 1024, seed=344),
    "geglu": geglu,
    "inplace_residual_ln_sums": inplace_ln_sums,
    "ln_parts_pe_fold": ln_parts_pe,
    "conv3x3_rowvec_residual": conv,
    "conv3x3_concat": lambda: conv(n=2, H=8, W=8, c1=640, c2=320, co=640, rowvec=False, residual=False, seed=350),
}


@pytest.mark.parametrize("name", sorted(PROBLEMS))
def test_schedule_invariance(name):
    run, check = PROBLEMS[name]()
    try:
        ops.set_option("gemm_ctas", 0)
        ops.set_option("gemm_stages", 0)
        base = run()
        torch.cuda.synchronize()
        r = check(base)
        assert r["ok"], f"{name}: max abs err {r['err']:.4g} > tol {r['tol']:.4g} (max |ref| {r['ref']:.4g})"
        for stages in RING_DEPTHS:
            ops.set_option("gemm_stages", stages)
            for ctas in GRID_CAPS:
                ops.set_option("gemm_ctas", ctas)
                outs = run()
                torch.cuda.synchronize()
                for i, (a, b) in enumerate(zip(base, outs)):
                    if not torch.equal(a, b):
                        diff = (a.float() - b.float()).abs()
                        rows = torch.nonzero(diff.reshape(-1, a.shape[-1]).amax(-1)).flatten()
                        raise AssertionError(f"{name}: output {i} differs at gemm_ctas={ctas} gemm_stages={stages}: "
                                             f"{rows.numel()} rows, first {rows[:8].tolist()}, max |diff| {diff.max().item():.4g}")
    finally:
        ops.set_option("gemm_ctas", 0)
        ops.set_option("gemm_stages", 0)
