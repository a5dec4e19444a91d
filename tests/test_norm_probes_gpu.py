"""Per-element normalisation tests (pytest -m gpu): GroupNorm on every path (5-D sets with both statistics kernels, the
frame-shard statistics + apply pair, the per-frame cluster kernel at every cluster size and its two-kernel fallback),
LayerNorm (ln5_kernel, ln_kernel), the LayerNorm folded into the next GEMM (row-statistics kernel and producer slices,
linear and GEGLU) and the SiLU / erf-GELU epilogues, against fp64 math on the same fp16 inputs with the bound derived in
tests/norm_probes.py.  Inputs give every (set, group) and row its own statistics, impulses at the schedules' edges and a
cancellation sweep; run with -s to see the measured envelope at mean / spread 32 .. 256."""
import pytest
import torch

from tests import norm_probes as P
from videoswap_b200 import ops

pytestmark = pytest.mark.gpu


def _opt(name, value, default):
    def wrap(fn):
        def run(*a):
            ops.set_option(name, value)
            try:
                return fn(*a)
            finally:
                ops.set_option(name, default)
        return run
    return wrap


def _gn(x1, x2, gamma, beta, eps, imgs_per_set, silu):
    return ops.groupnorm(x1, gamma, beta, P.GROUPS, eps, imgs_per_set=imgs_per_set, silu=silu, x2=x2)


_GN = {"v1": _gn, "v2": _opt("gn_stats_v2", 1, 0)(_gn)}
_GN_PAIR = _opt("gn_fused", 0, 1)(_gn)


def _shards(k):
    """The frame-sharded 5-D GroupNorm on one GPU: k shards add their sums into one buffer, each applies count_scale = k."""
    def run(x1, x2, gamma, beta, eps, F, silu):
        n, H, W, _ = x1.shape
        B, fs = n // F, F // k

        def shard(t, s):
            return None if t is None else t.view(B, F, H, W, -1)[:, s * fs:(s + 1) * fs].reshape(B * fs, H, W, -1).contiguous()

        sums = torch.zeros((B, P.GROUPS, 2), dtype=torch.float32, device=x1.device)
        for s in range(k):
            ops.groupnorm_stats(shard(x1, s), sums, P.GROUPS, fs, x2=shard(x2, s), zero_first=False)
        outs = [ops.groupnorm_apply(shard(x1, s), sums, gamma, beta, P.GROUPS, eps, fs, count_scale=k, silu=silu,
                                    x2=shard(x2, s)) for s in range(k)]
        return torch.cat([o.view(B, fs, H, W, -1) for o in outs], 1).reshape(n, H, W, -1)
    return run


def _ln(x, gamma, beta, pe, hw, F):
    return ops.layernorm(x, gamma, beta, pe=pe, hw=hw, F=F)


def _packed(W, geglu):
    if not geglu:
        return W, None, ops.EPI_LINEAR
    wp, bp = ops.pack_geglu(W, torch.zeros(W.shape[0], dtype=torch.float16, device=W.device))
    return wp, bp, ops.EPI_GEGLU


def _fold_stats(x, W, gamma, beta, pe, hw, F, residual, geglu):
    wp, bp, mode = _packed(W, geglu)
    return x, ops.ln_linear(x, wp, gamma, beta, bias=bp, pe=pe, hw=hw, frames=F, mode=mode)


def _fold_slices(x, W, gamma, beta, pe, hw, F, residual, geglu):
    """Producer x = x0 I + 0 (+ R): with no residual x0 itself, so the probed rows are exactly the chosen ones."""
    C = x.shape[1]
    wp, bp, mode = _packed(W, geglu)
    eye = torch.eye(C, dtype=torch.float16, device=x.device)
    R = None
    if residual:
        g = torch.Generator().manual_seed(C)
        R = (0.05 * torch.randn(x.shape, generator=g)).half().to(x.device)
    xu, out = ops.linear_ln_linear(x, eye, torch.zeros(C, device=x.device), wp, gamma, beta, residual=R, bias=bp, mode=mode,
                                   pe=pe, hw=hw, frames=F)
    if residual:
        assert torch.equal(xu, (x.float() + R.float()).half()), "producer residual add"
    return xu, out


def _geglu(A, W):
    wp, bp, mode = _packed(W, True)
    return ops.gemm(A, wp, bias=bp, mode=mode)


def _silu(x, sums, gamma, beta, eps):
    return ops.groupnorm_apply(x, sums, gamma, beta, P.GROUPS, eps, 1, silu=True)


CASES = {}
# 5-D GroupNorm (statistics over F frames): every UNet width, the up path's skip concats, the headline shape
for _v, _f in _GN.items():
    CASES.update({
        f"gn5d_320_{_v}": lambda f=_f: P.check_groupnorm(f, 2, 4, 16, 16, 320, seed=10),
        f"gn5d_640_{_v}": lambda f=_f: P.check_groupnorm(f, 2, 4, 16, 16, 640, silu=False, seed=11),
        f"gn5d_1280_{_v}": lambda f=_f: P.check_groupnorm(f, 2, 3, 8, 8, 1280, seed=12),
        f"gn5d_2560_{_v}": lambda f=_f: P.check_groupnorm(f, 2, 3, 8, 8, 2560, silu=False, seed=13),
        f"gn5d_cat_640_320_{_v}": lambda f=_f: P.check_groupnorm(f, 2, 4, 16, 16, 640, 320, seed=14),
        f"gn5d_cat_1280_640_{_v}": lambda f=_f: P.check_groupnorm(f, 2, 3, 8, 8, 1280, 640, silu=False, seed=15),
        f"gn5d_cat_1280_1280_{_v}": lambda f=_f: P.check_groupnorm(f, 2, 3, 8, 8, 1280, 1280, seed=16),
        f"gn5d_cat_640_640_{_v}": lambda f=_f: P.check_groupnorm(f, 2, 4, 16, 16, 640, 640, seed=17),
        f"gn5d_cat_320_320_{_v}": lambda f=_f: P.check_groupnorm(f, 2, 4, 32, 32, 320, 320, silu=False, seed=18),
        f"gn5d_headline_2x16x64x64x320_{_v}": lambda f=_f: P.check_groupnorm(f, 2, 16, 64, 64, 320, seed=19),
        f"gn5d_pixel_sweep_8x8_f4_{_v}": lambda f=_f: P.check_pixel_sweep(f, seed=20),
    })
CASES.update({
    f"gn5d_frame_shards_k{k}": lambda k=k: P.check_groupnorm(_shards(k), 2, 16, 32, 32, 320, k=k, launches=2, seed=30 + k)
    for k in (2, 4)
})
CASES["gn5d_frame_shards_k2_cat_640_320"] = lambda: P.check_groupnorm(_shards(2), 1, 8, 16, 16, 640, 320, k=2, seed=35)
# per-frame GroupNorm (transformer / motion-module norms, eps 1e-6): one shape per cluster size, then the fallback
for _name, (_H, _W, _C) in {"cluster16_64x64x320": (64, 64, 320), "cluster8_32x32x640": (32, 32, 640),
                            "cluster4_16x16x1280": (16, 16, 1280), "cluster2_8x16x1280": (8, 16, 1280),
                            "cluster1_8x8x1280": (8, 8, 1280)}.items():
    CASES[f"gn_frame_{_name}"] = lambda H=_H, W=_W, C=_C: P.check_groupnorm(_gn, 4, 1, H, W, C, silu=False, launches=2, seed=40 + C)
    CASES[f"gn_frame_{_name}_pair"] = lambda H=_H, W=_W, C=_C: P.check_groupnorm(_GN_PAIR, 4, 1, H, W, C, silu=False, seed=40 + C)
for _name, (_H, _W, _C) in {"45x60x320": (45, 60, 320), "23x30x640": (23, 30, 640), "90x160x320": (90, 160, 320)}.items():
    CASES[f"gn_frame_fallback_{_name}"] = lambda H=_H, W=_W, C=_C: P.check_groupnorm(_gn, 3, 1, H, W, C, silu=False, launches=2, seed=50 + H)
CASES["gn_frame_fused_silu_16x16x1280"] = lambda: P.check_groupnorm(_gn, 4, 1, 16, 16, 1280, silu=True, seed=60)
CASES["gn_frame_eps_1e-5_8x8x1280"] = lambda: P.check_groupnorm(_gn, 4, 1, 8, 8, 1280, eps=1e-5, silu=False, seed=61)
# LayerNorm: ln5_kernel (rows not a multiple of 2 RPW, frame-distinct PE rows) and the generic ln_kernel
for _C in (320, 640, 1280):
    CASES[f"ln5_{_C}"] = lambda C=_C: P.check_layernorm(_ln, 4096 + 2 * 32 // (C // 40) + 1, C, seed=70 + C)
    CASES[f"ln5_{_C}_pe"] = lambda C=_C: P.check_layernorm(_ln, 16 * 64 * 3 + 5, C, pe=True, hw=64, F=16, seed=71 + C)
for _C in (768, 2048):
    CASES[f"ln_generic_{_C}"] = lambda C=_C: P.check_layernorm(_ln, 1001, C, pe=True, hw=7, F=5, seed=72 + C)
# the folded LayerNorm, read through one-hot weights
for _C in (320, 640, 1280):
    CASES[f"fold_stats_{_C}"] = lambda C=_C: P.check_ln_fold(_fold_stats, 2 * 320 + 37, C, N=2 * C, seed=80 + C)
    CASES[f"fold_slices_{_C}"] = lambda C=_C: P.check_ln_fold(_fold_slices, 3 * 128 + 5, C, producer=True, seed=81 + C)
    CASES[f"fold_slices_{_C}_residual"] = lambda C=_C: P.check_ln_fold(_fold_slices, 1000, C, residual=True, producer=True, seed=82 + C)
CASES["fold_stats_320_pe"] = lambda: P.check_ln_fold(_fold_stats, 16 * 40, 320, N=960, pe=True, hw=40, F=16, seed=90)
CASES["fold_slices_320_motion_pe"] = lambda: P.check_ln_fold(_fold_slices, 2 * 16 * 64, 320, N=960, pe=True, hw=64, F=16,
                                                            residual=True, producer=True, seed=91)
CASES["fold_stats_320_geglu"] = lambda: P.check_ln_fold(_fold_stats, 700, 320, N=1280, geglu=True, seed=92)
CASES["fold_slices_640_geglu"] = lambda: P.check_ln_fold(_fold_slices, 700, 640, N=2560, geglu=True, producer=True, seed=93)
# epilogue activations
CASES["gelu_sig_probe"] = lambda: P.check_gelu(_geglu)
CASES["silu_probe"] = lambda: P.check_silu(_silu)


@pytest.mark.parametrize("name", sorted(CASES))
def test_norm_probes(name):
    r = CASES[name]()
    torch.cuda.synchronize()
    if r.get("report"):
        print(f"\n{name}: worst err / bound {r['err']:.4g}; {r['report']}")
    else:
        print(f"\n{name}: worst err / bound {r['err']:.4g}")
    assert r["ok"], f"{name}: {r.get('what', '')}: worst err / bound {r['err']:.4g}"
