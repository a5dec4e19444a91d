"""The power of the normalisation probes (tests/norm_probes.py), shown without a GPU.  A torch emulation of the kernels'
arithmetic -- shifted fp32 partial sums per block (per CTA) over the launch geometry of norm.cu, added block after
block, the one-pass GroupNorm variance, x a + b, SiLU, fp16 store; two-pass LayerNorm; the folded LayerNorm from row
statistics or producer column-tile slices; gelu_sig -- passes every comparator with 2x margin, and every planted bug
fails.  (Inside a block the emulation sums with torch reductions, not in the kernels' thread order.)  For three of the bugs the random-input
comparator of tests/kernel_checks.py (max|d| <= 2^-8 max|ref| + 2e-3, iid inputs) is shown to let them through."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import norm_probes as P

SMS = 132


def _split_group(C):
    """Group of every channel as the kernels map it, and with the bug that maps the first channel of the second group
    of a vector that straddles two groups to the first one (ga)."""
    cpg = C // P.GROUPS
    good = torch.arange(C) // cpg
    bad = good.clone()
    for v in range(C // 8):
        ga = (8 * v) // cpg
        if (8 * v + 7) // cpg != ga:
            bad[(ga + 1) * cpg] = ga
    return good, bad


def emulate_gn(mutation=None, sms=SMS):
    """gn(x1, x2, gamma, beta, eps, imgs_per_set, silu) with the statistics arithmetic of norm.cu: the blocks of gn_fill
    (or, per frame, the CTAs of gn_frame_fused_kernel) each sum x - k in fp32 with k the block's first pixel at the
    group's first channel, convert their partial to plain sums (gn_unshift), and the partials are added in fp32 one
    after the other (the global atomics / the cluster exchange); then gn_apply's x a + b, SiLU and the fp16 store.
    Inside a block the sums are torch reductions, not the kernels' thread / shared-atomic order."""
    def run(x1, x2, gamma, beta, eps, F_, silu):
        x = x1 if x2 is None else torch.cat([x1, x2], -1)
        n, H, W, C = x.shape
        hw, cpg = H * W, C // P.GROUPS
        ns = n // F_
        xs = x.reshape(ns, F_ * hw, C).float()
        good, bad = _split_group(C)
        cg = bad if mutation == "split_channel" else good
        ag = bad if mutation == "split_channel_apply" else good
        sched = P.gn_schedules(C, hw, F_, n, sms)
        fused = F_ == 1 and x2 is None and len(sched) > 1
        first = sched[1 if fused else 0][0]
        starts = torch.unique(first)
        bid = torch.searchsorted(starts, first)                        # block of every pixel
        nb = starts.numel()
        k = xs[:, starts][:, :, torch.arange(P.GROUPS) * cpg]           # [ns, blocks, G] shifts
        d = xs - k[:, :, cg][:, bid]
        if mutation == "tail_dropped":                                  # the tail loops' pixels never accumulated
            rows, ppb, nblk = P.gn_geometry(C, hw, F_, n, sms)
            for b in range(nblk):
                d[:, P.tail_pixels(b * ppb, min((b + 1) * ppb, F_ * hw), rows)] = 0
        sc = torch.zeros(ns, nb, C).index_add_(1, bid, d)
        qc = torch.zeros(ns, nb, C).index_add_(1, bid, d * d)
        sp = torch.zeros(ns, nb, P.GROUPS).index_add_(2, cg, sc)
        qp = torch.zeros(ns, nb, P.GROUPS).index_add_(2, cg, qc)
        m = (torch.bincount(bid, minlength=nb) * cpg).float()[None, :, None]
        mk = m * k
        Sb, Qb = sp + mk, qp + k * (2 * sp + mk)                        # gn_unshift
        if fused and mutation == "cluster_own":
            S, Q = nb * Sb, nb * Qb                                     # [ns, ncta, G]: each CTA its own partial x ncta
            ppc = hw // nb
        else:
            last = nb - 1 if fused and mutation == "last_cta" else nb
            S, Q = torch.zeros(ns, P.GROUPS), torch.zeros(ns, P.GROUPS)
            for b in range(last):
                S, Q = S + Sb[:, b], Q + Qb[:, b]
            S, Q = S[:, None], Q[:, None]
            ppc = F_ * hw
        if mutation == "set_shift":
            S, Q = S.roll(-1, 0), Q.roll(-1, 0)
        inv_n = torch.tensor(1.0 / (F_ * hw * cpg), dtype=torch.float32)
        mean = S * inv_n
        var = (Q * inv_n - mean * mean).clamp_min(0)
        rstd = torch.rsqrt(var + (1e-5 if mutation == "eps" else eps))
        if mutation == "rstd":
            rstd = rstd * 1.002
        a = rstd[..., ag] * gamma.float()                                  # [ns, slices, C]
        b = beta.float() - mean[..., ag] * a
        y = xs.reshape(ns, -1, ppc, C) * a[:, :, None] + b[:, :, None]
        if silu:
            y = y / (1 + torch.exp(-y))
        return y.half().reshape(n, H, W, C)
    return run


def emulate_ln(mutation=None):
    """ln(x, gamma, beta, pe, hw, F): two-pass fp32 row statistics (ln5_kernel); ln_row_ahead: row r + RPW's."""
    def run(x, gamma, beta, pe, hw, F_):
        rows, C = x.shape
        xf = x.float()
        mean = xf.mean(1, keepdim=True)
        var = ((xf - mean) ** 2).mean(1, keepdim=True)
        rstd = torch.rsqrt(var + 1e-5)
        if mutation == "ln_row_ahead":
            rpw = 32 // (C // 40)
            idx = (torch.arange(rows) + rpw) % rows
            mean, rstd = mean[idx], rstd[idx]
        y = (xf - mean) * rstd * gamma + beta
        if pe is not None:
            y = y + pe[(torch.arange(rows) // hw) % F_]
        return y.half()
    return run


def _gelu_sig(x, tanh=False, unclamped=False):
    if tanh:
        return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))
    xn = x if unclamped else x.clamp_min(-5.0)
    xc = xn.clamp_max(5.0)
    u = xc * xc
    q = u * 2.47135360e-05 + 7.37690930e-04
    q = q * u - 1.05988323e-01
    q = q * u - 2.30164247e+00
    return xn / (1 + torch.exp2(xc * q))


def emulate_fold(mutation=None, slices=False):
    """fold(x, W, gamma, beta, pe, hw, F, residual, geglu) -> (x, out): statistics per row (two-pass, or one-pass from
    128-column slices of the producer), rstd x' + (-mean rstd) gamma + beta through W, PE added, GEGLU on request."""
    def run(x, W, gamma, beta, pe, hw, F_, residual, geglu):
        rows, C = x.shape
        xf = x.float()
        if slices:
            sl = [xf[:, c:c + 128] for c in range(0, C, 128)]
            if mutation == "fold_last_slice":
                sl = sl[:-1]
            S = sum(s.sum(1, keepdim=True) for s in sl)
            Q = sum((s * s).sum(1, keepdim=True) for s in sl)
            mean = S / C
            rstd = torch.rsqrt((Q / C - mean * mean).clamp_min(0) + 1e-5)
        else:
            mean = xf.mean(1, keepdim=True)
            rstd = torch.rsqrt(((xf - mean) ** 2).mean(1, keepdim=True) + 1e-5)
        g16 = gamma.half().float()
        acc = (xf * g16) @ W.float().t()
        u = g16 @ W.float().t()
        c = beta @ W.float().t()
        y = rstd * acc + ((-mean * rstd) * u + c)
        if pe is not None:
            y = y + (pe @ W.float().t())[(torch.arange(rows) // hw) % F_]
        if geglu:
            h = W.shape[0] // 2
            y = y[:, :h] * _gelu_sig(y[:, h:], tanh=mutation == "tanh")
        return x, y.half()
    return run


def emulate_geglu(mutation=None):
    def run(A, W):
        h = (A.float() @ W.float().t())
        n = W.shape[0] // 2
        return (h[:, :n] * _gelu_sig(h[:, n:], mutation == "tanh", mutation == "unclamped")).half()
    return run


def emulate_silu(x, sums, gamma, beta, eps):
    xf = x.float()
    return (xf / (1 + torch.exp(-xf))).half()


C5 = dict(dev="cpu", sms=SMS)
CASES = {
    "gn5d_cat_640_320": lambda f: P.check_groupnorm(f, 2, 4, 8, 8, 640, 320, seed=14, **C5),
    "gn5d_cat_1280_640": lambda f: P.check_groupnorm(f, 2, 2, 4, 8, 1280, 640, silu=False, seed=15, **C5),
    "gn5d_320_16x16": lambda f: P.check_groupnorm(f, 2, 4, 16, 16, 320, seed=10, **C5),
    "gn5d_pixel_sweep_8x8_f4": lambda f: P.check_pixel_sweep(f, seed=20, **C5),
    "gn_frame_cluster16_64x64x320": lambda f: P.check_groupnorm(f, 2, 1, 64, 64, 320, silu=False, kinds=("distinct", "impulse"), seed=40, **C5),
    "gn_frame_cluster4_16x16x1280": lambda f: P.check_groupnorm(f, 2, 1, 16, 16, 1280, silu=False, launches=2, seed=41, **C5),
    "gn_frame_fallback_23x30x640": lambda f: P.check_groupnorm(f, 2, 1, 23, 30, 640, silu=False, seed=42, **C5),
}
LN_CASES = {
    "ln5_320": lambda f: P.check_layernorm(f, 4096 + 9, 320, seed=70, dev="cpu"),
    "ln5_1280_pe": lambda f: P.check_layernorm(f, 16 * 8 + 5, 1280, pe=True, hw=8, F=16, seed=71, dev="cpu"),
}
FOLD_CASES = {
    "fold_stats_320_pe": lambda f: P.check_ln_fold(f, 16 * 40, 320, N=960, pe=True, hw=40, F=16, seed=90, dev="cpu"),
    "fold_slices_640": lambda f: P.check_ln_fold(f, 3 * 128 + 5, 640, producer=True, seed=81, dev="cpu"),
    "fold_stats_320_geglu": lambda f: P.check_ln_fold(f, 300, 320, N=1280, geglu=True, seed=92, dev="cpu"),
}

# (emulation, case that must reject it)
MUTATIONS = {
    "set_s_plus_1": (lambda: emulate_gn("set_shift"), CASES["gn5d_320_16x16"]),
    "split_channel_in_group_ga": (lambda: emulate_gn("split_channel"), CASES["gn5d_cat_640_320"]),
    "split_channel_normalised_with_group_ga": (lambda: emulate_gn("split_channel_apply"), CASES["gn5d_320_16x16"]),
    "cluster_total_ncta_x_own": (lambda: emulate_gn("cluster_own"), CASES["gn_frame_cluster4_16x16x1280"]),
    "last_cta_partial_omitted": (lambda: emulate_gn("last_cta"), CASES["gn_frame_cluster4_16x16x1280"]),
    "eps_1e-5_for_1e-6": (lambda: emulate_gn("eps"), CASES["gn_frame_cluster4_16x16x1280"]),
    "tail_chunk_dropped": (lambda: emulate_gn("tail_dropped"), CASES["gn5d_pixel_sweep_8x8_f4"]),
    "rstd_x1.002": (lambda: emulate_gn("rstd"), CASES["gn5d_320_16x16"]),
    "ln_stats_row_rpw_ahead": (lambda: emulate_ln("ln_row_ahead"), LN_CASES["ln5_320"]),
    "fold_last_slice_missing": (lambda: emulate_fold("fold_last_slice", slices=True), FOLD_CASES["fold_slices_640"]),
    "tanh_gelu_in_fold": (lambda: emulate_fold("tanh"), FOLD_CASES["fold_stats_320_geglu"]),
    "tanh_gelu_in_geglu": (lambda: emulate_geglu("tanh"), lambda f: P.check_gelu(f, dev="cpu")),
    "gelu_numerator_unclamped": (lambda: emulate_geglu("unclamped"), lambda f: P.check_gelu(f, dev="cpu")),
}


def _msg(name, r):
    return f"{name}: worst err / bound {r['err']:.3g} ({r.get('what', '')})"


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_groupnorm_passes_with_margin(name):
    r = CASES[name](emulate_gn())
    assert r["ok"] and r["err"] <= 0.5, _msg(name, r)


@pytest.mark.parametrize("name", sorted(LN_CASES))
def test_emulated_layernorm_passes_with_margin(name):
    r = LN_CASES[name](emulate_ln())
    assert r["ok"] and r["err"] <= 0.5, _msg(name, r)


@pytest.mark.parametrize("name", sorted(FOLD_CASES))
def test_emulated_fold_passes_with_margin(name):
    r = FOLD_CASES[name](emulate_fold(slices="slices" in name))
    assert r["ok"] and r["err"] <= 0.5, _msg(name, r)


def test_emulated_epilogue_activations_pass():
    """Not held to 0.5: these bounds are the activations' own claimed error (gelu_sig: 1.2e-5 + 2^-20 max(x, 0); silu_f:
    its MUFU terms) plus one fp16 rounding, not twice a derived worst case, and the minimax fit of gelu_sig reaches
    0.97 of its claim.  The emulation computes the same formulas in fp32."""
    for r in (P.check_gelu(emulate_geglu(), dev="cpu"), P.check_silu(emulate_silu, dev="cpu")):
        assert r["ok"] and r["err"] <= 1.0, _msg("activation", r)


@pytest.mark.parametrize("name", sorted(MUTATIONS))
def test_planted_mutation_is_rejected(name):
    emu, case = MUTATIONS[name]
    r = case(emu())
    assert not r["ok"], _msg(name, r)


def _old_check(gn, per_frame, H, W, c1, c2=0, B=2, Fr=3, eps=1e-6, seed=100, mean=0.3):
    """tests/kernel_checks.py check_groupnorm on CPU: iid N(mean, 1.5^2) inputs, max|d| <= 2^-8 max|ref| + 2e-3."""
    g = torch.Generator().manual_seed(seed)
    n = B * Fr
    x1 = (torch.randn(n, H, W, c1, generator=g) * 1.5 + mean).half()
    x2 = (torch.randn(n, H, W, c2, generator=g) * 0.7 - 0.2).half() if c2 else None
    C = c1 + c2
    gamma = 1 + 0.1 * torch.randn(C, generator=g)
    beta = 0.1 * torch.randn(C, generator=g)
    out = gn(x1, x2, gamma, beta, eps, 1 if per_frame else Fr, True)
    x = (x1 if x2 is None else torch.cat([x1, x2], -1)).float().permute(0, 3, 1, 2)
    if per_frame:
        ref = F.group_norm(x, 32, gamma, beta, eps)
    else:
        ref = F.group_norm(x.reshape(B, Fr, C, H, W).transpose(1, 2), 32, gamma, beta, eps).transpose(1, 2).reshape(n, C, H, W)
    ref = F.silu(ref).permute(0, 2, 3, 1)
    err = (out.float() - ref).abs().max().item()
    return err <= 2 ** -8 * ref.abs().max().item() + 2e-3


# The bugs the random-input comparator lets through at the UNet's shapes ...
OLD_BLIND = {
    "set_s_plus_1": lambda: _old_check(emulate_gn("set_shift"), False, 64, 64, 320, B=2, Fr=16),
    "split_channel_normalised_with_group_ga": lambda: _old_check(emulate_gn("split_channel_apply"), False, 32, 32, 320, B=2, Fr=16),
    "eps_1e-5_for_1e-6": lambda: _old_check(emulate_gn("eps"), True, 16, 16, 1280, B=1, Fr=2),
}


@pytest.mark.parametrize("name", sorted(OLD_BLIND))
def test_random_input_comparator_passes_the_bug(name):
    """What the old suite could not see: the same planted bug passes the random-input comparator."""
    assert OLD_BLIND[name](), f"{name}: the random-input check caught it after all"


# ... and two it does catch there: counting one more channel in ga gives that group's sums cpg + 1 channels against a
# 1 / n for cpg (a ~3 % variance error at cpg = 10), and a cluster slice of 2560 elements per group is ~2 % off the
# whole image's statistics.
OLD_CATCHES = {
    "split_channel_in_group_ga": lambda: _old_check(emulate_gn("split_channel"), False, 32, 32, 320, B=2, Fr=16),
    "cluster_total_ncta_x_own_16x16x1280": lambda: _old_check(emulate_gn("cluster_own"), True, 16, 16, 1280, B=1, Fr=2),
    "cluster_total_ncta_x_own_64x64x320": lambda: _old_check(emulate_gn("cluster_own"), True, 64, 64, 320, B=1, Fr=2),
}


@pytest.mark.parametrize("name", sorted(OLD_CATCHES))
def test_random_input_comparator_rejects_the_bug(name):
    assert not OLD_CATCHES[name](), f"{name}: the random-input check let it through"
