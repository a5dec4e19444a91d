"""The GEMM / conv probes without a GPU: tests/gemm_probes.py's torch emulation of gemm_tc_kernel (producer odometer and
concat split, tile_pixel over pick_conv_tile's boxes, sub-pixel panels and shifted views, staged and direct epilogues)
runs through the same comparators the GPU test uses, at small shapes.  The emulation must pass exactly; each planted bug
must be rejected.  For each bug the verdict of the random-input comparator of tests/kernel_checks.py (max|d| <= 2^-8
max|ref| + 2e-3) is recorded as well: the precision bugs pass it."""
import math

import pytest
import torch

from tests import gemm_probes as P
from tests import kernel_checks as KC

CPU = "cpu"


def E(bug=None):
    return P.Emulator(bug)


EXACT_CASES = {
    "gemm_k72_rowvec_slice": lambda K: P.int_linear(K, CPU, 200, 96, 72, rowvec=True, seed=1),
    "gemm_rowvec_rv_mod": lambda K: P.int_linear(K, CPU, 300, 64, 64, rowvec=True, rv_mod=3, seed=2),
    "gemm_concat_residual": lambda K: P.int_linear(K, CPU, 150, 64, 128, K2=64, residual="sep", seed=3),
    "gemm_inplace_ln_sums_bn64": lambda K: P.int_linear(K, CPU, 200, 160, 64, bn=64, residual="inplace", ln_sums=True, seed=4),
    "gemm_ln_sums_auto": lambda K: P.int_linear(K, CPU, 130, 256, 64, ln_sums=True, seed=5),
    "conv_3x6x8_rowvec_residual": lambda K: P.int_conv(K, CPU, 3, 6, 8, 64, 32, rowvec=True, F_=2, residual=True, seed=6),
    "conv_concat_2x5x7": lambda K: P.int_conv(K, CPU, 2, 5, 7, 64, 32, c2=64, seed=7),
    "conv_1x1": lambda K: P.int_conv(K, CPU, 3, 1, 1, 64, 32, seed=8),
    "upsample_plain_3x4": lambda K: P.int_subpixel(K, CPU, 2, 3, 4, 64, 32, how="plain", seed=9),
    "upsample_packed_2x3": lambda K: P.int_subpixel(K, CPU, 1, 2, 3, 64, 32, how="packed", seed=10),
    "upsample_sized_both_odd": lambda K: P.int_subpixel(K, CPU, 2, 3, 4, 64, 32, OH=5, OW=7, seed=11),
    "upsample_sized_rows_odd": lambda K: P.int_subpixel(K, CPU, 2, 3, 4, 64, 32, OH=5, OW=8, seed=12),
    "upsample_sized_cols_odd": lambda K: P.int_subpixel(K, CPU, 2, 3, 4, 64, 32, OH=6, OW=7, seed=13),
    "onehot_gemm_rowvec_residual": lambda K: P.onehot_linear(K, CPU, 150, 128, 64, seed=14),
    "onehot_gemm_rv_mod_bn64": lambda K: P.onehot_linear(K, CPU, 150, 64, 64, rv_mod=3, bn=64, seed=15),
    "onehot_gemm_direct_n40": lambda K: P.onehot_linear(K, CPU, 150, 64, 40, seed=16),
    "onehot_gemm_direct_misaligned": lambda K: P.onehot_linear(K, CPU, 150, 64, 64, direct=True, seed=17),
    "two_term_k200": lambda K: P.two_term(K, CPU, 130, 200, 64, seed=18),
    "onehot_conv_3x5x6": lambda K: P.onehot_conv(K, CPU, 3, 5, 6, 64, seed=19),
    "onehot_upsample_3x4_to_5x7": lambda K: P.onehot_subpixel(K, CPU, 1, 3, 4, 64, 5, 7, seed=20),
}

BOUND_CASES = {
    "geglu_320": lambda K: P.geglu_case(K, CPU, 200, 320, seed=21),
    "quick_gelu_bn128": lambda K: P.qgelu_case(K, CPU, 150, 128, Kd=128, N=256, seed=22),
}

# planted bug -> the case that must reject it
MUTATIONS = {
    "odometer_early": EXACT_CASES["conv_3x6x8_rowvec_residual"],
    "concat_late": EXACT_CASES["gemm_concat_residual"],
    "image_ignored": EXACT_CASES["conv_3x6x8_rowvec_residual"],
    "panel_py_px_swapped": EXACT_CASES["upsample_plain_3x4"],
    "third_tap_unshifted": EXACT_CASES["upsample_sized_both_odd"],
    "rv_mod_ignored": EXACT_CASES["gemm_rowvec_rv_mod"],
    "ldrv_as_n": EXACT_CASES["gemm_k72_rowvec_slice"],
    "geglu_granule_64": BOUND_CASES["geglu_320"],
    "bias_fp16": EXACT_CASES["onehot_gemm_rowvec_residual"],
    "operands_bf16": EXACT_CASES["onehot_gemm_rowvec_residual"],
    "kblock_fp16": EXACT_CASES["two_term_k200"],
    "residual_before_rounding": EXACT_CASES["onehot_gemm_direct_misaligned"],
}


def _msg(name, r):
    return f"{name}: err {r['err']:.4g} ({r['what']})"


def test_every_planted_bug_has_a_case():
    assert sorted(MUTATIONS) == sorted(P.PLANTED)


@pytest.mark.parametrize("name", sorted(EXACT_CASES))
def test_emulation_is_exact(name):
    r = EXACT_CASES[name](E())
    assert r["ok"] and r["err"] == 0, _msg(name, r)


@pytest.mark.parametrize("name", sorted(BOUND_CASES))
def test_emulated_activations_within_bound(name):
    r = BOUND_CASES[name](E())
    assert r["ok"], _msg(name, r)


@pytest.mark.parametrize("bug", sorted(MUTATIONS))
def test_planted_bug_is_rejected(bug):
    r = MUTATIONS[bug](E(bug))
    assert not r["ok"], _msg(bug, r)


# ---------------------------------------------------------------------------------------------------- the old comparator
def _randn(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale


def _old_gemm(K, N=320, residual=True, direct=False, concat=False, rowvec=False, M=512, Kd=320, seed=400):
    """kernel_checks.check_gemm / _concat / _rowvec on iid N(0, 1) data (weights N(0, 1 / K))."""
    K2 = 64 if concat else 0
    A = _randn((M, Kd), seed).half()
    A2 = _randn((M, K2), seed + 1).half() if concat else None
    W = _randn((N, Kd + K2), seed + 2, 1 / math.sqrt(Kd + K2)).half()
    b = _randn((N,), seed + 3)
    R = _randn((M, N), seed + 4).half() if residual else None
    rv = P.table_slice(3, N, seed + 5, CPU, fine=True) if rowvec else None
    out = P.nan16((M, N + 8), CPU)[:, 4:4 + N] if direct else None
    out = K.gemm(A, W, bias=b, A2=A2, rowvec=rv, ppb=64, rv_mod=3 if rowvec else 0, residual=R, out=out)
    ref = (A.float() if A2 is None else torch.cat([A, A2], 1).float()) @ W.float().t() + b
    if rowvec:
        ref = ref + rv[(torch.arange(M) // 64) % 3]
    if residual:
        ref = ref + R.float()
    return KC._res(out, ref)["ok"]


def _old_conv(K, seed=410):
    """kernel_checks.check_conv3x3 with a row vector and residual, at a tile of 4 images."""
    n, H, W, ci, co = 3, 6, 8, 64, 64
    x = _randn((n, H, W, ci), seed).half()
    w = _randn((co, ci, 3, 3), seed + 1, 1 / math.sqrt(9 * ci)).half()
    b = _randn((co,), seed + 2)
    rv = _randn((2, co), seed + 3)
    R = _randn((n, H, W, co), seed + 4).half()
    out = K.conv3x3(x, K.pack_conv3x3(w), bias=b, rowvec=rv, ppb=2 * H * W, residual=R)
    ref = P.conv64(x, w).float() + b + rv[torch.arange(n) // 2][:, None, None, :] + R.float()
    return KC._res(out, ref)["ok"]


def _old_upsample(K, OH=6, OW=8, seed=420):
    """kernel_checks.check_upsample_conv (and its odd-size variant)."""
    x = _randn((2, 3, 4, 64), seed).half()
    w = _randn((64, 64, 3, 3), seed + 1, 1 / math.sqrt(9 * 64)).half()
    b = _randn((64,), seed + 2)
    out = K.upsample_sized(x, w, b, OH, OW) if (OH | OW) & 1 else K.upsample(x, w, b)
    return KC._res(out, P.conv64(P.upsample(x, OH, OW), w).float() + b)["ok"]


def _old_geglu(K, M=200, C=320, seed=430):
    A = _randn((M, C), seed).half()
    W = _randn((8 * C, C), seed + 1, 1 / math.sqrt(C)).half()
    b = _randn((8 * C,), seed + 2, 0.1).half()
    wp, bp = K.pack_geglu(W, b)
    out = K.gemm(A, wp, bias=bp, mode=P.GEGLU)
    v, g = (A.float() @ W.float().t() + b.float()).chunk(2, -1)
    return KC._res(out, v * torch.nn.functional.gelu(g))["ok"]


OLD = {
    "odometer_early": lambda K: _old_conv(K),
    "concat_late": lambda K: _old_gemm(K, concat=True),
    "image_ignored": lambda K: _old_conv(K),
    "panel_py_px_swapped": lambda K: _old_upsample(K),
    "third_tap_unshifted": lambda K: _old_upsample(K, 5, 7),
    "rv_mod_ignored": lambda K: _old_gemm(K, residual=False, rowvec=True, Kd=64),
    "ldrv_as_n": lambda K: _old_gemm(K, residual=False, rowvec=True, Kd=64),
    "geglu_granule_64": lambda K: _old_geglu(K),
    "bias_fp16": lambda K: _old_gemm(K),
    "operands_bf16": lambda K: _old_gemm(K),
    "kblock_fp16": lambda K: _old_gemm(K),
    "residual_before_rounding": lambda K: _old_gemm(K, N=64, direct=True),
}

# What the random-input comparator says about each planted bug (True = it lets the bug through).
OLD_PASSES = {
    "odometer_early": False,
    "concat_late": False,
    "image_ignored": False,
    "panel_py_px_swapped": False,
    "third_tap_unshifted": False,
    "rv_mod_ignored": False,
    "ldrv_as_n": False,
    "geglu_granule_64": False,
    "bias_fp16": True,
    "operands_bf16": True,
    "kblock_fp16": True,
    "residual_before_rounding": True,
}


def test_old_comparator_passes_the_correct_emulation():
    for name, check in OLD.items():
        assert check(E()), name


@pytest.mark.parametrize("bug", sorted(OLD))
def test_old_comparator_verdict(bug):
    """The recorded verdict of the random-input comparator on each planted bug holds."""
    assert OLD[bug](E(bug)) == OLD_PASSES[bug], f"{bug}: the random-input comparator {'passes' if not OLD_PASSES[bug] else 'rejects'} it"
