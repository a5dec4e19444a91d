"""The epilogue-slot instantiations (gemm_tc_kernel<BN, EPI, GemmParamsEpi>), K <= 640: the linears at BLOCK_N 128 / 160
with the RES, LNOUT, LNOUT + RES, LN and LN + RV epilogues and the cooperative GEGLUs (BLOCK_N 256, with and without a
folded LayerNorm), operands fetched into shared memory during the main loop.

Every case checks which instantiation ran (kernel names from torch.profiler) and holds the output to an exact
reference: integer-exact products and epilogue operands (tests/gemm_probes.py), or, where the epilogue itself rounds
(the LayerNorm statistics from partial sums, random fp16 data), bit for bit to the same launch with the slots switched
off (`gemm_epi_slot` 0), which is the epilogue that reads its operands from global memory."""
import pytest
import torch

from tests import gemm_probes as P
from tests.test_gemm_probes_gpu import K
from videoswap_b200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _gemm_kernels(fn):
    """Runs fn once under the profiler; returns (fn's result, names of the gemm_tc_kernel launches)."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        r = fn()
        torch.cuda.synchronize()
    return r, [e.name for e in prof.events() if "gemm_tc_kernel" in e.name]


def _slot_ran(names, bn):
    return len(names) == 1 and "GemmParamsEpi" in names[0] and f"<{bn}," in names[0].replace(" ", "")


def _no_slot(fn):
    ops.set_option("gemm_epi_slot", 0)
    try:
        return fn()
    finally:
        ops.set_option("gemm_epi_slot", 1)


# ---------------------------------------------------------------------------------------------------- integer-exact
INT_CASES = {
    **{f"res_bn{bn}": (bn, lambda bn=bn: P.int_linear(K, DEV, 128 * 9 + 77, 320, 320, bn=bn, residual="sep", seed=600 + bn))
       for bn in (128, 160)},
    **{f"lnout_bn{bn}": (bn, lambda bn=bn: P.int_linear(K, DEV, 128 * 9 + 77, 640, 640, bn=bn, ln_sums=True,
                                                        density=0.125, seed=610 + bn)) for bn in (128, 160)},
    **{f"lnout_inplace_res_bn{bn}": (bn, lambda bn=bn: P.int_linear(K, DEV, 128 * 9 + 77, 640, 320, bn=bn,
                                                                    residual="inplace", ln_sums=True, density=0.125,
                                                                    seed=620 + bn)) for bn in (128, 160)},
    # the last row tile holds 1 and 127 rows
    **{f"ragged_m{m}_bn{bn}": (bn, lambda m=m, bn=bn: P.int_linear(K, DEV, m, 320, 320, bn=bn, residual="inplace",
                                                                   ln_sums=True, density=0.125, seed=630 + m + bn))
       for m in (128 * 5 + 1, 128 * 5 + 127, 1) for bn in (128, 160)},
    # N not a multiple of BLOCK_N: the last column tile fetches fewer columns
    "partial_column_tile_bn128": (128, lambda: P.int_linear(K, DEV, 1025, 320, 320, bn=128, residual="sep", seed=640)),
}


@pytest.mark.parametrize("name", sorted(INT_CASES))
def test_slot_integer_exact(name):
    bn, case = INT_CASES[name]
    r, names = _gemm_kernels(case)
    assert _slot_ran(names, bn), names
    assert r["ok"] and r["err"] == 0, f"err {r['err']:.4g}: {r['what']}"


def _ln_case(M, N, Kd, bn, ppb=0, rv_mod=0, parts=0, seed=0, random=False):
    """Folded-LayerNorm GEMM out = la * acc + (lb * u + c) (+ rowvec[(row // ppb) % rv_mod]) through the descriptor.
    Integer data: la in {1/2, 1, 2}, lb, u, c, row vectors halves, ternary A and W, so every step is exact in fp32 and the
    fp64 reference is the answer.  parts > 0: the statistics come from `parts` (sum, sum of squares) slices instead
    (no exact reference: compared against the slot-less launch).  Returns (reference or None, launch, output buffer)."""
    g = torch.Generator().manual_seed(seed)
    if random:
        A = (torch.randn(M, Kd, generator=g) * 0.7).half().to(DEV)
        W = (torch.randn(N, Kd, generator=g) / Kd ** 0.5).half().to(DEV)
    else:
        A, W = P.ternary((M, Kd), seed, 0.125).to(DEV), P.ternary((N, Kd), seed + 1, 0.125).to(DEV)
    u, c = P.halves((N,), seed + 2).to(DEV), P.halves((N,), seed + 3).to(DEV)
    la = torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (M,), generator=g)]
    lb = P.halves((M,), seed + 4)
    stats = torch.stack([la, lb], 1).contiguous().to(DEV)
    lparts = None
    if parts:
        S = torch.randn(parts, M, generator=g) * 4
        Q = (S * S / 4 + torch.rand(parts, M, generator=g) * Kd / parts)
        lparts = torch.stack([S, Q], 2).contiguous().to(DEV)
    rv = P.table_slice(rv_mod, N, seed + 5, DEV) if ppb else None
    buf = P.nan16((M + 70, N + 64), DEV)
    out = buf[:M, 32:32 + N]

    def launch():
        out.fill_(float("nan"))
        ops._gemm_ex(A=A.data_ptr(), K1=Kd, lda1=Kd, Bw=W.data_ptr(), M=M, N=N, bias=c.data_ptr(), ln_u=u.data_ptr(),
                     ln_stats=0 if parts else stats.data_ptr(), ln_parts=lparts.data_ptr() if parts else 0,
                     ln_nparts=parts, rowvec=rv.data_ptr() if ppb else 0, ldrv=rv.stride(0) if ppb else 0,
                     pix_per_batch=ppb or 1, rv_mod=rv_mod, out=out.data_ptr(), ldc=out.stride(0), force_bn=bn)
        return out.clone()

    ref = None
    if not parts and not random:
        acc = A.double() @ W.double().t()
        ref = la.double().to(DEV)[:, None] * acc + lb.double().to(DEV)[:, None] * u.double() + c.double()
        if ppb:
            ref = ref + rv.double()[(torch.arange(M, device=DEV) // ppb) % rv_mod]
    return ref, launch, buf


# The slots take the LayerNorm rows of an even M (every tile's rows of every slice start 16-byte aligned); the last row
# tile of these holds 2, 78 or 126 rows.
LN_INT = {
    **{f"ln_stats_bn{bn}": (bn, dict(M=128 * 9 + 78, N=960, Kd=320, bn=bn, seed=700 + bn)) for bn in (128, 160)},
    # one frame per tile (256 rows a frame) and two (64 rows a frame), per-frame rows of a table slice
    **{f"ln_rv_ppb{ppb}_bn{bn}": (bn, dict(M=128 * 9 + 78, N=640, Kd=640, bn=bn, ppb=ppb, rv_mod=3, seed=710 + bn + ppb))
       for ppb in (64, 256) for bn in (128, 160)},
    "ln_rv_ragged_m2_bn160": (160, dict(M=128 * 4 + 2, N=320, Kd=320, bn=160, ppb=64, rv_mod=5, seed=720)),
    "ln_stats_ragged_m126_bn128": (128, dict(M=128 * 4 + 126, N=320, Kd=320, bn=128, seed=721)),
}


@pytest.mark.parametrize("name", sorted(LN_INT))
def test_slot_layernorm_integer_exact(name):
    bn, kw = LN_INT[name]
    ref, launch, buf = _ln_case(**kw)
    out, names = _gemm_kernels(launch)
    assert _slot_ran(names, bn), names
    M, N = kw["M"], kw["N"]
    r = P.merge(P.exact(out, ref, name), P.untouched(buf, (slice(0, M), slice(32, 32 + N)), name))
    assert r["ok"] and r["err"] == 0, f"err {r['err']:.4g}: {r['what']}"


@pytest.mark.parametrize("bn", [128, 160])
@pytest.mark.parametrize("parts", [1, 2, 4])
@pytest.mark.parametrize("M", [128 * 6 + 2, 128 * 6 + 126])
def test_slot_layernorm_parts_bitwise(M, parts, bn):
    _, launch, _ = _ln_case(M, 640, 640, bn, ppb=64 if parts == 2 else 0, rv_mod=4, parts=parts, seed=800 + parts + M)
    out, names = _gemm_kernels(launch)
    assert _slot_ran(names, bn), names
    ref, names0 = _gemm_kernels(lambda: _no_slot(launch))
    assert names0 and not any("GemmParamsEpi" in n for n in names0), names0
    assert torch.isfinite(out).all()
    r = P.bitwise(out, ref, f"ln parts {parts} M {M} bn {bn}")
    assert r["ok"], r["what"]


# ---------------------------------------------------------------------------------------------------- random fp16
def _random_linear(epi, M, N, Kd, bn, seed):
    g = torch.Generator().manual_seed(seed)
    A = (torch.randn(M, Kd, generator=g) * 0.7).half().to(DEV)
    W = (torch.randn(N, Kd, generator=g) / Kd ** 0.5).half().to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    R = torch.randn(M, N, generator=g).half().to(DEV)
    out = torch.empty(M, N, dtype=torch.float16, device=DEV)
    sums = torch.empty(ops.max_column_tiles(N, bn), M, 2, device=DEV)

    def launch():
        out.copy_(R)                                     # in-place residual, as the UNet's out-projections
        sums.fill_(float("nan"))
        ops.gemm(A, W, bias=b, residual=out if "RES" in epi else None, out=out, force_bn=bn,
                 ln_sums=sums if "LNOUT" in epi else None)
        return torch.cat([out.view(torch.int16).flatten().float(), sums.flatten()]) if "LNOUT" in epi else out.clone()
    return launch


@pytest.mark.parametrize("epi", ["RES", "LNOUT", "LNOUT+RES", "LN", "LN+RV"])
@pytest.mark.parametrize("bn", [128, 160])
def test_slot_random_fp16_equals_global_epilogue(epi, bn):
    """Random fp16 operands at a ragged M: the slot instantiation and the slot-less one give the same bits."""
    M, N, Kd = 128 * 40 + 78, 640, 320
    if epi.startswith("LN") and "OUT" not in epi:
        _, launch, _ = _ln_case(M, N, Kd, bn, ppb=64 if "RV" in epi else 0, rv_mod=16, parts=2, seed=900 + bn,
                                random=True)
    else:
        launch = _random_linear(epi, M, N, Kd, bn, 910 + bn)
    out, names = _gemm_kernels(launch)
    assert _slot_ran(names, bn), names
    ref, names0 = _gemm_kernels(lambda: _no_slot(launch))
    assert names0 and not any("GemmParamsEpi" in n for n in names0), names0
    if out.dtype == torch.float16:
        assert torch.isfinite(out).all()
        r = P.bitwise(out, ref, f"{epi} bn {bn}")
        assert r["ok"], r["what"]
    else:
        assert torch.equal(out.view(torch.int32), ref.view(torch.int32)), f"{epi} bn {bn}: output or row sums differ"


def test_long_k_keeps_its_instantiation():
    """K = 1280 (20 k-blocks) is not a short-K linear: it keeps the slot-less kernel."""
    launch = _random_linear("LNOUT+RES", 1024, 640, 1280, 160, 950)
    _, names = _gemm_kernels(launch)
    assert names and not any("GemmParamsEpi" in n for n in names), names


def test_layernorm_odd_m_keeps_its_instantiation():
    """An odd M would leave the LayerNorm rows of a slice 8-byte aligned: such a launch keeps the slot-less kernel."""
    kw = dict(M=128 * 4 + 77, N=320, Kd=320, bn=160, seed=960)
    ref, launch, buf = _ln_case(**kw)
    out, names = _gemm_kernels(launch)
    assert names and not any("GemmParamsEpi" in n for n in names), names
    r = P.exact(out, ref, "ln odd M")
    assert r["ok"] and r["err"] == 0, f"err {r['err']:.4g}: {r['what']}"


@pytest.mark.parametrize("ln", [False, True])
@pytest.mark.parametrize("C,M", [(320, 128 * 30 + 78), (640, 128 * 12 + 2)])
def test_slot_geglu_random_fp16_equals_global_epilogue(C, M, ln):
    """GEGLU [M, C] -> [M, 4 C] from a packed [8 C, C] weight (bias, and with ln the LayerNorm from two partial slices):
    the slot instantiation and the slot-less one give the same bits, on more tiles than a wave so both slots cycle."""
    g = torch.Generator().manual_seed(970 + C + ln)
    A = (torch.randn(M, C, generator=g) * 0.7).half().to(DEV)
    W = (torch.randn(8 * C, C, generator=g) / C ** 0.5).half().to(DEV)
    b, u = torch.randn(8 * C, generator=g).to(DEV), torch.randn(8 * C, generator=g).to(DEV)
    S = torch.randn(2, M, generator=g) * 4
    lparts = torch.stack([S, S * S / 4 + torch.rand(2, M, generator=g) * C / 2], 2).contiguous().to(DEV)
    out = torch.empty(M, 4 * C, dtype=torch.float16, device=DEV)

    def launch():
        out.fill_(float("nan"))
        ops._gemm_ex(A=A.data_ptr(), K1=C, lda1=C, Bw=W.data_ptr(), M=M, N=8 * C, bias=b.data_ptr(),
                     ln_u=u.data_ptr() if ln else 0, ln_parts=lparts.data_ptr() if ln else 0, ln_nparts=2 if ln else 0,
                     out=out.data_ptr(), ldc=4 * C, mode=ops.EPI_GEGLU)
        return out.clone()
    got, names = _gemm_kernels(launch)
    assert _slot_ran(names, 256), names
    ref, names0 = _gemm_kernels(lambda: _no_slot(launch))
    assert names0 and not any("GemmParamsEpi" in n for n in names0), names0
    assert torch.isfinite(got).all()
    r = P.bitwise(got, ref, f"geglu C {C} M {M} ln {ln}")
    assert r["ok"], r["what"]
