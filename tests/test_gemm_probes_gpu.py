"""Per-element probes of gemm_tc_kernel on an H100 (pytest -m gpu; inputs, references and comparators in
tests/gemm_probes.py).  Integer-exact products over every BLOCK_N, ragged M and K, concats, row-vector table slices,
in-place residuals, row-statistics slices, every conv-tile geometry of the 64x64, 56x96 and 45x60 latents, the skip
concats, the sub-pixel up-samplers (odd sizes too), the stride-2 convs and conv_in, held to an error of exactly 0 and
bit-identical across tile widths, grid caps and ring depths; one-hot precision probes bit-exact against the epilogue's
own rounding order on the staged and the direct-store path; GEGLU and quick-GELU on integer pre-activations within the
activations' claimed error.  Run with -s to see the activations' worst err / bound and the subnormal record."""
import pytest
import torch
import torch.nn.functional as F

from tests import downsample_checks as DC
from tests import gemm_probes as P
from videoswap_b200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ptr(t):
    return 0 if t is None else t.data_ptr()


class Kernel:
    """The gemm_probes backend over the library: ops.gemm / ops.conv3x3 where they reach the arguments, else the
    descriptor entry point (rv_mod, forced BLOCK_N of a conv, strided output and residual views)."""

    pack_conv3x3 = staticmethod(ops.pack_conv3x3)
    pack_conv_subpixel = staticmethod(ops.pack_conv_subpixel)
    pack_geglu = staticmethod(ops.pack_geglu)

    @staticmethod
    def gemm(A, W, bias=None, A2=None, rowvec=None, ppb=1, rv_mod=0, residual=None, out=None, ln_sums=None, bn=0,
             mode=P.LINEAR):
        M, K1 = A.shape
        N = W.shape[0]
        if out is None:
            out = torch.empty((M, N // 2 if mode == P.GEGLU else N), dtype=torch.float16, device=A.device)
        if not rv_mod and out.is_contiguous() and (residual is None or residual.is_contiguous()):
            return ops.gemm(A, W, bias=bias, residual=residual, A2=A2, rowvec=rowvec, pix_per_batch=ppb, mode=mode,
                            force_bn=bn, out=out, ln_sums=ln_sums)
        K2 = 0 if A2 is None else A2.shape[1]
        ops._gemm_ex(A=_ptr(A), K1=K1, lda1=K1, A2=_ptr(A2), K2=K2, lda2=K2, Bw=_ptr(W), M=M, N=N, bias=_ptr(bias),
                     rowvec=_ptr(rowvec), ldrv=0 if rowvec is None else rowvec.stride(0), pix_per_batch=ppb, rv_mod=rv_mod,
                     ln_sums_out=_ptr(ln_sums), residual=_ptr(residual), ldr=0 if residual is None else residual.stride(0),
                     out=_ptr(out), ldc=out.stride(0), mode=mode, force_bn=bn)
        return out

    @staticmethod
    def conv3x3(x, wp, bias=None, x2=None, rowvec=None, ppb=1, rv_mod=0, residual=None, out=None, bn=0):
        n, H, W, C1 = x.shape
        co = wp.shape[0]
        if not bn and not rv_mod and ppb % (H * W) == 0:
            return ops.conv3x3(x, wp, bias=bias, x2=x2, rowvec=rowvec, imgs_per_batch=ppb // (H * W), residual=residual,
                               out=out)
        if out is None:
            out = torch.empty((n, H, W, co), dtype=torch.float16, device=x.device)
        C2 = 0 if x2 is None else x2.shape[3]
        ops._gemm_ex(A=_ptr(x), K1=C1, lda1=C1, A2=_ptr(x2), K2=C2, lda2=C2, Bw=_ptr(wp), M=n * H * W, N=co, taps=9,
                     nimg=n, H=H, W=W, bias=_ptr(bias), rowvec=_ptr(rowvec), ldrv=0 if rowvec is None else rowvec.stride(0),
                     pix_per_batch=ppb, rv_mod=rv_mod, residual=_ptr(residual), ldr=co, out=_ptr(out), ldc=co, force_bn=bn)
        return out

    @staticmethod
    def upsample_sized(x, w, bias, OH, OW):
        return ops.upsample_conv3x3_sized(x, w, bias, OH, OW)

    @staticmethod
    def upsample_packed(x, wsub, bias):
        return ops.upsample_conv3x3_packed(x, wsub, bias)

    @staticmethod
    def upsample(x, w, bias):
        return ops.upsample_conv3x3(x, w, bias)


K = Kernel()


def _check(r):
    assert r["ok"] and r["err"] == 0, f"err {r['err']:.4g}: {r['what']}"


# ---------------------------------------------------------------------------------------------------- integer-exact
M_RAG = 128 * 5 + 77
LINEAR_CASES = {
    # every BLOCK_N, forced and automatic, with a row-vector table slice and a separate residual
    **{f"bn{bn}_rowvec_residual": (lambda bn=bn: P.int_linear(K, DEV, M_RAG, 640, 320, bn=bn, rowvec=True, residual="sep",
                                                                seed=100 + bn)) for bn in (0, 64, 128, 160, 256)},
    # partial last column tiles
    "n96_partial_tile": lambda: P.int_linear(K, DEV, 1025, 96, 320, seed=110),
    "n224_partial_tile": lambda: P.int_linear(K, DEV, 1025, 224, 320, residual="sep", seed=111),
    "n768_bn256": lambda: P.int_linear(K, DEV, 1101, 768, 320, bn=256, seed=112),
    "n224_bn256": lambda: P.int_linear(K, DEV, 300, 224, 64, bn=256, seed=113),
    # M < 128 (77 text rows: the cross-attention K / V), ragged M, M = 131072
    "m77_k768_kv": lambda: P.int_linear(K, DEV, 77, 1280, 768, seed=114),
    "m1_k320": lambda: P.int_linear(K, DEV, 1, 320, 320, residual="sep", seed=115),
    "m129_ragged": lambda: P.int_linear(K, DEV, 129, 320, 320, rowvec=True, seed=116),
    "m131072_k64": lambda: P.int_linear(K, DEV, 131072, 320, 64, rowvec=True, residual="sep", seed=117),
    # K not a multiple of 64 (TMA zero fill of the last k-block) and the product's K
    **{f"k{kd}": (lambda kd=kd: P.int_linear(K, DEV, M_RAG, 320, kd, residual="sep", seed=120 + kd))
       for kd in (8, 72, 200, 64, 320, 768, 1280, 5120)},
    # concat A | A2
    "concat_640_320": lambda: P.int_linear(K, DEV, 300, 640, 640, K2=320, residual="sep", seed=130),
    "concat_1280_1280_bn160": lambda: P.int_linear(K, DEV, M_RAG, 1280, 1280, K2=1280, bn=160, seed=131),
    # per-frame row vectors: (row // 64) % 3 of a table slice
    "rowvec_rv_mod": lambda: P.int_linear(K, DEV, M_RAG, 320, 320, rowvec=True, rv_mod=3, seed=132),
    "rowvec_rv_mod_bn256_residual": lambda: P.int_linear(K, DEV, M_RAG, 768, 320, bn=256, rowvec=True, rv_mod=5,
                                                         residual="sep", seed=133),
    # residual is out (the transformer's out-projections), with and without the row-statistics slices at every BN
    "inplace_residual": lambda: P.int_linear(K, DEV, M_RAG, 320, 320, residual="inplace", seed=134),
    **{f"inplace_ln_sums_bn{bn}": (lambda bn=bn: P.int_linear(K, DEV, M_RAG, 640, 64, bn=bn, residual="inplace",
                                                              ln_sums=True, density=0.125, seed=140 + bn))
       for bn in (0, 64, 128, 160, 256)},
    "ln_sums_n320_bn256": lambda: P.int_linear(K, DEV, 1101, 320, 64, bn=256, ln_sums=True, density=0.125, seed=150),
}


@pytest.mark.parametrize("name", sorted(LINEAR_CASES))
def test_gemm_integer_exact(name):
    _check(LINEAR_CASES[name]())


# every pick_conv_tile geometry the UNet's convs use: the level sizes of the 64x64, 56x96 and odd 45x60 latents at 2 .. 32
# images (TN > 1 tiles straddle image seams; TW / TH boxes overhang the right and bottom borders), and 1x1
CONV_LEVELS = [(2, 64, 64), (4, 32, 32), (16, 16, 16), (32, 8, 8), (2, 56, 96), (4, 28, 48), (16, 14, 24), (32, 7, 12),
               (2, 45, 60), (16, 45, 60), (3, 23, 30), (32, 23, 30), (32, 12, 15), (3, 12, 15), (3, 6, 8), (32, 6, 8),
               (3, 1, 1), (32, 1, 1)]
CONV_CASES = {
    **{f"level_{n}x{h}x{w}": (lambda n=n, h=h, w=w: P.int_conv(K, DEV, n, h, w, 64, 64, rowvec=True, F_=2, residual=True,
                                                               seed=200 + n + h + w)) for n, h, w in CONV_LEVELS},
    # the skip concats of the up path, at the levels they run on
    "concat_1280_1280": lambda: P.int_conv(K, DEV, 2, 8, 8, 1280, 1280, c2=1280, seed=240),
    "concat_1280_640": lambda: P.int_conv(K, DEV, 2, 16, 16, 1280, 640, c2=640, rowvec=True, residual=True, seed=241),
    "concat_640_320": lambda: P.int_conv(K, DEV, 2, 32, 32, 640, 320, c2=320, seed=242),
    "concat_320_320": lambda: P.int_conv(K, DEV, 2, 45, 60, 320, 320, c2=320, rowvec=True, F_=1, seed=243),
    # resnet conv with the time-embedding row (one per 16 frames) and the residual
    "temb_rowvec_16_frames": lambda: P.int_conv(K, DEV, 32, 8, 8, 640, 640, rowvec=True, F_=16, residual=True, seed=244),
    # conv_out: N = 4 and 8 on the direct-store path
    "conv_out_n4": lambda: P.int_conv(K, DEV, 2, 45, 60, 320, 4, seed=245),
    "conv_out_n8_residual": lambda: P.int_conv(K, DEV, 3, 23, 30, 64, 8, residual=True, seed=246),
}


@pytest.mark.parametrize("name", sorted(CONV_CASES))
def test_conv_integer_exact(name):
    _check(CONV_CASES[name]())


UPSAMPLE_CASES = {
    "plain_2x8x8": lambda: P.int_subpixel(K, DEV, 2, 8, 8, 64, 64, how="plain", seed=300),
    "plain_3x7x12": lambda: P.int_subpixel(K, DEV, 3, 7, 12, 128, 64, how="plain", seed=301),
    "packed_2x4x4": lambda: P.int_subpixel(K, DEV, 2, 4, 4, 64, 64, how="packed", seed=302),
    "packed_2x14x24": lambda: P.int_subpixel(K, DEV, 2, 14, 24, 64, 320, how="packed", seed=303),
    "sized_even_2x16x16": lambda: P.int_subpixel(K, DEV, 2, 16, 16, 64, 64, seed=304),
    # the 45x60 chain: 6x8 -> 12x15 (columns odd), 12x15 -> 23x30 (rows odd), 23x30 -> 45x60 (rows odd); both odd
    "sized_6x8_to_12x15": lambda: P.int_subpixel(K, DEV, 2, 6, 8, 64, 64, 12, 15, seed=305),
    "sized_12x15_to_23x30": lambda: P.int_subpixel(K, DEV, 2, 12, 15, 64, 64, 23, 30, seed=306),
    "sized_23x30_to_45x60": lambda: P.int_subpixel(K, DEV, 2, 23, 30, 64, 64, 45, 60, seed=307),
    "sized_12x8_to_23x15": lambda: P.int_subpixel(K, DEV, 3, 12, 8, 128, 64, 23, 15, seed=308),
    "sized_1x1_to_1x1": lambda: P.int_subpixel(K, DEV, 2, 1, 1, 64, 64, 1, 1, seed=309),
}


@pytest.mark.parametrize("name", sorted(UPSAMPLE_CASES))
def test_upsampler_integer_exact(name):
    _check(UPSAMPLE_CASES[name]())


@pytest.mark.parametrize("n,H,W", [(2, 16, 16), (2, 23, 30), (3, 45, 60), (2, 1, 1)])
def test_unet_downsampler_integer_exact(n, H, W):
    """The UNet's stride-2 down-sampler: im2col_s2 + the GEMM (pad 1 on every side), even and odd H, W."""
    x = P.ternary((n, H, W, 64), 400 + H).to(DEV)
    w = P.ternary((128, 64, 3, 3), 401 + H).to(DEV)
    b = P.halves((128,), 402 + H).to(DEV)
    out = ops.conv3x3_s2(x, ops.pack_conv3x3(w), b)
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), b.double(), stride=2, padding=1).permute(0, 2, 3, 1)
    _check(P.exact(out, ref, f"conv3x3_s2 {n}x{H}x{W}"))


def test_vae_downsampler_integer_exact():
    """The VAE encoder's implicit stride-2 conv (parity views, right / bottom padding): a cross-check of its probes."""
    x = P.ternary((2, 24, 40, 128), 410).to(DEV)
    w = P.ternary((128, 128, 3, 3), 411).to(DEV)
    b = P.halves((128,), 412).to(DEV)
    out = ops.downsample_conv3x3(x, ops.pack_conv3x3(w), b)
    ref, _ = DC.reference(x, w, b)
    _check(P.exact(out, ref, "VAE down-sampler 2x24x40"))


@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("n,H,W", [(2, 64, 64), (3, 45, 60), (1, 1, 1)])
def test_conv_in_integer_exact(n, H, W, tc):
    """conv_in: patch rows + the tensor-core GEMM, and the direct CUDA-core kernel."""
    x = P.ternary((n, H, W, 4), 420 + H, 0.5).to(DEV)
    w = P.ternary((320, 4, 3, 3), 421 + H, 0.5).to(DEV)
    b = P.halves((320,), 422 + H).to(DEV)
    out = ops.conv_in(x, w, b) if tc else ops.conv_in(x, w, b, scratch=None)
    _check(P.exact(out, P.conv64(x, w) + b.double(), f"conv_in {'tensor-core' if tc else 'direct'} {n}x{H}x{W}"))


# ---------------------------------------------------------------------------------------------------- invariance
def _configs(bns):
    for bn in bns:
        for stages in (0, 3):
            for ctas in (1, 3, 8):
                yield bn, stages, ctas


INVARIANT = {
    "gemm_rowvec_residual": (lambda bn: P.int_linear(K, DEV, M_RAG, 640, 1280, bn=bn, rowvec=True, residual="sep",
                                                     seed=500), (64, 128, 160, 256)),
    "gemm_concat_inplace_ln_sums": (lambda bn: P.int_linear(K, DEV, 1101, 640, 64, K2=64, bn=bn, residual="inplace",
                                                            ln_sums=True, density=0.125, seed=501), (64, 128, 160, 256)),
    "conv_concat_rowvec_residual": (lambda bn: P.int_conv(K, DEV, 3, 12, 15, 320, 320, c2=320, bn=bn, rowvec=True,
                                                          residual=True, seed=502), (64, 128, 160, 256)),
    "upsampler_23x30_to_45x60": (lambda bn: P.int_subpixel(K, DEV, 2, 23, 30, 64, 320, 45, 60, seed=503), (0,)),
}


@pytest.mark.parametrize("name", sorted(INVARIANT))
def test_exact_across_tile_width_grid_and_ring(name):
    """Exact results cannot depend on the schedule: every valid BLOCK_N x gemm_ctas 1 / 3 / 8 x gemm_stages 0 / 3."""
    run, bns = INVARIANT[name]
    try:
        for bn, stages, ctas in _configs(bns):
            ops.set_option("gemm_stages", stages)
            ops.set_option("gemm_ctas", ctas)
            r = run(bn)
            assert r["ok"] and r["err"] == 0, f"bn {bn} gemm_stages {stages} gemm_ctas {ctas}: {r['what']}"
    finally:
        ops.set_option("gemm_ctas", 0)
        ops.set_option("gemm_stages", 0)


# ---------------------------------------------------------------------------------------------------- one-hot probes
ONEHOT_CASES = {
    "m300_k320_n320": lambda: P.onehot_linear(K, DEV, 300, 320, 320, seed=600),
    "m77_k768_n768": lambda: P.onehot_linear(K, DEV, 77, 768, 768, seed=601),
    "m1101_k72_n96": lambda: P.onehot_linear(K, DEV, 1101, 72, 96, seed=602),
    "m130_k8_n64": lambda: P.onehot_linear(K, DEV, 130, 8, 64, seed=603),
    "m517_k1280_n640_bn160": lambda: P.onehot_linear(K, DEV, 517, 1280, 640, bn=160, seed=604),
    "m257_k5120_n1280": lambda: P.onehot_linear(K, DEV, 257, 5120, 1280, seed=605),
    "m717_k320_n768_bn256_rv_mod": lambda: P.onehot_linear(K, DEV, M_RAG, 320, 768, bn=256, rv_mod=3, seed=606),
    "m717_k200_n256_bn64": lambda: P.onehot_linear(K, DEV, M_RAG, 200, 256, bn=64, seed=607),
    # the direct-store epilogue: N not a multiple of 32, and an output 8 bytes off a 16-byte boundary
    "direct_n40": lambda: P.onehot_linear(K, DEV, M_RAG, 320, 40, seed=610),
    "direct_misaligned_out": lambda: P.onehot_linear(K, DEV, M_RAG, 320, 320, direct=True, seed=611),
    "direct_misaligned_out_rv_mod_bn256": lambda: P.onehot_linear(K, DEV, 300, 64, 256, bn=256, rv_mod=3, direct=True,
                                                                  seed=612),
    "direct_n40_no_residual": lambda: P.onehot_linear(K, DEV, 300, 64, 40, residual=False, seed=613),
    # two terms in the first and the last k-block per shape
    **{f"two_term_m{m}_k{kd}_n{n}": (lambda m=m, kd=kd, n=n: P.two_term(K, DEV, m, kd, n, seed=620 + kd))
       for m, kd, n in ((300, 320, 320), (77, 768, 768), (1101, 72, 96), (517, 1280, 640), (257, 5120, 1280),
                        (M_RAG, 200, 40))},
    # every (tap, channel) of a conv panel, borders reading their neighbour or the zero fill exactly
    "conv_2x45x60": lambda: P.onehot_conv(K, DEV, 2, 45, 60, 64, seed=630),
    "conv_3x6x8": lambda: P.onehot_conv(K, DEV, 3, 6, 8, 64, seed=631),
    "conv_32x7x12": lambda: P.onehot_conv(K, DEV, 32, 7, 12, 64, residual=False, seed=632),
    "conv_3x1x1": lambda: P.onehot_conv(K, DEV, 3, 1, 1, 64, seed=633),
    # every tap of every parity of the up-sampler, the third tap of an odd axis through the shifted view
    "upsampler_6x8_to_12x15": lambda: P.onehot_subpixel(K, DEV, 2, 6, 8, 64, 12, 15, seed=640),
    "upsampler_12x15_to_23x30": lambda: P.onehot_subpixel(K, DEV, 2, 12, 15, 64, 23, 30, seed=641),
    "upsampler_23x30_to_45x60": lambda: P.onehot_subpixel(K, DEV, 1, 23, 30, 64, 45, 60, seed=642),
    "upsampler_12x8_to_23x15": lambda: P.onehot_subpixel(K, DEV, 2, 12, 8, 64, 23, 15, seed=643),
    "upsampler_8x8_to_16x16": lambda: P.onehot_subpixel(K, DEV, 2, 8, 8, 64, 16, 16, seed=644),
}


@pytest.mark.parametrize("name", sorted(ONEHOT_CASES))
def test_one_hot_bit_exact(name):
    _check(ONEHOT_CASES[name]())


def test_subnormal_a_record():
    """Whether subnormal fp16 A values reach the tensor cores unflushed: recorded (run with -s), not asserted; normal
    rows of the same launch must be exact."""
    sub_ok, normal_ok = P.subnormal_probe(K, DEV)
    print(f"\nsubnormal fp16 A values honoured exactly: {sub_ok}")
    assert normal_ok


# ---------------------------------------------------------------------------------------------------- activations
@pytest.mark.parametrize("C", [320, 640, 1280])
def test_geglu_integer_preactivations(C):
    r = P.geglu_case(K, DEV, 128 * 3 + 77, C, seed=700 + C)
    print(f"\nGEGLU C {C}: worst err / bound {r['err']:.3g}")
    assert r["ok"], r


@pytest.mark.parametrize("bn", [128, 256])
def test_quick_gelu_integer_preactivations(bn):
    r = P.qgelu_case(K, DEV, 128 * 2 + 77, bn, seed=710 + bn)
    print(f"\nquick-GELU BLOCK_N {bn}: worst err / bound {r['err']:.3g}")
    assert r["ok"], r
