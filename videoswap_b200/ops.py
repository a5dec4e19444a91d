"""Thin torch-tensor wrappers over the per-kernel C-ABI entry points (torch is only used for device memory and the
current stream).  All activations are NHWC fp16 CUDA tensors.  Used by the parity tests and the host-side model."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib

GEGLU_GRANULE = 128
EPI_LINEAR, EPI_GEGLU, EPI_QUICK_GELU, EPI_RELU = 0, 1, 2, 3


def set_option(name: str, value: int):
    """Runtime options of the library, e.g. set_option("attn_tc", 0) forces the mma.sync attention kernel."""
    _lib.call("vs_set_option", name.encode(), int(value))


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _chk16(*ts):
    for t in ts:
        if t is not None:
            assert t.is_cuda and t.dtype == torch.float16 and t.is_contiguous(), "expected contiguous fp16 CUDA tensor"


def _chk32(*ts):
    for t in ts:
        if t is not None:
            assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), "expected contiguous fp32 CUDA tensor"


def _ptr(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def _out16(out, shape, device):
    """The caller's output tensor (checked) or a new one."""
    if out is None:
        return torch.empty(shape, dtype=torch.float16, device=device)
    _chk16(out)
    assert tuple(out.shape) == tuple(shape), f"out has shape {tuple(out.shape)}, expected {tuple(shape)}"
    return out


def _chk_rowvec(rv, N):
    """fp32 [rows, N] with unit column stride: a whole table or a column slice of a wider one (row stride = ldrv)."""
    if rv is not None:
        assert rv.is_cuda and rv.dtype == torch.float32 and rv.dim() == 2 and rv.shape[1] == N and rv.stride(1) == 1, \
            "expected an fp32 [rows, N] CUDA row-vector table with unit column stride"


def max_column_tiles(N, force_bn=0):
    """Upper bound on the column tiles of a GEMM (= LayerNorm partial-sum slices it writes): the automatic tile width is
    64 for N <= 64 and at least 128 otherwise."""
    bn = force_bn or (64 if N <= 64 else 128)
    return -(-N // bn)


def _gemm_ex(**fields):
    d = _lib.GemmDescStruct()
    d.taps = 1
    d.pix_per_batch = 1
    for k, v in fields.items():
        setattr(d, k, v)
    _lib.call("vs_gemm_ex", _stream(), C.byref(d))


def gemm(A, W, bias=None, residual=None, A2=None, rowvec=None, pix_per_batch=1, mode=EPI_LINEAR, force_bn=0, out=None,
         ln_sums=None):
    """out[M, N] = [A | A2] @ W^T (+bias +rowvec[row // pix_per_batch] +residual); GEGLU mode expects packed W/bias;
    EPI_QUICK_GELU mode gives quick_gelu(A @ W^T + bias) (bias only).
    out: the caller's [M, N] ([M, N/2] for GEGLU) tensor; it may be `residual` itself (in-place residual add, as the UNet's
    attention output projections run).  rowvec may be a column slice of a wider table.  ln_sums: [slices, M, 2] fp32
    (slices >= max_column_tiles(N, force_bn)) that receives, per column tile, each row's (sum, sum of squares) of the
    stored fp16 outputs."""
    _chk16(A, W, residual, A2)
    _chk32(bias, ln_sums)
    M, K1 = A.shape
    K2 = 0 if A2 is None else A2.shape[1]
    N = W.shape[0]
    assert W.shape[1] == K1 + K2
    _chk_rowvec(rowvec, N)
    oc = N // 2 if mode == EPI_GEGLU else N
    out = _out16(out, (M, oc), A.device)
    if ln_sums is not None:
        assert ln_sums.dim() == 3 and ln_sums.shape[1:] == (M, 2) and ln_sums.shape[0] >= max_column_tiles(N, force_bn)
    _gemm_ex(A=_ptr(A), K1=K1, lda1=K1, A2=_ptr(A2), K2=K2, lda2=K2, Bw=_ptr(W), M=M, N=N, bias=_ptr(bias),
             rowvec=_ptr(rowvec), ldrv=0 if rowvec is None else rowvec.stride(0), pix_per_batch=pix_per_batch,
             ln_sums_out=_ptr(ln_sums), residual=_ptr(residual), ldr=oc, out=_ptr(out), ldc=oc, mode=mode, force_bn=force_bn)
    return out


def pack_conv3x3(w):
    """[Co, Ci, 3, 3] fp16 -> [Co, 9*Ci] tap-major."""
    _chk16(w)
    co, ci = w.shape[:2]
    out = torch.empty((co, 9 * ci), dtype=torch.float16, device=w.device)
    _lib.call("vs_pack_conv3x3", _stream(), _p(w), co, ci, _p(out))
    return out


def pack_geglu(w, b):
    """FeedForward.net.0.proj [8C, C] / [8C] -> value/gate interleaved in GEGLU_GRANULE-row (128) granules (+ fp32 bias)."""
    _chk16(w, b)
    hidden, K = w.shape[0] // 2, w.shape[1]
    wout = torch.empty_like(w)
    bout = torch.empty((2 * hidden,), dtype=torch.float32, device=w.device)
    _lib.call("vs_pack_geglu", _stream(), _p(w), _p(b), hidden, K, _p(wout), _p(bout))
    return wout, bout


def conv3x3(x, w_packed, bias=None, x2=None, rowvec=None, imgs_per_batch=1, residual=None, out=None):
    """x: [N, H, W, C1] (+x2 [N, H, W, C2] channel concat), w_packed [Co, 9*(C1+C2)] -> [N, H, W, Co].
    rowvec[image // imgs_per_batch] is added (may be a column slice of a wider table); out: the caller's output tensor."""
    _chk16(x, w_packed, x2, residual)
    _chk32(bias)
    n, H, W, C1 = x.shape
    C2 = 0 if x2 is None else x2.shape[3]
    co = w_packed.shape[0]
    _chk_rowvec(rowvec, co)
    out = _out16(out, (n, H, W, co), x.device)
    _gemm_ex(A=_ptr(x), K1=C1, lda1=C1, A2=_ptr(x2), K2=C2, lda2=C2, Bw=_ptr(w_packed), M=n * H * W, N=co, taps=9, nimg=n,
             H=H, W=W, bias=_ptr(bias), rowvec=_ptr(rowvec), ldrv=0 if rowvec is None else rowvec.stride(0),
             pix_per_batch=imgs_per_batch * H * W, residual=_ptr(residual), ldr=co, out=_ptr(out), ldc=co)
    return out


def conv3x3_relu(x, w_packed, bias=None, out=None):
    """relu(conv3x3(x) + bias) in the conv's epilogue (one rounding to fp16): x [N, H, W, C] (C % 64 == 0), w_packed
    [Co, 9 C] (Co % 32 == 0) -> [N, H, W, Co]."""
    _chk16(x, w_packed)
    _chk32(bias)
    n, H, W, C1 = x.shape
    co = w_packed.shape[0]
    out = _out16(out, (n, H, W, co), x.device)
    _gemm_ex(A=_ptr(x), K1=C1, lda1=C1, Bw=_ptr(w_packed), M=n * H * W, N=co, taps=9, nimg=n, H=H, W=W, bias=_ptr(bias),
             out=_ptr(out), ldc=co, mode=EPI_RELU)
    return out


def t2i_image_in(frames):
    """uint8 frames [n, H, W, c] (c = 1 or 3; H, W multiples of 8) -> F.pixel_unshuffle(frames / 255 as fp16, 8) in NHWC:
    fp16 [n, H / 8, W / 8, 64 c], channel c' 64 + 8 i + j = pixel (8 y + i, 8 x + j) of channel c'."""
    assert frames.is_cuda and frames.dtype == torch.uint8 and frames.is_contiguous() and frames.dim() == 4, \
        "expected contiguous uint8 [n, H, W, c] CUDA frames"
    assert frames.data_ptr() % 8 == 0, "frames must be 8-byte aligned"
    n, H, W, c = frames.shape
    out = torch.empty((n, H // 8, W // 8, 64 * c), dtype=torch.float16, device=frames.device)
    _lib.call("vs_t2i_image_in", _stream(), _p(frames), n, H, W, c, _p(out))
    return out


def avgpool2x2(x):
    """AvgPool2d(2, stride 2) of x [N, H, W, C] (H, W even, C % 8 == 0) -> [N, H / 2, W / 2, C], fp32 sum, one rounding."""
    _chk16(x)
    n, H, W, Cc = x.shape
    out = torch.empty((n, H // 2, W // 2, Cc), dtype=torch.float16, device=x.device)
    _lib.call("vs_avgpool2x2", _stream(), _p(x), n, H, W, Cc, _p(out))
    return out


def scale_f16(x, scale, out=None):
    """fp16(fp32(x) * scale), as torch rounds an fp16 tensor times a Python float; out may be x (in place)."""
    _chk16(x)
    assert x.numel() % 8 == 0
    out = _out16(out, tuple(x.shape), x.device)
    _lib.call("vs_scale_f16", _stream(), _p(x), x.numel(), float(scale), _p(out))
    return out


def conv3x3_s2(x, w_packed, bias=None):
    _chk16(x, w_packed)
    n, H, W, Ci = x.shape
    co = w_packed.shape[0]
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    scratch = torch.empty((n * Ho * Wo, 9 * Ci), dtype=torch.float16, device=x.device)
    out = torch.empty((n, Ho, Wo, co), dtype=torch.float16, device=x.device)
    _lib.call("vs_conv3x3_s2", _stream(), _p(x), n, H, W, Ci, _p(w_packed), co, _p(bias), _p(scratch), _p(out))
    return out


def upsample_conv3x3(x, w, bias=None):
    """nearest-2x + conv3x3 (pad 1) as four sub-pixel convs: x [N, H, W, C], w [Co, C, 3, 3] (unpacked) -> [N, 2H, 2W, Co]."""
    _chk16(x, w)
    _chk32(bias)
    n, H, W, Ci = x.shape
    co = w.shape[0]
    wsub = torch.empty((16 * co * Ci,), dtype=torch.float16, device=x.device)
    out = torch.empty((n, 2 * H, 2 * W, co), dtype=torch.float16, device=x.device)
    _lib.call("vs_upsample_conv3x3", _stream(), _p(x), n, H, W, Ci, _p(w), co, _p(bias), _p(wsub), _p(out))
    return out


def pack_conv_subpixel(w):
    """[Co, Ci, 3, 3] fp16 -> the four sub-pixel panels of upsample_conv3x3, [4 parities (py * 2 + px), Co, 4 * Ci]."""
    _chk16(w)
    co, ci = w.shape[:2]
    out = torch.empty((4, co, 4 * ci), dtype=torch.float16, device=w.device)
    _lib.call("vs_pack_conv_subpixel", _stream(), _p(w), co, ci, _p(out))
    return out


def upsample_conv3x3_packed(x, wsub, bias=None):
    """upsample_conv3x3 on panels from pack_conv_subpixel: one tensor-core launch per output parity."""
    _chk16(x, wsub)
    _chk32(bias)
    n, H, W, Ci = x.shape
    co = wsub.shape[1]
    assert tuple(wsub.shape) == (4, co, 4 * Ci), "expected pack_conv_subpixel panels"
    out = torch.empty((n, 2 * H, 2 * W, co), dtype=torch.float16, device=x.device)
    for par in range(4):
        _gemm_ex(A=_ptr(x), K1=Ci, lda1=Ci, Bw=_ptr(wsub[par]), M=n * H * W, N=co, taps=4, sub_py=par >> 1, sub_px=par & 1,
                 nimg=n, H=H, W=W, bias=_ptr(bias), out=_ptr(out), ldc=co)
    return out


def upsample_conv3x3_sized(x, w, bias, OH, OW, out=None):
    """nearest up-sampling to OH x OW (2H or 2H - 1 rows, 2W or 2W - 1 columns) + conv3x3 (pad 1), as the UNet's up path
    runs it: x [N, H, W, C], w [Co, C, 3, 3] (unpacked) -> [N, OH, OW, Co].  `out` may be any contiguous fp16 buffer of at
    least N * OH * OW * Co elements; the result is its first N * OH * OW * Co elements."""
    _chk16(x, w, out)
    _chk32(bias)
    n, H, W, Ci = x.shape
    co = w.shape[0]
    panels = torch.empty((49 * co * Ci,), dtype=torch.float16, device=x.device)
    if out is None:
        out = torch.empty((n, OH, OW, co), dtype=torch.float16, device=x.device)
    assert out.is_contiguous() and out.numel() >= n * OH * OW * co
    _lib.call("vs_upsample_conv3x3_sized", _stream(), _p(x), n, H, W, Ci, _p(w), co, _p(bias), OH, OW, _p(panels), _p(out))
    return out


def upsample_nearest(x, OH, OW):
    """x [N, H, W, C] -> [N, OH, OW, C], out[y, x] = in[y // 2, x // 2] (OH in {2H - 1, 2H}, OW in {2W - 1, 2W})."""
    _chk16(x)
    n, H, W, Cc = x.shape
    out = torch.empty((n, OH, OW, Cc), dtype=torch.float16, device=x.device)
    _lib.call("vs_upsample_nearest", _stream(), _p(x), n, H, W, Cc, OH, OW, _p(out))
    return out


def groupnorm(x1, gamma, beta, groups, eps, imgs_per_set=1, silu=False, x2=None):
    """x1 [N, H, W, C1] (+ x2) -> normalised [N, H, W, C1+C2]; statistics over imgs_per_set images x (C/groups)."""
    _chk16(x1, x2)
    _chk32(gamma, beta)
    n, H, W, c1 = x1.shape
    c2 = 0 if x2 is None else x2.shape[3]
    sums = torch.empty((n // imgs_per_set, groups, 2), dtype=torch.float32, device=x1.device)
    out = torch.empty((n, H, W, c1 + c2), dtype=torch.float16, device=x1.device)
    _lib.call("vs_groupnorm", _stream(), _p(x1), c1, _p(x2), c2, n, H * W, imgs_per_set, groups, eps, _p(gamma), _p(beta),
              int(silu), _p(sums), _p(out))
    return out


def groupnorm_stats(x1, sums, groups, imgs_per_set, x2=None, zero_first=True):
    """Adds each set's per-group (sum, sum of squares) of x1 (+ x2) into sums [n / imgs_per_set, groups, 2] fp32 (zeroed
    first only with zero_first): the statistics half of the GroupNorm, as a frame shard computes it."""
    _chk16(x1, x2)
    _chk32(sums)
    n, H, W, c1 = x1.shape
    c2 = 0 if x2 is None else x2.shape[3]
    assert tuple(sums.shape) == (n // imgs_per_set, groups, 2)
    _lib.call("vs_groupnorm_stats", _stream(), _p(x1), c1, _p(x2), c2, n, H * W, imgs_per_set, groups, _p(sums),
              int(zero_first))
    return sums


def groupnorm_apply(x1, sums, gamma, beta, groups, eps, imgs_per_set, count_scale=1, silu=False, x2=None):
    """Normalises x1 (+ x2) with `sums` that cover count_scale times the local elements (all-reduced frame shards)."""
    _chk16(x1, x2)
    _chk32(sums, gamma, beta)
    n, H, W, c1 = x1.shape
    c2 = 0 if x2 is None else x2.shape[3]
    out = torch.empty((n, H, W, c1 + c2), dtype=torch.float16, device=x1.device)
    _lib.call("vs_groupnorm_apply", _stream(), _p(x1), c1, _p(x2), c2, n, H * W, imgs_per_set, groups, _p(sums), eps,
              _p(gamma), _p(beta), int(silu), int(count_scale), _p(out))
    return out


def layernorm(x, gamma, beta, pe=None, hw=1, F=1):
    _chk16(x)
    _chk32(gamma, beta, pe)
    rows, Cc = x.shape
    out = torch.empty_like(x)
    _lib.call("vs_layernorm", _stream(), _p(x), rows, Cc, _p(gamma), _p(beta), _p(pe), hw, F, _p(out))
    return out


def ln_linear(x, W, gamma, beta, bias=None, pe=None, hw=1, frames=1, mode=EPI_LINEAR):
    """LayerNorm(x)(+pe[(row // hw) % frames]) @ W^T + bias with the norm folded into the GEMM (C in 320/640/1280)."""
    _chk16(x, W)
    _chk32(gamma, beta, bias, pe)
    M, Cc = x.shape
    N = W.shape[0]
    dev = x.device
    wf = torch.empty_like(W)
    u = torch.empty((N,), dtype=torch.float32, device=dev)
    c = torch.empty((N,), dtype=torch.float32, device=dev)
    cpe = torch.empty((pe.shape[0], N), dtype=torch.float32, device=dev) if pe is not None else None
    stats = torch.empty((M, 2), dtype=torch.float32, device=dev)
    out = torch.empty((M, N // 2 if mode == EPI_GEGLU else N), dtype=torch.float16, device=dev)
    _lib.call("vs_ln_linear", _stream(), _p(x), M, Cc, _p(W), _p(bias), N, _p(gamma), _p(beta), _p(pe),
              0 if pe is None else pe.shape[0], hw, frames, mode, _p(wf), _p(u), _p(c), _p(cpe), _p(stats), _p(out))
    return out


def linear_ln_linear(x0, W0, b0, W, gamma, beta, residual=None, bias=None, mode=EPI_LINEAR, pe=None, hw=1, frames=1):
    """x = x0 @ W0^T + b0 (+ residual) [fp16]; out = (LayerNorm(x) (+ pe[(row // hw) % frames])) @ W^T + bias (or GEGLU),
    the LayerNorm's row statistics coming from the first GEMM's epilogue.  Returns (x, out)."""
    _chk16(x0, W0, W, residual)
    _chk32(b0, gamma, beta, bias, pe)
    M, K0 = x0.shape
    Cc, N = W0.shape[0], W.shape[0]
    dev = x0.device
    x = torch.empty((M, Cc), dtype=torch.float16, device=dev)
    wf = torch.empty_like(W)
    u = torch.empty((N,), dtype=torch.float32, device=dev)
    c = torch.empty((N,), dtype=torch.float32, device=dev)
    cpe = torch.empty((pe.shape[0], N), dtype=torch.float32, device=dev) if pe is not None else None
    cap = 16
    parts = torch.empty((cap, M, 2), dtype=torch.float32, device=dev)
    out = torch.empty((M, N // 2 if mode == EPI_GEGLU else N), dtype=torch.float16, device=dev)
    _lib.call("vs_linear_ln_linear", _stream(), _p(x0), M, K0, _p(W0), _p(b0), _p(residual), Cc, _p(x), _p(W), _p(bias), N,
              _p(gamma), _p(beta), _p(pe), 0 if pe is None else pe.shape[0], hw, frames, mode, _p(wf), _p(u), _p(c), _p(cpe),
              _p(parts), cap, _p(out))
    return x, out


def attention(q, k, v, heads, kv_div=1):
    """q [B, Nq, h*d], k/v [Bk, Nk, h*d] (may be strided views with contiguous last dim) -> [B, Nq, h*d]."""
    B, nq, Cc = q.shape
    nk = k.shape[1]
    d = Cc // heads
    for t in (q, k, v):
        assert t.dtype == torch.float16 and t.stride(2) == 1
    out = torch.empty((B, nq, Cc), dtype=torch.float16, device=q.device)
    _lib.call("vs_attention", _stream(), _p(q), q.stride(1), _p(k), k.stride(1), _p(v), v.stride(1), _p(out), Cc, B, nq, nk,
              heads, d, q.stride(0), k.stride(0), nq * Cc, kv_div)
    return out


def attention_probs(q, k, heads, kv_div=1):
    """softmax(q k^T / sqrt(d)) as a tensor [B, heads, Nq, Nk] fp16 (explicit-probability path of the attention controllers)."""
    B, nq, Cc = q.shape
    nk = k.shape[1]
    probs = torch.empty((B, heads, nq, nk), dtype=torch.float16, device=q.device)
    _lib.call("vs_attention_probs", _stream(), _p(q), q.stride(1), _p(k), k.stride(1), _p(probs), B, nq, nk, heads, Cc // heads,
              q.stride(0), k.stride(0), kv_div)
    return probs


def attention_apply_probs(probs, v, heads, kv_div=1):
    """O = P V: probs [B, heads, Nq, Nk] fp16, v [Bk, Nk, heads*d] -> [B, Nq, heads*d]."""
    _chk16(probs)
    B, _, nq, nk = probs.shape
    Cc = v.shape[2]
    out = torch.empty((B, nq, Cc), dtype=torch.float16, device=probs.device)
    _lib.call("vs_attention_apply_probs", _stream(), _p(probs), _p(v), v.stride(1), _p(out), Cc, B, nq, nk, heads, Cc // heads,
              v.stride(0), nq * Cc, kv_div)
    return out


def scores(q, k, out):
    """out[i, j] = q_i . k_j (fp16) for q [nq, d], k [nk, d]; out [nq, ld] with ld >= nk (columns nk .. ld - 1 untouched)."""
    _chk16(q, k, out)
    nq, d = q.shape
    nk = k.shape[0]
    assert k.shape[1] == d and out.dim() == 2 and out.shape[0] == nq and out.shape[1] >= nk
    _gemm_ex(A=_ptr(q), K1=d, lda1=d, Bw=_ptr(k), M=nq, N=nk, out=_ptr(out), ldc=out.shape[1])
    return out


def softmax_rows(s, n, scale):
    """In place on s [rows, ld] fp16: softmax(s * scale) over the first n columns (fp32 math), zeros in columns n .. ld - 1."""
    _chk16(s)
    rows, ld = s.shape
    _lib.call("vs_softmax_rows", _stream(), _p(s), rows, n, ld, float(scale))
    return s


def transpose_pad(x, rows_pad, out=None):
    """x [rows, cols] fp16 -> [cols, rows_pad] = x^T with zero columns rows .. rows_pad - 1."""
    _chk16(x)
    rows, cols = x.shape
    out = _out16(out, (cols, rows_pad), x.device)
    _lib.call("vs_transpose_pad", _stream(), _p(x), rows, cols, rows_pad, _p(out))
    return out


def vae_latent_in(z, divisor, wb):
    """post_quant_conv(z / divisor): z [n, 4, h, w] fp16 / fp32 NCHW, wb fp32 [20] (weight [4, 4], then bias [4]) ->
    NHWC fp16 [n, h, w, 4]."""
    assert z.is_cuda and z.dtype in (torch.float16, torch.float32) and z.is_contiguous() and z.dim() == 4 and z.shape[1] == 4, \
        "expected contiguous [n, 4, h, w] fp16 / fp32 CUDA latents"
    _chk32(wb)
    assert wb.numel() == 20
    n, _, h, w = z.shape
    out = torch.empty((n, h, w, 4), dtype=torch.float16, device=z.device)
    _lib.call("vs_vae_latent_in", _stream(), _p(z), int(z.dtype == torch.float32), n, h, w, float(divisor), _p(wb), _p(out))
    return out


IMG_SAMPLE, IMG_PT, IMG_NP, IMG_PIL = 0, 1, 2, 3


def image_postprocess(x, fmt):
    """Channels 0..2 of the decoder output x [n, H, W, C] (C % 8 == 0): IMG_SAMPLE fp16 [n, 3, H, W] as is; else
    y = clamp(x / 2 + 0.5, 0, 1) as IMG_PT fp32 [n, 3, H, W], IMG_NP fp32 [n, H, W, 3] or IMG_PIL uint8 [n, H, W, 3]."""
    _chk16(x)
    n, H, W, Cc = x.shape
    shape = (n, 3, H, W) if fmt in (IMG_SAMPLE, IMG_PT) else (n, H, W, 3)
    dtype = {IMG_SAMPLE: torch.float16, IMG_PT: torch.float32, IMG_NP: torch.float32, IMG_PIL: torch.uint8}[fmt]
    out = torch.empty(shape, dtype=dtype, device=x.device)
    _lib.call("vs_image_postprocess", _stream(), _p(x), n, H, W, Cc, fmt, _p(out))
    return out


def downsample_conv3x3(x, w_packed, bias=None):
    """Downsample2D(padding=0): conv3x3 with stride 2 of x zero-padded by one column on the right and one row at the
    bottom, x [N, H, W, C] (H, W even, C % 64 == 0), w_packed pack_conv3x3 [Co, 9 C] -> [N, H / 2, W / 2, Co]."""
    _chk16(x, w_packed)
    _chk32(bias)
    n, H, W, Ci = x.shape
    co = w_packed.shape[0]
    assert w_packed.shape[1] == 9 * Ci, "expected a pack_conv3x3 panel"
    out = torch.empty((n, H // 2, W // 2, co), dtype=torch.float16, device=x.device)
    _lib.call("vs_downsample_conv3x3", _stream(), _p(x), n, H, W, Ci, _p(w_packed), co, _p(bias), _p(out))
    return out


VAE_IN_U8_NHWC, VAE_IN_F16_NCHW, VAE_IN_F32_NCHW = 0, 1, 2


def vae_image_in(x):
    """Encoder input -> NHWC fp16 [n, H, W, 4] with channel 3 zero.  x: uint8 frames [n, H, W, 3] (normalised as
    VaeImageProcessor.preprocess does, 2 (u / 255) - 1) or fp16 / fp32 images [n, 3, H, W] in [-1, 1] (rounded to fp16)."""
    assert x.is_cuda and x.is_contiguous() and x.dim() == 4, "expected a contiguous 4-D CUDA tensor"
    if x.dtype == torch.uint8:
        assert x.shape[3] == 3, "uint8 frames are [n, H, W, 3]"
        src, (n, H, W) = VAE_IN_U8_NHWC, x.shape[:3]
    else:
        assert x.dtype in (torch.float16, torch.float32) and x.shape[1] == 3, "float images are [n, 3, H, W] fp16 / fp32"
        src = VAE_IN_F16_NCHW if x.dtype == torch.float16 else VAE_IN_F32_NCHW
        n, _, H, W = x.shape
    out = torch.empty((n, H, W, 4), dtype=torch.float16, device=x.device)
    _lib.call("vs_vae_image_in", _stream(), _p(x), src, n, H, W, _p(out))
    return out


def vae_moments(x, wb):
    """quant_conv in fp32: conv_out's x [n, h, w, 8] fp16, wb fp32 [72] (weight [8, 8], then bias [8]) -> the moments
    fp16 NCHW [n, 8, h, w] (mean, then logvar)."""
    _chk16(x)
    _chk32(wb)
    n, h, w, Cc = x.shape
    assert Cc == 8 and wb.numel() == 72
    out = torch.empty((n, 8, h, w), dtype=torch.float16, device=x.device)
    _lib.call("vs_vae_moments", _stream(), _p(x), n, h, w, _p(wb), _p(out))
    return out


def vae_posterior(params, noise=None, scale=1.0, video=False):
    """scale (mean + exp(0.5 clamp(logvar, -30, 20)) noise) from the moments params [n, 8, h, w] fp16 and noise
    [n, 4, h, w] fp16 (None: scale mean).  Output fp16 [n, 4, h, w], or with video=True [1, 4, n, h, w]."""
    _chk16(params, noise)
    n, c8, h, w = params.shape
    assert c8 == 8 and (noise is None or tuple(noise.shape) == (n, 4, h, w))
    out = torch.empty((1, 4, n, h, w) if video else (n, 4, h, w), dtype=torch.float16, device=params.device)
    _lib.call("vs_vae_posterior", _stream(), _p(params), _p(noise), n, h, w, float(scale), int(video), _p(out))
    return out


def clip_embed(ids, tok, pos):
    """CLIP token + position embedding: ids int32 [n, L] (CUDA, every id in [0, tok.shape[0]) -- the caller checks), tok
    fp16 [vocab, C], pos fp16 [>= L, C] -> fp16 [n L, C] = fp16(fp32(tok[ids]) + fp32(pos[t]))."""
    _chk16(tok, pos)
    assert ids.is_cuda and ids.dtype == torch.int32 and ids.is_contiguous() and ids.dim() == 2, "expected int32 [n, L] CUDA ids"
    n, L = ids.shape
    vocab, Cc = tok.shape
    assert pos.shape[1] == Cc and pos.shape[0] >= L
    out = torch.empty((n * L, Cc), dtype=torch.float16, device=tok.device)
    _lib.call("vs_clip_embed", _stream(), _p(ids), n, L, _p(tok), vocab, _p(pos), Cc, _p(out))
    return out


def causal_attention(qkv, nseq, L, heads, out=None):
    """Causal self-attention of nseq sequences of L <= 77 tokens from the fused QKV output qkv [nseq L, >= 3 C] (q, k, v
    in column blocks of C = heads * 64; may be a column slice with unit stride) -> [nseq L, C] (`out`: the caller's tensor,
    which may be a row-strided view)."""
    assert qkv.is_cuda and qkv.dtype == torch.float16 and qkv.dim() == 2 and qkv.stride(1) == 1 and qkv.shape[0] == nseq * L
    Cc = qkv.shape[1] // 3
    if out is None:
        out = torch.empty((nseq * L, Cc), dtype=torch.float16, device=qkv.device)
    assert out.is_cuda and out.dtype == torch.float16 and out.stride(1) == 1 and tuple(out.shape) == (nseq * L, Cc), \
        "out: fp16 [nseq L, C] CUDA tensor with unit column stride"
    _lib.call("vs_causal_attention", _stream(), _p(qkv), qkv.stride(0), _p(out), out.stride(0), nseq, L, heads, Cc // heads)
    return out


def temporal_attention(qkv, heads):
    """qkv [B, F, HW, 3C] -> [B, F, HW, C]: attention over the F axis for every (b, pixel, head)."""
    _chk16(qkv)
    B, F, HW, C3 = qkv.shape
    out = torch.empty((B, F, HW, C3 // 3), dtype=torch.float16, device=qkv.device)
    _lib.call("vs_temporal_attention", _stream(), _p(qkv), _p(out), B, F, HW, C3 // 3, heads)
    return out


def conv_in(x, w, bias, scratch="alloc"):
    """conv_in (3x3, pad 1): x [N, H, W, ci], w [co, ci, 3, 3] -> [N, H, W, co].  By default (ci == 4) patch rows + the
    tensor-core GEMM in a scratch buffer of (N H W + co) * 64 halves, as the UNet forward runs it; scratch=None selects
    the direct CUDA-core kernel (also used for ci != 4)."""
    _chk16(x, w)
    _chk32(bias)
    n, H, W, ci = x.shape
    co = w.shape[0]
    if isinstance(scratch, str):
        assert scratch == "alloc"
        scratch = torch.empty(((n * H * W + co) * 64,), dtype=torch.float16, device=x.device) if ci == 4 else None
    _chk16(scratch)
    if scratch is not None:
        assert scratch.numel() >= (n * H * W + co) * 64
    out = torch.empty((n, H, W, co), dtype=torch.float16, device=x.device)
    _lib.call("vs_conv_in", _stream(), _p(x), n, H, W, ci, _p(w), _p(bias), co, _p(scratch), _p(out))
    return out


def upsample2x(x):
    _chk16(x)
    n, H, W, Cc = x.shape
    out = torch.empty((n, 2 * H, 2 * W, Cc), dtype=torch.float16, device=x.device)
    _lib.call("vs_upsample2x", _stream(), _p(x), n, H, W, Cc, _p(out))
    return out


def ddim_coefficients(alpha_t: float, alpha_prev: float, eta: Optional[float] = None):
    """(c_x, c_e) with x_prev = c_x * x + c_e * eps  (DDIM, eta = 0).
    With `eta` given: (c_x, c_e, c_n) of diffusers 0.19.3's stochastic step, x_prev = c_x x + c_e eps + c_n z, with
    c_n = eta sqrt(variance(t, t_prev)) and c_e = sqrt(1 - a_p - c_n^2) - sqrt(a_p) sqrt(1 - a_t) / sqrt(a_t); at eta = 0
    the first two are the values above.  The same fp64 expression as vs_cfg_ddim_rescale_step's, so device coefficients
    rounded to fp32 reproduce the host-coefficient launch bit for bit."""
    import math
    if eta is None:
        c_x = math.sqrt(alpha_prev) / math.sqrt(alpha_t)
        c_e = math.sqrt(1.0 - alpha_prev) - math.sqrt(alpha_prev) * math.sqrt(1.0 - alpha_t) / math.sqrt(alpha_t)
        return c_x, c_e
    if eta < 0:
        raise ValueError(f"eta must be >= 0, got {eta}")
    at, ap = float(alpha_t), float(alpha_prev)
    c_n = 0.0 if eta == 0 else float(eta) * math.sqrt((1.0 - ap) / (1.0 - at) * (1.0 - at / ap))
    c_x = math.sqrt(ap) / math.sqrt(at)
    c_e = math.sqrt(1.0 - ap - c_n * c_n) - math.sqrt(ap) * math.sqrt(1.0 - at) / math.sqrt(at)
    return c_x, c_e, c_n


def cfg_ddim_step(eps2, latents, guidance, alpha_t=None, alpha_prev=None, cfg=True, out=None, coef=None):
    """coef: optional device tensor [2] fp32 (c_x, c_e) instead of host alphas (CUDA-graph replayable)."""
    assert eps2.dtype == latents.dtype and eps2.is_contiguous() and latents.is_contiguous()
    is_f32 = int(latents.dtype == torch.float32)
    if out is None:
        out = torch.empty_like(latents)
    if coef is not None:
        _chk32(coef)
        _lib.call("vs_cfg_ddim_step_dev", _stream(), _p(eps2), _p(latents), is_f32, latents.numel(), int(cfg), float(guidance),
                  _p(coef), _p(out))
        return out
    _lib.call("vs_cfg_ddim_step", _stream(), _p(eps2), _p(latents), is_f32, latents.numel(), int(cfg), float(guidance),
              float(alpha_t), float(alpha_prev), _p(out))
    return out


def cfg_ddim_rescale_step(eps2, latents, guidance, alpha_t=None, alpha_prev=None, eta=0.0, guidance_rescale=0.0,
                          noise=None, cfg=True, out=None, coef=None):
    """The CFG combine, diffusers' rescale_noise_cfg and DDIMScheduler.step with eta for S = latents.shape[0] samples in
    one launch (vs_cfg_ddim_rescale_step).  eps2: [2 S, ...] (uncond block first) under CFG, else [S, ...]; noise: the
    step's standard normal draw, latents' shape and dtype (needed when eta > 0).  coef: optional device tensor [4] fp32
    (c_x, c_e, c_n, guidance_rescale) instead of the host alphas / eta / guidance_rescale (CUDA-graph replayable)."""
    S = latents.shape[0]
    assert eps2.dtype == latents.dtype and eps2.is_contiguous() and latents.is_contiguous()
    assert eps2.numel() == latents.numel() * (2 if cfg else 1), "eps2 must hold (2 if cfg else 1) x latents' elements"
    if noise is not None:
        assert noise.dtype == latents.dtype and noise.is_contiguous() and noise.shape == latents.shape
    is_f32 = int(latents.dtype == torch.float32)
    if out is None:
        out = torch.empty_like(latents)
    n_s = latents.numel() // S
    if coef is not None:
        _chk32(coef)
        assert coef.numel() >= 4
        _lib.call("vs_cfg_ddim_rescale_step_dev", _stream(), _p(eps2), _p(latents), _p(noise), is_f32, S, n_s, int(cfg),
                  float(guidance), _p(coef), _p(out))
        return out
    _lib.call("vs_cfg_ddim_rescale_step", _stream(), _p(eps2), _p(latents), _p(noise), is_f32, S, n_s, int(cfg),
              float(guidance), float(alpha_t), float(alpha_prev), float(eta), float(guidance_rescale), _p(out))
    return out


def adapter_level(w0, b0, w1, b1, point_embedding, tracks, h, w, rate, point_mask=None, coord_fp16=True, scale=1.0):
    """One level of SparsePointAdapter: returns the NHWC fp16 map [F, h, w, C]."""
    _chk16(w0, b0, w1, b1)
    _chk32(point_embedding, tracks)
    mid, E = w0.shape
    Cc = w1.shape[0]
    F, P = tracks.shape[:2]
    ws = torch.empty((mid + Cc + P * (mid + Cc),), dtype=torch.float32, device=w0.device)
    out = torch.empty((F, h, w, Cc), dtype=torch.float16, device=w0.device)
    _lib.call("vs_adapter_level", _stream(), _p(w0), _p(b0), _p(w1), _p(b1), E, mid, Cc, _p(point_embedding), _p(tracks),
              _p(point_mask), F, P, h, w, float(rate), int(coord_fp16), float(scale), _p(ws), _p(out))
    return out


def dift_noise(moments, eps1, eps2, scaling_factor, sqrt_a, sqrt_1ma):
    """The DIFT UNet input fp32 [n E, 4, 1, h, w] = sqrt_a sf (mean + std eps1) + sqrt_1ma eps2 from the VAE moments
    fp16 [n, 8, h, w] of n frames and fp32 noise eps1, eps2 [n E, 4, h, w] (row r belongs to frame r // E)."""
    _chk16(moments)
    _chk32(eps1, eps2)
    n, c8, h, w = moments.shape
    assert c8 == 8 and eps1.shape == eps2.shape and eps1.dim() == 4 and tuple(eps1.shape[1:]) == (4, h, w)
    assert eps1.shape[0] % n == 0, "noise rows must be a whole ensemble per frame"
    E = eps1.shape[0] // n
    out = torch.empty((n * E, 4, 1, h, w), dtype=torch.float32, device=moments.device)
    _lib.call("vs_dift_noise", _stream(), _p(moments), _p(eps1), _p(eps2), n, E, h, w, float(scaling_factor), float(sqrt_a),
              float(sqrt_1ma), _p(out))
    return out


def dift_point_sample(feat, size, xy):
    """Ensemble mean of feat NHWC fp16 [n, E, h, w, C] up-sampled bilinearly (align_corners False) to size = (H, W),
    read at the pixels xy int32 [n, P, 2] = (x, y) inside the image -> fp32 [n, P, C]."""
    _chk16(feat)
    assert xy.is_cuda and xy.dtype == torch.int32 and xy.is_contiguous() and xy.dim() == 3 and xy.shape[2] == 2
    n, E, h, w, Cc = feat.shape
    assert xy.shape[0] == n
    P = xy.shape[1]
    out = torch.empty((n, P, Cc), dtype=torch.float32, device=feat.device)
    if P:
        _lib.call("vs_dift_point_sample", _stream(), _p(feat), n, E, h, w, Cc, int(size[0]), int(size[1]), _p(xy), P, _p(out))
    return out


def dift_ensemble_mean(feat):
    """feat NHWC fp16 [n, E, h, w, C] -> fp32 NCHW [n, C, h, w], the mean over E."""
    _chk16(feat)
    n, E, h, w, Cc = feat.shape
    out = torch.empty((n, Cc, h, w), dtype=torch.float32, device=feat.device)
    _lib.call("vs_dift_ensemble_mean", _stream(), _p(feat), n, E, h, w, Cc, _p(out))
    return out


def dift_point_cosine(vecs, src, src_row):
    """CosineSimilarity(dim=1, eps=1e-8) of vecs fp32 [n, P, C] against src[src_row] (src fp32 [S, C], src_row int32
    [n, P]) -> fp32 [n, P]."""
    _chk32(vecs, src)
    assert src_row.is_cuda and src_row.dtype == torch.int32 and src_row.is_contiguous()
    n, P, Cc = vecs.shape
    assert src.dim() == 2 and src.shape[1] == Cc and tuple(src_row.shape) == (n, P)
    conf = torch.empty((n, P), dtype=torch.float32, device=vecs.device)
    _lib.call("vs_dift_point_reduce", _stream(), _p(vecs), n, P, Cc, _p(src), _p(src_row), _p(conf), None, None, None, None)
    return conf


def dift_point_reduce(vecs, accept):
    """Per-point (sums [P, C], counts [P], means [P, C]) fp32 of vecs fp32 [n, P, C] over the frames where accept (bool /
    uint8 [n, P]) is set, accumulated in frame order; a point never accepted has mean 0."""
    _chk32(vecs)
    n, P, Cc = vecs.shape
    acc = accept.to(device=vecs.device, dtype=torch.uint8).contiguous()
    assert tuple(acc.shape) == (n, P)
    sums = torch.empty((P, Cc), dtype=torch.float32, device=vecs.device)
    means = torch.empty_like(sums)
    counts = torch.empty((P,), dtype=torch.float32, device=vecs.device)
    _lib.call("vs_dift_point_reduce", _stream(), _p(vecs), n, P, Cc, None, None, None, _p(acc), _p(sums), _p(counts), _p(means))
    return sums, counts, means
