"""Per-kernel parity checks: every CUDA kernel (called through the C-ABI) against a plain PyTorch fp32 restatement
of the same op on the same seeded inputs.  Each check returns {"err": max abs error, "ref": max |ref|, "tol": ...}.
Used by tests/test_kernels_gpu.py (pytest -m gpu) and tools/gpu_kernel_check.py (subprocess-isolated diagnostics)."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from videoswap_b200 import ops

DEV = "cuda"


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def _res(out, ref, rel=2 ** -8, abs_=2e-3):
    out, ref = out.float(), ref.float()
    err = (out - ref).abs().max().item()
    mx = ref.abs().max().item()
    tol = rel * mx + abs_
    bad = not (err <= tol) or not torch.isfinite(out).all().item()
    return {"err": err, "ref": mx, "tol": tol, "ok": not bad}


# ---------------------------------------------------------------------------------------------------- GEMM
def check_gemm(M=512, N=320, K=320, bias=True, residual=False, bn=0, seed=0):
    A = _rand((M, K), seed).half()
    W = _rand((N, K), seed + 1, 1 / math.sqrt(K)).half()
    b = _rand((N,), seed + 2).float() if bias else None
    R = _rand((M, N), seed + 3).half() if residual else None
    out = ops.gemm(A, W, bias=b, residual=R, force_bn=bn)
    ref = A.float() @ W.float().t()
    if bias:
        ref = ref + b
    if residual:
        ref = ref + R.float()
    return _res(out, ref)


def check_gemm_concat(M=300, N=640, K1=640, K2=320, seed=10):
    A = _rand((M, K1), seed).half()
    A2 = _rand((M, K2), seed + 1).half()
    W = _rand((N, K1 + K2), seed + 2, 1 / math.sqrt(K1 + K2)).half()
    b = _rand((N,), seed + 3).float()
    out = ops.gemm(A, W, bias=b, A2=A2)
    ref = torch.cat([A, A2], 1).float() @ W.float().t() + b
    return _res(out, ref)


def check_gemm_rowvec(M=256, N=320, K=64, seed=20):
    A = _rand((M, K), seed).half()
    W = _rand((N, K), seed + 1, 1 / math.sqrt(K)).half()
    rv = _rand((4, N), seed + 2).float()
    out = ops.gemm(A, W, rowvec=rv, pix_per_batch=64)
    ref = A.float() @ W.float().t() + rv.repeat_interleave(64, 0)
    return _res(out, ref)


def check_geglu(M=384, C=320, seed=30):
    A = _rand((M, C), seed).half()
    W = _rand((8 * C, C), seed + 1, 1 / math.sqrt(C)).half()
    b = _rand((8 * C,), seed + 2, 0.1).half()
    wp, bp = ops.pack_geglu(W, b)
    out = ops.gemm(A, wp, bias=bp, mode=ops.EPI_GEGLU)
    h = A.float() @ W.float().t() + b.float()
    v, g = h.chunk(2, -1)
    ref = v * F.gelu(g)
    return _res(out, ref)


# ---------------------------------------------------------------------------------------------------- conv
def _conv_ref(x_nhwc, w, b, stride=1):
    y = F.conv2d(x_nhwc.float().permute(0, 3, 1, 2), w.float(), None if b is None else b.float(), stride=stride, padding=1)
    return y.permute(0, 2, 3, 1)


def check_conv3x3(n=4, H=16, W=16, ci=320, co=320, rowvec=False, residual=False, seed=40):
    x = _rand((n, H, W, ci), seed).half()
    w = _rand((co, ci, 3, 3), seed + 1, 1 / math.sqrt(9 * ci)).half()
    b = _rand((co,), seed + 2).float()
    rv = _rand((n // 2, co), seed + 3).float() if rowvec else None
    R = _rand((n, H, W, co), seed + 4).half() if residual else None
    out = ops.conv3x3(x, ops.pack_conv3x3(w), bias=b, rowvec=rv, imgs_per_batch=2, residual=R)
    ref = _conv_ref(x, w, b)
    if rowvec:
        ref = ref + rv.repeat_interleave(2, 0)[:, None, None, :]
    if residual:
        ref = ref + R.float()
    return _res(out, ref)


def check_conv3x3_concat(n=2, H=8, W=8, c1=640, c2=320, co=640, seed=50):
    x1 = _rand((n, H, W, c1), seed).half()
    x2 = _rand((n, H, W, c2), seed + 1).half()
    w = _rand((co, c1 + c2, 3, 3), seed + 2, 1 / math.sqrt(9 * (c1 + c2))).half()
    b = _rand((co,), seed + 3).float()
    out = ops.conv3x3(x1, ops.pack_conv3x3(w), bias=b, x2=x2)
    ref = _conv_ref(torch.cat([x1, x2], -1), w, b)
    return _res(out, ref)


def check_conv3x3_odd_shape(n=3, H=7, W=12, ci=320, co=320, seed=55):
    return check_conv3x3(n=n, H=H, W=W, ci=ci, co=co, seed=seed) if n % 2 == 0 else _conv_odd(n, H, W, ci, co, seed)


def _conv_odd(n, H, W, ci, co, seed):
    x = _rand((n, H, W, ci), seed).half()
    w = _rand((co, ci, 3, 3), seed + 1, 1 / math.sqrt(9 * ci)).half()
    b = _rand((co,), seed + 2).float()
    out = ops.conv3x3(x, ops.pack_conv3x3(w), bias=b)
    return _res(out, _conv_ref(x, w, b))


def check_conv_out(n=2, H=16, W=16, ci=320, co=4, seed=60):
    return _conv_odd(n, H, W, ci, co, seed)


def check_conv_s2(n=2, H=16, W=16, ci=320, co=320, seed=70):
    x = _rand((n, H, W, ci), seed).half()
    w = _rand((co, ci, 3, 3), seed + 1, 1 / math.sqrt(9 * ci)).half()
    b = _rand((co,), seed + 2).float()
    out = ops.conv3x3_s2(x, ops.pack_conv3x3(w), bias=b)
    return _res(out, _conv_ref(x, w, b, stride=2))


def check_upsample_conv(n=2, H=8, W=8, ci=640, co=640, seed=75):
    """Upsample3D: nearest 2x + conv3x3 (resnet.py:54,67) through the sub-pixel decomposition."""
    x = _rand((n, H, W, ci), seed).half()
    w = _rand((co, ci, 3, 3), seed + 1, 1 / math.sqrt(9 * ci)).half()
    b = _rand((co,), seed + 2).float()
    out = ops.upsample_conv3x3(x, w, bias=b)
    up = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest")
    ref = F.conv2d(up, w.float(), b, padding=1).permute(0, 2, 3, 1)
    return _res(out, ref)


def check_conv_in(n=4, H=16, W=16, seed=80):
    x = _rand((n, H, W, 4), seed).half()
    w = _rand((320, 4, 3, 3), seed + 1, 1 / 6).half()
    b = _rand((320,), seed + 2).float()
    out = ops.conv_in(x, w, b)
    return _res(out, _conv_ref(x, w, b))


def check_upsample(n=2, H=5, W=6, c=640, seed=90):
    x = _rand((n, H, W, c), seed).half()
    out = ops.upsample2x(x)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1)
    return _res(out, ref, rel=0, abs_=0)


# ---------------------------------------------------------------------------------------------------- norms
def check_groupnorm(B=2, Fr=3, H=8, W=8, c1=320, c2=0, per_frame=False, silu=True, eps=1e-5, seed=100, mean=0.3):
    n = B * Fr
    x1 = (_rand((n, H, W, c1), seed) * 1.5 + mean).half()
    x2 = (_rand((n, H, W, c2), seed + 1) * 0.7 - 0.2).half() if c2 else None
    C = c1 + c2
    gamma = (1 + 0.1 * _rand((C,), seed + 2)).float()
    beta = (0.1 * _rand((C,), seed + 3)).float()
    out = ops.groupnorm(x1, gamma, beta, 32, eps, imgs_per_set=1 if per_frame else Fr, silu=silu, x2=x2)
    x = x1 if x2 is None else torch.cat([x1, x2], -1)
    x = x.float().permute(0, 3, 1, 2)                                # [n, C, H, W]
    if per_frame:
        ref = F.group_norm(x, 32, gamma, beta, eps)
    else:                                                            # 5-D GroupNorm: stats over (C/32, F, H, W)
        x5 = x.reshape(B, Fr, C, H, W).permute(0, 2, 1, 3, 4)
        ref = F.group_norm(x5, 32, gamma, beta, eps).permute(0, 2, 1, 3, 4).reshape(n, C, H, W)
    if silu:
        ref = F.silu(ref)
    return _res(out, ref.permute(0, 2, 3, 1))


def check_layernorm(rows=1000, C=320, pe=False, seed=110):
    x = (_rand((rows, C), seed) * 2 + 0.5).half()
    # gamma/beta are fp16 model weights in the product (the fast path keeps them as packed fp16): make them representable
    gamma = (1 + 0.1 * _rand((C,), seed + 1)).half().float()
    beta = (0.1 * _rand((C,), seed + 2)).half().float()
    Fr, hw = 5, 8
    table = _rand((24, C), seed + 3).float() if pe else None
    rows = (rows // (Fr * hw)) * Fr * hw if pe else rows
    x = x[:rows].contiguous()
    out = ops.layernorm(x, gamma, beta, pe=table, hw=hw, F=Fr)
    ref = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5)
    if pe:
        f_idx = (torch.arange(rows, device=DEV) // hw) % Fr
        ref = ref + table[f_idx]
    return _res(out, ref)


def check_ln_linear(rows=2000, C=320, N=960, pe=False, geglu=False, seed=115, hw=8):
    """LayerNorm (+ temporal PE) folded into the consuming GEMM vs LayerNorm -> linear / GEGLU in fp32."""
    x = (_rand((rows, C), seed) * 2 + 0.7).half()
    gamma = (1 + 0.1 * _rand((C,), seed + 1)).float()
    beta = (0.1 * _rand((C,), seed + 2)).float()
    Fr = 5
    table = _rand((24, C), seed + 3).float() if pe else None
    rows = (rows // (Fr * hw)) * Fr * hw
    x = x[:rows].contiguous()
    W = _rand((N, C), seed + 4, 1 / math.sqrt(C)).half()
    b = _rand((N,), seed + 5).float() if geglu else None
    y = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5)
    if pe:
        y = y + table[(torch.arange(rows, device=DEV) // hw) % Fr]
    ref = y @ W.float().t()
    if geglu:
        ref = ref + b
        h = N // 2
        ref = ref[:, :h] * F.gelu(ref[:, h:])
        Wp, bp = ops.pack_geglu(W, b.half())
        out = ops.ln_linear(x, Wp, gamma, beta, bias=bp, mode=ops.EPI_GEGLU)
    else:
        out = ops.ln_linear(x, W, gamma, beta, pe=table, hw=hw, frames=Fr)
    return _res(out, ref)


def check_linear_ln_linear(rows=2000, K0=320, C=320, N=960, residual=False, geglu=False, seed=160, mean=0.7):
    """Producer GEMM (row statistics from its epilogue) -> LayerNorm folded into the consumer GEMM, vs fp32 torch on the
    fp16 intermediate the producer actually stored."""
    x0 = (_rand((rows, K0), seed) * 2).half()
    W0 = _rand((C, K0), seed + 1, 1 / math.sqrt(K0)).half()
    b0 = (_rand((C,), seed + 2) + mean).float()
    R = (_rand((rows, C), seed + 3) * 1.5 - 0.4).half() if residual else None
    gamma = (1 + 0.1 * _rand((C,), seed + 4)).float()
    beta = (0.1 * _rand((C,), seed + 5)).float()
    W = _rand((N, C), seed + 6, 1 / math.sqrt(C)).half()
    b = _rand((N,), seed + 7).float() if geglu else None
    if geglu:
        Wp, bp = ops.pack_geglu(W, b.half())
        x, out = ops.linear_ln_linear(x0, W0, b0, Wp, gamma, beta, residual=R, bias=bp, mode=ops.EPI_GEGLU)
    else:
        x, out = ops.linear_ln_linear(x0, W0, b0, W, gamma, beta, residual=R)
    xr = x0.float() @ W0.float().t() + b0
    if residual:
        xr = xr.half().float() + R.float()
    r1 = _res(x, xr)
    y = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5)
    ref = y @ W.float().t()
    if geglu:
        ref = ref + b.half().float()
        h = N // 2
        ref = ref[:, :h] * F.gelu(ref[:, h:])
    r2 = _res(out, ref)
    r2["ok"] = r2["ok"] and r1["ok"]
    r2["producer_err"] = r1["err"]
    return r2


# ---------------------------------------------------------------------------------------------------- attention
def _mha_ref(q, k, v, heads):
    B, nq, C = q.shape
    d = C // heads
    qh = q.float().reshape(B, nq, heads, d).transpose(1, 2)
    kh = k.float().reshape(k.shape[0], -1, heads, d).transpose(1, 2)
    vh = v.float().reshape(v.shape[0], -1, heads, d).transpose(1, 2)
    s = qh @ kh.transpose(-1, -2) * d ** -0.5
    return (s.softmax(-1) @ vh).transpose(1, 2).reshape(B, nq, C)


def check_self_attention(B=3, N=200, C=320, seed=120):
    qkv = _rand((B, N, 3 * C), seed).half()
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    out = ops.attention(q, k, v, 8)
    return _res(out, _mha_ref(q, k, v, 8))


def check_self_attention_mma(**kw):
    """Same problem on the mma.sync kernel (the wgmma kernel is the default for d = 40 / 80)."""
    ops.set_option("attn_tc", 0)
    try:
        return check_self_attention(**kw)
    finally:
        ops.set_option("attn_tc", 1)


def check_cross_attention(B=2, Fr=3, N=100, C=640, nk=77, seed=130):
    q = _rand((B * Fr, N, C), seed).half()
    kv = _rand((B, nk, 2 * C), seed + 1).half()
    k, v = kv[..., :C], kv[..., C:]
    out = ops.attention(q, k, v, 8, kv_div=Fr)
    ref = _mha_ref(q, k.repeat_interleave(Fr, 0), v.repeat_interleave(Fr, 0), 8)
    return _res(out, ref)


def check_temporal_attention(B=2, Fr=16, HW=20, C=320, seed=140):
    qkv = _rand((B, Fr, HW, 3 * C), seed).half()
    out = ops.temporal_attention(qkv, 8)
    t = qkv.permute(0, 2, 1, 3).reshape(B * HW, Fr, 3 * C)
    ref = _mha_ref(t[..., :C], t[..., C:2 * C], t[..., 2 * C:], 8)
    ref = ref.reshape(B, HW, Fr, C).permute(0, 2, 1, 3)
    return _res(out, ref)


# ---------------------------------------------------------------------------------------------------- step
def check_cfg_ddim(dtype=torch.float16, seed=150):
    eps2 = _rand((2, 4, 4, 8, 8), seed).to(dtype)
    x = _rand((1, 4, 4, 8, 8), seed + 1).to(dtype)
    a_t, a_p, g = 0.0047, 0.0058, 7.5
    out = ops.cfg_ddim_step(eps2, x, g, a_t, a_p)
    e = eps2[0:1].float() + g * (eps2[1:2].float() - eps2[0:1].float())
    x0 = (x.float() - math.sqrt(1 - a_t) * e) / math.sqrt(a_t)
    ref = math.sqrt(a_p) * x0 + math.sqrt(1 - a_p) * e
    return _res(out, ref, rel=2 ** -9, abs_=1e-3)


def with_option(name, value, fn, restore):
    """Runs a check with a library option flipped (A/B coverage of alternative kernel paths)."""
    def run():
        ops.set_option(name, value)
        try:
            return fn()
        finally:
            ops.set_option(name, restore)
    return run


CHECKS = {
    # BN = 256 tiles (picked by the wave x feed model for wide N / many rows), with every epilogue specialisation
    "gemm_bn256": lambda: check_gemm(8192, 3840, 640, seed=7),
    "gemm_bn256_res": lambda: check_gemm(128 * 150 + 9, 1280, 320, residual=True, seed=8),
    "gemm_bn256_forced_tail": lambda: check_gemm(700, 768, 640, bn=256, seed=9),
    "conv_bn256": lambda: check_conv3x3(n=16, H=32, W=32, ci=320, co=1280, rowvec=True, residual=True),
    # odd row-tile counts, ragged M, small and large K, GEGLU, conv and concat shapes
    "gemm_pair_odd_m": lambda: check_gemm(128 * 3, 640, 1280, residual=True, seed=12),
    "gemm_pair_ragged_m": lambda: check_gemm(128 * 5 + 9, 1280, 1024, seed=13),
    "gemm_pair_small_k": lambda: check_gemm(128 * 7 + 3, 960, 320, seed=14),
    "geglu_pair_small_k": lambda: check_geglu(M=1000, C=320, seed=33),
    "conv_pair_odd": lambda: _conv_odd(3, 7, 12, 320, 320, 56),
    "single_gemm": lambda: check_gemm(1024, 1280, 1280, residual=True, seed=7),
    "single_gemm_bn256": with_option("gemm_stages", 3, lambda: check_gemm(8192, 3840, 640, seed=7), 0),
    "single_geglu": lambda: check_geglu(M=1000, C=640, seed=32),
    "single_conv": with_option("gemm_stages", 3, lambda: check_conv3x3(rowvec=True, residual=True), 0),
    "single_concat": with_option("gemm_stages", 3, lambda: check_gemm_concat(), 0),
    # tile counts that leave some CTAs of the persistent grid without work, or with one tile more than others
    "gemm_one_tile": lambda: check_gemm(100, 128, 64, seed=10),
    "gemm_149_tiles": lambda: check_gemm(128 * 149, 128, 128, residual=True, seed=11),
    # tensor-core attention: ragged query / key counts, many query blocks and key tiles, both head dims, cross-attention.
    # These ids (and the *_prefetch / *_respf* / *_resst* / *_pair* / single_* GEMM ids) come from the A/B switches of the
    # previous kernel generation and are kept as ids; each now runs its own configuration: the mma.sync attention path
    # ("attn_tc" = 0), a shallower GEMM operand ring ("gemm_stages" = 3 / 4), or another seed / ragged shape.
    "self_attn_d40_late_handoff": lambda: check_self_attention(B=2, N=601, C=320, seed=125),
    "self_attn_d40_nonpersistent": with_option("attn_tc", 0, lambda: check_self_attention(B=2, N=600, C=320, seed=121), 1),
    "self_attn_d80_nonpersistent": with_option("attn_tc", 0, lambda: check_self_attention(B=2, N=300, C=640, seed=123), 1),
    "self_attn_d40_persistent_n4096": lambda: check_self_attention(B=3, N=4096, C=320, seed=132),
    "self_attn_d40_poly2": with_option("attn_tc", 0, lambda: check_self_attention(B=2, N=4096, C=320, seed=124), 1),
    "self_attn_d40_poly3": lambda: check_self_attention(B=3, N=700, C=320, seed=127),
    "self_attn_d80_poly2": with_option("attn_tc", 0, lambda: check_self_attention(B=2, N=1024, C=640, seed=126), 1),
    "self_attn_d40_psmem": lambda: check_self_attention(B=1, N=4096, C=320, seed=130),
    "self_attn_d40_psmem_ragged": with_option("attn_tc", 0, lambda: check_self_attention(B=3, N=700, C=320, seed=127), 1),
    "self_attn_d80_psmem": lambda: check_self_attention(B=2, N=1100, C=640, seed=129),
    "cross_attn_d40_psmem": lambda: check_cross_attention(B=2, Fr=4, N=1024, C=320, seed=134),
    "cross_attn_d80_psmem": with_option("attn_tc", 0, lambda: check_cross_attention(B=2, Fr=8, N=1024, C=640, seed=133), 1),
    "self_attn_d40_mufu_only": lambda: check_self_attention(B=2, N=1024, C=320, seed=122),
    "self_attn_d40_free_running": with_option("attn_tc", 0, lambda: check_self_attention(B=2, N=1024, C=320, seed=122), 1),
    "self_attn_d40_softmax_epilogue": lambda: check_self_attention(B=2, N=4095, C=320, seed=131),
    "cross_attn_d40_softmax_epilogue": with_option("attn_tc", 0, lambda: check_cross_attention(B=2, Fr=4, N=1024, C=320, seed=134), 1),
    "self_attn_d40_many_items": lambda: check_self_attention(B=2, N=6144, C=320, seed=128),
    "self_attn_d80_many_items_odd_tiles": lambda: check_self_attention(B=6, N=1100, C=640, seed=129),     # nkt = 18, 5 q blocks
    "cross_attn_d80_many_items": lambda: check_cross_attention(B=2, Fr=8, N=1024, C=640, seed=133),
    # epilogue sub-tile counts, residual adds and partial column tiles at several BN
    "gemm_bn160_prefetch": with_option("gemm_stages", 3, lambda: check_gemm(512, 320, 320), 0),
    "gemm_residual_prefetch": with_option("gemm_stages", 4, lambda: check_gemm(128 * 150 + 9, 1280, 320, residual=True, seed=8), 0),
    "gemm_pair_prefetch": with_option("gemm_stages", 3, lambda: check_gemm(128 * 5 + 9, 1280, 1024, seed=13), 0),
    "conv3x3_epi_prefetch": with_option("gemm_stages", 4, lambda: check_conv3x3(rowvec=True, residual=True), 0),
    "ln_fuse_res_prefetch": with_option("gemm_stages", 3, lambda: check_linear_ln_linear(rows=128 * 150 + 37, residual=True, N=320, seed=161, mean=2.0), 0),
    "gemm_bn128_tail_prefetch": with_option("gemm_stages", 4, lambda: check_gemm(300, 768, 320, bn=128), 0),
    # residual epilogue: ragged M (rows outside the problem must not be touched), partial last column tile, conv geometry
    "gemm_residual_respf1": with_option("gemm_stages", 3, lambda: check_gemm(128 * 150 + 9, 1280, 320, residual=True, seed=8), 0),
    "gemm_residual_respf2": lambda: check_gemm(128 * 150 + 9, 1280, 320, residual=True, bn=128, seed=18),
    "gemm_residual_k320_respf1": with_option("gemm_stages", 3, lambda: check_gemm(128 * 301 + 77, 320, 320, residual=True, seed=21), 0),
    "gemm_residual_k320_respf2": with_option("gemm_stages", 4, lambda: check_gemm(128 * 301 + 77, 320, 320, residual=True, seed=21), 0),
    "gemm_residual_n96_respf2": lambda: check_gemm(128 * 3 + 5, 96, 320, residual=True, seed=22),
    "gemm_pair_residual_respf1": with_option("gemm_stages", 3, lambda: check_gemm(128 * 5 + 9, 1280, 1024, residual=True, seed=13), 0),
    "gemm_pair_residual_respf2": with_option("gemm_stages", 4, lambda: check_gemm(128 * 5 + 9, 1280, 1024, residual=True, seed=13), 0),
    "conv3x3_respf1": lambda: check_conv3x3(n=4, H=24, W=40, rowvec=True, residual=True, seed=41),
    "conv3x3_respf2": lambda: check_conv3x3(n=2, H=32, W=32, ci=640, co=640, rowvec=True, residual=True, seed=42),
    "ln_fuse_res_respf2": with_option("gemm_stages", 4, lambda: check_linear_ln_linear(rows=128 * 150 + 37, residual=True, N=320, seed=161, mean=2.0), 0),
    # residual epilogue with many tiles per CTA, ragged M, a partial last column tile (different sub-tile counts of
    # consecutive tiles), every BN, and short to long K
    "gemm_resst_l0_full": lambda: check_gemm(131072, 320, 320, residual=True, seed=31),
    "gemm_resst_ragged_many_tiles": lambda: check_gemm(128 * 901 + 77, 320, 320, residual=True, seed=32),
    "gemm_resst_n96_partial_tile": lambda: check_gemm(128 * 40 + 5, 96, 320, residual=True, seed=33),
    "gemm_resst_n224_bn160_partial": lambda: check_gemm(128 * 333 + 1, 224, 256, residual=True, bn=160, seed=34),
    "gemm_resst_bn128": lambda: check_gemm(128 * 300 + 9, 640, 320, residual=True, bn=128, seed=35),
    "gemm_resst_bn64": lambda: check_gemm(128 * 300 + 9, 320, 320, residual=True, bn=64, seed=36),
    "gemm_resst_k64": lambda: check_gemm(32768, 320, 64, residual=True, seed=37),
    "gemm_res_k384_register_path": lambda: check_gemm(4096, 320, 384, residual=True, seed=38),
    "gemm_res_k1280_register_path": lambda: check_gemm(32768, 320, 1280, residual=True, seed=40),
    "gemm_res_pair_k1024_register_path": lambda: check_gemm(128 * 64 + 9, 1280, 1024, residual=True, seed=39),
    "gemm_resst_off_register_path": lambda: check_gemm(128 * 302 + 1, 320, 320, residual=True, seed=23),
    "ln_fuse_res_resst_many_tiles": lambda: check_linear_ln_linear(rows=128 * 700 + 37, residual=True, N=320, seed=162, mean=2.0),
    "ln_fuse_res_resst_off": lambda: check_linear_ln_linear(rows=128 * 151 + 5, residual=True, N=320, seed=165, mean=-2.0),
    "gemm_bn160": lambda: check_gemm(512, 320, 320),
    "gemm_bn128_tail": lambda: check_gemm(300, 768, 320, bn=128),
    "gemm_bn64": lambda: check_gemm(130, 64, 128, bn=64),
    "gemm_residual": lambda: check_gemm(1024, 1280, 1280, residual=True),
    "gemm_small_m": lambda: check_gemm(77, 640, 768),
    "gemm_big_k": lambda: check_gemm(256, 320, 5120),
    "gemm_many_tiles": lambda: check_gemm(128 * 150 + 5, 320, 64),
    "gemm_qkv_rows": lambda: check_gemm(40000, 960, 320, residual=True, seed=5),
    "gemm_k64": lambda: check_gemm(128 * 300 + 77, 640, 64, bias=False, seed=6),
    "geglu_rows": lambda: check_geglu(M=20000, C=320, seed=31),
    "gemm_concat": check_gemm_concat,
    "gemm_rowvec": check_gemm_rowvec,
    "geglu": check_geglu,
    "conv3x3": lambda: check_conv3x3(),
    "conv3x3_epi": lambda: check_conv3x3(rowvec=True, residual=True),
    "conv3x3_w64": lambda: check_conv3x3(n=2, H=64, W=64, ci=64, co=160),
    "conv3x3_small": lambda: check_conv3x3(n=2, H=2, W=2, ci=1280, co=1280),
    "conv3x3_1x1": lambda: check_conv3x3(n=4, H=1, W=1, ci=1280, co=1280),
    "conv3x3_odd": lambda: _conv_odd(3, 7, 12, 320, 320, 55),
    "conv3x3_concat": check_conv3x3_concat,
    "conv_out": check_conv_out,
    "conv_s2": check_conv_s2,
    "conv_in": check_conv_in,
    "upsample_conv_subpixel": check_upsample_conv,
    "upsample_conv_subpixel_odd": lambda: check_upsample_conv(n=3, H=7, W=12, ci=320, co=320, seed=76),
    "upsample_conv_subpixel_1280": lambda: check_upsample_conv(n=4, H=16, W=16, ci=1280, co=1280, seed=77),
    "upsample": check_upsample,
    "gn5d_silu": lambda: check_groupnorm(),
    "gn5d_concat": lambda: check_groupnorm(c1=640, c2=320),
    "gn_frame": lambda: check_groupnorm(per_frame=True, silu=False, eps=1e-6),
    "gn5d_1280": lambda: check_groupnorm(B=1, Fr=2, H=4, W=4, c1=1280, c2=1280),
    # headline sizes: one statistics set = 16 frames x 64 x 64 x 10 channels = 655 360 elements with a mean 2-4x the spread
    "gn5d_c2_l0_mean3": lambda: check_groupnorm(B=2, Fr=16, H=64, W=64, c1=320, mean=3.0, seed=101),
    "gn5d_c2_l0_concat": lambda: check_groupnorm(B=1, Fr=16, H=64, W=64, c1=320, c2=320, mean=-6.0, seed=102),
    "gn5d_silu_stats_v2": with_option("gn_stats_v2", 1, lambda: check_groupnorm(), 0),
    "gn5d_concat_stats_v2": with_option("gn_stats_v2", 1, lambda: check_groupnorm(c1=640, c2=320), 0),
    "gn5d_c2_l0_mean3_stats_v2": with_option("gn_stats_v2", 1, lambda: check_groupnorm(B=2, Fr=16, H=64, W=64, c1=320, mean=3.0, seed=101), 0),
    # per-frame GroupNorm, single pass in a thread-block cluster: 16 / 8 / 4 / 1 CTAs per image, SiLU variant, and the
    # two-kernel path behind "gn_fused" = 0 (also taken when an image does not fit: 96x96 at 320 channels = 5.9 MB)
    "gn_frame_fused_l1": with_option("gn_fused", 1, lambda: check_groupnorm(B=2, Fr=3, H=32, W=32, c1=640, per_frame=True, silu=False, eps=1e-6, mean=-1.0, seed=104), 1),
    "gn_frame_fused_l0_cluster16": with_option("gn_fused", 1, lambda: check_groupnorm(B=2, Fr=4, H=64, W=64, c1=320, per_frame=True, silu=False, eps=1e-6, mean=2.0, seed=103), 1),
    "gn_frame_fused_l2": lambda: check_groupnorm(B=2, Fr=3, H=16, W=16, c1=1280, per_frame=True, silu=False, eps=1e-6, mean=0.5, seed=105),
    "gn_frame_fused_l3_silu": lambda: check_groupnorm(B=2, Fr=3, H=8, W=8, c1=1280, per_frame=True, silu=True, eps=1e-6, seed=106),
    "gn_frame_fused_odd": lambda: check_groupnorm(B=1, Fr=3, H=7, W=12, c1=320, per_frame=True, silu=False, eps=1e-6, seed=107),
    "gn_frame_two_kernels": with_option("gn_fused", 0, lambda: check_groupnorm(B=2, Fr=4, H=64, W=64, c1=320, per_frame=True, silu=False, eps=1e-6, mean=2.0, seed=103), 1),
    "gn_frame_too_large_for_cluster": lambda: check_groupnorm(B=1, Fr=2, H=96, W=96, c1=320, per_frame=True, silu=False, eps=1e-6, seed=108),
    "gn_frame_l0": lambda: check_groupnorm(B=2, Fr=4, H=64, W=64, c1=320, per_frame=True, silu=False, eps=1e-6, mean=2.0, seed=103),
    "ln_fold_qkv_320": lambda: check_ln_linear(),
    "ln_fold_qkv_pe_640": lambda: check_ln_linear(rows=1280, C=640, N=1920, pe=True, seed=116, hw=64),   # one frame per warp
    "ln_fold_q_1280": lambda: check_ln_linear(rows=700, C=1280, N=1280, seed=117),
    "ln_fold_geglu_320": lambda: check_ln_linear(rows=1500, C=320, N=2560, geglu=True, seed=118),
    "ln_fold_pe_mixed_warps": lambda: check_ln_linear(rows=40 * 7, C=320, N=960, pe=True, seed=119),
    # LayerNorm statistics emitted by the producing GEMM's epilogue (2 / 3 / 5 column tiles, residual, ragged rows, GEGLU)
    "ln_fuse_320_proj_in": lambda: check_linear_ln_linear(),
    "ln_fuse_320_res": lambda: check_linear_ln_linear(rows=128 * 150 + 37, residual=True, N=320, seed=161, mean=2.0),
    "ln_fuse_640_res_geglu": lambda: check_linear_ln_linear(rows=3000, K0=640, C=640, N=5120, residual=True, geglu=True, seed=162),
    "ln_fuse_1280_res": lambda: check_linear_ln_linear(rows=700, K0=1280, C=1280, N=3840, residual=True, seed=163, mean=-1.5),
    "ln_fuse_1280_pair": lambda: check_linear_ln_linear(rows=8192, K0=1280, C=1280, N=1280, residual=True, seed=164),
    "ln_320": lambda: check_layernorm(C=320),
    "ln_1280_pe": lambda: check_layernorm(rows=640, C=1280, pe=True),
    "self_attn_d40": lambda: check_self_attention(C=320),
    "self_attn_d80": lambda: check_self_attention(B=2, N=64, C=640),
    "self_attn_d160": lambda: check_self_attention(B=2, N=130, C=1280),
    "self_attn_tiny": lambda: check_self_attention(B=2, N=4, C=320),
    "self_attn_d40_n600": lambda: check_self_attention(B=2, N=600, C=320, seed=121),
    "self_attn_d40_n1024": lambda: check_self_attention(B=1, N=1024, C=320, seed=122),
    "self_attn_d80_n300": lambda: check_self_attention(B=2, N=300, C=640, seed=123),
    # the launch that is 88 % of the attention FLOPs of the benchmark: N = 4096 keys (64 key tiles), d = 40
    "self_attn_d40_n4096": lambda: check_self_attention(B=2, N=4096, C=320, seed=124),
    "self_attn_d40_n5376": lambda: check_self_attention(B=1, N=5376, C=320, seed=125),     # 448x768 video: 56x96 latent
    "self_attn_d80_n1024": lambda: check_self_attention(B=2, N=1024, C=640, seed=126),
    "cross_attn_d40_n4096": lambda: check_cross_attention(B=1, Fr=2, N=4096, C=320, seed=132),
    "self_attn_d40_mma": lambda: check_self_attention_mma(C=320),
    "self_attn_d80_mma": lambda: check_self_attention_mma(B=2, N=64, C=640),
    "cross_attn_d40": lambda: check_cross_attention(B=2, Fr=2, N=300, C=320, seed=131),
    "cross_attn": check_cross_attention,
    "temporal_attn_d40": lambda: check_temporal_attention(C=320),
    "temporal_attn_d40_scalar_stores": with_option("tattn_vst", 0, lambda: check_temporal_attention(C=320), 1),
    "temporal_attn_d80_f16": lambda: check_temporal_attention(B=2, Fr=16, HW=33, C=640, seed=141),
    "temporal_attn_d160_f3": lambda: check_temporal_attention(B=1, Fr=3, HW=7, C=1280),
    "temporal_attn_f24": lambda: check_temporal_attention(B=1, Fr=24, HW=5, C=640),
    "cfg_ddim_f16": lambda: check_cfg_ddim(torch.float16),
    "cfg_ddim_f32": lambda: check_cfg_ddim(torch.float32),
}
