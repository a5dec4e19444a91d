"""Per-element checks of the CLIP causal attention (causal_attn_kernel) and the quick-GELU GEMM epilogue against fp64 math
on the same fp16 inputs.  Kernel-agnostic like tests/attention_probes.py: the checks take the kernel as a callable, so
the same checks run the CUDA kernels (tests/test_text_encoder_gpu.py) and torch emulations of their arithmetic with
planted bugs (tests/test_text_encoder_cpu.py).

Causal attention.  qkv [n L, 3 C] (C = 12 heads x 64).  One-hot value probes: for sequence s, head h and channel c,
V[s, j, h 64 + c] = 1 for the probed key j = (c + 64 h + 7 s) % L and 0 otherwise, so out[s, i, h 64 + c] is the single
probability P_h[i, j] -- every key of every sequence is probed in every head.  The kernel computes
out = fp16(fp16(p~_j) / l) with the exact row maximum (A_j = 1 in the notation of attention_probes.py), so the bound of
the fused kernels applies unchanged: |out - p| <= (2^-9 + 2^-15) p + 2^-24 max_row(p) + 2^-24.  A probe of a future key
(j > i) must read exactly 0.

Quick-GELU epilogue.  y = fp16(v / (1 + 2^t)), t = min(-1.702 log2(e) v, 64), v = acc + bias in fp32: the activation is
within 2^-16.9 relative (common.cuh quick_gelu_f) and the output rounding adds 2^-11 relative or 2^-25 absolute below
2^-14, so |y - quick_gelu(v)| <= (2^-11 + 2^-16) |quick_gelu(v)| + 2^-25."""
from __future__ import annotations

import math

import torch

from tests import attention_probes as A

HEADS, D = 12, 64
C = HEADS * D
QG_REL, QG_FLOOR = 2.0 ** -11 + 2.0 ** -16, 2.0 ** -25


# ---------------------------------------------------------------------------------------------------- causal attention
def causal_qk(n, L, sigma=1.0, shift=0.0, sink=0.0, tail=False, seed=0):
    """q, k [n, L, C] fp16 with logits q.k / 8 of standard deviation sigma per head.  shift: head coordinate 0 adds +-shift
    to every logit of a row (the softmax is unchanged).  sink: head coordinate 1 adds `sink` to the logit of key 0 (an
    "attention sink" as real CLIP has).  tail: every real logit equals -20, so a padding key (logit 0) that leaks in takes
    ~all the mass."""
    g = torch.Generator().manual_seed(seed)
    if tail:
        q = torch.zeros(n, L, C)
        q[..., ::D] = float(torch.tensor(20.0 * 8 / 4).half())
        k = torch.randn(n, L, C, generator=g)
        k[..., ::D] = -4.0
        return q.half(), k.half()
    s = math.sqrt(sigma)
    q = torch.randn(n, L, C, generator=g) * s
    k = torch.randn(n, L, C, generator=g) * s
    if shift:
        q[..., ::D] = float(torch.tensor(shift * 8 / 8.0).half()) * (torch.randint(0, 2, (n, L, 1), generator=g) * 2.0 - 1.0)
        k[..., ::D] = 8.0
    if sink:
        q[..., 1::D] = float(torch.tensor(sink).half())
        k[..., 1::D] = 0.0
        k[:, 0, 1::D] = 8.0
    return q.half(), k.half()


def causal_probs(q, k):
    """fp64 softmax(q k^T / 8) with key j visible to query i iff j <= i: [n, heads, L, L]."""
    n, L, _ = q.shape
    qh = q.double().reshape(n, L, HEADS, D).transpose(1, 2)
    kh = k.double().reshape(n, L, HEADS, D).transpose(1, 2)
    s = qh @ kh.transpose(-1, -2) / 8.0
    mask = torch.triu(torch.ones(L, L, dtype=torch.bool, device=q.device), 1)
    return torch.softmax(s.masked_fill(mask, -math.inf), -1)


def probe_sel(n, L):
    """The probed key of every (sequence, head, channel): [n, heads, 64]."""
    return (torch.arange(HEADS * D).reshape(1, HEADS, D) + 7 * torch.arange(n).reshape(n, 1, 1)) % L


def check_causal(attn, n, L, sigmas=(1.0, 3.0, 6.0), shift=0.0, sink=0.0, tail=False, seed=0, dev="cuda"):
    """attn(qkv [n L, 3 C] fp16, n, L) -> [n L, C]: every key probed in every head, future keys exactly 0."""
    rs = []
    for i, sigma in enumerate((1.0,) if tail else sigmas):
        q, k = causal_qk(n, L, sigma, shift, sink, tail, seed + i)
        sel = probe_sel(n, L)
        v = A.one_hot_v(sel, L)
        qkv = torch.cat([q, k, v], -1).reshape(n * L, 3 * C).to(dev)
        out = attn(qkv, n, L).reshape(n, L, C).cpu()
        P = causal_probs(q, k)
        ref, pmax = A.probe_ref(P, sel)
        rs.append(A.compare(out, ref, pmax, what=f"L {L} sigma {sigma} shift {shift} sink {sink} tail {tail}"))
        future = sel.reshape(n, 1, C) > torch.arange(L).reshape(1, L, 1)
        rs.append(A.flag(bool((out[future.expand(n, L, C)] == 0).all()), f"a future key has weight (L {L})"))
        if sink:
            rs.append(A.flag(bool((P[:, :, 1:, 0] >= 0.9).all()), "the sink holds less than 90 % of the mass"))
    return A.merge(*rs)


# ---------------------------------------------------------------------------------------------------- quick-GELU
def quick_gelu64(v):
    v = v.double()
    return v * torch.sigmoid(1.702 * v)


def qgelu_inputs():
    """Every finite fp16 value in [-20, 20], then a spread out to +-65504 (fp16)."""
    allh = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    allh = allh[torch.isfinite(allh) & (allh.float().abs() <= 20)]
    big = torch.logspace(math.log10(20.0), math.log10(65504.0), 4000, dtype=torch.float64).half()
    return torch.cat([allh, big, -big, torch.tensor([65504.0, -65504.0]).half()])


def compare_qgelu(out, v32):
    """out fp16 against quick_gelu(v32) in fp64, per element."""
    ref = quick_gelu64(v32)
    o = out.double()
    bound = QG_REL * ref.abs() + QG_FLOOR
    finite = bool(torch.isfinite(o).all())
    err = ((o - ref).abs() / bound).max().item() if finite else math.inf
    return {"err": err, "tol": 1.0, "ok": finite and err <= 1.0, "what": "quick-GELU"}
