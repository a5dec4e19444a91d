"""Per-element attention checks: one-hot value probes, masked-tail problems and the explicit-probability pair against an
fp64 softmax of the same fp16 inputs.  Kernel-agnostic: every check takes the kernel as a callable, so the same checks
run the CUDA kernels (tests/test_attention_probes_gpu.py) and a torch emulation of their arithmetic with planted bugs
(tests/test_attention_probes_cpu.py).

One-hot value probes.  For head h and channel c, V[j(h, c), h d + c] = 1 and every other value is 0.  Then
out[:, h d + c] is P_h[:, j(h, c)], one probability per output element, read with relative precision instead of being
averaged with thousands of others.

Bound of the fused kernels (attention_tc.cu, attention.cu: attn_kernel and tattn_kernel).  With one-hot V, an output is
    out = fp16( fp16(p~_j) * A_j / l )
where p~_j = exp2(s_j sc - m_t sc) is the weight relative to the running maximum m_t of the key tile t holding key j,
A_j <= 1 the product of the rescale factors of the later tiles and l the fp32 normaliser in units of the final maximum
(l >= 1: the maximum key contributes 1).  Its error against the fp64 probability p = exp(s_j / sqrt(d) - ...) / sum:
  * P rounded to fp16: 2^-11 p, or, once p~_j is subnormal (< 2^-14), 2^-25 absolute in units of the running maximum,
    i.e. at most 2^-25 A_j / l <= 2^-25 max_row(p) after normalisation (max_row(p) = 1 / l);
  * the output rounded to fp16: 2^-11 p, or 2^-25 absolute below 2^-14;
  * exp2: ex2.approx.ftz.f32 (wgmma kernel) is within ~2^-22 relative, exp2f (mma.sync kernels) within 2 ulp; the
    argument s sc - m sc is formed from fp32 scores whose rounding is < 2^-16 relative to the largest logit here;
  * l: fp32 sums of <= 32 terms per thread, one update per key tile and two shuffles: < 2^-17 relative at 4096 keys,
    and the rescale factors hit O and l alike, so their ex2 error cancels.
Together: |out - p| <= (2^-10 + 2^-16) p + 2^-25 max_row(p) + 2^-25.  The comparator allows twice that,
    |out - p| <= (2^-9 + 2^-15) p + 2^-24 max_row(p) + 2^-24,
so a faithful kernel sits at <= 1/2 of the bound (two fp16 roundings of 2^-11 each can coincide; they do, within 2 %,
over the millions of probed elements of a sweep).  A planted 0.3 % error in the normaliser or a P rounded to bf16
(2^-8) still exceeds it; tests/test_attention_probes_cpu.py shows both on an emulation of the wgmma kernel.

attn_probs_kernel writes fp16(exp2((s - m) sc) / l) with the exact row maximum m: one rounding, so (2^-11 + 2^-16) p + 2^-25
with the same small terms; the comparator allows twice that.  attn_pv_kernel multiplies fp16 P and V exactly
into fp32 and adds: < (nk / 16 + 16) 2^-24 sum_j |p_j v_j| for the accumulator updates and the 16-term sums inside an
MMA, then one fp16 rounding of the output; doubled likewise.  With a one-hot V it adds one product to zeros, so its output
is P itself, bit for bit."""
from __future__ import annotations

import math

import torch

HEADS = 8
DEV = "cuda"                                      # where the checks put their inputs unless told otherwise
BKV_TC, STAGES_TC = 128, {40: 4, 80: 3}           # TCfg<D> in attention_tc.cu (test_attn_sass_cpu.py pins them)
BKV_MMA = 64                                      # ACfg<D>::BKV in attention.cu

REL, FLOOR = 2 * (2.0 ** -10 + 2.0 ** -16), 2.0 ** -24       # fused kernels (module docstring)
PROBS_REL = 2 * (2.0 ** -11 + 2.0 ** -16)                    # attn_probs_kernel: one fp16 rounding
PV_REL = 2 * 2.0 ** -11                                      # attn_pv_kernel: the output rounding ...


def pv_extra(nk):
    """... and the fp32 accumulation, per unit of sum_j |p_j v_j| (module docstring)."""
    return 2 * (nk / 16 + 16) * 2.0 ** -24


# ---------------------------------------------------------------------------------------------------- comparators
def compare(out, ref, pmax=0.0, rel=REL, extra=0.0, what=""):
    """|out - ref| <= rel |ref| + FLOOR pmax + FLOOR + extra per element; err = the largest err / bound."""
    out64, ref = out.double(), ref.double()
    bound = rel * ref.abs() + FLOOR * pmax + FLOOR + extra
    finite = bool(torch.isfinite(out64).all().item())
    ratio = ((out64 - ref).abs() / bound).max().item() if finite else math.inf
    return {"err": ratio, "tol": 1.0, "ref": ref.abs().max().item(), "ok": finite and ratio <= 1.0, "what": what}


def flag(ok, what):
    return {"err": 0.0 if ok else math.inf, "tol": 1.0, "ref": 0.0, "ok": bool(ok), "what": what}


def merge(*rs):
    """The worst sub-result (largest err / bound), ok only if every one is."""
    r = dict(max(rs, key=lambda x: x["err"]))
    r["ok"] = all(x["ok"] for x in rs)
    return r


# ---------------------------------------------------------------------------------------------------- references
def ref_probs(q, k, heads=HEADS, kv_div=1):
    """fp64 softmax(q k^T / sqrt(d)) of the fp16 inputs: [B, heads, nq, nk]; query batch b reads K batch b // kv_div."""
    B, nq, C = q.shape
    d = C // heads
    qh = q.double().reshape(B, nq, heads, d).transpose(1, 2)
    kh = k.double().reshape(k.shape[0], -1, heads, d).transpose(1, 2).repeat_interleave(kv_div, 0)
    return torch.softmax(qh @ kh.transpose(-1, -2) / math.sqrt(d), -1)


def probe_keys(Bk, d, nk, keys=None, offset=0):
    """The probed key of every (K/V batch, head, channel), [Bk, heads, d]: consecutive keys from `offset` (a sweep), or
    the listed keys in turn.  Successive K/V batches continue the sequence, so a frame that reads the wrong K/V batch
    reads other keys of other maps."""
    idx = torch.arange(Bk * HEADS * d).reshape(Bk, HEADS, d) + offset
    if keys is None:
        return idx % nk
    keys = torch.tensor(sorted(set(keys)))
    return keys[idx % len(keys)]


def one_hot_v(sel, nk):
    """V [Bk, nk, heads d] fp16 with V[b, sel[b, h, c], h d + c] = 1, zero elsewhere."""
    Bk, H, d = sel.shape
    v = torch.zeros(Bk, nk, H * d)
    v.scatter_(1, sel.reshape(Bk, 1, H * d), 1.0)
    return v.half()


def probe_ref(P, sel, kv_div=1):
    """What the probed output must be: out[b, :, h d + c] = P[b, h, :, sel[b // kv_div, h, c]], and max_row(p) per
    element."""
    B, H, nq, _ = P.shape
    d = sel.shape[2]
    s = sel.to(P.device).repeat_interleave(kv_div, 0)
    ref = P.gather(-1, s[:, :, None, :].expand(B, H, nq, d)).permute(0, 2, 1, 3).reshape(B, nq, H * d)
    pmax = P.amax(-1).permute(0, 2, 1)[..., None].expand(B, nq, H, d).reshape(B, nq, H * d)
    return ref, pmax


def edge_keys(nk, d):
    """Keys on the edges of both kernels' schedules: tile edges of 64 and 128, both sides of the wgmma ring wrap,
    the first key of the last tile, the last key."""
    ks = {0, 1, 63, 64, 127, 128, nk - 1, BKV_MMA * ((nk - 1) // BKV_MMA), BKV_TC * ((nk - 1) // BKV_TC)}
    if d in STAGES_TC:
        ks |= {BKV_TC * STAGES_TC[d] - 1, BKV_TC * STAGES_TC[d]}
    return sorted(x for x in ks if x < nk)


# ---------------------------------------------------------------------------------------------------- inputs
def random_qk(B, nq, nk, d, sigma=1.0, kv_div=1, shift=0.0, seed=0):
    """fp16 q [B, nq, heads d], k [B / kv_div, nk, heads d] with logits q.k / sqrt(d) of standard deviation sigma.  Each
    K batch is drawn independently, so each frame group has its own maps.  shift != 0: head coordinate 0 is
    q = +-alpha (sign per query) and k = beta for every key, which adds +-shift to every logit of a row and leaves the
    softmax unchanged: the kernels must subtract the row maximum before exp2."""
    g = torch.Generator().manual_seed(seed)
    s = math.sqrt(sigma)
    q = torch.randn(B, nq, HEADS * d, generator=g) * s
    k = torch.randn(B // kv_div, nk, HEADS * d, generator=g) * s
    if shift:
        beta = 8.0
        alpha = float(torch.tensor(shift * math.sqrt(d) / beta).half())
        sign = torch.randint(0, 2, (B, nq, 1), generator=g) * 2.0 - 1.0
        q[..., ::d] = alpha * sign
        k[..., ::d] = beta
    return q.half(), k.half()


def tail_qk(B, nq, nk, d, kv_div=1, seed=0):
    """Every real key has the same logit, a b / sqrt(d) ~ -20: q = a e_0 per head, k[:, e_0] = -b, other q coordinates
    0.  The softmax is exactly uniform, so a zero-filled padding key (logit 0) that leaks in takes ~all the mass."""
    g = torch.Generator().manual_seed(seed)
    b = 4.0
    a = float(torch.tensor(20.0 * math.sqrt(d) / b).half())
    q = torch.zeros(B, nq, HEADS * d)
    q[..., ::d] = a
    k = torch.randn(B // kv_div, nk, HEADS * d, generator=g)
    k[..., ::d] = -b
    return q.half(), k.half()


# ---------------------------------------------------------------------------------------------------- checks
def check_probes(attn, B, nq, nk, d, sigmas=(1.0,), kv_div=1, sweep=False, shift=0.0, tail=False, seed=0, dev=None):
    """One-hot probes of spatial / cross attention.  attn(q, k, v, heads, kv_div) -> out.  sweep: enough launches that
    every key of every map is probed once; otherwise the edge keys, each in many heads and channels."""
    dev = dev or DEV
    rs = []
    for i, sigma in enumerate(sigmas):
        if tail:
            q, k = tail_qk(B, nq, nk, d, kv_div, seed + i)
        else:
            q, k = random_qk(B, nq, nk, d, sigma, kv_div, shift, seed + i)
        q, k = q.to(dev), k.to(dev)
        P = ref_probs(q, k, HEADS, kv_div)
        Bk = k.shape[0]
        per = Bk * HEADS * d
        launches = -(-nk // per) if sweep else 1
        seen = torch.zeros(nk, dtype=torch.bool)
        for L in range(launches):
            sel = probe_keys(Bk, d, nk, None if sweep else edge_keys(nk, d), offset=L * per)
            seen[sel.flatten()] = True
            out = attn(q, k, one_hot_v(sel, nk).to(dev), HEADS, kv_div)
            ref, pmax = probe_ref(P, sel, kv_div)
            rs.append(compare(out, ref, pmax, what=f"sigma {sigma} launch {L}"))
        want = seen.all() if sweep else seen[edge_keys(nk, d)].all()
        rs.append(flag(bool(want), "a key was not probed"))
        del P
    return merge(*rs)


def temporal_qkv(B, F, HW, d, sigma=1.0, shift=0.0, seed=0):
    """qkv [B, F, HW, 3 heads d] fp16 with one-hot V: head h, channel c reads frame (c + h) % F (d >= 40 > F: every
    frame of every map in one launch)."""
    C = HEADS * d
    q, k = random_qk(B * HW, F, F, d, sigma, 1, shift, seed)                  # [B HW, F, C] each
    sel = (torch.arange(d)[None, :] + torch.arange(HEADS)[:, None]) % F       # [heads, d]
    v = one_hot_v(sel[None].expand(B * HW, HEADS, d).contiguous(), F)
    t = torch.cat([q, k, v], -1).reshape(B, HW, F, 3 * C).permute(0, 2, 1, 3).contiguous()
    return t, sel


def check_temporal_probes(tattn, B, F, HW, d, sigmas=(1.0, 3.0, 6.0), shift=0.0, seed=0, dev=None):
    """tattn(qkv, heads) -> [B, F, HW, C]: attention over the F frames of every pixel, probed at every frame."""
    dev = dev or DEV
    rs = []
    C = HEADS * d
    for i, sigma in enumerate(sigmas):
        qkv, sel = temporal_qkv(B, F, HW, d, sigma, shift, seed + i)
        qkv = qkv.to(dev)
        out = tattn(qkv, HEADS)
        t = qkv.permute(0, 2, 1, 3).reshape(B * HW, F, 3 * C)
        P = ref_probs(t[..., :C], t[..., C:2 * C])
        ref, pmax = probe_ref(P, sel[None].expand(B * HW, HEADS, d))
        ref = ref.reshape(B, HW, F, C).permute(0, 2, 1, 3)
        pmax = pmax.reshape(B, HW, F, C).permute(0, 2, 1, 3)
        rs.append(compare(out, ref, pmax, what=f"F {F} d {d} sigma {sigma} shift {shift}"))
    return merge(*rs)


def check_probs(probs_fn, B, nq, nk, d, kv_div=1, sigmas=(1.0, 3.0), tail=False, seed=0, dev=None):
    """probs_fn(q, k, heads, kv_div) -> [B, heads, nq, nk] fp16 against the fp64 softmax, element by element."""
    dev = dev or DEV
    rs = []
    for i, sigma in enumerate(sigmas):
        q, k = tail_qk(B, nq, nk, d, kv_div, seed + i) if tail else random_qk(B, nq, nk, d, sigma, kv_div, 0.0, seed + i)
        q, k = q.to(dev), k.to(dev)
        probs = probs_fn(q, k, HEADS, kv_div)
        rs.append(compare(probs, ref_probs(q, k, HEADS, kv_div), rel=PROBS_REL, what=f"probs sigma {sigma}"))
    return merge(*rs)


EDITS = ("scaled_rows", "zero_row", "zero_column", "refine_mix", "random_rows")


def edited_maps(P, kind, g):
    """A controller-style edit of fp16 maps [B, heads, nq, nk]: rows that no longer sum to 1, zero rows and columns, a
    refine-style word-column mix (AttentionRefine: base[..., mapper] alpha + edit (1 - alpha)), non-negative noise."""
    P = P.clone()
    nk = P.shape[-1]
    if kind == "scaled_rows":
        P[:, :, ::3] *= 2
    elif kind == "zero_row":
        P[:, :, 1::5] = 0
    elif kind == "zero_column":
        P[..., nk // 3] = 0
        P[..., nk - 1] = 0
    elif kind == "refine_mix":
        mapper = torch.randperm(nk, generator=g).to(P.device)
        alpha = (torch.rand(nk, generator=g) < 0.5).to(P.device, torch.float32)
        P = (P.float()[..., mapper] * alpha + P.float() * (1 - alpha)).half()
    elif kind == "random_rows":
        P = (torch.rand(P.shape, generator=g) * (4.0 / nk)).to(P.device).half()
    return P


def check_apply_probs(apply_fn, B, nq, nk, d, kv_div=1, seed=0, dev=None):
    """apply_fn(probs, v, heads, kv_div) -> [B, nq, heads d] on edited maps: against fp64 P V for random V (the kernel
    must not renormalise), and bit-identical to the probed columns of P for a one-hot V."""
    dev = dev or DEV
    g = torch.Generator().manual_seed(seed)
    q, k = random_qk(B, nq, nk, d, 3.0, kv_div, 0.0, seed)
    P0 = ref_probs(q, k, HEADS, kv_div).to(dev).half()
    v = torch.randn(B // kv_div, nk, HEADS * d, generator=g).half().to(dev)
    sel = probe_keys(B // kv_div, d, nk)
    vo = one_hot_v(sel, nk).to(dev)
    vh = v.double().reshape(B // kv_div, nk, HEADS, d).transpose(1, 2).repeat_interleave(kv_div, 0)
    rs = []
    for kind in EDITS:
        P = edited_maps(P0, kind, g)
        out = apply_fn(P, v, HEADS, kv_div)
        ref = (P.double() @ vh).transpose(1, 2).reshape(B, nq, HEADS * d)
        mag = (P.double() @ vh.abs()).transpose(1, 2).reshape(B, nq, HEADS * d)
        rs.append(compare(out, ref, rel=PV_REL, extra=pv_extra(nk) * mag, what=f"P V, {kind}"))
        ref1, _ = probe_ref(P.double(), sel, kv_div)
        out1 = apply_fn(P, vo, HEADS, kv_div)
        rs.append(flag(torch.equal(out1, ref1.half()), f"one-hot V does not return the columns of P ({kind})"))
    return merge(*rs)
