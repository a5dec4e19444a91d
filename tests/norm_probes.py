"""Per-element normalisation checks: GroupNorm (5-D sets, frame shards, per-frame cluster kernel and its fallback),
LayerNorm (ln5_kernel, ln_kernel) and the LayerNorm folded into the following GEMM, against fp64 math on the same fp16
inputs.  Kernel-agnostic: every check takes the kernel as a callable, so the same checks run the CUDA kernels
(tests/test_norm_probes_gpu.py) and a torch emulation of their arithmetic with planted bugs (tests/test_norm_probes_cpu.py).

Inputs that make mapping errors large.  Random inputs with one distribution everywhere give every (set, group) the same
statistics to ~0.1 %, so statistics read from the wrong set, group, row or CTA are nearly right.  Here
  * every (set, group) -- every row for LayerNorm -- has its own mean and spread (spread log-uniform in [0.05, 20], mean
    within +-4 spreads), every channel a small offset of its own and every pixel a smooth offset field, so wrong
    statistics are wrong by O(1) in normalised units and a CTA's own slice is not a sample of the whole image;
  * impulse probes: a group holds c0 everywhere and c0 + A at one (pixel, channel).  The impulse normalises to ~sqrt(n),
    every other element to ~-1/sqrt(n); if the statistics lose that pixel the variance collapses to eps and the impulse
    becomes ~A gamma / sqrt(eps); if another group counts it, two groups are wrong.  Each (set, group) of a launch has its
    impulse at another pixel of `edge_pixels` (first / last pixel of every image, shard, block and cluster slice, the
    tails of the 4-way unrolled loops, random pixels) and in another channel (the last channel of a group that splits an
    8-channel vector among them);
  * near-constant groups (spread 1e-3, so var ~ eps) and an exactly constant group (output beta): eps = 1e-5 and 1e-6
    give visibly different outputs;
  * a cancellation sweep: groups / rows with mean / spread = 0, 4, 16, 32, 64, 128, 256.

Bound.  GroupNorm computes y = fp16(silu?(x a + b)), a = rstd gamma, b = beta - mean a, from fp32 sums S = sum x,
Q = sum x^2 (variance Q / n - mean^2).  The sums are shifted (norm.cu gn_unshift): every block of the statistics kernel
(every CTA of the cluster kernel) sums d = x - k with k its first pixel's value at the group's first channel, converts
its partial to S_b = S'_b + m k, Q_b = Q'_b + k (2 S'_b + m k), and adds that to the global (cluster) total.  A shifted
term passes through at most d_loc fp32 additions (its thread's run of 8 channels x pixels, the shared atomics of the
threads holding the group), a block partial through the conversion and at most d_glob more (the global atomics of the
blocks or the ncta cluster partials, times the k frame shards); `gn_schedules` takes both from the launch geometry of
gn_fill / groupnorm_frame_fused with the device's SM count.  With u = 2^-24, per (set, group) from the actual inputs,
A1 = sum|d|, A2 = sum d^2, the largest over the schedules that can run:
    dS <= d_loc u A1 + (d_glob + 3) u (sum|x| + A1),  dQ <= (d_loc + 1) u A2 + (d_glob + 4) u (sum x^2 + A2),
    dmean = dS / n + 2 u |mean|,  dvar = dQ / n + 4 u E[x^2] + 2 |mean| dmean + dmean^2,
    drstd / rstd = the exact interval of 1 / sqrt(var + eps +- dvar) + 3 u (rsqrtf: 2 ulp; var + eps rounded).
Per element, with the exact a* = gamma / sqrt(var + eps):
    E = |x - mean| |a*| drstd + |a*| (1 + drstd) dmean + u (2 |x a*| + 2 |mean a*| + |beta| + |y0*|)
(the fp32 products and FMAs, the |mean a| 2^-24 term being the cancellation of x a against mean a); SiLU multiplies E by
max|silu'| = 1.1 and adds (8 + |y0|) u |silu(y0)| (__expf: ex2.approx of a rounded argument, __fdividef); the fp16 store
adds 2^-11 |y| (2^-25 below 2^-14).  The comparator allows twice that worst case.
LayerNorm (ln5_kernel, ln_kernel, ln_stats_kernel) uses a two-pass variance, sum (x - mean)^2, so dvar = (D + 4) u var +
dmean^2 with D = C / 16 + 8 (a lane's run plus the shuffles) and no cancellation; its apply adds up to five roundings of
|y|-sized terms (and the folded form the |mean a| term of its -mean rstd shift).  The fold from producer slices
(gemm.cu, EPI_F_LN) sums per-column-tile fp32 (sum, sum of squares) and uses an unshifted one-pass variance, with
D = C / 8 + 16 + slices.  The GEGLU fold feeds value and gate to gelu_sig in fp32, so its bound uses their pre-rounding
errors.

Envelope.  Separately from the bound, the product needs |y - y*| <= ulp16(|y*|) + 2^-14.  It is asserted for every
group or row with mean / spread <= 16; the cancellation sweep reports the same ratio at 32 .. 256.

erf-GELU of the GEGLU epilogue (common.cuh gelu_sig): |error| <= 1.2e-5 + 2^-20 max(x, 0) over all fp16 x (the logistic fit
is clamped at |x| = 5: beyond it the result is x / (1 + 2^(+-20.5)) with x clamped at -5), plus the fp16 rounding of the
output.  SiLU (silu_f) is probed through the GroupNorm apply with mean 0, rstd 1, gamma 1, beta 0."""
from __future__ import annotations

import math

import torch

DEV = "cuda"
GROUPS = 32
U = 2.0 ** -24
HALF = 2.0 ** -11           # fp16 rounding, relative
SUB = 2.0 ** -25            # fp16 rounding below 2^-14
FUSED_THREADS, FUSED_CAP = 480, 160 * 1024      # norm.cu kGnFusedThreads and the cluster kernel's per-CTA image bytes
RATIOS = (0.0, 4.0, 16.0, 32.0, 64.0, 128.0, 256.0)
ENVELOPE_MAX_RATIO = 16.0         # asserted up to here; 32 .. 256 are reported


def num_sms(dev):
    dev = torch.device(dev)
    return torch.cuda.get_device_properties(dev).multi_processor_count if dev.type == "cuda" else 132


# ---------------------------------------------------------------------------------------------------- comparators
def ulp16(y):
    """One fp16 ulp of |y| (2^-24 below 2^-14)."""
    e = torch.floor(torch.log2(y.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def compare(out, ref, bound, what=""):
    """|out - ref| <= bound per element; err = the largest err / bound."""
    finite = bool(torch.isfinite(out).all().item())
    ratio = ((out.double() - ref).abs() / bound).max().item() if finite else math.inf
    return {"err": ratio, "tol": 1.0, "ok": finite and ratio <= 1.0, "what": what}


def envelope(out, ref):
    """|out - ref| / (ulp16(ref) + 2^-14), per element."""
    return (out.double() - ref).abs() / (ulp16(ref) + 2.0 ** -14)


def flag(ok, what):
    return {"err": 0.0 if ok else math.inf, "tol": 1.0, "ok": bool(ok), "what": what}


def merge(*rs):
    """The worst sub-result (largest err / bound), ok only if every one is; reports are kept."""
    r = dict(max(rs, key=lambda x: x["err"]))
    r["ok"] = all(x["ok"] for x in rs)
    r["env"] = max(x.get("env", 0.0) for x in rs)
    bad = [x for x in rs if not x["ok"]]
    if bad:
        r["what"] = bad[0]["what"]
    r["report"] = "; ".join(x["report"] for x in rs if x.get("report"))
    return r


# ---------------------------------------------------------------------------------------------------- geometry
def gn_geometry(C, hw, imgs_per_set, nimg, sms):
    """gn_fill: (rows per block, pixels per block, blocks per set)."""
    cv = C // 8
    rows = max(1, 512 // cv)
    pps, nstat = imgs_per_set * hw, nimg // imgs_per_set
    want = -(-4 * sms // nstat)
    ppb = max(-(-pps // want), rows * 8)
    return rows, ppb, -(-pps // ppb)


def fused_ncta(C, hw):
    """groupnorm_frame_fused's cluster size, or 0 when the shape takes the statistics + apply pair."""
    if C % 8 or (FUSED_THREADS % (C // 8)):
        return 0
    img, ncta = hw * C * 2, 1
    while -(-img // ncta) > FUSED_CAP and ncta < 16:
        ncta *= 2
    return 0 if -(-img // ncta) > FUSED_CAP or hw % ncta else ncta


def gn_schedules(C, hw, imgs_per_set, nimg, sms, k=1):
    """The ways a GroupNorm can sum a set: [(first, d_loc, d_glob)] for the statistics kernel over k frame shards and, per
    frame, the cluster kernel.  first[p] is the first pixel of the block (CTA) that sums set pixel p, whose value at the
    group's first channel is that block's shift; d_loc is the most fp32 additions of a shifted term inside the block
    (8 channels x its thread's pixels, then the shared atomics of the threads holding the group), d_glob the most of a
    block partial (global atomics or the cluster's ncta partials, times the k shards)."""
    cpg = C // GROUPS
    fs = imgs_per_set // k
    rows, ppb, nblk = gn_geometry(C, hw, fs, nimg // k, sms)
    p = torch.arange(imgs_per_set * hw)
    shard = p // (fs * hw)
    out = [(shard * fs * hw + (p % (fs * hw)) // ppb * ppb, 8 * -(-ppb // rows) + (cpg // 8 + 2) * rows, nblk * k + 2)]
    ncta = fused_ncta(C, hw) if imgs_per_set == 1 else 0
    if ncta:
        rows_f, ppc = FUSED_THREADS // (C // 8), hw // ncta
        out.append((p // ppc * ppc, 8 * -(-ppc // rows_f) + (cpg // 8 + 2) * rows_f, ncta + 2))
    return out


def tail_pixels(lo, hi, rows):
    """Pixels [lo, hi) that the 4-way unrolled loops leave to their tail loop (thread r walks lo + r, lo + r + rows, ...)."""
    out = []
    for r in range(rows):
        n = max(0, -(-(hi - lo - r) // rows))
        out += [lo + r + rows * j for j in range(4 * (n // 4), n)]
    return out


def edge_pixels(C, hw, imgs_per_set, nimg, sms, k=1, seed=0, n_random=16):
    """Pixels of a set (index in [0, imgs_per_set hw)) on the edges of every schedule that can sum a set: images, frame
    shards, blocks of gn_fill (first, last and first / last tail pixel), cluster slices; and random ones."""
    pps = imgs_per_set * hw
    ps = set()
    for f in range(imgs_per_set):
        ps |= {f * hw, f * hw + hw - 1}
    for kk in (k, 1):
        fs = imgs_per_set // kk
        for s in range(kk):
            ps |= {s * fs * hw, (s + 1) * fs * hw - 1}
        rows, ppb, nblk = gn_geometry(C, hw, fs, nimg // kk, sms)
        for s in range(kk):
            for b in range(nblk):
                lo, hi = s * fs * hw + b * ppb, s * fs * hw + min((b + 1) * ppb, fs * hw)
                t = tail_pixels(lo, hi, rows)
                ps |= {lo, hi - 1} | ({t[0], t[-1]} if t else set())
    ncta = fused_ncta(C, hw)
    if ncta and imgs_per_set == 1:
        ppc, rows_f = hw // ncta, FUSED_THREADS // (C // 8)
        for r in range(ncta):
            t = tail_pixels(r * ppc, (r + 1) * ppc, rows_f)
            ps |= {r * ppc, (r + 1) * ppc - 1} | ({t[0], t[-1]} if t else set())
    g = torch.Generator().manual_seed(seed)
    ps |= set(torch.randint(0, pps, (n_random,), generator=g).tolist())
    return sorted(p for p in ps if 0 <= p < pps)


def split_channels(C):
    """Channels (within their group) worth an impulse: the last channel of every group whose last 8-channel vector also
    holds the next group, the first channel after a split, the group's first channel and a middle one."""
    cpg = C // GROUPS
    ch = []
    for g in range(GROUPS):
        if ((g + 1) * cpg) % 8:
            ch.append(cpg - 1)
        if (g * cpg) % 8:
            ch.append(0)
    return ch + [0, cpg - 1, cpg // 2, 1]


# ---------------------------------------------------------------------------------------------------- inputs
def group_distinct(nsets, npix, C, seed, ratios=None, near_constant=True, ngroups=GROUPS):
    """fp16 [nsets, npix, C]: every (set, group) its own mean / spread, channel offsets and a per-pixel offset field.
    ratios: mean / spread per group, cycled (the cancellation sweep).  near_constant: set 0 group 1 has spread 1e-3, set 0
    group 2 is exactly constant."""
    g = torch.Generator().manual_seed(seed)
    cpg = C // ngroups
    sd = torch.exp(torch.empty(nsets, ngroups).uniform_(math.log(0.05), math.log(20.0), generator=g))
    if ratios is None:
        mu = sd * torch.empty(nsets, ngroups).uniform_(-4.0, 4.0, generator=g)
    else:
        sd = torch.exp(torch.empty(nsets, ngroups).uniform_(math.log(0.05), math.log(2.0), generator=g))
        r = torch.tensor([ratios[i % len(ratios)] for i in range(ngroups)])
        sign = torch.randint(0, 2, (nsets, ngroups), generator=g) * 2.0 - 1.0
        mu = sd * r * sign
    if near_constant and ratios is None:
        sd[0, 1 % ngroups], mu[0, 1 % ngroups] = 1e-3, 2e-3
    z = torch.randn(nsets, npix, C, generator=g)
    z += 0.3 * torch.randn(1, 1, C, generator=g)                             # channel offsets
    t = torch.linspace(0, 1, npix)
    z += 0.5 * torch.sin(2 * math.pi * (t * 3 + torch.rand(nsets, 1, generator=g)))[..., None]   # pixel field
    x = z * sd.repeat_interleave(cpg, 1)[:, None] + mu.repeat_interleave(cpg, 1)[:, None]
    if near_constant and ratios is None:
        x[0, :, 2 * cpg:3 * cpg] = 2.0 ** -6
    return x.half()


def impulses(nsets, npix, C, pixels, chans, launch=0, seed=0):
    """fp16 [nsets, npix, C]: group (s, g) holds c0(s, g) = +-2^-5 except c0 + A (|A| in [2, 8]) at pixel
    pixels[(s G + g + launch G nsets) % len] and channel chans[(s + g + launch) % len] of the group.  Returns (x, where)."""
    g = torch.Generator().manual_seed(seed + launch)
    cpg = C // GROUPS
    c0 = (torch.randint(0, 2, (nsets, GROUPS), generator=g) * 2.0 - 1.0) * 2.0 ** -5
    amp = torch.randint(2, 9, (nsets, GROUPS), generator=g).float() * (torch.randint(0, 2, (nsets, GROUPS), generator=g) * 2.0 - 1.0)
    x = c0.repeat_interleave(cpg, 1)[:, None].expand(nsets, npix, C).clone()
    where = []
    for s in range(nsets):
        for gr in range(GROUPS):
            p = pixels[(s * GROUPS + gr + launch * GROUPS * nsets) % len(pixels)]
            c = gr * cpg + chans[(s + gr + launch) % len(chans)]
            x[s, p, c] += amp[s, gr]
            where.append((s, p, c))
    return x.half(), where


# ---------------------------------------------------------------------------------------------------- GroupNorm
def gn_ref_bound(x, gamma, beta, eps, silu, schedules):
    """x [nsets, npix, C] fp16 -> (y* fp64, per-element worst case W, mean / spread per (set, group) [nsets, 1, C]).
    The statistics error is the largest over `schedules` (gn_schedules)."""
    ns, npix, C = x.shape
    cpg = C // GROUPS
    xd = x.double()
    xg = xd.reshape(ns, npix, GROUPS, cpg)
    n = npix * cpg
    mean = xg.sum((1, 3)) / n
    ex2 = (xg * xg).sum((1, 3)) / n
    var = (xg - mean[:, None, :, None]).pow(2).sum((1, 3)) / n
    sabs, sq = xg.abs().sum((1, 3)), (xg * xg).sum((1, 3))
    dS = dQ = torch.zeros_like(mean)
    for first, d_loc, d_glob in schedules:
        d = xg - xg[:, first.to(xg.device), :, :1]                           # x - the block's shift
        a1, a2 = d.abs().sum((1, 3)), (d * d).sum((1, 3))
        del d
        dS = torch.maximum(dS, d_loc * U * a1 + (d_glob + 3) * U * (sabs + a1))
        dQ = torch.maximum(dQ, (d_loc + 1) * U * a2 + (d_glob + 4) * U * (sq + a2))
    dmean = dS / n + 2 * U * mean.abs()
    dvar = dQ / n + 4 * U * ex2 + 2 * mean.abs() * dmean + dmean ** 2
    r = 1 / torch.sqrt(var + eps)
    lo = var + eps - dvar
    r_hi = torch.where(lo > 0, 1 / torch.sqrt(lo.clamp_min(1e-300)), torch.full_like(lo, math.inf))
    drstd = torch.maximum(r_hi / r - 1, 1 - (1 / torch.sqrt(var + eps + dvar)) / r) + 3 * U
    ex = lambda t: t.repeat_interleave(cpg, 1)[:, None, :]                  # [ns, G] -> [ns, 1, C]
    gd, bd = gamma.double(), beta.double()
    a = ex(r) * gd
    y0 = (xd - ex(mean)) * a + bd
    e = ((xd - ex(mean)).abs() * a.abs() * ex(drstd) + a.abs() * (1 + ex(drstd)) * ex(dmean)
         + U * (2 * (xd * a).abs() + 2 * (ex(mean) * a).abs() + bd.abs() + y0.abs()))
    y = y0
    if silu:
        y = y0 * torch.sigmoid(y0)
        e = 1.1 * e + (8 + y0.abs()) * U * y.abs()
    e = torch.where(torch.isinf(ex(drstd)), math.inf, e)             # no bound: dvar >= var + eps
    w = e * (1 + HALF) + HALF * y.abs() + SUB
    ratio = ex(mean.abs() / torch.sqrt(var).clamp_min(1e-300))
    return y, w, ratio


def _params(C, seed, dev, affine=True):
    g = torch.Generator().manual_seed(seed)
    if not affine:
        return torch.ones(C, device=dev), torch.zeros(C, device=dev)
    gamma = (1 + 0.3 * torch.randn(C, generator=g)).half().float()
    beta = (0.2 * torch.randn(C, generator=g)).half().float()
    return gamma.to(dev), beta.to(dev)


def _gn_check(out, x, gamma, beta, eps, silu, schedules, what, report=False):
    y, w, ratio = gn_ref_bound(x, gamma, beta, eps, silu, schedules)
    return _check_rows(out.reshape(y.shape), y, w, ratio, what, report)


def check_groupnorm(gn, B, F, H, W, c1, c2=0, silu=True, eps=1e-6, kinds=("distinct", "impulse", "cancel"),
                    launches=1, k=1, seed=0, dev=None, sms=None):
    """gn(x1, x2, gamma, beta, eps, imgs_per_set, silu) -> out [n, H, W, C]: 5-D (F frames per set) or per-frame (F = 1,
    B images) GroupNorm.  x2 (c2 > 0) is the virtual concat.  k: frame shards summed into one buffer."""
    dev = dev or DEV
    sms = sms or num_sms(dev)
    C, hw, nimg = c1 + c2, H * W, B * F
    sched = gn_schedules(C, hw, F, nimg, sms, k)
    gamma, beta = _params(C, seed + 1, dev)
    rs = []
    for kind in kinds:
        for L in range(launches if kind == "impulse" else 1):
            if kind == "distinct":
                x = group_distinct(B, F * hw, C, seed + 2)
            elif kind == "cancel":
                x = group_distinct(B, F * hw, C, seed + 3, ratios=RATIOS)
            else:
                pix = edge_pixels(C, hw, F, nimg, sms, k, seed + 4)
                x, _ = impulses(B, F * hw, C, pix, split_channels(C), L, seed + 5)
            x = x.to(dev)
            xv = x.view(nimg, H, W, C)
            x1, x2 = (xv[..., :c1].contiguous(), xv[..., c1:].contiguous()) if c2 else (xv, None)
            out = gn(x1, x2, gamma, beta, eps, F, silu)
            rs.append(_gn_check(out, x, gamma, beta, eps, silu, sched, f"{kind} launch {L}", report=kind == "cancel"))
    return merge(*rs)


def check_pixel_sweep(gn, B=2, F=4, H=8, W=8, C=320, silu=False, eps=1e-6, seed=0, dev=None, sms=None):
    """Impulses at every pixel of every (set, group) over ceil(F H W / (B 32)) launches."""
    dev = dev or DEV
    sms = sms or num_sms(dev)
    hw, nimg = H * W, B * F
    sched = gn_schedules(C, hw, F, nimg, sms)
    gamma, beta = _params(C, seed + 1, dev)
    pix = list(range(F * hw))
    launches = -(-len(pix) // (B * GROUPS))
    seen, rs = set(), []
    for L in range(launches):
        x, where = impulses(B, F * hw, C, pix, split_channels(C), L, seed)
        seen |= {p for _, p, _ in where}
        x = x.to(dev)
        out = gn(x.view(nimg, H, W, C), None, gamma, beta, eps, F, silu)
        rs.append(_gn_check(out, x, gamma, beta, eps, silu, sched, f"sweep launch {L}"))
    rs.append(flag(len(seen) == len(pix), "a pixel was not probed"))
    return merge(*rs)


def check_silu(apply, dev=None):
    """silu_f through the GroupNorm apply: sums (0, n) with n = 2^15 elements per group and eps = 0 give mean 0 and
    rstd = rsqrtf(1); gamma 1, beta 0, so out = fp16(silu(x)) for every fp16 x in [-12, 12] and a spread of large ones."""
    dev = dev or DEV
    C, H, W, n_img = 256, 64, 64, 2
    vals = torch.arange(-0x7bff, 0x7c00, dtype=torch.int32)
    h = torch.where(vals < 0, (-vals) | 0x8000, vals).to(torch.int16).view(torch.float16).float()
    h = h[(h.abs() <= 12) | (torch.arange(h.numel()) % 37 == 0)]
    x = h.repeat(-(-n_img * H * W * C // h.numel()))[:n_img * H * W * C].reshape(n_img, H, W, C).half().to(dev)
    sums = torch.zeros(n_img, GROUPS, 2, device=dev)
    sums[..., 1] = float(H * W * (C // GROUPS))
    ones, zeros = torch.ones(C, device=dev), torch.zeros(C, device=dev)
    out = apply(x, sums, ones, zeros, 0.0)
    xd = x.double()
    y = xd * torch.sigmoid(xd)
    w = 1.1 * 3 * U * xd.abs() + (8 + xd.abs()) * U * y.abs()
    w = w * (1 + HALF) + HALF * y.abs() + SUB
    return compare(out, y, 2 * w, "silu probe")


# ---------------------------------------------------------------------------------------------------- LayerNorm
def ln_rows(rows, C, seed, cancel=False):
    """fp16 [rows, C]: every row its own mean / spread and channel offsets; row 1 has spread 1e-3, row 2 is constant.
    cancel: rows with mean / spread = RATIOS, cycled."""
    g = torch.Generator().manual_seed(seed)
    if cancel:
        sd = torch.exp(torch.empty(rows, 1).uniform_(math.log(0.05), math.log(2.0), generator=g))
        r = torch.tensor([RATIOS[i % len(RATIOS)] for i in range(rows)])[:, None]
        mu = r * sd * (torch.randint(0, 2, (rows, 1), generator=g) * 2.0 - 1.0)
    else:
        sd = torch.exp(torch.empty(rows, 1).uniform_(math.log(0.05), math.log(20.0), generator=g))
        mu = sd * torch.empty(rows, 1).uniform_(-4.0, 4.0, generator=g)
        sd[1], mu[1] = 1e-3, 2e-3
    x = (torch.randn(rows, C, generator=g) + 0.3 * torch.randn(1, C, generator=g)) * sd + mu
    if not cancel:
        x[2] = 0.75
    return x.half()


def ln_ref_bound(x, gamma, beta, pe_rows=None, two_pass=True, depth=None, folded=False):
    """x [rows, C] fp16 -> (y*, worst case W, mean / spread per row, W before the fp16 store).  two_pass: ln5 / ln_kernel / ln_stats statistics,
    else the one-pass producer-slice form.  folded: the GEMM epilogue's rstd x' + (-mean rstd) gamma + beta form."""
    C = x.shape[1]
    eps = 1e-5
    xd = x.double()
    depth = depth or (C // 16 + 8)
    mean = xd.mean(1, keepdim=True)
    var = (xd - mean).pow(2).mean(1, keepdim=True)
    dmean = depth * U * xd.abs().mean(1, keepdim=True) + 2 * U * mean.abs()
    if two_pass:
        dvar = (depth + 4) * U * var + dmean ** 2
    else:
        dvar = (depth + 4) * U * (xd * xd).mean(1, keepdim=True) + 2 * mean.abs() * dmean + dmean ** 2
    r = 1 / torch.sqrt(var + eps)
    lo = var + eps - dvar
    r_hi = torch.where(lo > 0, 1 / torch.sqrt(lo.clamp_min(1e-300)), torch.full_like(lo, math.inf))
    drstd = torch.maximum(r_hi / r - 1, 1 - (1 / torch.sqrt(var + eps + dvar)) / r) + 3 * U
    gd, bd = gamma.double(), beta.double()
    a = r * gd
    z = (xd - mean) * a
    y = z + bd
    pe = 0.0 if pe_rows is None else pe_rows.double()
    y = y + pe
    e = (xd - mean).abs() * a.abs() * drstd + a.abs() * (1 + drstd) * dmean
    e = e + U * (4 * z.abs() + (z + bd).abs() + y.abs() + (3 * (mean * a).abs() + (xd * a).abs() if folded else 0))
    e = torch.where(torch.isinf(drstd).expand_as(e), math.inf, e)
    w = e * (1 + HALF) + HALF * y.abs() + SUB
    return y, w, mean.abs() / torch.sqrt(var).clamp_min(1e-300), e


def _check_rows(out, y, w, ratio, what, report=False):
    """Bound on every element; the envelope on rows / groups with mean / spread <= ENVELOPE_MAX_RATIO; report: the
    envelope ratio at each cancellation ratio."""
    rs = [compare(out, y, 2 * w, what)]
    env = envelope(out, y)
    inside = (ratio <= ENVELOPE_MAX_RATIO * (1 + 1e-3)).expand_as(env)
    if inside.any():
        m = env[inside].max().item()
        rs.append({"err": 0.0, "env": m, "tol": 1.0, "ok": m <= 1.0, "what": what + " (envelope: 1 ulp + 2^-14)"})
    if report:
        parts = []
        nominal = torch.tensor(RATIOS, dtype=torch.float64, device=ratio.device)
        near = (torch.log1p(ratio)[..., None] - torch.log1p(nominal)).abs().argmin(-1)     # nearest swept ratio
        for i, rt in enumerate(RATIOS):
            sel = (near == i).expand_as(env)
            if sel.any():
                parts.append(f"{rt:g}: {env[sel].max().item():.3g} ulp")
        rs[0]["report"] = f"{what}: envelope / ulp by mean/spread " + ", ".join(parts)
    return merge(*rs)


def pe_table(C, seed, dev, frames=24):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(frames, C, generator=g).to(dev)


def check_layernorm(ln, rows, C, pe=False, hw=7, F=5, seed=0, dev=None):
    """ln(x, gamma, beta, pe, hw, F) -> [rows, C]; PE row (row // hw) % F, every PE row distinct."""
    dev = dev or DEV
    gamma, beta = _params(C, seed + 1, dev)
    table = pe_table(C, seed + 2, dev) if pe else None
    rs = []
    for cancel in (False, True):
        x = ln_rows(rows, C, seed + 3 + cancel, cancel).to(dev)
        out = ln(x, gamma, beta, table, hw, F)
        pr = table[(torch.arange(rows, device=dev) // hw) % F] if pe else None
        y, w, ratio, _ = ln_ref_bound(x, gamma, beta, pr)
        rs.append(_check_rows(out, y, w, ratio, f"ln C {C} rows {rows} cancel {cancel}", report=cancel))
    return merge(*rs)


def one_hot_w(N, C, shift=0, stride=1, dev=None):
    """W [N, C] fp16 with W[n, k(n)] = 1, k(n) = (n stride + shift) % C, and k."""
    k = (torch.arange(N) * stride + shift) % C
    w = torch.zeros(N, C)
    w[torch.arange(N), k] = 1.0
    return w.half().to(dev or DEV), k.to(dev or DEV)


def fold_depth(C):
    """Producer-slice statistics: a lane's 8-column chunks of every column tile, the shuffles and the slices."""
    return C // 8 + 16 + -(-C // 64)


def check_ln_fold(fold, rows, C, N=None, pe=False, hw=7, F=5, residual=False, producer=False, geglu=False, seed=0,
                  dev=None):
    """fold(x, W, gamma, beta, pe, hw, F, residual, geglu) -> (x_used, out) with one-hot weights.  Linear:
    out[:, n] = LN(x_used)[:, k(n)] (+ PE).  GEGLU (W = [value rows; gate rows], both one-hot):
    out[:, n] = LN[:, kv(n)] gelu(LN[:, kg(n)]).  producer: statistics from the producer GEMM's slices (one-pass)."""
    dev = dev or DEV
    N = N or C
    gamma, beta = _params(C, seed + 1, dev)
    table = pe_table(C, seed + 2, dev) if pe else None
    if geglu:
        Wv, kv = one_hot_w(N, C, shift=3, stride=1, dev=dev)
        Wg, kg = one_hot_w(N, C, shift=11, stride=7, dev=dev)
        W = torch.cat([Wv, Wg])
    else:
        W, k = one_hot_w(N, C, shift=3, stride=7, dev=dev)
    depth = fold_depth(C) if producer else None
    rs = []
    for cancel in (False, True):
        x = ln_rows(rows, C, seed + 3 + cancel, cancel).to(dev)
        xu, out = fold(x, W, gamma, beta, table, hw, F, residual, geglu)
        if not residual:
            rs.append(flag(torch.equal(xu, x), "the producer did not store x exactly"))
        pr = table[(torch.arange(rows, device=dev) // hw) % F] if pe else None
        y, w, ratio, e = ln_ref_bound(xu, gamma, beta, pr, not producer, depth, folded=True)
        what = f"fold C {C} N {N} {'slices' if producer else 'stats'}{' geglu' if geglu else ''} cancel {cancel}"
        if geglu:
            v, g, wv, wg = y[:, kv], y[:, kg], e[:, kv], e[:, kg]     # value and gate stay fp32
            gl = g * 0.5 * (1 + torch.erf(g / math.sqrt(2)))
            yy = v * gl
            e = gl.abs() * wv + v.abs() * (1.13 * wg + GELU_ABS + GELU_REL * g.clamp_min(0)) + 2 * U * yy.abs()
            rs.append(_check_rows(out, yy, e * (1 + HALF) + HALF * yy.abs() + SUB, ratio, what, report=cancel))
        else:
            rs.append(_check_rows(out, y[:, k], w[:, k], ratio, what, report=cancel))
    return merge(*rs)


# ---------------------------------------------------------------------------------------------------- GEGLU epilogue
GELU_ABS, GELU_REL = 1.2e-5, 2.0 ** -20         # gelu_sig's error: GELU_ABS + GELU_REL max(x, 0)


def gelu_gates(dev=None):
    """Every fp16 value in [-12, 12] (the clamp at |x| = 5 inside) and a spread of larger ones down to -65504."""
    vals = torch.arange(0, 0x7c00, dtype=torch.int32)
    pos = vals.to(torch.int16).view(torch.float16).float()
    h = torch.cat([pos, -pos])
    return h[(h.abs() <= 12) | (torch.arange(h.numel()) % 29 == 0)].to(dev or DEV)


def check_gelu(geglu, dev=None):
    """geglu(A, W) -> [M, hidden] with W = [value rows; gate rows] (value first, unpacked, no bias): A[:, K - 1] = 1 and
    the other columns hold the gates; value row n reads column K - 1, gate row n column n % (K - 1), so every output is
    fp16(gelu_sig(gate)) and is compared with the fp64 erf-GELU within gelu_sig's claimed error plus the fp16 rounding."""
    dev = dev or DEV
    K, hidden = 320, 1280
    gates = gelu_gates(dev)
    M = -(-gates.numel() // (K - 1))
    A = torch.ones(M * (K - 1), device=dev)
    A[:gates.numel()] = gates
    A = torch.cat([A.reshape(M, K - 1), torch.ones(M, 1, device=dev)], 1).half()
    Wv = torch.zeros(hidden, K, device=dev)
    Wv[:, K - 1] = 1
    Wg = torch.zeros(hidden, K, device=dev)
    Wg[torch.arange(hidden), torch.arange(hidden) % (K - 1)] = 1
    out = geglu(A, torch.cat([Wv, Wg]).half())
    g = A[:, (torch.arange(hidden, device=dev) % (K - 1))].double()
    y = g * 0.5 * (1 + torch.erf(g / math.sqrt(2)))
    e = GELU_ABS + GELU_REL * g.clamp_min(0) + 2 * U * y.abs()
    return compare(out, y, e * (1 + HALF) + HALF * y.abs() + SUB, "gelu probe")
