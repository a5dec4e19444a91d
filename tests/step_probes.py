"""Per-element checks of the denoising step's small kernels (pointwise.cu): the point adapter (`vs_adapter_level`:
f16_to_f32, small_linear twice, adapter_splat) and the time embedding (`vs_unet_time_embedding`: timestep_embedding,
then small_linear three times).  Kernel-agnostic: every check takes the kernel as a callable, so the same checks run
the CUDA kernels (tests/test_step_probes_gpu.py) and a torch emulation of their arithmetic with planted bugs
(tests/test_step_probes_cpu.py).

Adapter callables: fn(w0, b0, w1, b1, pe, tracks, h, w, rate, mask, coord_fp16, scale) -> NHWC fp16 [F, h, w, C], with
fp16 weights, fp32 point embeddings pe [P, E], fp32 tracks [F, P, 2] (x, y in pixels) and an int32 mask [P] or None.

Exact probes (no tolerance).
  * Integer-exact MLP.  Ternary fp16 weights, integer biases and embeddings make every first-layer pre-activation an
    integer that is >= 32 or <= -128, where silu_f gives x or (-)0 exactly (1 + __expf(-x) rounds to 1, or __expf
    overflows to inf); every fp32 partial sum is an integer far below 2^24 and every feature an integer of magnitude
    <= 2048, so exact in fp16.  `regimes` mixes both SiLU regimes with sparse weights; `dense` has +-1 embeddings over
    all E inputs and +-1 first-layer weights, and a one-hot second layer (column c reads hidden unit c mod mid), so
    every input column of both layers moves some output by at least 1: a dropped, duplicated or early-ending k pair
    and a skipped row of points all show.
  * Cells: every point sits on a cell (track = rate * (i, j), scale 1), different cells in every frame, so the map
    equals the features bit for bit and is zero elsewhere.
  * Dyadic geometry: tracks on quarter cells make the bilinear weights multiples of 1/16; with integer features every
    fp32 sum is exact and the only rounding is the final fp16 one, so the map equals `splat_ref` (an fp64 restatement
    of the reference's bilinear_interpolation, models/adapter_model.py:25-47) bit for bit.

Bounded probe (fp16 coordinate quantisation, tracks 512 .. 4096 px).  The kernel forms the same fp16 (or fp32) weights
as the reference, sums r16(feat) * wsum over the points in fp32 and rounds once; `splat_ref` sums the same products in
fp64.  With n the contributions at a cell and A = sum |feat w| there:
    |out - ref| <= s (n + 4) u A + k 2^-11 (1 + 2^-10) (|ref| + s (n + 4) u A) + k 2^-25,   u = 2^-24,
k = 2 fp16 roundings with coord_fp16 (r16(acc), then the product with the scale) and 1 without; n + 4 is the depth of
a term (wsum: up to 3 additions, the product, n accumulations).  The comparator allows twice that, and the set of
non-zero cells must equal the restatement's exactly.

Time embedding: fn(t [B]) -> (emb [B, 1280], proj [B, tproj_n]).  The reference forms the fp32 argument
t * exp(-ln(1e4) j / 160) as torch does; the kernel forms the same exponent, but expf (2 ulp) differs from torch's exp
by up to 3 ulp, so |arg_kernel - arg_torch| <= 8 u |arg|, and cosf / sinf add 2 ulp: ds = 8 u |arg| + 4 u |s|.  Each
small_linear row is a lane-strided fp32 dot product: a term passes through at most K / 64 + 9 roundings (its pair,
the lane's running sum, the five shuffles, the bias), so with g_K = (K / 32 + 10) u
    d(W x + b) <= |W| dx + g_K (|W| |x| + |b|),
and silu_f (__expf: 2 + 1.2 |x| ulp, __fdividef: 2 ulp) adds (8 + |x|) u |silu(x)| after a derivative of at most 1.1.
emb is held to the bound propagated from the sinusoid through both layers; every resnet's slice of proj to one layer's
bound applied to the kernel's own emb, under the resnet's own name.  The comparators allow twice the bound."""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
LEVELS = ((320, 8), (640, 16), (1280, 32), (1280, 64))      # (C, downsample rate) of SparsePointAdapter's four levels
E_DIM, MID = 1280, 128


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------ MLP
def exact_mlp(C, P, kind="regimes", E=E_DIM, mid=MID, seed=0):
    """(w0, b0, w1, b1) fp16, pe fp32 [P, E] and the exact features fp64 [P, C] (see the module docstring)."""
    g = _gen(seed)

    def ternary(shape, density):
        v = torch.randint(0, 2, shape, generator=g) * 2 - 1
        return v * (torch.rand(shape, generator=g) < density)

    if kind == "regimes":
        pe = ternary((P, E), 1 / 16)
        w0 = ternary((mid, E), 1 / 16)
        b0 = torch.where(torch.arange(mid) % 2 == 0, 48, -160)[torch.randperm(mid, generator=g)]
        w1 = ternary((C, mid), 1 / 8)
    elif kind == "dense":
        pe = torch.randint(0, 2, (P, E), generator=g) * 2 - 1
        w0 = torch.randint(0, 2, (mid, E), generator=g) * 2 - 1
        b0 = torch.full((mid,), 256)
        w1 = (torch.arange(mid)[None, :] == (torch.arange(C) % mid)[:, None]).long()
    else:
        raise ValueError(kind)
    b1 = torch.randint(-8, 9, (C,), generator=g)
    h = pe.double() @ w0.double().t() + b0.double()
    assert bool(((h >= 32) | (h <= -128)).all()), "pre-activations must stay in the exact SiLU regimes"
    feat = h.clamp_min(0) @ w1.double().t() + b1.double()
    assert feat.abs().max() <= 2048
    return (w0.half(), b0.half(), w1.half(), b1.half()), pe.float(), feat


# ------------------------------------------------------------------------------------------------------------ splat
def _rounder(coord_fp16):
    return (lambda v: float(np.float16(v))) if coord_fp16 else (lambda v: float(np.float32(v)))


def splat_ref(feat, tracks, h, w, rate, mask=None, coord_fp16=True):
    """fp64 restatement of the reference's per-point bilinear_interpolation: coordinates and the four weights in the
    tracks' dtype (fp16 with coord_fp16, else fp32; each op rounded once, as the reference's tensor ops do), feature x
    weight summed in fp64.  Returns (m [F, h, w, C] fp64 before the scale, A = sum |feat w| [F, h, w, C], n = the
    contributions per cell [F, h, w, 1])."""
    q = _rounder(coord_fp16)
    feat = feat.double()
    nf, npts = tracks.shape[:2]
    C = feat.shape[1]
    m = torch.zeros(nf, h, w, C, dtype=torch.float64)
    A = torch.zeros(nf, h, w, C, dtype=torch.float64)
    n = torch.zeros(nf, h, w, 1, dtype=torch.int64)
    fa = feat.abs()
    tr = tracks.double().tolist()
    for pt in range(npts):
        if mask is not None and not int(mask[pt]):
            continue
        for f in range(nf):
            px, py = q(tr[f][pt][0]), q(tr[f][pt][1])
            if px < 0 or py < 0:
                continue
            x, y = q(px / rate), q(py / rate)
            x1, y1 = int(x), int(y)
            xf, yf = q(x - x1), q(y - y1)
            x2, y2 = x1 + 1, y1 + 1
            x1, x2 = max(min(x1, w - 1), 0), max(min(x2, w - 1), 0)
            y1, y2 = max(min(y1, h - 1), 0), max(min(y2, h - 1), 0)
            ox, oy = q(1 - xf), q(1 - yf)
            ws = ((y1, x1, q(ox * oy)), (y1, x2, q(xf * oy)), (y2, x1, q(ox * yf)), (y2, x2, q(xf * yf)))
            for cy, cx, wt in ws:
                if wt != 0:
                    m[f, cy, cx] += feat[pt] * wt
                    A[f, cy, cx] += fa[pt] * abs(wt)
                    n[f, cy, cx] += 1
    return m, A, n


def round_map(m, coord_fp16, scale):
    """The kernel's output rounding of an exact map: fp16(r16(acc) * scale) with coord_fp16, else fp16(acc * scale)."""
    return (m.half().double() * scale).half() if coord_fp16 else (m * scale).half()


def _tracks_from_cells(cells, rate):
    return (cells.double() * rate).float()


def cell_tracks(F, P, h, w, rate, seed):
    """Every point on a cell, a different random cell arrangement in every frame (cells repeat only when P > h w)."""
    g = _gen(seed)
    out = torch.empty(F, P, 2)
    for f in range(F):
        idx = torch.cat([torch.randperm(h * w, generator=g) for _ in range(-(-P // (h * w)))])[:P]
        out[f] = _tracks_from_cells(torch.stack([idx % w, idx // w], 1), rate)
    return out


def _compare_exact(out, ref, what):
    out = out.detach().cpu()
    if out.shape != ref.shape:
        return {"ok": False, "err": float("inf"), "what": f"{what}: shape {tuple(out.shape)} != {tuple(ref.shape)}"}
    bad = ~((out == ref) | (torch.isnan(out) & torch.isnan(ref)))
    nbad = int(bad.sum())
    return {"ok": nbad == 0 and not bool(torch.isnan(out.float()).any()), "err": float(nbad),
            "what": f"{what}: {nbad} of {out.numel()} elements differ" + (f" (first at {bad.nonzero()[0].tolist()})" if nbad else "")}


def _run(fn, weights, pe, tracks, h, w, rate, mask, coord_fp16, scale, dev):
    w0, b0, w1, b1 = (t.to(dev) for t in weights)
    mk = None if mask is None else mask.to(device=dev, dtype=torch.int32)
    return fn(w0, b0, w1, b1, pe.to(dev).contiguous(), tracks.to(dev).contiguous(), h, w, rate, mk, coord_fp16, scale)


def check_adapter_cells(fn, level, P, kind="regimes", E=E_DIM, mid=MID, F=3, size=(512, 384), coord_fp16=True,
                        seed=0, dev="cuda"):
    """The MLP and the splat at exact cells: the map must equal the fp64 features bit for bit, everywhere."""
    C, rate = LEVELS[level]
    weights, pe, feat = exact_mlp(C, P, kind, E, mid, seed=seed)
    h, w = size[1] // rate, size[0] // rate
    tracks = cell_tracks(F, P, h, w, rate, seed + 1)
    out = _run(fn, weights, pe, tracks, h, w, rate, None, coord_fp16, 1.0, dev)
    m, _, _ = splat_ref(feat, tracks, h, w, rate, None, coord_fp16)
    return _compare_exact(out, round_map(m, coord_fp16, 1.0), f"level {level} P {P} {kind} E {E} mid {mid}")


# --------------------------------------------------------------------------------------------- dyadic geometry
def geometry_case(name, level):
    """(size (W, H), tracks [F, P, 2], mask or None) of one dyadic geometry case at `level`."""
    C, rate = LEVELS[level]
    size = (512, 384)
    mask = None
    if name in ("floor", "one_cell"):
        size = (480, 360) if name == "floor" else (rate + rate // 2 + 1, rate + 3)
    w, h = size[0] // rate, size[1] // rate
    g = _gen(1000 + level * 17 + len(name))
    q4 = rate / 4
    if name == "edges":
        # last column / row with the fraction 1/4 .. 3/4 (x2 / y2 clamp onto x1 / y1), exactly at w * rate, beyond the frame
        pts = [((w - 1) * rate + q4, 2 * rate + q4), (rate + 3 * q4, (h - 1) * rate + 2 * q4), ((w - 1) * rate + q4, (h - 1) * rate + 3 * q4),
               (w * rate, rate), (2 * rate, h * rate), (w * rate, h * rate), (5 * w * rate, 3 * h * rate), (w * rate + q4, 0.0)]
        tr = torch.tensor(pts)[None].repeat(3, 1, 1)
        tr[1] = tr[1].flip(0)                                  # other frames: the same points, other owners
        tr[2, :, 0] = tr[2, :, 0] * 0 + torch.tensor([(w - 1) * rate + 2 * q4] * 8)
    elif name == "signs":
        # negative (skipped), -0.0 (visible), and -1e-8: -0.0 in fp16 (visible with coord_fp16), invisible in fp32
        pts = [(-q4, rate), (rate, -3.0), (-0.0, 2 * rate + q4), (rate + q4, -0.0), (-0.0, -0.0), (-1e-8, rate + 2 * q4),
               (3 * rate, -1e-8), (-1e-8, -1e-8), (2 * rate + 3 * q4, rate + q4)]
        tr = torch.tensor(pts)[None].repeat(2, 1, 1)
        tr[1] = tr[1].roll(1, 0)
    elif name == "mask":
        P = 40
        tr = _tracks_from_cells(torch.stack([torch.randint(0, w, (2, P), generator=g),
                                             torch.randint(0, h, (2, P), generator=g)], -1), rate)
        tr = tr + (torch.randint(0, 4, tr.shape, generator=g) * q4)
        mask = torch.ones(P, dtype=torch.int32)
        mask[[0, P - 1, 17]] = 0
    elif name == "frames":
        Fn, P = 4, 5                                            # F != P: a frame / point index swap reads other tracks
        tr = _tracks_from_cells(torch.stack([torch.randint(0, w, (Fn, P), generator=g),
                                             torch.randint(0, h, (Fn, P), generator=g)], -1), rate)
        tr = tr + (torch.randint(0, 4, tr.shape, generator=g) * q4)
    elif name == "pile":
        P = 200                                                 # 200 points on one cell, quarter offsets over 4 cells
        base = torch.tensor([(w // 2) * rate, (h // 2) * rate], dtype=torch.float32)
        tr = (base + torch.randint(0, 4, (2, P, 2), generator=g) * q4)
    elif name == "floor":
        # 360 x 480 frames: level 3 is 5 x 7; points in the strip the floor cuts off and on the last full cells
        pts = [((w - 1) * rate + q4, rate), (w * rate + 2 * q4, (h - 1) * rate + q4), (rate, h * rate + 3 * q4),
               (size[0] - 1.0 - ((size[0] - 1) % q4), size[1] - 1.0 - ((size[1] - 1) % q4)), (0.0, 0.0)]
        tr = torch.tensor(pts)[None].repeat(2, 1, 1)
        tr[1, :, 0] = tr[1, :, 0].flip(0)
    elif name == "one_cell":
        pts = [(0.0, 0.0), (q4, 3 * q4), (rate + q4, 2 * q4), (2 * q4, rate), (3 * rate, 3 * rate)]
        tr = torch.tensor(pts)[None].repeat(2, 1, 1)
        tr[1] = tr[1].flip(0)
    else:
        raise ValueError(name)
    return size, tr.float(), mask


GEOMETRY = ("edges", "signs", "mask", "frames", "pile", "floor", "one_cell")


def check_adapter_geometry(fn, name, level, coord_fp16, scale=1.0, dev="cuda"):
    """A dyadic geometry case against the fp64 restatement, bit for bit."""
    C, rate = LEVELS[level]
    size, tracks, mask = geometry_case(name, level)
    P = tracks.shape[1]
    wts, pe, feat = exact_mlp(C, P, "regimes", seed=300 + level)
    h, w = size[1] // rate, size[0] // rate
    out = _run(fn, wts, pe, tracks, h, w, rate, mask, coord_fp16, scale, dev)
    m, _, _ = splat_ref(feat, tracks, h, w, rate, mask, coord_fp16)
    return _compare_exact(out, round_map(m, coord_fp16, scale), f"{name} level {level} fp16 coords {coord_fp16} scale {scale}")


# ------------------------------------------------------------------------------------------ fp16 quantisation
def quant_tracks(F, P, long_axis, seed):
    """Tracks 512 .. 4096 px on the long axis (fp16 steps 0.5, 1, 2 px), including values fp16 rounds onto a cell
    boundary (511.9 -> 512, 1023.9 -> 1024, ...), 0 .. 255 px on the other."""
    g = _gen(seed)
    t = torch.empty(F, P, 2, dtype=torch.float64)
    t[..., long_axis] = 512 + torch.rand(F, P, generator=g, dtype=torch.float64) * 3584
    t[..., 1 - long_axis] = torch.rand(F, P, generator=g, dtype=torch.float64) * 255
    special = torch.tensor([511.9, 1023.9, 2047.9, 4095.9, 767.8, 1535.7, 3071.1, 600.3, 2600.77, 1000.01])
    t[0, :special.numel(), long_axis] = special.double()
    t[1, :special.numel(), 1 - long_axis] = torch.tensor([13.31, 0.3, 7.99, 8.01, 100.7, 255.9, 31.97, 64.02, 3.3, 0.77]).double()
    return t.float()


def check_adapter_quant(fn, level, coord_fp16, long_axis=0, scale=1.0, P=24, F=2, dev="cuda"):
    """Non-dyadic coordinates: the support must equal the restatement's, values within twice the bound above."""
    C, rate = LEVELS[level]
    wts, pe, feat = exact_mlp(C, P, "regimes", seed=500 + level)
    size = [256, 256]
    size[long_axis] = 4096 + rate
    h, w = size[1] // rate, size[0] // rate
    tracks = quant_tracks(F, P, long_axis, seed=600 + level)
    out = _run(fn, wts, pe, tracks, h, w, rate, None, coord_fp16, scale, dev).detach().cpu().double()
    m, A, n = splat_ref(feat, tracks, h, w, rate, None, coord_fp16)
    ref = m * scale
    k = 2 if coord_fp16 else 1
    acc = scale * (n + 4).double() * U * A
    bound = acc + k * (2.0 ** -11 * (1 + 2.0 ** -10) * (ref.abs() + acc) + 2.0 ** -25)
    support_out = (out != 0).any(-1)
    support_ref = (round_map(m, coord_fp16, scale) != 0).any(-1)
    nsup = int((support_out != support_ref).sum())
    ratio = ((out - ref).abs() / (2 * bound)).max().item()
    ok = nsup == 0 and ratio <= 1.0 and bool(torch.isfinite(out).all())
    return {"ok": ok, "err": ratio, "what": f"level {level} fp16 coords {coord_fp16} axis {long_axis}: {nsup} cells "
            f"differ in support, worst err / comparator {ratio:.3g}"}


# ---------------------------------------------------------------------------------------------- time embedding
def tproj_layout(cfg):
    """[(resnet prefix, column offset, channels)] of the stacked time_emb_proj rows, in unet.cu's registration order:
    down blocks, mid block, up blocks."""
    boc, lpb = list(cfg.block_out_channels), cfg.layers_per_block
    names = [(f"down_blocks.{i}.resnets.{j}", boc[i]) for i in range(4) for j in range(lpb)]
    names += [("mid_block.resnets.0", boc[3]), ("mid_block.resnets.1", boc[3])]
    names += [(f"up_blocks.{i}.resnets.{j}", boc[3 - i]) for i in range(4) for j in range(lpb + 1)]
    out, off = [], 0
    for n, c in names:
        out.append((n, off, c))
        off += c
    return out


def time_param_names(cfg):
    return ["time_embedding.linear_1.weight", "time_embedding.linear_1.bias", "time_embedding.linear_2.weight",
            "time_embedding.linear_2.bias"] + [f"{n}.time_emb_proj.{s}" for n, _, _ in tproj_layout(cfg) for s in ("weight", "bias")]


def sinusoid_ref(t, dim):
    """(fp64 cos / sin at torch's fp32 argument, its kernel bound ds)."""
    half = dim // 2
    freq = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    arg = (t.float()[:, None] * freq[None, :]).double()
    s = torch.cat([torch.cos(arg), torch.sin(arg)], -1)
    ds = 8 * U * torch.cat([arg.abs(), arg.abs()], -1) + 4 * U * s.abs()
    return s, ds


def _silu(x):
    return x / (1 + torch.exp(-x))


def _silu_err(x):
    return (8 + x.abs()) * U * _silu(x).abs()


def linear_bound(W, x, b, dx):
    """(W x + b in fp64, its bound: |W| dx + g_K (|W| |x| + |b|))."""
    K = W.shape[1]
    gk = (K / 32 + 10) * U
    Wa = W.abs()
    return x @ W.t() + b, dx @ Wa.t() + gk * (x.abs() @ Wa.t() + b.abs())


def check_time_embedding(fn, sd, cfg, t, dev="cuda"):
    """emb against the fp64 chain with the propagated bound, every resnet's projection slice against one layer applied
    to the kernel's own emb.  `sd`: fp32 tensors holding the fp16 weights."""
    t = torch.as_tensor(t, dtype=torch.float32)
    emb, proj = fn(t.to(dev))
    emb, proj = emb.detach().cpu().double(), proj.detach().cpu().double()
    W = {k: sd[k].double() for k in time_param_names(cfg)}
    layout = tproj_layout(cfg)
    res = {"ok": True, "err": 0.0, "what": ""}

    def judge(name, out, ref, bound):
        if out.shape != ref.shape:
            res.update(ok=False, err=float("inf"), what=f"{name}: shape {tuple(out.shape)} != {tuple(ref.shape)}")
            return
        r = ((out - ref).abs() / (2 * bound)).max().item()
        if not (r <= 1.0):
            res["ok"] = False
        if not (r <= res["err"]):
            res.update(err=r, what=f"worst: {name}")

    s, ds = sinusoid_ref(t, cfg.block_out_channels[0])
    h1, dh1 = linear_bound(W["time_embedding.linear_1.weight"], s, W["time_embedding.linear_1.bias"], ds)
    a1, da1 = _silu(h1), 1.1 * dh1 + _silu_err(h1)
    e_ref, de = linear_bound(W["time_embedding.linear_2.weight"], a1, W["time_embedding.linear_2.bias"], da1)
    judge("emb", emb, e_ref, de)
    total = layout[-1][1] + layout[-1][2]
    if proj.shape[1] != total:
        res.update(ok=False, err=float("inf"), what=f"proj has {proj.shape[1]} columns, the resnets {total}")
        return res
    se = _silu(emb)
    for name, off, c in layout:
        p_ref, dp = linear_bound(W[f"{name}.time_emb_proj.weight"], se, W[f"{name}.time_emb_proj.bias"], _silu_err(emb))
        judge(name, proj[:, off:off + c], p_ref, dp)
    return res
