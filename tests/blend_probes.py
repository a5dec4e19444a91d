"""Per-element checks of the attention-controller blend (pointwise.cu `blend_mask_kernel` through `vs_blend_mask` /
`p2p.SpatialBlender._mask`, and `latent_blend_kernel` through `vs_latent_blend`).  Kernel-agnostic: a mask callable
fn(maps, alpha, h, w, th, both, res) -> mask [n_prompts, F, h, w] (maps: a list of per-layer [p, F, heads, r, words] fp16
tensors, alpha [p, words] fp32, res = (res_h, res_w)) and a latent callable fn(src, tgt, mask) -> (tgt', src') run the
CUDA kernels (tests/test_blend_probes_gpu.py) and a torch emulation of their arithmetic with planted bugs
(tests/test_blend_probes_cpu.py).

Reference (`mask_ref`): an fp64 restatement of the reference's SpatialBlender.get_mask (utils/p2p_utils/spatial_blend.py:
25-47): the word-weighted sum over words, the mean over layers x heads, max_pool2d(3, 1, 1), F.interpolate(size=(h, w))
nearest, division by the frame's max, `.gt(fp32(th))`, and with `both` the OR with prompt 0 of the same frame.  The source
indices of the resize are the ones torch computes, min(floor(dst * fp32(in / out)), in - 1); `src_index` pins them by
interpolating an index map with torch itself.  The 1 / (n_maps heads) factor of the mean cancels in the normalisation, so
a wrong mean factor cannot be seen here -- and does no harm.

Decision margin.  The maps are >= 0 and alpha is in {0, 1}, so the kernel's per-pixel value is a sum of the N = n_maps x
heads x (selected words) fp16 map values, added in fp32 in some order (lanes over words, then the warp shuffles): with
non-negative terms every partial sum is at most the total, so the sum is within gamma_(N-1) = (N - 1) u / (1 - (N - 1) u)
of the exact one (u = 2^-24).  The product with the fp32 mean factor adds one rounding, gamma_N in all; the factor's own
rounding is common to every pixel and cancels.  Pooling and resizing only select values, so the pooled pixel and the
frame's max are each within gamma_N of the exact ones, and the ratio adds one rounding:
    |r_kernel - r| <= M r,   M = (1 + gamma_N) / (1 - gamma_N) (1 + u) - 1 = (2 N + 1) u + O(N^2 u^2),
which is below (2 N + 6) u for N <= 6000 (the controllers' N is at most 5 x 8 x 77 = 3080).  A pixel is DECIDED when
r (1 - M) > fp32(th) (the kernel must give 1) or r (1 + M) <= fp32(th) (it must give 0: the test is strict); a frame whose
maps are all zero has 0 / 0 = NaN and must give 0.  Every decided pixel must match exactly; the undecided ones are
counted and must stay under 0.1 % so each case keeps its power.  With `both`, prompt 1's bit is the OR of two tri-state
decisions.

Exact cases (`dyadic`).  Map values k / 256, n_maps x heads = 8 and a one-hot alpha: every sum is a multiple of 2^-11
below 2^24 of them and the mean factor 1 / 8 is a power of two, so the kernel's pixels are exact; the ratio is the
correctly rounded fp32 quotient of exact values (double rounding through fp64 is innocuous for a quotient of 24-bit
operands), so every pixel is decided by fp32(p / max) > fp32(th), and the planted pixels at exactly p / max = th = 0.5
must give 0.

Latent blend (`check_latent`): tgt' = src + m (tgt - src) per (channel, frame, pixel) in fp32.  With 0/1 masks (all the
mask kernel makes) every element must be src or tgt bit for bit, in fp16 and fp32 and whether or not nvcc contracts
the update into an FMA.  The kernel selects at m = 0 and m = 1: the lerp alone returns s + fl(t - s), which misses t
wherever |t| << |s| (s = 1.1035, t = 2.4498e-05 gives 2.4557e-05 in fp16), and the inputs here span 2^-8 .. 2^8 so such
pairs occur.  Fractional masks: the difference, the product and the sum each round once,
    |v - ref| <= (2 u + u^2) (1 + u) m |tgt - src| + u |ref|  (the u^2 terms covered by a 1 + 8 u factor),
and fp16 targets are held to the set of values v rounds to (ddim_probes.beyond_rounding); the comparator allows twice
that, and src is never written."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from tests.ddim_probes import beyond_rounding

U = 2.0 ** -24
MAX_UNDECIDED = 1e-3


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def src_index(n_in: int, n_out: int) -> torch.Tensor:
    """The source index of every output row of F.interpolate(size=n_out, mode='nearest'), read off torch itself."""
    idx = torch.arange(n_in, dtype=torch.float32).reshape(1, 1, n_in, 1)
    got = F.interpolate(idx, size=(n_out, 1), mode="nearest")[0, 0, :, 0].long()
    scale = torch.tensor(n_in, dtype=torch.float32) / torch.tensor(n_out, dtype=torch.float32)
    formula = torch.floor(torch.arange(n_out, dtype=torch.float32) * scale).long().clamp_max(n_in - 1)
    assert torch.equal(got, formula), (n_in, n_out)
    return got


def margin(n_terms: int) -> float:
    g = n_terms * U / (1 - n_terms * U)
    return (1 + g) / (1 - g) * (1 + U) - 1


# ------------------------------------------------------------------------------------------------ reference
def mask_ref(maps, alpha, h, w, th, both, res, exact=False):
    """(tri-state mask [n_prompts, F, h, w] int8: 1, 0 or -1 = undecided, ratio r fp64)."""
    npr = 2 if both else 1
    rh, rw = res
    n_maps, (_, frames, heads, r, words) = len(maps), maps[0].shape
    al = alpha[:npr].double()
    m = torch.zeros(npr, frames, r, dtype=torch.float64)
    for it in maps:
        m += torch.einsum("pfhrw,pw->pfr", it[:npr].double(), al)
    m = (m / (n_maps * heads)).reshape(npr, frames, rh, rw)
    pooled = F.max_pool2d(m, 3, 1, 1)
    rs = pooled[:, :, src_index(rh, h)][:, :, :, src_index(rw, w)]
    mx = rs.amax((-2, -1), keepdim=True)
    ratio = rs / mx
    th32 = torch.tensor(th, dtype=torch.float32).item()
    out = torch.full(ratio.shape, -1, dtype=torch.int8)
    for p in range(npr):
        rp = ratio[p]
        if exact:
            one = rp.float().double() > th32
            zero = ~one
        else:
            M = margin(n_maps * heads * int((alpha[p] != 0).sum()))
            one = rp * (1 - M) > th32
            zero = rp * (1 + M) <= th32
        zero = zero | torch.isnan(rp)
        out[p][one] = 1
        out[p][zero] = 0
    if both:
        one = (out[0] == 1) | (out[1] == 1)
        zero = (out[0] == 0) & (out[1] == 0)
        out[1] = -1
        out[1][one] = 1
        out[1][zero] = 0
    return out, ratio


def check_mask(fn, case, report=False):
    maps, alpha, kw = make_case(**case)
    got = fn(maps, alpha, kw["h"], kw["w"], kw["th"], kw["both"], kw["res"]).cpu()
    ref, _ = mask_ref(maps, alpha, kw["h"], kw["w"], kw["th"], kw["both"], kw["res"], exact=kw["exact"])
    decided = ref >= 0
    wrong = int((decided & (got != ref.float())).sum())
    undecided = int((~decided).sum())
    frac = undecided / ref.numel()
    bad_values = int(((got != 0) & (got != 1)).sum())
    what = (f"{case['name']}: {wrong} wrong of {int(decided.sum())} decided pixels, {undecided} undecided "
            f"({100 * frac:.3g} %), {int((ref == 1).sum())} ones")
    if report:
        print(what)
    return {"ok": wrong == 0 and bad_values == 0 and frac < MAX_UNDECIDED and (not kw["exact"] or undecided == 0),
            "wrong": wrong, "undecided": undecided, "what": what}


# ------------------------------------------------------------------------------------------------ inputs
SEL = ((5, 70), (9, 40, 66))          # the selected words of prompts 0 and 1: words >= 64 are in the lanes' third stride


def _alpha(words, sel=SEL):
    a = torch.zeros(2, words)
    for p, ws in enumerate(sel):
        a[p, list(ws)] = 1
    return a


def _planted(rh, rw):
    """Corner and border pixels (and one interior pixel at an odd offset) for the unique maxima."""
    return [(0, 0), (0, rw - 1), (rh - 1, 0), (rh - 1, rw - 1), (0, rw // 2), (rh - 1, rw // 3), (rh // 2, 0),
            (rh // 3, rw - 1), (rh - 2, rw - 2)]


def random_maps(res, frames, n_maps, heads, words, seed, zero_frame=None, planted=True):
    """Softmax-like fp16 maps [2, F, heads, r, words] per layer: iid logits per (layer, prompt, frame, head, pixel, word),
    plus a blob on the prompt's selected words whose centre moves with the prompt, the frame and (a little) with the
    layer and head; frames f % 3 != 2 get a unique maximum at one corner / border pixel (cycling).  zero_frame: every map
    of that frame is 0."""
    rh, rw = res
    g = _gen(seed)
    yy, xx = torch.meshgrid(torch.arange(rh, dtype=torch.float32), torch.arange(rw, dtype=torch.float32), indexing="ij")
    centres = torch.rand(2, frames, 2, generator=g) * torch.tensor([rh, rw])
    sigma = 0.22 * min(rh, rw)
    plant = _planted(rh, rw)
    out = []
    for layer in range(n_maps):
        logits = torch.randn(2, frames, heads, rh * rw, words, generator=g)
        for p in range(2):
            for f in range(frames):
                for hd in range(heads):
                    cy = centres[p, f, 0] + 0.6 * (layer - n_maps / 2) + 0.4 * (hd % 3)
                    cx = centres[p, f, 1] - 0.5 * (hd % 2) + 0.3 * layer
                    blob = 4.0 * torch.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * sigma ** 2)).reshape(-1)
                    for wd in SEL[p]:
                        logits[p, f, hd, :, wd] += blob
                if planted and f % 3 != 2:
                    y, x = plant[(f + seed) % len(plant)]
                    for wd in SEL[p]:
                        logits[p, f, :, y * rw + x, wd] += 9.0
        mp = torch.softmax(logits, -1)
        if zero_frame is not None:
            mp[:, zero_frame] = 0
        out.append(mp.half())
    return out


def dyadic_maps(res, frames, seed, n_maps=2, heads=4, words=77, sel=((70,), (3,)), n_ties=6):
    """Map values k / 256; for each prompt's one selected word the sum over the 8 (layer, head) values is an integer field
    S / 256 with S in [0, 2040]: the maximum 2040 at (0, 0) (a source pixel of every resize), random values elsewhere, and n_ties islands (5 x 5 blocks of
    values <= 1020) centred on even pixels at exactly S = 1020, so their pooled value is exactly half the frame's max."""
    rh, rw = res
    g = _gen(seed)
    vals = torch.randint(0, 256, (n_maps, 2, frames, heads, rh * rw, words), generator=g).float()
    for p in range(2):
        for f in range(frames):
            S = torch.randint(0, 2041, (rh, rw), generator=g)
            for _ in range(n_ties):
                cy = 2 * int(torch.randint(2, max(3, (rh - 2) // 2), (1,), generator=g))
                cx = 2 * int(torch.randint(2, max(3, (rw - 2) // 2), (1,), generator=g))
                cy, cx = min(cy, rh - 1), min(cx, rw - 1)
                y0, x0 = max(cy - 2, 0), max(cx - 2, 0)
                S[y0:cy + 3, x0:cx + 3] = torch.randint(0, 1021, S[y0:cy + 3, x0:cx + 3].shape, generator=g)
                S[cy, cx] = 1020
            S[0, 0] = 2040
            S = S.reshape(-1)
            base, rem = S // 8, S % 8
            k = 0
            for layer in range(n_maps):
                for hd in range(heads):
                    vals[layer, p, f, hd, :, sel[p][0]] = (base + (k < rem).long()).float()
                    k += 1
    alpha = torch.zeros(2, words)
    for p in range(2):
        alpha[p, sel[p][0]] = 1
    return [(vals[layer] / 256).half() for layer in range(n_maps)], alpha


def make_case(name, res, size, frames, both, kind="random", n_maps=5, heads=8, words=77, th=0.3, seed=0, zero_frame=None):
    """(maps, alpha, kwargs) of one case."""
    if kind == "dyadic":
        maps, alpha = dyadic_maps(res, frames, seed)
        th = 0.5
    else:
        maps = random_maps(res, frames, n_maps, heads, words, seed, zero_frame=zero_frame)
        alpha = _alpha(words)
    return maps, alpha, {"h": size[0], "w": size[1], "th": th, "both": both, "res": res, "exact": kind == "dyadic"}


def _cases():
    shapes = [((16, 16), (64, 64)), ((16, 16), (16, 16)), ((16, 16), (8, 8)), ((16, 16), (24, 24)),
              ((14, 24), (56, 96)), ((14, 24), (14, 24)), ((14, 24), (7, 12)), ((14, 24), (21, 36)),
              ((32, 32), (128, 128)), ((32, 32), (32, 32)), ((32, 32), (8, 8))]
    cases = []
    for i, (res, size) in enumerate(shapes):
        big = res == (32, 32)
        cases.append(dict(name=f"{res[0]}x{res[1]}->{size[0]}x{size[1]} F{4 if big else 16} both", res=res, size=size,
                          frames=4 if big else 16, both=True, seed=100 + i))
        cases.append(dict(name=f"{res[0]}x{res[1]}->{size[0]}x{size[1]} F1 source", res=res, size=size, frames=1, both=False,
                          seed=200 + i))
    cases.append(dict(name="zero frame 16x16->64x64 F4 both", res=(16, 16), size=(64, 64), frames=4, both=True, seed=300,
                      zero_frame=1))
    cases.append(dict(name="zero frame 14x24->7x12 F3 source", res=(14, 24), size=(7, 12), frames=3, both=False, seed=301,
                      zero_frame=2))
    for i, (res, size) in enumerate([((16, 16), (64, 64)), ((14, 24), (7, 12)), ((16, 16), (24, 24))]):
        cases.append(dict(name=f"dyadic {res[0]}x{res[1]}->{size[0]}x{size[1]} F3 both", res=res, size=size, frames=3,
                          both=True, kind="dyadic", seed=400 + i))
    return {c["name"]: c for c in cases}


CASES = _cases()


# ------------------------------------------------------------------------------------------------ latent blend
def latent_inputs(C, frames, hw, dtype, kind, seed):
    """(src, tgt, mask): N(0, 1) values scaled by 2^k, k uniform in [-8, 8], so |tgt| << |src| (and the reverse) occurs;
    0/1 masks ('binary') or fractional ones in [0, 1] ('fraction')."""
    g = _gen(seed)

    def spread():
        return torch.randn(C, frames, hw, generator=g) * torch.exp2(torch.rand(C, frames, hw, generator=g) * 16 - 8)
    src, tgt = spread(), spread()
    if kind == "binary":
        mask = (torch.rand(frames, hw, generator=g) < 0.5).float()
    else:
        mask = torch.rand(frames, hw, generator=g)
        mask[:, :7] = torch.tensor([0.0, 1.0, 0.5, 0.25, 1 / 3, 0.999, 1e-4])
    return src.to(dtype), tgt.to(dtype), mask


def check_latent(fn, C, frames, hw, dtype, kind, seed=0, device="cpu"):
    src, tgt, mask = latent_inputs(C, frames, hw, dtype, kind, seed)
    src_d, tgt_d, mask_d = src.clone().to(device), tgt.to(device), mask.to(device)
    out, src_after = fn(src_d, tgt_d.clone(), mask_d)
    out, src_after = out.cpu(), src_after.cpu()
    untouched = torch.equal(src_after.view(torch.int16 if dtype == torch.float16 else torch.int32),
                            src.view(torch.int16 if dtype == torch.float16 else torch.int32))
    what = f"latent blend {kind} C{C} F{frames} hw{hw} {str(dtype)[6:]}"
    if kind == "binary":
        want = torch.where(mask[None].bool(), tgt, src)
        same = torch.equal(out.view(torch.int16 if dtype == torch.float16 else torch.int32),
                           want.view(torch.int16 if dtype == torch.float16 else torch.int32))
        return {"ok": same and untouched, "err": 0.0 if same else math.inf, "what": what + f": bit-exact {same}, src kept {untouched}"}
    s, t, m = src.double(), tgt.double(), mask.double()[None]
    ref = s + m * (t - s)
    bound = ((2 * U + U * U) * (1 + U) * m * (t - s).abs() + U * ref.abs()) * (1 + 8 * U)
    err = beyond_rounding(out, ref)
    ratio = (err / bound.clamp_min(1e-300)).max().item() if bool(torch.isfinite(err).all()) else math.inf
    return {"ok": ratio <= 2.0 and untouched, "err": ratio, "what": what + f": worst err / bound {ratio:.3g}, src kept {untouched}"}
