"""The power of the blend probes (tests/blend_probes.py), shown without a GPU.  A torch emulation of `blend_mask_kernel`
-- the alpha-weighted fp32 sum over layers, heads and words read through the layer-major, prompt-minor pointer table,
the fp32 mean factor, the 3 x 3 max pool with -inf padding, the fp32 nearest indices, the frame's max over the resized
pixels, the fp32 ratio and the strict test, the OR with prompt 0 -- matches every decided pixel of every case (the
dyadic ones on every pixel), and each planted bug is rejected by a named case.  The same for `latent_blend_kernel`,
where the plain lerp at m = 0 / 1 (the kernel before it selected) is among the rejected bugs."""
import functools

import pytest
import torch

from tests import blend_probes as B


def _pool(m, mutation):
    """3 x 3 max pool, stride 1, -inf padding, over the last two dims of m [F, rh, rw]; the own pixel is always read."""
    rh, rw = m.shape[-2:]
    pad = torch.nn.functional.pad(m, (1, 1, 1, 1), value=-float("inf"))
    out = m.clone()
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if mutation == "pool_4_neighbour" and dy != 0 and dx != 0:
                continue
            sh = pad[..., 1 + dy:1 + dy + rh, 1 + dx:1 + dx + rw].clone()
            if mutation == "pool_short_right" and dx == 1:
                sh[..., :, rw - 2] = -float("inf")          # the last column is never read as a neighbour
            if mutation == "pool_short_bottom" and dy == 1:
                sh[..., rh - 2, :] = -float("inf")
            out = torch.maximum(out, sh)
    return out


def _index(n_in, n_out, mutation):
    scale = torch.tensor(n_in, dtype=torch.float32) / torch.tensor(n_out, dtype=torch.float32)
    dst = torch.arange(n_out, dtype=torch.float32)
    if mutation == "nearest_rounded":
        src = torch.round(dst * scale)
    elif mutation == "nearest_half_offset":
        src = torch.floor((dst + 0.5) * scale)
    else:
        src = torch.floor(dst * scale)
    return src.long().clamp_max(n_in - 1)


def emulate_mask(mutation=None):
    def fn(maps, alpha, h, w, th, both, res):
        npr = 2 if both else 1
        n_maps, rh, rw = len(maps), res[0], res[1]
        flat = [it[q] for it in maps for q in range(npr)]                  # the host's pointer table
        frames, heads, r, words = flat[0].shape
        inv = torch.tensor(1.0 / (n_maps * heads), dtype=torch.float32)
        th32 = torch.tensor(th, dtype=torch.float32)
        out = torch.zeros(npr, frames, h, w)
        for pr in range(npr):
            a = alpha[0 if mutation == "prompt1_with_alpha0" else pr].clone()
            if mutation == "words_64_up_dropped":
                a[64:] = 0
            acc = torch.zeros(frames, r)
            for layer in range(n_maps):
                mp = flat[pr * n_maps + layer if mutation == "pointers_prompt_major" else layer * npr + pr].float()
                if mutation == "frame0_maps":
                    mp = mp[:1].expand_as(mp)
                if mutation == "head0_only":
                    mp = mp[:, :1]
                acc += (mp * a).sum((1, 3))
            m = (acc * inv).reshape(frames, rh, rw)
            pooled = _pool(m, mutation)
            rs = pooled[:, _index(rh, h, mutation)][:, :, _index(rw, w, mutation)]
            src = pooled if mutation == "normalise_before_resize" else rs
            mx = src.amax((-2, -1), keepdim=True)
            q = rs / mx
            bit = (q >= th32) if mutation == "greater_equal" else (q > th32)
            if both and pr > 0:
                first = out[0, :1].expand(frames, h, w) if mutation == "both_or_frame0" else out[0]
                bit = bit | (first != 0)
            out[pr] = bit.float()
        return out
    return fn


@functools.lru_cache(maxsize=None)
def _verdict(mutation, name):
    return B.check_mask(emulate_mask(mutation), B.CASES[name])


@pytest.mark.parametrize("name", sorted(B.CASES))
def test_emulation_matches_every_decided_pixel(name):
    r = B.check_mask(emulate_mask(), B.CASES[name], report=True)
    assert r["ok"], r["what"]


def test_resize_indices_are_torchs():
    """src_index reads torch's nearest indices; they are floor(dst * fp32(in / out)), which the rounded and the
    half-offset indices are not at the product shapes."""
    for n_in, n_out in ((16, 64), (16, 8), (16, 24), (14, 56), (14, 7), (24, 96), (24, 12), (24, 36), (14, 21), (32, 8)):
        assert torch.equal(B.src_index(n_in, n_out), _index(n_in, n_out, None))


# Each planted bug and the case that rejects it.
MUTATIONS = {
    "nearest_rounded": "16x16->64x64 F16 both",
    "nearest_half_offset": "16x16->8x8 F16 both",
    "pool_4_neighbour": "16x16->64x64 F16 both",
    "pool_short_right": "14x24->56x96 F16 both",
    "pool_short_bottom": "14x24->56x96 F16 both",
    "normalise_before_resize": "32x32->8x8 F1 source",
    "greater_equal": "dyadic 16x16->64x64 F3 both",
    "both_or_frame0": "16x16->16x16 F16 both",
    "prompt1_with_alpha0": "16x16->64x64 F16 both",
    "words_64_up_dropped": "14x24->7x12 F1 source",
    "frame0_maps": "14x24->14x24 F16 both",
    "head0_only": "16x16->24x24 F16 both",
    "pointers_prompt_major": "14x24->21x36 F16 both",
}


@pytest.mark.parametrize("bug", sorted(MUTATIONS))
def test_planted_bug_is_rejected(bug):
    r = _verdict(bug, MUTATIONS[bug])
    print(f"{bug}: {r['what']}")
    assert not r["ok"], r["what"]


# ---------------------------------------------------------------------------------------------------- latent blend
def emulate_latent(mutation=None):
    def fn(src, tgt, mask):
        s, t = src.float(), tgt.float()
        m = mask[None]
        if mutation == "mask_frame0":
            m = mask[None, :1].expand_as(m)
        v = s + m * (t - s)
        if mutation != "lerp_at_the_ends":
            v = torch.where(m == 0, s, torch.where(m == 1, t, v))
        if mutation == "fp16_lerp" and tgt.dtype == torch.float16:
            v = (s.half() + (m * (t - s)).half()).float()
        tgt.copy_(v.to(tgt.dtype))
        if mutation == "src_written":
            src.copy_(tgt)
        return tgt, src
    return fn


LATENT = [(4, 16, 64 * 64, torch.float16, "binary"), (4, 1, 56 * 96, torch.float32, "binary"),
          (4, 32, 8 * 8, torch.float16, "fraction"), (4, 3, 7 * 12, torch.float32, "fraction")]


@pytest.mark.parametrize("C,frames,hw,dtype,kind", LATENT)
def test_latent_emulation(C, frames, hw, dtype, kind):
    r = B.check_latent(emulate_latent(), C, frames, hw, dtype, kind)
    print(r["what"])
    assert r["ok"] and r["err"] <= 1.0, r["what"]


@pytest.mark.parametrize("bug,case", [("mask_frame0", LATENT[0]), ("fp16_lerp", LATENT[2]), ("src_written", LATENT[1]),
                                      ("lerp_at_the_ends", LATENT[0]), ("lerp_at_the_ends", LATENT[1])])
def test_latent_planted_bug_is_rejected(bug, case):
    r = B.check_latent(emulate_latent(bug), *case)
    assert not r["ok"], r["what"]
