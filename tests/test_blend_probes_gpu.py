"""Per-element tests of the attention-controller blend kernels (pytest -m gpu), with the reference, decision margin and
cases of tests/blend_probes.py: every case through `vs_blend_mask` directly and through `SpatialBlender._mask` (the
host's layer-major, prompt-minor pointer table), every decided pixel exact, the dyadic cases and their exact ties on
every pixel; the latent blend bit for bit with 0/1 masks and within its bound with fractional ones; and the argument
checks of `vs_blend_mask`, which reject before any launch."""
import ctypes as C

import pytest
import torch

from tests import blend_probes as B
from videoswap_b200 import _lib
from videoswap_b200.p2p import SpatialBlender

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _direct(maps, alpha, h, w, th, both, res):
    npr = 2 if both else 1
    flat = [m[q].cuda().contiguous() for m in maps for q in range(npr)]          # layer-major, prompt-minor
    ptrs = torch.tensor([t.data_ptr() for t in flat], dtype=torch.int64, device="cuda")
    frames, heads, _, words = flat[0].shape
    a = alpha[:npr].cuda().contiguous()
    mask = torch.full((npr, frames, h, w), float("nan"), device="cuda")
    _lib.call("vs_blend_mask", _stream(), C.c_void_p(ptrs.data_ptr()), len(maps), npr, frames, heads, res[0], res[1], words,
              C.c_void_p(a.data_ptr()), 1, h, w, float(th), int(both), C.c_void_p(mask.data_ptr()))
    torch.cuda.synchronize()
    return mask


def _blender(maps, alpha, h, w, th, both, res):
    sb = SpatialBlender(alpha.cuda(), th=(th, th), prompt_choose="both" if both else "source")
    mask = sb._mask([m.cuda() for m in maps], h, w)
    torch.cuda.synchronize()
    return mask


@pytest.mark.parametrize("name", sorted(B.CASES))
@pytest.mark.parametrize("path", ["vs_blend_mask", "SpatialBlender"])
def test_blend_mask_every_decided_pixel(name, path):
    r = B.check_mask(_direct if path == "vs_blend_mask" else _blender, B.CASES[name], report=True)
    assert r["ok"], r["what"]


def test_blend_mask_rejects_bad_arguments_before_any_launch():
    # sized for the largest accepted launch below (r = 32 x 32 pixels, 8 words); the rejected calls never launch
    maps = [torch.zeros(1, 1, 1, 32 * 32, 8, dtype=torch.float16, device="cuda")]
    ptrs = torch.tensor([maps[0].data_ptr()], dtype=torch.int64, device="cuda")
    alpha = torch.ones(1, 8, device="cuda")
    mask = torch.full((1, 1, 8, 8), float("nan"), device="cuda")

    def call(frames=1, heads=1, rh=4, rw=4, words=8, h=8, w=8, n_prompts=1):
        _lib.call("vs_blend_mask", _stream(), C.c_void_p(ptrs.data_ptr()), 1, n_prompts, frames, heads, rh, rw, words,
                  C.c_void_p(alpha.data_ptr()), 1, h, w, 0.3, 0, C.c_void_p(mask.data_ptr()))

    call()
    torch.cuda.synchronize()
    bad = [dict(rh=32, rw=33), dict(rh=1025, rw=1), dict(rh=-4, rw=-4), dict(rh=0), dict(rh=65536, rw=65536),
           dict(frames=0), dict(heads=0), dict(words=0), dict(h=0), dict(w=-8), dict(n_prompts=3), dict(n_prompts=0)]
    for kw in bad:
        n0 = _lib.lib().vs_launch_count()
        with pytest.raises(_lib.VSError, match="blend_mask"):
            call(**kw)
        assert _lib.lib().vs_launch_count() == n0, kw
    n0 = _lib.lib().vs_launch_count()
    call(rh=32, rw=32)                                  # r = 1024 is the largest map the kernel takes
    torch.cuda.synchronize()
    assert _lib.lib().vs_launch_count() == n0 + 1
    assert torch.equal(mask, torch.zeros_like(mask))    # all-zero maps: 0 / 0 gives 0 everywhere


# ------------------------------------------------------------------------------------------------ latent blend
def _latent(src, tgt, mask):
    ch, frames, hw = tgt.shape
    _lib.call("vs_latent_blend", _stream(), C.c_void_p(src.data_ptr()), C.c_void_p(tgt.data_ptr()),
              C.c_void_p(mask.data_ptr()), int(tgt.dtype == torch.float32), ch, frames, hw)
    torch.cuda.synchronize()
    return tgt, src


# 4 x 32 x 96 x 96 = 1 179 648 elements: 2.18 times the capped grid (132 SMs x 16 blocks x 256 threads = 540 672), so
# every thread goes round the grid-stride loop at least twice and some three times
LATENT = [(4, 1, 64 * 64), (4, 16, 64 * 64), (4, 16, 56 * 96), (4, 32, 8 * 8), (4, 32, 96 * 96)]


@pytest.mark.parametrize("C_,frames,hw", LATENT)
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("kind", ["binary", "fraction"])
def test_latent_blend(C_, frames, hw, dtype, kind):
    r = B.check_latent(_latent, C_, frames, hw, dtype, kind, seed=frames + hw, device="cuda")
    print(r["what"])
    assert r["ok"], r["what"]
