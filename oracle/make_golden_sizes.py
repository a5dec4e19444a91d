"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/unet_tiny_odd.pt and unet_full_arch_odd.pt by running the
REFERENCE's own model files (through oracle/diffusers_stub, as oracle/make_golden.py does) at latent sizes that are not
multiples of 8 -- the reference's forward_upsample_size path.  Run where the reference tree is checked out:
    VIDEOSWAP_REFERENCE=<checkout> python -m oracle.make_golden_sizes
The fixtures pin oracle/sized.py (tests/test_latent_sizes_cpu.py) wherever the reference is absent."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden import OUT, randn, run_case  # noqa: E402
from oracle.sized import level_sizes  # noqa: E402

# 9x13 -> 5x7 -> 3x4 -> 2x2: both axes odd at two up-samplers; 45x60 (a 360x480 video) -> 23x30 -> 12x15 -> 6x8: odd W at
# the first up-sampler, odd H at the other two, N = 2700 attention
CASES = {
    "tiny_odd": dict(boc=(32, 64, 128, 128), ctx=64, groups=8, batch=2, frames=2, h=9, w=13, edlora=True,
                     residuals=True, t=981, pe=24),
    "full_arch_odd": dict(boc=(320, 640, 1280, 1280), ctx=768, groups=32, batch=1, frames=2, h=45, w=60, edlora=True,
                          residuals=True, t=981, pe=24),
}


def make_inputs(case):
    """Shared by the golden maker and the tests: seeded sample [B, 4, F, h, w], embeddings and residuals on the ceil chain
    of level sizes (the same seeds as oracle/make_golden.py's cases)."""
    b, f, h, w = case["batch"], case["frames"], case["h"], case["w"]
    x = randn((b, 4, f, h, w), 2)
    ehs = randn((b, 16, 77, case["ctx"]), 3) if case["edlora"] else randn((b, 77, case["ctx"]), 3)
    res = None
    if case["residuals"]:
        res = [0.5 * randn((b * f, c, lh, lw), 10 + l) for l, (c, (lh, lw)) in enumerate(zip(case["boc"], level_sizes(h, w)))]
    return x, ehs, res


if __name__ == "__main__":
    import oracle.make_golden as G
    os.makedirs(OUT, exist_ok=True)
    G.make_inputs = make_inputs            # run_case draws its inputs through this name
    for n in sys.argv[1:] or list(CASES):
        run_case(n, CASES[n])
