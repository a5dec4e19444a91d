"""GPU parity tests (pytest -m gpu) aimed at the warp-specialised wgmma attention kernel (attention_tc.cu): a CTA covers
128 queries with two consumer warpgroups of 64 rows, streams 128-key K / V tiles through a ring of 4 stages at d = 40 and
3 at d = 80, and the two consumers take turns on the tensor cores.  The shapes below sit on the edges of that schedule."""
import pytest
import torch

from tests.kernel_checks import _flag, _rand, check_attn_dominant_key, check_cross_attention, check_self_attention
from videoswap_b200 import ops

pytestmark = pytest.mark.gpu

BKV = 128                    # TCfg<D>::BKV and ::STAGES in attention_tc.cu (test_attn_sass_cpu.py checks they match)
STAGES = {40: 4, 80: 3}


def check_deterministic(B=2, N=1000, C=320, seed=300, cross_frames=0):
    """Two launches on the same inputs are bit-identical: the kernel has no atomics, so a difference is a race in the
    K / V ring or in the consumers' hand-off."""
    if cross_frames:
        q = _rand((B * cross_frames, N, C), seed).half()
        kv = _rand((B, 77, 2 * C), seed + 1).half()
        k, v = kv[..., :C], kv[..., C:]
    else:
        qkv = _rand((B, N, 3 * C), seed).half()
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    kv_div = cross_frames or 1
    outs = [ops.attention(q, k, v, 8, kv_div=kv_div) for _ in range(3)]
    return _flag(all(torch.equal(outs[0], o) for o in outs[1:]), "attention output differs between launches")


def _ring(d, tiles, extra=0):
    return lambda: check_self_attention(B=2, N=BKV * tiles + extra, C=8 * d, seed=310 + tiles + d)


CASES = {
    # the last CTA's second consumer has no valid query row
    "idle_consumer_d40_n320": lambda: check_self_attention(B=2, N=64 * 5, C=320, seed=301),
    "idle_consumer_d80_n192": lambda: check_self_attention(B=2, N=64 * 3, C=640, seed=302),
    "idle_consumer_d40_n65": lambda: check_self_attention(B=3, N=65, C=320, seed=303),
    "idle_consumer_d80_n65": lambda: check_self_attention(B=3, N=65, C=640, seed=304),
    # key-tile counts of exactly the ring depth, one more, and a single key in the tile after the ring wraps
    "ring_depth_d40": _ring(40, STAGES[40]),
    "ring_depth_plus1_d40": _ring(40, STAGES[40] + 1),
    "ring_wrap_one_key_d40": _ring(40, STAGES[40], 1),
    "ring_depth_d80": _ring(80, STAGES[80]),
    "ring_depth_plus1_d80": _ring(80, STAGES[80] + 1),
    "ring_wrap_one_key_d80": _ring(80, STAGES[80], 1),
    # the row maximum jumps on the last key tile while the two consumers are at different tiles
    "dominant_key_late_d40": lambda: check_attn_dominant_key(B=2, N=BKV * 6 + 1, C=320, where="last", seed=320),
    "dominant_key_late_d80": lambda: check_attn_dominant_key(B=2, N=BKV * 3 + 1, C=640, where="last", seed=321),
    # cross-attention: K / V shared by the 16 frames of a CFG half, several 128-query blocks per frame
    "cross_kv_div16_d40": lambda: check_cross_attention(B=2, Fr=16, N=300, C=320, seed=330),
    "cross_kv_div16_d80": lambda: check_cross_attention(B=2, Fr=16, N=260, C=640, seed=331),
    # run-to-run determinism
    "deterministic_self_d40": lambda: check_deterministic(B=2, N=1000, C=320, seed=340),
    "deterministic_self_d80": lambda: check_deterministic(B=2, N=700, C=640, seed=341),
    "deterministic_cross_d40": lambda: check_deterministic(B=2, N=300, C=320, seed=342, cross_frames=16),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_attention_tc(name):
    r = CASES[name]()
    torch.cuda.synchronize()
    assert r["ok"], f"{name}: {r.get('what', '')} max abs err {r['err']:.4g} > tol {r['tol']:.4g} (max |ref| {r['ref']:.4g})"
