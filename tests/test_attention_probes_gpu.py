"""Per-element attention tests (pytest -m gpu) for all five attention kernels: one-hot value probes that read single
probabilities with relative precision, masked-tail problems whose exact answer is a uniform softmax, and the
explicit-probability pair on edited maps, each against an fp64 softmax of the same fp16 inputs with the bound derived in
tests/attention_probes.py.  Spatial cases run on the wgmma kernel (default, d = 40 / 80) and on the mma.sync kernel
(attn_tc = 0); d = 160 has only the latter."""
import pytest
import torch

from tests import attention_probes as A
from videoswap_b200 import ops

pytestmark = pytest.mark.gpu


def _attn(tc):
    def run(q, k, v, heads, kv_div):
        if tc:
            return ops.attention(q, k, v, heads, kv_div=kv_div)
        ops.set_option("attn_tc", 0)
        try:
            return ops.attention(q, k, v, heads, kv_div=kv_div)
        finally:
            ops.set_option("attn_tc", 1)
    return run


def _tattn(vst):
    def run(qkv, heads):
        ops.set_option("tattn_vst", vst)
        try:
            return ops.temporal_attention(qkv, heads)
        finally:
            ops.set_option("tattn_vst", 1)
    return run


def _temporal(F):
    """Every d and both store paths at F frames (F = 17 is the first with 32 padded frames, 32 the kernel's limit)."""
    def run():
        rs = []
        for d in (40, 80, 160):
            for vst in (1, 0):
                fn = _tattn(vst)
                rs.append(A.check_temporal_probes(fn, 2, F, 20, d, seed=500 + F + d))
                rs.append(A.check_temporal_probes(fn, 1, F, 12, d, sigmas=(1.0,), shift=40.0, seed=600 + F + d))
                rs.append(A.check_temporal_probes(fn, 1, F, 12, d, sigmas=(3.0,), shift=-40.0, seed=700 + F + d))
        return A.merge(*rs)
    return run


ALL = (1.0, 3.0, 6.0)
CASES = {}
for _k, _tc in (("tc", True), ("mma", False)):
    _a = _attn(_tc)
    CASES.update({
        # every key of every map probed: 7 launches of 640 keys at the headline shape, 2 of 1280 at d = 80
        f"sweep_self_d40_n4096_{_k}": lambda a=_a: A.check_probes(a, 2, 4096, 4096, 40, sigmas=(1.0, 3.0), sweep=True, seed=401),
        f"sweep_self_d80_n1100_{_k}": lambda a=_a: A.check_probes(a, 2, 1100, 1100, 80, sigmas=(1.0, 3.0), sweep=True, seed=403),
        # cross-attention: K / V shared by 16 frames; a frame reading the wrong K / V batch reads other keys of other maps
        f"sweep_cross_d40_nk77_{_k}": lambda a=_a: A.check_probes(a, 32, 300, 77, 40, sigmas=ALL, kv_div=16, sweep=True, seed=405),
        f"sweep_cross_d80_nk77_{_k}": lambda a=_a: A.check_probes(a, 32, 260, 77, 80, sigmas=ALL, kv_div=16, sweep=True, seed=408),
        # tile edges, ring wrap, first key of the last tile, last key, at three logit spreads
        f"edges_self_d40_n4096_{_k}": lambda a=_a: A.check_probes(a, 2, 4096, 4096, 40, sigmas=ALL, seed=411),
        f"edges_self_d40_n4095_{_k}": lambda a=_a: A.check_probes(a, 2, 4095, 4095, 40, sigmas=ALL, seed=414),
        f"edges_self_d40_n513_{_k}": lambda a=_a: A.check_probes(a, 3, 513, 513, 40, sigmas=ALL, seed=417),
        f"edges_self_d80_n1100_{_k}": lambda a=_a: A.check_probes(a, 2, 1100, 1100, 80, sigmas=ALL, seed=420),
        f"edges_self_d80_n385_{_k}": lambda a=_a: A.check_probes(a, 3, 385, 385, 80, sigmas=ALL, seed=423),
        # +-40 logit units on every score of a row: the max subtraction and the exp2 range
        f"shift_self_d40_n1024_{_k}": lambda a=_a: A.check_probes(a, 2, 1024, 1024, 40, sigmas=(1.0, 6.0), shift=40.0, sweep=True, seed=426),
        f"shift_self_d80_n513_{_k}": lambda a=_a: A.check_probes(a, 2, 513, 513, 80, sigmas=(1.0, 6.0), shift=-40.0, sweep=True, seed=428),
        # uniform softmax over the real keys: a zero-filled padding key (logit 0 against -20) would take all the mass
        f"tail_self_d40_n321_{_k}": lambda a=_a: A.check_probes(a, 2, 321, 321, 40, tail=True, sweep=True, seed=430),
        f"tail_self_d40_n385_{_k}": lambda a=_a: A.check_probes(a, 2, 385, 385, 40, tail=True, sweep=True, seed=431),
        f"tail_self_d80_n321_{_k}": lambda a=_a: A.check_probes(a, 2, 321, 321, 80, tail=True, sweep=True, seed=432),
        f"tail_self_d80_n385_{_k}": lambda a=_a: A.check_probes(a, 2, 385, 385, 80, tail=True, sweep=True, seed=433),
        f"tail_cross_d40_nk77_{_k}": lambda a=_a: A.check_probes(a, 32, 300, 77, 40, kv_div=16, tail=True, sweep=True, seed=434),
        f"tail_cross_d80_nk77_{_k}": lambda a=_a: A.check_probes(a, 32, 130, 77, 80, kv_div=16, tail=True, sweep=True, seed=435),
    })
_m = _attn(True)                 # d = 160 always runs on the mma.sync kernel
CASES.update({
    "sweep_self_d160_n336": lambda: A.check_probes(_m, 2, 336, 336, 160, sigmas=ALL, sweep=True, seed=440),
    "sweep_cross_d160_nk77": lambda: A.check_probes(_m, 32, 256, 77, 160, sigmas=ALL, kv_div=16, sweep=True, seed=443),
    "edges_self_d160_n1024": lambda: A.check_probes(_m, 2, 1024, 1024, 160, sigmas=ALL, seed=446),
    "shift_self_d160_n256": lambda: A.check_probes(_m, 2, 256, 256, 160, sigmas=(1.0, 6.0), shift=40.0, sweep=True, seed=449),
    "tail_self_d160_n321": lambda: A.check_probes(_m, 2, 321, 321, 160, tail=True, sweep=True, seed=451),
    "tail_cross_d160_nk77": lambda: A.check_probes(_m, 32, 64, 77, 160, kv_div=16, tail=True, sweep=True, seed=452),
})
CASES.update({f"temporal_f{F}": _temporal(F) for F in (1, 2, 15, 16, 17, 24, 32)})
for _d in (40, 80, 160):
    CASES.update({
        f"probs_self_d{_d}": lambda d=_d: A.merge(*[A.check_probs(ops.attention_probs, 2, nk, nk, d, seed=460 + nk)
                                                     for nk in (64, 256, 321)]),
        f"probs_cross_d{_d}": lambda d=_d: A.merge(*[A.check_probs(ops.attention_probs, 4, 200, 77, d, kv_div=kd, seed=470 + kd)
                                                      for kd in (1, 2)]),
        f"probs_tail_d{_d}": lambda d=_d: A.merge(A.check_probs(ops.attention_probs, 2, 321, 321, d, tail=True, seed=480),
                                                  A.check_probs(ops.attention_probs, 4, 100, 77, d, kv_div=2, tail=True, seed=481)),
        f"apply_probs_edited_d{_d}": lambda d=_d: A.merge(A.check_apply_probs(ops.attention_apply_probs, 2, 256, 256, d, seed=490),
                                                          A.check_apply_probs(ops.attention_apply_probs, 4, 200, 77, d, kv_div=2,
                                                                              seed=491)),
    })


@pytest.mark.parametrize("name", sorted(CASES))
def test_attention_probes(name):
    r = CASES[name]()
    torch.cuda.synchronize()
    assert r["ok"], f"{name}: {r.get('what', '')}: worst err / bound {r['err']:.4g}"
