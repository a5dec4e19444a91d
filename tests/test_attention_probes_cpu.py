"""The power of the attention probes (tests/attention_probes.py), shown without a GPU: a torch emulation of the wgmma
kernel's arithmetic (attention_tc.cu: 128-key tiles, online maximum, P rounded to fp16 relative to the running maximum,
fp32 O and l, fp16 output) and of attn_probs_kernel must pass the comparators with at least 2x margin at the shapes the
GPU tests use, and every planted bug in that arithmetic must fail them."""
import math

import pytest
import torch

from tests import attention_probes as A

LOG2E = 1.4426950408889634


def _sc(d):
    """scale_log2 as the kernels compute it, in fp32."""
    return torch.tensor(LOG2E, dtype=torch.float32) / torch.tensor(float(d)).sqrt()


class TcEmulation:
    """attn(q, k, v, heads, kv_div) with the wgmma kernel's arithmetic and an optional planted mutation.  The softmax
    part does not depend on V, so it is kept while the same q / k tensors come back with other probes."""
    BKV, STAGES = A.BKV_TC, A.STAGES_TC

    def __init__(self, mutation=None, **kw):
        self.mutation, self.kw = mutation, kw
        self._qk = (None, None)

    def _softmax(self, q, k, heads, kv_div):
        B, nq, C = q.shape
        d, nk, Bk = C // heads, k.shape[1], k.shape[0]
        sc = _sc(d)
        self.kidx = torch.arange(B) % Bk if self.mutation == "kv_batch_mod" else torch.arange(B) // kv_div
        qh = q.float().reshape(B, nq, heads, d).transpose(1, 2)
        nkt = -(-nk // self.BKV)
        kh = torch.zeros(Bk, nkt * self.BKV, C)                # TMA zero-fills keys beyond nk
        kh[:, :nk] = k.float()
        kh = kh.reshape(Bk, -1, heads, d).transpose(1, 2)
        m = torch.full((B, heads, nq, 1), -math.inf)
        l = torch.zeros(B, heads, nq, 1)
        self.tiles, prev_alpha = [], None
        for t in range(nkt):
            keys = torch.arange(t * self.BKV, (t + 1) * self.BKV)
            s = qh @ kh[self.kidx][:, :, keys].transpose(-1, -2)
            masked = keys >= nk
            if self.mutation == "unmask_pad":
                masked &= keys != nk
            s[..., masked] = -math.inf
            mx = torch.maximum(m, s.amax(-1, keepdim=True))
            alpha = torch.exp2((m - mx) * sc)
            ms = mx * sc
            p = torch.exp2((s.double() * sc.double() - ms.double()).float())      # fmaf(s, sc, -ms)
            if self.mutation == "tile_scale":
                lo, hi = self.kw["keys"]
                p[..., (keys >= lo) & (keys < hi)] *= 1.03
            l = l * alpha + p.sum(-1, keepdim=True)
            p16 = p.bfloat16().float() if self.mutation == "p_bf16" else p.half().float()
            a_o = prev_alpha if self.mutation == "stale_alpha" and t == self.STAGES[d] else alpha
            self.tiles.append((keys, p16, a_o))
            prev_alpha, m = alpha, mx
        self.inv = 1.0 / l
        if self.mutation == "normaliser":
            self.inv = self.inv * self.kw["factor"]

    def __call__(self, q, k, v, heads, kv_div=1):
        if self._qk[0] is not q or self._qk[1] is not k:
            self._softmax(q, k, heads, kv_div)
            self._qk = (q, k)
        B, nq, C = q.shape
        nk = v.shape[1]
        vp = torch.zeros(v.shape[0], len(self.tiles) * self.BKV, C)
        vp[:, :nk] = v.float()
        vh = vp[self.kidx].reshape(B, -1, heads, C // heads).transpose(1, 2)
        o = torch.zeros(B, heads, nq, C // heads)
        for keys, p16, a_o in self.tiles:
            o = o * a_o + p16 @ vh[:, :, keys]
        return (o * self.inv).half().transpose(1, 2).reshape(B, nq, C)


def emulate_probs(mutation=None):
    """probs_fn with attn_probs_kernel's arithmetic: fp32 scores, exact row maximum, fp32 normaliser, one fp16 rounding."""
    def run(q, k, heads, kv_div=1):
        B, nq, C = q.shape
        d = C // heads
        sc = _sc(d)
        qh = q.float().reshape(B, nq, heads, d).transpose(1, 2)
        kh = k.float().reshape(k.shape[0], -1, heads, d).transpose(1, 2).repeat_interleave(kv_div, 0)
        s = qh @ kh.transpose(-1, -2)
        e = torch.exp2((s - s.amax(-1, keepdim=True)) * sc)
        p = e * (1.0 / e.sum(-1, keepdim=True))
        if mutation == "near_1e-3":
            p = torch.where((p > 5e-4) & (p < 2e-3), p * 1.05, p)
        return p.half()
    return run


# the GPU tests' shapes (one query batch instead of two where the CPU time needs it)
CASES = {
    "sweep_d40_n4096": lambda a: A.check_probes(a, 1, 4096, 4096, 40, sigmas=(1.0,), sweep=True, seed=11, dev="cpu"),
    "edges_d40_n4096": lambda a: A.check_probes(a, 1, 4096, 4096, 40, sigmas=(3.0, 6.0), seed=12, dev="cpu"),
    "sweep_d80_n1100": lambda a: A.check_probes(a, 1, 1100, 1100, 80, sigmas=(1.0, 3.0), sweep=True, seed=13, dev="cpu"),
    "shift_d40_n1024": lambda a: A.check_probes(a, 1, 1024, 1024, 40, sigmas=(1.0,), shift=40.0, sweep=True, seed=14, dev="cpu"),
    "shift_d80_n513": lambda a: A.check_probes(a, 1, 513, 513, 80, sigmas=(3.0,), shift=-40.0, seed=15, dev="cpu"),
    "tail_d40_n321": lambda a: A.check_probes(a, 2, 321, 321, 40, tail=True, sweep=True, seed=16, dev="cpu"),
    "tail_d80_n385": lambda a: A.check_probes(a, 2, 385, 385, 80, tail=True, sweep=True, seed=17, dev="cpu"),
    "tail_cross_d40_nk77": lambda a: A.check_probes(a, 32, 300, 77, 40, kv_div=16, tail=True, sweep=True, seed=18, dev="cpu"),
    "cross_d40_nk77": lambda a: A.check_probes(a, 32, 300, 77, 40, sigmas=(1.0, 3.0), kv_div=16, sweep=True, seed=19, dev="cpu"),
}
PROBS_CASES = {
    "probs_d40_nk256": lambda f: A.check_probs(f, 2, 256, 256, 40, seed=20, dev="cpu"),
    "probs_cross_d80_nk77": lambda f: A.check_probs(f, 4, 200, 77, 80, kv_div=2, seed=21, dev="cpu"),
    "probs_tail_d40_nk321": lambda f: A.check_probs(f, 2, 321, 321, 40, tail=True, seed=22, dev="cpu"),
}

# (mutation, its parameters, the case that must reject it); the first three are the errors the random-input check of
# tests/kernel_checks.py lets through at this shape
MUTATIONS = {
    "tile128_x1.03": ("tile_scale", {"keys": (5 * 128, 6 * 128)}, "sweep_d40_n4096"),
    "tile64_x1.03": ("tile_scale", {"keys": (11 * 64, 12 * 64)}, "sweep_d40_n4096"),
    "normaliser_x1.01": ("normaliser", {"factor": 1.01}, "sweep_d40_n4096"),
    "normaliser_x1.003": ("normaliser", {"factor": 1.003}, "sweep_d40_n4096"),
    "stale_alpha_after_ring_wrap": ("stale_alpha", {}, "sweep_d40_n4096"),
    "p_rounded_to_bf16": ("p_bf16", {}, "sweep_d40_n4096"),
    "padding_key_unmasked": ("unmask_pad", {}, "tail_d40_n321"),
    "kv_batch_b_mod_bk": ("kv_batch_mod", {}, "cross_d40_nk77"),
}


def _msg(name, r):
    return f"{name}: worst err / bound {r['err']:.3g} ({r.get('what', '')})"


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_kernel_passes_with_margin(name):
    r = CASES[name](TcEmulation())
    assert r["ok"] and r["err"] <= 0.5, _msg(name, r)


@pytest.mark.parametrize("name", sorted(PROBS_CASES))
def test_emulated_probs_pass_with_margin(name):
    r = PROBS_CASES[name](emulate_probs())
    assert r["ok"] and r["err"] <= 0.5, _msg(name, r)


@pytest.mark.parametrize("name", sorted(MUTATIONS))
def test_planted_mutation_is_rejected(name):
    mutation, kw, case = MUTATIONS[name]
    r = CASES[case](TcEmulation(mutation, **kw))
    assert not r["ok"], _msg(name, r)


def test_probabilities_near_1e3_off_by_5_percent_are_rejected():
    r = PROBS_CASES["probs_d40_nk256"](emulate_probs("near_1e-3"))
    assert not r["ok"], _msg("near_1e-3", r)
