"""The power of the CFG + DDIM probes (tests/ddim_probes.py), shown without a GPU.  A torch emulation of
`cfg_ddim_kernel` -- the library's fp32 coefficients from the fp32 alphas, the guidance lerp and the two-term update in
fp32, the fp16 or fp32 store -- stays within every bound (half of what the comparator allows) at every step of all three
schedules, and every planted bug fails the comparator.  For each bug the random-input comparator of tests/kernel_checks.py (one (a_t, a_p) pair, rel 2^-9,
abs 1e-3) is shown to catch it or let it through."""
import numpy as np
import pytest
import torch

from tests import ddim_probes as D
from tests import kernel_checks as KC
from videoswap_b200.scheduler import DDIMInverseScheduler, DDIMScheduler

N = 4097             # odd


def emulate(mutation=None):
    """step(eps, x, g, cfg, a_t, a_p) with cfg_ddim_kernel's arithmetic, optionally with one planted bug."""
    def step(eps, x, g, cfg, a_t, a_p):
        if mutation == "alphas_swapped":
            a_t, a_p = a_p, a_t
        c_x, c_e = D.library_coefficients(a_t, a_p)
        if mutation == "coefficients_fp16":
            c_x, c_e = np.float16(c_x), np.float16(c_e)
        c_x, c_e = float(c_x), float(c_e)
        n = x.numel()
        e = eps[:n].float()
        if cfg:
            ec = eps[n:2 * n].float()
            if mutation == "uncond_cond_swapped":
                e, ec = ec, e
            e = e + g * (ec - e)
        elif mutation == "nocfg_reads_second_half":
            e = torch.as_strided(eps, (n,), (1,), eps.storage_offset() + n).float()
        return (torch.tensor(c_x, dtype=torch.float32) * x.float() + torch.tensor(c_e, dtype=torch.float32) * e).to(x.dtype)
    return step


def scheduler_alphas(set_alpha_to_one=False):
    """alphas(schedule, t) from the project's schedulers (set_alpha_to_one=True plants final_alpha_cumprod = 1)."""
    fwd = DDIMScheduler(set_alpha_to_one=set_alpha_to_one)
    fwd.set_timesteps(D.STEPS)
    inv = {}
    for conv in ("0.19.3", "0.21"):
        inv[conv] = DDIMInverseScheduler(convention=conv, set_alpha_to_one=set_alpha_to_one)
        inv[conv].set_timesteps(D.STEPS)

    def alphas(schedule, t):
        return fwd.alphas(t) if schedule == "forward" else inv[schedule.split("_")[1]].alphas(t)
    return alphas


CASES = [(s, dt, cfg) for s in D.SCHEDULES for dt in (torch.float16, torch.float32) for cfg in (True, False)]


def _run_all(step, alphas):
    return [D.check_schedule(step, alphas, s, dt, cfg, N, seed=7) for s, dt, cfg in CASES]


def test_the_schedules_use_the_restated_alphas():
    """Every (a_t, a_p) of the project's schedulers equals the restated table, including both ends."""
    alphas = scheduler_alphas()
    for s in D.SCHEDULES:
        ts = [t for t, _, _ in D.pairs(s)]
        sched = DDIMScheduler() if s == "forward" else DDIMInverseScheduler(convention=s.split("_")[1])
        sched.set_timesteps(D.STEPS)
        assert list(sched.timesteps) == ts, s
        for t, a_t, a_p in D.pairs(s):
            assert alphas(s, t) == (a_t, a_p), (s, t)
    ac = D.alphas_cumprod()
    assert D.pairs("forward")[-1] == (1, ac[1].item(), ac[0].item())
    assert D.pairs("inverse_0.19.3")[-1] == (981, ac[981].item(), ac[999].item())
    assert D.pairs("inverse_0.21")[0] == (1, ac[0].item(), ac[1].item())


def test_emulation_within_every_bound():
    worst = 0.0
    for r in _run_all(emulate(), scheduler_alphas()):
        print(r["what"])
        assert r["err"] <= D.TOL / 2, r["what"]
        worst = max(worst, r["err"])
    print(f"worst err / bound over {len(CASES)} cases x 50 steps: {worst:.3g}")


def test_device_coefficients_in_fp64_stay_within_the_bound():
    """ops.ddim_coefficients (fp64, rounded to fp32 when uploaded) with the kernel's arithmetic."""
    from videoswap_b200 import ops

    def step_coef(eps, x, g, cfg, c_x, c_e):
        n = x.numel()
        e = eps[:n].float()
        if cfg:
            e = e + g * (eps[n:2 * n].float() - e)
        cx, ce = torch.tensor([c_x, c_e], dtype=torch.float32)
        return (cx * x.float() + ce * e).to(x.dtype)
    for s, dt, cfg in CASES:
        r = D.check_coefficients(step_coef, s, dt, cfg, N, ops.ddim_coefficients, seed=8)
        assert r["err"] <= D.TOL / 2, r["what"]


MUTATIONS = {
    "coefficients_fp16": (emulate("coefficients_fp16"), scheduler_alphas()),
    "uncond_cond_swapped": (emulate("uncond_cond_swapped"), scheduler_alphas()),
    "alphas_swapped": (emulate("alphas_swapped"), scheduler_alphas()),
    "final_alpha_cumprod_one": (emulate(), scheduler_alphas(set_alpha_to_one=True)),
    "nocfg_reads_second_half": (emulate("nocfg_reads_second_half"), scheduler_alphas()),
}


@pytest.mark.parametrize("bug", sorted(MUTATIONS))
def test_planted_bug_is_rejected(bug):
    rs = _run_all(*MUTATIONS[bug])
    bad = [r["what"] for r in rs if not r["ok"]]
    print(f"{bug}: rejected by {len(bad)} of {len(rs)} cases, e.g. {bad[:1]}")
    assert bad, bug


# ---------------------------------------------------------------------------------------------------- the old comparator
def _old(step, cfg=True, dtype=torch.float16, seed=150):
    """kernel_checks.check_cfg_ddim / _nocfg: one (a_t, a_p) pair with the alphas written into the check, 1 024
    elements, rel 2^-9, abs 1e-3."""
    n = 4 * 4 * 8 * 8
    eps, x = D.inputs(n, dtype, cfg, seed)
    a_t, a_p = (0.0047, 0.0058) if cfg else (0.0058, 0.0047)
    out = step(eps, x, 7.5, cfg, a_t, a_p)
    ref, _ = D.ddim_ref_bound(eps, x, 7.5, cfg, a_t, a_p)
    return KC._res(out, ref, rel=2 ** -9, abs_=1e-3)["ok"]


OLD = {
    "coefficients_fp16": lambda: _old(emulate("coefficients_fp16")),
    "uncond_cond_swapped": lambda: _old(emulate("uncond_cond_swapped")),
    "alphas_swapped": lambda: _old(emulate("alphas_swapped")),
    # the old check takes its alphas from literals, never from a scheduler: a wrong end of the table cannot reach it
    "final_alpha_cumprod_one": lambda: _old(emulate()),
    "nocfg_reads_second_half": lambda: _old(emulate("nocfg_reads_second_half"), cfg=False),
}

# What the random-input comparator says about each planted bug (True = it lets the bug through).
OLD_PASSES = {
    "coefficients_fp16": True,
    "uncond_cond_swapped": False,
    "alphas_swapped": False,
    "final_alpha_cumprod_one": True,
    "nocfg_reads_second_half": False,
}


def test_old_comparator_passes_the_correct_emulation():
    assert _old(emulate()) and _old(emulate(), cfg=False)


@pytest.mark.parametrize("bug", sorted(OLD))
def test_old_comparator_verdict(bug):
    """The recorded verdict of the single-pair comparator on each planted bug holds."""
    assert OLD[bug]() == OLD_PASSES[bug], bug
