"""Model-level parity helpers: the native UNet / pipeline (through the C-ABI) vs the CPU oracle on seeded inputs."""
from __future__ import annotations

import math
import os

import torch

from oracle import unet3d_oracle as O
from videoswap_b200 import (AnimateDiffUNet3DModel, DDIMScheduler, SparsePointAdapter, VideoSwapPipeline,
                            adapter_param_shapes, seeded_state_dict, unet_param_shapes)

GOLD = os.path.join(os.path.dirname(__file__), "golden")
_CACHE = {}


def psnr(out: torch.Tensor, ref: torch.Tensor) -> float:
    out, ref = out.float().cpu(), ref.float().cpu()
    mse = ((out - ref) ** 2).mean().item()
    rng = (ref.max() - ref.min()).item()
    return float("inf") if mse == 0 else 10 * math.log10(rng * rng / mse)


def randn(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def get_model():
    """Full SD-1.5 + AnimateDiff architecture with seeded weights: (native model on cuda fp16, fp32 state dict)."""
    if "m" not in _CACHE:
        m = AnimateDiffUNet3DModel(init="empty")
        sd = seeded_state_dict(unet_param_shapes(m.cfg), seed=0)
        m.load_state_dict(sd)
        m = m.half().cuda()
        # the oracle sees the SAME fp16-rounded weights, so the comparison isolates kernel arithmetic
        sd16 = {k: (v.half().float() if not k.endswith(".pe") else v) for k, v in sd.items()}
        _CACHE["m"] = (m, sd16)
    return _CACHE["m"]


def fresh_model():
    """A second, independent model instance (own native handle and workspace) with random weights made on the GPU."""
    m = AnimateDiffUNet3DModel(init="empty")
    g = torch.Generator(device="cuda").manual_seed(0)
    sd = {}
    for name, shape in unet_param_shapes(m.cfg).items():
        if name.endswith(".pe"):
            continue
        if len(shape) >= 2:
            sd[name] = ((torch.rand(shape, device="cuda", generator=g) * 2 - 1) / math.sqrt(math.prod(shape[1:]))).half()
        elif name.endswith(".weight"):
            sd[name] = (1 + 0.1 * torch.randn(shape, device="cuda", generator=g)).half()
        else:
            sd[name] = (0.02 * torch.randn(shape, device="cuda", generator=g)).half()
    m.load_state_dict(sd, strict=False, assign=True)
    return m.half().cuda()


def nhwc_tap_to_ncfhw(t, B):
    n, h, w, c = t.shape
    return t.float().cpu().reshape(B, n // B, h, w, c).permute(0, 4, 1, 2, 3)


def unet_vs_oracle(B=1, Fr=2, hw=8, edlora=True, residuals=False, t=981, taps=False, w=None):
    m, sd = get_model()
    w = hw if w is None else w                      # non-square latents (the reference's usual 448x768 -> 56x96)
    x = randn((B, 4, Fr, hw, w), 2)
    ehs = randn((B, 16, 77, 768), 3) if edlora else randn((B, 77, 768), 3)
    res = None
    if residuals:
        boc = m.cfg.block_out_channels
        res = [0.5 * randn((B * Fr, c, max(hw >> l, 1), max(w >> l, 1)), 10 + l) for l, c in enumerate(boc)]
    x16, e16 = x.half(), ehs.half()
    res16 = [r.half() for r in res] if res else None
    otaps, ntaps = ({}, {}) if taps else (None, None)
    with torch.no_grad():
        ref = O.unet_forward(sd, O.OracleConfig(), x16.float(), t, e16.float(), [r.float() for r in res16] if res16 else None,
                             taps=otaps)
    out = m(x16.cuda(), t, e16.cuda(), down_block_additional_residuals=[r.cuda() for r in res16] if res16 else None,
            return_dict=False, _taps=ntaps)[0]
    torch.cuda.synchronize()
    r = {"psnr": psnr(out, ref), "max_err": (out.float().cpu() - ref).abs().max().item(), "ref_max": ref.abs().max().item(),
         "finite": bool(torch.isfinite(out).all().item())}
    if taps:
        r["taps"] = {}
        for k, v in ntaps.items():
            if k in otaps:
                o = nhwc_tap_to_ncfhw(v, B)
                r["taps"][k] = {"psnr": psnr(o, otaps[k]), "max_err": (o - otaps[k]).abs().max().item(),
                                "ref_max": otaps[k].abs().max().item()}
    return r


def unet_vs_reference_golden(name="full_arch_small"):
    """tests/golden/unet_<name>.pt was produced by the REFERENCE's own model files (oracle/make_golden.py)."""
    from oracle.make_golden import make_inputs
    g = torch.load(os.path.join(GOLD, f"unet_{name}.pt"))
    case = g["case"]
    m, _ = get_model()
    x, ehs, res = make_inputs(case)
    res16 = [r.half().cuda() for r in res] if res else None
    out = m(x.half().cuda(), case["t"], ehs.half().cuda(), down_block_additional_residuals=res16, return_dict=False)[0]
    torch.cuda.synchronize()
    return {"psnr": psnr(out, g["out"]), "max_err": (out.float().cpu() - g["out"]).abs().max().item()}


def pipeline_vs_oracle(steps=3, Fr=2, hw=8, guidance=7.5):
    m, sd = get_model()
    pipe = VideoSwapPipeline(m, DDIMScheduler())
    lat = randn((1, 4, Fr, hw, hw), 21)
    pos = randn((1, 16, 77, 768), 22).half()
    neg = randn((1, 16, 77, 768), 23).half()
    # run only `steps` iterations of the 50-step schedule on both sides
    sched = O.DDIM()
    ts = sched.timesteps(50)[:steps]
    ref = lat.half().float()
    ehs2 = torch.cat([neg, pos]).float()
    nat = lat.half().cuda()
    from videoswap_b200 import ops
    pipe.scheduler.set_timesteps(50)
    for t in ts:
        with torch.no_grad():
            ref = O.denoise_step(sd, O.OracleConfig(), sched, ref, t, 50, ehs2, guidance)
        eps = m(torch.cat([nat] * 2), t, torch.cat([neg, pos]).cuda(), return_dict=False)[0]
        a_t, a_p = pipe.scheduler.alphas(t)
        nat = ops.cfg_ddim_step(eps, nat, guidance, a_t, a_p)
    torch.cuda.synchronize()
    return {"psnr": psnr(nat, ref), "max_err": (nat.float().cpu() - ref).abs().max().item()}


def _conditions(Fr, img, P=24, seed=51):
    """Synthetic TAP conditions (SURVEY 8d C3): tracks U[0, img) with some invisible, point embeddings N(0,1)."""
    g = torch.Generator().manual_seed(seed)
    tracks = torch.rand((Fr, P, 2), generator=g) * img
    tracks[0, 0] = -1.0
    tracks[Fr - 1, P - 1, 1] = -1.0
    emb = torch.randn((P, 1280), generator=g)
    return {"pred_tracks": tracks[None], "img_size": (img, img), "point_embedding": emb[None], "index_list": list(range(P - 1))}


def pipeline_call_vs_oracle(iters=3, Fr=2, hw=16, guidance=7.5, t2i_scale=4.0, t2i_end=0.0):
    """VideoSwapPipeline.__call__ (conditions -> adapter, residual window, CFG, DDIM, final rearrange) vs the oracle's
    restatement of pipeline_videoswap.py:525-610.  `t2i_end` = 0 closes the adapter window after iteration 0; the strong
    t2i scale makes a wrongly open (or never opened) window cost > 15 dB against the oracle."""
    m, sd = get_model()
    ad = SparsePointAdapter(init="empty")
    asd = seeded_state_dict(adapter_param_shapes(), seed=5)
    ad.load_state_dict(asd)
    ad = ad.half().cuda()
    pipe = VideoSwapPipeline(m, DDIMScheduler(), adapter=ad)
    cond = _conditions(Fr, hw * 8)
    lat = randn((1, 4, Fr, hw, hw), 21).half()
    pos, neg = randn((1, 16, 77, 768), 22).half(), randn((1, 16, 77, 768), 23).half()
    out = pipe(pos.cuda(), lat.cuda(), negative_prompt_embeds=neg.cuda(), conditions=cond, num_inference_steps=50,
               guidance_scale=guidance, t2i_guidance_scale=t2i_scale, t2i_start=0.0, t2i_end=t2i_end, max_iters=iters).videos
    torch.cuda.synchronize()
    # oracle: the reference's fp16 adapter arithmetic, then the fp32 loop on the fp16-rounded maps
    asd16 = {k: v.half() for k, v in asd.items()}
    maps = O.adapter_forward(asd16, cond["pred_tracks"][0].half(), cond["img_size"], cond["point_embedding"][0].half(),
                             index_list=cond["index_list"])
    state = [(mm * t2i_scale).float() for mm in maps]
    with torch.no_grad():
        ref = O.denoise_loop(sd, O.OracleConfig(), lat.float(), pos.float(), neg.float(), 50, guidance, state, 0.0, t2i_end,
                             max_iters=iters)
        ref_no_window = O.denoise_loop(sd, O.OracleConfig(), lat.float(), pos.float(), neg.float(), 50, guidance, state, 0.0, 1.0,
                                       max_iters=iters)
        ref_never = O.denoise_loop(sd, O.OracleConfig(), lat.float(), pos.float(), neg.float(), 50, guidance, None, 0.0, 1.0,
                                   max_iters=iters)
    return {"psnr": psnr(out, ref), "shape": tuple(out.shape), "ref_shape": tuple(ref.shape),
            "psnr_if_window_ignored": psnr(out, ref_no_window), "psnr_if_never_applied": psnr(out, ref_never)}


def invert_vs_oracle(iters=3, Fr=2, hw=8, convention="0.19.3"):
    from videoswap_b200 import DDIMInverseScheduler
    m, sd = get_model()
    pipe = VideoSwapPipeline(m, DDIMScheduler(), inverse_scheduler=DDIMInverseScheduler(convention=convention))
    lat = randn((1, 4, Fr, hw, hw), 61).half()
    emb = randn((1, 77, 768), 62).half()
    out = pipe.invert(emb.cuda(), lat.cuda(), num_inference_steps=50, max_iters=iters).latents
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = O.invert_loop(sd, O.OracleConfig(), lat.float(), emb.float(), 50, convention, max_iters=iters)
    return {"psnr": psnr(out, ref), "max_err": (out.float().cpu() - ref).abs().max().item()}


def adapter_fp16_vs_golden():
    """Product default (coord_fp16=True, the reference's fp16 inference arithmetic) vs the fixture the reference's own
    SparsePointAdapter produced in half precision."""
    from oracle.make_golden import adapter_fp16_inputs, densify
    g = torch.load(os.path.join(GOLD, "adapter_fp16.pt"))
    ref = densify(g["maps_sparse"])
    ad = SparsePointAdapter(init="empty")
    ad.load_state_dict(seeded_state_dict(adapter_param_shapes(), seed=5))
    ad = ad.half().cuda()
    tracks, emb, size, index_list = adapter_fp16_inputs()
    maps = ad(tracks.cuda(), size, emb.half().cuda(), index_list=index_list, coord_fp16=True, as_nchw=True)
    torch.cuda.synchronize()
    errs = [(m.float().cpu() - r.float()).abs().max().item() for m, r in zip(maps, ref)]
    refs = [r.float().abs().max().item() for r in ref]
    # the support (which cells a point touches) must be identical: that is what the fp16 coordinate quantisation decides
    same_support = [bool(((m.float().cpu() != 0).any(1) == (r != 0).any(1)).all()) for m, r in zip(maps, ref)]
    return {"errs": errs, "refs": refs, "same_support": same_support}


def adapter_vs_golden():
    from oracle.make_golden import densify
    g = torch.load(os.path.join(GOLD, "adapter.pt"))
    ref = densify(g["maps_sparse"])
    ad = SparsePointAdapter(init="empty")
    ad.load_state_dict(seeded_state_dict(adapter_param_shapes(), seed=5))
    ad = ad.cuda()
    maps = ad(g["tracks"].cuda(), g["size"], g["emb"].cuda(), coord_fp16=False, as_nchw=True)
    torch.cuda.synchronize()
    errs = [(m.float().cpu() - r).abs().max().item() for m, r in zip(maps, ref)]
    refs = [r.abs().max().item() for r in ref]
    return {"errs": errs, "refs": refs}


def edlora_merge_vs_oracle(Fr=2, hw=8, alpha=0.6, rank=4):
    """formats.merge_edlora_into_unet on the NATIVE model (parameters on the GPU, re-packed lazily) vs the oracle run on
    independently merged weights; then restore_unet brings the parameters back bit for bit (the OUTPUT is compared in dB: the
    GroupNorm statistics use float atomics, so two forwards of the same weights agree to ~70 dB, not bit for bit)."""
    from videoswap_b200 import formats
    m, sd = get_model()
    g = torch.Generator().manual_seed(77)
    lora = {}
    for k, w in sd.items():
        dn = formats.lora_down_name(k)
        if dn == k or "motion_modules" in k or not any(s in k for s in ("down_blocks.0.", "mid_block.", "up_blocks.3.attentions.2.")):
            continue
        down, up = 0.1 * torch.randn((rank, w.shape[1]), generator=g), 0.1 * torch.randn((w.shape[0], rank), generator=g)
        if w.dim() == 4:
            down, up = down[:, :, None, None], up[:, :, None, None]
        lora[dn], lora[dn.replace("lora_down", "lora_up")] = down, up
    merged = dict(sd)
    for dn in [k for k in lora if "lora_down" in k]:
        k = dn.replace("lora_down.", "")
        d = lora[dn.replace("lora_down", "lora_up")].squeeze() @ lora[dn].squeeze()
        merged[k] = (sd[k] + alpha * d.reshape(sd[k].shape)).half().float()
    x, ehs = randn((1, 4, Fr, hw, hw), 2).half(), randn((1, 16, 77, 768), 3).half()
    before = m(x.cuda(), 981, ehs.cuda(), return_dict=False)[0].clone()
    saved = {k: p.detach().clone() for k, p in m.named_parameters() if k in {d.replace("lora_down.", "") for d in lora}}
    backup = formats.merge_edlora_into_unet(m, lora, alpha, strict=True)
    try:
        out = m(x.cuda(), 981, ehs.cuda(), return_dict=False)[0].clone()
        with torch.no_grad():
            ref = O.unet_forward(merged, O.OracleConfig(), x.float(), 981, ehs.float(), None)
    finally:
        formats.restore_unet(m, backup)
    after = m(x.cuda(), 981, ehs.cuda(), return_dict=False)[0]
    torch.cuda.synchronize()
    return {"pairs": len(lora) // 2, "touched": len(backup), "psnr": psnr(out, ref), "psnr_unmerged_vs_merged_ref": psnr(before, ref),
            "restored_params_bit_exact": all(torch.equal(p, saved[k]) for k, p in m.named_parameters() if k in saved) and len(saved) == len(backup),
            "psnr_restored_vs_before": psnr(after, before)}
