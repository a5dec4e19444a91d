"""Parity helpers for the attention controllers (SURVEY.md 8f-2): the native explicit-probability attention, the hook through
AnimateDiffUNet3DModel.forward against the oracle's hook, and the device-native controllers replayed against the fixtures
the reference's own AttentionStore / AttentionRefine / AttentionReplace / SpatialBlender produced (oracle/make_golden_p2p.py)."""
from __future__ import annotations

import os

import torch

from oracle import make_golden_p2p as G
from oracle import unet3d_oracle as O
from tests import attention_probes as A
from tests import unet_checks as U
from videoswap_b200 import ops, p2p

GOLD = os.path.join(os.path.dirname(__file__), "golden")
DEV = "cuda"


def explicit_attention_check(B=3, N=256, NK=None, C=1280, kv_div=1, seed=170):
    """probs = softmax(q k^T / sqrt(d)) to HBM, then O = P V (d = C / 8).  The probabilities element by element against
    the fp64 softmax and O against fp64 P V of the probabilities the kernel wrote, both with the bounds of
    tests/attention_probes.py ("probs" / "out": err = the worst err / bound); O also against fp32 torch."""
    g = torch.Generator().manual_seed(seed)
    NK = N if NK is None else NK
    q = torch.randn((B, N, C), generator=g).half().to(DEV)
    kv = torch.randn((B // kv_div, NK, 2 * C), generator=g).half().to(DEV)
    k, v = kv[..., :C], kv[..., C:]
    probs = ops.attention_probs(q, k, 8, kv_div=kv_div)
    out = ops.attention_apply_probs(probs, v, 8, kv_div=kv_div)
    torch.cuda.synchronize()
    d = C // 8
    qh = q.float().reshape(B, N, 8, d).transpose(1, 2)
    kh = k.float().repeat_interleave(kv_div, 0).reshape(B, NK, 8, d).transpose(1, 2)
    vh = v.float().repeat_interleave(kv_div, 0).reshape(B, NK, 8, d).transpose(1, 2)
    pr = (qh @ kh.transpose(-1, -2) * d ** -0.5).softmax(-1)
    ref = (pr @ vh).transpose(1, 2).reshape(B, N, C)
    vd = v.double().repeat_interleave(kv_div, 0).reshape(B, NK, 8, d).transpose(1, 2)
    pv = (probs.double() @ vd).transpose(1, 2).reshape(B, N, C)
    mag = (probs.double() @ vd.abs()).transpose(1, 2).reshape(B, N, C)
    return {"probs": A.compare(probs, A.ref_probs(q, k, 8, kv_div), rel=A.PROBS_REL),
            "out": A.compare(out, pv, rel=A.PV_REL, extra=A.pv_extra(NK) * mag),
            "row_sum_err": (probs.float().sum(-1) - 1).abs().max().item(),
            "out_err": (out.float() - ref).abs().max().item(), "out_ref": ref.abs().max().item()}


class _Recorder:
    """Oracle-side twin of p2p.AttentionStore's `forward` (device-agnostic): keeps what the hook saw."""

    def __init__(self, edit=None):
        self.maps, self.edit = [], edit

    def __call__(self, probs, is_cross, place):
        self.maps.append((place, is_cross, probs.detach().clone()))
        return self.edit(probs, is_cross, place) if self.edit else probs


def unet_hook_vs_oracle(Fr=2, hw=16, edit=False):
    """One UNet forward ([2,...] CFG batch) with a controller registered: the maps the native hook delivers and the epsilon
    (after an in-place edit of the conditional half when `edit`) vs the oracle's hook."""
    m, sd = U.get_model()
    x = U.randn((2, 4, Fr, hw, hw), 2).half()
    ehs = U.randn((2, 16, 77, 768), 3).half()

    def edit_fn(probs, is_cross, place):      # a controller that really changes the maps: flatten the cond half of cross maps
        if is_cross:
            h = probs.shape[0] // 2
            probs[h:] = 0.5 * probs[h:] + 0.5 / probs.shape[-1]
        return probs

    class Ctl(p2p.AttentionControl):
        def __init__(self):
            super().__init__()
            self.LOW_RESOURCE = True
            self.seen = []

        def forward(self, attn, is_cross, place):
            self.seen.append((place, is_cross, attn.detach().clone()))
            return edit_fn(attn, is_cross, place) if edit else attn
    ctl = Ctl()
    n = p2p.register_attention_control(m, ctl)
    try:
        out = m(x.cuda(), 981, ehs.cuda(), return_dict=False)[0]
        torch.cuda.synchronize()
    finally:
        p2p.register_attention_control(m, None)
    rec = _Recorder(edit_fn if edit else None)
    O.ATTN_HOOK = rec
    try:
        with torch.no_grad():
            ref = O.unet_forward(sd, O.OracleConfig(), x.float(), 981, ehs.float())
    finally:
        O.ATTN_HOOK = None
    assert len(ctl.seen) == len(rec.maps), (len(ctl.seen), len(rec.maps))
    worst = 1e9
    for (p1, c1, a), (p2_, c2, b) in zip(ctl.seen, rec.maps):
        assert (p1, c1) == (p2_, c2) and tuple(a.shape) == tuple(b.shape), ((p1, c1, a.shape), (p2_, c2, b.shape))
        worst = min(worst, U.psnr(a, b))
    return {"registered": n, "calls": len(ctl.seen), "min_map_psnr": worst, "eps_psnr": U.psnr(out, ref),
            "order": [(p_, c) for p_, c, _ in ctl.seen]}


def replay_vs_reference_fixture(kind="refine"):
    """The scenario of oracle/make_golden_p2p.py replayed on the GPU with the device-native controllers."""
    g = torch.load(os.path.join(GOLD, f"p2p_{kind}.pt"))
    c = g["controller"]
    store = p2p.AttentionStore()
    store.LOW_RESOURCE = True
    for step in range(G.N_STEPS):
        for li, (place, is_cross) in enumerate(G.LAYERS):
            store(G.synth_map(step, li, G.FRAMES, is_cross, 1).half().to(DEV), is_cross, place)
        store.step_callback(G.synth_latents(step, 1).half().to(DEV))

    def blender(alpha, se, choose):
        b = p2p.SpatialBlender(alpha, th=c["th"], NUM_DDIM_STEPS=G.N_STEPS, prompt_choose=choose)
        b.start_blend, b.end_blend = se
        return b
    common = dict(num_steps=G.N_STEPS, cross_replace_alpha=c["cross_replace_alpha"], self_replace_steps=0.0,
                  latent_blend=blender(c["latent_alpha_layers"], c["latent_start_end"], "both"), additional_attention_store=store,
                  attention_blend=blender(c["attn_alpha_layers"], c["attn_start_end"], "source"), image_height=G.IMG, image_width=G.IMG)
    ctl = p2p.AttentionRefine(c["mapper"], c["alphas"], **common) if kind == "refine" else p2p.AttentionReplace(c["mapper"], **common)
    ctl.num_self_replace = tuple(c["num_self_replace"])
    map_err, lat_err, mask_mismatch = 0.0, 0.0, 0
    for step in range(G.N_STEPS):
        for li, (place, is_cross) in enumerate(G.LAYERS):
            attn = G.synth_map(step, li, 2 * G.FRAMES, is_cross, 2).half().to(DEV)
            out = ctl(attn, is_cross, place)
            if li in g["edited"][step]:
                map_err = max(map_err, (out[G.FRAMES:].float().cpu() - g["edited"][step][li]).abs().max().item())
        x = ctl.step_callback(G.synth_latents(step, 2).half().to(DEV))
        lat_err = max(lat_err, (x.float().cpu() - g["latents"][step]).abs().max().item())
    torch.cuda.synchronize()
    masks = [m.float().cpu() for m in ctl.latent_blend.mask_list]
    for a, b in zip(masks, g["latent_masks"]):
        mask_mismatch += int((a != b).sum().item())
    return {"map_err": map_err, "latent_err": lat_err, "mask_mismatch": mask_mismatch, "mask_pixels": sum(m.numel() for m in masks),
            "n_masks": (len(masks), len(g["latent_masks"]))}


# ---------------------------------------------------------------------------------------------------- whole flow
class _RecordingBlender(p2p.SpatialBlender):
    """The product blender, remembering every mask it computed (in call order)."""

    def _mask(self, maps, target_h, target_w):
        m = super()._mask(maps, target_h, target_w)
        self.__dict__.setdefault("all_masks", []).append(m.float().cpu())
        return m


class _TorchBlender(p2p.SpatialBlender):
    """Checker-side restatement of SpatialBlender.get_mask / the blend in plain torch (spatial_blend.py:25-63,141-142), so the
    oracle loop below does not execute the CUDA blend kernels it is checking.  A mask is a THRESHOLDED quantity: a pixel
    within fp16 noise of the threshold may flip between the fp16 device maps and the fp32 oracle maps and would then send the
    two (chaotic) denoising trajectories apart.  So the checker counts its disagreements with the masks the product computed
    (`forced`, in call order) and continues with the product's mask: mask computation and everything downstream of it are
    checked separately."""
    forced = None
    mismatch = 0
    pixels = 0

    def _mask(self, maps, target_h, target_w):
        own = self._own_mask(maps, target_h, target_w)
        if self.forced is None:
            return own
        given = self.forced.pop(0).to(own)
        type(self).mismatch += int((own != given).sum())
        type(self).pixels += own.numel()
        return given

    def _own_mask(self, maps, target_h, target_w):
        import torch.nn.functional as F
        items = [m[None] if m.dim() == 4 else m for m in maps]
        p, frames, heads, r, words = items[0].shape
        res_h = int((r * (target_h / target_w)) ** 0.5)
        res_w = int(r / res_h)
        n_prompts = 1 if self.prompt_choose == "source" else p
        cat = torch.cat([it[:n_prompts].float().reshape(n_prompts, frames, heads, res_h, res_w, words).permute(0, 2, 1, 3, 4, 5)
                         for it in items], dim=1)                                    # p (layers heads) c h w words
        alpha = self.alpha_layers[:n_prompts].float().reshape(n_prompts, 1, 1, 1, 1, words)
        mm = (cat * alpha).sum(-1).mean(1)
        mm = F.max_pool2d(mm, (3, 3), (1, 1), padding=(1, 1))
        mask = F.interpolate(mm, size=(target_h, target_w))
        mask = mask / mask.max(-2, keepdims=True)[0].max(-1, keepdims=True)[0]
        mask = mask.gt(self.th[0])
        if self.prompt_choose == "both":
            mask = mask[:1] + mask
        return mask.float()

    def __call__(self, attention_store, step_in_store=None, target_h=None, target_w=None, x_t=None):
        if target_h is None and target_w is None and x_t is not None:
            target_h, target_w = x_t.shape[-2:]
        self.counter += 1
        mask = self._mask(attention_store["down_cross"][2:4] + attention_store["up_cross"][:3], target_h, target_w)
        self.mask_list.append(mask[0][:, None])
        if x_t is None:
            return mask
        if self.start_blend < self.counter < self.end_blend:
            x_t = x_t[:1] + mask[:, None] * (x_t - x_t[:1])
        return x_t


def _edit_controller(store, blender_cls, n_steps):
    """AttentionRefine with everything switched on for all steps: cross refine (a new word at position 3, the others mapped
    1:1), masked self-attention replacement and latent blend from the first callback on."""
    mapper = torch.arange(77)[None].clone()
    mapper[0, 3] = -1
    alphas = torch.ones(1, 77)
    alphas[0, 3] = 0.0
    words = torch.zeros(2, 77)
    words[:, 2] = 1.0
    words[1, 3] = 1.0

    def blender(choose, start, end):
        # threshold 0.92: with seeded random weights the normalised maps live in [0.85, 1] (median 0.92) -> ~half the pixels
        b = blender_cls(words, th=(0.92, 0.92), NUM_DDIM_STEPS=n_steps, prompt_choose=choose)
        b.start_blend, b.end_blend = start, end
        return b
    ctl = p2p.AttentionRefine(mapper, alphas, num_steps=n_steps, cross_replace_alpha=p2p.time_words_alpha(n_steps, 1.0),
                              self_replace_steps=1.0, latent_blend=blender("both", 0, 10 ** 6), additional_attention_store=store,
                              attention_blend=blender("source", 0, 10 ** 6), image_height=512, image_width=512)
    return ctl


def edit_flow_vs_oracle(n_steps=2, Fr=2, hw=64):
    """The `use_blend: true` loop of a shipped config, shortened to n_steps: DDIM inversion with an AttentionStore registered
    (no CFG), then the CFG editing loop with AttentionRefine + masked self-attention replacement + latent blend, through the
    product surface (pipe.invert / pipe.__call__ with `controller=`) at the shipped resolution (64x64 latents: only the
    16x16 / 8x8 levels are controlled and the blend reads up_cross[:3], all 16x16 -- at other input sizes the reference's own
    SpatialBlender concatenates maps of different resolutions and fails) against the same flow on the CPU oracle (oracle UNet
    with its attention hook, p2p's device-agnostic controller logic on CPU tensors -- itself pinned to the reference's
    classes by replay_vs_reference_fixture -- and the torch restatement of the blend above)."""
    from videoswap_b200 import DDIMInverseScheduler, DDIMScheduler, VideoSwapPipeline
    m, sd = U.get_model()
    lat0 = U.randn((1, 4, Fr, hw, hw), 91).half()
    src = U.randn((1, 16, 77, 768), 92).half()
    tgt = U.randn((1, 16, 77, 768), 93).half()
    neg = U.randn((1, 16, 77, 768), 94).half()
    # ---- native
    pipe = VideoSwapPipeline(m, DDIMScheduler(), inverse_scheduler=DDIMInverseScheduler())
    store = p2p.AttentionStore()
    store.LOW_RESOURCE = True
    p2p.register_attention_control(pipe, store)
    try:
        inv = pipe.invert(src.cuda(), lat0.cuda(), num_inference_steps=50, controller=store, max_iters=n_steps).latents
        ctl = _edit_controller(store, _RecordingBlender, n_steps)
        p2p.register_attention_control(pipe, ctl)
        out = pipe(tgt.cuda(), inv, negative_prompt_embeds=neg.cuda(), num_inference_steps=50, guidance_scale=7.5, controller=ctl,
                   max_iters=n_steps).videos
        torch.cuda.synchronize()
    finally:
        p2p.register_attention_control(pipe, None)
    # ---- oracle
    ostore = p2p.AttentionStore()
    ostore.LOW_RESOURCE = True
    sched = O.DDIM()
    x = lat0.float()
    with torch.no_grad():
        O.ATTN_HOOK = ostore
        try:
            for i, t in enumerate(sched.inverse_timesteps(50)[:n_steps]):
                x = sched.inverse_step(O.unet_forward(sd, O.OracleConfig(), x, t, src.float()), t, x, 50)
                x = ostore.step_callback(x)
            oinv = x
            octl = _edit_controller(ostore, _TorchBlender, n_steps)
            # the two blenders of the native controller were called in this order: attention blend per controlled self-attention
            # layer, latent blend once per step -- the oracle's blenders are called in the same order
            octl.attention_blend.forced = list(ctl.attention_blend.all_masks)
            octl.latent_blend.forced = list(ctl.latent_blend.all_masks)
            _TorchBlender.mismatch = _TorchBlender.pixels = 0
            O.ATTN_HOOK = octl
            ehs2 = torch.cat([neg, tgt]).float()
            for i, t in enumerate(sched.timesteps(50)[:n_steps]):
                x = O.denoise_step(sd, O.OracleConfig(), sched, x, t, 50, ehs2, 7.5)
                x = octl.step_callback(x)
        finally:
            O.ATTN_HOOK = None
    ref = x.permute(0, 2, 1, 3, 4).reshape(Fr, 4, hw, hw)
    fill = torch.stack([mm.float().cpu() for mm in ctl.latent_blend.mask_list]).mean().item()
    return {"inversion_psnr": U.psnr(inv, oinv), "edit_psnr": U.psnr(out, ref), "stored_maps": sum(len(v) for v in store.attention_store.values()),
            "mask_mismatch": _TorchBlender.mismatch, "mask_pixels": _TorchBlender.pixels, "mask_fill": fill,
            "masks_checked": (len(ctl.attention_blend.all_masks), len(ctl.latent_blend.all_masks)),
            "unused_forced": (len(octl.attention_blend.forced), len(octl.latent_blend.forced)), "steps": (store.cur_step, ctl.cur_step)}
