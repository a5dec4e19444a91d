"""TEST INFRASTRUCTURE ONLY.  Golden vectors for the attention controllers (SURVEY.md 8f-2), produced by the REFERENCE's own
classes -- utils/p2p_utils/attention_store.AttentionStore, attention_util.make_controller -> AttentionRefine /
AttentionReplace, spatial_blend.SpatialBlender -- imported unmodified from the reference checkout (through oracle/diffusers_stub;
a whitespace tokenizer stands in for CLIP's, it only drives the reference's own word alignment).

Scenario (everything seeded): an inversion pass stores the maps / latents of N steps (LOW_RESOURCE, batch = F frames), then an
editing pass under CFG feeds [uncond | cond] maps through the edit controller layer by layer (the UNet's call order: down
2 x (self, cross), mid (self, cross), up 3 x (self, cross) -- the layers below 32^2 queries at 512^2) and calls
`step_callback` on the latents after every step.  Recorded: the controller's tensors, every edited cond-half map of two
layers per step, the blend masks and the latents after each callback.   python -m oracle.make_golden_p2p"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden")

N_STEPS, FRAMES, HEADS, RES, WORDS, IMG, LAT = 6, 2, 2, 16, 77, 32, 8
LAYERS = [("down", False), ("down", True), ("down", False), ("down", True), ("mid", False), ("mid", True),
          ("up", False), ("up", True), ("up", False), ("up", True), ("up", False), ("up", True)]
SRC, TGT = "a cat walking on the grass", "a dog walking on the grass"
BLEND_WORDS = [["cat"], ["dog"]]


class WordTokenizer:
    """encode: [bos] + one id per whitespace word + [eos]; decode: the words back."""

    def __init__(self):
        self.vocab = {"<bos>": 0, "<eos>": 1}

    def encode(self, text):
        ids = [0]
        for w in text.split(" "):
            ids.append(self.vocab.setdefault(w, len(self.vocab)))
        return ids + [1]

    def decode(self, ids):
        inv = {v: k for k, v in self.vocab.items()}
        return " ".join(inv[int(i)] for i in ids)


def synth_map(step, layer, batch, is_cross, phase):
    """Deterministic probability maps [batch, heads, RES, t] (rows sum to 1), fp16-representable values."""
    g = torch.Generator().manual_seed(1000 * phase + 37 * step + layer)
    t = WORDS if is_cross else RES
    logits = 2.0 * torch.randn((batch, HEADS, RES, t), generator=g)
    return logits.softmax(-1).half().float()


def synth_latents(step, phase):
    g = torch.Generator().manual_seed(5000 * phase + step)
    return torch.randn((1, 4, FRAMES, LAT, LAT), generator=g).half().float()


def load_reference_p2p():
    from oracle.ref_loader import load_reference, REFERENCE_ROOT  # noqa: F401  (puts the stubs + reference on sys.path)
    load_reference()
    import importlib
    au = importlib.import_module("videoswap.utils.p2p_utils.attention_util")
    st = importlib.import_module("videoswap.utils.p2p_utils.attention_store")
    return au, st


def run(kind):
    au, st = load_reference_p2p()
    tok = WordTokenizer()
    store = st.AttentionStore()
    store.LOW_RESOURCE = True                                     # inversion: no CFG (pipeline_videoswap.py:241)
    for step in range(N_STEPS):
        for li, (place, is_cross) in enumerate(LAYERS):
            store(synth_map(step, li, FRAMES, is_cross, 1), is_cross, place)
        store.step_callback(synth_latents(step, 1))
    ctl = au.make_controller(tok, [SRC, TGT], is_replace_controller=(kind == "replace"), cross_replace_steps=0.5,
                             self_replace_steps=0.5, blend_words=BLEND_WORDS, additional_attention_store=store,
                             blend_th=(0.3, 0.3), NUM_DDIM_STEPS=N_STEPS, blend_latents=True, blend_self_attention=True,
                             image_height=IMG, image_width=IMG)
    rec = {"edited": [], "latents": [], "latent_masks": None}
    for step in range(N_STEPS):
        outs = {}
        for li, (place, is_cross) in enumerate(LAYERS):
            attn = synth_map(step, li, 2 * FRAMES, is_cross, 2)    # [uncond | cond]
            out = ctl(attn, is_cross, place)
            if li in (1, 7, 10):                                  # down cross #0, up cross #0, up self #2
                outs[li] = out[FRAMES:].clone()
        rec["edited"].append(outs)
        x = ctl.step_callback(synth_latents(step, 2))
        rec["latents"].append(x.clone())
    rec["latent_masks"] = [m.clone() for m in ctl.latent_blend.mask_list]
    rec["controller"] = {
        "kind": kind, "mapper": ctl.mapper.cpu(), "alphas": getattr(ctl, "alphas", torch.zeros(0)).cpu(),
        "cross_replace_alpha": ctl.cross_replace_alpha.cpu(), "num_self_replace": tuple(ctl.num_self_replace),
        "latent_alpha_layers": ctl.latent_blend.alpha_layers.cpu(), "attn_alpha_layers": ctl.attention_blend.alpha_layers.cpu(),
        "latent_start_end": (ctl.latent_blend.start_blend, ctl.latent_blend.end_blend),
        "attn_start_end": (ctl.attention_blend.start_blend, ctl.attention_blend.end_blend), "th": tuple(ctl.latent_blend.th)}
    torch.save(rec, os.path.join(OUT, f"p2p_{kind}.pt"))
    print(kind, "mapper", tuple(ctl.mapper.shape), "edited maps", len(rec["edited"]) * 3, "mask sum",
          [float(m.sum()) for m in rec["latent_masks"]], "latents", float(torch.stack(rec["latents"]).abs().sum()))


if __name__ == "__main__":
    for k in sys.argv[1:] or ["refine", "replace"]:
        run(k)
