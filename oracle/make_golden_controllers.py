"""TEST INFRASTRUCTURE ONLY.  Golden tensors for the prompt-driven controller construction (`p2p.make_controller`), produced by
the REFERENCE's own `attention_util.make_controller` (with its ptp_utils / seq_aligner / spatial_blend), imported unmodified
from the reference checkout (oracle/ref_loader.py), over the prompt table below.  Every row's reference controller goes
through `p2p.from_reference`, and the fixture keeps the attributes of that native twin -- the values a controller built from
the prompts natively must equal.

The table covers refinement with inserted and deleted words, equal-length swaps (replacement, including words that the
tokenizer splits into different numbers of tokens), multi-word and repeated blend words, ED-LoRA concept prompts (blend
words and per-word steps looked up as the layer-0 concept tokens), a `replace_other` prompt, float / pair / dict
cross_replace_steps, float and pair self_replace_steps, and rows without blending.  The tokenizer is
oracle/chunk_tokenizer.py, which splits words longer than four characters.  REFUSED lists the calls the reference rejects.

    VIDEOSWAP_REFERENCE=<checkout> python -m oracle.make_golden_controllers        -> tests/golden/controllers.pt"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "controllers.pt")


def R(name, src, tgt, replace=False, cross=0.5, self_=0.5, words=None, th=(0.3, 0.3), steps=50, hw=(512, 512),
      concepts=(), blend_latents=True, blend_self=True):
    return dict(name=name, prompts=[src, tgt], is_replace=replace, cross=cross, self_=self_, words=words, th=th, steps=steps,
                hw=hw, concepts=tuple(concepts), blend_latents=blend_latents, blend_self=blend_self)


ROWS = [
    R("refine_insert", "a cat walking on the grass", "a fluffy kitten walking on the grass", cross=0.2,
      words=[["cat"], ["fluffy", "kitten"]]),
    R("refine_delete", "a silver jeep driving down a curvy road in the countryside",
      "a car driving down a curvy road in the countryside", self_=(0.2, 0.7), words=[["silver", "jeep"], ["car"]],
      th=(0.1, 0.1), hw=(448, 768)),
    R("refine_edlora", "a kitten playing with a ball of yarn", "a <catA1> <catA2> playing with a ball of yarn",
      cross={"default_": (0.1, 0.6), "<catA1>": 0.3}, words=[["kitten"], ["<catA1>", "<catA2>"]], th=(0.2, 0.2), steps=4,
      hw=(256, 256), concepts=("<catA1>", "<catA2>")),
    R("refine_insert_split_words", "a kitten playing with a ball of yarn", "a small puppy playing with a ball of yarn",
      self_=(0.0, 0.5), words=[["kitten"], ["small", "puppy"]], steps=4, hw=(256, 256)),
    R("refine_replace_other", "a man walking on the beach at sunset",
      "a <hermione1> <hermione2> walking on the snowy mountain at sunset", cross=0.5, self_=0.3,
      words=[["man"], ["<hermione1>", "<hermione2>"]], concepts=("<hermione1>", "<hermione2>")),
    R("refine_dict_no_default", "a brown horse running across a meadow", "a white unicorn running across a meadow",
      cross={"unicorn": (0.2, 0.9), "missing": 0.5}, self_=0.3, words=[["brown", "horse"], ["white", "unicorn"]],
      hw=(448, 768)),
    R("refine_repeated_word", "a cat chasing another cat", "a tiger chasing another tiger", cross=(0.1, 0.4), self_=0.2,
      words=[["cat"], ["tiger"]], steps=20),
    R("refine_latent_blend_only", "a red sports car on a bridge", "a blue pickup truck on a bridge", cross=0.0, self_=0.0,
      words=[["red", "sports", "car"], ["blue", "pickup", "truck"]], blend_self=False),
    R("refine_no_blend", "a dog sitting on a bench", "a corgi sitting on a wooden bench", cross=0.3, words=None),
    R("replace_swap", "a cat walking on the grass", "a dog walking on the grass", replace=True, words=[["cat"], ["dog"]]),
    R("replace_token_counts", "a cat sleeping on a red sofa", "a elephant sleeping on a green sofa", replace=True,
      cross=0.4, self_=(0.0, 0.5), words=[["cat"], ["elephant"]], hw=(448, 768)),
    R("replace_token_counts_back", "a elephant sleeping on a green sofa", "a cat sleeping on a red sofa", replace=True,
      cross={"default_": 0.4, "cat": (0.0, 0.2)}, words=[["elephant"], ["cat"]], steps=4, hw=(64, 64)),
    R("replace_edlora", "a cat sitting on a chair", "a <catA1> sitting on a chair", replace=True, cross=0.3, self_=0.0,
      words=[["cat"], ["<catA1>"]], concepts=("<catA1>",)),
    R("replace_no_blend", "a cat walking on the grass", "a fox walking on the grass", replace=True, words="None"),
]

# calls the reference rejects: (name, prompts, is_replace, exception type name)
REFUSED = [
    ("replace_word_counts_differ", ["a cat walking on the grass", "a fluffy kitten walking on the grass"], True, "ValueError"),
]


def concept_cfg(tokenizer, concepts):
    """What load_new_concept leaves behind for ED-LoRA concepts: 16 tokens `<name_i>` each, in the tokenizer and the cfg."""
    cfg = {}
    for c in concepts:
        names = [f"<{c}_{i}>" for i in range(16)]
        tokenizer.add_tokens(names)
        cfg[c] = {"concept_token_ids": [tokenizer.convert_tokens_to_ids(n) for n in names], "concept_token_names": names}
    return cfg


def tokenizer_for(row):
    from oracle.chunk_tokenizer import ChunkTokenizer
    tok = ChunkTokenizer()
    if row["concepts"]:
        tok.new_concept_cfg = concept_cfg(tok, row["concepts"])
    return tok


def controller_kwargs(row):
    return dict(is_replace_controller=row["is_replace"], cross_replace_steps=row["cross"], self_replace_steps=row["self_"],
                blend_words=row["words"], blend_th=row["th"], NUM_DDIM_STEPS=row["steps"], blend_latents=row["blend_latents"],
                blend_self_attention=row["blend_self"], image_height=row["hw"][0], image_width=row["hw"][1])


def native_attributes(ctl):
    """The attributes the fixture pins (tensors only), from a native controller."""
    out = {"mapper": ctl.mapper.cpu(), "cross_replace_alpha": ctl.cross_replace_alpha.cpu(),
           "num_self_replace": torch.tensor(ctl.num_self_replace), "image_hw": torch.tensor([ctl.image_height, ctl.image_width])}
    if hasattr(ctl, "alphas"):
        out["alphas"] = ctl.alphas.cpu()
    for tag, b in (("latent_blend", ctl.latent_blend), ("attention_blend", ctl.attention_blend)):
        if b is not None:
            out[tag] = {"alpha_layers": b.alpha_layers.cpu(), "start_end": torch.tensor([b.start_blend, b.end_blend]),
                        "th": torch.tensor(b.th, dtype=torch.float64), "choose_both": torch.tensor(b.prompt_choose == "both")}
    return out


def main():
    from oracle.ref_loader import load_reference
    load_reference()
    import importlib
    au = importlib.import_module("videoswap.utils.p2p_utils.attention_util")
    st = importlib.import_module("videoswap.utils.p2p_utils.attention_store")
    from videoswap_b200 import p2p
    fixture = {}
    for row in ROWS:
        tok = tokenizer_for(row)
        pieces = {}
        for p in row["prompts"]:
            for w in tok.tokenize(p):
                assert pieces.setdefault(tok.convert_tokens_to_ids(w), w) == w, f"hash collision in {row['name']}"
        kw = controller_kwargs(row)
        cross = kw["cross_replace_steps"]
        kw["cross_replace_steps"] = dict(cross) if isinstance(cross, dict) else cross     # the reference adds 'default_'
        ref = au.make_controller(tok, list(row["prompts"]), additional_attention_store=st.AttentionStore(), **kw)
        fixture[row["name"]] = native_attributes(p2p.from_reference(ref, p2p.AttentionStore(), row["steps"]))
        print(row["name"], tuple(ref.mapper.shape), "blend", ref.latent_blend is not None, ref.attention_blend is not None)
    for name, prompts, is_replace, exc in REFUSED:
        try:
            au.make_controller(tokenizer_for({"concepts": ()}), prompts, is_replace, 0.5, additional_attention_store=st.AttentionStore(),
                               NUM_DDIM_STEPS=50)
        except Exception as e:  # noqa: BLE001
            assert type(e).__name__ == exc, (name, e)
            print(name, "refused:", type(e).__name__)
        else:
            raise AssertionError(f"the reference accepted {name}")
    torch.save(fixture, OUT)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
