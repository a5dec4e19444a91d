"""TEST INFRASTRUCTURE ONLY.  Golden vectors for the CLIP text encoder (videoswap_b200/text.py) and the text half of ED-LoRA
(videoswap_b200/formats.py), written to tests/golden/clip_text.pt.  Runs on the CPU where transformers is installed:

  last_hidden_state / hidden_states   transformers' own CLIPTextModel (SD-1.5 config, attn_implementation="eager", fp32)
                                      with weights seeded_state_dict(clip_text_param_shapes(), SEED) -- regenerated from the
                                      seed by the tests, not stored -- for a short prompt, the empty prompt, a full 77-token
                                      sequence and one with concept ids >= 49408 after resize_token_embeddings(49408 + 16)
  merge_lora_into_weight(..., 'text_encoder')   utils/convert_edlora_to_diffusers.py:36-81 of the reference  } that module
  load_new_concept                              utils/convert_edlora_to_diffusers.py:4-33                      } imports only
                                      `copy`, so it is loaded as a file from the checkout oracle/ref_loader names
                                      (VIDEOSWAP_REFERENCE); load_new_concept runs on a small transformers model with the
                                      tests' stub tokenizer.
    VIDEOSWAP_REFERENCE=/path/to/VideoSwap python -m oracle.make_golden_text"""
import importlib.util
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "clip_text.pt")
SEED = 9                       # = videoswap_b200.text.SEED
# Rows kept of each sequence's outputs (the fixture stays small): the first 24 tokens of the short, empty and concept
# sequences (every real token, BOS to EOS, and the first paddings) and all 77 of the full one, which covers every position.
KEEP = [24, 24, 77, 24]
TAP_TOKENS = 24
CONCEPT_SEED = 21
RANK, ALPHA = 4, 0.7


def reference_module():
    from oracle import ref_loader
    path = os.path.join(ref_loader.REFERENCE_ROOT, "videoswap", "utils", "convert_edlora_to_diffusers.py")
    if not os.path.exists(path):
        raise RuntimeError("set VIDEOSWAP_REFERENCE to a checkout of showlab/VideoSwap")
    spec = importlib.util.spec_from_file_location("ref_convert_edlora", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def sequences(g):
    """ids [4, 77]: short prompt, empty prompt, a full 77-token sequence, one with the 16 concept ids >= 49408."""
    from tests.stub_tokenizer import BOS, EOS
    rows = []
    for body in (torch.randint(0, BOS, (10,), generator=g).tolist(), [], torch.randint(0, BOS, (75,), generator=g).tolist(),
                 torch.randint(0, BOS, (3,), generator=g).tolist() + list(range(49408, 49424)) + [320, 1125]):
        r = [BOS] + body + [EOS]
        rows.append(r + [EOS] * (77 - len(r)))
    return torch.tensor(rows)


def encoder_fixture():
    import transformers
    from transformers import CLIPTextConfig, CLIPTextModel
    from videoswap_b200.spec import clip_text_param_shapes
    from videoswap_b200.weights import seeded_state_dict
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                         max_position_embeddings=77, hidden_act="quick_gelu", layer_norm_eps=1e-5, projection_dim=768,
                         attn_implementation="eager")
    model = CLIPTextModel(cfg).eval()
    sd = seeded_state_dict(clip_text_param_shapes(), seed=SEED)
    model.load_state_dict(sd, strict=True)
    keys = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.resize_token_embeddings(49408 + 16)
    g = torch.Generator().manual_seed(CONCEPT_SEED)
    concept_rows = (0.02 * torch.randn(16, 768, generator=g)).half()        # fp16 values: the native table holds them exactly
    with torch.no_grad():
        model.get_input_embeddings().weight[49408:] = concept_rows.float()
        ids = sequences(g)
        out = model(ids, output_hidden_states=True)
    # stored in fp16 (the fp32 outputs rounded once): the tests allow for that rounding
    taps = {i: torch.stack([out.hidden_states[i][0, :TAP_TOKENS], out.hidden_states[i][3, :TAP_TOKENS]]).half()
            for i in (1, 6, 12)}
    last = torch.cat([out.last_hidden_state[s, :k] for s, k in enumerate(KEEP)]).half()
    return {"seed": SEED, "transformers_version": transformers.__version__, "input_ids": ids, "concept_rows": concept_rows,
            "keep": KEEP, "last_hidden_state": last, "tap_sequences": [0, 3], "tap_tokens": TAP_TOKENS, "hidden_states": taps,
            "keys": keys}


def small_te_state_dict(dtype, C=16, F=32):
    """Real key names of layers 0 and 11 (the six LoRA sites plus their biases and norms) at a small width."""
    g = torch.Generator().manual_seed(3)
    sd = {}
    for i in (0, 11):
        p = f"text_model.encoder.layers.{i}"
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[f"{p}.self_attn.{n}.weight"] = torch.randn(C, C, generator=g)
            sd[f"{p}.self_attn.{n}.bias"] = torch.randn(C, generator=g)
        sd[f"{p}.layer_norm1.weight"] = torch.randn(C, generator=g)
        sd[f"{p}.mlp.fc1.weight"] = torch.randn(F, C, generator=g)
        sd[f"{p}.mlp.fc1.bias"] = torch.randn(F, generator=g)
        sd[f"{p}.mlp.fc2.weight"] = torch.randn(C, F, generator=g)
    sd["text_model.embeddings.token_embedding.weight"] = torch.randn(40, C, generator=g)
    return {k: v.to(dtype) for k, v in sd.items()}


def lora_for(sd):
    g = torch.Generator().manual_seed(4)
    lora = {}
    for k, w in sd.items():
        for site in ("q_proj", "k_proj", "v_proj", "out_proj", "fc1", "fc2"):
            if k.endswith(f".{site}.weight"):
                base = k[:-len("weight")]
                lora[base + "lora_down.weight"] = 0.3 * torch.randn(RANK, w.shape[1], generator=g)
                lora[base + "lora_up.weight"] = 0.3 * torch.randn(w.shape[0], RANK, generator=g)
    return lora


def merge_fixture(ref):
    out = {"alpha": ALPHA}
    for name, dtype in (("fp32", torch.float32), ("fp16", torch.float16)):
        sd = small_te_state_dict(dtype)
        lora = lora_for(sd)
        merged = ref.merge_lora_into_weight(sd, lora, model_type="text_encoder", alpha=ALPHA)
        # the reference then load_state_dict()s the merged dict into parameters of the original dtype
        out[name] = {"lora": lora, "merged": {k: v.to(dtype) for k, v in merged.items()}}
    return out


def concept_fixture(ref):
    from types import SimpleNamespace

    from transformers import CLIPTextConfig, CLIPTextModel
    from tests.stub_tokenizer import StubTokenizer
    torch.manual_seed(5)
    te = CLIPTextModel(CLIPTextConfig(vocab_size=100, hidden_size=32, intermediate_size=64, num_hidden_layers=1,
                                      num_attention_heads=2, max_position_embeddings=77))
    g = torch.Generator().manual_seed(6)
    base = te.get_input_embeddings().weight.detach().clone()
    emb = {"<cat1>": torch.randn(16, 32, generator=g), "<dog2>": torch.randn(16, 32, generator=g)}
    pipe = SimpleNamespace(tokenizer=StubTokenizer(base_vocab=100), text_encoder=te)
    _, cfg = ref.load_new_concept(pipe, emb, enable_edlora=True)
    return {"base_table": base, "embedding": emb, "cfg": cfg, "table": te.get_input_embeddings().weight.detach().clone()}


def main():
    ref = reference_module()
    fx = encoder_fixture()
    fx["merge"] = merge_fixture(ref)
    fx["concept"] = concept_fixture(ref)
    torch.save(fx, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 2 ** 20:.2f} MB), transformers {fx['transformers_version']}")


if __name__ == "__main__":
    main()
