"""CPU side of the CLIP text encoder: the fp32 oracle (tests/clip_oracle.py) against the fixture transformers wrote
(oracle/make_golden_text.py) and, where transformers is installed, against a live model; the host mirror's keys; the
ED-LoRA text helpers of formats.py against the reference's own functions; and the power of the GPU tests' comparators,
shown on torch emulations of the causal-attention and quick-GELU arithmetic with planted bugs."""
import math
import os

import pytest
import torch

from tests import attention_probes as A
from tests import clip_oracle as CO
from tests import clip_probes as CP
from videoswap_b200 import formats
from videoswap_b200.spec import CLIPTextConfig, clip_text_param_shapes
from videoswap_b200.text import SEED, check_config
from videoswap_b200.weights import seeded_state_dict

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "clip_text.pt")


@pytest.fixture(scope="module")
def fx():
    return torch.load(GOLDEN, weights_only=False)


def seeded_sd(fx):
    sd = seeded_state_dict(clip_text_param_shapes(), seed=fx["seed"])
    tok = sd["text_model.embeddings.token_embedding.weight"]
    sd["text_model.embeddings.token_embedding.weight"] = torch.cat([tok, fx["concept_rows"].float()])
    return sd


# ---------------------------------------------------------------------------------------------------- oracle
def _close_to_fp16_ref(got, ref16):
    """|got - transformers| <= 1e-4 max|ref|, seen through the fixture's one fp16 rounding of transformers' fp32 output
    (half an fp16 ulp: 2^-11 relative, 2^-25 absolute below the normal range)."""
    ref = ref16.float()
    return bool(((got - ref).abs() <= 1e-4 * ref.abs().max() + 2.0 ** -11 * ref.abs() + 2.0 ** -25).all())


def test_oracle_reproduces_transformers_fixture(fx):
    assert fx["seed"] == SEED
    with torch.no_grad():
        out, hidden = CO.text_model(seeded_sd(fx), fx["input_ids"])
    assert _close_to_fp16_ref(torch.cat([out[s, :k] for s, k in enumerate(fx["keep"])]), fx["last_hidden_state"])
    T = fx["tap_tokens"]
    for i, t in fx["hidden_states"].items():
        got = torch.stack([hidden[i][s, :T] for s in fx["tap_sequences"]])
        assert _close_to_fp16_ref(got, t), i


def test_oracle_matches_live_transformers():
    transformers = pytest.importorskip("transformers")
    cfg = transformers.CLIPTextConfig(vocab_size=1000, hidden_size=768, intermediate_size=3072, num_hidden_layers=2,
                                      num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu",
                                      attn_implementation="eager")
    torch.manual_seed(0)
    model = transformers.CLIPTextModel(cfg).eval()
    ids = torch.randint(0, 1000, (3, 77))
    with torch.no_grad():
        ref = model(ids, output_hidden_states=True)
        out, hidden = CO.text_model(model.state_dict(), ids, layers=2)
    assert (out - ref.last_hidden_state).abs().max() <= 1e-4 * ref.last_hidden_state.abs().max()
    for a, b in zip(hidden, ref.hidden_states):
        assert (a - b).abs().max() <= 1e-4 * b.abs().max()


# ---------------------------------------------------------------------------------------------------- host mirror
def test_host_keys_and_parameter_count(fx):
    shapes = clip_text_param_shapes()
    assert dict(shapes) == {k: tuple(v) for k, v in fx["keys"].items() if not k.endswith("position_ids")}
    assert len(shapes) == 196 and sum(math.prod(s) for s in shapes.values()) == 123_060_480


@pytest.mark.parametrize("field,value", [("hidden_act", "gelu"), ("hidden_size", 1024), ("num_attention_heads", 16),
                                         ("max_position_embeddings", 78)])
def test_other_configs_are_rejected(field, value):
    with pytest.raises(ValueError, match=field):
        check_config(CLIPTextConfig(**{field: value}))


class _Params:
    """The named_parameters / resize / get_input_embeddings surface of the native CLIPTextModel, on CPU tensors."""

    def __init__(self, sd):
        self.sd = {k: v.clone() for k, v in sd.items()}
        self.dirty = 0

    def named_parameters(self):
        return iter(self.sd.items())

    def mark_weights_dirty(self):
        self.dirty += 1

    def resize_token_embeddings(self, n):
        k = "text_model.embeddings.token_embedding.weight"
        old = self.sd[k]
        self.sd[k] = torch.cat([old, torch.zeros(n - old.shape[0], old.shape[1], dtype=old.dtype)])

    def get_input_embeddings(self):
        return type("E", (), {"weight": self.sd["text_model.embeddings.token_embedding.weight"]})()


@pytest.mark.parametrize("dtype", ["fp32", "fp16"])
def test_text_lora_merge_and_restore_match_reference(fx, dtype):
    from oracle.make_golden_text import small_te_state_dict
    sd = small_te_state_dict(torch.float32 if dtype == "fp32" else torch.float16)
    case = fx["merge"][dtype]
    m = _Params(sd)
    backup = formats.merge_edlora_into_text_encoder(m, case["lora"], fx["merge"]["alpha"])
    assert m.dirty == 1 and len(backup) == 12
    for k, v in case["merged"].items():
        assert torch.equal(m.sd[k], v), k
    tok = "text_model.embeddings.token_embedding.weight"
    m.sd[tok][-1] = 3.0                                   # a concept row written after the merge
    formats.restore_text_encoder(m, backup)
    for k, v in sd.items():
        if k != tok:
            assert torch.equal(m.sd[k], v), k
    assert bool((m.sd[tok][-1] == 3.0).all()), "restore must leave the token embedding alone"


def test_load_new_concept_matches_reference(fx):
    from tests.stub_tokenizer import StubTokenizer
    c = fx["concept"]
    te = _Params({"text_model.embeddings.token_embedding.weight": c["base_table"]})
    cfg = formats.load_new_concept(StubTokenizer(base_vocab=100), te, c["embedding"])
    assert cfg == c["cfg"]
    assert torch.equal(te.get_input_embeddings().weight, c["table"])


# ---------------------------------------------------------------------------------------------------- causal attention
LOG2E = 1.4426950408889634


def emulate_causal(mutation=None):
    """attn(qkv, n, L) with causal_attn_kernel's arithmetic: 80 padded keys (zero K / V), fp32 scores, the mask before
    the row maximum, p = exp2(s sc - m sc), fp32 l, fp16(p) V in fp32, times 1 / l, fp16 out."""
    def run(qkv, n, L):
        H, D, C = CP.HEADS, CP.D, CP.C
        x = qkv.float().reshape(n, L, 3, H, D)
        q, k, v = (torch.zeros(n, H, 80, D) for _ in range(3))
        q[:, :, :L], k[:, :, :L], v[:, :, :L] = (x[:, :, i].transpose(1, 2) for i in range(3))
        if mutation == "head_plus_1_k":
            k = k.roll(-1, 1)
        sc = torch.tensor(LOG2E, dtype=torch.float32) / (torch.tensor(768.0).sqrt() if mutation == "scale_768" else 8.0)
        s = q @ k.transpose(-1, -2)
        i, j = torch.arange(80)[:, None], torch.arange(80)[None, :]
        masked = (j > i) | (j >= L)
        if mutation == "diag_masked":
            masked = (j >= i) | (j >= L)
        elif mutation == "next_visible":
            masked = (j > i + 1) | (j >= L)
        elif mutation == "pad_unmasked":
            masked = (j > i) & (j < L)
        s = s.masked_fill(masked, -math.inf)
        m = s.amax(-1, keepdim=True)
        p = torch.exp2((s.double() * sc.double() - (m * sc).double()).float())
        l = p.sum(-1, keepdim=True)
        p16 = p.bfloat16().float() if mutation == "p_bf16" else p.half().float()
        o = (p16 @ v) * (1.0 / l)
        return o[:, :, :L].half().transpose(1, 2).reshape(n * L, C)
    return run


CAUSAL_CASES = {
    "L77": lambda a: CP.check_causal(a, 3, 77, seed=1, dev="cpu"),
    "L17": lambda a: CP.check_causal(a, 2, 17, seed=2, dev="cpu"),
    "L1": lambda a: CP.check_causal(a, 2, 1, seed=3, dev="cpu"),
    "L77_shift": lambda a: CP.check_causal(a, 2, 77, sigmas=(1.0,), shift=40.0, seed=4, dev="cpu"),
    "L77_sink": lambda a: CP.check_causal(a, 2, 77, sigmas=(1.0,), sink=12.0, seed=5, dev="cpu"),
    "L65_tail": lambda a: CP.check_causal(a, 2, 65, tail=True, seed=6, dev="cpu"),
}
CAUSAL_MUTATIONS = {
    "key_i_masked_for_query_i": ("diag_masked", "L77"),
    "key_i_plus_1_visible": ("next_visible", "L77"),
    "padding_keys_77_79_unmasked": ("pad_unmasked", "L65_tail"),
    "scale_1_over_sqrt_768": ("scale_768", "L77"),
    "head_h_reads_head_h_plus_1_k": ("head_plus_1_k", "L77"),
    "p_rounded_to_bf16": ("p_bf16", "L77"),
}


@pytest.mark.parametrize("name", sorted(CAUSAL_CASES))
def test_emulated_causal_attention_passes_with_margin(name):
    r = CAUSAL_CASES[name](emulate_causal())
    assert r["ok"] and r["err"] <= 0.5, r


@pytest.mark.parametrize("name", sorted(CAUSAL_MUTATIONS))
def test_planted_causal_attention_bug_is_rejected(name):
    mutation, case = CAUSAL_MUTATIONS[name]
    r = CAUSAL_CASES[case](emulate_causal(mutation))
    assert not r["ok"], r


# ---------------------------------------------------------------------------------------------------- quick-GELU
def emulate_qgelu(mutation=None):
    """The epilogue's arithmetic on v (fp32): v / (1 + 2^min(-1.702 log2(e) v, 64)), rounded to fp16."""
    def run(v):
        v = v.float()
        if mutation == "tanh_gelu":
            y = 0.5 * v * (1 + torch.tanh(math.sqrt(2 / math.pi) * (v + 0.044715 * v ** 3)))
        elif mutation == "unclamped_exponent":      # sigmoid as e^z / (1 + e^z): e^z overflows for v > 52
            e = torch.exp(1.702 * v)
            y = v * e / (1 + e)
        else:
            c = (1.7 if mutation == "c_1.7" else 1.702) * LOG2E
            t = (-c * v).clamp(max=20.0 if mutation == "exponent_clamped_at_20" else 64.0)
            y = v / (1 + torch.exp2(t))
        return y.half()
    return run


def test_emulated_quick_gelu_passes():
    v = CP.qgelu_inputs().float()
    r = CP.compare_qgelu(emulate_qgelu()(v), v)
    assert r["ok"], r


@pytest.mark.parametrize("mutation", ["c_1.7", "tanh_gelu", "unclamped_exponent", "exponent_clamped_at_20"])
def test_planted_quick_gelu_bug_is_rejected(mutation):
    v = CP.qgelu_inputs().float()
    r = CP.compare_qgelu(emulate_qgelu(mutation)(v), v)
    assert not r["ok"], (mutation, r)
