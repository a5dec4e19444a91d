"""`p2p.make_controller` against the reference's own make_controller (tests/golden/controllers.pt, written by
oracle/make_golden_controllers.py), and the host-side parts of `VideoSwapPipeline.validation`: prompt construction,
`lora_path` parsing, the `select_point` -> `index_list` mapping and the point drawing."""
import os

import pytest
import torch

from oracle import make_golden_controllers as M
from oracle.chunk_tokenizer import ChunkTokenizer
from videoswap_b200 import p2p
from videoswap_b200 import pipeline as P

GOLD = torch.load(os.path.join(os.path.dirname(__file__), "golden", "controllers.pt"), weights_only=True)


def _build(row, **extra):
    tok = M.tokenizer_for(row)
    return p2p.make_controller(tok, list(row["prompts"]), additional_attention_store=p2p.AttentionStore(), device="cpu",
                               **M.controller_kwargs(row), **extra)


def _assert_equal(got, want, where):
    assert set(got) == set(want), (where, sorted(got), sorted(want))
    for k, v in want.items():
        if isinstance(v, dict):
            _assert_equal(got[k], v, f"{where}.{k}")
        else:
            assert got[k].dtype == v.dtype and torch.equal(got[k], v), f"{where}.{k}"


@pytest.mark.parametrize("row", M.ROWS, ids=[r["name"] for r in M.ROWS])
def test_make_controller_equals_reference(row):
    ctl = _build(row)
    assert isinstance(ctl, p2p.AttentionReplace if row["is_replace"] else p2p.AttentionRefine)
    _assert_equal(M.native_attributes(ctl), GOLD[row["name"]], row["name"])


def test_fixture_covers_the_table():
    assert sorted(GOLD) == sorted(r["name"] for r in M.ROWS)
    refine = GOLD["refine_insert"]
    assert (refine["mapper"] == -1).any() and (refine["alphas"] == 0).any(), "an inserted word must map to -1"
    back = GOLD["replace_token_counts"]["mapper"][0]
    assert ((back > 0) & (back < 1)).any(), "a swap with different token counts must spread the source token"


def test_concept_cfg_given_explicitly_equals_tokenizer_attribute():
    row = next(r for r in M.ROWS if r["name"] == "refine_edlora")
    tok = M.tokenizer_for(row)
    cfg = tok.new_concept_cfg
    del tok.new_concept_cfg
    ctl = p2p.make_controller(tok, list(row["prompts"]), additional_attention_store=p2p.AttentionStore(), device="cpu",
                              new_concept_cfg=cfg, **M.controller_kwargs(row))
    _assert_equal(M.native_attributes(ctl), GOLD[row["name"]], row["name"])
    plain = p2p.make_controller(tok, list(row["prompts"]), additional_attention_store=p2p.AttentionStore(), device="cpu",
                                **M.controller_kwargs(row))
    # bound, each concept is one added token; as written, '<catA1>' is split into '<cat' 'A1>'
    assert ctl.latent_blend.alpha_layers[1].nonzero().flatten().tolist() == [2, 3]
    assert plain.latent_blend.alpha_layers[1].nonzero().flatten().tolist() == [2, 3, 4, 5]


def test_dict_cross_replace_steps_is_not_modified():
    row = next(r for r in M.ROWS if r["name"] == "refine_dict_no_default")
    steps = dict(row["cross"])
    _build(dict(row, cross=steps))
    assert steps == row["cross"]


@pytest.mark.parametrize("name,prompts,is_replace,exc", M.REFUSED, ids=[r[0] for r in M.REFUSED])
def test_refused_like_the_reference(name, prompts, is_replace, exc):
    import builtins
    with pytest.raises(getattr(builtins, exc), match="same length"):
        p2p.make_controller(ChunkTokenizer(), prompts, is_replace, 0.5, additional_attention_store=p2p.AttentionStore(),
                            NUM_DDIM_STEPS=50, device="cpu")


def test_native_controller_needs_steps_store_and_two_prompts():
    tok, pr = ChunkTokenizer(), ["a cat", "a dog"]
    with pytest.raises(ValueError, match="NUM_DDIM_STEPS"):
        p2p.make_controller(tok, pr, False, 0.5, additional_attention_store=p2p.AttentionStore(), device="cpu")
    with pytest.raises(ValueError, match="additional_attention_store"):
        p2p.make_controller(tok, pr, False, 0.5, NUM_DDIM_STEPS=4, device="cpu")
    with pytest.raises(ValueError, match="prompts"):
        p2p.make_controller(tok, pr + ["a fox"], False, 0.5, additional_attention_store=p2p.AttentionStore(),
                            NUM_DDIM_STEPS=4, device="cpu")


def test_word_inds_split_words_and_indices():
    tok = ChunkTokenizer()
    text = "a fluffy kitten walking on the grass"          # fluf|fy kitt|en walk|ing gras|s
    assert p2p.get_word_inds(text, "fluffy", tok) == [2, 3]
    assert p2p.get_word_inds(text, "kitten", tok) == [4, 5]
    assert p2p.get_word_inds(text, 2, tok) == [4, 5]
    assert p2p.get_word_inds(text, "walking", tok) == [6, 7]
    assert p2p.get_word_inds(text, "grass", tok) == [10, 11]
    assert p2p.get_word_inds(text, "dog", tok) == []
    assert p2p.get_word_inds("a cat chasing another cat", "cat", tok) == [2, 7]


# ---------------------------------------------------------------------------------------------------- validation, host side
def test_edit_prompts():
    assert P.edit_prompts("a cat walking on the grass", {"replace": "cat -> <catA1> <catA2>"}) == \
        ("cat", "<catA1> <catA2>", "a <catA1> <catA2> walking on the grass")
    # str.replace replaces every occurrence; replace_other works on the target prompt
    assert P.edit_prompts("a cat chasing a cat", {"replace": " cat->dog "})[2] == "a dog chasing a dog"
    src, tgt, prompt = P.edit_prompts("a man walking on the beach", {"replace": "man -> <h1> <h2>",
                                                                     "replace_other": "beach -> snowy mountain"})
    assert (src, tgt, prompt) == ("man", "<h1> <h2>", "a <h1> <h2> walking on the snowy mountain")
    # replace_other is checked against the target prompt: a word the first replacement removed is refused
    with pytest.raises(ValueError, match="replace_other"):
        P.edit_prompts("a man on a horse", {"replace": "horse -> bike", "replace_other": "horse -> camel"})
    with pytest.raises(ValueError, match="source prompt"):
        P.edit_prompts("a cat on the grass", {"replace": "dog -> fox"})


def test_parse_lora_path():
    assert P.parse_lora_path("models/x/edlora_model-latest.pth---0.7") == ("models/x/edlora_model-latest.pth", 0.7, True)
    assert P.parse_lora_path("models/lora.pth---1") == ("models/lora.pth", 1.0, False)
    with pytest.raises(ValueError, match="---"):
        P.parse_lora_path("models/lora.pth")


def test_select_index_list():
    cond = {"point_name2id": {"head": 0, "tail": 3, "left_ear": 5}}
    assert P.select_index_list(cond, ["tail", "head"]) == [3, 0]
    assert P.select_index_list(cond, None) is None and P.select_index_list(cond, []) is None
    with pytest.raises(KeyError):
        P.select_index_list(cond, ["nose"])


def test_draw_points_in_place_only_inside_discs():
    from PIL import Image
    import numpy as np
    frames = [Image.new("RGB", (64, 48), (10, 20, 30)) for _ in range(3)]
    tracks = torch.tensor([[[10.0, 10.0], [40.0, 20.0], [-1.0, 5.0]],
                           [[30.0, 30.0], [5.0, 40.0], [20.0, 20.0]]])        # 2 frames of tracks for 3 frames
    out = P.draw_points(frames, {"pred_tracks": tracks, "index_list": [0, 2]})
    assert len(out) == 2 and out[0] is frames[0], "drawn in place; frames without tracks are left out"
    a = np.asarray(out[0])
    changed = np.argwhere((a != (10, 20, 30)).any(-1))
    assert len(changed) and all((x - 10) ** 2 + (y - 10) ** 2 <= 36 for y, x in changed), "only point 0 is visible and selected"
    assert tuple(a[10, 10]) == (0, 255, 0)
    b = np.asarray(out[1])
    assert tuple(b[30, 30]) == (0, 255, 0) and tuple(b[20, 20]) == (0, 255, 0) and tuple(b[40, 5]) == (10, 20, 30)
    assert np.asarray(frames[2]).max() == 30
