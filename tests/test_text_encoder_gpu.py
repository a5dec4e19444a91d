"""The CLIP text encoder on an H100: the causal-attention kernel and the quick-GELU epilogue per element against fp64
(tests/clip_probes.py), the embedding bit-exact against torch, the whole encoder against transformers' fixture and the
fp32 oracle, batch invariance, and the pipeline's prompt encoding (plain and ED-LoRA)."""
import os

import pytest
import torch

import videoswap_b200 as V
from tests import clip_oracle as CO
from tests import clip_probes as CP
from tests import unet_checks as U
from tests.stub_tokenizer import StubTokenizer
from videoswap_b200 import _lib, formats, ops
from videoswap_b200.spec import clip_text_param_shapes
from videoswap_b200.text import TOKEN_EMBEDDING

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "clip_text.pt")


def _launches():
    return _lib.lib().vs_launch_count()


# ---------------------------------------------------------------------------------------------------- causal attention
def _attn_into_nan_buffer(qkv, n, L):
    """The kernel's output as a view into a NaN-filled buffer (row stride 800 > 768): nothing outside it may be written."""
    buf = torch.full((n * L + 2, 800), float("nan"), dtype=torch.float16, device="cuda")
    view = buf[1:n * L + 1, 8:8 + CP.C]
    ops.causal_attention(qkv, n, L, CP.HEADS, out=view)
    outside = buf.clone()
    outside[1:n * L + 1, 8:8 + CP.C] = 0
    assert bool(torch.isnan(outside[0]).all() and torch.isnan(outside[-1]).all() and torch.isnan(outside[:, :8]).all()
                and torch.isnan(outside[:, 8 + CP.C:]).all()), "the kernel wrote outside its output"
    return view


@pytest.mark.parametrize("L", [77, 1, 2, 16, 17, 64, 65])
def test_causal_attention_probes(L):
    rs = [CP.check_causal(_attn_into_nan_buffer, 3, L, seed=L)]
    rs.append(CP.check_causal(_attn_into_nan_buffer, 2, L, sigmas=(1.0,), shift=40.0, seed=L + 100))
    rs.append(CP.check_causal(_attn_into_nan_buffer, 2, L, sigmas=(3.0,), shift=-40.0, seed=L + 200))
    rs.append(CP.check_causal(_attn_into_nan_buffer, 2, L, tail=True, seed=L + 300))
    if L >= 16:
        rs.append(CP.check_causal(_attn_into_nan_buffer, 2, L, sigmas=(1.0,), sink=12.0, seed=L + 400))
    r = CP.A.merge(*rs)
    print(f"\ncausal attention L {L}: worst err / bound {r['err']:.3g} ({r['what']})")
    assert r["ok"] and r["err"] <= 1.0, r


def test_causal_attention_rejects_bad_shapes():
    qkv = torch.zeros(78, 3 * CP.C, dtype=torch.float16, device="cuda")
    with pytest.raises(_lib.VSError, match="L <= 77"):
        ops.causal_attention(qkv, 1, 78, CP.HEADS)
    with pytest.raises(_lib.VSError, match="head dim"):
        ops.causal_attention(qkv[:77], 1, 77, 8)


# ---------------------------------------------------------------------------------------------------- quick-GELU GEMM
def _qgelu_problem(M=17 * 77, K=768, N=3072):
    """x [M, K] holding every probe value, one-hot W[n, n % K] = 1, bias b: out[m, n] = quick_gelu(fp32(x[m, n % K] + b[n]))."""
    vals = CP.qgelu_inputs()
    g = torch.Generator().manual_seed(1)
    x = vals[torch.arange(M * K) % len(vals)][torch.randperm(M * K, generator=g)].reshape(M, K)
    w = torch.zeros(N, K, dtype=torch.float16)
    w[torch.arange(N), torch.arange(N) % K] = 1
    b = torch.zeros(N)
    b[K:] = torch.randint(-16, 17, (N - K,), generator=g).float() / 16
    v32 = x.float()[:, torch.arange(N) % K] + b
    return x.cuda(), w.cuda(), b.cuda(), v32


@pytest.mark.parametrize("bn", [0, 128, 256])
def test_quick_gelu_epilogue_per_element_and_schedule_invariant(bn):
    x, w, b, v32 = _qgelu_problem()
    base = ops.gemm(x, w, bias=b, mode=ops.EPI_QUICK_GELU, force_bn=bn)
    r = CP.compare_qgelu(base.cpu(), v32)
    print(f"\nquick-GELU epilogue (BLOCK_N {bn or 'auto'}): worst err / bound {r['err']:.3g}")
    assert r["ok"], r
    try:
        for ctas in (1, 2, 3, 5, 8):
            ops.set_option("gemm_ctas", ctas)
            out = ops.gemm(x, w, bias=b, mode=ops.EPI_QUICK_GELU, force_bn=bn)
            assert torch.equal(out, base), f"gemm_ctas {ctas}"
    finally:
        ops.set_option("gemm_ctas", 0)


def test_quick_gelu_epilogue_rejects_other_arguments():
    x, w, b, _ = _qgelu_problem(M=128)
    with pytest.raises(_lib.VSError, match="quick-GELU"):
        ops.gemm(x, w, bias=b, mode=ops.EPI_QUICK_GELU, force_bn=160)
    with pytest.raises(_lib.VSError, match="quick-GELU"):
        ops.gemm(x, w, bias=b, residual=torch.zeros(128, 3072, dtype=torch.float16, device="cuda"), mode=ops.EPI_QUICK_GELU)


# ---------------------------------------------------------------------------------------------------- embedding
@pytest.fixture(scope="module")
def model():
    """Seeded full-size weights, resized to 49408 + 16 rows with the fixture's concept rows."""
    fx = torch.load(GOLDEN, weights_only=False)
    m = V.CLIPTextModel()
    m.resize_token_embeddings(49408 + 16)
    m.get_input_embeddings().weight[49408:] = fx["concept_rows"].cuda().half()
    return m, fx


def test_embedding_bit_exact(model):
    m, _ = model
    g = torch.Generator().manual_seed(3)
    for n, L in ((17, 77), (2, 5), (1, 1)):
        ids = torch.randint(0, 49424, (n, L), generator=g)
        tok = m.get_input_embeddings().weight
        pos = m.state_dict()["text_model.embeddings.position_embedding.weight"]
        out = ops.clip_embed(ids.int().cuda(), tok, pos)
        assert torch.equal(out.view(n, L, -1), tok[ids.cuda()] + pos[:L])


def test_out_of_range_id_raises_before_any_launch(model):
    m, _ = model
    for bad in (49424, -1):
        ids = torch.full((2, 77), 49407)
        ids[1, 5] = bad
        n0 = _launches()
        with pytest.raises(ValueError, match="outside the token embedding"):
            m(ids)
        assert _launches() == n0


# ---------------------------------------------------------------------------------------------------- whole encoder
def test_encoder_vs_transformers_fixture(model):
    m, fx = model
    out = m(fx["input_ids"], output_hidden_states=True)
    assert out.last_hidden_state.dtype == torch.float16 and tuple(out[0].shape) == (4, 77, 768)
    assert len(out.hidden_states) == 13
    kept = torch.cat([out.last_hidden_state[s, :k] for s, k in enumerate(fx["keep"])])     # the rows the fixture keeps
    db = U.psnr(kept, fx["last_hidden_state"])
    T = fx["tap_tokens"]
    taps = {i: U.psnr(torch.stack([out.hidden_states[i][s, :T] for s in fx["tap_sequences"]]), t)
            for i, t in fx["hidden_states"].items()}
    print(f"\nCLIP text encoder vs transformers {fx['transformers_version']}: last_hidden_state {db:.1f} dB, taps "
          + ", ".join(f"{i}: {v:.1f} dB" for i, v in taps.items()))
    assert db >= 40.0 and min(taps.values()) >= 40.0


def _batch17(seed=7):
    g = torch.Generator().manual_seed(seed)
    rows = []
    for i in range(17):
        n = int(torch.randint(0, 76, (1,), generator=g))
        r = [49406] + torch.randint(0, 49406, (n,), generator=g).tolist() + [49407]
        rows.append(r + [49407] * (77 - len(r)))
    return torch.tensor(rows)


def test_encoder_vs_fp32_oracle_and_batch_invariance(model):
    m, _ = model
    ids = _batch17()
    out = m(ids).last_hidden_state
    sd = {k: v.float() for k, v in m.state_dict().items()}
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            ref, _ = CO.text_model(sd, ids.cuda())
            ref16, _ = CO.text_model(sd, ids[:, :16].cuda())
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    db = U.psnr(out, ref)
    db16 = U.psnr(m(ids[:, :16]).last_hidden_state, ref16)
    alone = [m(ids[i:i + 1]).last_hidden_state[0] for i in range(17)]
    worst = min(U.psnr(a, out[i]) for i, a in enumerate(alone))
    same = all(torch.equal(a, out[i]) for i, a in enumerate(alone))
    print(f"\nbatch 17 vs fp32 oracle: {db:.1f} dB (L = 16: {db16:.1f} dB); alone vs in the batch: "
          f"{'bit-identical' if same else f'{worst:.1f} dB'}")
    assert db >= 40.0 and db16 >= 40.0 and worst >= 70.0


def test_state_dict_round_trip_and_partial_load(model):
    m, _ = model
    sd = m.state_dict()
    assert set(sd) == set(clip_text_param_shapes()) and sd[TOKEN_EMBEDDING].shape[0] == 49424
    ids = _batch17(9)[:3]
    ref = m(ids).last_hidden_state.clone()
    m2 = V.CLIPTextModel(init="empty")
    r = m2.load_state_dict({**{k: v.float().cpu() for k, v in sd.items()}, "text_model.embeddings.position_ids": torch.arange(77)[None]})
    assert r.missing_keys == []
    assert torch.equal(m2(ids).last_hidden_state, ref)
    w = "text_model.encoder.layers.3.mlp.fc1.weight"
    m2.load_state_dict({w: torch.zeros(3072, 768)}, strict=False)
    assert not torch.equal(m2(ids).last_hidden_state, ref)
    m2.load_state_dict({w: sd[w]}, strict=False)
    assert torch.equal(m2(ids).last_hidden_state, ref)
    with pytest.raises(KeyError, match="unexpected"):
        m2.load_state_dict({"text_model.pooler.weight": torch.zeros(1)}, strict=False)
    with pytest.raises(KeyError, match="missing"):
        m2.load_state_dict({w: sd[w]})


# ---------------------------------------------------------------------------------------------------- pipeline
@pytest.fixture(scope="module")
def pipe(model):
    m, _ = model
    unet, _ = U.get_model()
    return V.VideoSwapPipeline(unet, V.DDIMScheduler(), text_encoder=m, tokenizer=StubTokenizer())


def test_encode_prompt_plain_and_edlora(pipe):
    p = pipe
    p.set_new_concept_cfg(None)
    e = p.encode_prompt("a cat on a sofa", "blurry")
    assert tuple(e.shape) == (2, 77, 768)
    assert torch.equal(e[0], p.text_encoder(p.tokenizer(["blurry"], max_length=77).input_ids)[0][0])
    e2 = p.encode_prompt("a cat on a sofa")                 # uncond "" by default
    assert torch.equal(e2[0], p.text_encoder(p.tokenizer([""], max_length=77).input_ids)[0][0])
    assert tuple(p.encode_prompt("a cat", do_classifier_free_guidance=False).shape) == (1, 77, 768)

    te = p.text_encoder
    g = torch.Generator().manual_seed(11)
    tok = StubTokenizer(base_vocab=te.get_input_embeddings().weight.shape[0])     # new ids follow the rows the model has
    p.tokenizer = tok
    rows_before = te.get_input_embeddings().weight.shape[0]
    cfg = formats.load_new_concept(tok, te, {"<cat1>": 0.02 * torch.randn(16, 768, generator=g)})
    assert te.get_input_embeddings().weight.shape[0] == len(tok) and len(tok) > rows_before
    p.set_new_concept_cfg(cfg)
    prompt = "a <cat1> on a sofa"
    e = p.encode_prompt(prompt, "blurry")
    assert tuple(e.shape) == (2, 16, 77, 768)
    assert all(torch.equal(e[0, i], e[0, 0]) for i in range(16)), "the negative must be repeated 16 times bitwise"
    bound = formats.bind_concept_prompt(prompt, cfg)
    for i in (0, 7, 15):
        one = te(tok([bound[i]], max_length=77).input_ids)[0][0]
        assert U.psnr(e[1, i], one) >= 70.0, i
    assert not torch.equal(e[1, 0], e[1, 15])
    p.set_new_concept_cfg(None)


def test_text_lora_merge_restore_bit_exact(pipe):
    te = pipe.text_encoder
    ids = _batch17(13)[:2]
    before = te(ids).last_hidden_state.clone()
    g = torch.Generator().manual_seed(12)
    lora = {}
    for i in (0, 5, 11):
        for site in ("self_attn.q_proj", "self_attn.v_proj", "self_attn.out_proj", "mlp.fc1", "mlp.fc2"):
            w = te.state_dict()[f"text_model.encoder.layers.{i}.{site}.weight"]
            lora[f"text_model.encoder.layers.{i}.{site}.lora_down.weight"] = 0.05 * torch.randn(4, w.shape[1], generator=g)
            lora[f"text_model.encoder.layers.{i}.{site}.lora_up.weight"] = 0.05 * torch.randn(w.shape[0], 4, generator=g)
    backup = formats.merge_edlora_into_text_encoder(te, lora, 0.7)
    assert len(backup) == 15
    assert U.psnr(te(ids).last_hidden_state, before) < 60.0, "the merge must change the output"
    formats.restore_text_encoder(te, backup)
    assert torch.equal(te(ids).last_hidden_state, before)


def test_pipeline_prompt_equals_embeddings(pipe):
    p = pipe
    p.set_new_concept_cfg(None)
    lat = U.randn((1, 4, 2, 8, 8), 21).half().cuda()
    e = p.encode_prompt("a dog running", "low quality")
    assert torch.equal(p.encode_prompt("a dog running", "low quality"), e)
    a = p(prompt="a dog running", negative_prompt="low quality", latents=lat, max_iters=2).videos
    b = p(e[1:], lat, negative_prompt_embeds=e[:1], max_iters=2).videos
    # the UNet's GroupNorm statistics are summed with atomics, so two denoising runs agree to the last bits only
    db = U.psnr(a, b)
    print(f"\npipe(prompt=...) vs pipe(prompt_embeds=encode_prompt(...)): {'bit-identical' if torch.equal(a, b) else f'{db:.1f} dB'}")
    assert db >= 60.0
    with pytest.raises(ValueError, match="exactly one"):
        p(e[1:], lat, prompt="a dog")
    with pytest.raises(ValueError, match="latents"):
        p(prompt="a dog")
    p.vae = V.AutoencoderKL()
    try:
        from PIL import Image
        g = torch.Generator().manual_seed(22)
        frames = [Image.fromarray(torch.randint(0, 256, (64, 64, 3), generator=g, dtype=torch.uint8).numpy(), "RGB")
                  for _ in range(2)]
        e1 = p.encode_prompt("a dog running", do_classifier_free_guidance=False, plain=True)
        x = p.invert(prompt="a dog running", video=frames, generator=torch.Generator("cuda").manual_seed(0), max_iters=2).latents
        y = p.invert(e1, video=frames, generator=torch.Generator("cuda").manual_seed(0), max_iters=2).latents
        # GroupNorm statistics (VAE encoder, UNet) are summed with atomics: two runs agree to the last bits only
        assert U.psnr(x, y) >= 60.0
        lat2 = p.prepare_image_latents(frames, torch.Generator("cuda").manual_seed(0))
        assert U.psnr(p.invert(prompt="a dog running", latents=lat2, max_iters=2).latents,
                      p.invert(e1, lat2, max_iters=2).latents) >= 60.0
    finally:
        p.vae = None
